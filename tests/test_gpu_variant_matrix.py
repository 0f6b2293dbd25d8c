"""Every shipped kernel instantiation, launched and compared with the oracle.

The cases are generated from the kernel ledger of the built library (tests/kernel_ledger.py), not chosen by hand: each
ledger key is mapped to a driver that selects exactly that instantiation --

  FIN / FOUT  source format (and content) / destination dtype and format
  TMA         a pitch-aligned source (`to_image`) vs a tight odd-width tensor (or a CUDA array)
  TW          EASU: renderScale 0.75 (60-column tile) vs 0.9 (72); the fused kernel: anisotropic output sizes, as
              its 72-column tile only fits its shared-memory budget when the source tile is short
  PAIRED      PostProcessor with a UNORM output (EASU writes the outside-radius groups, RCAS skips them)
  OPQ         a BGRX8 source
  ANYIO       an ArrayImage source and/or destination (TMA=1: a pitched source with an array destination)
  S           MSAA sources; repitch / expand: the host-memory entry and an R32G32B32_FLOAT source

-- and torch.profiler (CUDA activity) records which kernels each case actually launched: the set of normalised keys a
case launches must equal the set it claims, and the union over the module must cover the ledger minus EXCLUDED.

Every result is compared with the CPU oracle (oracle/pyoracle.py; oracle/frontend.py for the resolve), never with
another GPU path: strict math bit for bit (float outputs too); fast math per pass on identical inputs <= 1 LSB (UNORM8),
<= 1 code (UNORM10), <= 1e-3 * max(1, |ref|) (FP16 / FP32); fast math composed (paired context path, fused kernel)
<= 4 LSB with < 1e-4 of channel values beyond 1 LSB (test_gpu_fsr_parity.py).  97x61 sources give partial tiles in
both dimensions; the radius with an off-centre projection centre puts filtered, bilinear and copy groups in one image."""
import time
from collections import defaultdict

import numpy as np
import pytest

from tests import kernel_ledger as kl

pytestmark = pytest.mark.gpu

W, H = 97, 61
PROJ = (0.42, 0.47, 0.58, 0.53)
RADIUS = 0.4
SHARP = 0.8
FUSED_72 = (108, 96)  # out->in 0.90 wide, 0.64 tall: the 72-column tile with and without the TMA landing zone
PAIRED_RCAS_PLAIN = "the paired RCAS reads the context's own 256-byte-pitched intermediate, which always has a tensor " \
                    "map; its plain-load build only runs if the driver cannot encode one, which no API input causes"
EXCLUDED = {
    ("strict", "rcas_rcp_selftest_kernel", ()): "device self-test of RCAS's reciprocal (test_gpu_fsr_parity.py)",
    ("fast", "rcas_rcp_selftest_kernel", ()): "device self-test of RCAS's reciprocal (test_gpu_fsr_parity.py)",
    ("", "nis_div_selftest_kernel", ()): "device self-test of NIS's in-range division (test_gpu_nis_parity.py)",
}
for _m in kl.MODES:
    for _f in (kl.RGBA8, kl.RGB10A2):
        for _a in (0, 1):
            EXCLUDED[(_m, "rcas_kernel", (_f, _f, 0, 1, 0, _a))] = PAIRED_RCAS_PLAIN

BGRX8, RGB32F = 5, 6
STATE = {"t0": None, "launched": set(), "maxima": defaultdict(float), "ran": set()}


# ---- inputs ------------------------------------------------------------------------------------------------------
def _content(fmt, w, h, seed):
    """numpy (H, W, 4) source of API format fmt: natural UNORM content, floats spanning about [-0.1, 1.2]; the X byte
    of BGRX8 holds noise, which the kernels must read as alpha 1"""
    from openvr_fsr_b200 import synth
    if fmt == kl.RGB10A2:
        return synth.natural_rgb10a2(w, h, seed)
    px = synth.natural_rgba8(w, h, seed)
    if fmt in (kl.RGBA16F, kl.RGBA32F):
        return (px.astype(np.float32) / 200.0 - 0.1).astype(np.float16 if fmt == kl.RGBA16F else np.float32)
    if fmt == BGRX8:
        px[..., 3] = np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)
    return px


def _dtype(fmt):
    import torch
    return {kl.RGBA16F: torch.float16, kl.RGBA32F: torch.float32}.get(fmt, torch.uint8)


def _np_dtype(fmt):
    return {kl.RGBA16F: np.float16, kl.RGBA32F: np.float32}.get(fmt, np.uint8)


def _tag(fmt):
    """the format argument of the API calls (None: the tensor dtype says it)"""
    return fmt if fmt in (kl.BGRA8, kl.RGB10A2, BGRX8) else None


def _place(arr, fmt, where, dev):
    """'tma': pitch-aligned device image; 'tight': packed rows (odd width: no TMA); 'array': CUDA array"""
    import torch
    import openvr_fsr_b200 as ovr
    if where == "tma":
        return ovr.to_image(arr, dev)
    t = torch.from_numpy(arr).to(dev)
    if where == "tight":
        return t
    return ovr.ArrayImage(arr.shape[1], arr.shape[0], fmt).upload(t)


def _outputs(fmt, w, h, dev, kinds):
    import openvr_fsr_b200 as ovr
    return [ovr.ArrayImage(w, h, fmt) if k == "array" else ovr.alloc_image(w, h, _dtype(fmt), dev) for k in kinds]


def _host(d):
    import openvr_fsr_b200 as ovr
    return (d.download() if isinstance(d, ovr.ArrayImage) else d).cpu().numpy()


# ---- comparison --------------------------------------------------------------------------------------------------
def _units(a, fmt):
    """UNORM channel codes as int32 (RGB10A2: the four fields of the packed word)"""
    from openvr_fsr_b200 import synth
    return synth.unpack_rgb10a2(a) if fmt == kl.RGB10A2 else a.astype(np.int32)


def _check(got, want, fmt, mode, composed):
    """(None if within the bound else a description, the fast-math error in LSB / codes / relative units)"""
    if mode == "strict":
        if got.shape == want.shape and np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8)):
            return None, 0.0
        n = int((np.ascontiguousarray(got).view(np.uint8) != np.ascontiguousarray(want).view(np.uint8)).sum()) if got.shape == want.shape else -1
        return f"strict: {n} bytes differ", 0.0
    if fmt in (kl.RGBA16F, kl.RGBA32F):
        g, w = got.astype(np.float64), want.astype(np.float64)
        err = float(np.nanmax(np.abs(g - w) / np.maximum(1.0, np.abs(w)))) if np.isfinite(g).all() else float("inf")
        return (None if err <= 1e-3 else f"fast: relative error {err:.3g} > 1e-3"), err
    d = np.abs(_units(got, fmt) - _units(want, fmt))
    err = float(d.max())
    if composed:
        beyond = float((d > 1).mean())
        ok = err <= 4 and beyond < 1e-4
        return (None if ok else f"fast composed: max {err:.0f}, {beyond:.2e} beyond 1"), err
    return (None if err <= 1 else f"fast: max {err:.0f} > 1"), err


# ---- cases -------------------------------------------------------------------------------------------------------
class Case:
    """keys: the instantiations the case launches; run(dev) -> [(label, got, want, out format, composed)]"""

    def __init__(self, family, mode, keys, run, name):
        self.family, self.mode, self.keys, self.run, self.name = family, mode, frozenset(keys), run, name


def _mathmode(mode):
    import openvr_fsr_b200 as ovr
    return ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST


def _debug(args):
    return sum(args) % 3 == 0  # the debug tint on about a third of the cases


def _seed(key):
    return 1 + sum((i + 3) * a for i, a in enumerate(key[2])) + len(key[1])


def _stateless(key, content=None):
    """EASU / RCAS / NVScaler / NVSharpen / CAS / fused: one ovrfsr_dispatch_* call per I/O layout.  content(fmt, w, h,
    seed) -> source array (default: _content)"""
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    mode, kernel, args = key
    p = dict(zip(kl.PARAMS[kernel], args))
    fin, fout, tma, anyio = p["FIN"], p.get("FOUT"), p.get("TMA", 0), p.get("ANYIO", 0)
    sfmt = BGRX8 if (p.get("OPQ") or (fin == kl.BGRA8 and kernel in ("nis_scaler_kernel", "nis_sharpen_kernel", "cas_sharpen_kernel",
                                                                       "cas_scale_kernel") and fout == kl.RGBA16F)) else fin
    debug = _debug(args)
    mm = _mathmode(mode)
    # source placement and destinations: (source where, [destination kinds])
    if anyio:
        layouts = [("tma", ["array"])] if tma else [("array", ["pitched", "array"])]
    else:
        layouts = [("tma" if tma else "tight", ["pitched"])]
    ow, oh = W, H
    composed = False
    if kernel == "easu_kernel":
        ow, oh = ovr.output_size(W, H, 0.9 if p["TW"] == 72 else 0.75)
        uc = po.upscale_constants(0, True, W, H, ow, oh, proj=PROJ, radius=RADIUS)
        call = lambda s, d, sf, df: ovr.fsr_easu(s, d, uc.words(), mm, src_fmt=sf, dst_fmt=df)  # noqa: E731
        oracle = lambda src, df: po.easu(src, ow, oh, uc, out_dtype=_np_dtype(fout), src_fmt=sfmt, dst_fmt=df)  # noqa: E731
    elif kernel == "rcas_kernel":
        sc = po.sharpen_constants(0, True, W, H, proj=PROJ, radius=RADIUS, sharpness=SHARP, debug=debug)
        call = lambda s, d, sf, df: ovr.fsr_rcas(s, d, sc.words(), mm, src_fmt=sf, dst_fmt=df)  # noqa: E731
        oracle = lambda src, df: po.rcas(src, sc, out_dtype=_np_dtype(fout), src_fmt=sfmt, dst_fmt=df)  # noqa: E731
    elif kernel in ("nis_scaler_kernel", "nis_sharpen_kernel"):
        scaler = kernel == "nis_scaler_kernel"
        if scaler:
            ow, oh = ovr.output_size(W, H, 0.75)
        cfg, ok = po.nis_config(not scaler, 0, True, W, H, ow, oh, proj=PROJ, radius=RADIUS, sharpness=SHARP, debug=debug)
        assert ok
        fn = ovr.nis_scaler if scaler else ovr.nis_sharpen
        call = lambda s, d, sf, df: fn(s, d, bytes(cfg), mm, src_fmt=sf, dst_fmt=df)  # noqa: E731
        oracle = (lambda src, df: po.nis_scaler(src, ow, oh, cfg, out_dtype=_np_dtype(fout), src_fmt=sfmt, dst_fmt=df)) if scaler \
            else (lambda src, df: po.nis_sharpen(src, cfg, out_dtype=_np_dtype(fout), src_fmt=sfmt, dst_fmt=df))
    elif kernel in ("cas_sharpen_kernel", "cas_scale_kernel"):
        sharpen_only = kernel == "cas_sharpen_kernel"
        if not sharpen_only:
            ow, oh = ovr.output_size(W, H, 0.75)
            # no TMA variant: both placements run the one instantiation
            layouts = [("tma" if fin in kl.PACKED32 and mode == "fast" else "tight", ["pitched"])]
        kc = po.cas_setup(SHARP, 1.0, W, H, ow, oh)
        call = lambda s, d, sf, df: ovr.cas(s, d, kc.words(), sharpen_only, mm, src_fmt=sf, dst_fmt=df)  # noqa: E731
        oracle = lambda src, df: po.cas(src, ow, oh, kc, sharpen_only, out_dtype=_np_dtype(fout), src_fmt=sfmt, dst_fmt=df)  # noqa: E731
    elif kernel == "fsr_fused_kernel":
        fout = p["FOUT"]
        ow, oh = FUSED_72 if p["TW"] == 72 else ovr.output_size(W, H, 0.75)
        uc = po.upscale_constants(0, True, W, H, ow, oh, proj=PROJ, radius=RADIUS)
        sc = po.sharpen_constants(0, True, ow, oh, proj=PROJ, radius=RADIUS, sharpness=SHARP, debug=debug)
        call = lambda s, d, sf, df: ovr.fsr_fused(s, d, uc.words(), sc.words(), mm, src_fmt=sf, dst_fmt=df)  # noqa: E731

        def oracle(src, df):
            return po.rcas(po.easu(src, ow, oh, uc, src_fmt=sfmt, dst_fmt=df), sc, src_fmt=df, dst_fmt=df)
        composed = True
    else:
        raise AssertionError(key)

    def run(dev):
        src = (content or _content)(sfmt, W, H, _seed(key))
        want = oracle(src, _tag(fout))
        out = []
        for where, kinds in layouts:
            s = _place(src, sfmt, where, dev)
            for kind, d in zip(kinds, _outputs(fout, ow, oh, dev, kinds)):
                call(s, d, None if where == "array" else _tag(sfmt), None if kind == "array" else _tag(fout))
                out.append((f"{where}->{kind}", _host(d), want, fout, composed))
        return out
    return Case(kernel, mode, {key}, run, kl.describe(key))


def _paired(mode, fin, tw, tma, anyio, content=None):
    """the context path with a UNORM output: paired EASU + RCAS, both eyes (apply_pair / apply_pair_into)"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    scale = 0.9 if tw == 72 else 0.75
    unorm = kl.RGB10A2 if fin == kl.RGB10A2 else kl.RGBA8
    debug = _debug((fin, tw, tma, anyio))
    layered = anyio and not tma and fin in (kl.RGB10A2, kl.RGBA32F)
    keys = {(mode, "easu_kernel", (fin, unorm, tw, tma, 1, anyio)), (mode, "rcas_kernel", (unorm, unorm, 1, 1, 0, anyio))}

    def run(dev):
        ow, oh = ovr.output_size(W, H, scale)
        eyes = [(content or _content)(fin, W, H, 40 + fin + 2 * e) for e in (0, 1)]
        pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=scale, sharpness=SHARP, radius=RADIUS, projCentre=PROJ,
                                          debugMode=debug, mathMode=_mathmode(mode)))
        if anyio and layered:
            lay = ovr.ArrayImage(W, H, fin, layers=2).upload(torch.stack([torch.from_numpy(e).to(dev) for e in eyes]))
            srcs = (lay, lay)
        else:
            srcs = tuple(_place(e, fin, "tma" if tma else ("array" if anyio else "tight"), dev) for e in eyes)
        if anyio:
            dsts = _outputs(unorm, ow, oh, dev, ["array", "array"])
            pp.apply_pair_into(srcs[0], srcs[1], dsts[0], dsts[1], fmt=None if not tma and anyio else _tag(fin))
            got = [_host(d) for d in dsts]
        else:
            got = [t.cpu().numpy() for t in pp.apply_pair(srcs[0], srcs[1], fmt=_tag(fin))]
        torch.cuda.synchronize()
        pp.close()
        out = []
        for e in (0, 1):
            uc = po.upscale_constants(e, True, W, H, ow, oh, proj=PROJ, radius=RADIUS)
            sc = po.sharpen_constants(e, True, ow, oh, proj=PROJ, radius=RADIUS, sharpness=SHARP, debug=debug)
            mid = po.easu(eyes[e], ow, oh, uc, src_fmt=fin, dst_fmt=_tag(unorm))
            want = po.rcas(mid, sc, src_fmt=_tag(unorm), dst_fmt=_tag(unorm))
            out.append((f"eye {e}{' (layer 1)' if layered and e else ''}", got[e], want, unorm, True))
        return out
    return Case("paired", mode, keys, run, f"{mode}:paired FIN={kl.FORMAT_NAMES[fin]} TW={tw} TMA={tma} ANYIO={anyio}"
                + (" layered" if layered else ""))


def _resolve(key):
    import openvr_fsr_b200 as ovr
    from oracle import frontend
    from openvr_fsr_b200 import synth
    fmt, s = key[2]
    # S = 0 (scalar fetches): an odd count; for the 4-byte formats also 2 samples, which used to pick a vector variant
    counts = [s] if s else ([3, 2] if fmt in kl.PACKED32 else [3])

    def run(dev):
        import torch
        out = []
        for n in counts:
            rng = np.random.default_rng(7 * n + fmt)
            if fmt == kl.RGBA8:
                raw = synth.uniform_rgba8(W * n, H, n)
                raw[..., 3] = rng.integers(0, 256, (H, W * n), dtype=np.uint8)
            elif fmt == kl.RGB10A2:
                raw = synth.uniform_rgb10a2(W * n, H, n)
            else:
                raw = rng.uniform(-0.1, 1.2, (H, W * n, 4)).astype(_np_dtype(fmt))
            src = ovr.alloc_image(W * n, H, _dtype(fmt), dev).copy_(torch.from_numpy(raw).to(dev))
            dst = ovr.alloc_image(W, H, _dtype(fmt), dev)
            ovr.resolve_msaa(src, dst, n, fmt=_tag(fmt))
            out.append((f"{n} samples", dst.cpu().numpy(), frontend.resolve_msaa(raw, n, fmt), fmt, False))
        return out
    return Case("resolve_msaa_kernel", "strict", {key}, run, kl.describe(key) + f" ({'/'.join(map(str, counts))} samples)")


def _host_entry():
    """ovrfsr_apply_host with tight host rows: the upload and the download are re-pitched on the device"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    keys = {("", "repitch_rows_kernel", ()), ("strict", "easu_kernel", (kl.RGBA8, kl.RGBA8, 60, 1, 1, 0)),
            ("strict", "rcas_kernel", (kl.RGBA8, kl.RGBA8, 1, 1, 0, 0))}

    def run(dev):
        ow, oh = ovr.output_size(W, H, 0.75)
        img = _content(kl.RGBA8, W, H, 5)
        src = torch.from_numpy(img).pin_memory()
        dst = torch.zeros((oh, ow, 4), dtype=torch.uint8).pin_memory()
        pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=0.75, sharpness=SHARP, radius=RADIUS, projCentre=PROJ))
        pp.apply_host(0, src, dst)
        torch.cuda.synchronize()
        pp.close()
        uc = po.upscale_constants(0, True, W, H, ow, oh, proj=PROJ, radius=RADIUS)
        sc = po.sharpen_constants(0, True, ow, oh, proj=PROJ, radius=RADIUS, sharpness=SHARP)
        return [("host", dst.numpy(), po.rcas(po.easu(img, ow, oh, uc), sc), kl.RGBA8, False)]
    return Case("host entry", "strict", keys, run, "strict:apply_host (tight host rows)")


def _rgb32f_source(content=None):
    """an R32G32B32_FLOAT eye: expanded to RGBA32F (alpha 1), then the paired passes"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    keys = {("", "expand_rgb32f_kernel", ()), ("strict", "easu_kernel", (kl.RGBA32F, kl.RGBA8, 60, 0, 1, 0)),
            ("strict", "rcas_kernel", (kl.RGBA8, kl.RGBA8, 1, 1, 0, 0))}

    def run(dev):
        ow, oh = ovr.output_size(W, H, 0.75)
        rgba = (content or _content)(kl.RGBA32F, W, H, 9)
        rgb = np.ascontiguousarray(rgba[..., :3])
        pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=0.75, sharpness=SHARP, radius=RADIUS, projCentre=PROJ))
        got = pp.apply(0, torch.from_numpy(rgb).to(dev), fmt=RGB32F).cpu().numpy()
        pp.close()
        uc = po.upscale_constants(0, True, W, H, ow, oh, proj=PROJ, radius=RADIUS)
        sc = po.sharpen_constants(0, True, ow, oh, proj=PROJ, radius=RADIUS, sharpness=SHARP)
        return [("rgb32f", got, po.rcas(po.easu(rgb, ow, oh, uc, src_fmt=RGB32F), sc), kl.RGBA8, False)]
    return Case("rgb32f source", "strict", keys, run, "strict:apply (R32G32B32_FLOAT source)")


def case_for(key, content=None):
    """the case that launches `key`; content(fmt, w, h, seed) replaces the sources of the FSR / NIS / CAS drivers"""
    mode, kernel, args = key
    p = dict(zip(kl.PARAMS[kernel], args))
    if kernel == "easu_kernel" and p["PAIRED"]:
        return _paired(mode, p["FIN"], p["TW"], p["TMA"], p["ANYIO"], content)
    if kernel == "rcas_kernel" and p["PAIRED"]:
        return _paired(mode, p["FIN"], 60, 1, p["ANYIO"], content)
    if kernel in ("easu_kernel", "rcas_kernel", "nis_scaler_kernel", "nis_sharpen_kernel", "cas_sharpen_kernel",
                  "cas_scale_kernel", "fsr_fused_kernel"):
        return _stateless(key, content)
    if kernel == "resolve_msaa_kernel":
        return _resolve(key)
    if kernel == "repitch_rows_kernel":
        return _host_entry()
    if kernel == "expand_rgb32f_kernel":
        return _rgb32f_source(content)
    return None


def _cases(ledger_keys, family):
    """the cases of one family, generated from the ledger: every key not yet launched by an earlier case gets one"""
    cases, claimed, missing = [], set(STATE["launched"]), []
    for key in sorted(k for k in ledger_keys if k[1] == family and k not in EXCLUDED):
        if key in claimed:
            continue
        c = case_for(key)
        if c is None:
            missing.append(kl.describe(key))
            continue
        assert key in c.keys, (kl.describe(key), c.name)
        claimed |= c.keys
        cases.append(c)
    assert not missing, "ledger keys without a driver:\n" + "\n".join(missing)
    return cases


# ---- recording launches --------------------------------------------------------------------------------------------
def _session(cases, dev):
    """run the cases under one torch.profiler session, a separator kernel (torch's spin kernel) after each; returns
    [(the library kernels recorded in the case's window, the library's launch count for the case, comparisons)]"""
    import torch
    import openvr_fsr_b200 as ovr
    from torch.profiler import ProfilerActivity, profile
    spans, results = [], []
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.cuda._sleep(1000)
        torch.cuda.synchronize()
        for c in cases:
            n0 = ovr.kernel_launches()
            results.append(c.run(dev))
            torch.cuda.synchronize()
            spans.append(ovr.kernel_launches() - n0)
            torch.cuda._sleep(1)
            torch.cuda.synchronize()
    events = sorted((e.start_ns(), e.name()) for e in prof.profiler.kineto_results.events()
                    if e.device_type() == torch.autograd.DeviceType.CUDA)
    windows, cur = [], []
    for _, name in events:
        if "spin_kernel" in name:
            windows.append(cur)
            cur = []
        elif kl.normalise(name) is not None:
            cur.append(kl.normalise(name))
    # aligned from the end: the case windows are the ones closed by the last len(cases) separators
    windows = ([[]] * len(cases) + windows)[-len(cases):]
    return list(zip(windows, spans, results))


def _run_recorded(cases, dev):
    """[(case, launched keys, comparisons)].  CUPTI can miss the first launches of a session: a case whose window holds
    fewer launches than the library counted is recorded again, alone."""
    out = []
    for c, (win, n, res) in zip(cases, _session(cases, dev)):
        if len(win) != n:
            print(f"  re-recording {c.name}: {len(win)} of {n} launches recorded")
            win, n, res = _session([c], dev)[0]
        assert len(win) == n, f"{c.name}: the profiler recorded {len(win)} of the {n} launches the library counted"
        out.append((c, set(win), res))
    return out


@pytest.fixture(scope="module")
def shipped(built_lib):
    STATE["t0"] = STATE["t0"] or time.monotonic()
    return set(kl.ledger(built_lib))


FAMILIES = ["easu_kernel", "rcas_kernel", "nis_scaler_kernel", "nis_sharpen_kernel", "cas_sharpen_kernel", "cas_scale_kernel",
            "fsr_fused_kernel", "resolve_msaa_kernel", "repitch_rows_kernel", "expand_rgb32f_kernel"]


def _run_family(family, shipped, dev):
    if family in STATE["ran"]:
        return
    STATE["ran"].add(family)
    cases = _cases(shipped, family)
    failures = []
    for mode in ("strict", "fast", ""):
        group = [c for c in cases if (c.mode if c.mode in ("strict", "fast") else "") == mode]
        if not group:
            continue
        for c, got_keys, res in _run_recorded(group, dev):
            STATE["launched"] |= got_keys
            if got_keys != c.keys:
                failures.append(f"{c.name}: launched {sorted(map(kl.describe, got_keys))}, expected {sorted(map(kl.describe, c.keys))}")
            for label, got, want, fmt, composed in res:
                msg, err = _check(got, want, fmt, c.mode, composed)
                if c.mode == "fast":
                    fam = f"{c.family}{' (composed)' if composed else ''} -> {kl.FORMAT_NAMES[fmt]}"
                    STATE["maxima"][fam] = max(STATE["maxima"][fam], err)
                if msg:
                    failures.append(f"{c.name} [{label}]: {msg}")
    print(f"{family}: {len(cases)} cases")
    assert not failures, f"{len(failures)} failures:\n" + "\n".join(failures)


@pytest.mark.parametrize("family", FAMILIES)
def test_every_variant_matches_the_oracle(cuda, shipped, family):
    _run_family(family, shipped, cuda)


def test_launched_and_compared_covers_the_ledger(cuda, shipped):
    for family in FAMILIES:
        try:
            _run_family(family, shipped, cuda)
        except AssertionError:
            pass  # reported by that family's test; coverage is judged on what ran
    target = shipped - set(EXCLUDED)
    covered = STATE["launched"] & target
    print(f"\nlaunched and compared vs ledger: {len(covered)}/{len(target)} ({len(shipped)} shipped, {len(EXCLUDED)} excluded)")
    print("excluded:")
    for k, why in sorted(EXCLUDED.items()):
        print(f"  {kl.describe(k)}: {why}")
    print("fast-math maxima (LSB / code, or relative for float outputs):")
    for fam, v in sorted(STATE["maxima"].items()):
        print(f"  {fam}: {v:.3g}")
    print(f"module wall time: {time.monotonic() - STATE['t0']:.1f} s")
    assert set(EXCLUDED) <= shipped, "an exclusion names a kernel the library no longer ships"
    assert not STATE["launched"] - shipped, "launched kernels the ledger does not list"
    assert covered == target, "never launched:\n" + "\n".join(sorted(map(kl.describe, target - covered)))
