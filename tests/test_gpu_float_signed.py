"""Every float-source kernel against the oracle on signed, HDR and tiny texels.

scRGB eye textures (R16G16B16A16_FLOAT) hold negative channels and float render targets produce -0 routinely, so a
float source is not the [0, 1] content of the variant matrix.  This module runs the matrix's drivers
(tests/test_gpu_variant_matrix.py) on every ledger key whose source format is RGBA16F or RGBA32F -- EASU, RCAS, NVScaler,
NVSharpen, CAS sharpen / upscale and the fused kernel, both math modes, every target format, plain / CUDA-array I/O, the
paired context path -- with finite content made of blocks of:

  zeros       a random-sign zero field
  bands       -0 / +0 bands and a flat -0.25 block
  impulses    isolated texels from -2 to 7.5 on a random-sign zero field
  scrgb       natural content over about -0.5 .. 7.5
  subnormal   FP16 subnormals (k * 2^-24, |k| < 1024) and signed zeros: dark areas
  highlights  natural scRGB content with +-65504 texels
  ringzeros   +0 / -0 texels with sparse 0.5s (RCAS's ring min / max on zeros of both signs)
  beyond16    (FP32 sources) natural content over about -5e4 .. 1.5e5 with +-3e6 texels

and, as named regressions, the 48x36 RGBA32F image with flat +-0 bands, negative texels and impulses into an RGBA32F
target at scales 1.0 / 0.75 / 0.5, the 97x61 partial-tile shape, the R32G32B32_FLOAT expansion path and one stateful
PostProcessor.apply per FSR and NIS into a float target.

Strict math compares bytes, the sign of zero included.  Fast math runs the same content: UNORM targets keep the matrix's
bounds (<= 1 LSB / code per pass, composed <= 4 LSB); float targets keep <= 1e-3 * max(1, |ref|) plus a term that scales
with the largest texel in the output's footprint (see FOOTPRINT_ULPS; below 1e-5 within scRGB range); equal infinities of one sign match (an FP16 store of 65520 or
more is +inf on both sides), a NaN never does, nor an infinity against a finite value.  The ties of min / max on +-0
that this content forms are pinned by the checker's rule (oracle/ovr_glue.h; tests/test_gpu_minmax_rule.py)."""
import time

import numpy as np
import pytest

from tests import kernel_ledger as kl
from tests import test_gpu_variant_matrix as vm

pytestmark = pytest.mark.gpu

FLOAT_FORMATS = (kl.RGBA16F, kl.RGBA32F)
FAMILIES = ["easu_kernel", "rcas_kernel", "nis_scaler_kernel", "nis_sharpen_kernel", "cas_sharpen_kernel", "cas_scale_kernel",
            "fsr_fused_kernel"]
STATE = {"t0": None, "launched": set(), "ran": set(), "maxima": {}}
# Fast math on float targets: |got - ref| <= 1e-3 * max(1, |ref|) + FOOTPRINT_ULPS * 2^-23 * M, with M the largest
# magnitude of that channel within FOOTPRINT texels of the output's source position.  The second term is the part of
# the error that scales with the texels the filter combines: a tap weight that differs from the reference's by a
# rounding (regrouped taps, approximate reciprocals) times a +-65504 or 3e6 texel moves an output near 1 by more than
# 1e-3 (measured on H100: 0.0049 next to 65504 texels, EASU -> FP16; 0.003 next to 3e6 texels, NVScaler).  The reference's
# result is ill-conditioned there, as between two D3D11 GPUs.  On content within scRGB range M <= 7.5 and the term is
# below 1e-5: the matrix's bound.
FOOTPRINT = 5        # texels: EASU's 4x4 taps, NVScaler's 6x6, CAS / RCAS 3x3, plus the output -> source rounding
FOOTPRINT_ULPS = 8    # the measured worst cases above are below 1 ulp of M
ZERO_FAMILIES = ("zeros", "bands", "impulses", "subnormal", "ringzeros")  # each must hold -0 texels


# ---- content -------------------------------------------------------------------------------------------------------
def _signed_zeros(rng, shape):
    return np.where(rng.random(shape) < 0.5, -0.0, 0.0)


def _natural(w, h, seed, lo, hi):
    from openvr_fsr_b200 import synth
    return synth.natural_rgba8(w, h, seed).astype(np.float64) / 255.0 * (hi - lo) + lo


def _families(fmt, w, h, seed):
    rng = np.random.default_rng(seed)
    shape = (h, w, 4)
    zeros = _signed_zeros(rng, shape)
    bands = np.zeros(shape)  # by assignment: -0.0 + (+0.0) would be +0
    bands[:, (np.arange(w) // 3) % 3 == 0, :] = -0.0
    bands[(np.arange(h) // 4) % 3 == 2, :, :] = -0.25
    impulses = _signed_zeros(rng, shape)
    hit = rng.random((h, w)) < 0.05
    impulses[hit] = rng.choice([-2.0, -0.5, 0.25, 1.0, 3.0, 7.5], size=(int(hit.sum()), 4))
    scrgb = _natural(w, h, seed, -0.5, 7.5)
    k = rng.integers(-1023, 1024, shape).astype(np.float64)
    subnormal = np.where(k == 0, _signed_zeros(rng, shape), k * 2.0 ** -24)
    highlights = _natural(w, h, seed + 1, -0.5, 7.5)
    hit = rng.random((h, w)) < 0.03
    highlights[hit] = rng.choice([-65504.0, 65504.0], size=(int(hit.sum()), 4))
    fams = {"zeros": zeros, "bands": bands, "impulses": impulses, "scrgb": scrgb, "subnormal": subnormal,
            "highlights": highlights, "ringzeros": ring_zeros(rng, shape)}
    if fmt == kl.RGBA32F:
        beyond = _natural(w, h, seed + 2, -5.0e4, 1.5e5)
        hit = rng.random((h, w)) < 0.03
        beyond[hit] = rng.choice([-3.0e6, 3.0e6], size=(int(hit.sum()), 4))
        fams["beyond16"] = beyond
    for name in ZERO_FAMILIES:
        f = fams[name].astype(np.float16 if fmt == kl.RGBA16F else np.float32)
        assert (np.signbit(f) & (f == 0)).any(), f"content family {name} holds no -0"
    return fams


def ring_zeros(rng, shape):
    """+0 / -0 texels with sparse 0.5s: RCAS's ring min / max meet zeros of both signs with a positive maximum, and a
    -0 / +0 lobe reaches the output through the zero products of its neighbours"""
    return rng.choice([0.0, -0.0, 0.5], p=[0.5, 0.3, 0.2], size=shape)


def signed_content(fmt, w, h, seed, exclude=()):
    """(h, w, 4) float16 / float32 source: 12x10-texel blocks of the content families but `exclude`, the block pattern
    shifted by seed (other formats: the variant matrix's content)"""
    if fmt not in FLOAT_FORMATS:
        return vm._content(fmt, w, h, seed)
    fams = [f for name, f in _families(fmt, w, h, seed).items() if name not in exclude]
    sel = (np.arange(w)[None, :] // 12 + 3 * (np.arange(h)[:, None] // 10) + seed) % len(fams)
    out = np.zeros((h, w, 4))
    for i, f in enumerate(fams):
        out = np.where((sel == i)[..., None], f, out)
    return out.astype(np.float16 if fmt == kl.RGBA16F else np.float32)


def section8_content(w=48, h=36, seed=8):
    """DESIGN section 8's case: a random-sign zero field, a -0 band, a +0 band, a flat -0.25 block and 12 impulses"""
    rng = np.random.default_rng(seed)
    a = _signed_zeros(rng, (h, w, 4))
    a[:, w // 6:w // 6 + 6] = -0.0
    a[:, w // 2 - 3:w // 2 + 3] = 0.0
    a[h // 4:h // 4 + 12, 2 * w // 3:2 * w // 3 + 12] = -0.25
    for _ in range(12):
        a[rng.integers(0, h), rng.integers(0, w), :3] = rng.choice([-1.0, -0.25, 0.5, 1.0, 2.0], size=3)
    return a.astype(np.float32)


# ---- comparison ----------------------------------------------------------------------------------------------------
def footprint_magnitude(src, out_shape):
    """(oh, ow, 4): per channel, the largest |texel| within FOOTPRINT texels of each output pixel's source position"""
    from scipy.ndimage import maximum_filter
    a = maximum_filter(np.abs(src.astype(np.float64)), size=(2 * FOOTPRINT + 1, 2 * FOOTPRINT + 1, 1), mode="nearest")
    h, w = src.shape[:2]
    oh, ow = out_shape[:2]
    sy = np.minimum(((np.arange(oh) + 0.5) * h / oh).astype(int), h - 1)
    sx = np.minimum(((np.arange(ow) + 0.5) * w / ow).astype(int), w - 1)
    m = a[sy][:, sx]
    if m.shape[2] < 4:  # an R32G32B32_FLOAT source: alpha reads as 1
        m = np.concatenate([m, np.ones(m.shape[:2] + (1,))], axis=2)
    return m


def check(got, want, fmt, mode, composed, src=None):
    """(None if within the bound else a description, the fast-math error in units of the relative bound 1e-3).  src:
    the pass's source, for the footprint term of the float-target bound (None: no such term)"""
    if mode == "strict" or fmt not in FLOAT_FORMATS:
        return vm._check(got, want, fmt, mode, composed)
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}", float("inf")
    g, w = got.astype(np.float64), want.astype(np.float64)
    gi, wi = np.isinf(g), np.isinf(w)
    nan = np.isnan(g) | np.isnan(w)
    wrong_class = nan | (gi != wi) | (gi & wi & (np.sign(g) != np.sign(w)))
    if wrong_class.any():
        i = tuple(np.argwhere(wrong_class)[0])
        return f"fast: {int(wrong_class.sum())} NaN / infinity mismatches, first at {i}: {g[i]!r} vs {w[i]!r}", float("inf")
    fin = ~(gi | wi)
    m = footprint_magnitude(src, got.shape) if src is not None else np.zeros(got.shape)
    allowed = 1e-3 * np.maximum(1.0, np.abs(w)) + FOOTPRINT_ULPS * 2.0 ** -23 * m
    ratio = np.abs(g[fin] - w[fin]) / allowed[fin]  # equal infinities are matched above
    err = 1e-3 * float(ratio.max()) if ratio.size else 0.0
    if err > 1e-3:
        i = tuple(np.argwhere(fin)[int(np.argmax(ratio))])
        return f"fast: error {abs(g[i] - w[i]):.3g} > {allowed[i]:.3g} at {i}: {g[i]!r} vs {w[i]!r} (footprint max {m[i]:.3g})", err
    return None, err


def _describe_strict_diff(got, want):
    """words that differ, and how many of them differ only in the sign of a zero"""
    if got.dtype.kind != "f" or got.shape != want.shape:
        return ""
    diff = np.ascontiguousarray(got).view(np.uint8).reshape(got.shape + (-1,)) != \
        np.ascontiguousarray(want).view(np.uint8).reshape(want.shape + (-1,))
    words = diff.any(axis=-1)
    zero_sign = words & (got == 0) & (want == 0)
    i = tuple(np.argwhere(words)[0]) if words.any() else None
    return f" ({int(words.sum())} words, {int(zero_sign.sum())} only the sign of a zero; first at {i}: " \
           f"{got[i]!r} vs {want[i]!r})" if i else ""


# ---- ledger cases --------------------------------------------------------------------------------------------------
def _float_keys(shipped):
    return {k for k in shipped if k[1] in FAMILIES and dict(zip(kl.PARAMS[k[1]], k[2]))["FIN"] in FLOAT_FORMATS}


@pytest.fixture(scope="module")
def float_keys(built_lib):
    STATE["t0"] = STATE["t0"] or time.monotonic()
    keys = _float_keys(set(kl.ledger(built_lib)))
    assert keys, "the ledger lists no float-source kernels"
    return keys


def _run_family(family, keys, dev):
    """the cases of one family.  A driver of the variant matrix launches the kernels it claims whatever the content (the
    launch switches look at formats and layouts, never at texel values), which test_gpu_variant_matrix.py records with
    torch.profiler; here a case must make at least one launch per claimed kernel, and its claims count as launched."""
    import torch
    import openvr_fsr_b200 as ovr
    if family in STATE["ran"]:
        return
    STATE["ran"].add(family)
    cases, claimed, srcs = [], set(), []

    def content(fmt, w, h, seed):  # signed_content, remembered for the footprint term of the fast bound
        srcs.append(signed_content(fmt, w, h, seed))
        return srcs[-1]
    for key in sorted(k for k in keys if k[1] == family):
        if key in claimed or key in STATE["launched"]:
            continue
        c = vm.case_for(key, content)
        assert c is not None and key in c.keys, kl.describe(key)
        claimed |= c.keys
        cases.append(c)
    failures = []
    for c in cases:
        n0 = ovr.kernel_launches()
        srcs.clear()
        res = c.run(dev)
        torch.cuda.synchronize()
        n = ovr.kernel_launches() - n0
        if n < len(c.keys):
            failures.append(f"{c.name}: {n} launches for {len(c.keys)} claimed kernels")
        else:
            STATE["launched"] |= c.keys
        for label, got, want, fmt, composed in res:
            # float targets come from the single-source drivers; the two-eye (paired) case has UNORM targets
            msg, err = check(got, want, fmt, c.mode, composed, srcs[-1] if len(srcs) == 1 else None)
            if c.mode == "fast":
                fam = f"{c.family}{' (composed)' if composed else ''} -> {kl.FORMAT_NAMES[fmt]}"
                STATE["maxima"][fam] = max(STATE["maxima"].get(fam, 0.0), err)
            if msg:
                extra = _describe_strict_diff(got, want) if c.mode == "strict" else ""
                failures.append(f"{c.name} [{label}]: {msg}{extra}")
    print(f"{family}: {len(cases)} cases")
    assert not failures, f"{len(failures)} failures:\n" + "\n".join(failures)


@pytest.mark.parametrize("family", FAMILIES)
def test_float_source_matches_the_oracle(cuda, float_keys, family):
    _run_family(family, float_keys, cuda)


def test_every_float_source_key_launched(cuda, float_keys):
    for family in FAMILIES:
        try:
            _run_family(family, float_keys, cuda)
        except AssertionError:
            pass  # reported by that family's test; coverage is judged on what ran
    covered = STATE["launched"] & float_keys
    print(f"\nfloat-source keys launched and compared: {len(covered)}/{len(float_keys)}")
    print("fast-math maxima (LSB / code, or for float targets the error in units of the bound, scaled to 1e-3):")
    for fam, v in sorted(STATE["maxima"].items()):
        print(f"  {fam}: {v:.3g}")
    print(f"module wall time: {time.monotonic() - STATE['t0']:.1f} s")
    assert covered == float_keys, "never launched:\n" + "\n".join(sorted(map(kl.describe, float_keys - covered)))


# ---- named regressions ---------------------------------------------------------------------------------------------
def _strict_equal(got, want, what):
    msg, _ = vm._check(got, want, kl.RGBA32F, "strict", False)
    assert msg is None, f"{what}: {msg}{_describe_strict_diff(got, want)}"


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("scale", [1.0, 0.75, 0.5])
def test_section8_easu_rgba32f(cuda, scale, mode):
    """48x36 RGBA32F source with flat +-0 bands, negative texels and impulses -> RGBA32F, then RCAS on the result"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    src = section8_content()
    h, w = src.shape[:2]
    ow, oh = ovr.output_size(w, h, scale)
    uc = po.upscale_constants(0, True, w, h, ow, oh, radius=2.0)
    sc = po.sharpen_constants(0, True, ow, oh, radius=2.0, sharpness=0.9)
    mm = ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST
    out = torch.empty((oh, ow, 4), dtype=torch.float32, device=cuda)
    ovr.fsr_easu(torch.from_numpy(src).to(cuda), out, uc.words(), mm)
    sharp = torch.empty_like(out)
    want = po.easu(src, ow, oh, uc, out_dtype=np.float32)
    ovr.fsr_rcas(torch.from_numpy(want).to(cuda), sharp, sc.words(), mm)
    torch.cuda.synchronize()
    want_r = po.rcas(want, sc, out_dtype=np.float32)
    for what, got, ref in (("EASU", out.cpu().numpy(), want), ("RCAS", sharp.cpu().numpy(), want_r)):
        if mode == "strict":
            _strict_equal(got, ref, f"{what} {w}x{h} -> {ow}x{oh}")
        else:
            msg, _ = check(got, ref, kl.RGBA32F, "fast", False, src if what == "EASU" else want)
            assert msg is None, f"{what} {w}x{h} -> {ow}x{oh}: {msg}"


@pytest.mark.parametrize("fout", [kl.RGBA16F, kl.RGBA32F])
@pytest.mark.parametrize("fin", [kl.RGBA16F, kl.RGBA32F])
def test_rcas_signed_zero_ring(cuda, fin, fout):
    """strict RCAS on a whole 97x61 image of ring_zeros content (every group inside the radius), three seeds: the ring
    min / max ties between -0 and +0 decide the sign of zero outputs"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    w, h = 97, 61
    sc = po.sharpen_constants(0, True, w, h, proj=vm.PROJ, radius=2.0, sharpness=vm.SHARP)
    odt = np.float16 if fout == kl.RGBA16F else np.float32
    for seed in (1, 2, 3):
        src = ring_zeros(np.random.default_rng(seed), (h, w, 4)).astype(np.float16 if fin == kl.RGBA16F else np.float32)
        out = torch.empty((h, w, 4), dtype=torch.float16 if fout == kl.RGBA16F else torch.float32, device=cuda)
        ovr.fsr_rcas(torch.from_numpy(src).to(cuda), out, sc.words(), ovr.MATH_STRICT)
        torch.cuda.synchronize()
        _strict_equal(out.cpu().numpy(), po.rcas(src, sc, out_dtype=odt), f"seed {seed}")


@pytest.mark.parametrize("kernel", ["easu", "rcas", "nis_scaler", "nis_sharpen", "cas_sharpen", "cas_scale"])
def test_partial_tiles_97x61_signed(cuda, kernel):
    """the 97x61 partial-tile shape with DESIGN section 8's content, strict, RGBA32F -> RGBA32F"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    w, h = 97, 61
    src = section8_content(w, h, seed=97)
    t = torch.from_numpy(src).to(cuda)
    ow, oh = (w, h) if kernel in ("rcas", "nis_sharpen", "cas_sharpen") else ovr.output_size(w, h, 0.75)
    out = torch.empty((oh, ow, 4), dtype=torch.float32, device=cuda)
    mm = ovr.MATH_STRICT
    if kernel == "easu":
        uc = po.upscale_constants(0, True, w, h, ow, oh, proj=vm.PROJ, radius=vm.RADIUS)
        ovr.fsr_easu(t, out, uc.words(), mm)
        want = po.easu(src, ow, oh, uc, out_dtype=np.float32)
    elif kernel == "rcas":
        sc = po.sharpen_constants(0, True, w, h, proj=vm.PROJ, radius=vm.RADIUS, sharpness=vm.SHARP)
        ovr.fsr_rcas(t, out, sc.words(), mm)
        want = po.rcas(src, sc, out_dtype=np.float32)
    elif kernel.startswith("nis"):
        scaler = kernel == "nis_scaler"
        cfg, ok = po.nis_config(not scaler, 0, True, w, h, ow, oh, proj=vm.PROJ, radius=vm.RADIUS, sharpness=vm.SHARP)
        assert ok
        (ovr.nis_scaler if scaler else ovr.nis_sharpen)(t, out, bytes(cfg), mm)
        want = po.nis_scaler(src, ow, oh, cfg, out_dtype=np.float32) if scaler else po.nis_sharpen(src, cfg, out_dtype=np.float32)
    else:
        sharpen_only = kernel == "cas_sharpen"
        kc = po.cas_setup(vm.SHARP, 1.0, w, h, ow, oh)
        ovr.cas(t, out, kc.words(), sharpen_only, mm)
        want = po.cas(src, ow, oh, kc, sharpen_only, out_dtype=np.float32)
    torch.cuda.synchronize()
    _strict_equal(out.cpu().numpy(), want, f"{kernel} {w}x{h} -> {ow}x{oh}")


@pytest.mark.parametrize("fout", [kl.RGBA16F, kl.RGBA32F])
@pytest.mark.parametrize("path", ["fsr", "nis", "rgb32f"])
def test_postprocessor_apply_float_target(cuda, path, fout):
    """one stateful PostProcessor.apply per path into a float target, strict: FSR (EASU -> float -> RCAS), NIS
    (NVScaler) on an RGBA16F / RGBA32F eye, and an R32G32B32_FLOAT eye through the expansion and FSR"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    w, h, scale = vm.W, vm.H, 0.75
    fin = kl.RGBA32F if path == "rgb32f" else fout
    # an FP16 intermediate holds no texel beyond 65504: such a texel would reach RCAS as an infinity (a non-finite input)
    src = signed_content(fin, w, h, 11 + fin, exclude=("beyond16",) if fout == kl.RGBA16F else ())
    feed, sfmt = (np.ascontiguousarray(src[..., :3]), vm.RGB32F) if path == "rgb32f" else (src, None)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, useNis=path == "nis", renderScale=scale, sharpness=vm.SHARP,
                                      radius=vm.RADIUS, projCentre=vm.PROJ, outputFormat=fout, mathMode=ovr.MATH_STRICT))
    got = pp.apply(0, torch.from_numpy(feed).to(cuda), fmt=sfmt).cpu().numpy()
    pp.close()
    ow, oh = ovr.output_size(w, h, scale)
    odt = np.float16 if fout == kl.RGBA16F else np.float32
    if path == "nis":
        cfg, ok = po.nis_config(False, 0, True, w, h, ow, oh, proj=vm.PROJ, radius=vm.RADIUS, sharpness=vm.SHARP)
        assert ok
        want = po.nis_scaler(feed, ow, oh, cfg, out_dtype=odt)
    else:
        uc = po.upscale_constants(0, True, w, h, ow, oh, proj=vm.PROJ, radius=vm.RADIUS)
        sc = po.sharpen_constants(0, True, ow, oh, proj=vm.PROJ, radius=vm.RADIUS, sharpness=vm.SHARP)
        want = po.rcas(po.easu(feed, ow, oh, uc, out_dtype=odt, src_fmt=sfmt), sc, out_dtype=odt)
    assert got.dtype == want.dtype, (got.dtype, want.dtype)
    _strict_equal(got, want, f"{path} -> {kl.FORMAT_NAMES[fout]}")
