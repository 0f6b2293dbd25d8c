"""Every float-source kernel and the context path against the oracle on infinite and NaN texels.

An R16G16B16A16_FLOAT render target overflows to +-inf at 65520, and a NaN from one bad shader pixel reaches the
compositor as it is; an FP32 eye texture can hold signalling NaNs with payloads.  This module runs the drivers of
tests/test_gpu_float_signed.py (themselves those of the variant matrix) on every ledger key whose source format is
RGBA16F or RGBA32F, both math modes, with content made of 12x10-texel blocks of finite scRGB content holding:

  one       sparse +inf / -inf / NaN in one colour channel
  three     sparse texels whose three colour channels are each +inf, -inf or NaN
  alphanan  NaN alpha only
  bits      RGBA16F: the half patterns 0x7c00, 0xfc00, 0x7e00 and the signalling 0x7c01 (and 0xfe01);
            RGBA32F: +-inf and signalling / quiet NaNs with payloads (0x7f800001, 0xff800001, 0x7fc00001, 0xffc00000, 0x7fa5a5a5)
  beside    +-inf texels next to +-0 and next to +-65504, on a random-sign zero field
  infblock  a whole block of +inf colour (alpha 1): whole EASU / CAS footprints of +inf
  finite    the content with no non-finite texel, so that the fast bound keeps pixels to hold to

and, over the blocks: a one-colour 18x18 window of +inf colour aligned to the 16x16 group (2, 1), which the RCAS
cases' radius puts inside (RCAS's one-colour group skip, rcas_flat_group, runs there; the RCAS cases assert it with the
window rule of tests/test_gpu_rcas_flat.py), non-finite texels at the four image corners (outside the radius, where the bilinear copy
reads them), along the image edges and along the source columns and rows that the 64-column / 32-row tile boundaries of
the kernels map to (their halo texels).

Strict math.  UNORM targets: every byte equal.  Float targets: every word that is not NaN equal bit for bit, the sign of
zero and of infinity included, and NaN at exactly the same words.  NaN payloads are not compared: the device's
arithmetic and FP16 store produce canonical NaNs (0x7fffffff, 0x7fff), the checker keeps x86's (the quietened input, or
0xffc00000 / 0x7e00), and D3D11 leaves NaN payloads unspecified.  Finite words keep the byte comparison of the variant
matrix.

Fast math: containment, not a bound.  An output whose footprint -- the source texels within REACH texels of the
nearest-texel source position of test_gpu_float_signed.footprint_magnitude -- holds no non-finite texel keeps the bounds
of test_gpu_float_signed.check.  REACH is a hand-set bound per kernel: its farthest tap as the source positions of
tests/test_resample_footprint_host.py place it, plus one texel for the nearest-texel mapping.  It is not derived from
those positions; a REACH that is too small shows as a class or bound failure at outputs taken as finite.  An output
whose footprint holds a non-finite texel must be written -- every destination holds a sentinel before the launch:
the test's own, and the paired context's, which apply_pair allocates on its first call, so that the compared call is
the second one into the same images -- and its class mismatches with the
checker (NaN / +inf / -inf / finite) are counted and reported, not bounded: fast math's reciprocals and regrouped sums
turn inf - inf, inf * 0 and inf / inf into NaN where the reference's order does not, and the reverse.  Only strict
math pins those pixels (DESIGN section 3).

The ledger part of the module takes about 92 s, and the whole module about 100 s, on one H100 80GB HBM3 at a 700 W
power limit."""
import time

import numpy as np
import pytest

from tests import kernel_ledger as kl
from tests import test_gpu_float_signed as fs
from tests import test_gpu_variant_matrix as vm

pytestmark = pytest.mark.gpu

FAMILIES = fs.FAMILIES
CONTENT = ("one", "three", "alphanan", "bits", "beside", "infblock", "finite")
NONFINITE_CONTENT = CONTENT[:-1]  # each must hold a non-finite texel wherever it is placed
F16_BITS = (0x7c00, 0xfc00, 0x7e00, 0x7c01, 0xfe01)
F32_BITS = (0x7f800000, 0xff800000, 0x7f800001, 0xff800001, 0x7fc00001, 0xffc00000, 0x7fa5a5a5)
# a hand-set bound, not derived: source texels between an output's nearest-texel source position and the farthest tap
# it reads, plus one for that mapping: EASU's 4x4 window and bilinear copy, RCAS's cross, NVScaler's 6x6 window and chroma tap, NVSharpen's 5x5,
# CAS's 3x3 (the upscale's 4x4 of bilinear windows); EASU -> RCAS (fused, paired) adds one output pixel
REACH = {"easu_kernel": 3, "rcas_kernel": 2, "nis_scaler_kernel": 4, "nis_sharpen_kernel": 3, "cas_sharpen_kernel": 2,
         "cas_scale_kernel": 3, "fsr_fused_kernel": 4, "paired": 4, "rgb32f source": 4}
SENTINEL = 0xA5
STATE = {"t0": None, "launched": set(), "ran": set(), "maxima": {}, "stats": {}}


# ---- content -------------------------------------------------------------------------------------------------------
def _types(fmt):
    return (np.float16, np.uint16) if fmt == kl.RGBA16F else (np.float32, np.uint32)


def _inf_nan(fmt):
    """(+inf, -inf, quiet NaN) bit patterns of the format"""
    return (0x7c00, 0xfc00, 0x7e00) if fmt == kl.RGBA16F else (0x7f800000, 0xff800000, 0x7fc00000)


def _per_block(rng, w, h, n):
    """n random texels in every 12x10 block: (ys, xs)"""
    ys, xs = [], []
    for by in range(0, h, 10):
        for bx in range(0, w, 12):
            ys += list(rng.integers(by, min(by + 10, h), n))
            xs += list(rng.integers(bx, min(bx + 12, w), n))
    return np.array(ys), np.array(xs)


def _families(fmt, w, h, seed):
    """{name: (h, w, 4) unsigned bit patterns of the format}"""
    ft, ut = _types(fmt)
    rng = np.random.default_rng(seed)
    pinf, ninf, qnan = _inf_nan(fmt)
    nonfinite = np.array([pinf, ninf, qnan, qnan | (0x8000 if fmt == kl.RGBA16F else 0x80000000)], dtype=ut)

    def base(s):
        return fs._natural(w, h, seed + s, -0.5, 7.5).astype(ft).view(ut).copy()
    one = base(0)
    ys, xs = _per_block(rng, w, h, 1)
    one[ys, xs, rng.integers(0, 3, len(ys))] = rng.choice(nonfinite, len(ys))
    three = base(1)
    ys, xs = _per_block(rng, w, h, 1)
    three[ys, xs, :3] = rng.choice(nonfinite, (len(ys), 3))
    alphanan = base(2)
    ys, xs = _per_block(rng, w, h, 1)
    alphanan[ys, xs, 3] = rng.choice(nonfinite[2:], len(ys))
    bits = base(3)
    ys, xs = _per_block(rng, w, h, 2)
    pats = np.array(F16_BITS if fmt == kl.RGBA16F else F32_BITS, dtype=ut)
    half = len(ys) // 2
    bits[ys[:half], xs[:half], rng.integers(0, 4, half)] = rng.choice(pats, half)
    bits[ys[half:], xs[half:], :3] = rng.choice(pats, (len(ys) - half, 3))
    beside = fs._signed_zeros(rng, (h, w, 4)).astype(ft).view(ut).copy()
    big = np.array([np.float16(65504).view(np.uint16), np.float16(-65504).view(np.uint16)] if fmt == kl.RGBA16F else
                   [np.float32(65504).view(np.uint32), np.float32(-65504).view(np.uint32)], dtype=ut)
    ys, xs = _per_block(rng, w, h, 1)
    # an infinity with +-65504 on its right, +-65504 or +-0 on its left, and the field's +-0 above and below
    beside[ys, np.minimum(xs + 1, w - 1), :3] = rng.choice(big, (len(ys), 1))
    beside[ys, np.maximum(xs - 1, 0), :3] = rng.choice(np.concatenate([big, [0, 0x8000 if fmt == kl.RGBA16F else 0x80000000]])
                                                       .astype(ut), (len(ys), 1))
    beside[ys, xs, :3] = rng.choice(nonfinite[:2], (len(ys), 1))
    infblock = np.zeros((h, w, 4), dtype=ut)
    infblock[..., :3] = pinf
    infblock[..., 3] = ft(1).view(ut)
    return {"one": one, "three": three, "alphanan": alphanan, "bits": bits, "beside": beside, "infblock": infblock,
            "finite": base(4)}


def _overlays(u, fmt, rng):
    """the +inf one-colour window, the corners, the image edges and the tile-boundary lines, on bit patterns u"""
    h, w = u.shape[:2]
    ft, ut = _types(fmt)
    pinf, ninf, qnan = _inf_nan(fmt)
    vals = np.array([pinf, ninf, qnan], dtype=ut)
    for y, x in ((0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1)):
        u[y, x, rng.integers(0, 3)] = rng.choice(vals)
    for x in range(3, w - 1, 17):
        u[0 if x % 2 else h - 1, x, :3] = rng.choice(vals)
    for y in range(4, h - 1, 13):
        u[y, 0 if y % 2 else w - 1, rng.integers(0, 3)] = rng.choice(vals)
    # the source columns / rows where 64 x 32 output tiles meet, at the matrix's scales (0.75, 0.9; the fused kernel's
    # 0.64 tall), one texel either side: the halo of both tiles
    for x in (46, 49, 57):
        if x < w:
            u[5 + x % 7::19, x, rng.integers(0, 3)] = rng.choice(vals)
    for y in (22, 25, 28):
        if y < h:
            u[y, 7 + y % 5::23, :3] = rng.choice(vals)
    if w >= 50 and h >= 34:  # the 18x18 cross window of 16x16 group (2, 1)
        u[15:33, 31:49, :3] = pinf
        u[15:33, 31:49, 3] = ft(1).view(ut)
    return u


def nonfinite_content(fmt, w, h, seed):
    """(h, w, 4) float16 / float32 source: 12x10-texel blocks of the content families, the block pattern shifted by
    seed, and the overlays (other formats: the variant matrix's content)"""
    if fmt not in fs.FLOAT_FORMATS:
        return vm._content(fmt, w, h, seed)
    ft, ut = _types(fmt)
    fams = _families(fmt, w, h, seed)
    sel = (np.arange(w)[None, :] // 12 + 3 * (np.arange(h)[:, None] // 10) + seed) % len(CONTENT)
    u = np.zeros((h, w, 4), dtype=ut)
    for i, name in enumerate(CONTENT):
        u = np.where((sel == i)[..., None], fams[name], u)  # bit patterns: payloads and signalling NaNs survive
        if name in NONFINITE_CONTENT and (sel == i).any():
            held = u[sel == i].view(ft)
            assert not np.isfinite(held).all(), f"content family {name} holds no non-finite texel"
    return _overlays(u, fmt, np.random.default_rng(seed)).view(ft)


# ---- comparison ----------------------------------------------------------------------------------------------------
def tainted(src, out_shape, reach):
    """(oh, ow): the outputs whose footprint (source texels within `reach` of the output's source position, the mapping
    of test_gpu_float_signed.footprint_magnitude) holds a non-finite texel"""
    from scipy.ndimage import maximum_filter
    bad = ~np.isfinite(src.astype(np.float32)).all(axis=-1)
    near = maximum_filter(bad, size=2 * reach + 1, mode="nearest")
    h, w = src.shape[:2]
    oh, ow = out_shape[:2]
    sy = np.minimum(((np.arange(oh) + 0.5) * h / oh).astype(int), h - 1)
    sx = np.minimum(((np.arange(ow) + 0.5) * w / ow).astype(int), w - 1)
    return near[sy][:, sx]


def strict_check(got, want, fmt):
    """None, or what differs: UNORM targets byte for byte; float targets every non-NaN word bit for bit, NaN at the
    same words (payloads not compared)"""
    if fmt not in fs.FLOAT_FORMATS or got.shape != want.shape:
        return vm._check(got, want, fmt, "strict", False)[0]
    gn, wn = np.isnan(got), np.isnan(want)
    if (gn != wn).any():
        i = tuple(np.argwhere(gn != wn)[0])
        return f"strict: NaN at {int((gn != wn).sum())} words the checker has none (or the reverse), first at {i}: " \
               f"{got[i]!r} vs {want[i]!r}"
    g, w = got.copy(), want.copy()
    g[gn] = 0
    w[wn] = 0
    msg = vm._check(g, w, fmt, "strict", False)[0]
    return msg and msg + fs._describe_strict_diff(g, w)


def _classes(a):
    return np.select([np.isnan(a), np.isposinf(a), np.isneginf(a)], [1, 2, 3], 0)


def _unwritten(got, want, taint):
    """tainted pixels that still hold the sentinel (and are not what the checker wants)"""
    gb = np.ascontiguousarray(got).view(np.uint8).reshape(got.shape[:2] + (-1,))
    wb = np.ascontiguousarray(want).view(np.uint8).reshape(want.shape[:2] + (-1,))
    return taint & (gb == SENTINEL).all(axis=-1) & (gb != wb).any(axis=-1)


def check(got, want, fmt, mode, composed, src, reach):
    """(None or a description, the fast-math error as test_gpu_float_signed.check gives it, statistics)"""
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}", float("inf"), {}
    taint = tainted(src, got.shape, reach) if src is not None else np.zeros(got.shape[:2], bool)
    st = {"outputs": int(taint.size), "tainted": int(taint.sum()), "class mismatches": 0}
    if fmt in fs.FLOAT_FORMATS:
        g = got.astype(np.float32)
        st["nan"], st["inf"] = int(np.isnan(g).sum()), int(np.isinf(g).sum())
    unwritten = _unwritten(got, want, taint)
    if unwritten.any():
        i = tuple(np.argwhere(unwritten)[0])
        return f"{int(unwritten.sum())} outputs with a non-finite footprint left unwritten, first at {i}", float("inf"), st
    if mode == "strict":
        return strict_check(got, want, fmt), 0.0, st
    if fmt in fs.FLOAT_FORMATS:
        cm = (_classes(got.astype(np.float32)) != _classes(want.astype(np.float32))) & taint[..., None]
        st["class mismatches"] = int(cm.sum())
        zero = np.zeros((), got.dtype)
        g, w = np.where(taint[..., None], zero, got), np.where(taint[..., None], zero, want)
        clean = np.where(np.isfinite(src.astype(np.float32)), src, 0).astype(src.dtype) if src is not None else None
        msg, err = fs.check(g, w, fmt, mode, composed, clean)
    else:
        msg, err = vm._check(np.where(taint[..., None], want, got), want, fmt, mode, composed)
    return msg, err, st


# ---- ledger cases --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def float_keys(built_lib):
    STATE["t0"] = STATE["t0"] or time.monotonic()
    keys = fs._float_keys(set(kl.ledger(built_lib)))
    assert keys, "the ledger lists no float-source kernels"
    return keys


def _poisoned_outputs(fmt, w, h, dev, kinds):
    """vm._outputs, every destination filled with the sentinel byte"""
    import torch
    import openvr_fsr_b200 as ovr
    outs = _plain_outputs(fmt, w, h, dev, kinds)
    for d in outs:
        if isinstance(d, ovr.ArrayImage):
            es = torch.empty((), dtype=d._dtype()).element_size()
            d.upload(torch.full((d.height, d.width, 4 * es), SENTINEL, dtype=torch.uint8, device=dev).view(d._dtype()))
        else:
            d.view(torch.uint8).fill_(SENTINEL)
    return outs


_plain_outputs = vm._outputs



def _poisoned_apply_pair(plain):
    """PostProcessor.apply_pair whose outputs hold the sentinel when the compared call runs: the context allocates them
    on the first call and keeps them, so they are poisoned and written a second time"""
    def apply_pair(pp, *args, **kwargs):
        import torch
        first = plain(pp, *args, **kwargs)
        torch.cuda.synchronize()
        for t in first:
            t.view(torch.uint8).fill_(SENTINEL)
        second = plain(pp, *args, **kwargs)
        assert [t.data_ptr() for t in second] == [t.data_ptr() for t in first], "apply_pair moved its outputs"
        return second
    return apply_pair


def rcas_inf_flat_groups(src):
    """the inside 16x16 groups of the RCAS cases whose 18x18 cross window is one RGB of +inf (tests/test_gpu_rcas_flat.py's
    window rule, with the sharpen constants of the variant matrix's RCAS driver)"""
    from oracle import pyoracle as po
    from tests import test_gpu_rcas_flat as rf
    h, w = src.shape[:2]
    fmt = kl.RGBA16F if src.dtype == np.float16 else kl.RGBA32F
    words = po.sharpen_constants(0, True, w, h, proj=vm.PROJ, radius=vm.RADIUS, sharpness=vm.SHARP).words()
    flat, _, _ = rf._classify(src, fmt, words)
    return [(gx, gy) for gx, gy in flat if np.isposinf(src[gy * 16, gx * 16, :3]).all()]


def _run_family(family, keys, dev, monkeypatch):
    """the cases of one family, as test_gpu_float_signed._run_family runs them"""
    import torch
    import openvr_fsr_b200 as ovr
    if family in STATE["ran"]:
        return
    STATE["ran"].add(family)
    cases, claimed, srcs = [], set(), []

    def content(fmt, w, h, seed):
        srcs.append(nonfinite_content(fmt, w, h, seed))
        return srcs[-1]
    for key in sorted(k for k in keys if k[1] == family):
        if key in claimed or key in STATE["launched"]:
            continue
        c = vm.case_for(key, content)
        assert c is not None and key in c.keys, kl.describe(key)
        claimed |= c.keys
        cases.append(c)
    failures = []
    monkeypatch.setattr(vm, "_outputs", _poisoned_outputs)
    monkeypatch.setattr(ovr.PostProcessor, "apply_pair", _poisoned_apply_pair(ovr.PostProcessor.apply_pair))
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
        if c.family == "rcas_kernel" and not rcas_inf_flat_groups(srcs[-1]):
            failures.append(f"{c.name}: no inside group with a one-colour +inf window (rcas_flat_group not reached)")
        for i, (label, got, want, fmt, composed) in enumerate(res):
            src = srcs[i] if len(srcs) == len(res) else srcs[-1]  # the paired case: one source per eye
            msg, err, st = check(got, want, fmt, c.mode, composed, src, REACH[c.family])
            agg = STATE["stats"].setdefault((c.family, c.mode), {})
            for k, v in st.items():
                agg[k] = agg.get(k, 0) + v
            if c.mode == "fast":
                fam = f"{c.family}{' (composed)' if composed else ''} -> {kl.FORMAT_NAMES[fmt]}"
                STATE["maxima"][fam] = max(STATE["maxima"].get(fam, 0.0), err)
            if msg:
                failures.append(f"{c.name} [{label}]: {msg}")
    monkeypatch.undo()
    print(f"{family}: {len(cases)} cases")
    assert not failures, f"{len(failures)} failures:\n" + "\n".join(failures)


@pytest.mark.parametrize("family", FAMILIES)
def test_float_source_nonfinite_matches_the_oracle(cuda, float_keys, family, monkeypatch):
    _run_family(family, float_keys, cuda, monkeypatch)


def test_every_float_source_key_launched_nonfinite(cuda, float_keys, monkeypatch):
    for family in FAMILIES:
        try:
            _run_family(family, float_keys, cuda, monkeypatch)
        except AssertionError:
            pass  # reported by that family's test; coverage is judged on what ran
    covered = STATE["launched"] & float_keys
    print(f"\nfloat-source keys launched and compared on non-finite content: {len(covered)}/{len(float_keys)}")
    print("per family and mode: outputs, outputs with a non-finite texel in their footprint, NaN / inf output words "
          "(float targets), fast-math class mismatches at those outputs (not bounded):")
    for (fam, mode), st in sorted(STATE["stats"].items()):
        print(f"  {fam} {mode}: {st.get('outputs', 0)} outputs, {st.get('tainted', 0)} tainted, {st.get('nan', 0)} NaN, "
              f"{st.get('inf', 0)} inf, {st.get('class mismatches', 0)} class mismatches")
    print("fast-math maxima at untainted outputs (LSB / code, or for float targets the error in units of the bound):")
    for fam, v in sorted(STATE["maxima"].items()):
        print(f"  {fam}: {v:.3g}")
    print(f"module wall time: {time.monotonic() - STATE['t0']:.1f} s")
    assert covered == float_keys, "never launched:\n" + "\n".join(sorted(map(kl.describe, float_keys - covered)))
    for (fam, mode), st in STATE["stats"].items():
        assert 0 < st["tainted"] < st["outputs"], f"{fam} {mode}: {st['tainted']} of {st['outputs']} outputs tainted"


def test_content_holds_every_pattern():
    """the blocks and overlays put every listed bit pattern, signalling NaNs included, into the source"""
    for fmt in fs.FLOAT_FORMATS:
        ft, ut = _types(fmt)
        seen = set()
        for seed in range(1, 8):
            u = nonfinite_content(fmt, vm.W, vm.H, seed).view(ut)
            seen |= set(np.unique(u).tolist())
        pats = F16_BITS if fmt == kl.RGBA16F else F32_BITS
        assert set(pats) <= seen, sorted(hex(p) for p in set(pats) - seen)
        src = nonfinite_content(fmt, vm.W, vm.H, 3)
        assert np.isposinf(src[15:33, 31:49, :3]).all()
        t = tainted(src, (vm.H, vm.W), REACH["easu_kernel"])
        assert 0.2 < t.mean() < 0.95, t.mean()


@pytest.mark.parametrize("fout", [kl.RGBA16F, kl.RGBA32F])
@pytest.mark.parametrize("fin", [kl.RGBA16F, kl.RGBA32F])
def test_easu_bilinear_zero_weights(cuda, fin, fout):
    """EASU at render scale 0.5, every group outside the radius: every other output column and row samples at an exact
    texel centre, a tap weight of 0.  The checker still adds that tap (c00 * 1 + c10 * 0), so an infinite texel next to
    the centre makes a NaN; strict math must give the same words, NaN at the same words"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    from tests import test_oracle_nonfinite_host as nh
    from tests import test_resample_footprint_host as fp
    F = np.float32
    src = nonfinite_content(fin, vm.W, vm.H, 9 + fin)
    ow, oh = ovr.output_size(vm.W, vm.H, 0.5)
    odt = np.float16 if fout == kl.RGBA16F else np.float32
    # the pixels whose x weight is 0 and whose zero-weighted x neighbour is non-finite while the centre texel is not
    p = np.arange(ow)
    s = fp.snap_subtexel(fp.mul_add_unfused(p.astype(F) / F(ow), F(vm.W), F(-0.5)))
    zero_x = p[(s == np.floor(s)) & (s >= 0) & (s + 1 < vm.W)]
    x0 = np.floor(s[zero_x]).astype(int)
    fin_rows = np.isfinite(src[..., :3].astype(np.float32)).all(-1)
    assert (fin_rows[:, x0] & ~fin_rows[:, x0 + 1]).any(), "no zero-weight tap reads a non-finite texel"
    for inside in (False, True):
        uc = nh._everywhere(po.upscale_constants(0, True, vm.W, vm.H, ow, oh, proj=vm.PROJ, radius=vm.RADIUS), inside)
        out = torch.empty((oh, ow, 4), dtype=vm._dtype(fout), device=cuda)
        out.view(torch.uint8).fill_(SENTINEL)
        ovr.fsr_easu(ovr.to_image(src, cuda), out, uc.words(), ovr.MATH_STRICT)
        torch.cuda.synchronize()
        want = po.easu(src, ow, oh, uc, out_dtype=odt)
        if not inside:
            assert np.isnan(want[:, zero_x, :3]).any()
        msg = strict_check(out.cpu().numpy(), want, fout)
        assert msg is None, f"{'filter' if inside else 'bilinear copy'}: {msg}"


@pytest.mark.parametrize("fout", [kl.RGBA16F, kl.RGBA32F])
@pytest.mark.parametrize("fin", [kl.RGBA16F, kl.RGBA32F])
def test_nis_sharpen_every_block_inside(cuda, fin, fout):
    """NVSharpen with every 32x32 block inside the radius: the variant matrix's geometry (radius 0.4 about (40, 28))
    puts none of its blocks inside, so the filter and its centre tap -- a bilinear sample whose zero-weighted
    neighbours are still added, so an infinite neighbour makes a NaN -- only run here"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    from tests import test_oracle_nonfinite_host as nh
    src = nonfinite_content(fin, vm.W, vm.H, 13 + fin)
    cfg, ok = po.nis_config(True, 0, True, vm.W, vm.H, vm.W, vm.H, proj=vm.PROJ, radius=vm.RADIUS, sharpness=vm.SHARP)
    assert ok
    cfg = nh._everywhere(cfg, True)
    odt = np.float16 if fout == kl.RGBA16F else np.float32
    for mode in ("strict", "fast"):
        out = torch.empty((vm.H, vm.W, 4), dtype=vm._dtype(fout), device=cuda)
        out.view(torch.uint8).fill_(SENTINEL)
        ovr.nis_sharpen(ovr.to_image(src, cuda), out, bytes(cfg), vm._mathmode(mode))
        torch.cuda.synchronize()
        want = po.nis_sharpen(src, cfg, out_dtype=odt)
        msg, _, _ = check(out.cpu().numpy(), want, fout, mode, False, src, REACH["nis_sharpen_kernel"])
        assert msg is None, f"{mode}: {msg}"


# ---- the context path ----------------------------------------------------------------------------------------------
SHARP = 0.8


def _strict_same(got, want, what):
    assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
    msg = strict_check(got, want, {np.dtype(np.float16): kl.RGBA16F, np.dtype(np.float32): kl.RGBA32F}.get(got.dtype, kl.RGBA8))
    assert msg is None, f"{what}: {msg}"


def _beyond_fp16(w, h, seed):
    """finite RGBA32F linear light with blocks and sparse texels from 6.6e4 to 1e6, of both signs"""
    rng = np.random.default_rng(seed)
    a = fs._natural(w, h, seed, -0.5, 7.5)
    hit = rng.random((h, w)) < 0.04
    a[hit, :3] = rng.uniform(6.6e4, 1e6, (int(hit.sum()), 3)) * rng.choice([-1.0, 1.0], (int(hit.sum()), 3))
    a[h // 3:h // 3 + 9, w // 3:w // 3 + 9, :3] = rng.uniform(6.6e4, 1e6, (9, 9, 3))
    return a.astype(np.float32)


def _fsr_chain(src, scale, radius, out_dtype, src_fmt=None, eye=0, one=True, proj=(.5, .5, .5, .5)):
    """(the oracle chain of the context's FSR path, EASU's intermediate stored in the output's format)"""
    from oracle import pyoracle as po
    h, w = src.shape[:2]
    ow, oh = po.output_size(w, h, scale)
    sc = po.sharpen_constants(eye, one, ow, oh, proj=proj, radius=radius, sharpness=SHARP)
    if scale == 1.0:
        return po.rcas(src, sc, out_dtype=out_dtype, src_fmt=src_fmt), None
    uc = po.upscale_constants(eye, one, w, h, ow, oh, proj=proj, radius=radius)
    mid = po.easu(src, ow, oh, uc, out_dtype=out_dtype, src_fmt=src_fmt)
    return po.rcas(mid, sc, out_dtype=out_dtype), mid


def _nis_chain(src, scale, radius, out_dtype, src_fmt=None):
    from oracle import pyoracle as po
    h, w = src.shape[:2]
    ow, oh = po.output_size(w, h, scale)
    cfg, ok = po.nis_config(scale == 1.0, 0, True, w, h, ow, oh, radius=radius, sharpness=SHARP)
    assert ok
    return po.nis_sharpen(src, cfg, out_dtype=out_dtype, src_fmt=src_fmt) if scale == 1.0 else \
        po.nis_scaler(src, ow, oh, cfg, out_dtype=out_dtype, src_fmt=src_fmt)


def _cfg(scale, radius, out_dtype, **kw):
    import openvr_fsr_b200 as ovr
    fmt = {np.uint8: ovr.FORMAT_AUTO, np.float16: ovr.FORMAT_RGBA16F, np.float32: ovr.FORMAT_RGBA32F}[out_dtype]
    return ovr.Config(fsrEnabled=True, renderScale=scale, sharpness=SHARP, radius=radius, outputFormat=fmt,
                      mathMode=ovr.MATH_STRICT, **kw)


@pytest.mark.parametrize("scale", [0.75, 1.0])
@pytest.mark.parametrize("kind", ["RGBA32F", "RGB32F"])
def test_ctx_fsr_fp16_output_makes_infinities(cuda, kind, scale):
    """finite FP32 eyes beyond 65504 into an RGBA16F output: at 0.75 EASU's RGBA16F intermediate rounds them to +-inf
    and RCAS reads those; at 1.0 RCAS reads the source and only its FP16 store overflows"""
    import torch
    import openvr_fsr_b200 as ovr
    src = _beyond_fp16(vm.W, vm.H, 31)
    feed, fmt = (np.ascontiguousarray(src[..., :3]), vm.RGB32F) if kind == "RGB32F" else (src, None)
    for radius in (0.4, 2.0):
        pp = ovr.PostProcessor(_cfg(scale, radius, np.float16))
        got = pp.apply(0, torch.from_numpy(feed).to(cuda), fmt=fmt).cpu().numpy()
        pp.close()
        want, mid = _fsr_chain(feed, scale, radius, np.float16, src_fmt=fmt)
        if scale != 1.0:
            assert np.isinf(mid).any() and (np.isinf(mid) & (mid < 0)).any(), "the checker's intermediate holds no -inf / +inf"
        assert np.isinf(want).any()
        _strict_same(got, want, f"{kind} -> RGBA16F scale {scale} radius {radius}")


@pytest.mark.parametrize("fused", [False, True])
def test_ctx_fsr_beyond_fp16_into_rgba8(cuda, fused):
    """the same eyes into RGBA8: the paired dispatches, or the fused kernel"""
    import torch
    import openvr_fsr_b200 as ovr
    src = _beyond_fp16(vm.W, vm.H, 32)
    t = torch.from_numpy(src).to(cuda)
    pp = ovr.PostProcessor(_cfg(0.75, 0.4, np.uint8, fusedFsr=fused))
    n0 = ovr.kernel_launches()
    got = pp.apply(0, t).cpu().numpy()
    n = ovr.kernel_launches() - n0
    pp.close()
    assert n == (1 if fused else 2), n
    _strict_same(got, _fsr_chain(src, 0.75, 0.4, np.uint8)[0], f"fused={fused}")


@pytest.mark.parametrize("out_dtype", [np.float16, np.uint8])
def test_ctx_nis_beyond_fp16(cuda, out_dtype):
    import torch
    import openvr_fsr_b200 as ovr
    src = _beyond_fp16(vm.W, vm.H, 33)
    pp = ovr.PostProcessor(_cfg(0.75, 0.4, out_dtype, useNis=True))
    got = pp.apply(0, torch.from_numpy(src).to(cuda)).cpu().numpy()
    pp.close()
    want = _nis_chain(src, 0.75, 0.4, out_dtype)
    if out_dtype == np.float16:
        assert np.isinf(want).any()
    _strict_same(got, want, f"NIS -> {np.dtype(out_dtype).name}")


def _fp16_eye(w, h, seed):
    return nonfinite_content(kl.RGBA16F, w, h, seed)


def test_ctx_msaa_resolve_of_opposite_infinities(cuda):
    """4x MSAA RGBA16F with a +inf and a -inf sample in some texels: the resolve's sum is NaN there, then FSR"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import frontend as fe
    eye = fs._natural(vm.W, vm.H, 4, -0.5, 7.5).astype(np.float16)
    ms = np.repeat(eye, 4, axis=1)
    rng = np.random.default_rng(4)
    ys0, xs0 = _per_block(rng, vm.W, vm.H, 1)
    ms[ys0, 4 * xs0 + 1, :3] = np.inf
    ms[ys0, 4 * xs0 + 2, :3] = -np.inf
    ys, xs = _per_block(rng, vm.W, vm.H, 1)
    ms[ys, 4 * xs + 3, rng.integers(0, 4, len(ys))] = np.nan
    reads = fe.resolve_msaa(ms, 4, kl.RGBA16F)
    assert np.isnan(reads[ys0, xs0, :3]).all()  # +inf + -inf: the resolve's sum is NaN at those texels
    for out_dtype in (np.float16, np.uint8):
        pp = ovr.PostProcessor(_cfg(0.75, 0.4, out_dtype))
        got = pp.apply(0, torch.from_numpy(ms).to(cuda), samples=4).cpu().numpy()
        pp.close()
        _strict_same(got, _fsr_chain(reads, 0.75, 0.4, out_dtype)[0], f"MSAA -> {np.dtype(out_dtype).name}")


@pytest.mark.parametrize("path", ["fsr", "nis"])
def test_ctx_srtm_nonfinite(cuda, path):
    """OVRFSR_FLAG_SRTM / OVRFSR_FLAG_SRTM_NIS on RGBA16F eyes holding +-inf and NaN: F(inf) = inf * rcp(inf) = NaN"""
    import torch
    import openvr_fsr_b200 as ovr
    from tests import test_gpu_nis_srtm as gn
    from tests import test_gpu_srtm as gs
    eye = _fp16_eye(vm.W, vm.H, 5)
    for out_dtype in (np.uint8, np.float16, np.float32):
        scale = 0.75
        if path == "fsr":
            pp = ovr.PostProcessor(_cfg(scale, 0.4, out_dtype, srtm=True))
            want = gs._chain(eye, 0, True, scale, 0.4, out_dtype)
        else:
            pp = ovr.PostProcessor(_cfg(scale, 0.4, out_dtype, useNis=True, srtmNis=True))
            want = gn._chain(eye, 0, True, scale, 0.4, out_dtype)
        got = pp.apply(0, torch.from_numpy(eye).to(cuda)).cpu().numpy()
        pp.close()
        _strict_same(got, want, f"{path} SRTM -> {np.dtype(out_dtype).name}")


def test_ctx_shared_texture_unequal_radii(cuda):
    """one RGBA16F texture holding both eyes, with +-inf and NaN texels, and a different radius override per eye:
    each 16x16 block is the oracle's all-inside or all-outside result, by the two-radius rule"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    from tests import test_gpu_focus_radius as fr
    iw, ih, scale = 2 * vm.W, vm.H, 0.75
    tex = _fp16_eye(iw, ih, 6)
    ow, oh = po.output_size(iw, ih, scale)
    pp = ovr.PostProcessor(_cfg(scale, 0.5, np.float16))
    proj = (.5, .5, .5, .5)
    rl, rr = 0.3, 0.8
    pp.set_focus_radius(0, rl)
    pp.set_focus_radius(1, rr)
    t = torch.from_numpy(tex).to(cuda)
    left = pp.apply(ovr.EYE_LEFT, t, ovr.TextureBounds(0.0, 0.0, 0.5, 1.0))
    pp.apply(ovr.EYE_RIGHT, t, ovr.TextureBounds(0.5, 0.0, 1.0, 1.0))
    got = left.cpu().numpy()
    pp.close()
    rsq = [po.upscale_constants(0, True, iw, ih, ow, oh, radius=r).radius[1] for r in (rl, rr)]
    centre = list(po.sharpen_constants(0, False, ow, oh, proj=proj).imageCentre)
    m = fr._mask((oh, ow), 16, 16, centre, *rsq)
    assert m.any() and not m.all()
    uin, uout = (fr._all(po.upscale_constants(0, False, iw, ih, ow, oh, proj=proj), k) for k in (True, False))
    mid = fr._select(m, po.easu(tex, ow, oh, uin, out_dtype=np.float16), po.easu(tex, ow, oh, uout, out_dtype=np.float16))
    sin, sout = (fr._all(po.sharpen_constants(0, False, ow, oh, proj=proj, sharpness=SHARP), k) for k in (True, False))
    want = fr._select(m, po.rcas(mid, sin, out_dtype=np.float16), po.rcas(mid, sout, out_dtype=np.float16))
    _strict_same(got, want, "shared texture")


def test_ctx_array_source(cuda):
    """one CUDA-array RGBA16F eye holding +-inf and NaN, FSR into an RGBA16F array destination"""
    import torch
    import openvr_fsr_b200 as ovr
    eye = _fp16_eye(vm.W, vm.H, 7)
    ow, oh = ovr.output_size(vm.W, vm.H, 0.75)
    src_a = ovr.ArrayImage(vm.W, vm.H, ovr.FORMAT_RGBA16F).upload(torch.from_numpy(eye).to(cuda))
    dst_a = ovr.ArrayImage(ow, oh, ovr.FORMAT_RGBA16F)
    pp = ovr.PostProcessor(_cfg(0.75, 0.4, np.float16))
    pp.apply_into(0, src_a, dst_a)
    got = dst_a.download().cpu().numpy()
    pp.close()
    for a in (src_a, dst_a):
        a.release()
        a.close()
    _strict_same(got, _fsr_chain(eye, 0.75, 0.4, np.float16)[0], "array source")
