"""RCAS's one-colour group path against the oracle.

An inside-radius 16x16 group whose cross window (every b / d / e / f / h texel its pixels read: the group plus a 1-texel
ring, zeros outside the image) has one RGB stores its first pixel's filter value in every row (rcas_flat_group in
fsr_kernels.cuh).  The fixtures paint into natural content: exactly one group's window; the window minus one ring texel
on each of the four sides (filtered); a rectangle off the group grid; border groups (a nonzero colour next to the zero
ring is filtered, black RGB under nonzero alpha is skipped); partial right / bottom groups; windows flat in two channels
only (filtered); RGB-flat windows under varying alpha (skipped); and, in float sources, one-colour windows of -0, NaN
and HDR texels.  No two painted windows overlap.  A numpy mirror of the window rule asserts that each fixture is what
its role says (a ring fixture's window differs from its first texel in exactly the one intended texel) and that every
fixture has both one-colour and filtered inside groups.

Strict math is compared bit for bit with the oracle (NaN outputs by position), fast math within 1 code of a UNORM
target and within 1e-3 (relative above 1) of a float target.  Sources RGBA8, BGRA8, BGRX8, RGB10A2, RGBA16F and RGBA32F, placed as TMA (pitch-aligned), plain-load (tight
rows) and CUDA-array sources; RGBA8, RGB10A2 and FP32 targets; several sharpness values, debug tint on and off; the
plain dispatch and the paired context path with outside groups.

Builds of the kernel with a wrong window test or a wrong stored value fail here: a test without the ring, a test that
leaves out the window's last column (second half-warp at columns 1-16), and one-colour groups storing the centre
texel instead of the filter value."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RGBA8, BGRA8, RGBA16F, RGBA32F, RGB10A2, BGRX8 = 0, 1, 2, 3, 4, 5
W, H = 189, 125  # 12 x 8 groups, the last column and row partial (13 pixels)
PROJ, RADIUS = (0.30, 0.40, 0.62, 0.55), 0.55


def _windows(w=W, h=H):
    """{(gx, gy): (x0, x1, y0, y1)} inclusive pixel rectangle of each group's 18x18 window (may leave the image)"""
    return {(gx, gy): (gx * 16 - 1, gx * 16 + 16, gy * 16 - 1, gy * 16 + 16)
            for gy in range((h + 15) // 16) for gx in range((w + 15) // 16)}


def _inside(words, gx, gy):
    c, r2 = [int(w) for w in words[4:8]], int(words[9])
    m = 0xFFFFFFFF
    d = lambda a, b: ((a - b) & m) * ((a - b) & m) & m  # noqa: E731
    x, y = gx * 16 + 8, gy * 16 + 8
    return ((d(c[0], x) + d(c[1], y)) & m) <= r2 or ((d(c[2], x) + d(c[3], y)) & m) <= r2


def _rgb_bits(img, fmt):
    """(H, W, 3) integer keys of the RGB bits each texel decodes from"""
    from openvr_fsr_b200 import synth
    if fmt == RGB10A2:
        return synth.unpack_rgb10a2(img)[..., :3].astype(np.int64)
    if fmt in (RGBA16F, RGBA32F):
        return np.ascontiguousarray(img[..., :3]).view(np.uint16 if fmt == RGBA16F else np.uint32).astype(np.int64)
    return img[..., :3].astype(np.int64)


def _classify(img, fmt, words):
    """(one-colour inside groups, filtered inside groups, outside groups) by the window rule"""
    h, w = img.shape[:2]
    key = np.zeros((h + 18, w + 18, 3), np.int64)  # zeros outside the image, as Texture2D.Load reads there
    key[1:h + 1, 1:w + 1] = _rgb_bits(img, fmt)
    flat, filt, outside = [], [], []
    for (gx, gy) in _windows(w, h):
        if not _inside(words, gx, gy):
            outside.append((gx, gy))
            continue
        win = key[gy * 16:gy * 16 + 18, gx * 16:gx * 16 + 18]
        (flat if (win == win[1, 1]).all() else filt).append((gx, gy))
    return flat, filt, outside


def _encode(val, alpha, fmt, rng):
    """float RGB values in [0, 1] (or any float for float formats) + alpha in [0, 1] -> the source array"""
    from openvr_fsr_b200 import synth
    if fmt in (RGBA16F, RGBA32F):
        return np.concatenate([val, alpha[..., None]], -1).astype(np.float16 if fmt == RGBA16F else np.float32)
    if fmt == RGB10A2:
        return synth.pack_rgb10a2(np.round(np.clip(val, 0, 1) * 1023).astype(np.int64),
                                  np.round(alpha * 3).astype(np.int64))
    out = np.empty(val.shape[:2] + (4,), np.uint8)
    out[..., :3] = np.round(np.clip(val, 0, 1) * 255).astype(np.uint8)
    out[..., 3] = np.round(alpha * 255).astype(np.uint8)
    if fmt in (BGRA8, BGRX8):
        out[..., :3] = out[..., 2::-1]
    if fmt == BGRX8:
        out[..., 3] = rng.integers(0, 256, val.shape[:2], dtype=np.uint8)
    return out


# Fixture roles, by group.  No two painted windows overlap (their groups are two or more apart in x or y), so every
# fixture is what it says when the kernel sees it; _check_roles asserts that with the numpy mirror.
RING = {(3, 1): (-1, 8), (5, 1): (16, 8), (7, 1): (8, -1), (9, 1): (8, 16)}  # one ring texel left / right / top / bottom
FLAT = {(1, 1): "one window", (5, 3): "one window", (3, 3): "RGB under varying alpha",
        (0, 7): "black, left border and partial bottom", (11, 2): "black, partial right",
        (11, 7): "black under varying alpha, partial corner"}
FLAT_FLOAT = {(7, 3): "-0", (9, 3): "NaN", (1, 5): "HDR"}
FILTERED = {(1, 3): "flat in two channels", (11, 0): "colour, top border and partial right",
            (11, 4): "colour, partial right", (3, 7): "colour, partial bottom"}


def _fixture(fmt, seed):
    from openvr_fsr_b200 import synth
    rng = np.random.default_rng(seed)
    val = synth.natural_f32(W, H, seed).astype(np.float64)
    alpha = np.ones((H, W))
    q = 1023.0 if fmt == RGB10A2 else 255.0
    step = 1.0 / q if fmt not in (RGBA16F, RGBA32F) else 1.0 / 64

    def paint(x0, x1, y0, y1, rgb, a=None):
        xs, ys = slice(max(x0, 0), min(x1, W - 1) + 1), slice(max(y0, 0), min(y1, H - 1) + 1)
        val[ys, xs] = rgb
        if a is not None:
            alpha[ys, xs] = a(alpha[ys, xs].shape)

    win = _windows()
    colours = [(0.2, 0.6, 0.35), (0.9, 0.1, 0.5), (0.41, 0.73, 0.12), (0.66, 0.33, 0.95)]
    # off the group grid, clear of every other fixture's window
    paint(40, 150, 70, 105, colours[3])
    # the window minus one ring texel, one per side: filtered
    for g, (dx, dy) in RING.items():
        paint(*win[g], colours[1])
        val[g[1] * 16 + dy, g[0] * 16 + dx] = (0.5, 0.5, 0.5)
    # flat in two channels only: filtered
    x0, x1, y0, y1 = win[1, 3]
    paint(x0, x1, y0, y1, colours[3])
    val[y0 + 1:y1:2, x0 + 1:x1:2, seed % 3] += step
    # a nonzero colour next to the zero ring (border and partial groups): filtered
    paint(*win[11, 0], colours[2])
    paint(*win[11, 4], colours[0])
    paint(*win[3, 7], colours[1])
    # one-colour windows: exactly one group's window, twice; RGB-flat under varying alpha; black RGB under nonzero
    # alpha next to the zero ring at the left border and in partial right / bottom groups
    paint(*win[1, 1], colours[0])
    paint(*win[5, 3], colours[2])
    paint(*win[3, 3], colours[2], a=lambda s: rng.integers(0, 4, s) / 3)
    paint(*win[0, 7], (0.0, 0.0, 0.0), a=lambda s: np.full(s, 1.0))
    paint(*win[11, 2], (0.0, 0.0, 0.0), a=lambda s: np.full(s, 2 / 3))
    paint(*win[11, 7], (0.0, 0.0, 0.0), a=lambda s: rng.integers(1, 4, s) / 3)
    if fmt in (RGBA16F, RGBA32F):
        paint(*win[7, 3], (-0.0, -0.0, -0.0))
        paint(*win[9, 3], (np.nan, 0.25, 0.5))
        paint(*win[1, 5], (3.5, 12.0, 0.75))
    return _encode(val, alpha, fmt, rng)


def _check_roles(img, fmt):
    """every fixture is what its role says, by the window rule (all groups taken as inside)"""
    key = np.zeros((H + 18, W + 18, 3), np.int64)
    key[1:H + 1, 1:W + 1] = _rgb_bits(img, fmt)
    window = lambda g: key[g[1] * 16:g[1] * 16 + 18, g[0] * 16:g[0] * 16 + 18]  # noqa: E731
    differs = lambda g: (window(g) != window(g)[1, 1]).any(-1)  # noqa: E731
    for g, (dx, dy) in RING.items():
        want = np.zeros((18, 18), bool)
        want[dy + 1, dx + 1] = True
        assert (differs(g) == want).all(), f"ring fixture {g}: the window differs from its first texel elsewhere"
    flat = {**FLAT, **(FLAT_FLOAT if fmt in (RGBA16F, RGBA32F) else {})}
    for g, what in flat.items():
        assert not differs(g).any(), f"one-colour fixture {g} ({what}) is not one colour"
    for g, what in FILTERED.items():
        assert differs(g).any(), f"filtered fixture {g} ({what}) is one colour"


def _place(arr, fmt, where, dev):
    import torch
    import openvr_fsr_b200 as ovr
    if where == "tma":
        return ovr.to_image(arr, dev)
    t = torch.from_numpy(arr).to(dev)
    return t if where == "tight" else ovr.ArrayImage(arr.shape[1], arr.shape[0], fmt).upload(t)


def _tag(fmt):
    return fmt if fmt in (BGRA8, RGB10A2, BGRX8) else None


def _compare(got, want, mode, out):
    if out == "f32":
        nan = np.isnan(want)
        assert (np.isnan(got) == nan).all(), "NaN outputs differ from the oracle"
        got, want = np.where(nan, 0, got).astype(np.float32), np.where(nan, 0, want).astype(np.float32)
        if mode == "fast":
            # test_gpu_float_signed.py's float-target bound (its ulp term is negligible at these magnitudes)
            err = np.abs(got.astype(np.float64) - want) / np.maximum(1.0, np.abs(want.astype(np.float64)))
            assert err.max() <= 1e-3, f"fast: relative error {err.max():.2e}"
            return
    if mode == "strict" or out == "f32":
        bad = int((np.ascontiguousarray(got).view(np.uint8) != np.ascontiguousarray(want).view(np.uint8)).sum())
        assert bad == 0, f"{bad} bytes differ from the oracle"
        return
    from openvr_fsr_b200 import synth
    codes = (lambda a: synth.unpack_rgb10a2(a)) if out == RGB10A2 else (lambda a: a.astype(np.int32))
    d = np.abs(codes(got) - codes(want))
    assert d.max() <= 1, f"fast: max {d.max()} LSB"


UNORM = [RGBA8, BGRA8, BGRX8, RGB10A2]
FLOATS = [RGBA16F, RGBA32F]


def _check_fixture(src, fmt, words, want_outside):
    flat, filt, outside = _classify(src, fmt, words)
    need = 1 if want_outside else 3
    assert len(flat) >= need and len(filt) >= need, f"{len(flat)} one-colour and {len(filt)} filtered inside groups"
    assert bool(outside) == want_outside
    return flat


def _run_plain(cuda, src, fmt, where, sc, mode, out):
    import torch
    import openvr_fsr_b200 as ovr
    mm = ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST
    s = _place(src, fmt, where, cuda)
    sfmt = None if where == "array" else _tag(fmt)
    if out == "f32":
        d = torch.zeros((H, W, 4), dtype=torch.float32, device=cuda)
        ovr.fsr_rcas(s, d, sc.words(), mm, src_fmt=sfmt)
    elif where == "array":
        d = ovr.ArrayImage(W, H, out)
        ovr.fsr_rcas(s, d, sc.words(), mm, src_fmt=None)
        return d.download().cpu().numpy()
    else:
        d = ovr.alloc_image(W, H, torch.uint8, cuda)
        ovr.fsr_rcas(s, d, sc.words(), mm, src_fmt=sfmt, dst_fmt=_tag(out))
    torch.cuda.synchronize()
    return d.cpu().numpy()


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("where", ["tma", "tight", "array"])
@pytest.mark.parametrize("fmt", UNORM + FLOATS)
def test_rcas_flat_groups_plain_dispatch(cuda, fmt, where, mode):
    from oracle import pyoracle as po
    if fmt in FLOATS and where == "tma":
        pytest.skip("float sources take plain loads only")
    cases = [(2.0, (0.5, 0.5, 0.5, 0.5), 0.2, False), (RADIUS, PROJ, 0.9, False), (2.0, (0.5, 0.5, 0.5, 0.5), 2.0, True)]
    for radius, proj, sharp, debug in cases:
        sc = po.sharpen_constants(0, True, W, H, proj=proj, radius=radius, sharpness=sharp, debug=debug)
        src = _fixture(fmt, seed=int(sharp * 10) + fmt)
        _check_roles(src, fmt)
        flat = _check_fixture(src, fmt, sc.words(), radius < 2.0)
        outs = ["f32"] if fmt in FLOATS else [RGB10A2] if fmt == RGB10A2 else [RGBA8, "f32"]
        for out in outs:
            if out == "f32" and where == "array":
                continue
            got = _run_plain(cuda, src, fmt, where, sc, mode, out)
            want = po.rcas(src, sc, out_dtype=np.float32 if out == "f32" else np.uint8, src_fmt=_tag(fmt),
                           dst_fmt=None if out == "f32" else _tag(out))
            _compare(got, want, mode, out)
            if out == "f32" and mode == "strict" and fmt in (RGBA8, RGBA32F):
                # a build that stores the centre texel instead of the filter value must fail: some one-colour group's
                # reference output differs from its texel
                cen = src[..., :3].astype(np.float32) / (255.0 if fmt == RGBA8 else 1.0)
                diff = [g for g in flat if not np.array_equal(want[g[1] * 16, g[0] * 16, :3].view(np.uint32),
                                                              cen[g[1] * 16, g[0] * 16].view(np.uint32))]
                assert diff, "no one-colour group whose RCAS value differs from its texel"


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("where", ["tma", "tight"])
@pytest.mark.parametrize("fmt", [RGBA8, RGB10A2])
def test_rcas_flat_groups_paired(cuda, fmt, where, mode):
    """the context path (paired EASU + RCAS, both eyes) at scale 0.75: one-colour source blocks around the eye centres
    become one-colour windows of the intermediate; the radius leaves outside groups, which the paired EASU writes
    straight to the final image"""
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    from oracle import pyoracle as po
    mm = ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST
    sw, sh = 94, 70
    ow, oh = ovr.output_size(sw, sh, 0.75)
    eyes, mids = [], []
    for e in (0, 1):
        uc = po.upscale_constants(e, True, sw, sh, ow, oh, proj=PROJ, radius=RADIUS)
        sc = po.sharpen_constants(e, True, ow, oh, proj=PROJ, radius=RADIUS, sharpness=0.8)
        val = synth.natural_f32(sw, sh, 40 + e).astype(np.float64)
        val[8:40, 8:40] = (0.2, 0.6, 0.35)
        val[20:54, 44:78] = (0.9, 0.1, 0.5)
        val[56:70, 0:30] = (0.0, 0.0, 0.0)
        rng = np.random.default_rng(e)
        src = _encode(val, rng.integers(1, 4, (sh, sw)) / 3, fmt, rng)
        mid = po.easu(src, ow, oh, uc, src_fmt=_tag(fmt), dst_fmt=_tag(fmt))
        flat, filt, outside = _classify(mid, fmt, sc.words())
        assert flat and filt and outside, f"eye {e}: {len(flat)} one-colour, {len(filt)} filtered, {len(outside)} outside"
        eyes.append(src)
        mids.append((mid, sc))
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=0.75, sharpness=0.8, radius=RADIUS, projCentre=PROJ,
                                      mathMode=mm))
    srcs = [_place(e, fmt, where, cuda) for e in eyes]
    got = [t.cpu().numpy() for t in pp.apply_pair(srcs[0], srcs[1], fmt=_tag(fmt))]
    torch.cuda.synchronize()
    pp.close()
    for e in (0, 1):
        mid, sc = mids[e]
        want = po.rcas(mid, sc, src_fmt=_tag(fmt), dst_fmt=_tag(fmt))
        _compare(got[e], want, mode, fmt)
