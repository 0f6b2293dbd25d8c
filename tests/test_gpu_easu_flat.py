"""EASU's one-colour group path against the oracle.

An inside-radius 16x16 group whose footprint (every f / g / j / k texel its pixels use) has one RGB stores f without
running the filter (easu_flat_group in fsr_kernels.cuh).  The fixtures paint one-colour rectangles into natural content:
exactly a group block's footprint, the same minus its last column or last row (so the footprint rule is tested at its
edges), rectangles off the group grid, rectangles over the image border (clamp to edge), rectangles flat in two of the
three channels only (must be filtered) and flat in RGB under varying alpha (must be skipped); plus an image of one colour.
A numpy mirror of the footprint rule asserts that every fixture has both one-colour and filtered inside groups, so the
test cannot pass without running both paths.

Strict math is compared bit for bit with the oracle, fast math with the per-pass tolerances of
test_gpu_variant_matrix.py.  Formats RGBA8, BGRA8, BGRX8 and RGB10A2, placed as TMA (pitch-aligned), plain-load (tight
rows) and CUDA-array sources; the plain dispatch and the paired context path; scales 0.75, 0.5 and 0.9."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RGBA8, BGRA8, RGB10A2, BGRX8 = 0, 1, 4, 5
W, H = 125, 93
PROJ, RADIUS = (0.30, 0.40, 0.62, 0.55), 0.55
FLAT = (0.2, 0.6, 0.35)


def _f32(u):
    return np.array([u], dtype=np.uint32).view(np.float32)[0]


def _pos(p, scale, offs):
    """easu_pos: (float)p * scale, then + offs, each rounded to binary32"""
    return np.float32(np.float32(p) * scale) + offs


def _footprints(words, ow, oh):
    """{(gx, gy): (x0, x1, y0, y1)} source texel rectangle of each group's f / g / j / k, unclamped"""
    c0x, c0y, c0z, c0w = (_f32(words[i]) for i in range(4))
    fp = {}
    for gy in range((oh + 15) // 16):
        for gx in range((ow + 15) // 16):
            x0, y0 = gx * 16, gy * 16
            x1, y1 = min(x0 + 15, ow - 1), min(y0 + 15, oh - 1)
            fp[gx, gy] = (int(np.floor(_pos(x0, c0x, c0z))), int(np.floor(_pos(x1, c0x, c0z))) + 1,
                          int(np.floor(_pos(y0, c0y, c0w))), int(np.floor(_pos(y1, c0y, c0w))) + 1)
    return fp


def _inside(words, gx, gy):
    """group_inside(): wrapping u32 distance of the group centre to either eye centre"""
    c, r2 = [int(w) for w in words[16:20]], int(words[21])
    m = 0xFFFFFFFF
    d = lambda a, b: ((a - b) & m) * ((a - b) & m) & m  # noqa: E731
    x, y = gx * 16 + 8, gy * 16 + 8
    return ((d(c[0], x) + d(c[1], y)) & m) <= r2 or ((d(c[2], x) + d(c[3], y)) & m) <= r2


def _rgb_key(img, fmt):
    from openvr_fsr_b200 import synth
    rgb = synth.unpack_rgb10a2(img)[..., :3] if fmt == RGB10A2 else img[..., :3]
    return rgb.astype(np.int64) @ np.array([1, 1 << 10, 1 << 20])


def _classify(img, fmt, words, ow, oh):
    """(one-colour inside groups, filtered inside groups, outside groups) by the footprint rule, on the clamped source"""
    key = _rgb_key(img, fmt)
    h, w = key.shape
    flat = filt = outside = 0
    for (gx, gy), (x0, x1, y0, y1) in _footprints(words, ow, oh).items():
        if not _inside(words, gx, gy):
            outside += 1
            continue
        xs, ys = np.clip(np.arange(x0, x1 + 1), 0, w - 1), np.clip(np.arange(y0, y1 + 1), 0, h - 1)
        if np.all(key[np.ix_(ys, xs)] == key[ys[0], xs[0]]):
            flat += 1
        else:
            filt += 1
    return flat, filt, outside


def _paint(img, fmt, x0, x1, y0, y1, rgb=FLAT, vary=None, rng=None):
    """one colour on the clamped rectangle; vary = a channel index that gets a +-1 code pattern (flat in two
    channels only), or 'alpha' for random alpha under one RGB"""
    h, w = img.shape[:2]
    xs, ys = slice(max(x0, 0), min(x1, w - 1) + 1), slice(max(y0, 0), min(y1, h - 1) + 1)
    sub_h, sub_w = ys.stop - ys.start, xs.stop - xs.start
    if sub_h <= 0 or sub_w <= 0:
        return
    if fmt == RGB10A2:
        codes = np.broadcast_to(np.round(np.array(rgb) * 1023).astype(np.int64), (sub_h, sub_w, 3)).copy()
        alpha = np.full((sub_h, sub_w), 3, np.int64)
    else:
        codes = np.broadcast_to(np.round(np.array(rgb) * 255).astype(np.int64), (sub_h, sub_w, 3)).copy()
        alpha = np.full((sub_h, sub_w), 255, np.int64)
        if fmt == BGRA8 or fmt == BGRX8:
            codes = codes[..., ::-1].copy()
    if vary == "alpha":
        alpha = rng.integers(0, 4 if fmt == RGB10A2 else 256, (sub_h, sub_w))
    elif vary is not None:
        codes[..., vary] += (np.add.outer(np.arange(sub_h), np.arange(sub_w)) % 2)
    if fmt == RGB10A2:
        from openvr_fsr_b200 import synth
        img[ys, xs] = synth.pack_rgb10a2(codes, alpha)
    else:
        img[ys, xs, :3] = codes.astype(np.uint8)
        img[ys, xs, 3] = alpha.astype(np.uint8)


def _fixture(fmt, words, ow, oh, seed, whole=False):
    from openvr_fsr_b200 import synth
    rng = np.random.default_rng(seed)
    img = synth.natural_rgb10a2(W, H, seed) if fmt == RGB10A2 else synth.natural_rgba8(W, H, seed)
    if fmt == BGRX8:
        img[..., 3] = rng.integers(0, 256, (H, W), dtype=np.uint8)
    if whole:
        _paint(img, fmt, 0, W - 1, 0, H - 1, vary="alpha", rng=rng)
        return img
    fp = _footprints(words, ow, oh)
    ngx, ngy = (ow + 15) // 16, (oh + 15) // 16
    # a 2x2 block of groups, exactly its footprint
    x0, _, y0, _ = fp[1, 1]
    _, x1, _, y1 = fp[2, 2]
    _paint(img, fmt, x0, x1, y0, y1)
    # one group's footprint minus its last column, one minus its last row: both must be filtered
    a = fp[4 % ngx, 1]
    _paint(img, fmt, a[0], a[1] - 1, a[2], a[3], rgb=(0.9, 0.1, 0.5))
    b = fp[1, 3 % ngy]
    _paint(img, fmt, b[0], b[1], b[2], b[3] - 1, rgb=(0.05, 0.05, 0.05))
    # over the right / bottom image border (clamp to edge) and across the last partial group
    c = fp[ngx - 2, ngy - 2]
    _paint(img, fmt, c[0], W + 4, c[2], H + 4, rgb=(1.0, 1.0, 1.0))
    # over the top-left border, off the group grid
    _paint(img, fmt, -3, fp[1, 0][1] + 3, -3, 9, rgb=(0.0, 0.0, 0.0))
    # flat in RGB under random alpha (skipped), and flat in two channels only (filtered)
    d = fp[5 % ngx, 3 % ngy]
    _paint(img, fmt, d[0] - 2, d[1] + 1, d[2] - 1, d[3] + 2, rgb=(0.4, 0.3, 0.8), vary="alpha", rng=rng)
    e = fp[3, 4 % ngy]
    _paint(img, fmt, e[0] - 1, e[1] + 1, e[2] - 1, e[3] + 1, rgb=(0.7, 0.7, 0.2), vary=int(seed) % 3)
    # under a radius mask: the exact footprints of the first and the last inside group
    inside = [g for g in sorted(fp, key=lambda g: (g[1], g[0])) if _inside(words, *g)]
    for g, rgb in ((inside[0], (0.3, 0.3, 0.9)), (inside[-1], (0.6, 0.8, 0.1))):
        _paint(img, fmt, *fp[g], rgb=rgb)
    return img


def _place(arr, fmt, where, dev):
    import torch
    import openvr_fsr_b200 as ovr
    if where == "tma":
        return ovr.to_image(arr, dev)
    t = torch.from_numpy(arr).to(dev)
    return t if where == "tight" else ovr.ArrayImage(arr.shape[1], arr.shape[0], fmt).upload(t)


def _tag(fmt):
    return fmt if fmt in (BGRA8, RGB10A2, BGRX8) else None


def _codes(a, fmt):
    from openvr_fsr_b200 import synth
    return synth.unpack_rgb10a2(a) if fmt == RGB10A2 else a.astype(np.int32)


def _compare(got, want, mode, fmt, composed=False):
    if mode == "strict" or fmt == "f32":
        assert got.shape == want.shape
        bad = int((np.ascontiguousarray(got).view(np.uint8) != np.ascontiguousarray(want).view(np.uint8)).sum())
        assert bad == 0, f"{bad} bytes differ from the oracle"
        return
    d = np.abs(_codes(got, fmt) - _codes(want, fmt))
    if composed:
        assert d.max() <= 4 and (d > 1).mean() < 1e-4, f"fast composed: max {d.max()}, {(d > 1).mean():.2e} beyond 1"
    else:
        assert d.max() <= 1, f"fast: max {d.max()} LSB"


FORMATS = [RGBA8, BGRA8, BGRX8, RGB10A2]
PLACES = ["tma", "tight", "array"]
SCALES = [0.75, 0.5, 0.9]


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("where", PLACES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_easu_flat_groups_plain_dispatch(cuda, fmt, where, scale, mode):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    mm = ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST
    ow, oh = ovr.output_size(W, H, scale)
    out_fmt = RGB10A2 if fmt == RGB10A2 else RGBA8
    for radius, proj in ((2.0, (0.5, 0.5, 0.5, 0.5)), (RADIUS, PROJ)):
        uc = po.upscale_constants(0, True, W, H, ow, oh, proj=proj, radius=radius)
        words = uc.words()
        src = _fixture(fmt, words, ow, oh, seed=int(scale * 100) + fmt)
        flat, filt, outside = _classify(src, fmt, words, ow, oh)
        assert flat >= 2 and filt >= 2, f"fixture exercises {flat} one-colour and {filt} filtered inside groups"
        assert (outside > 0) == (radius < 2.0)
        s = _place(src, fmt, where, cuda)
        sfmt = None if where == "array" else _tag(fmt)
        want = po.easu(src, ow, oh, uc, src_fmt=_tag(fmt), dst_fmt=_tag(out_fmt))
        if where == "array":
            d = ovr.ArrayImage(ow, oh, out_fmt)
            ovr.fsr_easu(s, d, words, mm, src_fmt=sfmt)
            got = d.download().cpu().numpy()
        else:
            d = ovr.alloc_image(ow, oh, torch.uint8, cuda)
            ovr.fsr_easu(s, d, words, mm, src_fmt=sfmt, dst_fmt=_tag(out_fmt))
            torch.cuda.synchronize()
            got = d.cpu().numpy()
        _compare(got, want, mode, out_fmt)
        if mode == "strict" and where == "tma":
            # FP32 output: the stored one-colour pixels are f itself, before any quantisation
            d32 = ovr.alloc_image(ow, oh, torch.float32, cuda)
            ovr.fsr_easu(s, d32, words, mm, src_fmt=sfmt)
            torch.cuda.synchronize()
            want32 = po.easu(src, ow, oh, uc, out_dtype=np.float32, src_fmt=_tag(fmt))
            _compare(d32.cpu().numpy(), want32, mode, "f32")


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_easu_one_colour_image(cuda, fmt, mode):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    mm = ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST
    ow, oh = ovr.output_size(W, H, 0.75)
    out_fmt = RGB10A2 if fmt == RGB10A2 else RGBA8
    uc = po.upscale_constants(0, True, W, H, ow, oh, radius=2.0)
    src = _fixture(fmt, uc.words(), ow, oh, seed=7 + fmt, whole=True)
    assert _classify(src, fmt, uc.words(), ow, oh)[1:] == (0, 0)
    d = ovr.alloc_image(ow, oh, torch.uint8, cuda)
    ovr.fsr_easu(ovr.to_image(src, cuda), d, uc.words(), mm, src_fmt=_tag(fmt), dst_fmt=_tag(out_fmt))
    torch.cuda.synchronize()
    want = po.easu(src, ow, oh, uc, src_fmt=_tag(fmt), dst_fmt=_tag(out_fmt))
    _compare(d.cpu().numpy(), want, mode, out_fmt)


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("where", PLACES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_easu_flat_groups_paired(cuda, fmt, where, mode):
    """the context path: paired EASU (outside groups straight to the final image) + RCAS, both eyes"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    mm = ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST
    ow, oh = ovr.output_size(W, H, 0.75)
    unorm = RGB10A2 if fmt == RGB10A2 else RGBA8
    eyes, consts = [], []
    for e in (0, 1):
        uc = po.upscale_constants(e, True, W, H, ow, oh, proj=PROJ, radius=RADIUS)
        src = _fixture(fmt, uc.words(), ow, oh, seed=20 + 3 * e + fmt)
        flat, filt, outside = _classify(src, fmt, uc.words(), ow, oh)
        assert flat >= 2 and filt >= 2 and outside > 0, f"eye {e}: {flat} one-colour, {filt} filtered, {outside} outside groups"
        eyes.append(src)
        consts.append(uc)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=0.75, sharpness=0.8, radius=RADIUS, projCentre=PROJ,
                                      mathMode=mm))
    srcs = [_place(e, fmt, where, cuda) for e in eyes]
    if where == "array":
        dsts = [ovr.ArrayImage(ow, oh, unorm) for _ in (0, 1)]
        pp.apply_pair_into(srcs[0], srcs[1], dsts[0], dsts[1])
        got = [d.download().cpu().numpy() for d in dsts]
    else:
        got = [t.cpu().numpy() for t in pp.apply_pair(srcs[0], srcs[1], fmt=_tag(fmt))]
    torch.cuda.synchronize()
    pp.close()
    for e in (0, 1):
        sc = po.sharpen_constants(e, True, ow, oh, proj=PROJ, radius=RADIUS, sharpness=0.8)
        mid = po.easu(eyes[e], ow, oh, consts[e], src_fmt=_tag(fmt), dst_fmt=_tag(unorm))
        want = po.rcas(mid, sc, src_fmt=_tag(unorm), dst_fmt=_tag(unorm))
        _compare(got[e], want, mode, unorm, composed=True)
