"""The checker contains a non-finite texel: one +inf, -inf or NaN changes only the outputs whose footprint reads it.

A finite field gets one +inf, -inf or NaN texel, in one colour channel or in all three, at an interior texel, on an
image edge, at a corner and at the texels where 64 x 32 output tiles meet.  Every restated pass (EASU filtered and its
bilinear copy, RCAS filtered and copied, NVScaler and NVSharpen inside and outside the radius, CAS sharpen and upscale)
then runs on the field with and without it, and the outputs whose bits change (a NaN counts as one value) must all be
outputs whose source footprint holds that texel.  The footprints are the per-kernel source positions restated in
tests/test_resample_footprint_host.py: EASU's 4x4 window at floor(pos) - 1 .. + 2 and its bilinear taps, RCAS's cross,
NVScaler's 6x6 window and chroma tap, CAS's 3x3 (the upscale's f - 1 .. f + 2), clamped to the image where the pass
clamps.  That the change is not empty, and the footprint not the whole image, shows the bound is neither too small nor
vacuous; this is what the GPU containment check of tests/test_gpu_float_nonfinite.py measures fast math against."""
import numpy as np
import pytest

from tests import test_resample_footprint_host as fp

F = np.float32
W, H, SCALE = 97, 41, 0.75
U32 = 0xFFFFFFFF


def _field():
    from openvr_fsr_b200 import synth
    return (synth.natural_rgba8(W, H, 17).astype(F) / F(200.0) - F(0.1)).astype(F)


def _everywhere(consts, inside):
    """the same constants with every group inside (R^2 = 2^32 - 1) or outside (centres (0, 0), R^2 = 0)"""
    for i in range(4):
        consts.imageCentre[i] = 0
    consts.radius[1] = U32 if inside else 0
    return consts


def _c0(words):
    return np.array(words, dtype=np.uint32).view(F)


def _span(lo, hi, n, clamp):
    """per-pixel tap interval [lo, hi] as the pass reads it: clamped to the image (Gather / SampleLevel) or not (Load)"""
    return (fp.clampi(lo, 0, n - 1), fp.clampi(hi, 0, n - 1)) if clamp else (lo, hi)


def _box(sx, sy, tx, ty):
    """(oh, ow): the outputs whose x interval sx holds tx and y interval sy holds ty"""
    return ((sy[0] <= ty) & (ty <= sy[1]))[:, None] & ((sx[0] <= tx) & (tx <= sx[1]))[None, :]


def _passes():
    """{name: (run(src) -> float32 output, footprint(tx, ty) -> (oh, ow) bool)}"""
    from oracle import pyoracle as po
    ow, oh = po.output_size(W, H, SCALE)
    px, py = np.arange(ow), np.arange(oh)
    out = {}
    for inside in (True, False):
        tag = "filter" if inside else "copy"
        uc = _everywhere(po.upscale_constants(0, True, W, H, ow, oh, radius=0.5), inside)
        c0 = _c0(uc.const0)
        if inside:  # fsr_kernels.cuh: 12 taps within floor(pos) - 1 .. floor(pos) + 2 of each axis
            fx, fy = fp.ifloor(fp.easu_pos(px, c0[0], c0[2])), fp.ifloor(fp.easu_pos(py, c0[1], c0[3]))
            sx, sy = _span(fx - 1, fx + 2, W, True), _span(fy - 1, fy + 2, H, True)
        else:       # the bilinear copy: taps b0, b0 + 1 of the snapped position
            bx = fp._bilinear_taps(px, F(uc.radius[2]), np.int64(W))
            by = fp._bilinear_taps(py, F(uc.radius[3]), np.int64(H))
            sx, sy = _span(bx, bx + 1, W, True), _span(by, by + 1, H, True)
        out[f"easu {tag}"] = (lambda s, uc=uc: po.easu(s, ow, oh, uc, out_dtype=F),
                              lambda tx, ty, sx=sx, sy=sy: _box(sx, sy, tx, ty))
        sc = _everywhere(po.sharpen_constants(0, True, W, H, radius=0.5, sharpness=0.8), inside)
        qx, qy = np.arange(W), np.arange(H)

        def cross(tx, ty, qx=qx, qy=qy):  # Texture2D.Load of the cross, zeros outside the image
            dx, dy = tx - qx[None, :], ty - qy[:, None]
            return (np.abs(dx) + np.abs(dy)) <= 1
        out[f"rcas {tag}"] = (lambda s, sc=sc: po.rcas(s, sc, out_dtype=F), cross)
        for sharpen in (False, True):
            nw, nh = (W, H) if sharpen else (ow, oh)
            cfg, ok = po.nis_config(sharpen, 0, True, W, H, nw, nh, radius=0.5, sharpness=0.8)
            assert ok
            cfg = _everywhere(cfg, inside)
            nx, ny = np.arange(nw), np.arange(nh)
            wx, wy = fp.ifloor(fp.nis_pos(nx, F(cfg.kScaleX))), fp.ifloor(fp.nis_pos(ny, F(cfg.kScaleY)))
            win = (_span(wx - 2, wx + 3, W, True), _span(wy - 2, wy + 3, H, True))
            cx = fp.ifloor(fp.snap_subtexel(fp.mul_add_unfused((nx.astype(F) + F(0.5)) * F(cfg.kDstNormX), F(W), F(-0.5))))
            cy = fp.ifloor(fp.snap_subtexel(fp.mul_add_unfused((ny.astype(F) + F(0.5)) * F(cfg.kDstNormY), F(H), F(-0.5))))
            chroma = (_span(cx, cx + 1, W, True), _span(cy, cy + 1, H, True))
            run = (lambda s, cfg=cfg: po.nis_sharpen(s, cfg, out_dtype=F)) if sharpen else \
                (lambda s, cfg=cfg: po.nis_scaler(s, ow, oh, cfg, out_dtype=F))
            out[f"{'nis sharpen' if sharpen else 'nis scaler'} {tag}"] = (
                run, lambda tx, ty, win=win, chroma=chroma: _box(*win, tx, ty) | _box(*chroma, tx, ty))
    kc = po.cas_setup(0.8, 1.0, W, H, W, H)
    qx, qy = np.arange(W), np.arange(H)
    out["cas sharpen"] = (lambda s: po.cas(s, W, H, kc, True, out_dtype=F),
                          lambda tx, ty: _box(_span(qx - 1, qx + 1, W, True), _span(qy - 1, qy + 1, H, True), tx, ty))
    ku = po.cas_setup(0.8, 1.0, W, H, ow, oh)
    k0 = _c0(ku.const0)
    fx, fy = fp.ifloor(fp.easu_pos(px, k0[0], k0[2])), fp.ifloor(fp.easu_pos(py, k0[1], k0[3]))
    out["cas upscale"] = (lambda s: po.cas(s, ow, oh, ku, False, out_dtype=F),
                          lambda tx, ty: _box(_span(fx - 1, fx + 2, W, True), _span(fy - 1, fy + 2, H, True), tx, ty))
    return out


def _places():
    """interior, edges, corners, and the source texels the first 64 x 32 output tile boundary maps to"""
    from oracle import pyoracle as po
    ow, oh = po.output_size(W, H, SCALE)
    c0 = _c0(po.upscale_constants(0, True, W, H, ow, oh).const0)
    bx, by = int(fp.ifloor(fp.easu_pos(64, c0[0], c0[2]))), int(fp.ifloor(fp.easu_pos(32, c0[1], c0[3])))
    return {"interior": (W // 3, H // 2), "left edge": (0, H // 2), "bottom edge": (W // 2, H - 1), "corner": (W - 1, 0),
            "tile x": (bx, H // 3), "tile x+1": (bx + 1, H // 3), "tile y": (W // 4, by), "tile xy": (bx, by)}


def _changed(a, b):
    """outputs any of whose words differ in bits, every NaN one value"""
    same = (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    return ~same.all(axis=-1)


@pytest.fixture(scope="module")
def passes():
    return _passes()


@pytest.mark.parametrize("name", ["easu filter", "easu copy", "rcas filter", "rcas copy", "nis scaler filter",
                                  "nis scaler copy", "nis sharpen filter", "nis sharpen copy", "cas sharpen",
                                  "cas upscale"])
def test_one_nonfinite_texel_stays_in_its_footprint(passes, name):
    run, footprint = passes[name]
    field = _field()
    base = run(field)
    assert np.isfinite(base).all()
    bad, reached = [], 0
    with np.errstate(invalid="ignore"):
        for where, (tx, ty) in _places().items():
            fpm = footprint(tx, ty)
            assert fpm.any() and fpm.sum() <= 64, (where, int(fpm.sum()))
            for value in (np.inf, -np.inf, np.nan):
                for channels in (slice(0, 1), slice(0, 3)):
                    src = field.copy()
                    src[ty, tx, channels] = value
                    ch = _changed(run(src), base)
                    reached += int(ch.any())
                    if (ch & ~fpm).any():
                        y, x = np.argwhere(ch & ~fpm)[0]
                        bad.append(f"{value} in {channels} at {where} ({tx}, {ty}) changed output ({x}, {y}), outside "
                                   f"its footprint ({int((ch & ~fpm).sum())} such outputs)")
    assert not bad, "\n".join(bad)
    assert reached, f"{name}: no non-finite texel changed any output"
