"""The checker's side of OVRFSR_FLAG_SRTM: AMD's simple reversible tone mapper (ffx_fsr1.h, FsrSrtmF / FsrSrtmInvF)
around the unchanged restated FSR passes of oracle/pyoracle.py.  TEST INFRASTRUCTURE ONLY.

    F(c) = c * rcp(max3(c.rgb) + 1)                     FsrSrtmF:    {0 .. FP16_MAX} -> {0 .. 1}
    G(c) = c * rcp(max(1/32768, 1 - max3(c.rgb)))       FsrSrtmInvF: back, with a peak of 32768

Both in binary32 (numpy float32 arithmetic: IEEE add, IEEE divide for the true reciprocal, IEEE multiply), alpha
untouched.  max3 is max(max(r, g), b) under the pinned min / max rule (oracle/ovr_glue.h: NaN ignored, -0 < +0); np.fmax
ignores NaN the same way, and the sign of a zero maximum cannot reach the result (m + 1 and 1 - m are the same for +-0).
Inputs outside the map's domain (negative, NaN, +-inf, max3 <= -1) simply go through the formula.

A pass with the tone map is the plain oracle pass between the maps: F on every decoded source texel (the decode is exact
into binary32, so the mapped RGBA32F copy is what the pass reads; RCAS's out-of-image zeros need no map, F(+0) = +0), the
pass into RGBA32F (exact), G, then the target's encode -- done by the oracle's own store, through its RCAS copy path with
every group outside the radius and no tint (OutputTexture = 1 x InputTexture)."""
from __future__ import annotations

import numpy as np

from oracle import pyoracle as po

_ONE = np.float32(1.0)
_FLOOR = np.float32(1.0 / 32768.0)


def srtm(rgb, inverse=False) -> np.ndarray:
    """FsrSrtmF (inverse=False) / FsrSrtmInvF on the last axis (3 channels) of an array, in binary32"""
    c = np.array(rgb, dtype=np.float32)
    assert c.shape[-1] == 3
    m = np.fmax(np.fmax(c[..., 0], c[..., 1]), c[..., 2])
    with np.errstate(all="ignore"):
        k = _ONE / (np.fmax(_FLOOR, _ONE - m) if inverse else m + _ONE)
        return (c * k[..., None]).astype(np.float32)


def _map_rgb(img32, inverse):
    out = img32.copy()
    out[..., :3] = srtm(img32[..., :3], inverse)
    return out


def _float_source(src):
    if src.dtype not in (np.float16, np.float32):
        raise ValueError("the tone map is defined for float sources only (UNORM sources are display-referred)")
    return src.astype(np.float32)  # binary16 -> binary32 is exact, as the kernels' and the oracle's decodes


def encode(img32, out_dtype, dst_fmt=None):
    """the oracle's store of an RGBA32F image into out_dtype (uint8: RGBA8, float16: RGBA16F): its RCAS copy path"""
    if np.dtype(out_dtype) == np.float32 and dst_fmt is None:
        return img32.copy()
    h, w = img32.shape[:2]
    c = po.SharpenConstants()
    c.const0[0] = int(np.float32(1.0).view(np.uint32))
    # odd centres: centre - (16 g + 8) is odd, so its square is never 0 mod 2^32 and no group is inside radius^2 = 0
    c.imageCentre[:] = [1, 1, 1, 1]
    c.radius[:] = [0, 0, w, h]
    return po.rcas(np.ascontiguousarray(img32), c, out_dtype=out_dtype, dst_fmt=dst_fmt)


def easu(src, out_w, out_h, consts, out_dtype=np.uint8, srtm_in=False, srtm_out=False, nthreads=1, dst_fmt=None):
    """the restated EASU with F on its texels read (srtm_in) and G on its pixels stored (srtm_out)"""
    s = _float_source(src)
    if srtm_in:
        s = _map_rgb(s, False)
    o = po.easu(np.ascontiguousarray(s), out_w, out_h, consts, out_dtype=np.float32, nthreads=nthreads)
    if srtm_out:
        o = _map_rgb(o, True)
    return encode(o, out_dtype, dst_fmt)


def rcas(src, consts, out_dtype=np.uint8, srtm_in=False, srtm_out=False, nthreads=1, dst_fmt=None):
    """the restated RCAS with F on its texels read (srtm_in) and G on its pixels stored (srtm_out)"""
    s = _float_source(src)
    if srtm_in:
        s = _map_rgb(s, False)
    o = po.rcas(np.ascontiguousarray(s), consts, out_dtype=np.float32, nthreads=nthreads)
    if srtm_out:
        o = _map_rgb(o, True)
    return encode(o, out_dtype, dst_fmt)
