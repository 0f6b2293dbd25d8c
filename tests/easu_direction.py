"""EASU's direction test, restated, and content that sits on its threshold.

FsrEasuF (ffx_fsr1.h:389-395; oracle/fsr_oracle.c:202-209) normalises the blended direction with a branch:

    zro = dir.x^2 + dir.y^2 < 1/32768      zro: dir = (1, dir.y), else dir / |dir|

so a pixel whose dir^2 sits within an ulp or two of 2^-15 turns its anisotropic kernel by up to 90 degrees on a
last-bit difference in how dir^2 was computed.  Random content almost never lands there; the generators below put a
large share of the output pixels within a few ulps of it on purpose, and `easu` restates the oracle's easu_pixel in
numpy float32 (every operation rounded on its own, as `-ffp-contract=off` compiles the oracle) so that a test can
count, per pixel, how far dir^2 is from the threshold and which branch the oracle took.  tests/test_easu_direction_host.py
holds the restatement to the oracle bit for bit, which is what makes its dir^2 trustworthy.

Content is finite and >= 0 here, so min / max are numpy's (the oracle's HLSL rule differs only at NaN and signed zeros).
"""
from __future__ import annotations

import numpy as np

from openvr_fsr_b200 import synth

F = np.float32
RGBA8, BGRA8, RGBA16F, RGBA32F, RGB10A2, BGRX8 = 0, 1, 2, 3, 4, 5
THRESHOLD = F(1.0 / 32768.0)
_T_BITS = int(THRESHOLD.view(np.int32))


def _f(u):
    return np.array([u], dtype=np.uint32).view(np.float32)[0]


def prx_lo_rcp(a):
    """ffx_a.h APrxLoRcpF1: 0x7ef07ebb - bits(a)"""
    return (np.uint32(0x7ef07ebb) - a.view(np.uint32)).view(np.float32)


def prx_lo_rsq(a):
    """ffx_a.h APrxLoRsqF1: 0x5f347d74 - (bits(a) >> 1)"""
    return (np.uint32(0x5f347d74) - (a.view(np.uint32) >> np.uint32(1))).view(np.float32)


def decode(src, fmt):
    """(H, W, 4) source of API format fmt -> float32 rgba as ovo_texel reads it (UNORM: v / 255 or v / 1023 rounded
    once; FP16: exact)"""
    if fmt == RGBA32F:
        return src.astype(F)
    if fmt == RGBA16F:
        return src.astype(F)
    if fmt == RGB10A2:
        c = synth.unpack_rgb10a2(src).astype(F)
        return np.concatenate([c[..., :3] / F(1023.0), c[..., 3:] / F(3.0)], axis=-1)
    c = src.astype(F) / F(255.0)
    if fmt in (BGRA8, BGRX8):
        c = c[..., [2, 1, 0, 3]]
    return c


def ulps_from_threshold(dir2):
    """signed distance of each dir^2 (>= +0) from 2^-15, in ulps: 0 is the threshold itself, -1 the float below it"""
    return dir2.astype(F).view(np.int32).astype(np.int64) - _T_BITS


def easu(src, fmt, words, ow, oh):
    """FsrEasuF at every output pixel, every group taken as inside the radius (oracle/fsr_oracle.c:166-243).
    Returns (rgb float32 (oh, ow, 3), dir^2 float32 (oh, ow), zro bool (oh, ow))."""
    t = decode(src, fmt)
    h, w = t.shape[:2]
    c0 = [_f(int(words[i])) for i in range(4)]
    ppx = np.arange(ow, dtype=np.uint32).astype(F) * c0[0] + c0[2]
    ppy = np.arange(oh, dtype=np.uint32).astype(F) * c0[1] + c0[3]
    fpx, fpy = np.floor(ppx), np.floor(ppy)
    ppx, ppy = ppx - fpx, ppy - fpy
    ix, iy = fpx.astype(np.int64), fpy.astype(np.int64)
    ppx, ppy = np.broadcast_to(ppx[None, :], (oh, ow)), np.broadcast_to(ppy[:, None], (oh, ow))

    def tex(dx, dy):
        ys = np.clip(iy + dy, 0, h - 1)
        xs = np.clip(ix + dx, 0, w - 1)
        return t[ys[:, None], xs[None, :], :3]

    b, c, e, f, g, hh = tex(0, -1), tex(1, -1), tex(-1, 0), tex(0, 0), tex(1, 0), tex(2, 0)
    i, j, k, l, n, o = tex(-1, 1), tex(0, 1), tex(1, 1), tex(2, 1), tex(0, 2), tex(1, 2)

    def luma2(q):
        return q[..., 2] * F(0.5) + (q[..., 0] * F(0.5) + q[..., 1])

    bL, cL, eL, fL, gL, hL = map(luma2, (b, c, e, f, g, hh))
    iL, jL, kL, lL, nL, oL = map(luma2, (i, j, k, l, n, o))

    one = F(1.0)
    dirx = np.zeros((oh, ow), F)
    diry = np.zeros((oh, ow), F)
    ln = np.zeros((oh, ow), F)
    for wt, lA, lB, lC, lD, lE in (((one - ppx) * (one - ppy), bL, eL, fL, gL, jL),
                                   (ppx * (one - ppy), cL, fL, gL, hL, kL),
                                   ((one - ppx) * ppy, fL, iL, jL, kL, nL),
                                   (ppx * ppy, gL, jL, kL, lL, oL)):
        # FsrEasuSetF (fsr_oracle.c:121-138)
        dc, cb = lD - lC, lC - lB
        lenX = prx_lo_rcp(np.maximum(np.abs(dc), np.abs(cb)))
        dX = lD - lB
        dirx = dirx + dX * wt
        lenX = np.minimum(one, np.maximum(F(0.0), np.abs(dX) * lenX))
        lenX = lenX * lenX
        ln = ln + lenX * wt
        ec, ca = lE - lC, lC - lA
        lenY = prx_lo_rcp(np.maximum(np.abs(ec), np.abs(ca)))
        dY = lE - lA
        diry = diry + dY * wt
        lenY = np.minimum(one, np.maximum(F(0.0), np.abs(dY) * lenY))
        lenY = lenY * lenY
        ln = ln + lenY * wt

    dir2 = dirx * dirx + diry * diry
    zro = dir2 < THRESHOLD
    dirR = np.where(zro, one, prx_lo_rsq(dir2))
    dirx = np.where(zro, one, dirx) * dirR
    diry = diry * dirR
    ln = ln * F(0.5)
    ln = ln * ln
    stretch = (dirx * dirx + diry * diry) * prx_lo_rcp(np.maximum(np.abs(dirx), np.abs(diry)))
    len0 = one + (stretch - one) * ln
    len1 = one + F(-0.5) * ln
    lob = F(0.5) + F((1.0 / 4.0 - 0.04) - 0.5) * ln
    clp = prx_lo_rcp(lob)

    aC = np.zeros((oh, ow, 3), F)
    aW = np.zeros((oh, ow), F)
    for ox, oy, q in ((0, -1, b), (1, -1, c), (-1, 1, i), (0, 1, j), (0, 0, f), (-1, 0, e),
                      (1, 1, k), (2, 1, l), (2, 0, hh), (1, 0, g), (1, 2, o), (0, 2, n)):
        offx, offy = F(ox) - ppx, F(oy) - ppy
        vx = offx * dirx + offy * diry
        vy = offx * (-diry) + offy * dirx
        vx = vx * len0
        vy = vy * len1
        d2 = np.minimum(vx * vx + vy * vy, clp)
        wB = F(2.0 / 5.0) * d2 + F(-1.0)
        wA = lob * d2 + F(-1.0)
        wB = wB * wB
        wA = wA * wA
        wB = F(25.0 / 16.0) * wB + F(-(25.0 / 16.0 - 1.0))
        wq = wB * wA
        aC = aC + q * wq[..., None]
        aW = aW + wq
    r = one / aW
    mn = np.minimum(np.minimum(f, np.minimum(g, j)), k)
    mx = np.maximum(np.maximum(f, np.maximum(g, j)), k)
    pix = np.minimum(mx, np.maximum(mn, aC * r[..., None]))
    return pix, dir2, zro


def near_threshold(dir2, zro, within=2):
    """(pixels within +-`within` ulps of 2^-15, of which the oracle took zro, of which it did not)"""
    near = np.abs(ulps_from_threshold(dir2)) <= within
    return int(near.sum()), int((near & zro).sum()), int((near & ~zro).sum())


# ---- content --------------------------------------------------------------------------------------------------------
# Float sources.  Every value is a multiple of 2^-29 below 2^-5 (R and B: of 2^-28), so the luma sum
# B*0.5 + (R*0.5 + G) and every luma difference is exact: luma is exactly c + G(y) whatever the chroma does, dir.x is
# exactly 0, and each feature's dir.y = lE - lA is exactly D = K * 2^-29.  K = 2965821 puts D 0.8 ulp above
# fl(2^-7.5), so fl(D^2) is about 2 ulps above 2^-15, and the rounding of the four-term blend (weights summing to 1
# within an ulp or two) spreads the pixels' dir^2 over a few ulps on both sides of the threshold.  G rises by D over
# every two rows, in steps that alternate between floor(K/2) and ceil(K/2) units, so lE - lC and lC - lA are both
# about D/2: lenY saturates, lenX is 0 and the kernel is as anisotropic as EASU makes it.  The ramp restarts every
# PERIOD rows (to stay below 2^-5); the features whose cross spans a restart are far from the threshold.
Q = 2.0 ** -29
K_STEP = 2965821
PERIOD = 8
CHROMA_C = 2.0 ** -7


def float_ramp(w, h, fmt, seed, k=K_STEP):
    """iso-luminant chroma texture over a luma ramp along y whose per-feature dir^2 sits on 2^-15 (RGBA32F); for
    RGBA16F the same recipe rounded to half, whose coarser grid spreads the features over a wider band around it"""
    rng = np.random.default_rng(seed)
    i = np.arange(h) % PERIOD
    g = ((i // 2) * k + (i % 2) * (k // 2)) * Q
    c = CHROMA_C
    # chroma: R = c + t, B = c - t, t a multiple of 2^-28 in [-c, c), in 1-3 texel cells along both axes
    cells = rng.integers(-(1 << 21), 1 << 21, (h + 3, w + 3))
    cy = np.cumsum(rng.integers(1, 3, h + 2))[:h] // 2
    cx = np.cumsum(rng.integers(1, 3, w + 2))[:w] // 2
    tch = cells[cy[:, None], cx[None, :]] * 2.0 ** -28
    img = np.empty((h, w, 4), np.float64)
    img[..., 0] = c + tch
    img[..., 1] = g[:, None]
    img[..., 2] = c - tch
    img[..., 3] = 1.0
    return img.astype(np.float16 if fmt == RGBA16F else np.float32)


# UNORM sources.  2-D cells of two colours that differ by (+k+1, +1, -k) codes in 8 bits (x4 in 10 bits): the luma
# step is 1.5 codes (0.0059, dir^2 = 3.5e-5 at an edge feature), so blends of edge and flat features sweep dir^2
# through 2^-15 while R and B swing hard -- a branch flip there moves the output by many codes.
def unorm_cells(w, h, fmt, seed, k):
    rng = np.random.default_rng(seed)
    unit = 4 if fmt == RGB10A2 else 1
    top = 1023 if fmt == RGB10A2 else 255
    step = np.array([k + 1, 1, -k]) * unit
    base = np.array([rng.integers(0, top - step[0] - 2 * unit), rng.integers(2 * unit, top - 2 * unit),
                     rng.integers(-step[2] + 2 * unit, top)])
    # cell edges at irregular spacings (1-4 texels) in both axes, two colours in a random pattern
    ey = np.cumsum(rng.integers(1, 5, h + 4))
    ex = np.cumsum(rng.integers(1, 5, w + 4))
    rows = np.searchsorted(ey, np.arange(h), side="right")
    cols = np.searchsorted(ex, np.arange(w), side="right")
    pick = rng.integers(0, 2, (rows.max() + 1, cols.max() + 1))[rows[:, None], cols[None, :]]
    rgb = base[None, None, :] + pick[..., None] * step[None, None, :]
    return _pack(rgb, fmt)


def flat_luma(w, h, fmt, seed):
    """luma equal up to its last bits under hard chroma edges: G fixed, R + B fixed, R random per 1-3 texel cell, so
    every luma difference EASU's features divide by each other is decode rounding (DESIGN.md §3's decode lesson)"""
    rng = np.random.default_rng(seed)
    top = 1023 if fmt == RGB10A2 else 255
    cells = rng.integers(0, top + 1, (h + 3, w + 3))
    cy = np.cumsum(rng.integers(1, 3, h + 2))[:h] // 2
    cx = np.cumsum(rng.integers(1, 3, w + 2))[:w] // 2
    r = cells[cy[:, None], cx[None, :]]
    rgb = np.stack([r, np.full_like(r, top // 3), top - r], axis=-1)
    return _pack(rgb, fmt)


def _pack(rgb, fmt):
    h, w = rgb.shape[:2]
    if fmt == RGB10A2:
        return synth.pack_rgb10a2(rgb, np.full((h, w), 3))
    out = np.empty((h, w, 4), np.uint8)
    out[..., :3] = rgb[..., ::-1] if fmt in (BGRA8, BGRX8) else rgb
    out[..., 3] = 255
    return out


# The cases: (name, source format, in w, in h, render scale, seed, generator, UNORM step k, near-threshold minimum).
# Sizes are non-round; render scale 0.77 takes EASU's 60-column tile, 0.9 the 72-column one.  min_near is the number
# of pixels whose dir^2 is within 2 ulps of 2^-15 that each case promises (tests/test_easu_direction_host.py), set a
# little under the count measured with `easu`: 16599 and 8820 for the two FP32 ramps, 3 for the FP16 one, whose
# 11-bit texels cannot hold a feature's dir.y to the last bit.  The UNORM cases promise none: a UNORM luma difference
# is a multiple of 1/510 (1/2046) plus decode rounding, so no edge puts dir.y within an ulp of 2^-7.5, and blends of
# edge and flat features reach the 2-ulp band only by coincidence (none in 2-D iso-luminant cells at these sizes).
# They still cross the threshold in both directions, and `flat` is the decode lesson's content.
CASES = {
    # name: (fmt, iw, ih, scale, seed, kind, k, min_near)
    "ramp_f32_s077": (RGBA32F, 157, 113, 0.77, 3, "ramp", 0, 15000),
    "ramp_f32_s090": (RGBA32F, 131, 97, 0.9, 4, "ramp", 0, 8000),
    "ramp_f16_s077": (RGBA16F, 157, 113, 0.77, 5, "ramp", 0, 2),
    "cells_rgba8_s077": (RGBA8, 157, 113, 0.77, 6, "cells", 3, 0),
    "cells_bgra8_s090": (BGRA8, 131, 97, 0.9, 7, "cells", 5, 0),
    "cells_rgb10a2_s077": (RGB10A2, 157, 113, 0.77, 8, "cells", 2, 0),
    "flat_rgba8_s077": (RGBA8, 157, 113, 0.77, 9, "flat", 0, 0),
    "flat_rgb10a2_s090": (RGB10A2, 131, 97, 0.9, 10, "flat", 0, 0),
}


def case_source(name):
    """(H, W, 4) source array of case `name`"""
    fmt, iw, ih, scale, seed, kind, k, _ = CASES[name]
    if kind == "ramp":
        return float_ramp(iw, ih, fmt, seed)
    if kind == "cells":
        return unorm_cells(iw, ih, fmt, seed, k)
    return flat_luma(iw, ih, fmt, seed)
