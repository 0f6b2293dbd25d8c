"""The checker's side of OVRFSR_FLAG_PERCEPTUAL: the gamma-2.0 maps and the sRGB encode around the unchanged restated
passes of oracle/pyoracle.py, composed with the maps of OVRFSR_FLAG_SRTM (tests/srtm_oracle.py) and OVRFSR_FLAG_FINITE
(tests/finite_rule.py).  TEST INFRASTRUCTURE ONLY.

    P(c)   = copysign(sqrt(|c|), c)      on R, G, B of every texel a pass reads
    P^-1(c) = c * |c|                     on R, G, B of every pixel a pass stores
    code(v) = #{k in 1..255 : v >= T[k]}  the sRGB encode of an RGBA8 store with perceptual-out (NaN, v <= 0 -> 0)

sqrt and the product are correctly rounded binary32 operations in numpy as on the device.  T is the committed table
(openvr_fsr_b200/csrc/srgb_table.inc), which tests/test_perceptual_host.py holds to a fresh decimal generation and to a
float64 sRGB encode.

A pass with bits is the plain oracle pass between the maps: read = finite-in, F, P on every decoded source texel (the
decode is exact into binary32, so the mapped RGBA32F copy is what the pass reads; RCAS's out-of-image zeros need no map,
F(+0) = P(+0) = +0), the pass into RGBA32F (exact), then store = P^-1, G, and finite-out or the target's encode.  The
encode is the oracle's own store (srtm_oracle.encode); an RGBA8 target with perceptual-out takes code() on R, G and B
and the oracle's UNORM alpha.  With no bits this gives the plain oracle's bytes."""
from __future__ import annotations

import re
from pathlib import Path

import numpy as np

from oracle import pyoracle as po
from tests import finite_rule as fr
from tests import srtm_oracle as so

ROOT = Path(__file__).resolve().parents[1]
# the plain passes, taken before any test replaces the module's names with the wrappers below
_EASU, _RCAS, _NIS_SCALER, _NIS_SHARPEN = po.easu, po.rcas, po.nis_scaler, po.nis_sharpen
TABLE_INC = ROOT / "openvr_fsr_b200" / "csrc" / "srgb_table.inc"

# OVRFSR_PASS_* (include/ovrfsr.h)
SRTM_IN, SRTM_OUT, FINITE_IN, FINITE_OUT, PERCEPTUAL_IN, PERCEPTUAL_OUT = 1, 2, 16, 32, 128, 512
READ_BITS = SRTM_IN | FINITE_IN | PERCEPTUAL_IN
STORE_BITS = SRTM_OUT | FINITE_OUT | PERCEPTUAL_OUT


def table_words() -> np.ndarray:
    """the 256 committed thresholds as binary32 bit patterns"""
    words = re.findall(r"0x([0-9a-f]{8})u", TABLE_INC.read_text())
    assert len(words) == 256, len(words)
    return np.array([int(w, 16) for w in words], dtype=np.uint32)


_T = table_words().view(np.float32)


def p_fwd(c):
    c = np.asarray(c, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        return np.copysign(np.sqrt(np.abs(c)), c).astype(np.float32)


def p_inv(c):
    c = np.asarray(c, dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        return (c * np.abs(c)).astype(np.float32)


def srgb_code(v) -> np.ndarray:
    """the encode of linear binary32 values: the number of thresholds T[1..255] at or below v; NaN -> 0"""
    v = np.asarray(v, dtype=np.float32)
    k = np.searchsorted(_T[1:], np.where(np.isnan(v), np.float32(0), v), side="right")
    return k.astype(np.uint8)


def read_map(img32, bits):
    """finite-in, F, P on the channels each takes (img32: RGBA32F)"""
    out = np.array(img32, dtype=np.float32)
    if bits & FINITE_IN:
        out = fr.finite_in(out)
    if bits & SRTM_IN:
        out[..., :3] = so.srtm(out[..., :3])
    if bits & PERCEPTUAL_IN:
        out[..., :3] = p_fwd(out[..., :3])
    return out


def store(img32, bits, out_dtype, dst_fmt=None):
    """P^-1, G, then finite-out or the target's encode, of an RGBA32F pass result"""
    o = np.array(img32, dtype=np.float32)
    if bits & PERCEPTUAL_OUT:
        o[..., :3] = p_inv(o[..., :3])
    if bits & SRTM_OUT:
        o[..., :3] = so.srtm(o[..., :3], inverse=True)
    enc = _encode(o, out_dtype, dst_fmt)
    if enc.dtype == np.uint8:
        if bits & PERCEPTUAL_OUT:
            enc[..., :3] = srgb_code(o[..., :3])
        return enc
    return fr.finite_out(enc) if bits & FINITE_OUT else enc


def _encode(img32, out_dtype, dst_fmt=None):
    """srtm_oracle.encode through the plain RCAS: the oracle's store of an RGBA32F image"""
    if np.dtype(out_dtype) == np.float32 and dst_fmt is None:
        return img32.copy()
    h, w = img32.shape[:2]
    c = po.SharpenConstants()
    c.const0[0] = int(np.float32(1.0).view(np.uint32))
    c.imageCentre[:] = [1, 1, 1, 1]  # no group inside radius^2 = 0 (srtm_oracle.encode)
    c.radius[:] = [0, 0, w, h]
    return _RCAS(np.ascontiguousarray(img32), c, out_dtype=out_dtype, dst_fmt=dst_fmt)


def _source(src, src_fmt):
    if src_fmt == 6:  # R32G32B32_FLOAT: the kernels read its RGBA32F expansion (alpha 1)
        s = np.ones(src.shape[:2] + (4,), dtype=np.float32)
        s[..., :3] = src
        return s
    return so._float_source(src)


def easu(src, out_w, out_h, consts, out_dtype=np.uint8, bits=0, src_fmt=None, dst_fmt=None, nthreads=1):
    o = _EASU(np.ascontiguousarray(read_map(_source(src, src_fmt), bits)), out_w, out_h, consts, out_dtype=np.float32,
              nthreads=nthreads)
    return store(o, bits, out_dtype, dst_fmt)


def rcas(src, consts, out_dtype=np.uint8, bits=0, src_fmt=None, dst_fmt=None, nthreads=1):
    o = _RCAS(np.ascontiguousarray(read_map(_source(src, src_fmt), bits)), consts, out_dtype=np.float32,
              nthreads=nthreads)
    return store(o, bits, out_dtype, dst_fmt)


def nis_scaler(src, out_w, out_h, cfg, out_dtype=np.uint8, bits=0, src_fmt=None, dst_fmt=None, nthreads=1):
    o = _NIS_SCALER(np.ascontiguousarray(read_map(_source(src, src_fmt), bits)), out_w, out_h, cfg,
                    out_dtype=np.float32, nthreads=nthreads)
    return store(o, bits, out_dtype, dst_fmt)


def nis_sharpen(src, cfg, out_dtype=np.uint8, bits=0, src_fmt=None, dst_fmt=None, nthreads=1):
    o = _NIS_SHARPEN(np.ascontiguousarray(read_map(_source(src, src_fmt), bits)), cfg, out_dtype=np.float32,
                    nthreads=nthreads)
    return store(o, bits, out_dtype, dst_fmt)


def ctx_bits(flags, nis, upscale, unorm_out):
    """the pass bits a context gives each pass (capi.cu, prepare_resources): (easu, rcas, nis, intermediate dtype)"""
    srtm, srtm_nis, finite, perc = flags & 2, flags & 4, flags & 8, flags & 16
    easu_b = rcas_b = nis_b = 0
    if srtm and not nis:
        easu_b, rcas_b = SRTM_IN, SRTM_OUT | (0 if upscale else SRTM_IN)
    if srtm_nis and nis:
        nis_b = SRTM_IN | SRTM_OUT
    if perc:
        easu_b |= PERCEPTUAL_IN
        rcas_b |= PERCEPTUAL_OUT | (0 if upscale else PERCEPTUAL_IN)
        nis_b |= (PERCEPTUAL_IN | PERCEPTUAL_OUT) if nis else 0
    plain_mid = not ((srtm and not nis) or perc)
    mid = None if plain_mid else (np.float16 if unorm_out else np.float32)
    if finite:
        both = FINITE_IN | FINITE_OUT
        easu_b |= both
        rcas_b |= both if (not upscale or mid is not None or not unorm_out) else 0
        nis_b |= both
    return easu_b, rcas_b, nis_b, mid


def ctx_plan(flags, nis, upscale, src_fmt, out_fmt):
    """the rest of the plan (csrc/plan.h, make_plan) from ctx_bits, for an ovrfsr_format source src_fmt and the output
    format out_fmt prepare_resources accepted: (easu, rcas, nis bits, intermediate dtype or None for the output's
    format, paired, fused tried, sRGB-encoded output).  A UNORM source gets no bits; the pairing needs a UNORM output
    and an intermediate in its format; the output is sRGB-encoded for PERCEPTUAL with a float source into RGBA8."""
    float_src = src_fmt in (2, 3, 6)  # RGBA16F, RGBA32F, RGB32F
    unorm_out = out_fmt in (0, 4)     # RGBA8, RGB10A2
    easu_b, rcas_b, nis_b, mid = ctx_bits(flags, nis, upscale, unorm_out) if float_src else (0, 0, 0, None)
    paired = not nis and upscale and unorm_out and mid is None
    return easu_b, rcas_b, nis_b, mid, paired, paired and bool(flags & 1), float_src and bool(flags & 16) and out_fmt == 0


def fsr_chain(src, uc, sc, out_w, out_h, out_dtype, flags, upscale=True, src_fmt=None):
    """the checker of a context's FSR path with config flags `flags` on a float source (no pairing, no fused kernel)"""
    easu_b, rcas_b, _, mid = ctx_bits(flags, False, upscale, np.dtype(out_dtype) == np.uint8)
    if not upscale:
        return rcas(src, sc, out_dtype, rcas_b, src_fmt)
    m = easu(src, out_w, out_h, uc, mid if mid is not None else out_dtype, easu_b, src_fmt)
    return rcas(m, sc, out_dtype, rcas_b)


def nis_chain(src, cfg, out_w, out_h, out_dtype, flags, upscale=True, src_fmt=None):
    _, _, nis_b, _ = ctx_bits(flags, True, upscale, np.dtype(out_dtype) == np.uint8)
    if upscale:
        return nis_scaler(src, out_w, out_h, cfg, out_dtype, nis_b, src_fmt)
    return nis_sharpen(src, cfg, out_dtype, nis_b, src_fmt)
