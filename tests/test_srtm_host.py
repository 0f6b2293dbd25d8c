"""AMD's reversible tone map (OVRFSR_FLAG_SRTM) without a GPU: the checker's two maps (tests/srtm_oracle.py) on densely sampled float32 values
of the whole FP16 range, the round-trip bounds DESIGN.md section 4 states, the special inputs outside the map's domain,
and the C ABI refusing the pass flags for UNORM sources before anything is launched."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
FP16_MAX = 65504.0
# relative error of G(F(x)) against x, per band of x, binary32 maps (the oracle's; the GPU's are the same operations)
BANDS_B32 = [((0.0, 1.0), 3.2e-7), ((1.0, 4.0), 6.0e-7), ((4.0, 64.0), 7.8e-6), ((64.0, 1024.0), 1.2e-4)]
# through an RGBA16F intermediate (the tone-mapped value rounded to binary16), x in (0, 1]: relative where F(x) is an FP16
# normal, absolute below that (F(x) ~ x there, FP16 subnormals are spaced 2^-24: half a step, plus G's rounding)
B16_REL, B16_ABS = 6.6e-4, 3.0e-8


@pytest.fixture(scope="module")
def samples():
    """every 61st float32 in (0, 65504] plus the band edges, as (x, x/2, 0) triples"""
    top = int(np.float32(FP16_MAX).view(np.uint32))
    bits = np.concatenate([np.arange(1, top + 1, 61, dtype=np.uint32),
                           np.float32([1.0, 4.0, 64.0, 1024.0, FP16_MAX]).view(np.uint32)])
    x = np.unique(bits).view(np.float32)
    return np.stack([x, (x * np.float32(0.5)).astype(np.float32), np.zeros_like(x)], -1)


def _rel(got, want):
    g, w = got.astype(np.float64), want.astype(np.float64)
    pos = w > 0
    return np.abs(g - w)[pos] / w[pos]


def test_forward_maps_fp16_range_into_unit_interval(samples):
    from tests import srtm_oracle as so
    f = so.srtm(samples)
    assert np.isfinite(f).all() and (f >= 0).all() and (f < 1).all()
    # the largest value is 0.9999848; F(65504) itself rounds one ulp below it (k = 1 / 65505 and x * k round twice)
    assert f[:, 0].max() == np.float32(0.9999848) and f[-1, 0] == np.nextafter(np.float32(0.9999848), np.float32(0))
    assert (f[:, 2] == 0).all()  # a zero channel stays zero


@pytest.mark.parametrize("band,bound", BANDS_B32, ids=[f"{lo:g}-{hi:g}" for (lo, hi), _ in BANDS_B32])
def test_round_trip_binary32(samples, band, bound):
    from tests import srtm_oracle as so
    lo, hi = band
    c = samples[(samples[:, 0] > lo) & (samples[:, 0] <= hi)]
    g = so.srtm(so.srtm(c), inverse=True)
    err = _rel(g[:, :2], c[:, :2])
    assert err.size and err.max() <= bound, err.max()


def test_round_trip_top_band_is_capped(samples):
    """x in (1024, 65504]: F(x) rounds within 2^-24 of 1, so G's 1 - m reaches its 1/32768 floor and G caps at 32768"""
    from tests import srtm_oracle as so
    c = samples[samples[:, 0] > 1024.0]
    g = so.srtm(so.srtm(c), inverse=True)
    assert g.max() <= 32768.0 and g[-1, 0] == np.float32(32767.5)
    assert _rel(g[:, :2], c[:, :2]).max() <= 0.5


def test_round_trip_through_binary16_up_to_one(samples):
    """the RGBA16F intermediate the ctx uses for a UNORM output (which clips at 1)"""
    from tests import srtm_oracle as so
    c = samples[samples[:, 0] <= 1.0]
    f = so.srtm(c)
    g = so.srtm(f.astype(np.float16).astype(np.float32), inverse=True)
    normal = f[:, :2] >= 2.0 ** -14
    d = np.abs(g[:, :2].astype(np.float64) - c[:, :2])
    assert (d[normal] / c[:, :2][normal]).max() <= B16_REL
    assert d[~normal].max() <= B16_ABS


def test_inverse_never_exceeds_32768():
    """G over every 7th float32 in [0, 1] (and 1 itself, where 1 - m is 0): at most 32768 x the input's largest channel"""
    from tests import srtm_oracle as so
    bits = np.concatenate([np.arange(0, int(np.float32(1.0).view(np.uint32)) + 1, 7, dtype=np.uint32),
                           np.float32([1.0, 0.9999848, np.nextafter(np.float32(1), np.float32(0))]).view(np.uint32)])
    x = bits.view(np.float32)
    g = so.srtm(np.stack([x, x, x], -1), inverse=True)
    assert g.max() == 32768.0 and (g <= 32768.0).all()
    assert (g[:, 0] <= np.float32(32768.0) * x).all()


def test_outside_the_domain_follows_the_formula():
    """signed zeros, subnormals, negatives, max3 = -1, NaN and infinity: no clamp, what IEEE arithmetic gives"""
    from tests import srtm_oracle as so
    tiny = np.float32(2.0 ** -140)
    c = np.array([[0.0, -0.0, 0.0], [tiny, -tiny, 0.0], [-0.5, -0.5, -0.5], [-1.0, -2.0, -3.0], [np.nan, 1.0, 0.5],
                  [np.inf, 1.0, 0.0], [-4.0, 1.0, 0.0]], np.float32)
    f = so.srtm(c)
    assert np.array_equal(f[0].view(np.uint32), c[0].view(np.uint32))  # k = 1: signs of zero kept
    assert np.array_equal(f[1].view(np.uint32), c[1].view(np.uint32))  # subnormals pass through
    assert (f[2] == -1.0).all()                                        # m = -0.5: k = 2
    assert f[3, 0] == -np.inf and f[3, 1] == -np.inf                   # m = -1: k = 1 / 0 = inf
    assert np.isnan(f[4, 0]) and f[4, 1] == 0.5 and f[4, 2] == 0.25    # max3 ignores the NaN channel (the pinned rule)
    assert np.isnan(f[5, 0]) and f[5, 1] == 0.0 and f[5, 2] == 0.0     # m = inf: inf x 0 is NaN, finite x 0 = 0
    assert f[6, 0] == -2.0 and f[6, 1] == 0.5                          # m = 1 from the positive channel
    g = so.srtm(np.array([[2.0, 0.5, -1.0], [np.nan, 0.5, 0.0]], np.float32), inverse=True)
    assert (g[0] == np.float32([2.0, 0.5, -1.0]) * np.float32(32768.0)).all()  # 1 - m < 0: the 1/32768 floor
    assert np.isnan(g[1, 0]) and g[1, 1] == 1.0


def test_oracle_passes_match_the_maps_around_the_plain_passes():
    """the checker's passes with the tone map against the composition they document: F on the decoded source, the plain
    pass in RGBA32F, G, the target's encode -- and that encode is the oracle's own store, bit for bit"""
    from oracle import pyoracle as po
    from openvr_fsr_b200 import synth
    from tests import srtm_oracle as so
    w, h = 41, 29
    src = (synth.natural_rgba8(w, h, 5).astype(np.float32) / 255.0 * 12.0 - 0.5).astype(np.float16)
    ow, oh = po.output_size(w, h, 0.75)
    uc = po.upscale_constants(0, True, w, h, ow, oh, radius=0.5)
    sc = po.sharpen_constants(0, True, ow, oh, radius=0.5, sharpness=0.8, debug=True)
    # the encode through the oracle's copy path is its store: same bytes as the plain passes writing the target directly
    for dt in (np.uint8, np.float16):
        plain32 = po.easu(src, ow, oh, uc, out_dtype=np.float32)
        assert np.array_equal(so.encode(plain32, dt).view(np.uint8), po.easu(src, ow, oh, uc, out_dtype=dt).view(np.uint8))
        assert np.array_equal(so.easu(src, ow, oh, uc, out_dtype=dt).view(np.uint8), po.easu(src, ow, oh, uc, out_dtype=dt).view(np.uint8))
        assert np.array_equal(so.rcas(plain32, sc, out_dtype=dt).view(np.uint8), po.rcas(plain32, sc, out_dtype=dt).view(np.uint8))
    f = src.astype(np.float32)
    f[..., :3] = so.srtm(f[..., :3])
    mid = so.easu(src, ow, oh, uc, out_dtype=np.float32, srtm_in=True)
    assert np.array_equal(mid.view(np.uint32), po.easu(f, ow, oh, uc, out_dtype=np.float32).view(np.uint32))
    out = so.rcas(mid, sc, out_dtype=np.float16, srtm_out=True)
    r = po.rcas(mid, sc, out_dtype=np.float32)
    r[..., :3] = so.srtm(r[..., :3], inverse=True)
    assert np.array_equal(out.view(np.uint16), r.astype(np.float16).view(np.uint16))
    with pytest.raises(ValueError):  # UNORM sources are display-referred: no tone map
        so.rcas(synth.natural_rgba8(w, h, 5), sc, srtm_in=True)


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def _img(fmt, w=64, h=32, addr=0x7f0000000000):
    from openvr_fsr_b200 import _lib as L
    bpp = {L.FORMAT_RGBA16F: 8, L.FORMAT_RGBA32F: 16}.get(fmt, 4)
    return L.Image(addr, w, h, w * bpp, fmt, 1, 0, 0)


@pytest.mark.parametrize("src_fmt", [0, 1, 4, 5])  # RGBA8, BGRA8, RGB10A2, BGRX8
@pytest.mark.parametrize("flags", [1, 2, 3])
def test_pass_flags_rejected_for_unorm_sources(built_lib, src_fmt, flags):
    """OVRFSR_ERR_UNSUPPORTED before any launch: a fake device pointer is never touched, no device is needed"""
    from openvr_fsr_b200 import _lib as L
    dst_fmt = L.FORMAT_RGB10A2 if src_fmt == L.FORMAT_RGB10A2 else L.FORMAT_RGBA8
    uc, sc = (C.c_uint32 * 24)(), (C.c_uint32 * 12)()
    s, d = _img(src_fmt), _img(dst_fmt, addr=0x7f0000100000)
    assert L.lib().ovrfsr_dispatch_fsr_easu_ex(C.byref(s), C.byref(d), uc, L.MATH_STRICT, flags, None) == L.ERR_UNSUPPORTED
    assert L.lib().ovrfsr_dispatch_fsr_rcas_ex(C.byref(s), C.byref(d), sc, L.MATH_FAST, flags, None) == L.ERR_UNSUPPORTED


def test_unknown_pass_flags_rejected(built_lib):
    from openvr_fsr_b200 import _lib as L
    s, d = _img(L.FORMAT_RGBA16F), _img(L.FORMAT_RGBA16F, addr=0x7f0000100000)
    for flags in (4, 8, -1, 0x100 | 1):
        assert L.lib().ovrfsr_dispatch_fsr_easu_ex(C.byref(s), C.byref(d), (C.c_uint32 * 24)(), 1, flags, None) == L.ERR_INVALID
        assert L.lib().ovrfsr_dispatch_fsr_rcas_ex(C.byref(s), C.byref(d), (C.c_uint32 * 12)(), 1, flags, None) == L.ERR_INVALID


def test_srtm_symbols_and_flags_declared(built_lib):
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    header = (ROOT / "include" / "ovrfsr.h").read_text()
    assert re.search(r"#define OVRFSR_FLAG_SRTM 2\b", header)
    assert re.search(r"#define OVRFSR_PASS_SRTM_IN 1\b", header) and re.search(r"#define OVRFSR_PASS_SRTM_OUT 2\b", header)
    lib = C.CDLL(str(built_lib))
    for name in ("ovrfsr_dispatch_fsr_easu_ex", "ovrfsr_dispatch_fsr_rcas_ex"):
        assert hasattr(lib, name) and name in L.SYMBOLS
        assert re.search(r"OVRFSR_API int " + name + r"\(const ovrfsr_image \*src, const ovrfsr_image \*dst, const uint32_t consts",
                         header)
    assert ovr.Config(srtm=True).to_c().flags == L.FLAG_SRTM
    assert ovr.Config(srtm=True, fusedFsr=True).to_c().flags == L.FLAG_SRTM | L.FLAG_FUSED_FSR
    cfg_h = (ROOT / "openvr_fsr_b200" / "csrc" / "config.h").read_text()
    assert re.search(r"bool srtm = false;", cfg_h)
    assert "OVRFSR_FLAG_SRTM" in (ROOT / "openvr_fsr_b200" / "csrc" / "postprocessor.cpp").read_text()
