"""OVRFSR_FLAG_PERCEPTUAL without a GPU: the flag's and the pass bits' values in every layer, that the other bits stay
unknown, the config round trip, the argument checks of the four _ex dispatches (refused before anything is launched, so
fake device addresses are never touched) -- from Python and from a plain C program --, the C++ drop-in's field, the
committed sRGB table against a fresh generation and a float64 encode, the maps, and the checker with the maps off."""
import ctypes as C
import dataclasses
import importlib.util
import inspect
import os
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import perceptual_oracle as pq

ROOT = Path(__file__).resolve().parents[1]
INC = ROOT / "include"
EX = ("ovrfsr_dispatch_fsr_easu_ex", "ovrfsr_dispatch_fsr_rcas_ex", "ovrfsr_dispatch_nis_scaler_ex", "ovrfsr_dispatch_nis_sharpen_ex")
PERC = pq.PERCEPTUAL_IN | pq.PERCEPTUAL_OUT


def _img(fmt, w=64, h=32, addr=0x7f0000000000):
    from openvr_fsr_b200 import _lib as L
    bpp = {L.FORMAT_RGBA16F: 8, L.FORMAT_RGBA32F: 16}.get(fmt, 4)
    return L.Image(addr, w, h, w * bpp, fmt, 1, 0, 0)


def _consts(name):
    if "nis" in name:
        return C.cast(C.create_string_buffer(256), C.c_void_p)
    return (C.c_uint32 * (24 if "easu" in name else 12))()


def test_values_in_every_layer(built_lib):
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    header = (INC / "ovrfsr.h").read_text()
    assert re.search(r"#define OVRFSR_FLAG_PERCEPTUAL 16\b", header) and L.FLAG_PERCEPTUAL == 16
    assert re.search(r"#define OVRFSR_PASS_PERCEPTUAL_IN 128\b", header) and L.PASS_PERCEPTUAL_IN == pq.PERCEPTUAL_IN == 128
    assert re.search(r"#define OVRFSR_PASS_PERCEPTUAL_OUT 512\b", header) and L.PASS_PERCEPTUAL_OUT == pq.PERCEPTUAL_OUT == 512
    # no pass bit is defined as 4, 8, 64 or 0x100: those stay unknown
    bits = {int(v, 0) for v in re.findall(r"#define OVRFSR_PASS_\w+ (\w+)", header)}
    assert bits == {1, 2, 16, 32, 128, 512}, bits
    assert ovr.Config(perceptual=True).to_c().flags == L.FLAG_PERCEPTUAL
    assert ovr.Config(perceptual=True, srtm=True, finite=True).to_c().flags == L.FLAG_PERCEPTUAL | L.FLAG_SRTM | L.FLAG_FINITE
    cfg_h = (ROOT / "openvr_fsr_b200" / "csrc" / "config.h").read_text()
    assert re.search(r"bool perceptual = false;", cfg_h)
    assert "OVRFSR_FLAG_PERCEPTUAL" in (ROOT / "openvr_fsr_b200" / "csrc" / "postprocessor.cpp").read_text()
    for fn in (ovr.fsr_easu, ovr.fsr_rcas, ovr.nis_scaler, ovr.nis_sharpen):
        params = inspect.signature(fn).parameters
        assert "perceptual_in" in params and "perceptual_out" in params, fn.__name__
    assert "perceptual_in" not in inspect.signature(ovr.fsr_fused).parameters  # the fused dispatch has no pass bits


def test_config_round_trip(built_lib):
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    cfg = ovr.Config(fsrEnabled=True, renderScale=0.75, perceptual=True)
    pp = ovr.PostProcessor(cfg)  # ovrfsr_create: no GPU work
    try:
        got = L.Config()
        assert L.lib().ovrfsr_get_config(pp._ctx, C.byref(got)) == L.OK and got.flags == L.FLAG_PERCEPTUAL
        pp.set_config(dataclasses.replace(cfg, perceptual=False, finite=True))
        assert L.lib().ovrfsr_get_config(pp._ctx, C.byref(got)) == L.OK and got.flags == L.FLAG_FINITE
    finally:
        pp.close()


@pytest.mark.parametrize("name", EX)
@pytest.mark.parametrize("src_fmt", [0, 1, 4, 5])  # RGBA8, BGRA8, RGB10A2, BGRX8
@pytest.mark.parametrize("flags", [128, 512, PERC, 128 | 1, 512 | 2 | 32, PERC | 51])
def test_perceptual_bits_rejected_for_unorm_sources(built_lib, name, src_fmt, flags):
    from openvr_fsr_b200 import _lib as L
    dst_fmt = L.FORMAT_RGB10A2 if src_fmt == L.FORMAT_RGB10A2 else L.FORMAT_RGBA8
    s, d = _img(src_fmt), _img(dst_fmt, addr=0x7f0000100000)
    for mode in (L.MATH_STRICT, L.MATH_FAST):
        assert getattr(L.lib(), name)(C.byref(s), C.byref(d), _consts(name), mode, flags, None) == L.ERR_UNSUPPORTED


@pytest.mark.parametrize("name", EX)
@pytest.mark.parametrize("src_fmt", [2, 3])  # RGBA16F, RGBA32F
def test_unknown_bits_with_the_perceptual_bits_rejected(built_lib, name, src_fmt):
    from openvr_fsr_b200 import _lib as L
    s, d = _img(src_fmt), _img(L.FORMAT_RGBA16F, addr=0x7f0000100000)
    for flags in (4 | 128, 8 | 512, 64 | PERC, 0x100 | 128, 0x100 | 512, 1024 | PERC, 256 | 51, -1):
        assert getattr(L.lib(), name)(C.byref(s), C.byref(d), _consts(name), L.MATH_STRICT, flags, None) == L.ERR_INVALID


def test_plain_c_program(tmp_path, built_lib):
    """tests/c/perceptual_abi.c: the flag and the pass bits of the _ex dispatches from C11 against the in-tree library"""
    if shutil.which("gcc") is None:
        pytest.skip("gcc not installed")
    exe = tmp_path / "perceptual_abi"
    libdir = Path(built_lib).parent
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", str(INC),
                           str(ROOT / "tests/c/perceptual_abi.c"), "-o", str(exe), "-L", str(libdir), "-lovrfsr",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([str(exe)], capture_output=True, text=True, env={**os.environ, "TZ": "UTC"})
    assert out.returncode == 0, out.stdout + out.stderr
    assert "perceptual_abi: ok" in out.stdout


def test_cpp_perceptual_driver_compiles():
    """the drop-in's Config::perceptual driver builds with a plain host compiler; the GPU test builds and runs it"""
    cuda_inc = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda")) / "include"
    if shutil.which("g++") is None or not (cuda_inc / "cuda_runtime.h").exists():
        pytest.skip("g++ or the CUDA headers are not installed")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(INC),
                               "-I", str(ROOT / "openvr_fsr_b200/csrc"), "-I", str(cuda_inc), "-c",
                               str(ROOT / "tests/cpp/pp_perceptual_selftest.cpp"), "-o", str(Path(d) / "pp.o")])


# ---- the sRGB table ----------------------------------------------------------------------------------------------
def _generator():
    spec = importlib.util.spec_from_file_location("gen_srgb_table", ROOT / "tools" / "gen_srgb_table.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_committed_table_is_a_fresh_generation():
    gen = _generator()
    fresh = gen.thresholds()
    assert np.array_equal(pq.table_words(), np.array(fresh, dtype=np.uint32))
    assert pq.TABLE_INC.read_text() == gen.render(fresh)


def test_table_strictly_increasing_and_bracketing_the_boundaries():
    from decimal import Decimal
    gen = _generator()
    t = pq.table_words().view(np.float32)
    assert t[0] == 0 and (np.diff(t) > 0).all() and t[1] > 0 and t[255] < 1
    for k in range(1, 256):
        b = gen.srgb_to_linear((Decimal(k) - Decimal("0.5")) / Decimal(255))
        assert Decimal(float(t[k])) >= b > Decimal(float(np.nextafter(t[k], np.float32(0))))


def _srgb_f64(v):
    """a float64 statement of the encode: round(255 * linear_to_srgb(sat(v)))"""
    v = np.asarray(v, dtype=np.float32)
    v = np.clip(np.where(np.isnan(v), np.float32(0), v).astype(np.float64), 0.0, 1.0)
    s = np.where(v <= 0.0031308, v * 12.92, 1.055 * np.power(v, 1 / 2.4) - 0.055)
    return np.floor(s * 255 + 0.5).astype(np.uint8)


def test_table_encode_equals_float64_on_every_fp16_word():
    x = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16).astype(np.float32)
    x = x[~np.isinf(x)]
    assert np.array_equal(pq.srgb_code(x), _srgb_f64(x))


def test_table_encode_equals_float64_on_a_dense_fp32_sweep():
    lo, hi = np.float32(1e-5).view(np.uint32), np.float32(1.01).view(np.uint32)
    x = np.arange(lo, hi, 5, dtype=np.uint32).view(np.float32)
    t = pq.table_words()
    around = (t[1:, None].astype(np.int64) + np.arange(-2, 3)[None, :]).astype(np.uint32).view(np.float32).ravel()
    special = np.array([0.0, -0.0, -1.0, -np.inf, np.inf, np.nan, 1e-45, 2.0, 65504.0], dtype=np.float32)
    for v in (x, around, special):
        assert np.array_equal(pq.srgb_code(v), _srgb_f64(v))
    # the thresholds themselves: code k at T[k], k - 1 one ulp below
    tk = t[1:].view(np.float32)
    assert np.array_equal(pq.srgb_code(tk), np.arange(1, 256))
    assert np.array_equal(pq.srgb_code(np.nextafter(tk, np.float32(0))), np.arange(0, 255))


# ---- the maps ----------------------------------------------------------------------------------------------------
def test_inverse_of_forward_within_one_ulp_on_every_fp16_word():
    x = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16).astype(np.float32)
    y = pq.p_inv(pq.p_fwd(x))
    fin = np.isfinite(x)
    assert (np.isnan(y) == np.isnan(x)).all() and np.array_equal(y[np.isinf(x)], x[np.isinf(x)])
    d = np.abs(y[fin].view(np.int32).astype(np.int64) - x[fin].view(np.int32).astype(np.int64))
    assert d.max() <= 1, int(d.max())
    assert np.array_equal(np.signbit(y[fin]), np.signbit(x[fin]))  # -0 stays -0, negatives stay negative


def test_maps_are_sign_preserving_gamma_two():
    x = np.array([0.0, -0.0, 0.25, -0.25, 4.0, -9.0, np.inf, -np.inf], dtype=np.float32)
    assert np.array_equal(pq.p_fwd(x), np.array([0.0, -0.0, 0.5, -0.5, 2.0, -3.0, np.inf, -np.inf], dtype=np.float32))
    assert np.array_equal(np.signbit(pq.p_fwd(x)), np.signbit(x))
    assert np.array_equal(pq.p_inv(np.array([0.5, -3.0], dtype=np.float32)), np.array([0.25, -9.0], dtype=np.float32))


# ---- the checker ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_dtype", [np.uint8, np.float16, np.float32])
def test_checker_with_the_maps_off_is_the_plain_oracle(out_dtype):
    from oracle import pyoracle as po
    rng = np.random.default_rng(3)
    w, h = 37, 29
    src = rng.uniform(-0.2, 1.5, (h, w, 4)).astype(np.float16)
    ow, oh = po.output_size(w, h, 0.75)
    uc = po.upscale_constants(0, True, w, h, ow, oh, radius=0.4)
    sc = po.sharpen_constants(0, True, w, h, radius=0.4, sharpness=0.6)
    cfg, ok = po.nis_config(True, 0, True, w, h, w, h, radius=0.4, sharpness=0.6)
    assert ok
    pairs = [(pq.easu(src, ow, oh, uc, out_dtype), po.easu(src, ow, oh, uc, out_dtype=out_dtype)),
             (pq.rcas(src, sc, out_dtype), po.rcas(src, sc, out_dtype=out_dtype)),
             (pq.nis_sharpen(src, cfg, out_dtype), po.nis_sharpen(src, cfg, out_dtype=out_dtype))]
    for got, want in pairs:
        assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


def test_checker_rgba8_store_is_the_srgb_code():
    """an RGBA8 store with perceptual-out: code() of P^-1 on R, G, B and the oracle's alpha"""
    from oracle import pyoracle as po
    rng = np.random.default_rng(4)
    src = rng.uniform(0, 1, (24, 40, 4)).astype(np.float32)
    sc = po.sharpen_constants(0, True, 40, 24, radius=0.4, sharpness=0.6)
    lin = pq.rcas(src, sc, np.float32, pq.PERCEPTUAL_IN | pq.PERCEPTUAL_OUT)
    got = pq.rcas(src, sc, np.uint8, pq.PERCEPTUAL_IN | pq.PERCEPTUAL_OUT)
    assert np.array_equal(got[..., :3], pq.srgb_code(lin[..., :3]))
    assert np.array_equal(got[..., 3], po.rcas(src, sc, out_dtype=np.uint8)[..., 3])
    # brighter than the plain UNORM store of the same linear values in the midtones
    mid = (lin[..., :3] > 0.05) & (lin[..., :3] < 0.5)
    assert (got[..., :3][mid].astype(int) > np.floor(lin[..., :3][mid] * 255 + 0.5)).all()
