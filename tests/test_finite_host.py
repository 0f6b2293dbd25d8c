"""OVRFSR_FLAG_FINITE without a GPU: the flag's and the pass bits' values in every layer, the config round trip, the
argument checks of the four _ex dispatches (refused before anything is launched, so fake device addresses are never
touched) -- from Python and from a plain C program --, the C++ drop-in's field, and the host statement of the two maps
that the GPU tests hold the kernels to."""
import ctypes as C
import dataclasses
import os
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import finite_rule as fr

ROOT = Path(__file__).resolve().parents[1]
INC = ROOT / "include"
EX = ("ovrfsr_dispatch_fsr_easu_ex", "ovrfsr_dispatch_fsr_rcas_ex", "ovrfsr_dispatch_nis_scaler_ex", "ovrfsr_dispatch_nis_sharpen_ex")


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
    assert re.search(r"#define OVRFSR_FLAG_FINITE 8\b", header) and L.FLAG_FINITE == 8
    assert re.search(r"#define OVRFSR_PASS_FINITE_IN 16\b", header) and L.PASS_FINITE_IN == 16
    assert re.search(r"#define OVRFSR_PASS_FINITE_OUT 32\b", header) and L.PASS_FINITE_OUT == 32
    assert ovr.Config(finite=True).to_c().flags == L.FLAG_FINITE
    assert ovr.Config(finite=True, srtm=True, fusedFsr=True).to_c().flags == L.FLAG_FINITE | L.FLAG_SRTM | L.FLAG_FUSED_FSR
    assert ovr.Config().to_c().flags == 0
    cfg_h = (ROOT / "openvr_fsr_b200" / "csrc" / "config.h").read_text()
    assert re.search(r"bool finite = false;", cfg_h)
    assert "OVRFSR_FLAG_FINITE" in (ROOT / "openvr_fsr_b200" / "csrc" / "postprocessor.cpp").read_text()
    import inspect
    for fn in (ovr.fsr_easu, ovr.fsr_rcas, ovr.nis_scaler, ovr.nis_sharpen):
        params = inspect.signature(fn).parameters
        assert "finite_in" in params and "finite_out" in params, fn.__name__
    assert "finite_in" not in inspect.signature(ovr.fsr_fused).parameters  # the fused dispatch has no pass bits


def test_config_round_trip(built_lib):
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    cfg = ovr.Config(fsrEnabled=True, renderScale=0.75, finite=True)
    pp = ovr.PostProcessor(cfg)  # ovrfsr_create: no GPU work
    try:
        got = L.Config()
        assert L.lib().ovrfsr_get_config(pp._ctx, C.byref(got)) == L.OK and got.flags == L.FLAG_FINITE
        pp.set_config(dataclasses.replace(cfg, finite=False, srtm=True))  # a reset, nothing to release yet
        assert L.lib().ovrfsr_get_config(pp._ctx, C.byref(got)) == L.OK and got.flags == L.FLAG_SRTM
    finally:
        pp.close()


@pytest.mark.parametrize("name", EX)
@pytest.mark.parametrize("src_fmt", [0, 1, 4, 5])  # RGBA8, BGRA8, RGB10A2, BGRX8
@pytest.mark.parametrize("flags", [16, 32, 48, 16 | 1, 32 | 2, 51])
def test_finite_bits_rejected_for_unorm_sources(built_lib, name, src_fmt, flags):
    from openvr_fsr_b200 import _lib as L
    dst_fmt = L.FORMAT_RGB10A2 if src_fmt == L.FORMAT_RGB10A2 else L.FORMAT_RGBA8
    s, d = _img(src_fmt), _img(dst_fmt, addr=0x7f0000100000)
    for mode in (L.MATH_STRICT, L.MATH_FAST):
        assert getattr(L.lib(), name)(C.byref(s), C.byref(d), _consts(name), mode, flags, None) == L.ERR_UNSUPPORTED


@pytest.mark.parametrize("name", EX)
@pytest.mark.parametrize("src_fmt", [2, 3])  # RGBA16F, RGBA32F
def test_unknown_bits_with_the_finite_bits_rejected(built_lib, name, src_fmt):
    from openvr_fsr_b200 import _lib as L
    s, d = _img(src_fmt), _img(L.FORMAT_RGBA16F, addr=0x7f0000100000)
    for flags in (4 | 16, 8 | 32, 64 | 48, 0x100 | 16, -1):
        assert getattr(L.lib(), name)(C.byref(s), C.byref(d), _consts(name), L.MATH_STRICT, flags, None) == L.ERR_INVALID


def test_plain_c_program(tmp_path, built_lib):
    """tests/c/finite_abi.c: the flag and the pass bits of the _ex dispatches from C11 against the in-tree library"""
    if shutil.which("gcc") is None:
        pytest.skip("gcc not installed")
    exe = tmp_path / "finite_abi"
    libdir = Path(built_lib).parent
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", str(INC),
                           str(ROOT / "tests/c/finite_abi.c"), "-o", str(exe), "-L", str(libdir), "-lovrfsr",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([str(exe)], capture_output=True, text=True, env={**os.environ, "TZ": "UTC"})
    assert out.returncode == 0, out.stdout + out.stderr
    assert "finite_abi: ok" in out.stdout


def test_cpp_finite_driver_compiles():
    """the drop-in's Config::finite driver builds with a plain host compiler; the GPU test builds and runs the same file"""
    cuda_inc = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda")) / "include"
    if shutil.which("g++") is None or not (cuda_inc / "cuda_runtime.h").exists():
        pytest.skip("g++ or the CUDA headers are not installed")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(INC),
                               "-I", str(ROOT / "openvr_fsr_b200/csrc"), "-I", str(cuda_inc), "-c",
                               str(ROOT / "tests/cpp/pp_finite_selftest.cpp"), "-o", str(Path(d) / "pp.o")])


# ---- the host statement of the maps -----------------------------------------------------------------------------
def test_finite_in_over_every_fp16_word():
    u = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    x = u.view(np.float16)
    y = fr.finite_in(x)
    fin = np.isfinite(x)
    assert np.array_equal(y[fin].view(np.uint16), u[fin])  # +-0, subnormals, negatives: bit for bit
    assert (y[np.isnan(x)].view(np.uint16) == 0).all()  # NaN -> +0, whatever its sign and payload
    assert (y[x == np.inf] == 65504).all() and (y[x == -np.inf] == -65504).all()
    assert np.isfinite(y).all()


def test_finite_in_keeps_fp32_beyond_fp16():
    words = np.array([0, 0x80000000, 1, 0x807fffff, 0x7f7fffff, 0xff7fffff, 0x477fe000, 0x477fe001, 0x7f800000, 0xff800000,
                      0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fa5a5a5], dtype=np.uint32)
    x = words.view(np.float32)
    y = fr.finite_in(x).view(np.uint32)
    assert np.array_equal(y[:8], words[:8])  # +-0, subnormals, +-FLT_MAX, 65504 and the next float: bit for bit
    assert np.array_equal(y[8:10], np.array([0x477fe000, 0xc77fe000], dtype=np.uint32))  # +-inf -> +-65504
    assert (y[10:] == 0).all()  # quiet and signalling NaNs of either sign, with payloads -> +0


def test_finite_out_before_an_fp16_store_is_convert_then_map():
    """clamp then round == round then map +-inf to +-65504, across the binary32 values around 65504 / 65520"""
    lo, hi = np.float32(65000).view(np.uint32), np.float32(70000).view(np.uint32)
    x = np.arange(lo, hi, dtype=np.uint32).view(np.float32)
    x = np.concatenate([x, -x, np.array([np.inf, -np.inf, np.nan, 3e38, -3e38], dtype=np.float32)])
    with np.errstate(over="ignore"):
        assert np.array_equal(fr.fp16_store(x).view(np.uint16), fr.finite_out(x.astype(np.float16)).view(np.uint16))
    assert np.isfinite(fr.fp16_store(x)).all()
    assert fr.fp16_store(np.float32(65519.99)) == 65504 and fr.fp16_store(np.float32(-65520)) == -65504


def test_finite_out_fp32():
    x = np.array([np.inf, -np.inf, np.nan, -0.0, 1e38, -1e-45], dtype=np.float32)
    y = fr.finite_out(x)
    assert y[0] == np.finfo(np.float32).max and y[1] == -np.finfo(np.float32).max and y[2].view(np.uint32) == 0
    assert np.array_equal(y[3:].view(np.uint32), x[3:].view(np.uint32))
