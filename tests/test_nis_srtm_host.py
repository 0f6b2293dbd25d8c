"""OVRFSR_FLAG_SRTM_NIS without a GPU: the bit's value and its round trip through a ctx's config, the argument validation
of ovrfsr_dispatch_nis_scaler_ex / _sharpen_ex (refused before anything is launched, so fake device addresses are never
touched), the exports and declarations of every layer -- from Python and from a plain C program -- and that the
checker's NIS chain with the maps off is the plain oracle pass, byte for byte."""
import ctypes as C
import os
import re
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
INC = ROOT / "include"
EX = ("ovrfsr_dispatch_nis_scaler_ex", "ovrfsr_dispatch_nis_sharpen_ex")


def _img(fmt, w=64, h=32, addr=0x7f0000000000):
    from openvr_fsr_b200 import _lib as L
    bpp = {L.FORMAT_RGBA16F: 8, L.FORMAT_RGBA32F: 16}.get(fmt, 4)
    return L.Image(addr, w, h, w * bpp, fmt, 1, 0, 0)


def _cfg256():
    from openvr_fsr_b200 import _lib as L
    return C.create_string_buffer(256), L


def test_flag_value_and_config_round_trip(built_lib):
    import dataclasses
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    header = (INC / "ovrfsr.h").read_text()
    assert re.search(r"#define OVRFSR_FLAG_SRTM_NIS 4\b", header) and L.FLAG_SRTM_NIS == 4
    assert ovr.Config(srtmNis=True).to_c().flags == L.FLAG_SRTM_NIS
    assert ovr.Config(srtmNis=True, srtm=True).to_c().flags == L.FLAG_SRTM_NIS | L.FLAG_SRTM
    assert ovr.Config().to_c().flags == 0
    cfg = ovr.Config(fsrEnabled=True, useNis=True, renderScale=0.75, srtmNis=True)
    pp = ovr.PostProcessor(cfg)  # ovrfsr_create: no GPU work
    try:
        got = L.Config()
        assert L.lib().ovrfsr_get_config(pp._ctx, C.byref(got)) == L.OK and got.flags == L.FLAG_SRTM_NIS
        pp.set_config(dataclasses.replace(cfg, srtmNis=False, srtm=True))  # a reset, nothing to release yet
        assert L.lib().ovrfsr_get_config(pp._ctx, C.byref(got)) == L.OK and got.flags == L.FLAG_SRTM
    finally:
        pp.close()


@pytest.mark.parametrize("name", EX)
@pytest.mark.parametrize("src_fmt", [0, 1, 4, 5])  # RGBA8, BGRA8, RGB10A2, BGRX8
@pytest.mark.parametrize("flags", [1, 2, 3])
def test_pass_flags_rejected_for_unorm_sources(built_lib, name, src_fmt, flags):
    buf, L = _cfg256()
    dst_fmt = L.FORMAT_RGB10A2 if src_fmt == L.FORMAT_RGB10A2 else L.FORMAT_RGBA8
    s, d = _img(src_fmt), _img(dst_fmt, addr=0x7f0000100000)
    for mode in (L.MATH_STRICT, L.MATH_FAST):
        assert getattr(L.lib(), name)(C.byref(s), C.byref(d), buf, mode, flags, None) == L.ERR_UNSUPPORTED


@pytest.mark.parametrize("name", EX)
@pytest.mark.parametrize("src_fmt", [2, 3])  # RGBA16F, RGBA32F
def test_unknown_pass_flags_rejected(built_lib, name, src_fmt):
    buf, L = _cfg256()
    s, d = _img(src_fmt), _img(L.FORMAT_RGBA16F, addr=0x7f0000100000)
    for flags in (4, 8, -1, 0x100 | 1):
        assert getattr(L.lib(), name)(C.byref(s), C.byref(d), buf, L.MATH_STRICT, flags, None) == L.ERR_INVALID


@pytest.mark.parametrize("name", EX)
def test_image_checks_come_first(built_lib, name):
    """the _ex entry points validate their images exactly as the plain dispatches do, whatever the pass flags"""
    buf, L = _cfg256()
    plain = getattr(L.lib(), name[:-3])
    ok_s, ok_d = _img(L.FORMAT_RGBA16F), _img(L.FORMAT_RGBA16F, addr=0x7f0000100000)
    cases = [
        (_img(L.FORMAT_RGB32F), ok_d),                                     # RGB32F: expand first
        (ok_s, _img(L.FORMAT_BGRA8, addr=0x7f0000100000)),                 # BGRA8 destination
        (L.Image(0, 64, 32, 512, L.FORMAT_RGBA16F, 1, 0, 0), ok_d),        # null source
        (L.Image(0x7f0000000000, 64, 32, 100, L.FORMAT_RGBA16F, 1, 0, 0), ok_d),  # pitch too small
    ]
    for s, d in cases:
        want = plain(C.byref(s), C.byref(d), buf, L.MATH_STRICT, None)
        assert want in (L.ERR_INVALID, L.ERR_UNSUPPORTED)
        for flags in (0, 1, 2, 3):
            assert getattr(L.lib(), name)(C.byref(s), C.byref(d), buf, L.MATH_STRICT, flags, None) == want
    assert getattr(L.lib(), name)(C.byref(ok_s), C.byref(ok_d), None, L.MATH_STRICT, 3, None) == L.ERR_INVALID


def test_symbols_exported_and_declared(built_lib):
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    header = (INC / "ovrfsr.h").read_text()
    lib = C.CDLL(str(built_lib))
    for name in EX:
        assert hasattr(lib, name) and name in L.SYMBOLS
        assert re.search(r"OVRFSR_API int " + name + r"\(const ovrfsr_image \*src, const ovrfsr_image \*dst, const void \*cfg256,"
                         r"\s+int math_mode, int pass_flags, void \*stream\);", header)
    import inspect
    for fn in (ovr.nis_scaler, ovr.nis_sharpen):
        params = inspect.signature(fn).parameters
        assert "srtm_in" in params and "srtm_out" in params
    cfg_h = (ROOT / "openvr_fsr_b200" / "csrc" / "config.h").read_text()
    assert re.search(r"bool srtmNis = false;", cfg_h)
    assert "OVRFSR_FLAG_SRTM_NIS" in (ROOT / "openvr_fsr_b200" / "csrc" / "postprocessor.cpp").read_text()


def test_plain_c_program(tmp_path, built_lib):
    """tests/c/nis_srtm_abi.c: the flag and the _ex dispatches from C11 against the in-tree library"""
    if shutil.which("gcc") is None:
        pytest.skip("gcc not installed")
    exe = tmp_path / "nis_srtm_abi"
    libdir = Path(built_lib).parent
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", str(INC),
                           str(ROOT / "tests/c/nis_srtm_abi.c"), "-o", str(exe), "-L", str(libdir), "-lovrfsr",
                           f"-Wl,-rpath,{libdir}"])
    out = subprocess.run([str(exe)], capture_output=True, text=True, env={**os.environ, "TZ": "UTC"})
    assert out.returncode == 0, out.stdout + out.stderr
    assert "nis_srtm_abi: ok" in out.stdout


def test_cpp_nis_srtm_driver_compiles():
    """the drop-in's Config::srtmNis driver builds with a plain host compiler; the GPU test builds and runs the same file"""
    cuda_inc = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda")) / "include"
    if shutil.which("g++") is None or not (cuda_inc / "cuda_runtime.h").exists():
        pytest.skip("g++ or the CUDA headers are not installed")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(INC),
                               "-I", str(ROOT / "openvr_fsr_b200/csrc"), "-I", str(cuda_inc), "-c",
                               str(ROOT / "tests/cpp/pp_nis_srtm_selftest.cpp"), "-o", str(Path(d) / "pp.o")])


@pytest.mark.parametrize("scale", [0.75, 1.0], ids=["scaler", "sharpen"])
def test_checker_chain_without_the_maps_is_the_plain_pass(scale):
    """tests/test_gpu_nis_srtm.py's checker: F, the NIS oracle into RGBA32F, G, the oracle's encode.  With F and G off it
    must write the bytes of the plain oracle pass into each target format, which pins the RGBA32F hop and the encode"""
    import numpy as np
    from oracle import pyoracle as po
    from openvr_fsr_b200 import synth
    from tests.test_gpu_nis_srtm import nis_pass
    w, h = 97, 61
    src = synth.natural_rgba16f(w, h, 5, peak=1000.0)
    ow, oh = po.output_size(w, h, scale)
    cfg, ok = po.nis_config(scale == 1.0, 0, True, w, h, ow, oh, radius=0.5, sharpness=0.8, debug=True)
    assert ok
    for dt in (np.uint8, np.float16, np.float32):
        got = nis_pass(src, cfg, ow, oh, scale != 1.0, dt, srtm_in=False, srtm_out=False)
        want = po.nis_scaler(src, ow, oh, cfg, out_dtype=dt) if scale != 1.0 else po.nis_sharpen(src, cfg, out_dtype=dt)
        assert got.dtype == want.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8)), np.dtype(dt).name
