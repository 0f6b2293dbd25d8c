"""ovrfsr_set_sharpness / ovrfsr_clear_sharpness without a GPU: argument validation, the symbols every layer exports and
declares, and that the calls are host work only -- before the first apply and across set_config alike.  That a
rejected value leaves the previous one in place shows in the output, so tests/test_gpu_live_sharpness.py checks that
too."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture
def pp(built_lib):
    import openvr_fsr_b200 as ovr
    p = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=0.75, sharpness=0.9))  # ovrfsr_create: no GPU work
    yield p
    p.close()


@pytest.mark.parametrize("sharpness", [math.nan, math.inf, -math.inf, -0.01, 1.01])
def test_set_sharpness_rejects_bad_values(pp, sharpness):
    from openvr_fsr_b200 import _lib as L
    pp.set_sharpness(0.4)
    with pytest.raises(L.OvrFsrError) as e:
        pp.set_sharpness(sharpness)
    assert e.value.status == L.ERR_INVALID


@pytest.mark.parametrize("sharpness", [0.0, -0.0, 1.0, 0.5, 0.37])
def test_set_sharpness_accepts_the_closed_range(pp, sharpness):
    pp.set_sharpness(sharpness)


def test_sharpness_null_ctx_is_rejected(built_lib):
    from openvr_fsr_b200 import _lib as L
    assert L.lib().ovrfsr_set_sharpness(None, 0.5) == L.ERR_INVALID
    assert L.lib().ovrfsr_clear_sharpness(None) == L.ERR_INVALID


def test_sharpness_before_first_apply_and_after_set_config_needs_no_device(pp):
    """host memory only: accepted on a ctx that never touched a GPU, across set_config (whose reset does nothing on an
    uninitialised ctx), alongside the focus and radius calls; on a machine without a GPU a device call would fail"""
    import dataclasses
    pp.set_sharpness(0.2)
    pp.set_focus(0, 0.4, 0.6)
    pp.set_focus_radius(1, 1.0)
    pp.set_config(dataclasses.replace(pp.config, sharpness=0.3))
    pp.set_sharpness(1.0)
    pp.clear_focus(0)
    pp.clear_focus_radius(1)  # the sharpness override stays
    pp.clear_sharpness()
    pp.clear_sharpness()  # clearing without an override is fine


def test_sharpness_symbols_exported_and_declared(built_lib):
    from openvr_fsr_b200 import _lib as L
    lib = C.CDLL(str(built_lib))
    header = (ROOT / "include" / "ovrfsr.h").read_text()
    assert re.search(r"OVRFSR_API int ovrfsr_set_sharpness\(ovrfsr_ctx \*ctx, float sharpness\);", header)
    assert re.search(r"OVRFSR_API int ovrfsr_clear_sharpness\(ovrfsr_ctx \*ctx\);", header)
    for name in ("ovrfsr_set_sharpness", "ovrfsr_clear_sharpness"):
        assert hasattr(lib, name) and name in L.SYMBOLS
    pp_h = (ROOT / "openvr_fsr_b200" / "csrc" / "postprocessor.h").read_text()
    assert "bool SetSharpness(float sharpness);" in pp_h and "bool ClearSharpness();" in pp_h
    from openvr_fsr_b200.api import PostProcessor
    assert callable(PostProcessor.set_sharpness) and callable(PostProcessor.clear_sharpness)


def test_cpp_sharpness_driver_compiles():
    """the drop-in's SetSharpness driver builds with a plain host compiler; the GPU test builds and runs the same file"""
    cuda_inc = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda")) / "include"
    if shutil.which("g++") is None or not (cuda_inc / "cuda_runtime.h").exists():
        pytest.skip("g++ or the CUDA headers are not installed")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT / "include"),
                               "-I", str(ROOT / "openvr_fsr_b200/csrc"), "-I", str(cuda_inc), "-c",
                               str(ROOT / "tests/cpp/pp_sharpness_selftest.cpp"), "-o", str(Path(d) / "pp.o")])
