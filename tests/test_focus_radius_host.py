"""ovrfsr_set_focus_radius / ovrfsr_clear_focus_radius without a GPU: argument validation, the symbols every layer
exports and declares, and that the calls are host work only -- before the first apply and after set_config alike.
That a rejected value leaves the previous one in place shows in the output, so tests/test_gpu_focus_radius.py checks
it."""
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
    p = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=0.75, radius=0.3))  # ovrfsr_create: no GPU work
    yield p
    p.close()


@pytest.mark.parametrize("eye,radius", [(0, math.nan), (1, math.inf), (0, -math.inf), (1, -0.1), (0, 4.0001),
                                        (2, 0.5), (-1, 0.5)])
def test_set_focus_radius_rejects_bad_arguments(pp, eye, radius):
    from openvr_fsr_b200 import _lib as L
    pp.set_focus_radius(0, 1.5)
    with pytest.raises(L.OvrFsrError) as e:
        pp.set_focus_radius(eye, radius)
    assert e.value.status == L.ERR_INVALID


@pytest.mark.parametrize("radius", [0.0, -0.0, 4.0, 0.3, 2.0])
def test_set_focus_radius_accepts_the_closed_range(pp, radius):
    for eye in (0, 1):
        pp.set_focus_radius(eye, radius)


def test_clear_focus_radius_rejects_bad_eye_and_null_ctx(pp):
    from openvr_fsr_b200 import _lib as L
    for eye in (2, -1):
        with pytest.raises(L.OvrFsrError):
            pp.clear_focus_radius(eye)
    assert L.lib().ovrfsr_set_focus_radius(None, 0, .5) == L.ERR_INVALID
    assert L.lib().ovrfsr_clear_focus_radius(None, 0) == L.ERR_INVALID


def test_focus_radius_before_first_apply_and_after_set_config_needs_no_device(pp):
    """host memory only: accepted on a ctx that never touched a GPU, across set_config (whose reset does nothing on an
    uninitialised ctx), and independent of the focus calls; on a machine without a GPU a device call would fail"""
    import dataclasses
    pp.set_focus_radius(0, 0.3)
    pp.set_focus_radius(1, 1.0)
    pp.set_focus(0, 0.4, 0.6)
    pp.clear_focus(0)  # leaves the radius override
    pp.set_config(dataclasses.replace(pp.config, radius=0.7))
    pp.set_focus_radius(0, 4.0)
    pp.clear_focus_radius(1)  # leaves eye 0's override and any focus alone
    pp.clear_focus_radius(1)  # clearing an eye without an override is fine
    pp.set_focus(1, 0.5, 0.5)
    pp.clear_focus_radius(0)
    pp.clear_focus(1)


def test_focus_radius_symbols_exported_and_declared(built_lib):
    from openvr_fsr_b200 import _lib as L
    lib = C.CDLL(str(built_lib))
    header = (ROOT / "include" / "ovrfsr.h").read_text()
    assert re.search(r"OVRFSR_API int ovrfsr_set_focus_radius\(ovrfsr_ctx \*ctx, int eye, float radius\);", header)
    assert re.search(r"OVRFSR_API int ovrfsr_clear_focus_radius\(ovrfsr_ctx \*ctx, int eye\);", header)
    for name in ("ovrfsr_set_focus_radius", "ovrfsr_clear_focus_radius"):
        assert hasattr(lib, name) and name in L.SYMBOLS
    pp_h = (ROOT / "openvr_fsr_b200" / "csrc" / "postprocessor.h").read_text()
    assert "bool SetFocusRadius(EVREye eEye, float radius);" in pp_h and "bool ClearFocusRadius(EVREye eEye);" in pp_h
    from openvr_fsr_b200.api import PostProcessor
    assert callable(PostProcessor.set_focus_radius) and callable(PostProcessor.clear_focus_radius)


def test_cpp_focus_radius_driver_compiles():
    """the drop-in's SetFocusRadius driver builds with a plain host compiler; the GPU test builds and runs the same file"""
    cuda_inc = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda")) / "include"
    if shutil.which("g++") is None or not (cuda_inc / "cuda_runtime.h").exists():
        pytest.skip("g++ or the CUDA headers are not installed")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT / "include"),
                               "-I", str(ROOT / "openvr_fsr_b200/csrc"), "-I", str(cuda_inc), "-c",
                               str(ROOT / "tests/cpp/pp_focus_radius_selftest.cpp"), "-o", str(Path(d) / "pp.o")])
