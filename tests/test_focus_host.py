"""ovrfsr_set_focus / ovrfsr_clear_focus without a GPU: argument validation, the symbols every layer exports and
declares, and that setting a focus before the first apply is host work only."""
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


@pytest.mark.parametrize("eye,x,y", [(2, .5, .5), (-1, .5, .5), (0, math.nan, .5), (1, .5, math.nan), (0, math.inf, .5),
                                     (1, .5, -math.inf), (0, -0.01, .5), (1, .5, 1.01), (0, 1.5, 0.0)])
def test_set_focus_rejects_bad_arguments(pp, eye, x, y):
    from openvr_fsr_b200 import _lib as L
    with pytest.raises(L.OvrFsrError) as e:
        pp.set_focus(eye, x, y)
    assert e.value.status == L.ERR_INVALID


def test_clear_focus_rejects_bad_eye_and_null_ctx(pp):
    from openvr_fsr_b200 import _lib as L
    for eye in (2, -1):
        with pytest.raises(L.OvrFsrError):
            pp.clear_focus(eye)
    assert L.lib().ovrfsr_set_focus(None, 0, .5, .5) == L.ERR_INVALID
    assert L.lib().ovrfsr_clear_focus(None, 0) == L.ERR_INVALID


def test_set_focus_before_first_apply_needs_no_device(pp):
    """host memory only: accepted on a ctx that never touched a GPU (the corners of [0, 1] included), and clearing
    works the same way; on a machine without a GPU a device call would fail"""
    for eye, (x, y) in ((0, (0.0, 0.0)), (1, (1.0, 1.0)), (0, (0.3, 0.7)), (1, (-0.0, 0.5))):
        pp.set_focus(eye, x, y)
    pp.clear_focus(0)
    pp.clear_focus(1)
    pp.clear_focus(1)  # clearing an eye without a focus is fine


def test_focus_symbols_exported_and_declared(built_lib):
    from openvr_fsr_b200 import _lib as L
    lib = C.CDLL(str(built_lib))
    header = (ROOT / "include" / "ovrfsr.h").read_text()
    for name in ("ovrfsr_set_focus", "ovrfsr_clear_focus"):
        assert hasattr(lib, name) and name in L.SYMBOLS
        assert re.search(r"OVRFSR_API int " + name + r"\(ovrfsr_ctx \*ctx, int eye", header)
    pp_h = (ROOT / "openvr_fsr_b200" / "csrc" / "postprocessor.h").read_text()
    assert "bool SetFocus(EVREye eEye, float x, float y);" in pp_h and "bool ClearFocus(EVREye eEye);" in pp_h
    from openvr_fsr_b200.api import PostProcessor
    assert callable(PostProcessor.set_focus) and callable(PostProcessor.clear_focus)


def test_cpp_focus_driver_compiles():
    """the drop-in's SetFocus driver builds with a plain host compiler; the GPU test builds and runs the same file"""
    cuda_inc = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda")) / "include"
    if shutil.which("g++") is None or not (cuda_inc / "cuda_runtime.h").exists():
        pytest.skip("g++ or the CUDA headers are not installed")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT / "include"),
                               "-I", str(ROOT / "openvr_fsr_b200/csrc"), "-I", str(cuda_inc), "-c",
                               str(ROOT / "tests/cpp/pp_focus_selftest.cpp"), "-o", str(Path(d) / "pp.o")])
