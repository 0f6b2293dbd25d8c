"""The context's pass plan without a GPU: make_plan (csrc/plan.h, what prepare_resources runs) for every use_nis, render
scale 1 and 0.75, output format, source format and flags 0..31 that prepare_resources accepts, against the statement the
GPU tests check the context path with (perceptual_oracle.ctx_bits and ctx_plan) and the rules of include/ovrfsr.h."""
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest

from tests import perceptual_oracle as pq

ROOT = Path(__file__).resolve().parents[1]
RGBA8, BGRA8, RGBA16F, RGBA32F, RGB10A2, BGRX8, RGB32F = range(7)  # ovrfsr_format
FUSED, SRTM, SRTM_NIS, FINITE, PERCEPTUAL = 1, 2, 4, 8, 16        # OVRFSR_FLAG_*
FLOAT_SOURCES = (RGBA16F, RGBA32F, RGB32F)


def _plans():
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("g++ not installed")
    with tempfile.TemporaryDirectory() as d:
        exe = Path(d) / "plan_dump"
        subprocess.check_call([cxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT / "openvr_fsr_b200/csrc"),
                               str(ROOT / "tests/cpp/plan_dump.cpp"), "-o", str(exe)])
        out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    return [tuple(map(int, line.split())) for line in out.splitlines()]


def _accepted(src, out):
    """prepare_resources' output formats (DetermineOutputFormat): 10-bit in <-> 10-bit out, or a float output"""
    return out in (RGBA16F, RGBA32F) or out == (RGB10A2 if src == RGB10A2 else RGBA8)


def test_make_plan_states_the_rule():
    rows = _plans()
    assert len(rows) == 2 * 2 * 5 * 7 * 32
    checked = 0
    for nis, upscale, cfg_out, src, flags, out, paired, fused, mid, srgb, easu, rcas, nis_b in rows:
        if not _accepted(src, out):
            continue
        checked += 1
        where = dict(nis=nis, upscale=upscale, cfg_out=cfg_out, src=src, flags=flags)
        float_src = src in FLOAT_SOURCES
        unorm_out = out in (RGBA8, RGB10A2)
        # ovrfsr.h: SRTM (on the FSR path) and PERCEPTUAL with a float source rule out the pairing and the fused kernel,
        # and make the intermediate RGBA16F for a UNORM output and RGBA32F for a float one
        mapped = float_src and bool(flags & PERCEPTUAL or (flags & SRTM and not nis))
        assert paired == (not nis and upscale and unorm_out and not mapped), where
        assert fused == (paired and bool(flags & FUSED)), where
        assert srgb == (float_src and bool(flags & PERCEPTUAL) and out == RGBA8), where
        if not nis and upscale:
            assert mid == ((RGBA16F if unorm_out else RGBA32F) if mapped else out), where
        # the bits of every pass that runs; a pass that does not run gets none
        want = dict(easu=0, rcas=0, nis=0)
        if float_src:
            e, r, n, _ = pq.ctx_bits(flags, bool(nis), bool(upscale), out == RGBA8)
            want = dict(easu=e, rcas=r, nis=n)
        runs = {"nis"} if nis else ({"easu", "rcas"} if upscale else {"rcas"})
        got = dict(easu=easu, rcas=rcas, nis=nis_b)
        for name in ("easu", "rcas", "nis"):
            assert got[name] == (want[name] if name in runs else 0), (name, where)
        # the whole plan as tests/test_gpu_frame_fuzz.py takes it from the checker's one statement
        e, r, n, pmid, ppaired, pfused, psrgb = pq.ctx_plan(flags, bool(nis), bool(upscale), src, out)
        assert (ppaired, pfused, psrgb) == (bool(paired), bool(fused), bool(srgb)), where
        if not nis and upscale:
            assert mid == {None: out, np.float16: RGBA16F, np.float32: RGBA32F}[pmid], where
        for name, bits in (("easu", e), ("rcas", r), ("nis", n)):
            assert got[name] == (bits if name in runs else 0), (name, where)
    assert checked == 2 * 2 * 32 * 7 * 4  # each source: AUTO, its UNORM output and the two float outputs
