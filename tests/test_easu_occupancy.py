"""Resident CTAs per SM of the headline EASU kernels, from the built library's resource usage (cuobjdump -res-usage, no
GPU needed), the way tests/test_sass_budget.py pins their instruction counts.  Strict EASU is issue-latency-bound: its
speed follows the warps resident per SM, and four 256-thread CTAs fit only while the registers stay at 64 or fewer and
the C2 tile at 32 bytes per texel (colour and features; the luma plane and the TMA landing zone share the feature tile).
Fast math needs ~78 registers, so three.  H100 (sm_90): 65,536 registers and 228 KiB of
shared memory per SM, 1 KiB of it reserved per CTA; registers are allocated per warp in 256s, shared memory in 128 B."""
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po

REGS_PER_SM, SMEM_PER_SM, SMEM_RESERVED_PER_CTA, THREADS = 65536, 228 * 1024, 1024, 256
C2 = (1683, 1869, 2244, 2492)  # bench.py's workload: in w, in h, out w, out h
# easu_kernel<RGBA8, RGBA8, 60, TMA, PAIRED, !ANYIO>: what bench.py's two-pass headline launches
HEADLINE = "11easu_kernelILi0ELi0ELi60ELb1ELb1ELb0E"


@pytest.fixture(scope="module")
def usage(built_lib):
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    try:
        out = subprocess.run([exe, "-res-usage", str(built_lib)], capture_output=True, text=True, check=True).stdout
    except FileNotFoundError:
        pytest.skip("cuobjdump not installed")
    res = {}
    for name, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out):
        res[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    return res


def c2_dynamic_smem():
    """easu_launch_t's dynamic shared memory at C2 with a TMA source (csrc/kernels.inc)"""
    w = po.upscale_constants(0, True, *C2, radius=2.0).words()
    c0x, c0y = w[:2].view(np.float32)
    tile_w = (int(np.ceil(np.float32(63) * c0x)) + 5 + 3) & ~3
    tile_h = int(np.ceil(np.float32(31) * c0y)) + 5
    cols = tile_w + 4
    stride = 60 if cols <= 60 else 72
    assert stride == 60, "C2 runs the 60-texel stride"
    return stride * tile_h * 32


@pytest.mark.parametrize("mode, ctas", [("strict_math", 4), ("fast_math", 3)])
def test_headline_easu_fits_its_ctas_per_sm(usage, mode, ctas):
    (ru,) = [v for k, v in usage.items() if mode + HEADLINE in k]
    regs = (ru["REG"] + 7) // 8 * 8
    assert regs * THREADS * ctas <= REGS_PER_SM, ru
    per_cta = (c2_dynamic_smem() + ru["SHARED"] + SMEM_RESERVED_PER_CTA + 127) // 128 * 128
    assert per_cta * ctas <= SMEM_PER_SM, (per_cta, ru)


def test_no_easu_instantiation_spills(usage):
    easu = {k: v for k, v in usage.items() if "11easu_kernelI" in k}
    assert len(easu) == 256
    assert not {k: v for k, v in easu.items() if v["STACK"] or v["LOCAL"]}
