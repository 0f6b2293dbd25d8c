"""The checker's HLSL min / max / saturate, pinned on the host.

D3D11 leaves the sign of min(+0, -0) / max(+0, -0) to the implementation and C leaves it to the C library (glibc
returns the first operand), so the checker states its own rule (oracle/ovr_glue.h): NaN-ignoring, -0 < +0, independent
of operand order -- IEEE 754-2019 minimumNumber / maximumNumber, what sm_90a's FMNMX computes
(tests/test_gpu_minmax_rule.py).  Here: the exported helpers against a plain statement of that rule on every ordered
pair of {+-0, +-1, +-2^-149, +-65504, +-inf, NaNs of both signs, quiet and signalling, with payloads}; the reference shims' min / max / clamp / saturate (oracle/ref_shim) compiled
on their own and compared with the helpers; no libm min / max left in the checker's sources."""
import ctypes as C
import math
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
# the operands of tests/cuda/minmax_probe.cu, in its order: +-0, +-1, +-2^-149, +-65504, NaN, +-inf, and the NaNs
# 0x7f800001 / 0xff800001 (signalling), 0x7fc00001, 0xffc00000.  A Python float cannot carry a signalling float32 NaN
# (the conversion quietens it), so here they are NaNs like the others; the device probe reads their exact bits.
NAN_BITS = (0x7f800001, 0xff800001, 0x7fc00001, 0xffc00000)
VALUES = [0.0, -0.0, 1.0, -1.0, 2.0 ** -149, -(2.0 ** -149), 65504.0, -65504.0, math.nan, math.inf, -math.inf] + \
    [float(np.uint32(b).view(np.float32)) for b in NAN_BITS]


def rule_min(a, b):
    """IEEE 754-2019 minimumNumber"""
    if math.isnan(a):
        return b
    if math.isnan(b):
        return a
    if a != b:
        return a if a < b else b
    return a if math.copysign(1.0, a) < 0 else b


def rule_max(a, b):
    """IEEE 754-2019 maximumNumber"""
    if math.isnan(a):
        return b
    if math.isnan(b):
        return a
    if a != b:
        return a if a > b else b
    return b if math.copysign(1.0, a) < 0 else a


def rule_sat(a):
    return rule_min(1.0, rule_max(0.0, a))


def bits(x):
    """float32 bits, every NaN as one value (the rule says which operand, not which NaN payload)"""
    return "nan" if math.isnan(x) else int(np.float32(x).view(np.uint32))


def test_rule_statement_is_order_independent_and_ignores_nan():
    for a in VALUES:
        for b in VALUES:
            assert bits(rule_min(a, b)) == bits(rule_min(b, a)) and bits(rule_max(a, b)) == bits(rule_max(b, a))
            if not (math.isnan(a) and math.isnan(b)):
                assert not math.isnan(rule_min(a, b)) and not math.isnan(rule_max(a, b))
    assert bits(rule_min(0.0, -0.0)) == 0x80000000 and bits(rule_max(-0.0, 0.0)) == 0
    assert bits(rule_sat(-0.0)) == 0 and bits(rule_sat(math.nan)) == 0
    assert bits(rule_sat(math.inf)) == 0x3f800000 and bits(rule_sat(-math.inf)) == 0
    assert rule_min(math.nan, -math.inf) == -math.inf and rule_max(math.inf, math.nan) == math.inf


def test_checker_helpers_follow_the_rule_on_every_pair():
    from oracle import pyoracle as po
    lib = po.oracle_lib()
    bad = []
    for a in VALUES:
        for b in VALUES:
            for name, got, want in (("min", lib.ovo_hlsl_min(a, b), rule_min(a, b)),
                                    ("max", lib.ovo_hlsl_max(a, b), rule_max(a, b))):
                if bits(got) != bits(want):
                    bad.append(f"{name}({a!r}, {b!r}) = {got!r}, the rule says {want!r}")
        if bits(lib.ovo_hlsl_saturate(a)) != bits(rule_sat(a)):
            bad.append(f"saturate({a!r}) = {lib.ovo_hlsl_saturate(a)!r}, the rule says {rule_sat(a)!r}")
    assert not bad, "\n".join(bad)


SHIM_TU = r"""
#include <cmath>
#include <cstdint>
#include <cstring>
#include "ovr_glue.h"
namespace ref {
#include "ref_shim/amd_shim.h"
}
namespace nis {
#include "ref_shim/hlsl_intrinsics.inc"
}
extern "C" {
float amd_min(float a, float b) { return ref::min(a, b); }
float amd_max(float a, float b) { return ref::max(a, b); }
float amd_min3(float a, float b) { return ref::min(ref::AF3(a, a, a), ref::AF3(b, b, b)).y; }
float amd_max3(float a, float b) { return ref::max(ref::AF3(a, a, a), ref::AF3(b, b, b)).z; }
float amd_clamp(float x, float lo, float hi) { return ref::clamp(x, lo, hi); }
float amd_sat(float a) { return ref::ASatF1(a); }
float amd_min3f1(float a, float b, float c) { return ref::AMin3F1(a, b, c); }
float amd_max3f1(float a, float b, float c) { return ref::AMax3F1(a, b, c); }
float hlsl_min(float a, float b) { return nis::min(a, b); }
float hlsl_max(float a, float b) { return nis::max(a, b); }
float hlsl_sat(float a) { return nis::saturate(a); }
}
"""


@pytest.fixture(scope="module")
def shims(tmp_path_factory):
    """the min / max of the reference shims (oracle/ref_shim), compiled without the reference sources"""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.fail("no C++ compiler: the shims cannot be compiled")
    d = tmp_path_factory.mktemp("shims")
    (d / "shims.cpp").write_text(SHIM_TU)
    so = d / "libshims.so"
    subprocess.run([cxx, "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-std=c++17", "-shared", "-w",
                    f"-I{ROOT / 'oracle'}", "-o", str(so), str(d / "shims.cpp")], check=True)
    lib = C.CDLL(str(so))
    for name, n in (("amd_min", 2), ("amd_max", 2), ("amd_min3", 2), ("amd_max3", 2), ("amd_clamp", 3), ("amd_sat", 1),
                    ("amd_min3f1", 3), ("amd_max3f1", 3), ("hlsl_min", 2), ("hlsl_max", 2), ("hlsl_sat", 1)):
        getattr(lib, name).argtypes = [C.c_float] * n
        getattr(lib, name).restype = C.c_float
    return lib


def test_reference_shims_use_the_checker_rule(shims):
    bad = []

    def check(what, got, want):
        if bits(got) != bits(want):
            bad.append(f"{what} = {got!r}, the checker gives {want!r}")
    for a in VALUES:
        check(f"ASatF1({a!r})", shims.amd_sat(a), rule_sat(a))
        check(f"saturate({a!r})", shims.hlsl_sat(a), rule_sat(a))
        for b in VALUES:
            for name in ("amd_min", "amd_min3", "hlsl_min"):
                check(f"{name}({a!r}, {b!r})", getattr(shims, name)(a, b), rule_min(a, b))
            for name in ("amd_max", "amd_max3", "hlsl_max"):
                check(f"{name}({a!r}, {b!r})", getattr(shims, name)(a, b), rule_max(a, b))
            for c in VALUES:
                check(f"clamp({a!r}, {b!r}, {c!r})", shims.amd_clamp(a, b, c), rule_min(rule_max(a, b), c))
                check(f"AMin3F1({a!r}, {b!r}, {c!r})", shims.amd_min3f1(a, b, c), rule_min(a, rule_min(b, c)))
                check(f"AMax3F1({a!r}, {b!r}, {c!r})", shims.amd_max3f1(a, b, c), rule_max(a, rule_max(b, c)))
    assert not bad, f"{len(bad)} differences, e.g.\n" + "\n".join(bad[:20])


def test_no_libm_min_max_in_the_checker():
    """the checker's bits may not depend on the host's C library: every min / max goes through ovo_min / ovo_max"""
    hits = []
    for p in sorted((ROOT / "oracle").rglob("*")):
        if p.suffix not in (".c", ".h", ".inc", ".cpp"):
            continue
        code = re.sub(r"/\*.*?\*/|//[^\n]*", "", p.read_text(), flags=re.S)
        for m in re.finditer(r"\b(?:std::)?f(?:min|max)[fl]?\s*\(", code):
            hits.append(f"{p.relative_to(ROOT)}: {m.group(0)}")
    assert not hits, "\n".join(hits)
