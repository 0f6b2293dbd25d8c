"""What sm_90a's min / max / saturate do with signed zeros, subnormals and NaN, against the checker's pinned rule.

tests/cuda/minmax_probe.cu evaluates fminf / fmaxf on every ordered pair of {+-0, +-1, +-2^-149, +-65504, +-inf, NaN,
the signalling NaNs 0x7f800001 / 0xff800001 and the quiet 0x7fc00001 / 0xffc00000},
__saturatef on each value, on each product of two values and on each fused multiply-add of three (the kernels saturate
products and sums), and the nested forms the filters use (EASU's and RCAS's four-texel min / max, EASU's de-ring clamp,
NIS's three-texel ranges, CAS's AMin3F1 / AMax3F1, RCAS's lobe clamp) on every triple / quadruple.  It is built with
-fmad=false (the strict kernels' flag) and -fmad=true (the fast kernels'), its SASS is checked to be FMNMX for min / max
and FADD.SAT / FMUL.SAT / FFMA.SAT for saturate -- the instructions the kernels execute -- and each build runs once.  Every result
must equal the checker's helpers (oracle/ovr_glue.h ovo_min / ovo_max / ovo_sat): IEEE 754-2019 minimumNumber /
maximumNumber, NaN ignored and -0 < +0 whatever the operand order (tests/test_minmax_rule_host.py pins the helpers)."""
import math
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import kernel_ledger as kl
from tests.test_minmax_rule_host import VALUES, bits

pytestmark = pytest.mark.gpu

PROBE = Path(__file__).resolve().parent / "cuda" / "minmax_probe.cu"


def _nvcc():
    p = Path("/usr/local/cuda/bin/nvcc")
    return str(p) if p.exists() else "nvcc"


def _sass_functions(exe):
    out = subprocess.run([kl._tool("cuobjdump"), "-sass", str(exe)], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+([A-Z][A-Z0-9_.]*)", line)
            if m:
                funcs[cur].append(m.group(1))
    return funcs


def _expected(lib, form, ix):
    mn, mx, sat = lib.ovo_hlsl_min, lib.ovo_hlsl_max, lib.ovo_hlsl_saturate
    v = [VALUES[i] for i in ix]
    if form == "min2":
        return mn(v[0], v[1])
    if form == "max2":
        return mx(v[0], v[1])
    if form == "sat":
        return sat(v[0])
    if form == "satmul":
        return sat(float(np.float32(v[0]) * np.float32(v[1])))
    if form == "satfma":  # the float64 product of two floats is exact; no operand set here rounds a float64 midpoint
        return sat(float(np.float32(v[0] * v[1] + v[2])))
    if form == "min3l":
        return mn(mn(v[0], v[1]), v[2])
    if form == "max3l":
        return mx(mx(v[0], v[1]), v[2])
    if form == "min3r":
        return mn(v[0], mn(v[1], v[2]))
    if form == "max3r":
        return mx(v[0], mx(v[1], v[2]))
    if form == "clamp":
        return mn(v[1], mx(v[0], v[2]))
    if form == "lobe":
        return mx(-0.1875, mn(mx(v[0], mx(v[1], v[2])), 0.0))
    if form == "min4":
        return mn(mn(v[0], mn(v[1], v[2])), v[3])
    if form == "max4":
        return mx(mx(v[0], mx(v[1], v[2])), v[3])
    raise AssertionError(form)


@pytest.mark.parametrize("fmad", ["false", "true"])
def test_device_min_max_saturate_follow_the_checker_rule(cuda, tmp_path, fmad):
    from oracle import pyoracle as po
    exe = tmp_path / f"minmax_probe_fmad_{fmad}"
    subprocess.run([_nvcc(), "-O2", "-gencode", "arch=compute_90a,code=sm_90a", f"-fmad={fmad}", "-o", str(exe), str(PROBE)],
                   check=True, capture_output=True, text=True)

    funcs = _sass_functions(exe)
    for name, ops in funcs.items():
        if "probe_sat_forms" in name:
            assert "FMUL.SAT" in ops and "FFMA.SAT" in ops, f"{name}: saturated product / FMA not as FMUL.SAT / FFMA.SAT: {ops}"
        elif "probe_sat" in name:
            assert "FADD.SAT" in ops, f"{name}: saturate not as FADD.SAT: {ops}"
        else:
            assert "FMNMX" in ops, f"{name}: no FMNMX: {ops}"
            assert not any(o.startswith(("FSEL", "FSETP", "FSET")) for o in ops), f"{name}: min / max not as FMNMX: {ops}"
    assert len(funcs) == 5, sorted(funcs)

    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    lib = po.oracle_lib()
    counts, bad = {}, []
    with np.errstate(invalid="ignore", over="ignore"):  # inf * 0, inf - inf and 65504^2 are operands here
        for line in r.stdout.splitlines():
            form, *idx, word = line.split()
            ix = [int(i) for i in idx]
            got = float(np.uint32(int(word, 16)).view(np.float32))
            want = _expected(lib, form, ix)
            counts[form] = counts.get(form, 0) + 1
            if bits(got) != bits(want):
                bad.append(f"{form}{tuple(VALUES[i] for i in ix)}: device {word} ({got!r}), checker {want!r}")
    n = len(VALUES)
    assert counts == {"min2": n * n, "max2": n * n, "sat": n, "min3l": n ** 3, "max3l": n ** 3, "min3r": n ** 3,
                      "max3r": n ** 3, "clamp": n ** 3, "lobe": n ** 3, "min4": n ** 4, "max4": n ** 4, "satmul": n * n,
                      "satfma": n ** 3}, counts
    # what the device did on the ties the rule is about, printed for the record
    pairs = {(f, tuple(map(int, i))): w for f, *i, w in (ln.split() for ln in r.stdout.splitlines())}
    print(f"-fmad={fmad}: fminf(+0,-0)={pairs[('min2', (0, 1))]} fminf(-0,+0)={pairs[('min2', (1, 0))]} "
          f"fmaxf(+0,-0)={pairs[('max2', (0, 1))]} fmaxf(-0,+0)={pairs[('max2', (1, 0))]} "
          f"__saturatef(-0)={pairs[('sat', (1,))]} __saturatef(-0*1)={pairs[('satmul', (1, 2))]} "
          f"__saturatef(fmaf(-1,+0,-0))={pairs[('satfma', (3, 0, 1))]} fminf(NaN,-1)={pairs[('min2', (8, 3))]}; "
          f"{sum(counts.values())} results, {len(bad)} differ from the checker")
    assert not bad, f"{len(bad)} results differ from the checker, e.g.\n" + "\n".join(bad[:20])
    assert not math.isnan(float(np.uint32(int(pairs[("min2", (8, 3))], 16)).view(np.float32)))
