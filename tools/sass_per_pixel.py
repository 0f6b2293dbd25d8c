"""Dev tool: static SASS instructions per output pixel, per stage, of the two strict kernels the bench.py headline runs
(C2, RGBA8 -> RGBA8, TMA, paired with RCAS), with each stage's opcode mix.  Builds on tools/sass_loops.py's view of a
kernel: every backward branch is a loop, its body size is its static instruction count.

  easu filter  : the per-pixel loop of stage 3 (unrolled x2, so body / 2 pixels)
  rcas decode  : the flat-index tile decode loop (unrolled x4: body / 4 texels), x 66*34 texels / 2048 pixels
  rcas rest    : every instruction outside that loop (the 8-pixel filter column, unrolled), / 8 pixels

Static counts, not executed ones: a count here is what one pass through the code issues.
usage: python tools/sass_per_pixel.py [libovrfsr.so]"""
import re
import subprocess
import sys
from collections import Counter
from pathlib import Path

EASU = "strict_math11easu_kernelILi0ELi0ELi60ELb1ELb1ELb0E"   # <RGBA8, RGBA8, 60, TMA, PAIRED, !ANYIO>
RCAS = "strict_math11rcas_kernelILi0ELi0ELb1ELb1ELb0ELb0E"    # <RGBA8, RGBA8, TMA, PAIRED, !OPQ, !ANYIO>
RCAS_TEXELS_PER_PX = 66 * 34 / (64 * 32)


def _op(s):
    return re.sub(r"^@!?U?P\d+\s+", "", s).split()[0].split(".")[0]


def kernels(so):
    out = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True, check=True).stdout
    res = {}
    for b in re.split(r"\n\s*Function : ", out)[1:]:
        name = b.split("\n", 1)[0].strip()
        if EASU in name or RCAS in name:
            ins = [re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", l) for l in b.split("\n")]
            res["easu" if EASU in name else "rcas"] = [(int(m.group(1), 16), m.group(2).strip()) for m in ins if m]
    return res


def loops(ins):
    """(first, last) instruction index of every backward branch"""
    addr = {a: i for i, (a, _) in enumerate(ins)}
    res = []
    for i, (_, s) in enumerate(ins):
        m = re.search(r"\bBRA(?:\.U)?(?:\.\w+)*\s+(?:!?U?P\d+,\s*)?(0x[0-9a-f]+)", s)
        if m and int(m.group(1), 16) in addr and addr[int(m.group(1), 16)] <= i:
            res.append((addr[int(m.group(1), 16)], i))
    return res


def per_pixel(so):
    k = kernels(so)
    e, r = [s for _, s in k["easu"]], [s for _, s in k["rcas"]]
    # EASU: the innermost large loop is stage 3's filter loop
    el = [(a, b) for a, b in loops(k["easu"]) if b - a + 1 >= 500]
    fa, fb = min(el, key=lambda ab: ab[1] - ab[0])
    # RCAS: the decode loop is its only loop with an STS
    rl = [(a, b) for a, b in loops(k["rcas"]) if any(_op(s) == "STS" for s in r[a:b + 1])]
    da, db = max(rl, key=lambda ab: ab[1] - ab[0])
    rest = r[:da] + r[db + 1:]
    return {
        "easu_filter": {"per_px": (fb - fa + 1) / 2, "mix": Counter(_op(s) for s in e[fa:fb + 1])},
        "easu_total_static": {"per_px": None, "mix": Counter(_op(s) for s in e), "n": len(e)},
        "rcas_decode": {"per_px": (db - da + 1) / 4 * RCAS_TEXELS_PER_PX, "mix": Counter(_op(s) for s in r[da:db + 1])},
        "rcas_rest": {"per_px": len(rest) / 8, "mix": Counter(_op(s) for s in rest)},
        "rcas_total_static": {"per_px": None, "mix": Counter(_op(s) for s in r), "n": len(r)},
    }


if __name__ == "__main__":
    so = Path(sys.argv[1]) if len(sys.argv) > 1 else Path(__file__).resolve().parents[1] / "openvr_fsr_b200" / "libovrfsr.so"
    for stage, v in per_pixel(so).items():
        head = f"{v['per_px']:.1f} per px" if v["per_px"] is not None else f"{v['n']} instructions"
        print(f"{stage:18s} {head}: " + " ".join(f"{o}:{n}" for o, n in v["mix"].most_common(16)))
