"""The kernel ledger: every __global__ function the built library ships, as normalised keys.

A key is (mode, kernel, args): mode is "strict" / "fast" for the kernels of the two math-mode builds (the
ovrfsr::strict_math / ovrfsr::fast_math inline namespaces, device_common.cuh) and "" for the kernels that exist once:
the MSAA resolve and the division self-test (strict build only, outside those namespaces) and the host-entry helpers
of capi.cu; args are the template arguments as ints (bools as 0 / 1).  The same key comes out of cu++filt's spelling
(`easu_kernel<(int)0, (int)2, (int)60, (bool)1, ...>`) and of __cxa_demangle's, which torch.profiler reports
(`easu_kernel<0, 2, 60, true, ...>`), so a launch recorded on the GPU can be matched against the shipped list.

expected_keys() restates the launch switches of csrc/kernels.inc as the set of instantiations they produce; the
closed-form count of each family sits next to the switch it mirrors there."""
from __future__ import annotations

import re
import shutil
import subprocess
from collections import Counter

RGBA8, BGRA8, RGBA16F, RGBA32F, RGB10A2 = 0, 1, 2, 3, 4
FORMAT_NAMES = {RGBA8: "RGBA8", BGRA8: "BGRA8", RGBA16F: "RGBA16F", RGBA32F: "RGBA32F", RGB10A2: "RGB10A2"}
PACKED32 = (RGBA8, BGRA8, RGB10A2)  # 4-byte texels: the formats a TMA tensor map can describe
# OVRFSR_FORMAT_SWITCH: {RGBA8, BGRA8, RGBA16F, RGBA32F} -> {RGBA8, RGBA16F, RGBA32F}; RGB10A2 -> {RGB10A2, RGBA16F, RGBA32F}
PAIRS = [(i, o) for i in (RGBA8, BGRA8, RGBA16F, RGBA32F) for o in (RGBA8, RGBA16F, RGBA32F)] + \
        [(RGB10A2, o) for o in (RGB10A2, RGBA16F, RGBA32F)]
MODES = ("strict", "fast")

# template parameter names per kernel, in declaration order
PARAMS = {
    "easu_kernel": ("FIN", "FOUT", "TW", "TMA", "PAIRED", "ANYIO"),
    "rcas_kernel": ("FIN", "FOUT", "TMA", "PAIRED", "OPQ", "ANYIO"),
    "nis_scaler_kernel": ("FIN", "FOUT", "TMA", "ANYIO"),
    "nis_sharpen_kernel": ("FIN", "FOUT", "ANYIO"),
    "cas_sharpen_kernel": ("FIN", "FOUT", "TMA"),
    "cas_scale_kernel": ("FIN", "FOUT"),
    "fsr_fused_kernel": ("FIN", "FMID", "FOUT", "TW", "TMA"),
    "resolve_msaa_kernel": ("FMT", "S"),
    "repitch_rows_kernel": (),
    "expand_rgb32f_kernel": (),
    "rcas_rcp_selftest_kernel": (),
    "nis_div_selftest_kernel": (),
}

# closed forms of the family sizes (the comments beside the switches in csrc/kernels.inc state the same products)
FAMILY_COUNTS = {
    "easu_kernel": 2 * 2 * 2 * (15 + 5 + 9 + 3),        # modes x TW x ANYIO x (plain + paired + TMA + TMA paired)
    "rcas_kernel": 2 * 2 * (15 + 9 + 2 + 2 + 3 + 3),    # modes x ANYIO x (plain + TMA + paired + TMA paired + OPQ + TMA OPQ)
    "nis_scaler_kernel": 2 * 2 * (15 + 9),              # modes x ANYIO x (plain + TMA)
    "nis_sharpen_kernel": 2 * 2 * 15,                   # modes x ANYIO x pairs
    "cas_sharpen_kernel": 2 * (15 + 9),                 # modes x (plain + TMA)
    "cas_scale_kernel": 2 * 15,                         # modes x pairs
    "fsr_fused_kernel": 2 * 2 * (5 + 3),                # modes x TW x (plain + TMA), FOUT = FMID = the UNORM intermediate
    "resolve_msaa_kernel": 4 * 4 - 2,                   # formats x S in {0, 2, 4, 8}, minus S = 2 for the 4-byte formats
    "repitch_rows_kernel": 1,
    "expand_rgb32f_kernel": 1,
    "rcas_rcp_selftest_kernel": 2,                      # one per math mode
    "nis_div_selftest_kernel": 1,                       # strict only
}

_KERNEL = re.compile(r"(?:\b(strict|fast)_math::)?(\w+_kernel)(?:<([^<>]*)>)?\(")


def _arg(tok: str) -> int:
    tok = re.sub(r"^\((?:unsigned )?(?:int|bool|long)\)", "", tok.strip())
    if tok in ("true", "false"):
        return int(tok == "true")
    return int(tok.rstrip("uU"))


def normalise(demangled: str):
    """(mode, kernel, args) of a demangled kernel name in cu++filt's or __cxa_demangle's spelling; None when the name
    is not one of this library's kernels."""
    m = _KERNEL.search(demangled)
    if not m or m.group(2) not in PARAMS:
        return None
    args = tuple(_arg(a) for a in m.group(3).split(",")) if m.group(3) else ()
    if len(args) != len(PARAMS[m.group(2)]):
        raise ValueError(f"{m.group(2)} has {len(args)} template arguments, the ledger knows {len(PARAMS[m.group(2)])}: {demangled}")
    return (m.group(1) or "", m.group(2), args)


def describe(key) -> str:
    mode, kernel, args = key
    parts = []
    for name, v in zip(PARAMS[kernel], args):
        parts.append(f"{name}={FORMAT_NAMES.get(v, v)}" if name in ("FIN", "FOUT", "FMID", "FMT") else f"{name}={v}")
    return f"{mode + ':' if mode else ''}{kernel}<{', '.join(parts)}>"


def _tool(name: str) -> str:
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not shutil.which(exe):
        raise FileNotFoundError(name)
    return exe


def mangled_kernels(lib_path) -> list[str]:
    """The .text.<mangled> section names of every cubin in the library (cuobjdump -elf)"""
    r = subprocess.run([_tool("cuobjdump"), "-elf", str(lib_path)], capture_output=True, text=True, timeout=900)
    if r.returncode != 0:
        raise RuntimeError(f"cuobjdump -elf failed: {r.stderr[-500:]}")
    return sorted(set(re.findall(r"\s\.text\.(_Z\w+)", r.stdout)))


def demangle(names: list[str]) -> list[str]:
    r = subprocess.run([_tool("cu++filt")], input="\n".join(names) + "\n", capture_output=True, text=True, timeout=300)
    if r.returncode != 0:
        raise RuntimeError(f"cu++filt failed: {r.stderr[-500:]}")
    out = r.stdout.splitlines()
    assert len(out) == len(names), "cu++filt returned a different number of lines"
    return out


def ledger(lib_path) -> dict:
    """{key: demangled name} for every __global__ function of the library; a kernel the ledger cannot parse raises"""
    out = {}
    for name in demangle(mangled_kernels(lib_path)):
        key = normalise(name)
        if key is None:
            raise ValueError(f"a kernel the ledger does not know: {name}")
        assert key not in out, f"two functions normalise to {key}"
        out[key] = name
    return out


def expected_keys() -> set:
    """The instantiations the launch switches of csrc/kernels.inc and csrc/capi.cu can produce"""
    keys = set()
    paired = [(i, o) for i, o in PAIRS if o in (RGBA8, RGB10A2)]
    for m in MODES:
        for anyio in (0, 1):
            for tw in (60, 72):
                for tma in (0, 1):
                    for (i, o) in PAIRS:
                        if tma and i not in PACKED32:
                            continue
                        keys.add((m, "easu_kernel", (i, o, tw, tma, 0, anyio)))
                        if (i, o) in paired:
                            keys.add((m, "easu_kernel", (i, o, tw, tma, 1, anyio)))
            for tma in (0, 1):
                for (i, o) in PAIRS:
                    if tma and i not in PACKED32:
                        continue
                    keys.add((m, "rcas_kernel", (i, o, tma, 0, 0, anyio)))
                    if i == o and i in (RGBA8, RGB10A2):
                        keys.add((m, "rcas_kernel", (i, o, tma, 1, 0, anyio)))
                    if i == BGRA8:
                        keys.add((m, "rcas_kernel", (i, o, tma, 0, 1, anyio)))
                    keys.add((m, "nis_scaler_kernel", (i, o, tma, anyio)))
            for (i, o) in PAIRS:
                keys.add((m, "nis_sharpen_kernel", (i, o, anyio)))
        for (i, o) in PAIRS:
            keys.add((m, "cas_scale_kernel", (i, o)))
            for tma in (0, 1):
                if tma and i not in PACKED32:
                    continue
                keys.add((m, "cas_sharpen_kernel", (i, o, tma)))
        for fin in (RGBA8, BGRA8, RGBA16F, RGBA32F, RGB10A2):
            mid = RGB10A2 if fin == RGB10A2 else RGBA8
            for tw in (60, 72):
                for tma in (0, 1):
                    if tma and fin not in PACKED32:
                        continue
                    keys.add((m, "fsr_fused_kernel", (fin, mid, mid, tw, tma)))
        keys.add((m, "rcas_rcp_selftest_kernel", ()))
    for fmt in (RGBA8, RGBA16F, RGBA32F, RGB10A2):
        for s in (0, 2, 4, 8):
            if s == 2 and fmt in PACKED32:
                continue
            keys.add(("", "resolve_msaa_kernel", (fmt, s)))
    keys |= {("", "repitch_rows_kernel", ()), ("", "expand_rgb32f_kernel", ()), ("", "nis_div_selftest_kernel", ())}
    return keys


def family_counts(keys) -> Counter:
    return Counter(k[1] for k in keys)
