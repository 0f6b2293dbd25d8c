"""OVRFSR_FLAG_SRTM_NIS on the H100: AMD's reversible tone map around NVScaler and NVSharpen, against the checker.

The checker is tests/srtm_oracle.py's F on the decoded source (an RGBA32F copy), the unchanged restated pass
(oracle/pyoracle.py's nis_scaler / nis_sharpen) into RGBA32F, G, and the oracle's own encode into the target format.

Stateless: every float-source nis_scaler_kernel / nis_sharpen_kernel instantiation the ledger lists, through
ovrfsr_dispatch_nis_scaler_ex / _sharpen_ex with each pass bit alone and both, on signed / HDR / +-65504 content and on
in-domain HDR content.  Strict math is compared to the bit on both.  Fast math is bounded on the in-domain content only,
in tone-mapped space (F in float64 on both sides, since G amplifies any difference near 1) for float targets and in LSB
for RGBA8; out-of-domain values that reach G's 1/32768 floor have no fast-math bound (see tests/test_gpu_srtm.py).

The context path: C2-shaped RGBA16F, RGBA32F, RGB32F and 4x-multisampled RGBA16F eyes at peaks 4 and 1000, NVScaler
(renderScale 0.75) and NVSharpen (renderScale 1), into RGBA8, RGBA16F and RGBA32F, radius 0.5 / 2.0 with the debug tint
on and off, every apply entry, CUDA-array source and destination, a shared texture, a graph replay, a focus, a radius
override and a sharpness override; strict output equal to the checker, fast output within the bound measured on an
H100; UNORM sources and the FSR path unchanged by the bit; the C++ drop-in's Config::srtmNis."""
import dataclasses
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import kernel_ledger as kl
from tests import srtm_oracle as so
from tests import test_gpu_float_signed as fs
from tests import test_gpu_srtm as gs
from tests import test_gpu_variant_matrix as vm

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
FLAG_SETS = [(1, 0), (0, 1), (1, 1)]
NT = os.cpu_count() or 1
SHARP = 0.8
# fast math, measured on one H100 80GB HBM3 (DESIGN.md section 4), with headroom: tone-mapped space / RGBA8 codes
FAST_TONE, FAST_LSB = 2e-3, 4
MAXIMA = {}


def nis_pass(src, cfg, out_w, out_h, scaler, out_dtype, srtm_in=True, srtm_out=True):
    """the checker of one NIS pass with the tone map: F on the decoded source, the restated pass into RGBA32F, G, the
    oracle's encode into out_dtype"""
    from oracle import pyoracle as po
    s = np.ascontiguousarray(src.astype(np.float32))  # binary16 -> binary32 is exact, as the decodes
    if srtm_in:
        s[..., :3] = so.srtm(s[..., :3])
    o = po.nis_scaler(s, out_w, out_h, cfg, out_dtype=np.float32, nthreads=NT) if scaler else \
        po.nis_sharpen(s, cfg, out_dtype=np.float32, nthreads=NT)
    if srtm_out:
        o[..., :3] = so.srtm(o[..., :3], inverse=True)
    return so.encode(o, out_dtype)


def _tone_err(got, want):
    return gs._tone_err(got, want)


# ---- stateless dispatches, ledger-driven ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nis_keys(built_lib):
    keys = sorted(k for k in kl.ledger(built_lib) if k[1] in ("nis_scaler_kernel", "nis_sharpen_kernel") and
                  dict(zip(kl.PARAMS[k[1]], k[2]))["FIN"] in fs.FLOAT_FORMATS)
    assert len(keys) == 2 * 2 * 2 * 6, len(keys)  # modes x kernels x ANYIO x (float source, output) pairs
    return keys


def _run_key(key, dev, content, flags):
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    mode, kernel, args = key
    p = dict(zip(kl.PARAMS[kernel], args))
    fin, fout, anyio = p["FIN"], p["FOUT"], p["ANYIO"]
    mm = vm._mathmode(mode)
    src = content(fin, vm.W, vm.H, vm._seed(key))
    sin, sout = flags
    scaler = kernel == "nis_scaler_kernel"
    ow, oh = ovr.output_size(vm.W, vm.H, 0.75) if scaler else (vm.W, vm.H)
    cfg, ok = po.nis_config(not scaler, 0, True, vm.W, vm.H, ow, oh, proj=vm.PROJ, radius=vm.RADIUS, sharpness=SHARP,
                            debug=vm._debug(args))
    assert ok
    fn = ovr.nis_scaler if scaler else ovr.nis_sharpen
    want = nis_pass(src, cfg, ow, oh, scaler, vm._np_dtype(fout), sin, sout)
    layouts = [("array", ["pitched", "array"])] if anyio else [("tight", ["pitched"])]
    out = []
    for where, kinds in layouts:
        s = vm._place(src, fin, where, dev)
        for kind, d in zip(kinds, vm._outputs(fout, ow, oh, dev, kinds)):
            n0 = ovr.kernel_launches()
            fn(s, d, bytes(cfg), mm, srtm_in=sin, srtm_out=sout)
            assert ovr.kernel_launches() == n0 + 1
            out.append((f"{where}->{kind}", vm._host(d)))
    return want, out, fout


@pytest.mark.parametrize("kernel", ["nis_scaler_kernel", "nis_sharpen_kernel"])
@pytest.mark.parametrize("content", ["signed", "in_domain"])
def test_dispatch_ex_matches_the_oracle(cuda, nis_keys, kernel, content):
    gen = fs.signed_content if content == "signed" else gs.in_domain
    failures, n = [], 0
    for key in (k for k in nis_keys if k[1] == kernel):
        if key[0] == "fast" and content == "signed":
            continue  # out-of-domain values through G: strict math pins them, fast math has no bound there
        for flags in FLAG_SETS:
            want, outs, fout = _run_key(key, cuda, gen, flags)
            for label, got in outs:
                n += 1
                name = f"{kl.describe(key)} in={flags[0]} out={flags[1]} [{label}]"
                if key[0] == "strict":
                    msg, err = vm._check(got, want, fout, "strict", False)
                elif flags == (0, 1):
                    # G alone on a pass over linear light: its input leaves [0, 1) (HDR texels, negative overshoot), so
                    # values meet G's 1/32768 floor and a last-bit difference comes out x32768 (measured on H100: 7.0 in
                    # tone-mapped space).  Strict math above pins these outputs; fast math only the NaN classes.
                    g, w = got.astype(np.float64), want.astype(np.float64)
                    msg = None if np.array_equal(np.isnan(g), np.isnan(w)) else "fast: NaN where the oracle has none"
                    err = 0.0
                elif fout in fs.FLOAT_FORMATS:
                    err, same = _tone_err(got, want)
                    msg = None if same and err <= FAST_TONE else f"tone-mapped error {err:.3g} (NaN classes agree: {same})"
                else:
                    err = float(np.abs(got.astype(np.int32) - want.astype(np.int32)).max())
                    msg = None if err <= FAST_LSB else f"{err:.0f} LSB"
                if key[0] == "fast":
                    k = f"{kernel} -> {kl.FORMAT_NAMES[fout]}"
                    MAXIMA[k] = max(MAXIMA.get(k, 0.0), err)
                if msg:
                    failures.append(f"{name}: {msg}")
    print(f"\n{kernel} / {content}: {n} outputs compared; fast maxima: " +
          ", ".join(f"{k}: {v:.3g}" for k, v in sorted(MAXIMA.items()) if k.startswith(kernel)))
    assert not failures, f"{len(failures)} failures:\n" + "\n".join(failures[:20])


@pytest.mark.parametrize("scaler", [True, False], ids=["scaler", "sharpen"])
def test_zero_flags_launch_the_plain_dispatch(cuda, scaler):
    """pass_flags == 0 through the _ex entry points gives the bytes of the plain entry points"""
    import ctypes as C
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    from oracle import pyoracle as po
    src = fs.signed_content(kl.RGBA16F, vm.W, vm.H, 3)
    ow, oh = ovr.output_size(vm.W, vm.H, 0.75) if scaler else (vm.W, vm.H)
    cfg, _ = po.nis_config(not scaler, 0, True, vm.W, vm.H, ow, oh, proj=vm.PROJ, radius=vm.RADIUS, sharpness=SHARP)
    s = torch.from_numpy(src).to(cuda)
    a, b = (torch.empty((oh, ow, 4), dtype=torch.float16, device=cuda) for _ in range(2))
    (ovr.nis_scaler if scaler else ovr.nis_sharpen)(s, a, bytes(cfg), ovr.MATH_FAST)
    si, di = ovr.image_of(s), ovr.image_of(b)
    buf = C.create_string_buffer(bytes(cfg), 256)
    fn = L.lib().ovrfsr_dispatch_nis_scaler_ex if scaler else L.lib().ovrfsr_dispatch_nis_sharpen_ex
    assert fn(C.byref(si), C.byref(di), buf, ovr.MATH_FAST, 0, torch.cuda.current_stream().cuda_stream) == L.OK
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---- the context path ----------------------------------------------------------------------------------------------
SCALES = {"scaler": 0.75, "sharpen": 1.0}


def _eyes(peak, dtype=np.float16, full=False):
    (left, right), _ = gs._eyes("C2", peak, full)
    return left.astype(dtype), right.astype(dtype)


def _chain(src, eye, one, scale, radius, out_dtype, proj=(.5, .5, .5, .5), debug=False, sharp=SHARP, srtm=True):
    """the checker of a ctx's NIS pass: NVScaler below scale 1, NVSharpen at scale 1; src is what the pass reads"""
    from oracle import pyoracle as po
    h, w = src.shape[:2]
    ow, oh = po.output_size(w, h, scale)
    cfg, ok = po.nis_config(scale == 1.0, eye, one, w, h, ow, oh, proj=proj, radius=radius, sharpness=sharp, debug=debug)
    assert ok
    return nis_pass(src, cfg, ow, oh, scale != 1.0, out_dtype, srtm, srtm)


def _cfg(scale, radius, out_dtype, strict=True, debug=False, srtmNis=True, **kw):
    import openvr_fsr_b200 as ovr
    return ovr.Config(fsrEnabled=True, useNis=True, renderScale=scale, sharpness=SHARP, radius=radius, debugMode=debug,
                      outputFormat=gs._out_fmt(out_dtype), mathMode=ovr.MATH_STRICT if strict else ovr.MATH_FAST,
                      srtmNis=srtmNis, **kw)


_same = gs._same


@pytest.mark.parametrize("peak", [4.0, 1000.0])
@pytest.mark.parametrize("path", list(SCALES))
def test_ctx_strict_entries(cuda, path, peak):
    """every apply entry, strict, against the checker"""
    import torch
    import openvr_fsr_b200 as ovr
    scale = SCALES[path]
    left, right = _eyes(peak)
    t = [torch.from_numpy(e).to(cuda) for e in (left, right)]
    h, w = left.shape[:2]
    ow, oh = ovr.output_size(w, h, scale)
    pp = ovr.PostProcessor(_cfg(scale, 0.5, np.uint8))
    outs = pp.apply_pair(t[0], t[1])
    for e in (0, 1):
        _same(outs[e].cpu().numpy(), _chain((left, right)[e], e, True, scale, 0.5, np.uint8), f"apply_pair eye {e}")
    pp.set_config(_cfg(scale, 2.0, np.float16, debug=True))
    for e in (0, 1):
        _same(pp.apply(e, t[e]).cpu().numpy(), _chain((left, right)[e], e, True, scale, 2.0, np.float16, debug=True), f"apply eye {e}")
    # apply_into, CUDA-array source and destination
    pp.set_config(_cfg(scale, 0.5, np.float32))
    src_a = ovr.ArrayImage(w, h, ovr.FORMAT_RGBA16F).upload(t[1])
    dst_a = ovr.ArrayImage(ow, oh, ovr.FORMAT_RGBA32F)
    pp.apply_into(1, src_a, dst_a)
    _same(dst_a.download().cpu().numpy(), _chain(right, 1, True, scale, 0.5, np.float32), "apply_into array->array")
    # apply_pair_into
    pp.set_config(_cfg(scale, 0.5, np.uint8, debug=True))
    dl, dr = (ovr.alloc_image(ow, oh, torch.uint8, cuda) for _ in range(2))
    pp.apply_pair_into(t[0], t[1], dl, dr)
    for e, d in ((0, dl), (1, dr)):
        _same(d.cpu().numpy(), _chain((left, right)[e], e, True, scale, 0.5, np.uint8, debug=True), f"apply_pair_into eye {e}")
    # apply_host, pinned memory
    hs = torch.from_numpy(left).pin_memory()
    hd = torch.empty((oh, ow, 4), dtype=torch.uint8).pin_memory()
    pp.apply_host(0, hs, hd)
    torch.cuda.synchronize()
    _same(hd.numpy(), _chain(left, 0, True, scale, 0.5, np.uint8, debug=True), "apply_host")
    for a in (src_a, dst_a):
        a.release()
        a.close()
    pp.close()


def _source(kind, peak):
    """(what the ctx is given, its format tag, MSAA sample count, what the pass reads) for one eye"""
    from oracle import frontend as fe
    left, _ = _eyes(peak, np.float32 if kind in ("RGBA32F", "RGB32F") else np.float16)
    if kind == "RGB32F":
        rgb = np.ascontiguousarray(left[..., :3])
        reads = np.concatenate([rgb, np.ones_like(rgb[..., :1])], axis=-1)
        return rgb, vm.RGB32F, 1, reads
    if kind == "MSAA4":
        from tests.test_gpu_frontend import _msaa
        ms = _msaa(left, 4, 21, kl.RGBA16F)
        return ms, None, 4, fe.resolve_msaa(ms, 4, kl.RGBA16F)
    return left, None, 1, left


@pytest.mark.parametrize("peak", [4.0, 1000.0])
@pytest.mark.parametrize("kind", ["RGBA16F", "RGBA32F", "RGB32F", "MSAA4"])
@pytest.mark.parametrize("path", list(SCALES))
def test_ctx_sources_and_outputs(cuda, path, kind, peak):
    """every float source the flag covers into every output format, radius 0.5 / 2.0 with the debug tint on and off"""
    import torch
    import openvr_fsr_b200 as ovr
    scale = SCALES[path]
    feed, fmt, samples, reads = _source(kind, peak)
    t = torch.from_numpy(feed).to(cuda)
    for i, out_dtype in enumerate((np.uint8, np.float16, np.float32)):
        for radius, debug in ((0.5, i % 2 == 0), (2.0, i % 2 == 1)):
            pp = ovr.PostProcessor(_cfg(scale, radius, out_dtype, debug=debug))
            got = pp.apply(0, t, fmt=fmt, samples=samples).cpu().numpy()
            pp.close()
            _same(got, _chain(reads, 0, True, scale, radius, out_dtype, debug=debug),
                  f"{kind} -> {np.dtype(out_dtype).name} r={radius} debug={debug}")


@pytest.mark.parametrize("path", list(SCALES))
def test_ctx_shared_texture(cuda, path):
    """one texture holding both eyes side by side: processed once, both centres tested"""
    import torch
    import openvr_fsr_b200 as ovr
    scale = SCALES[path]
    left, _ = _eyes(1000.0)
    both = np.ascontiguousarray(np.concatenate([left, left[:, ::-1]], axis=1))
    tb = torch.from_numpy(both).to(cuda)
    proj = (0.45, 0.5, 0.55, 0.5)
    pp = ovr.PostProcessor(_cfg(scale, 2.0, np.float16, projCentre=proj, debug=True))
    got = pp.apply(0, tb, bounds=ovr.TextureBounds(0, 0, 0.5, 1)).cpu().numpy()
    pp.apply(1, tb, bounds=ovr.TextureBounds(0.5, 0, 1, 1))  # the same texture again: not processed twice
    _same(got, _chain(both, 0, False, scale, 2.0, np.float16, proj=proj, debug=True), "shared texture")
    pp.close()


@pytest.mark.parametrize("path", list(SCALES))
def test_ctx_focus_radius_and_sharpness_overrides(cuda, path):
    """the latched focus, radius override and sharpness override, with the tone map, on every apply: apply_pair, then
    a changed set through apply"""
    import torch
    import openvr_fsr_b200 as ovr
    scale = SCALES[path]
    left, right = _eyes(1000.0)
    t = [torch.from_numpy(e).to(cuda) for e in (left, right)]
    pp = ovr.PostProcessor(_cfg(scale, 0.5, np.uint8))
    steps = [(((0.3, 0.4), (0.7, 0.6)), (1.0, 0.3), 0.2), (((0.6, 0.5), (0.4, 0.45)), (0.0, 2.0), 0.9)]
    for step, (foci, radii, sharp) in enumerate(steps):
        for e in (0, 1):
            pp.set_focus(e, *foci[e])
            pp.set_focus_radius(e, radii[e])
        pp.set_sharpness(sharp)
        outs = pp.apply_pair(t[0], t[1]) if step == 0 else [pp.apply(e, t[e]) for e in (0, 1)]
        for e in (0, 1):
            want = _chain((left, right)[e], e, True, scale, radii[e], np.uint8, proj=foci[e] + foci[e], sharp=sharp)
            _same(outs[e].cpu().numpy(), want, f"step {step} eye {e}")
    pp.close()


def test_ctx_graph_replay(cuda):
    """apply_pair captured into a CUDA graph and replayed on new content: the replay's output is the checker's"""
    import torch
    import openvr_fsr_b200 as ovr
    left, right = _eyes(1000.0)
    scale = SCALES["scaler"]
    pp = ovr.PostProcessor(_cfg(scale, 0.5, np.float16))
    t = [torch.from_numpy(e).to(cuda) for e in (left, right)]
    pp.apply_pair(t[0], t[1])  # lazy init outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = pp.apply_pair(t[0], t[1], stream=torch.cuda.current_stream(cuda))
    l2, r2 = _eyes(4.0)
    t[0].copy_(torch.from_numpy(l2))
    t[1].copy_(torch.from_numpy(r2))
    g.replay()
    torch.cuda.synchronize()
    for e in (0, 1):
        _same(outs[e].cpu().numpy(), _chain((l2, r2)[e], e, True, scale, 0.5, np.float16), f"replay eye {e}")
    pp.close()


@pytest.mark.parametrize("out_dtype", [np.uint8, np.float16, np.float32], ids=["RGBA8", "RGBA16F", "RGBA32F"])
def test_ctx_fast(cuda, out_dtype):
    """fast math on the ctx path, both NIS passes and peaks, radius 0.5 / 2.0, the debug tint on and off.  The bound is
    the worst case measured on one H100 (DESIGN.md section 4) with headroom."""
    import torch
    import openvr_fsr_b200 as ovr
    worst = 0.0
    for path, scale in SCALES.items():
        for peak in (4.0, 1000.0):
            left, right = _eyes(peak)
            for radius, debug in ((0.5, False), (2.0, True)):
                pp = ovr.PostProcessor(_cfg(scale, radius, out_dtype, strict=False, debug=debug))
                outs = pp.apply_pair(torch.from_numpy(left).to(cuda), torch.from_numpy(right).to(cuda))
                for e in (0, 1):
                    got = outs[e].cpu().numpy()
                    want = _chain((left, right)[e], e, True, scale, radius, out_dtype, debug=debug)
                    if out_dtype == np.uint8:
                        err = float(np.abs(got.astype(np.int32) - want.astype(np.int32)).max())
                    else:
                        err, same = _tone_err(got, want)
                        assert same, f"{path} peak {peak}: NaN classes differ"
                    worst = max(worst, err)
                pp.close()
    print(f"\nctx fast worst case ({np.dtype(out_dtype).name}): {worst:.3g}")
    assert worst <= (FAST_LSB if out_dtype == np.uint8 else FAST_TONE), worst


@pytest.mark.parametrize("case", ["rgba8", "rgb10a2", "fsr", "fsr_rcas"])
def test_bit_ignored_where_it_does_not_apply(cuda, case):
    """UNORM sources on the NIS path, and float sources on the FSR path (with and without OVRFSR_FLAG_SRTM): the same
    bytes with the bit on and off"""
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    w, h = 421, 467
    fmt = None
    if case == "rgb10a2":
        src, fmt = synth.natural_rgb10a2(w, h, 3), ovr.FORMAT_RGB10A2
    elif case == "rgba8":
        src = synth.natural_rgba8(w, h, 3)
    else:
        src = synth.natural_rgba16f(w, h, 3, peak=1000.0)
    t = torch.from_numpy(src).to(cuda)
    scale = 1.0 if case == "fsr_rcas" else 0.75
    for srtm in ((False, True) if case.startswith("fsr") else (False,)):
        res = []
        for bit in (False, True):
            pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, useNis=not case.startswith("fsr"), renderScale=scale, radius=0.5,
                                              srtm=srtm, srtmNis=bit, mathMode=ovr.MATH_STRICT))
            res.append(pp.apply(0, t, fmt=fmt).cpu().numpy().copy())
            pp.close()
        _same(res[1], res[0], f"{case} srtm={srtm}")


def test_both_bits_follow_the_path(cuda):
    """a config with OVRFSR_FLAG_SRTM and OVRFSR_FLAG_SRTM_NIS tone-maps whichever path runs: set_config toggles use_nis"""
    import torch
    import openvr_fsr_b200 as ovr
    left, _ = _eyes(1000.0)
    t = torch.from_numpy(left).to(cuda)
    cfg = _cfg(0.75, 0.5, np.uint8, srtm=True)
    pp = ovr.PostProcessor(cfg)
    _same(pp.apply(0, t).cpu().numpy(), _chain(left, 0, True, 0.75, 0.5, np.uint8), "NIS with both bits")
    pp.set_config(dataclasses.replace(cfg, useNis=False))
    _same(pp.apply(0, t).cpu().numpy(), gs._chain(left, 0, True, 0.75, 0.5, np.uint8), "FSR with both bits")
    pp.set_config(dataclasses.replace(cfg, srtmNis=False))
    _same(pp.apply(0, t).cpu().numpy(), _chain(left, 0, True, 0.75, 0.5, np.uint8, srtm=False), "NIS with OVRFSR_FLAG_SRTM only")
    pp.close()


def test_cpp_dropin_config_srtm_nis(cuda, built_lib, tmp_path):
    """vr::PostProcessor with Config::useNis and Config::srtmNis on an RGBA16F pair (tests/cpp/pp_nis_srtm_selftest.cpp)
    gives the checker's bytes"""
    exe = tmp_path / "pp_nis_srtm_selftest"
    pkg = ROOT / "openvr_fsr_b200"
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-I", str(pkg / "csrc"), "-I", str(ROOT / "include"),
                           str(ROOT / "tests/cpp/pp_nis_srtm_selftest.cpp"), "-o", str(exe), "-L", str(pkg), "-lovrfsr",
                           "-Xlinker", f"-rpath={pkg}"])
    left, right = _eyes(1000.0)
    h, w = left.shape[:2]
    scale = SCALES["scaler"]
    ins = [tmp_path / f"in{e}.rgba16f" for e in (0, 1)]
    outs = [tmp_path / f"out{e}.rgba" for e in (0, 1)]
    for p, img in zip(ins, (left, right)):
        p.write_bytes(img.tobytes())
    out = subprocess.run([str(exe), *map(str, ins), str(w), str(h), str(scale), str(SHARP), "0.5", *map(str, outs)],
                         capture_output=True, text=True)
    assert out.returncode == 0 and "pp_nis_srtm_selftest: ok" in out.stdout, out.stdout + out.stderr
    from oracle import pyoracle as po
    ow, oh = po.output_size(w, h, scale)
    for e in (0, 1):
        got = np.frombuffer(outs[e].read_bytes(), dtype=np.uint8).reshape(oh, ow, 4)
        _same(got, _chain((left, right)[e], e, True, scale, 0.5, np.uint8), f"drop-in eye {e}")
