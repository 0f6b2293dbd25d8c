"""OVRFSR_FLAG_SRTM on the H100: AMD's reversible tone map around EASU and RCAS, against the checker's maps.

Stateless: every float-source easu_kernel / rcas_kernel instantiation the ledger lists, except the paired ones (the
tone map turns the pairing off), through ovrfsr_dispatch_fsr_easu_ex / _rcas_ex with each pass-flag combination, on
the signed / HDR / +-65504 content of tests/test_gpu_float_signed.py.  Strict math is compared to the bit.  Fast math:
on in-domain content (finite, >= 0) within 1e-3 per pass in tone-mapped space -- an output that went through G is
mapped back through F in float64 on both sides, because G amplifies any difference near 1 -- and <= 1 LSB on UNORM
targets; on the out-of-domain content the rules of test_gpu_float_signed.check where no G ran (through G, out-of-domain
values meet its 1/32768 floor and a last-bit difference comes out x32768: strict math pins those, fast math only the
NaN classes).

The context path: C2- and C3a-shaped RGBA16F eyes (synth.natural_rgba16f at its default peak 4 and at a peak of 1000),
radius 0.5 / 2.0, every apply entry, CUDA-array source and destination, a shared texture, a focus, the debug tint,
RCAS alone, a CUDA-graph replay, strict output equal to the oracle chain F -> EASU -> intermediate (RGBA16F for a UNORM
output, RGBA32F for a float one) -> RCAS -> G; fast output within the bound measured here; UNORM sources and use_nis
unchanged by the flag; the C++ drop-in's Config::srtm."""
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import kernel_ledger as kl
from tests import srtm_oracle as so
from tests import test_gpu_float_signed as fs
from tests import test_gpu_variant_matrix as vm

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
FLAG_SETS = [(1, 0), (0, 1), (1, 1)]
NT = os.cpu_count() or 1
MAXIMA = {}


def _f64(a):
    """F in float64 on the rgb of an image (alpha as is): the space the filters run in"""
    c = a.astype(np.float64)
    with np.errstate(all="ignore"):
        c[..., :3] /= np.fmax(np.fmax(c[..., 0], c[..., 1]), c[..., 2])[..., None] + 1.0
    return c


def in_domain(fmt, w, h, seed):
    """finite, non-negative HDR content: natural over 0 .. 7.5 with 3 % of the texels at 65504 and a zero block"""
    rng = np.random.default_rng(seed)
    a = fs._natural(w, h, seed, 0.0, 7.5)
    hit = rng.random((h, w)) < 0.03
    a[hit] = 65504.0
    a[: h // 4, : w // 4] = 0.0
    a[..., 3] = 1.0
    return a.astype(np.float16 if fmt == kl.RGBA16F else np.float32)


def _tone_err(got, want):
    """largest |F(got) - F(want)| over finite pixels, and whether the NaN / infinity classes agree"""
    g, w = _f64(got), _f64(want)
    same_class = np.array_equal(np.isnan(g), np.isnan(w))
    fin = np.isfinite(g) & np.isfinite(w)
    return (float(np.abs(g[fin] - w[fin]).max()) if fin.any() else 0.0), same_class


# ---- stateless dispatches, ledger-driven ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def srtm_keys(built_lib):
    keys = sorted(k for k in kl.ledger(built_lib) if k[1] in ("easu_kernel", "rcas_kernel") and
                  dict(zip(kl.PARAMS[k[1]], k[2]))["FIN"] in fs.FLOAT_FORMATS and not dict(zip(kl.PARAMS[k[1]], k[2]))["PAIRED"])
    assert len(keys) == 2 * (2 * 2 * 6 + 2 * 6), len(keys)  # modes x (EASU: TW x ANYIO x pairs + RCAS: ANYIO x pairs)
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
    if kernel == "easu_kernel":
        ow, oh = ovr.output_size(vm.W, vm.H, 0.9 if p["TW"] == 72 else 0.75)
        uc = po.upscale_constants(0, True, vm.W, vm.H, ow, oh, proj=vm.PROJ, radius=vm.RADIUS)
        call = lambda s, d: ovr.fsr_easu(s, d, uc.words(), mm, srtm_in=sin, srtm_out=sout)  # noqa: E731
        want = so.easu(src, ow, oh, uc, out_dtype=vm._np_dtype(fout), srtm_in=sin, srtm_out=sout, nthreads=NT)
    else:
        ow, oh = vm.W, vm.H
        sc = po.sharpen_constants(0, True, vm.W, vm.H, proj=vm.PROJ, radius=vm.RADIUS, sharpness=vm.SHARP,
                                  debug=vm._debug(args))
        call = lambda s, d: ovr.fsr_rcas(s, d, sc.words(), mm, srtm_in=sin, srtm_out=sout)  # noqa: E731
        want = so.rcas(src, sc, out_dtype=vm._np_dtype(fout), srtm_in=sin, srtm_out=sout, nthreads=NT)
    layouts = [("array", ["pitched", "array"])] if anyio else [("tight", ["pitched"])]
    out = []
    for where, kinds in layouts:
        s = vm._place(src, fin, where, dev)
        for kind, d in zip(kinds, vm._outputs(fout, ow, oh, dev, kinds)):
            n0 = ovr.kernel_launches()
            call(s, d)
            assert ovr.kernel_launches() == n0 + 1
            out.append((f"{where}->{kind}", vm._host(d)))
    return src, want, out, fout


@pytest.mark.parametrize("kernel", ["easu_kernel", "rcas_kernel"])
@pytest.mark.parametrize("content", ["signed", "in_domain"])
def test_dispatch_ex_matches_the_oracle(cuda, srtm_keys, kernel, content):
    gen = fs.signed_content if content == "signed" else in_domain
    failures, n = [], 0
    for key in (k for k in srtm_keys if k[1] == kernel):
        for flags in FLAG_SETS:
            src, want, outs, fout = _run_key(key, cuda, gen, flags)
            for label, got in outs:
                n += 1
                name = f"{kl.describe(key)} in={flags[0]} out={flags[1]} [{label}]"
                if key[0] == "strict" or fout not in fs.FLOAT_FORMATS:
                    msg, err = vm._check(got, want, fout, key[0], False)
                elif content == "in_domain":
                    err, same = _tone_err(got, want)
                    msg = None if same and err <= 1e-3 else f"tone-mapped error {err:.3g} (NaN classes agree: {same})"
                elif not flags[1]:
                    # out-of-domain texels: check()'s rules on the tone-mapped output, footprint of the mapped source
                    msg, err = fs.check(got, want, fout, "fast", False, _f64(src) if flags[0] else src)
                else:
                    # Out-of-domain texels through G: no fast-math bound exists.  A negative, >= 1 or overflowing value
                    # reaches G's 1/32768 floor, so a last-bit difference of the filter comes out x32768 (measured on
                    # H100: -1.89e6 vs -2.13e6 next to 3e6 texels), and FP16 outputs cross 65520 into infinity on one
                    # side only.  Strict math above pins these bit for bit; fast math is held to the NaN classes.
                    g, w = got.astype(np.float64), want.astype(np.float64)
                    msg = None if np.array_equal(np.isnan(g), np.isnan(w)) else "fast: NaN where the oracle has none"
                    err = 0.0
                if key[0] == "fast":
                    k = f"{kernel} {content} -> {kl.FORMAT_NAMES[fout]}"
                    MAXIMA[k] = max(MAXIMA.get(k, 0.0), err)
                if msg:
                    failures.append(f"{name}: {msg}")
    print(f"\n{kernel} / {content}: {n} outputs compared; fast maxima: " +
          ", ".join(f"{k}: {v:.3g}" for k, v in sorted(MAXIMA.items()) if k.startswith(f"{kernel} {content}")))
    assert not failures, f"{len(failures)} failures:\n" + "\n".join(failures[:20])


def test_zero_flags_launch_the_plain_dispatch(cuda):
    """pass_flags == 0 through the _ex entry points gives the bytes of the plain entry points"""
    import ctypes as C
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    from oracle import pyoracle as po
    src = fs.signed_content(kl.RGBA16F, vm.W, vm.H, 3)
    ow, oh = ovr.output_size(vm.W, vm.H, 0.75)
    uc = po.upscale_constants(0, True, vm.W, vm.H, ow, oh, proj=vm.PROJ, radius=vm.RADIUS)
    s = torch.from_numpy(src).to(cuda)
    a, b = (torch.empty((oh, ow, 4), dtype=torch.float16, device=cuda) for _ in range(2))
    ovr.fsr_easu(s, a, uc.words(), ovr.MATH_FAST)
    si, di = ovr.image_of(s), ovr.image_of(b)
    words = (C.c_uint32 * 24)(*[int(x) for x in uc.words()])
    assert L.lib().ovrfsr_dispatch_fsr_easu_ex(C.byref(si), C.byref(di), words, ovr.MATH_FAST, 0,
                                               torch.cuda.current_stream().cuda_stream) == L.OK
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---- the context path ----------------------------------------------------------------------------------------------
SHAPES = {"C2": (1683, 1869, 0.75), "C3a": (2244, 2492, 1.3)}
SMALL = 4  # the matrix below runs at 1/4 of each side (same render scale); one full-size pair per shape checks the rest
SHARP = 0.8


def _eyes(shape, peak, full=False):
    from openvr_fsr_b200 import synth
    w, h, scale = SHAPES[shape]
    if not full:
        w, h = w // SMALL, h // SMALL
    left = synth.natural_rgba16f(w, h, 5, peak=peak)
    return (left, np.ascontiguousarray(np.roll(left, 16, axis=1))), scale


def _chain(src, eye, only_one, scale, radius, out_dtype, proj=(.5, .5, .5, .5), debug=False, sharp=SHARP, srtm=True):
    """the oracle's F -> EASU -> intermediate -> RCAS -> G (RCAS alone at scale 1: F and G in the one pass)"""
    from oracle import pyoracle as po
    h, w = src.shape[:2]
    ow, oh = po.output_size(w, h, scale)
    sc = po.sharpen_constants(eye, only_one, ow, oh, proj=proj, radius=radius, sharpness=sharp, debug=debug)
    if scale == 1.0:
        return so.rcas(src, sc, out_dtype=out_dtype, srtm_in=srtm, srtm_out=srtm, nthreads=NT)
    uc = po.upscale_constants(eye, only_one, w, h, ow, oh, proj=proj, radius=radius)
    mid = (np.float32 if out_dtype != np.uint8 else np.float16) if srtm else out_dtype
    m = so.easu(src, ow, oh, uc, out_dtype=mid, srtm_in=srtm, nthreads=NT)
    return so.rcas(m, sc, out_dtype=out_dtype, srtm_out=srtm, nthreads=NT)


def _out_fmt(dtype):
    import openvr_fsr_b200 as ovr
    return {np.uint8: ovr.FORMAT_AUTO, np.float16: ovr.FORMAT_RGBA16F, np.float32: ovr.FORMAT_RGBA32F}[dtype]


def _cfg(scale, radius, out_dtype, strict=True, debug=False, srtm=True, **kw):
    import openvr_fsr_b200 as ovr
    return ovr.Config(fsrEnabled=True, renderScale=scale, sharpness=SHARP, radius=radius, debugMode=debug,
                      outputFormat=_out_fmt(out_dtype), mathMode=ovr.MATH_STRICT if strict else ovr.MATH_FAST, srtm=srtm, **kw)


def _same(got, want, what):
    g, w = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert g.shape == w.shape and g.dtype == w.dtype, (what, g.shape, w.shape, g.dtype, w.dtype)
    diff = g.view(np.uint8) != w.view(np.uint8)
    assert not diff.any(), f"{what}: {int(diff.sum())} bytes differ"


@pytest.mark.parametrize("peak", [4.0, 1000.0])
@pytest.mark.parametrize("shape", ["C2", "C3a"])
def test_ctx_strict_entries(cuda, shape, peak):
    """every apply entry, strict, against the oracle chain"""
    import torch
    import openvr_fsr_b200 as ovr
    (left, right), scale = _eyes(shape, peak)
    t = [torch.from_numpy(e).to(cuda) for e in (left, right)]
    h, w = left.shape[:2]
    ow, oh = ovr.output_size(w, h, scale)
    # apply_pair, radius 0.5, RGBA8 output (RGBA16F intermediate)
    pp = ovr.PostProcessor(_cfg(scale, 0.5, np.uint8))
    outs = pp.apply_pair(t[0], t[1])
    for e in (0, 1):
        _same(outs[e].cpu().numpy(), _chain((left, right)[e], e, True, scale, 0.5, np.uint8), f"apply_pair eye {e}")
    # set_config to a float output: a reset, the intermediate reallocated as RGBA32F; apply, radius 2.0, debug tint
    pp.set_config(_cfg(scale, 2.0, np.float16, debug=True))
    for e in (0, 1):
        _same(pp.apply(e, t[e]).cpu().numpy(), _chain((left, right)[e], e, True, scale, 2.0, np.float16, debug=True), f"apply eye {e}")
    # apply_into, CUDA-array source and destination, RGBA32F output
    pp.set_config(_cfg(scale, 0.5, np.float32))
    src_a = ovr.ArrayImage(w, h, ovr.FORMAT_RGBA16F).upload(t[1])
    dst_a = ovr.ArrayImage(ow, oh, ovr.FORMAT_RGBA32F)
    pp.apply_into(1, src_a, dst_a)
    _same(dst_a.download().cpu().numpy(), _chain(right, 1, True, scale, 0.5, np.float32), "apply_into array->array")
    # apply_pair_into with a focus per eye
    pp.set_config(_cfg(scale, 0.5, np.uint8))
    foci = ((0.3, 0.4), (0.7, 0.6))
    for e in (0, 1):
        pp.set_focus(e, *foci[e])
    dl, dr = (ovr.alloc_image(ow, oh, torch.uint8, cuda) for _ in range(2))
    pp.apply_pair_into(t[0], t[1], dl, dr)
    for e, d in ((0, dl), (1, dr)):
        _same(d.cpu().numpy(), _chain((left, right)[e], e, True, scale, 0.5, np.uint8, proj=foci[e] + foci[e]), f"focus eye {e}")
    pp.clear_focus(0)
    pp.clear_focus(1)
    # apply_host, pinned memory
    hs = torch.from_numpy(left).pin_memory()
    hd = torch.empty((oh, ow, 4), dtype=torch.uint8).pin_memory()
    pp.apply_host(0, hs, hd)
    torch.cuda.synchronize()
    _same(hd.numpy(), _chain(left, 0, True, scale, 0.5, np.uint8), "apply_host")
    for a in (src_a, dst_a):
        a.release()
        a.close()
    pp.close()


@pytest.mark.parametrize("peak", [4.0, 1000.0])
def test_ctx_shared_texture_and_sharpen_only(cuda, peak):
    """one texture holding both eyes (processed once), and renderScale 1 (RCAS alone: F and G in one pass, the
    outside-radius copy in tone-mapped space with the debug tint)"""
    import torch
    import openvr_fsr_b200 as ovr
    (left, _), scale = _eyes("C2", peak)
    both = np.ascontiguousarray(np.concatenate([left, left[:, ::-1]], axis=1))
    tb = torch.from_numpy(both).to(cuda)
    proj = (0.45, 0.5, 0.55, 0.5)
    pp = ovr.PostProcessor(_cfg(scale, 2.0, np.uint8, projCentre=proj))
    got = pp.apply(0, tb, bounds=ovr.TextureBounds(0, 0, 1, 1)).cpu().numpy()
    _same(got, _chain(both, 0, True, scale, 2.0, np.uint8, proj=proj), "one-eye texture")
    pp.set_config(_cfg(scale, 2.0, np.float16, projCentre=proj))
    got = pp.apply(0, tb, bounds=ovr.TextureBounds(0, 0, 0.5, 1)).cpu().numpy()
    pp.apply(1, tb, bounds=ovr.TextureBounds(0.5, 0, 1, 1))  # the same texture again: not processed twice
    _same(got, _chain(both, 0, False, scale, 2.0, np.float16, proj=proj), "shared texture")
    for radius, debug in ((0.5, True), (2.0, False)):
        pp.set_config(_cfg(1.0, radius, np.float16, debug=debug))
        got = pp.apply(0, torch.from_numpy(left).to(cuda)).cpu().numpy()
        _same(got, _chain(left, 0, True, 1.0, radius, np.float16, debug=debug), f"RCAS alone r={radius}")
    pp.close()


@pytest.mark.parametrize("shape", ["C2", "C3a"])
def test_ctx_full_size_pair(cuda, shape):
    """one full-size pair per shape, peak 1000, strict, RGBA8 output"""
    import torch
    import openvr_fsr_b200 as ovr
    (left, right), scale = _eyes(shape, 1000.0, full=True)
    pp = ovr.PostProcessor(_cfg(scale, 0.5, np.uint8))
    outs = pp.apply_pair(torch.from_numpy(left).to(cuda), torch.from_numpy(right).to(cuda))
    for e in (0, 1):
        _same(outs[e].cpu().numpy(), _chain((left, right)[e], e, True, scale, 0.5, np.uint8), f"{shape} eye {e}")
    pp.close()


@pytest.mark.parametrize("out_dtype", [np.uint8, np.float16, np.float32], ids=["RGBA8", "RGBA16F", "RGBA32F"])
def test_ctx_fast(cuda, out_dtype):
    """fast math on the ctx path, both shapes and peaks, radius 0.5 / 2.0, the debug tint on and off.  Measured on one
    H100 before the bounds were set (DESIGN.md section 4): the bounds are the measured worst case with headroom."""
    import torch
    import openvr_fsr_b200 as ovr
    worst = 0.0
    for shape in SHAPES:
        for peak in (4.0, 1000.0):
            (left, right), scale = _eyes(shape, peak)
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
                        assert same, f"{shape} peak {peak}: NaN classes differ"
                    worst = max(worst, err)
                pp.close()
    MAXIMA[f"ctx fast -> {np.dtype(out_dtype).name}"] = worst
    print(f"\nctx fast worst case ({np.dtype(out_dtype).name}): {worst:.3g}")
    assert worst <= (4 if out_dtype == np.uint8 else 2e-3), worst


def test_ctx_graph_replay(cuda):
    """apply_pair captured into a CUDA graph and replayed on new content: the replay's output is the oracle's"""
    import torch
    import openvr_fsr_b200 as ovr
    (left, right), scale = _eyes("C2", 1000.0)
    pp = ovr.PostProcessor(_cfg(scale, 0.5, np.float16))
    t = [torch.from_numpy(e).to(cuda) for e in (left, right)]
    pp.apply_pair(t[0], t[1])  # lazy init outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = pp.apply_pair(t[0], t[1], stream=torch.cuda.current_stream(cuda))
    (l2, r2), _ = _eyes("C2", 4.0)
    t[0].copy_(torch.from_numpy(l2))
    t[1].copy_(torch.from_numpy(r2))
    g.replay()
    torch.cuda.synchronize()
    for e in (0, 1):
        _same(outs[e].cpu().numpy(), _chain((l2, r2)[e], e, True, scale, 0.5, np.float16), f"replay eye {e}")
    pp.close()


@pytest.mark.parametrize("case", ["unorm", "nis", "rgb10a2"])
def test_flag_ignored_where_it_does_not_apply(cuda, case):
    """UNORM sources and use_nis: the same bytes with the flag on and off"""
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    w, h = 421, 467
    if case == "rgb10a2":
        src, fmt = synth.natural_rgb10a2(w, h, 3), ovr.FORMAT_RGB10A2
    elif case == "unorm":
        src, fmt = synth.natural_rgba8(w, h, 3), None
    else:
        src, fmt = synth.natural_rgba16f(w, h, 3, peak=1000.0), None
    t = torch.from_numpy(src).to(cuda)
    res = []
    for srtm in (False, True):
        pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, useNis=case == "nis", renderScale=0.75, radius=0.5, srtm=srtm,
                                          mathMode=ovr.MATH_STRICT))
        res.append(pp.apply(0, t, fmt=fmt).cpu().numpy().copy())
        pp.close()
    _same(res[1], res[0], case)


def test_cpp_dropin_config_srtm(cuda, built_lib, tmp_path):
    """vr::PostProcessor with Config::srtm on an RGBA16F pair (tests/cpp/pp_srtm_selftest.cpp) gives the oracle's bytes"""
    exe = tmp_path / "pp_srtm_selftest"
    pkg = ROOT / "openvr_fsr_b200"
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-I", str(pkg / "csrc"), "-I", str(ROOT / "include"),
                           str(ROOT / "tests/cpp/pp_srtm_selftest.cpp"), "-o", str(exe), "-L", str(pkg), "-lovrfsr",
                           "-Xlinker", f"-rpath={pkg}"])
    (left, right), scale = _eyes("C2", 1000.0)
    h, w = left.shape[:2]
    ins = [tmp_path / f"in{e}.rgba16f" for e in (0, 1)]
    outs = [tmp_path / f"out{e}.rgba" for e in (0, 1)]
    for p, img in zip(ins, (left, right)):
        p.write_bytes(img.tobytes())
    out = subprocess.run([str(exe), *map(str, ins), str(w), str(h), str(scale), str(SHARP), "0.5", *map(str, outs)],
                         capture_output=True, text=True)
    assert out.returncode == 0 and "pp_srtm_selftest: ok" in out.stdout, out.stdout + out.stderr
    from oracle import pyoracle as po
    ow, oh = po.output_size(w, h, scale)
    for e in (0, 1):
        got = np.frombuffer(outs[e].read_bytes(), dtype=np.uint8).reshape(oh, ow, 4)
        _same(got, _chain((left, right)[e], e, True, scale, 0.5, np.uint8), f"drop-in eye {e}")
