"""OVRFSR_FLAG_FINITE on the GPU: every float-source kernel with the OVRFSR_PASS_FINITE_* bits, and the context path with
the flag, against the oracle.

The bits are runtime arguments of the same instantiations, so a pass with finite-in and finite-out runs the filter it
runs without them on finite_in(source), and maps what it stores (tests/finite_rule.py):

  launch(IN | OUT, src) == finite_out(launch(no bits, finite_in(src)))

Section by section:
  1/2  every RGBA16F / RGBA32F source key of the ledger in the five families that take the bits, on the content of
       tests/test_gpu_float_nonfinite.py: strict math equals finite_out(oracle pass on finite_in(src)) at every word,
       with no NaN and no infinity on either side; fast math keeps test_gpu_float_signed.check's bounds at every
       output pixel (no taint exception).  The stateless keys run through the _ex dispatches, the paired ones through
       a context with the flag (UNORM intermediate: finite-in on the eye only), the fused ones through a context with
       the flag and OVRFSR_FLAG_FUSED_FSR.  Each key must be launched with the bits.
  3    the context cases of test_gpu_float_nonfinite.py with the flag: every output word finite, and per pass equal
       to the checker where the checker exists.
  4    finite content: the bits change no output bit, for every key.
  5    the flag changes no plan (kernel launches per apply), and nothing for UNORM sources.
  6    the maps themselves, through RCAS's outside-radius copy (an identity on float texels without them): every FP16
       word, the listed FP32 words, and the FP16 store of binary32 values around 65504 / 65520.
  7    the C++ drop-in's Config::finite."""
import dataclasses
import functools
import os
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import finite_rule as fr
from tests import kernel_ledger as kl
from tests import test_gpu_float_nonfinite as nf
from tests import test_gpu_float_signed as fs
from tests import test_gpu_variant_matrix as vm

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
FAMILIES = ("easu_kernel", "rcas_kernel", "nis_scaler_kernel", "nis_sharpen_kernel", "fsr_fused_kernel")
# The fused kernel's 72-column tile only holds a float source tile up to out->in 0.757 tall while needing more than
# about 0.8 wide (fsr_fused.cuh); the context scales both axes alike, and the stateless fused dispatch takes no pass
# bits, so no entry point launches these keys with finite-in.
FUSED_72_REASON = "no entry point launches the float-source 72-column fused kernel with finite-in"
STATE = {"launched": set(), "ran": set()}


# ---- the bits on, in the API and in the checker -----------------------------------------------------------------
def finite_on(monkeypatch):
    """every FSR / NIS dispatch with OVRFSR_PASS_FINITE_IN | _OUT, every context with OVRFSR_FLAG_FINITE, and every
    oracle pass as finite_out(pass(finite_in(src)))"""
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    for name in ("fsr_easu", "fsr_rcas", "nis_scaler", "nis_sharpen"):
        monkeypatch.setattr(ovr, name, functools.partial(getattr(ovr, name), finite_in=True, finite_out=True))
    monkeypatch.setattr(ovr, "Config", functools.partial(ovr.Config, finite=True))
    for name in ("easu", "rcas", "nis_scaler", "nis_sharpen"):
        def mapped(src, *a, _f=getattr(po, name), **k):
            return fr.finite_out(_f(fr.finite_in(src), *a, **k))
        monkeypatch.setattr(po, name, mapped)


def _fused_ctx(key, content):
    """a float-source fused key through a context with OVRFSR_FLAG_FUSED_FSR (and, under finite_on, the flag)"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    mode, _, args = key
    fin = args[0]

    def run(dev):
        src = content(fin, vm.W, vm.H, vm._seed(key))
        ow, oh = ovr.output_size(vm.W, vm.H, 0.75)
        pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=0.75, sharpness=vm.SHARP, radius=vm.RADIUS,
                                          projCentre=vm.PROJ, mathMode=vm._mathmode(mode), fusedFsr=True))
        got = pp.apply(0, torch.from_numpy(src).to(dev)).cpu().numpy()
        torch.cuda.synchronize()
        pp.close()
        uc = po.upscale_constants(0, True, vm.W, vm.H, ow, oh, proj=vm.PROJ, radius=vm.RADIUS)
        sc = po.sharpen_constants(0, True, ow, oh, proj=vm.PROJ, radius=vm.RADIUS, sharpness=vm.SHARP)
        return [("context", got, po.rcas(po.easu(src, ow, oh, uc), sc), kl.RGBA8, True)]
    return vm.Case("fsr_fused_kernel", mode, {key}, run, kl.describe(key) + " (context)")


def _case(key, content):
    if key[1] == "fsr_fused_kernel":
        return _fused_ctx(key, content)
    return vm.case_for(key, content)


@pytest.fixture(scope="module")
def finite_keys(built_lib):
    keys = {k for k in fs._float_keys(set(kl.ledger(built_lib))) if k[1] in FAMILIES}
    assert keys, "the ledger lists no float-source kernels"
    return keys


def _reachable(keys):
    return {k for k in keys if not (k[1] == "fsr_fused_kernel" and k[2][3] == 72)}


def _cases(keys, family):
    cases, claimed = [], set()
    for key in sorted(k for k in _reachable(keys) if k[1] == family):
        if key in claimed:
            continue
        c = _case(key, nf.nonfinite_content)
        assert key in c.keys, kl.describe(key)
        claimed |= c.keys
        cases.append(c)
    return cases


def _all_finite(a, fmt):
    return fmt not in fs.FLOAT_FORMATS or bool(np.isfinite(a.astype(np.float32)).all())


# ---- 1 / 2: every float-source key on non-finite content ---------------------------------------------------------
def _run_family(family, keys, dev, monkeypatch):
    import torch
    import openvr_fsr_b200 as ovr
    if family in STATE["ran"]:
        return
    STATE["ran"].add(family)
    srcs = []

    def content(fmt, w, h, seed):
        srcs.append(nf.nonfinite_content(fmt, w, h, seed))
        return srcs[-1]
    cases = _cases(keys, family)
    failures = []
    finite_on(monkeypatch)
    for c0 in cases:
        key = sorted(c0.keys & keys)[0]
        c = _case(key, content)
        srcs.clear()
        n0 = ovr.kernel_launches()
        res = c.run(dev)
        torch.cuda.synchronize()
        n = ovr.kernel_launches() - n0
        if n < len(c.keys):
            failures.append(f"{c.name}: {n} launches for {len(c.keys)} claimed kernels")
        else:
            STATE["launched"] |= c.keys
        for i, (label, got, want, fmt, composed) in enumerate(res):
            src = srcs[i] if len(srcs) == len(res) else srcs[-1]
            if not (_all_finite(got, fmt) and _all_finite(want, fmt)):
                failures.append(f"{c.name} [{label}]: a non-finite word with the bits on "
                                f"(device {not _all_finite(got, fmt)}, checker {not _all_finite(want, fmt)})")
                continue
            if c.mode == "strict":
                msg = nf.strict_check(got, want, fmt)
            elif fmt in fs.FLOAT_FORMATS:
                msg = fs.check(got, want, fmt, c.mode, composed, fr.finite_in(src))[0]
            else:
                msg = vm._check(got, want, fmt, c.mode, composed)[0]
            if msg:
                failures.append(f"{c.name} [{label}]: {msg}")
    monkeypatch.undo()
    print(f"{family}: {len(cases)} cases")
    assert not failures, f"{len(failures)} failures:\n" + "\n".join(failures)


@pytest.mark.parametrize("family", FAMILIES)
def test_finite_bits_match_the_oracle(cuda, finite_keys, family, monkeypatch):
    _run_family(family, finite_keys, cuda, monkeypatch)


def test_every_float_source_key_launched_with_the_bits(cuda, finite_keys, monkeypatch):
    for family in FAMILIES:
        try:
            _run_family(family, finite_keys, cuda, monkeypatch)
        except AssertionError:
            pass  # reported by that family's test; coverage is judged on what ran
    reach = _reachable(finite_keys)
    covered = STATE["launched"] & finite_keys
    left = finite_keys - reach
    print(f"\nfloat-source keys launched with the finite bits: {len(covered)}/{len(finite_keys)}; "
          f"{len(left)} unreachable ({FUSED_72_REASON})")
    assert left and all(k[1] == "fsr_fused_kernel" for k in left)
    assert covered == reach, "never launched:\n" + "\n".join(sorted(map(kl.describe, reach - covered)))


# ---- 4: finite content: the bits change nothing --------------------------------------------------------------------
@pytest.mark.parametrize("family", FAMILIES)
def test_bits_change_nothing_on_finite_content(cuda, finite_keys, family, monkeypatch):
    import torch

    def content(fmt, w, h, seed):
        if fmt not in fs.FLOAT_FORMATS:
            return vm._content(fmt, w, h, seed)
        if seed % 2:
            return fs.signed_content(fmt, w, h, seed)
        blocks = nf.nonfinite_content(fmt, w, h, seed)
        return np.where(np.isfinite(blocks.astype(np.float32)), blocks, 0).astype(blocks.dtype)
    failures = []
    for c0 in _cases(finite_keys, family):
        key = sorted(c0.keys & finite_keys)[0]
        off = _case(key, content).run(cuda)
        torch.cuda.synchronize()
        finite_on(monkeypatch)
        on = _case(key, content).run(cuda)
        torch.cuda.synchronize()
        monkeypatch.undo()
        for (label, g_off, _, fmt, _), (_, g_on, _, _, _) in zip(off, on):
            if not _all_finite(g_off, fmt):
                continue  # an output beyond the destination's range: the bits clamp it (section 3 checks those)
            if not np.array_equal(np.ascontiguousarray(g_off).view(np.uint8), np.ascontiguousarray(g_on).view(np.uint8)):
                failures.append(f"{kl.describe(key)} [{label}]: the bits changed a finite output")
    assert not failures, "\n".join(failures)


# ---- 3: the context path with the flag ----------------------------------------------------------------------------
def _finite_words(got, what):
    if got.dtype != np.uint8:
        assert np.isfinite(got.astype(np.float32)).all(), f"{what}: non-finite output"


@pytest.mark.parametrize("scale", [0.75, 1.0])
@pytest.mark.parametrize("kind", ["RGBA32F", "RGB32F"])
def test_ctx_beyond_fp16_into_rgba16f(cuda, kind, scale, monkeypatch):
    """finite FP32 eyes beyond 65504 into RGBA16F: EASU's RGBA16F intermediate and the output clamp to +-65504
    instead of rounding to +-inf"""
    import torch
    import openvr_fsr_b200 as ovr
    src = nf._beyond_fp16(vm.W, vm.H, 31)
    feed, fmt = (np.ascontiguousarray(src[..., :3]), vm.RGB32F) if kind == "RGB32F" else (src, None)
    plain = nf._fsr_chain(feed, scale, 0.4, np.float16, src_fmt=fmt)[0]
    assert np.isinf(plain).any()
    finite_on(monkeypatch)
    for radius in (0.4, 2.0):
        pp = ovr.PostProcessor(nf._cfg(scale, radius, np.float16))
        got = pp.apply(0, torch.from_numpy(feed).to(cuda), fmt=fmt).cpu().numpy()
        pp.close()
        _finite_words(got, kind)
        nf._strict_same(got, nf._fsr_chain(feed, scale, radius, np.float16, src_fmt=fmt)[0], f"{kind} scale {scale} radius {radius}")


@pytest.mark.parametrize("fused", [False, True])
def test_ctx_beyond_fp16_into_rgba8(cuda, fused, monkeypatch):
    import torch
    import openvr_fsr_b200 as ovr
    src = nf._fp16_eye(vm.W, vm.H, 32)
    finite_on(monkeypatch)
    pp = ovr.PostProcessor(nf._cfg(0.75, 0.4, np.uint8, fusedFsr=fused))
    n0 = ovr.kernel_launches()
    got = pp.apply(0, torch.from_numpy(src).to(cuda)).cpu().numpy()
    n = ovr.kernel_launches() - n0
    pp.close()
    assert n == (1 if fused else 2), n
    nf._strict_same(got, nf._fsr_chain(src, 0.75, 0.4, np.uint8)[0], f"fused={fused}")


@pytest.mark.parametrize("out_dtype", [np.float16, np.float32, np.uint8])
@pytest.mark.parametrize("scale", [0.75, 1.0])
def test_ctx_nis(cuda, out_dtype, scale, monkeypatch):
    import torch
    import openvr_fsr_b200 as ovr
    finite_on(monkeypatch)
    for src in (nf._beyond_fp16(vm.W, vm.H, 33), nf._fp16_eye(vm.W, vm.H, 34)):
        pp = ovr.PostProcessor(nf._cfg(scale, 0.4, out_dtype, useNis=True))
        got = pp.apply(0, torch.from_numpy(src).to(cuda)).cpu().numpy()
        pp.close()
        _finite_words(got, "NIS")
        nf._strict_same(got, nf._nis_chain(src, scale, 0.4, out_dtype), f"NIS {src.dtype} -> {np.dtype(out_dtype).name}")


def test_ctx_msaa_resolve_of_opposite_infinities(cuda, monkeypatch):
    """the resolve's NaN (+inf + -inf) is mapped by the passes that read the resolved copy"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import frontend as fe
    eye = fs._natural(vm.W, vm.H, 4, -0.5, 7.5).astype(np.float16)
    ms = np.repeat(eye, 4, axis=1)
    rng = np.random.default_rng(4)
    ys, xs = nf._per_block(rng, vm.W, vm.H, 1)
    ms[ys, 4 * xs + 1, :3] = np.inf
    ms[ys, 4 * xs + 2, :3] = -np.inf
    reads = fe.resolve_msaa(ms, 4, kl.RGBA16F)
    assert np.isnan(reads[ys, xs, :3]).all()
    finite_on(monkeypatch)
    for out_dtype in (np.float16, np.uint8):
        pp = ovr.PostProcessor(nf._cfg(0.75, 0.4, out_dtype))
        got = pp.apply(0, torch.from_numpy(ms).to(cuda), samples=4).cpu().numpy()
        pp.close()
        _finite_words(got, "MSAA")
        nf._strict_same(got, nf._fsr_chain(reads, 0.75, 0.4, out_dtype)[0], f"MSAA -> {np.dtype(out_dtype).name}")


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_ctx_entries_overrides_and_tone_map(cuda, mode, monkeypatch):
    """with the flag, every output word is finite: apply_pair / apply_pair_into, apply_into with CUDA arrays, a shared
    texture with unequal per-eye radii, focus / focus-radius / sharpness overrides, and SRTM / SRTM_NIS with the flag
    (F(65504) is finite) -- on RGBA16F eyes holding +-inf and NaN, into RGBA16F and RGBA32F"""
    import torch
    import openvr_fsr_b200 as ovr
    finite_on(monkeypatch)
    mm = vm._mathmode(mode)
    left, right = (torch.from_numpy(nf._fp16_eye(vm.W, vm.H, s)).to(cuda) for s in (40, 41))
    ow, oh = ovr.output_size(vm.W, vm.H, 0.75)
    for out_dtype in (np.float16, np.float32):
        for extra in ({}, {"srtm": True}, {"useNis": True, "srtmNis": True}, {"useNis": True}):
            cfg = dataclasses.replace(nf._cfg(0.75, 0.4, out_dtype, **extra), mathMode=mm)
            assert cfg.finite
            pp2 = ovr.PostProcessor(cfg)
            outs = [t.cpu().numpy() for t in pp2.apply_pair(left, right)]
            dl, dr = (torch.empty((oh, ow, 4), dtype=vm._dtype(kl.RGBA16F if out_dtype == np.float16 else kl.RGBA32F), device=cuda)
                      for _ in range(2))
            pp2.apply_pair_into(left, right, dl, dr)
            outs += [dl.cpu().numpy(), dr.cpu().numpy()]
            pp2.set_focus(0, 0.3, 0.6)
            pp2.set_focus_radius(1, 0.9)
            pp2.set_sharpness(0.2)
            outs += [pp2.apply(0, left).cpu().numpy(), pp2.apply(1, right).cpu().numpy()]
            torch.cuda.synchronize()
            pp2.close()
            for i, o in enumerate(outs):
                _finite_words(o, f"{mode} {extra} -> {np.dtype(out_dtype).name} output {i}")


def test_ctx_shared_texture_and_arrays(cuda, monkeypatch):
    import torch
    import openvr_fsr_b200 as ovr
    finite_on(monkeypatch)
    # one RGBA16F texture holding both eyes, a different radius per eye
    tex = torch.from_numpy(nf._fp16_eye(2 * vm.W, vm.H, 6)).to(cuda)
    pp = ovr.PostProcessor(nf._cfg(0.75, 0.5, np.float16))
    pp.set_focus_radius(0, 0.3)
    pp.set_focus_radius(1, 0.8)
    got = pp.apply(ovr.EYE_LEFT, tex, ovr.TextureBounds(0.0, 0.0, 0.5, 1.0)).cpu().numpy()
    pp.close()
    _finite_words(got, "shared texture")
    # a CUDA-array source and a CUDA-array destination
    eye = nf._fp16_eye(vm.W, vm.H, 7)
    ow, oh = ovr.output_size(vm.W, vm.H, 0.75)
    src_a = ovr.ArrayImage(vm.W, vm.H, ovr.FORMAT_RGBA16F).upload(torch.from_numpy(eye).to(cuda))
    dst_a = ovr.ArrayImage(ow, oh, ovr.FORMAT_RGBA16F)
    pp = ovr.PostProcessor(nf._cfg(0.75, 0.4, np.float16))
    pp.apply_into(0, src_a, dst_a)
    got = dst_a.download().cpu().numpy()
    pp.close()
    for a in (src_a, dst_a):
        a.release()
        a.close()
    _finite_words(got, "array source")
    nf._strict_same(got, nf._fsr_chain(eye, 0.75, 0.4, np.float16)[0], "array source")


# ---- 5: plans and formats ------------------------------------------------------------------------------------------
PLANS = {
    "paired": dict(scale=0.75, out=np.uint8),
    "fused": dict(scale=0.75, out=np.uint8, fusedFsr=True),
    "float output": dict(scale=0.75, out=np.float16),
    "rcas only": dict(scale=1.0, out=np.float32),
    "nvscaler": dict(scale=0.75, out=np.float16, useNis=True),
    "nvsharpen": dict(scale=1.0, out=np.uint8, useNis=True),
    "resolve": dict(scale=0.75, out=np.float16, samples=4),
    "expand": dict(scale=0.75, out=np.uint8, rgb32f=True),
}


@pytest.mark.parametrize("plan", list(PLANS))
def test_flag_changes_no_plan(cuda, plan):
    import torch
    import openvr_fsr_b200 as ovr
    p = dict(PLANS[plan])
    scale, out, samples, rgb = p.pop("scale"), p.pop("out"), p.pop("samples", 1), p.pop("rgb32f", False)
    eye = nf._fp16_eye(vm.W, vm.H, 50)
    feed = np.repeat(eye, samples, axis=1) if samples > 1 else eye
    fmt = None
    if rgb:
        feed, fmt = np.ascontiguousarray(eye[..., :3].astype(np.float32)), vm.RGB32F
    counts = []
    for finite in (False, True):
        pp = ovr.PostProcessor(nf._cfg(scale, 0.4, out, finite=finite, **p))
        t = torch.from_numpy(feed).to(cuda)
        pp.apply(0, t, fmt=fmt, samples=samples)  # allocations happen here
        n0 = ovr.kernel_launches()
        pp.apply(0, t, fmt=fmt, samples=samples)
        torch.cuda.synchronize()
        counts.append(ovr.kernel_launches() - n0)
        pp.close()
    assert counts[0] == counts[1] and counts[0] > 0, counts


@pytest.mark.parametrize("path", ["fsr", "fused", "nis"])
def test_unorm_sources_ignore_the_flag(cuda, path):
    import torch
    import openvr_fsr_b200 as ovr
    extra = {"fsr": {}, "fused": {"fusedFsr": True}, "nis": {"useNis": True}}[path]
    for fmt in (kl.RGBA8, kl.RGB10A2, vm.BGRX8):
        src = vm._content(fmt, vm.W, vm.H, 60 + fmt)
        outs = []
        for finite in (False, True):
            pp = ovr.PostProcessor(nf._cfg(0.75, 0.4, np.uint8, finite=finite, **extra))
            outs.append(pp.apply(0, torch.from_numpy(src).to(cuda), fmt=vm._tag(fmt)).cpu().numpy())
            pp.close()
        assert np.array_equal(outs[0], outs[1]), (path, fmt)


# ---- 6: the maps, through RCAS's outside-radius copy ---------------------------------------------------------------
def _rcas_copy(src, out_dtype, dev, mode, **bits):
    """RCAS with every group outside the radius and the tint off: the copy 1 x texel, through the pass's maps"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    from tests import test_oracle_nonfinite_host as nh
    h, w = src.shape[:2]
    sc = nh._everywhere(po.sharpen_constants(0, True, w, h, sharpness=0.5), False)
    out = torch.empty((h, w, 4), dtype=torch.float16 if out_dtype == np.float16 else torch.float32, device=dev)
    ovr.fsr_rcas(torch.from_numpy(src).to(dev), out, sc.words(), vm._mathmode(mode), **bits)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_helpers_exhaustive(cuda, mode):
    # finite-in over every FP16 word (16384 texels x 4 channels), stored exactly as binary32
    h16 = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16).reshape(128, 128, 4)
    got = _rcas_copy(h16, np.float32, cuda, mode, finite_in=True)
    want = fr.finite_in(h16).astype(np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # finite-in over FP32 words: +-0, subnormals, +-FLT_MAX, +-inf, quiet / signalling NaNs with payloads
    words = np.array([0, 0x80000000, 1, 0x807fffff, 0x00800000, 0x7f7fffff, 0xff7fffff, 0x477fe000, 0x477fe001, 0xc77fe001,
                      0x7f800000, 0xff800000, 0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fa5a5a5, 0xffffffff],
                     dtype=np.uint32)
    f32 = np.resize(words, 64 * 64 * 4).view(np.float32).reshape(64, 64, 4)
    got = _rcas_copy(f32, np.float32, cuda, mode, finite_in=True)
    assert np.array_equal(got.view(np.uint32), fr.finite_in(f32).view(np.uint32))
    # finite-out before an FP16 store, across the binary32 range around 65504 / 65520 (and +-inf, NaN, +-FLT_MAX)
    lo, hi = np.float32(65000).view(np.uint32), np.float32(66000).view(np.uint32)
    x = np.arange(lo, hi, dtype=np.uint32).view(np.float32)
    x = np.concatenate([x, -x, np.array([np.inf, -np.inf, np.nan, 3.4e38, -3.4e38, 0.0, -0.0], dtype=np.float32)])
    n = -(-x.size // (4 * 256)) * 4 * 256
    grid = np.resize(x, n).reshape(-1, 256, 4)
    got = _rcas_copy(grid, np.float16, cuda, mode, finite_out=True)
    assert np.array_equal(got.view(np.uint16), fr.fp16_store(grid).view(np.uint16))
    # without the bits the same copy keeps the infinities: the maps, not the copy, remove them
    assert np.isinf(_rcas_copy(grid, np.float16, cuda, mode)).any()


# ---- 7: the C++ drop-in --------------------------------------------------------------------------------------------
def test_cpp_dropin_config_finite(cuda, built_lib, tmp_path, monkeypatch):
    """vr::PostProcessor with Config::finite on an RGBA16F pair holding +-inf and NaN (tests/cpp/pp_finite_selftest.cpp)
    gives the checker's bytes on finite_in(eyes), which differ from the bytes without the flag"""
    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("nvcc not installed")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = tmp_path / "pp_finite_selftest"
    pkg = ROOT / "openvr_fsr_b200"
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", str(pkg / "csrc"), "-I", str(ROOT / "include"),
                           str(ROOT / "tests/cpp/pp_finite_selftest.cpp"), "-o", str(exe), "-L", str(pkg), "-lovrfsr",
                           "-Xlinker", f"-rpath={pkg}"])
    eyes = [nf._fp16_eye(vm.W, vm.H, s) for s in (70, 71)]
    ins = [tmp_path / f"in{e}.rgba16f" for e in (0, 1)]
    outs = [tmp_path / f"out{e}.rgba" for e in (0, 1)]
    for p, img in zip(ins, eyes):
        p.write_bytes(img.tobytes())
    scale, sharp, radius = 0.75, 0.8, 0.5
    out = subprocess.run([str(exe), *map(str, ins), str(vm.W), str(vm.H), str(scale), str(sharp), str(radius), *map(str, outs)],
                         capture_output=True, text=True, env={**os.environ})
    assert out.returncode == 0 and "pp_finite_selftest: ok" in out.stdout, out.stdout + out.stderr
    from oracle import pyoracle as po
    ow, oh = po.output_size(vm.W, vm.H, scale)

    def chain(src, e):
        uc = po.upscale_constants(e, True, vm.W, vm.H, ow, oh, radius=radius)
        sc = po.sharpen_constants(e, True, ow, oh, radius=radius, sharpness=sharp)
        return po.rcas(po.easu(src, ow, oh, uc), sc)
    for e in (0, 1):
        got = np.frombuffer(outs[e].read_bytes(), dtype=np.uint8).reshape(oh, ow, 4)
        assert not np.array_equal(got, chain(eyes[e], e)), "the flag changed nothing on an eye holding +-inf and NaN"
        assert np.array_equal(got, chain(fr.finite_in(eyes[e]), e)), f"drop-in eye {e}"
