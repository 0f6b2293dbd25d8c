"""OVRFSR_FLAG_PERCEPTUAL on the GPU: every float-source kernel with the OVRFSR_PASS_PERCEPTUAL_* bits, the maps and the
sRGB encode themselves, the context path with the flag, and the C++ drop-in, against tests/perceptual_oracle.py.

  1  every RGBA16F / RGBA32F source key of EASU, RCAS, NVScaler and NVSharpen in the ledger (the paired EASU keys
     excepted: a pass with the perceptual bits never pairs), through the _ex dispatches, with each perceptual bit alone
     and both, also with the SRTM and FINITE bits, on in-range, HDR, signed and (with FINITE) non-finite content, into
     every target the key stores (RGBA8, RGBA16F, RGBA32F).  Strict math equals the checker at every word; fast math
     stays within 4 codes of an RGBA8 target and 2e-3 (relative above 1) of a float target in the pass's filter domain.
  2  the maps and the encode, through RCAS's outside-radius copy (tint off), in both math modes, bit for bit: every
     FP16 word, FP32 words around all 255 thresholds, NaN, +-0 and negatives.
  3  the context path: RGBA16F, RGBA32F, RGB32F and 4x MSAA eyes; FSR at 0.75 / 1.0 / 1.3 and NIS at 0.75 / 1.0; RGBA8
     (sRGB), RGBA16F and RGBA32F outputs; radius 0.5 and 2.0; tint on and off -- strict math equals the checker, and the
     returned format carries OVRFSR_FORMAT_SRGB_BIT exactly for the RGBA8 output.  Every apply entry, CUDA arrays, a
     shared texture, a graph replay, the overrides and SRTM / SRTM_NIS / FINITE with the flag.  The plan launches what
     the SRTM plan launches; UNORM sources ignore the flag.
  4  the C++ drop-in's Config::perceptual and the colour space it hands on."""
import dataclasses
import functools
import os
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import kernel_ledger as kl
from tests import perceptual_oracle as pq
from tests import test_gpu_float_nonfinite as nf
from tests import test_gpu_float_signed as fs
from tests import test_gpu_variant_matrix as vm

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
FAMILIES = ("easu_kernel", "rcas_kernel", "nis_scaler_kernel", "nis_sharpen_kernel")
P_IN, P_OUT = pq.PERCEPTUAL_IN, pq.PERCEPTUAL_OUT
SRTM = pq.SRTM_IN | pq.SRTM_OUT
FINITE = pq.FINITE_IN | pq.FINITE_OUT
_KW = {pq.SRTM_IN: "srtm_in", pq.SRTM_OUT: "srtm_out", pq.FINITE_IN: "finite_in", pq.FINITE_OUT: "finite_out",
       P_IN: "perceptual_in", P_OUT: "perceptual_out"}


# ---- content ---------------------------------------------------------------------------------------------------------
def _in_range(fmt, w, h, seed):
    a = fs._natural(w, h, seed, 0.0, 1.0)
    return a.astype(np.float16 if fmt == kl.RGBA16F else np.float32)


def _hdr(fmt, w, h, seed):
    a = fs._natural(w, h, seed, 0.0, 1.0) ** 2.2 * 4.0
    hit = np.random.default_rng(seed).random((h, w)) < 0.05
    a[hit, :3] *= 24.0  # highlights up to ~100
    return a.astype(np.float16 if fmt == kl.RGBA16F else np.float32)


CONTENT = {"in-range": _in_range, "hdr": _hdr, "signed": fs.signed_content, "non-finite": nf.nonfinite_content}
# (pass bits, content): each perceptual bit alone and both, and both with the SRTM and FINITE bits
COMBOS = [(P_IN | P_OUT, "in-range"), (P_IN, "hdr"), (P_OUT, "signed"), (P_IN | P_OUT, "hdr"), (P_IN | P_OUT | SRTM, "hdr"),
          (P_IN | P_OUT | FINITE, "non-finite"), (P_IN | P_OUT | SRTM | FINITE, "signed")]


def _bits_on(monkeypatch, bits):
    """every FSR / NIS dispatch with `bits`, and every oracle pass as the checker's pass with them"""
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    kw = {name: True for b, name in _KW.items() if bits & b}
    for name in ("fsr_easu", "fsr_rcas", "nis_scaler", "nis_sharpen"):
        monkeypatch.setattr(ovr, name, functools.partial(getattr(ovr, name), **kw))
    for name in ("easu", "rcas", "nis_scaler", "nis_sharpen"):
        monkeypatch.setattr(po, name, functools.partial(getattr(pq, name), bits=bits))


# ---- 1: every float-source key ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def keys(built_lib):
    ks = set()
    for k in fs._float_keys(set(kl.ledger(built_lib))):
        p = dict(zip(kl.PARAMS[k[1]], k[2]))
        if k[1] in FAMILIES and not p.get("PAIRED"):
            ks.add(k)
    assert ks, "the ledger lists no float-source kernels"
    return ks


def _fast_domain(a, bits, fmt):
    """a float target's words in the pass's filter domain (the store maps undone), alpha as is"""
    x = a.astype(np.float32).copy()
    if bits & pq.SRTM_OUT:
        x[..., :3] = pq.so.srtm(x[..., :3])
    if bits & P_OUT:
        x[..., :3] = pq.p_fwd(x[..., :3])
    return x


def _fast_check(got, want, fmt, bits):
    if fmt == kl.RGBA8:
        d = np.abs(got.astype(int) - want.astype(int))
        return None if d.max() <= 4 else f"fast: {int(d.max())} codes off (bound 4)"
    g, w = _fast_domain(got, bits, fmt), _fast_domain(want, bits, fmt)
    same = (g == w) | (np.isnan(g) & np.isnan(w))
    with np.errstate(invalid="ignore", over="ignore"):
        ok = same | (np.abs(g - w) <= 2e-3 * np.maximum(1.0, np.abs(w)))
    if ok.all():
        return None
    i = tuple(np.argwhere(~ok)[0])
    return f"fast: {int((~ok).sum())} words beyond 2e-3, first at {i}: {g[i]!r} vs {w[i]!r}"


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("combo", range(len(COMBOS)))
def test_every_float_source_key_matches_the_checker(cuda, keys, family, combo, monkeypatch):
    import torch
    import openvr_fsr_b200 as ovr
    bits, content = COMBOS[combo]
    _bits_on(monkeypatch, bits)
    failures, ran = [], 0
    for key in sorted(k for k in keys if k[1] == family):
        c = vm.case_for(key, CONTENT[content])
        n0 = ovr.kernel_launches()
        res = c.run(cuda)
        torch.cuda.synchronize()
        assert ovr.kernel_launches() > n0, kl.describe(key)
        ran += 1
        for label, got, want, fmt, _ in res:
            msg = nf.strict_check(got, want, fmt) if c.mode == "strict" else _fast_check(got, want, fmt, bits)
            if msg:
                failures.append(f"{c.name} [{label}]: {msg}")
    print(f"{family} bits={bits} on {content}: {ran} keys")
    assert ran and not failures, f"{len(failures)} failures:\n" + "\n".join(failures)


# ---- 2: the maps and the encode ----------------------------------------------------------------------------------------
def _copy_consts(w, h):
    from oracle import pyoracle as po
    from tests import test_oracle_nonfinite_host as nh
    return nh._everywhere(po.sharpen_constants(0, True, w, h, sharpness=0.5), False)


def _rcas_copy(src, out_dtype, dev, mode, bits):
    """RCAS with every group outside the radius and the tint off: the copy 1 x texel through the pass's maps"""
    import torch
    import openvr_fsr_b200 as ovr
    h, w = src.shape[:2]
    out = torch.empty((h, w, 4), dtype={np.uint8: torch.uint8, np.float16: torch.float16, np.float32: torch.float32}[out_dtype],
                      device=dev)
    ovr.fsr_rcas(torch.from_numpy(src).to(dev), out, _copy_consts(w, h).words(), vm._mathmode(mode),
                 **{name: True for b, name in _KW.items() if bits & b})
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _grid(x):
    n = -(-x.size // (4 * 64)) * 4 * 64
    return np.resize(x, n).reshape(-1, 64, 4)


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_maps_and_encode_bit_for_bit(cuda, mode):
    # every FP16 word through P then P^-1, stored as RGBA32F (the round trip itself) and as RGBA8 (its sRGB code)
    h16 = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16).reshape(128, 128, 4)
    sc = _copy_consts(128, 128)
    for out_dtype in (np.float32, np.uint8, np.float16):
        got = _rcas_copy(h16, out_dtype, cuda, mode, P_IN | P_OUT)
        want = pq.rcas(h16, sc, out_dtype, P_IN | P_OUT)
        msg = nf.strict_check(got, want, {np.float32: kl.RGBA32F, np.float16: kl.RGBA16F, np.uint8: kl.RGBA8}[out_dtype])
        assert msg is None, f"FP16 words -> {np.dtype(out_dtype).name}: {msg}"
    rt = _rcas_copy(h16, np.float32, cuda, mode, P_IN | P_OUT)
    assert np.array_equal(np.isnan(rt), np.isnan(h16.astype(np.float32)))
    # FP32 words at and one ulp around all 255 thresholds, and values whose square lands there (perceptual-out alone)
    t = pq.table_words()[1:].astype(np.int64)
    around = (t[:, None] + np.arange(-1, 2)[None, :]).astype(np.uint32).view(np.float32).ravel()
    roots = np.sqrt(around).astype(np.float32).view(np.uint32).astype(np.int64)
    roots = (roots[:, None] + np.arange(-2, 3)[None, :]).astype(np.uint32).view(np.float32).ravel()
    special = np.array([np.nan, -np.nan, 0.0, -0.0, -1e-30, -0.25, -1.0, -np.inf, np.inf, 1e-45, 1.0, 2.0, 65504.0],
                       dtype=np.float32)
    for vals, bits in ((np.concatenate([around, special]), P_IN | P_OUT), (np.concatenate([roots, special]), P_OUT)):
        g = _grid(vals)
        wsc = _copy_consts(g.shape[1], g.shape[0])
        for out_dtype, fmt in ((np.uint8, kl.RGBA8), (np.float32, kl.RGBA32F)):
            got = _rcas_copy(g, out_dtype, cuda, mode, bits)
            msg = nf.strict_check(got, pq.rcas(g, wsc, out_dtype, bits), fmt)
            assert msg is None, f"bits {bits} -> {np.dtype(out_dtype).name}: {msg}"
        codes = _rcas_copy(g, np.uint8, cuda, mode, bits)[..., :3]
        lin = pq.p_inv(pq.p_fwd(g[..., :3])) if bits & P_IN else pq.p_inv(g[..., :3])
        assert np.array_equal(codes, pq.srgb_code(lin))
    # the squares of `roots` reach every code
    assert len(np.unique(_rcas_copy(_grid(roots), np.uint8, cuda, mode, P_OUT)[..., :3])) == 256


# ---- 3: the context path -------------------------------------------------------------------------------------------------
def _cfg(path, scale, radius, out_dtype, tint=False, **kw):
    import openvr_fsr_b200 as ovr
    fmt = {np.uint8: ovr.FORMAT_AUTO, np.float16: ovr.FORMAT_RGBA16F, np.float32: ovr.FORMAT_RGBA32F}[out_dtype]
    return ovr.Config(fsrEnabled=True, useNis=path == "nis", renderScale=scale, sharpness=vm.SHARP, radius=radius,
                      outputFormat=fmt, mathMode=ovr.MATH_STRICT, debugMode=tint, **{"perceptual": True, **kw})


def _flags(cfg):
    return cfg.to_c().flags


def _want(path, src, scale, radius, out_dtype, flags, tint=False, src_fmt=None, eye=0, one=True, w=None, h=None):
    from oracle import pyoracle as po
    h0, w0 = src.shape[:2]
    w, h = w or w0, h or h0
    ow, oh = po.output_size(w, h, scale)
    if path == "nis":
        cfg, ok = po.nis_config(scale == 1.0, eye, one, w, h, ow, oh, radius=radius, sharpness=vm.SHARP, debug=tint)
        assert ok
        return pq.nis_chain(src, cfg, ow, oh, out_dtype, flags, scale != 1.0, src_fmt)
    uc = po.upscale_constants(eye, one, w, h, ow, oh, radius=radius)
    sc = po.sharpen_constants(eye, one, ow, oh, radius=radius, sharpness=vm.SHARP, debug=tint)
    return pq.fsr_chain(src, uc, sc, ow, oh, out_dtype, flags, scale != 1.0, src_fmt)


def _eye(kind, seed):
    """(what the ctx is fed, its fmt, samples, what the passes read)"""
    from oracle import frontend as fe
    a = _hdr(kl.RGBA32F, vm.W, vm.H, seed)
    a[::7, ::5, :3] *= -0.3  # a few negative (scRGB) texels
    if kind == "RGBA16F":
        e = a.astype(np.float16)
        return e, None, 1, e
    if kind == "RGBA32F":
        return a, None, 1, a
    if kind == "RGB32F":
        rgb = np.ascontiguousarray(a[..., :3])
        return rgb, vm.RGB32F, 1, rgb
    ms = np.repeat(a.astype(np.float16), 4, axis=1)
    ms[:, 1::4, :3] *= np.float16(0.5)
    return ms, None, 4, fe.resolve_msaa(ms, 4, kl.RGBA16F)


@pytest.mark.parametrize("path,scale", [("fsr", 0.75), ("fsr", 1.0), ("fsr", 1.3), ("nis", 0.75), ("nis", 1.0)])
@pytest.mark.parametrize("kind", ["RGBA16F", "RGBA32F", "RGB32F", "MSAA4"])
def test_ctx_matches_the_checker(cuda, kind, path, scale):
    import torch
    import openvr_fsr_b200 as ovr
    feed, fmt, samples, reads = _eye(kind, 11)
    src_fmt = vm.RGB32F if kind == "RGB32F" else None
    t = torch.from_numpy(feed).to(cuda)
    for out_dtype in (np.uint8, np.float16, np.float32):
        for radius in (0.5, 2.0):
            for tint in (False, True):
                cfg = _cfg(path, scale, radius, out_dtype, tint)
                pp = ovr.PostProcessor(cfg)
                got = pp.apply(0, t, fmt=fmt, samples=samples).cpu().numpy()
                tag = pp.last_output_format & ovr.FORMAT_SRGB_BIT
                pp.close()
                what = f"{kind} {path} {scale} -> {np.dtype(out_dtype).name} radius {radius} tint {tint}"
                assert bool(tag) == (out_dtype == np.uint8), what
                nf._strict_same(got, _want(path, reads, scale, radius, out_dtype, _flags(cfg), tint, src_fmt), what)


@pytest.mark.parametrize("extra", [{}, {"srtm": True}, {"useNis": True, "srtmNis": True}, {"finite": True},
                                   {"srtm": True, "finite": True}, {"useNis": True, "srtmNis": True, "finite": True}])
def test_ctx_entries_and_flag_combinations(cuda, extra):
    """apply_pair, apply_pair_into (tagged and untagged destinations), apply_into with CUDA arrays, apply_host, and
    focus / focus-radius / sharpness overrides, with the other float flags"""
    import torch
    import openvr_fsr_b200 as ovr
    path = "nis" if extra.get("useNis") else "fsr"
    extra = {k: v for k, v in extra.items() if k != "useNis"}
    eyes = [nf._fp16_eye(vm.W, vm.H, s) if extra.get("finite") else _hdr(kl.RGBA16F, vm.W, vm.H, s) for s in (40, 41)]
    left, right = (torch.from_numpy(e).to(cuda) for e in eyes)
    ow, oh = ovr.output_size(vm.W, vm.H, 0.75)
    for out_dtype in (np.uint8, np.float16):
        cfg = _cfg(path, 0.75, 0.5, out_dtype, **extra)
        flags = _flags(cfg)
        want = [_want(path, e, 0.75, 0.5, out_dtype, flags, eye=i) for i, e in enumerate(eyes)]
        pp = ovr.PostProcessor(cfg)
        a, b = pp.apply_pair(left, right)
        nf._strict_same(a.cpu().numpy(), want[0], f"{extra} apply_pair left")
        nf._strict_same(b.cpu().numpy(), want[1], f"{extra} apply_pair right")
        assert bool(pp.last_output_format & ovr.FORMAT_SRGB_BIT) == (out_dtype == np.uint8)
        tdt = {np.uint8: torch.uint8, np.float16: torch.float16}[out_dtype]
        dfmt = ovr.FORMAT_RGBA8 if out_dtype == np.uint8 else ovr.FORMAT_RGBA16F
        for tag in ((0, ovr.FORMAT_SRGB_BIT) if out_dtype == np.uint8 else (0,)):
            dl, dr = (torch.zeros((oh, ow, 4), dtype=tdt, device=cuda) for _ in range(2))
            pp.apply_pair_into(left, right, dl, dr, dst_fmt=dfmt | tag)
            nf._strict_same(dl.cpu().numpy(), want[0], f"{extra} apply_pair_into tag {tag}")
            nf._strict_same(dr.cpu().numpy(), want[1], f"{extra} apply_pair_into tag {tag}")
        # a host round trip
        hs = torch.from_numpy(eyes[0]).pin_memory()
        hd = torch.zeros((oh, ow, 4), dtype=tdt).pin_memory()
        pp.apply_host(0, hs, hd)
        torch.cuda.synchronize()
        nf._strict_same(hd.numpy(), want[0], f"{extra} apply_host")
        # the overrides
        pp.set_focus(0, 0.3, 0.6)
        pp.set_focus_radius(0, 0.9)
        pp.set_sharpness(0.2)
        got = pp.apply(0, left).cpu().numpy()
        pp.close()
        cfg2 = dataclasses.replace(cfg, sharpness=0.2, radius=0.9, projCentre=(0.3, 0.6, 0.5, 0.5))
        ref = ovr.PostProcessor(cfg2)
        nf._strict_same(got, ref.apply(0, left).cpu().numpy(), f"{extra} overrides")
        ref.close()


def test_ctx_arrays_shared_texture_and_graph(cuda):
    import torch
    import openvr_fsr_b200 as ovr
    eye = _hdr(kl.RGBA16F, vm.W, vm.H, 7)
    ow, oh = ovr.output_size(vm.W, vm.H, 0.75)
    cfg = _cfg("fsr", 0.75, 0.5, np.uint8)
    want = _want("fsr", eye, 0.75, 0.5, np.uint8, _flags(cfg))
    # a CUDA-array source and a CUDA-array destination, tagged as sRGB and not
    src_a = ovr.ArrayImage(vm.W, vm.H, ovr.FORMAT_RGBA16F).upload(torch.from_numpy(eye).to(cuda))
    for tag in (0, ovr.FORMAT_SRGB_BIT):
        dst_a = ovr.ArrayImage(ow, oh, ovr.FORMAT_RGBA8)
        dst_a.image.format |= tag
        pp = ovr.PostProcessor(cfg)
        pp.apply_into(0, src_a, dst_a)
        dst_a.image.format &= ~ovr.FORMAT_SRGB_BIT
        got = dst_a.download().cpu().numpy()
        pp.close()
        dst_a.release()
        dst_a.close()
        nf._strict_same(got, want, f"arrays, destination tag {tag}")
    src_a.release()
    src_a.close()
    # one texture holding both eyes
    tex = np.concatenate([eye, _hdr(kl.RGBA16F, vm.W, vm.H, 8)], axis=1)
    pp = ovr.PostProcessor(cfg)
    got = pp.apply(ovr.EYE_LEFT, torch.from_numpy(tex).to(cuda), ovr.TextureBounds(0.0, 0.0, 0.5, 1.0)).cpu().numpy()
    assert pp.last_output_format & ovr.FORMAT_SRGB_BIT
    pp.close()
    nf._strict_same(got, _want("fsr", tex, 0.75, 0.5, np.uint8, _flags(cfg), one=False), "shared texture")
    # a captured graph replays the perceptual plan on new content
    l = torch.from_numpy(eye).to(cuda)
    pp = ovr.PostProcessor(cfg)
    dst = torch.zeros((oh, ow, 4), dtype=torch.uint8, device=cuda)
    pp.apply_into(0, l, dst)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pp.apply_into(0, l, dst, stream=torch.cuda.current_stream(cuda))
    eye2 = _hdr(kl.RGBA16F, vm.W, vm.H, 9)
    l.copy_(torch.from_numpy(eye2).to(cuda))
    dst.zero_()
    g.replay()
    torch.cuda.synchronize()
    nf._strict_same(dst.cpu().numpy(), _want("fsr", eye2, 0.75, 0.5, np.uint8, _flags(cfg)), "graph replay")
    del g
    pp.close()


PLANS = [("fsr", 0.75, np.uint8), ("fsr", 0.75, np.float16), ("fsr", 1.0, np.uint8), ("nis", 0.75, np.uint8),
         ("nis", 1.0, np.float32)]


@pytest.mark.parametrize("plan", range(len(PLANS)))
def test_plan_launches_what_the_srtm_plan_launches(cuda, plan):
    import torch
    import openvr_fsr_b200 as ovr
    path, scale, out_dtype = PLANS[plan]
    t = torch.from_numpy(_hdr(kl.RGBA16F, vm.W, vm.H, 50)).to(cuda)
    counts = []
    for kw in ({"perceptual": False, **({"srtmNis": True} if path == "nis" else {"srtm": True})}, {}):
        pp = ovr.PostProcessor(_cfg(path, scale, 0.5, out_dtype, **kw))
        pp.apply(0, t)
        n0 = ovr.kernel_launches()
        pp.apply(0, t)
        torch.cuda.synchronize()
        counts.append(ovr.kernel_launches() - n0)
        pp.close()
    assert counts[0] == counts[1] > 0, counts


@pytest.mark.parametrize("path", ["fsr", "fused", "nis"])
def test_unorm_sources_ignore_the_flag(cuda, path):
    import torch
    import openvr_fsr_b200 as ovr
    extra = {"fsr": {}, "fused": {"fusedFsr": True}, "nis": {}}[path]
    for fmt in (kl.RGBA8, kl.RGB10A2, vm.BGRX8):
        src = vm._content(fmt, vm.W, vm.H, 60 + fmt)
        outs = []
        for perceptual in (False, True):
            pp = ovr.PostProcessor(_cfg("nis" if path == "nis" else "fsr", 0.75, 0.4, np.uint8, perceptual=perceptual, **extra))
            outs.append(pp.apply(0, torch.from_numpy(src).to(cuda), fmt=vm._tag(fmt)).cpu().numpy())
            assert not pp.last_output_format & ovr.FORMAT_SRGB_BIT
            pp.close()
        assert np.array_equal(outs[0], outs[1]), (path, fmt)


# ---- 4: the C++ drop-in --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("targets", [False, True])
def test_cpp_dropin(cuda, built_lib, tmp_path, targets):
    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("nvcc not installed")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = tmp_path / "pp_perceptual_selftest"
    pkg = ROOT / "openvr_fsr_b200"
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", str(pkg / "csrc"), "-I", str(ROOT / "include"),
                           str(ROOT / "tests/cpp/pp_perceptual_selftest.cpp"), "-o", str(exe), "-L", str(pkg), "-lovrfsr",
                           "-Xlinker", f"-rpath={pkg}"])
    eyes = [_hdr(kl.RGBA16F, vm.W, vm.H, s) for s in (70, 71)]
    ins = [tmp_path / f"in{e}.rgba16f" for e in (0, 1)]
    for p, img in zip(ins, eyes):
        p.write_bytes(img.tobytes())
    scale, radius = 0.75, 0.5
    from oracle import pyoracle as po
    ow, oh = po.output_size(vm.W, vm.H, scale)
    for perceptual in (0, 1):
        outs = [tmp_path / f"out{perceptual}{e}.rgba" for e in (0, 1)]
        out = subprocess.run([str(exe), *map(str, ins), str(vm.W), str(vm.H), str(scale), str(vm.SHARP), str(radius),
                              str(perceptual), str(int(targets)), *map(str, outs)], capture_output=True, text=True,
                             env={**os.environ})
        assert out.returncode == 0 and "pp_perceptual_selftest: ok" in out.stdout, out.stdout + out.stderr
        for e in (0, 1):
            got = np.frombuffer(outs[e].read_bytes(), dtype=np.uint8).reshape(oh, ow, 4)
            if perceptual:
                nf._strict_same(got, _want("fsr", eyes[e], scale, radius, np.uint8, 16, eye=e), f"drop-in eye {e}")
