"""ovrfsr_set_focus_radius: each eye's mask radius is set every frame, without a reset, and latched on the GPU with the
focus when the frame runs.  An apply with radius override r gives the bits of an apply whose config radius is r --
checked against the oracle in strict math, against a ctx configured with that radius in fast math -- on every ctx
path, with and without a focus; a shared texture tests centre pair 0 against the left eye's radius and pair 1 against
the right eye's; the override costs no reset, follows a captured CUDA graph across replays, and a frame never sees a
radius that was not set."""
import dataclasses
import subprocess
import threading
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]

IW, IH, SCALE, SHARP = 211, 157, 0.75, 0.9
# per-eye radius sequences that differ between the eyes and change every frame (0 and 4 are the ends of the range)
RADII_L = [0.3, 0.5, 0.0, 1.0, 2.0, 4.0]
RADII_R = [1.0, 0.0, 4.0, 0.3, 0.5, 2.0]
FOCI = [(0.5, 0.5), (0.2, 0.3), (0.8, 0.7), (0.0, 1.0), (0.35, 0.6), (0.6, 0.4)]
U32 = 0xFFFFFFFF


def _oracle(img, eye, one, proj, radius, mode, scale=SCALE, sharp=SHARP):
    """strict oracle output of one eye: mode 'fsr' (EASU -> RCAS, also what the fused kernel gives; RCAS alone at scale
    1), 'nis' (NVScaler at scale < 1, NVSharpen at scale 1)"""
    from oracle import pyoracle as po
    ih, iw = img.shape[:2]
    ow, oh = po.output_size(iw, ih, scale)
    if mode == "nis":
        cfg, _ = po.nis_config(scale == 1.0, eye, one, iw, ih, ow, oh, proj=proj, radius=radius, sharpness=sharp)
        return po.nis_sharpen(img, cfg) if scale == 1.0 else po.nis_scaler(img, ow, oh, cfg)
    sc = po.sharpen_constants(eye, one, ow, oh, proj=proj, radius=radius, sharpness=sharp)
    mid = img if scale == 1.0 else po.easu(img, ow, oh, po.upscale_constants(eye, one, iw, ih, ow, oh, proj=proj, radius=radius))
    return po.rcas(mid, sc)


def _eyes(torch, dev, seed=3):
    from openvr_fsr_b200 import synth
    left, right = synth.stereo_pair("natural", IW, IH, seed)
    return (left, right), (torch.from_numpy(left).to(dev), torch.from_numpy(right).to(dev))


PATHS = {  # name: (Config kwargs, oracle mode)
    "fsr": (dict(renderScale=SCALE), "fsr"),
    "fused": (dict(renderScale=SCALE, fusedFsr=True), "fsr"),
    "rcas": (dict(renderScale=1.0), "fsr"),
    "nis_scaler": (dict(renderScale=SCALE, useNis=True), "nis"),
    "nis_sharpen": (dict(renderScale=1.0, useNis=True), "nis"),
}


@pytest.mark.parametrize("focus", [False, True])
@pytest.mark.parametrize("path", list(PATHS))
def test_radius_sequence_matches_oracle_strict(cuda, path, focus):
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    kw, mode = PATHS[path]
    (left, right), (tl, tr) = _eyes(torch, cuda)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, sharpness=SHARP, radius=0.5, mathMode=ovr.MATH_STRICT, **kw))
    for i, (rl, rr) in enumerate(zip(RADII_L, RADII_R)):
        fl, fr = (FOCI[i], FOCI[-1 - i]) if focus else ((.5, .5), (.5, .5))
        if focus:
            pp.set_focus(0, *fl)
            pp.set_focus(1, *fr)
        pp.set_focus_radius(0, rl)
        pp.set_focus_radius(1, rr)
        # a rejected value leaves the one just set
        assert L.lib().ovrfsr_set_focus_radius(pp._ctx, 0, 4.5) == L.ERR_INVALID
        assert L.lib().ovrfsr_set_focus_radius(pp._ctx, 1, float("nan")) == L.ERR_INVALID
        for eye, (img, t, f, r) in enumerate(((left, tl, fl, rl), (right, tr, fr, rr))):
            got = pp.apply(eye, t).cpu().numpy()
            want = _oracle(img, eye, True, f + f, r, mode, scale=kw["renderScale"])
            assert np.array_equal(got, want), (path, eye, f, r)
    pp.close()


@pytest.mark.parametrize("path", list(PATHS))
def test_radius_fast_math_equals_configured_radius(cuda, path):
    """fast math: the same bits as a ctx whose config radius (and projection centre) is the override (and focus)"""
    import torch
    import openvr_fsr_b200 as ovr
    kw, _ = PATHS[path]
    _, (tl, tr) = _eyes(torch, cuda, 5)
    cfg = ovr.Config(fsrEnabled=True, sharpness=SHARP, radius=0.5, mathMode=ovr.MATH_FAST, **kw)
    pp = ovr.PostProcessor(cfg)
    for i, (rl, rr) in enumerate(zip(RADII_L, RADII_R)):
        fl, fr = FOCI[i], FOCI[-1 - i]
        pp.set_focus_radius(0, rl)
        pp.set_focus_radius(1, rr)
        use_focus = i % 2 == 1
        if use_focus:
            pp.set_focus(0, *fl)
            pp.set_focus(1, *fr)
        else:
            pp.clear_focus(0), pp.clear_focus(1)
        for eye, t, r in ((0, tl, rl), (1, tr, rr)):
            ref = ovr.PostProcessor(dataclasses.replace(cfg, radius=r, **({"projCentre": fl + fr} if use_focus else {})))
            assert torch.equal(pp.apply(eye, t), ref.apply(eye, t)), (path, eye, r, use_focus)
            ref.close()
    pp.close()


@pytest.mark.parametrize("path", list(PATHS))
def test_override_equal_to_config_radius_gives_reference_bytes(cuda, path):
    import torch
    import openvr_fsr_b200 as ovr
    kw, _ = PATHS[path]
    _, (tl, tr) = _eyes(torch, cuda, 7)
    cfg = ovr.Config(fsrEnabled=True, sharpness=SHARP, radius=0.3, projCentre=(.45, .5, .55, .5), **kw)
    pp, ref = ovr.PostProcessor(cfg), ovr.PostProcessor(cfg)
    want = [ref.apply(0, tl).clone(), ref.apply(1, tr).clone()]
    pp.set_focus_radius(0, 0.3)
    pp.set_focus_radius(1, 0.3)
    assert torch.equal(pp.apply(0, tl), want[0]) and torch.equal(pp.apply(1, tr), want[1])
    # radius 0: no block centre is a circle centre here, so every block the 0.3 circle holds changes its output
    pp.set_focus_radius(0, 0.0)
    pp.set_focus_radius(1, 0.0)
    assert not torch.equal(pp.apply(0, tl), want[0]) and not torch.equal(pp.apply(1, tr), want[1])
    pp.clear_focus_radius(0)
    assert torch.equal(pp.apply(0, tl), want[0]) and not torch.equal(pp.apply(1, tr), want[1])
    pp.clear_focus_radius(1)
    assert torch.equal(pp.apply(0, tl), want[0]) and torch.equal(pp.apply(1, tr), want[1])
    # a new config radius applies to the eyes without an override only, and set_config keeps the override
    pp.set_focus_radius(1, 0.3)
    pp.set_config(dataclasses.replace(cfg, radius=0.7))
    ref.set_config(dataclasses.replace(cfg, radius=0.7))
    assert torch.equal(pp.apply(0, tl), ref.apply(0, tl)) and torch.equal(pp.apply(1, tr), want[1])
    pp.close(), ref.close()


def _mask(shape, bw, bh, centre, r0sq, r1sq):
    """per-pixel inside flag of the two-radius rule: block (bx, by) is inside when its centre is within r0 of centre
    pair 0 or within r1 of pair 1, in wrapping u32 arithmetic like the kernels and the shaders"""
    h, w = shape
    by, bx = np.meshgrid(np.arange((h + bh - 1) // bh, dtype=np.uint32), np.arange((w + bw - 1) // bw, dtype=np.uint32),
                         indexing="ij")
    cx, cy = bx * np.uint32(bw) + np.uint32(bw // 2), by * np.uint32(bh) + np.uint32(bh // 2)
    c = [np.uint32(v) for v in centre]
    with np.errstate(over="ignore"):
        d1 = (c[0] - cx) * (c[0] - cx) + (c[1] - cy) * (c[1] - cy)
        d2 = (c[2] - cx) * (c[2] - cx) + (c[3] - cy) * (c[3] - cy)
    inside = (d1 <= np.uint32(r0sq)) | (d2 <= np.uint32(r1sq))
    return np.repeat(np.repeat(inside, bh, axis=0), bw, axis=1)[:h, :w]


def _all(consts, inside):
    """the same constants with every block inside (R^2 = 2^32 - 1) or every block outside: centres (0, 0) are never a
    block centre (those are odd multiples of half a block), so with R^2 = 0 no squared distance qualifies"""
    for i in range(4):
        consts.imageCentre[i] = 0
    consts.radius[1] = U32 if inside else 0
    return consts


def _select(mask, a, b):
    return np.where(mask[..., None], a, b)


@pytest.mark.parametrize("focus", [False, True])
@pytest.mark.parametrize("path", ["fsr", "fused", "rcas", "nis_scaler", "nis_sharpen"])
def test_shared_texture_tests_each_centre_against_its_eyes_radius(cuda, path, focus):
    """one texture holding both eyes: the per-block selection, under the two-radius rule, between the oracle's
    all-inside and all-outside results -- per pass for FSR (EASU's 16x16 groups, then RCAS on that image); equal radii
    reduce to the plain oracle"""
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    from oracle import pyoracle as po
    kw, mode = PATHS[path]
    scale = kw["renderScale"]
    tex_np = synth.natural_rgba8(320, 120, 21)
    tex = torch.from_numpy(tex_np).to(cuda)
    iw, ih = 320, 120
    ow, oh = po.output_size(iw, ih, scale)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, sharpness=SHARP, radius=0.5, **kw))
    fl, fr = ((0.3, 0.4), (0.7, 0.6)) if focus else ((.5, .5), (.5, .5))
    if focus:
        pp.set_focus(0, *fl)
        pp.set_focus(1, *fr)
    proj = fl + fr
    for rl, rr in ((0.3, 0.8), (1.0, 0.2), (0.0, 2.0), (0.6, 0.6)):
        pp.set_focus_radius(0, rl)
        pp.set_focus_radius(1, rr)
        left = pp.apply(ovr.EYE_LEFT, tex, ovr.TextureBounds(0.0, 0.0, 0.5, 1.0))
        right = pp.apply(ovr.EYE_RIGHT, tex, ovr.TextureBounds(0.5, 0.0, 1.0, 1.0))
        assert left.data_ptr() == right.data_ptr()
        got = left.cpu().numpy()
        if rl == rr:
            assert np.array_equal(got, _oracle(tex_np, 0, False, proj, rl, mode, scale=scale)), (path, rl)
            continue
        rsq = [po.upscale_constants(0, True, iw, ih, ow, oh, radius=r).radius[1] for r in (rl, rr)]
        if mode == "nis":
            sharpen = scale == 1.0
            centre = list(po.nis_config(sharpen, 0, False, iw, ih, ow, oh, proj=proj, radius=0.5)[0].imageCentre)
            cin, cout = (_all(po.nis_config(sharpen, 0, False, iw, ih, ow, oh, proj=proj, radius=0.5, sharpness=SHARP)[0], k)
                         for k in (True, False))
            run = (lambda c: po.nis_sharpen(tex_np, c)) if sharpen else (lambda c: po.nis_scaler(tex_np, ow, oh, c))
            m = _mask((oh, ow), 32, 32 if sharpen else 24, centre, *rsq)
            want = _select(m, run(cin), run(cout))
        else:
            centre = list(po.sharpen_constants(0, False, ow, oh, proj=proj).imageCentre)
            m = _mask((oh, ow), 16, 16, centre, *rsq)
            mid = tex_np
            if scale != 1.0:
                uin, uout = (_all(po.upscale_constants(0, False, iw, ih, ow, oh, proj=proj), k) for k in (True, False))
                mid = _select(m, po.easu(tex_np, ow, oh, uin), po.easu(tex_np, ow, oh, uout))
            sin, sout = (_all(po.sharpen_constants(0, False, ow, oh, proj=proj, sharpness=SHARP), k) for k in (True, False))
            want = _select(m, po.rcas(mid, sin), po.rcas(mid, sout))
        assert m.any() and not m.all(), (path, rl, rr)  # the case separates the two radii
        assert np.array_equal(got, want), (path, rl, rr)
    pp.close()


def test_radius_needs_no_reset(cuda):
    """output images stay where they are, each apply launches the same kernels (the copy is not a launch), and the
    debugMode timing keeps sampling"""
    import torch
    import openvr_fsr_b200 as ovr
    _, (tl, tr) = _eyes(torch, cuda, 15)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.5, debugMode=True))
    ptrs = [pp.apply(0, tl).data_ptr(), pp.apply(1, tr).data_ptr()]
    n0 = ovr.kernel_launches()
    pp.apply(0, tl), pp.apply(1, tr)
    per_frame = ovr.kernel_launches() - n0
    for i, r in enumerate(RADII_L * 3):
        pp.set_focus_radius(i % 2, r)
        n0 = ovr.kernel_launches()
        assert [pp.apply(0, tl).data_ptr(), pp.apply(1, tr).data_ptr()] == ptrs
        assert ovr.kernel_launches() - n0 == per_frame
        torch.cuda.synchronize()
    ms, n = pp.gpu_time_ms()
    assert n >= 6 and 0.0 < ms < 50.0
    pp.close()


def test_radius_follows_a_captured_graph(cuda):
    import torch
    import openvr_fsr_b200 as ovr
    (left, right), (tl, tr) = _eyes(torch, cuda, 17)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.5))
    pp.set_focus_radius(0, 0.3)
    pp.set_focus_radius(1, 1.0)
    pp.apply_pair(tl, tr)  # lazy init outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        a, b = pp.apply_pair(tl, tr, stream=torch.cuda.current_stream(cuda))
    for i, (rl, rr) in enumerate(zip(RADII_L, RADII_R)):
        pp.set_focus_radius(0, rl)
        pp.set_focus_radius(1, rr)
        fl, fr = FOCI[i], FOCI[-1 - i]
        pp.set_focus(0, *fl)
        pp.set_focus(1, *fr)
        a.zero_(), b.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(a.cpu().numpy(), _oracle(left, 0, True, fl + fl, rl, "fsr")), (rl, fl)
        assert np.array_equal(b.cpu().numpy(), _oracle(right, 1, True, fr + fr, rr, "fsr")), (rr, fr)
    pp.clear_focus(0), pp.clear_focus(1)
    pp.clear_focus_radius(0)  # the captured copy now reads the config radius for the left eye
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(a.cpu().numpy(), _oracle(left, 0, True, (.5, .5, .5, .5), 0.5, "fsr"))
    assert np.array_equal(b.cpu().numpy(), _oracle(right, 1, True, (.5, .5, .5, .5), RADII_R[-1], "fsr"))
    pp.clear_focus_radius(1)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(b.cpu().numpy(), _oracle(right, 1, True, (.5, .5, .5, .5), 0.5, "fsr"))
    del g
    pp.close()


@pytest.mark.parametrize("with_focus", [False, True])
def test_radius_updates_from_another_thread_never_tear(cuda, with_focus):
    """A thread cycles the left eye's radius through three values while 200 frames run: every frame is one of the three
    oracle outputs (both radius words of the block are published by one 64-bit store).  With the focus cycling through
    three points too, a copy may combine the radius of one update with the centre pairs of another, and the two
    centre pairs with each other (each pair whole): every frame is one of those 3 x 3 x 3 oracle outputs."""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    (left, _), (tl, _) = _eyes(torch, cuda, 19)
    ow, oh = po.output_size(IW, IH, SCALE)
    radii = [0.25, 0.45, 0.7]
    points = [(0.25, 0.3), (0.5, 0.5), (0.75, 0.7)] if with_focus else [(0.5, 0.5)]
    want = {}
    for k, r in enumerate(radii):
        for i, pi in enumerate(points):
            for j, pj in enumerate(points):
                uc = po.upscale_constants(0, True, IW, IH, ow, oh, proj=pi + pi, radius=r)
                sc = po.sharpen_constants(0, True, ow, oh, proj=pi + pi, radius=r, sharpness=SHARP)
                other = po.upscale_constants(0, True, IW, IH, ow, oh, proj=pj + pj, radius=r)
                for c in (uc, sc):
                    c.imageCentre[2], c.imageCentre[3] = other.imageCentre[2], other.imageCentre[3]
                want[po.rcas(po.easu(left, ow, oh, uc), sc).tobytes()] = (k, i, j)
    assert len({v[0] for v in want.values()}) == 3  # the three radii give three images
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.5))
    pp.set_focus_radius(0, radii[0])
    pp.set_focus(0, *points[0])
    stop = threading.Event()

    def cycle():
        n = 0
        while not stop.is_set():
            pp.set_focus_radius(0, radii[n % 3])
            if with_focus:
                pp.set_focus(0, *points[(n // 3 + n) % 3])
            n += 1

    th = threading.Thread(target=cycle)
    th.start()
    try:
        for _ in range(200):
            assert pp.apply(0, tl).cpu().numpy().tobytes() in want
    finally:
        stop.set()
        th.join()
    pp.close()


def test_radius_apply_pair_array_destination_and_apply_host(cuda):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    (left, right), (tl, tr) = _eyes(torch, cuda, 9)
    ow, oh = po.output_size(IW, IH, SCALE)
    cfg = ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.5)
    pair, into, host = ovr.PostProcessor(cfg), ovr.PostProcessor(cfg), ovr.PostProcessor(cfg)
    arr = [ovr.ArrayImage(ow, oh), ovr.ArrayImage(ow, oh)]
    src = [torch.from_numpy(left).pin_memory(), torch.from_numpy(right).pin_memory()]
    dst = [torch.empty((oh, ow, 4), dtype=torch.uint8).pin_memory() for _ in range(2)]
    for i, (rl, rr) in enumerate(zip(RADII_L, RADII_R)):
        fl, fr = FOCI[i], FOCI[-1 - i]
        for p in (pair, into, host):
            p.set_focus_radius(0, rl)
            p.set_focus_radius(1, rr)
            if i % 2:
                p.set_focus(0, *fl), p.set_focus(1, *fr)
            else:
                p.clear_focus(0), p.clear_focus(1)
        if not i % 2:
            fl = fr = (.5, .5)
        a, b = pair.apply_pair(tl, tr)
        for eye, t in ((0, tl), (1, tr)):
            into.apply_into(eye, t, arr[eye])
            host.apply_host(eye, src[eye], dst[eye])
        torch.cuda.synchronize()
        wa, wb = _oracle(left, 0, True, fl + fl, rl, "fsr"), _oracle(right, 1, True, fr + fr, rr, "fsr")
        assert np.array_equal(a.cpu().numpy(), wa) and np.array_equal(b.cpu().numpy(), wb), (rl, rr)
        assert np.array_equal(arr[0].download().cpu().numpy(), wa) and np.array_equal(arr[1].download().cpu().numpy(), wb)
        assert np.array_equal(dst[0].numpy(), wa) and np.array_equal(dst[1].numpy(), wb)
    for p in (pair, into, host):
        p.close()
    for d in arr:
        d.close()


@pytest.mark.parametrize("use_nis", [0, 1])
def test_cpp_dropin_set_focus_radius(cuda, built_lib, tmp_path, use_nis):
    """vr::PostProcessor::SetFocusRadius before the first Apply, across a Reset, then ClearFocusRadius
    (tests/cpp/pp_focus_radius_selftest.cpp)"""
    from openvr_fsr_b200 import synth
    exe = tmp_path / "pp_focus_radius_selftest"
    pkg = ROOT / "openvr_fsr_b200"
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-I", str(pkg / "csrc"), "-I", str(ROOT / "include"),
                           str(ROOT / "tests/cpp/pp_focus_radius_selftest.cpp"), "-o", str(exe), "-L", str(pkg), "-lovrfsr",
                           "-Xlinker", f"-rpath={pkg}"])
    eyes = synth.stereo_pair("natural", IW, IH, 23)
    radii = (0.2, 1.5)
    ins = [tmp_path / f"in{e}.rgba" for e in (0, 1)]
    outs = [tmp_path / f"{k}{e}.rgba" for k in ("set", "clear") for e in (0, 1)]
    for p, img in zip(ins, eyes):
        p.write_bytes(img.tobytes())
    args = [str(exe), *map(str, ins), str(IW), str(IH), str(SCALE), str(SHARP), "0.5", str(use_nis),
            *(str(r) for r in radii), *map(str, outs)]
    out = subprocess.run(args, capture_output=True, text=True)
    assert out.returncode == 0 and "pp_focus_radius_selftest: ok" in out.stdout, out.stdout + out.stderr
    from oracle import pyoracle as po
    ow, oh = po.output_size(IW, IH, SCALE)
    mode = "nis" if use_nis else "fsr"
    centre = (.5, .5, .5, .5)
    for e in (0, 1):
        got = [np.frombuffer(outs[k * 2 + e].read_bytes(), dtype=np.uint8).reshape(oh, ow, 4) for k in (0, 1)]
        assert np.array_equal(got[0], _oracle(eyes[e], e, True, centre, radii[e], mode))
        assert np.array_equal(got[1], _oracle(eyes[e], e, True, centre, 0.5, mode))
