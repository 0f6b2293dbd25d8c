"""ovrfsr_set_focus: the radius mask follows a per-eye focus that is set every frame and latched on the GPU when the
frame runs.  An apply with focus (x, y) gives the bits of an apply whose proj_centre is (x, y) -- checked against the
oracle in strict math, against a ctx configured with that projection centre in fast math -- on every ctx path; the
focus costs no reset, follows a captured CUDA graph across replays, and is never torn inside an (x, y) pair."""
import subprocess
import threading
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]

IW, IH, SCALE, SHARP = 211, 157, 0.75, 0.9
FOCI = [(0.5, 0.5), (0.2, 0.3), (0.8, 0.7), (0.0, 1.0), (0.35, 0.6)]


def _oracle(img, eye, one, proj, radius, mode, scale=SCALE, sharp=SHARP):
    """strict oracle output of one eye: mode 'fsr' (EASU -> RCAS, also what the fused kernel gives), 'nis' (NVScaler at
    scale < 1, NVSharpen at scale 1)"""
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
    "nis_scaler": (dict(renderScale=SCALE, useNis=True), "nis"),
    "nis_sharpen": (dict(renderScale=1.0, useNis=True), "nis"),
}


@pytest.mark.parametrize("radius", [0.3, 0.5])
@pytest.mark.parametrize("path", list(PATHS))
def test_focus_sequence_matches_oracle_strict(cuda, path, radius):
    import torch
    import openvr_fsr_b200 as ovr
    kw, mode = PATHS[path]
    (left, right), (tl, tr) = _eyes(torch, cuda)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, sharpness=SHARP, radius=radius, mathMode=ovr.MATH_STRICT, **kw))
    for i, fl in enumerate(FOCI):
        fr = FOCI[-1 - i]
        pp.set_focus(0, *fl)
        pp.set_focus(1, *fr)
        for eye, (img, t, f) in enumerate(((left, tl, fl), (right, tr, fr))):
            got = pp.apply(eye, t).cpu().numpy()
            want = _oracle(img, eye, True, f + f, radius, mode, scale=kw["renderScale"])
            assert np.array_equal(got, want), (path, eye, f)
    pp.close()


@pytest.mark.parametrize("path", list(PATHS))
def test_focus_fast_math_equals_projection_centre(cuda, path):
    """fast math: the same bits as a ctx whose proj_centre is the focus (the same kernels read the same words)"""
    import dataclasses
    import torch
    import openvr_fsr_b200 as ovr
    kw, _ = PATHS[path]
    _, (tl, tr) = _eyes(torch, cuda, 5)
    cfg = ovr.Config(fsrEnabled=True, sharpness=SHARP, radius=0.3, mathMode=ovr.MATH_FAST, **kw)
    pp = ovr.PostProcessor(cfg)
    for fl, fr in zip(FOCI, FOCI[::-1]):
        pp.set_focus(0, *fl)
        pp.set_focus(1, *fr)
        ref = ovr.PostProcessor(dataclasses.replace(cfg, projCentre=fl + fr))
        for eye, t in ((0, tl), (1, tr)):
            assert torch.equal(pp.apply(eye, t), ref.apply(eye, t)), (path, eye)
        ref.close()
    pp.close()


def test_focus_apply_into_array_destination(cuda):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    (left, right), (tl, tr) = _eyes(torch, cuda, 7)
    ow, oh = po.output_size(IW, IH, SCALE)
    dst = [ovr.ArrayImage(ow, oh), ovr.ArrayImage(ow, oh)]
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.3))
    for fl, fr in zip(FOCI[1:], FOCI[:0:-1]):
        pp.set_focus(0, *fl)
        pp.set_focus(1, *fr)
        for eye, (img, t, f) in enumerate(((left, tl, fl), (right, tr, fr))):
            pp.apply_into(eye, t, dst[eye])
            assert np.array_equal(dst[eye].download().cpu().numpy(), _oracle(img, eye, True, f + f, 0.3, "fsr"))
    pp.close()
    for d in dst:
        d.close()


def test_focus_apply_pair_and_apply_host(cuda):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    (left, right), (tl, tr) = _eyes(torch, cuda, 9)
    ow, oh = po.output_size(IW, IH, SCALE)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.5))
    host = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.5))
    src = [torch.from_numpy(left).pin_memory(), torch.from_numpy(right).pin_memory()]
    dst = [torch.empty((oh, ow, 4), dtype=torch.uint8).pin_memory() for _ in range(2)]
    for fl, fr in zip(FOCI, FOCI[::-1]):
        for p in (pp, host):
            p.set_focus(0, *fl)
            p.set_focus(1, *fr)
        a, b = pp.apply_pair(tl, tr)
        for eye in (0, 1):
            host.apply_host(eye, src[eye], dst[eye])
        torch.cuda.synchronize()
        wa, wb = _oracle(left, 0, True, fl + fl, 0.5, "fsr"), _oracle(right, 1, True, fr + fr, 0.5, "fsr")
        assert np.array_equal(a.cpu().numpy(), wa) and np.array_equal(b.cpu().numpy(), wb)
        assert np.array_equal(dst[0].numpy(), wa) and np.array_equal(dst[1].numpy(), wb)
    pp.close(), host.close()


def test_focus_shared_texture_takes_both_eyes_foci(cuda):
    """one texture holding both eyes: centre pair 0 is the left eye's focus, pair 1 the right eye's"""
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    tex_np = synth.natural_rgba8(320, 120, 21)
    tex = torch.from_numpy(tex_np).to(cuda)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.3))
    for fl, fr in ((FOCI[1], FOCI[2]), (FOCI[3], FOCI[1])):
        pp.set_focus(0, *fl)
        pp.set_focus(1, *fr)
        left = pp.apply(ovr.EYE_LEFT, tex, ovr.TextureBounds(0.0, 0.0, 0.5, 1.0))
        right = pp.apply(ovr.EYE_RIGHT, tex, ovr.TextureBounds(0.5, 0.0, 1.0, 1.0))
        assert left.data_ptr() == right.data_ptr()
        assert np.array_equal(left.cpu().numpy(), _oracle(tex_np, 0, False, fl + fr, 0.3, "fsr"))
    pp.close()


def test_focus_at_projection_centre_and_clear_give_reference_bytes(cuda):
    import torch
    import openvr_fsr_b200 as ovr
    proj = (.45, .5, .55, .5)
    _, (tl, tr) = _eyes(torch, cuda, 13)
    cfg = ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.3, projCentre=proj)
    pp, ref = ovr.PostProcessor(cfg), ovr.PostProcessor(cfg)
    want = [ref.apply(0, tl).clone(), ref.apply(1, tr).clone()]
    pp.set_focus(0, proj[0], proj[1])
    pp.set_focus(1, proj[2], proj[3])
    assert torch.equal(pp.apply(0, tl), want[0]) and torch.equal(pp.apply(1, tr), want[1])
    pp.set_focus(0, 0.1, 0.9)
    pp.set_focus(1, 0.9, 0.1)
    assert not torch.equal(pp.apply(0, tl), want[0]) and not torch.equal(pp.apply(1, tr), want[1])
    pp.clear_focus(0)
    assert torch.equal(pp.apply(0, tl), want[0]) and not torch.equal(pp.apply(1, tr), want[1])
    pp.clear_focus(1)
    assert torch.equal(pp.apply(0, tl), want[0]) and torch.equal(pp.apply(1, tr), want[1])
    pp.close(), ref.close()


def test_focus_needs_no_reset(cuda):
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
    for i, f in enumerate(FOCI * 3):
        pp.set_focus(i % 2, *f)
        n0 = ovr.kernel_launches()
        assert [pp.apply(0, tl).data_ptr(), pp.apply(1, tr).data_ptr()] == ptrs
        assert ovr.kernel_launches() - n0 == per_frame
        torch.cuda.synchronize()
    ms, n = pp.gpu_time_ms()
    assert n >= 6 and 0.0 < ms < 50.0
    pp.close()


def test_focus_follows_a_captured_graph(cuda):
    import torch
    import openvr_fsr_b200 as ovr
    (left, right), (tl, tr) = _eyes(torch, cuda, 17)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.3))
    pp.set_focus(0, *FOCI[1])
    pp.set_focus(1, *FOCI[2])
    pp.apply_pair(tl, tr)  # lazy init outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        a, b = pp.apply_pair(tl, tr, stream=torch.cuda.current_stream(cuda))
    for fl, fr in zip(FOCI, FOCI[::-1]):
        pp.set_focus(0, *fl)
        pp.set_focus(1, *fr)
        a.zero_(), b.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(a.cpu().numpy(), _oracle(left, 0, True, fl + fl, 0.3, "fsr"))
        assert np.array_equal(b.cpu().numpy(), _oracle(right, 1, True, fr + fr, 0.3, "fsr"))
    pp.clear_focus(0)  # the captured copy now reads the projection centre
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(a.cpu().numpy(), _oracle(left, 0, True, (.5, .5, .5, .5), 0.3, "fsr"))
    del g
    pp.close()


def test_focus_updates_from_another_thread_never_tear_a_pair(cuda):
    """A thread cycles the focus through three points while 200 frames run: a frame may mix the two centre pairs of
    its block (one per update), never the x of one update with the y of another -- so every frame is one of the 9
    oracle outputs of (pair 0 from point i, pair 1 from point j)."""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    (left, _), (tl, _) = _eyes(torch, cuda, 19)
    ow, oh = po.output_size(IW, IH, SCALE)
    points = [(0.25, 0.3), (0.5, 0.5), (0.75, 0.7)]
    want = {}
    for i, pi in enumerate(points):
        for j, pj in enumerate(points):
            uc = po.upscale_constants(0, True, IW, IH, ow, oh, proj=pi + pi, radius=0.3)
            sc = po.sharpen_constants(0, True, ow, oh, proj=pi + pi, radius=0.3, sharpness=SHARP)
            other = po.upscale_constants(0, True, IW, IH, ow, oh, proj=pj + pj, radius=0.3)
            for c in (uc, sc):
                c.imageCentre[2], c.imageCentre[3] = other.imageCentre[2], other.imageCentre[3]
            want[po.rcas(po.easu(left, ow, oh, uc), sc).tobytes()] = (i, j)
    assert len({want[k] for k in want if want[k][0] == want[k][1]}) == 3  # the three points give three images
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=0.3))
    pp.set_focus(0, *points[0])
    stop = threading.Event()

    def cycle():
        k = 0
        while not stop.is_set():
            pp.set_focus(0, *points[k % 3])
            k += 1

    th = threading.Thread(target=cycle)
    th.start()
    try:
        for _ in range(200):
            assert pp.apply(0, tl).cpu().numpy().tobytes() in want
    finally:
        stop.set()
        th.join()
    pp.close()


@pytest.mark.parametrize("use_nis", [0, 1])
def test_cpp_dropin_set_focus(cuda, built_lib, tmp_path, use_nis):
    """vr::PostProcessor::SetFocus before the first Apply, across a Reset, then ClearFocus (tests/cpp/pp_focus_selftest.cpp)"""
    from openvr_fsr_b200 import synth
    exe = tmp_path / "pp_focus_selftest"
    pkg = ROOT / "openvr_fsr_b200"
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-I", str(pkg / "csrc"), "-I", str(ROOT / "include"),
                           str(ROOT / "tests/cpp/pp_focus_selftest.cpp"), "-o", str(exe), "-L", str(pkg), "-lovrfsr",
                           "-Xlinker", f"-rpath={pkg}"])
    eyes = synth.stereo_pair("natural", IW, IH, 23)
    foci = ((0.3, 0.4), (0.7, 0.6))
    ins = [tmp_path / f"in{e}.rgba" for e in (0, 1)]
    outs = [tmp_path / f"{k}{e}.rgba" for k in ("focus", "clear") for e in (0, 1)]
    for p, img in zip(ins, eyes):
        p.write_bytes(img.tobytes())
    args = [str(exe), *map(str, ins), str(IW), str(IH), str(SCALE), str(SHARP), "0.3", str(use_nis),
            *(str(v) for f in foci for v in f), *map(str, outs)]
    out = subprocess.run(args, capture_output=True, text=True)
    assert out.returncode == 0 and "pp_focus_selftest: ok" in out.stdout, out.stdout + out.stderr
    from oracle import pyoracle as po
    ow, oh = po.output_size(IW, IH, SCALE)
    mode = "nis" if use_nis else "fsr"
    for e in (0, 1):
        got = [np.frombuffer(outs[k * 2 + e].read_bytes(), dtype=np.uint8).reshape(oh, ow, 4) for k in (0, 1)]
        assert np.array_equal(got[0], _oracle(eyes[e], e, True, foci[e] + foci[e], 0.3, mode))
        assert np.array_equal(got[1], _oracle(eyes[e], e, True, (.5, .5, .5, .5), 0.3, mode))
