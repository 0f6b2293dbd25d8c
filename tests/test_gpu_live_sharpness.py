"""ovrfsr_set_sharpness: the sharpness is changed every frame, without a reset, and latched on the GPU with the focus
when the frame runs.  An apply with sharpness override s gives the bytes of an apply whose config sharpness is s --
checked against the oracle in strict math, against a ctx configured with s in fast math -- on every ctx path (paired
FSR, fused, RCAS alone, SRTM, NVScaler, NVSharpen) and every apply entry point, with no focus, with a focus, and with a
focus and a radius override.  The override costs no reset, follows a captured CUDA graph across replays, survives
set_config, and a frame never sees a sharpness that was not set."""
import dataclasses
import subprocess
import threading
from pathlib import Path

import numpy as np
import pytest

from tests import test_gpu_focus_radius as fr
from tests import test_gpu_srtm as gs

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]

IW, IH, SCALE, CFG_SHARP = 211, 157, 0.75, 0.75
# both ends of the range, and either side of NIS's slider switch at 0.5
SHARPS = [0.0, 0.05, 0.37, 0.5, 0.62, 0.9, 1.0]
FOCI = [(0.5, 0.5), (0.2, 0.3), (0.8, 0.7), (0.0, 1.0), (0.35, 0.6), (0.6, 0.4), (0.45, 0.55)]
RADII = [0.3, 0.5, 0.0, 1.0, 2.0, 4.0, 0.7]
CENTRE = ((.5, .5), (.5, .5))

PATHS = {  # name: (Config kwargs, oracle mode)
    "fsr": (dict(renderScale=SCALE), "fsr"),
    "fused": (dict(renderScale=SCALE, fusedFsr=True), "fsr"),
    "rcas": (dict(renderScale=1.0), "fsr"),
    "srtm": (dict(renderScale=SCALE, srtm=True), "srtm"),
    "srtm_rcas": (dict(renderScale=1.0, srtm=True), "srtm"),
    "nis_scaler": (dict(renderScale=SCALE, useNis=True), "nis"),
    "nis_sharpen": (dict(renderScale=1.0, useNis=True), "nis"),
}


def _eyes(torch, dev, mode, seed=3):
    """UNORM eyes, or HDR RGBA16F eyes for the SRTM paths"""
    from openvr_fsr_b200 import synth
    if mode == "srtm":
        left = synth.natural_rgba16f(IW, IH, seed, peak=4.0)
        right = np.ascontiguousarray(np.roll(left, 16, axis=1))
    else:
        left, right = synth.stereo_pair("natural", IW, IH, seed)
    return (left, right), (torch.from_numpy(left).to(dev), torch.from_numpy(right).to(dev))


def _want(mode, img, eye, one, proj, radius, scale, sharp):
    """strict oracle output of one eye at sharpness `sharp` (RGBA8 output)"""
    if mode == "srtm":
        return gs._chain(img, eye, one, scale, radius, np.uint8, proj=proj, sharp=sharp)
    return fr._oracle(img, eye, one, proj, radius, mode, scale=scale, sharp=sharp)


@pytest.mark.parametrize("latch", ["sharpness", "focus", "focus_radius"])
@pytest.mark.parametrize("path", list(PATHS))
def test_sharpness_sequence_matches_oracle_strict(cuda, path, latch):
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L
    kw, mode = PATHS[path]
    (left, right), (tl, tr) = _eyes(torch, cuda, mode)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, sharpness=CFG_SHARP, radius=0.5, mathMode=ovr.MATH_STRICT, **kw))
    for i, s in enumerate(SHARPS):
        pp.set_sharpness(s)
        # a rejected value leaves the one just set
        assert L.lib().ovrfsr_set_sharpness(pp._ctx, 1.01) == L.ERR_INVALID
        assert L.lib().ovrfsr_set_sharpness(pp._ctx, float("nan")) == L.ERR_INVALID
        focus = (FOCI[i], FOCI[-1 - i]) if latch != "sharpness" else CENTRE
        radius = (RADII[i], RADII[-1 - i]) if latch == "focus_radius" else (0.5, 0.5)
        if latch != "sharpness":
            pp.set_focus(0, *focus[0]), pp.set_focus(1, *focus[1])
        if latch == "focus_radius":
            pp.set_focus_radius(0, radius[0]), pp.set_focus_radius(1, radius[1])
        for eye, (img, t) in enumerate(((left, tl), (right, tr))):
            got = pp.apply(eye, t).cpu().numpy()
            want = _want(mode, img, eye, True, focus[eye] + focus[eye], radius[eye], kw["renderScale"], s)
            assert np.array_equal(got, want), (path, latch, eye, s)
    pp.close()


@pytest.mark.parametrize("path", list(PATHS))
def test_sharpness_fast_math_equals_configured_sharpness(cuda, path):
    """fast math: the same bits as a ctx whose config sharpness (and projection centre) is the override (and focus)"""
    import torch
    import openvr_fsr_b200 as ovr
    kw, mode = PATHS[path]
    _, (tl, tr) = _eyes(torch, cuda, mode, 5)
    cfg = ovr.Config(fsrEnabled=True, sharpness=CFG_SHARP, radius=0.5, mathMode=ovr.MATH_FAST, **kw)
    pp = ovr.PostProcessor(cfg)
    for i, s in enumerate(SHARPS):
        pp.set_sharpness(s)
        fl, fr_ = FOCI[i], FOCI[-1 - i]
        use_focus = i % 2 == 1
        if use_focus:
            pp.set_focus(0, *fl), pp.set_focus(1, *fr_)
        else:
            pp.clear_focus(0), pp.clear_focus(1)
        for eye, t in ((0, tl), (1, tr)):
            ref = ovr.PostProcessor(dataclasses.replace(cfg, sharpness=s, **({"projCentre": fl + fr_} if use_focus else {})))
            assert torch.equal(pp.apply(eye, t), ref.apply(eye, t)), (path, eye, s, use_focus)
            ref.close()
    pp.close()


@pytest.mark.parametrize("path", list(PATHS))
def test_override_equal_to_config_clear_and_set_config(cuda, path):
    """an override equal to the config sharpness gives the reference bytes; clear restores the config's bytes; a
    set_config with another sharpness keeps the override, which then wins until it is cleared"""
    import torch
    import openvr_fsr_b200 as ovr
    kw, mode = PATHS[path]
    _, (tl, tr) = _eyes(torch, cuda, mode, 7)
    cfg = ovr.Config(fsrEnabled=True, sharpness=0.37, radius=0.5, **kw)
    pp, ref = ovr.PostProcessor(cfg), ovr.PostProcessor(cfg)
    want = [ref.apply(0, tl).clone(), ref.apply(1, tr).clone()]
    pp.set_sharpness(0.37)
    assert torch.equal(pp.apply(0, tl), want[0]) and torch.equal(pp.apply(1, tr), want[1])
    pp.set_sharpness(0.9)
    assert not torch.equal(pp.apply(0, tl), want[0]) and not torch.equal(pp.apply(1, tr), want[1])
    pp.clear_sharpness()
    assert torch.equal(pp.apply(0, tl), want[0]) and torch.equal(pp.apply(1, tr), want[1])
    pp.set_sharpness(0.37)
    pp.set_config(dataclasses.replace(cfg, sharpness=0.9))
    assert torch.equal(pp.apply(0, tl), want[0]) and torch.equal(pp.apply(1, tr), want[1])
    pp.clear_sharpness()
    ref.set_config(dataclasses.replace(cfg, sharpness=0.9))
    for eye, t in ((0, tl), (1, tr)):
        assert torch.equal(pp.apply(eye, t), ref.apply(eye, t)), eye
    pp.close(), ref.close()


@pytest.mark.parametrize("path", ["fsr", "fused", "rcas", "nis_scaler", "nis_sharpen"])
def test_sharpness_every_entry_point(cuda, path):
    """apply_pair, apply_pair_into CUDA arrays, apply_into from a CUDA-array source into a CUDA array, apply_host"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    kw, mode = PATHS[path]
    scale = kw["renderScale"]
    (left, right), (tl, tr) = _eyes(torch, cuda, mode, 9)
    ow, oh = po.output_size(IW, IH, scale)
    cfg = ovr.Config(fsrEnabled=True, sharpness=CFG_SHARP, radius=0.5, **kw)
    pair, pair_into, into, host = (ovr.PostProcessor(cfg) for _ in range(4))
    arr_pair = [ovr.ArrayImage(ow, oh), ovr.ArrayImage(ow, oh)]
    arr_src = [ovr.ArrayImage(IW, IH).upload(tl), ovr.ArrayImage(IW, IH).upload(tr)]
    arr_dst = [ovr.ArrayImage(ow, oh), ovr.ArrayImage(ow, oh)]
    src = [torch.from_numpy(left).pin_memory(), torch.from_numpy(right).pin_memory()]
    dst = [torch.empty((oh, ow, 4), dtype=torch.uint8).pin_memory() for _ in range(2)]
    for i, s in enumerate(SHARPS):
        for p in (pair, pair_into, into, host):
            p.set_sharpness(s)
            if i % 2:
                p.set_focus(0, *FOCI[i]), p.set_focus(1, *FOCI[-1 - i])
            else:
                p.clear_focus(0), p.clear_focus(1)
        focus = (FOCI[i], FOCI[-1 - i]) if i % 2 else CENTRE
        a, b = pair.apply_pair(tl, tr)
        pair_into.apply_pair_into(tl, tr, arr_pair[0], arr_pair[1])
        for eye in (0, 1):
            into.apply_into(eye, arr_src[eye], arr_dst[eye])
            host.apply_host(eye, src[eye], dst[eye])
        torch.cuda.synchronize()
        for eye, img, got in ((0, left, a), (1, right, b)):
            want = _want(mode, img, eye, True, focus[eye] + focus[eye], 0.5, scale, s)
            assert np.array_equal(got.cpu().numpy(), want), ("apply_pair", eye, s)
            assert np.array_equal(arr_pair[eye].download().cpu().numpy(), want), ("apply_pair_into", eye, s)
            assert np.array_equal(arr_dst[eye].download().cpu().numpy(), want), ("apply_into", eye, s)
            assert np.array_equal(dst[eye].numpy(), want), ("apply_host", eye, s)
    for p in (pair, pair_into, into, host):
        p.close()
    for d in arr_pair + arr_src + arr_dst:
        d.close()


@pytest.mark.parametrize("path", ["fsr", "fused", "rcas", "nis_scaler", "nis_sharpen"])
def test_sharpness_shared_texture(cuda, path):
    """one texture holding both eyes: both halves at the override, processed once per frame"""
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    kw, mode = PATHS[path]
    tex_np = synth.natural_rgba8(320, 120, 21)
    tex = torch.from_numpy(tex_np).to(cuda)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, sharpness=CFG_SHARP, radius=0.5, **kw))
    proj = (0.3, 0.4, 0.7, 0.6)
    pp.set_focus(0, *proj[:2]), pp.set_focus(1, *proj[2:])
    for s in SHARPS:
        pp.set_sharpness(s)
        left = pp.apply(ovr.EYE_LEFT, tex, ovr.TextureBounds(0.0, 0.0, 0.5, 1.0))
        right = pp.apply(ovr.EYE_RIGHT, tex, ovr.TextureBounds(0.5, 0.0, 1.0, 1.0))
        assert left.data_ptr() == right.data_ptr()
        assert np.array_equal(left.cpu().numpy(), _want(mode, tex_np, 0, False, proj, 0.5, kw["renderScale"], s)), (path, s)
    pp.close()


@pytest.mark.parametrize("path", ["fsr", "nis_scaler"])
def test_sharpness_needs_no_reset(cuda, path):
    """output images stay where they are, and each apply launches the kernels a frame without an override launches
    (the copy is not a launch)"""
    import torch
    import openvr_fsr_b200 as ovr
    kw, mode = PATHS[path]
    _, (tl, tr) = _eyes(torch, cuda, mode, 15)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, sharpness=CFG_SHARP, radius=0.5, **kw))
    ptrs = [pp.apply(0, tl).data_ptr(), pp.apply(1, tr).data_ptr()]
    n0 = ovr.kernel_launches()
    pp.apply(0, tl), pp.apply(1, tr)
    per_frame = ovr.kernel_launches() - n0
    for s in SHARPS * 2:
        pp.set_sharpness(s)
        n0 = ovr.kernel_launches()
        assert [pp.apply(0, tl).data_ptr(), pp.apply(1, tr).data_ptr()] == ptrs
        assert ovr.kernel_launches() - n0 == per_frame
    torch.cuda.synchronize()
    pp.close()


def test_sharpness_follows_a_captured_graph(cuda):
    import torch
    import openvr_fsr_b200 as ovr
    (left, right), (tl, tr) = _eyes(torch, cuda, "fsr", 17)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=CFG_SHARP, radius=0.5))
    pp.set_sharpness(0.2)
    pp.apply_pair(tl, tr)  # lazy init outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        a, b = pp.apply_pair(tl, tr, stream=torch.cuda.current_stream(cuda))
    for s in SHARPS:
        pp.set_sharpness(s)
        a.zero_(), b.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(a.cpu().numpy(), _want("fsr", left, 0, True, (.5,) * 4, 0.5, SCALE, s)), s
        assert np.array_equal(b.cpu().numpy(), _want("fsr", right, 1, True, (.5,) * 4, 0.5, SCALE, s)), s
    pp.clear_sharpness()  # the captured copy now reads the config's words
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(a.cpu().numpy(), _want("fsr", left, 0, True, (.5,) * 4, 0.5, SCALE, CFG_SHARP))
    del g
    pp.close()


@pytest.mark.parametrize("path", ["fsr", "nis_scaler"])
def test_sharpness_updates_from_another_thread_never_tear(cuda, path):
    """A thread alternates the sharpness between 0.2 and 0.9 while 200 frames run.  FSR reads one word: every frame is
    one of the two oracle outputs.  NIS reads two pairs, each published whole: every frame is one of the four
    strength / limit combinations of the two NISConfigs ovrfsr_make_nis_config builds."""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    kw, mode = PATHS[path]
    (left, _), (tl, _) = _eyes(torch, cuda, mode, 19)
    ow, oh = po.output_size(IW, IH, SCALE)
    values = (0.2, 0.9)
    cfg = ovr.Config(fsrEnabled=True, sharpness=CFG_SHARP, radius=0.5, **kw)
    if mode == "fsr":
        want = {_want(mode, left, 0, True, (.5,) * 4, 0.5, SCALE, s).tobytes() for s in values}
        assert len(want) == 2
    else:
        raw = [ovr.make_nis_config(dataclasses.replace(cfg, sharpness=s), False, 0, True, IW, IH, ow, oh)[0] for s in values]
        # bytes 32..39: kSharpStrengthMin / Scale, 40..47: kSharpLimitMin / Scale
        want = {po.nis_scaler(left, ow, oh, po.NISConfig.from_buffer_copy(a[:40] + b[40:48] + a[48:])).tobytes()
                for a in raw for b in raw}
        assert len(want) == 4
    pp = ovr.PostProcessor(cfg)
    pp.set_sharpness(values[0])
    stop = threading.Event()

    def cycle():
        n = 0
        while not stop.is_set():
            pp.set_sharpness(values[n % 2])
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


def test_capture_names_the_override(cuda, tmp_path):
    """F7 capture with config sharpness 0.9 and override 0.3: the file is named _s30_ and holds the 0.3 frame"""
    import torch
    import openvr_fsr_b200 as ovr
    (left, _), (tl, _) = _eyes(torch, cuda, "fsr", 21)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=0.9, radius=0.5))
    pp.set_sharpness(0.3)
    pp.request_capture(str(tmp_path))
    pp.apply(0, tl)
    torch.cuda.synchronize()
    path = Path(pp.last_capture_path())
    assert path.parent == tmp_path and "_fsr_s30_r50" in path.name, path
    img, _ = ovr.load_dds(str(path))
    assert np.array_equal(img, _want("fsr", left, 0, True, (.5,) * 4, 0.5, SCALE, 0.3))
    pp.close()


@pytest.mark.parametrize("use_nis", [0, 1])
def test_cpp_dropin_set_sharpness(cuda, built_lib, tmp_path, use_nis):
    """vr::PostProcessor::SetSharpness before the first Apply, across a Reset, then ClearSharpness
    (tests/cpp/pp_sharpness_selftest.cpp)"""
    from openvr_fsr_b200 import synth
    exe = tmp_path / "pp_sharpness_selftest"
    pkg = ROOT / "openvr_fsr_b200"
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-I", str(pkg / "csrc"), "-I", str(ROOT / "include"),
                           str(ROOT / "tests/cpp/pp_sharpness_selftest.cpp"), "-o", str(exe), "-L", str(pkg), "-lovrfsr",
                           "-Xlinker", f"-rpath={pkg}"])
    eyes = synth.stereo_pair("natural", IW, IH, 23)
    override = 0.37
    ins = [tmp_path / f"in{e}.rgba" for e in (0, 1)]
    outs = [tmp_path / f"{k}{e}.rgba" for k in ("set", "clear") for e in (0, 1)]
    for p, img in zip(ins, eyes):
        p.write_bytes(img.tobytes())
    args = [str(exe), *map(str, ins), str(IW), str(IH), str(SCALE), str(CFG_SHARP), "0.5", str(use_nis), str(override),
            *map(str, outs)]
    out = subprocess.run(args, capture_output=True, text=True)
    assert out.returncode == 0 and "pp_sharpness_selftest: ok" in out.stdout, out.stdout + out.stderr
    from oracle import pyoracle as po
    ow, oh = po.output_size(IW, IH, SCALE)
    mode = "nis" if use_nis else "fsr"
    for e in (0, 1):
        got = [np.frombuffer(outs[k * 2 + e].read_bytes(), dtype=np.uint8).reshape(oh, ow, 4) for k in (0, 1)]
        assert np.array_equal(got[0], _want(mode, eyes[e], e, True, (.5,) * 4, 0.5, SCALE, override))
        assert np.array_equal(got[1], _want(mode, eyes[e], e, True, (.5,) * 4, 0.5, SCALE, CFG_SHARP))
