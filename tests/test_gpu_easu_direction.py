"""EASU's direction threshold on the device: every EASU filter launch on content whose dir^2 sits on 2^-15.

FsrEasuF's `zro = dir.x^2 + dir.y^2 < 1/32768` turns the anisotropic kernel by up to 90 degrees on a last-bit
difference in dir^2 (tests/easu_direction.py).  The cases of tests/easu_direction.py -- FP32 / FP16 luma ramps under
iso-luminant chroma with most pixels within a few ulps of the threshold, UNORM iso-luminant cells, UNORM luma flat to
the last bit under chroma edges -- run through every kernel whose pixels go through easu_filter / easu_filter_fast:

  * the plain dispatch (`easu_kernel`, PAIRED=0): pitch-aligned (TMA loader for UNORM sources) and tight odd-width
    sources, CUDA-array sources into pitched and CUDA-array destinations, into the UNORM target and RGBA16F / RGBA32F;
  * the paired context path (`easu_kernel`, PAIRED=1, then RCAS): a PostProcessor with a UNORM output, both eyes;
  * the fused kernel (`fsr_fused_kernel`) at render scale 0.77 (60-column tile) and at an anisotropic size that takes
    its 72-column tile;

each at render scale 0.77 and 0.9 (EASU's 60- and 72-column tiles), every group inside the radius.  Strict math is
compared with the oracle bit for bit; fast math per pass within test_gpu_variant_matrix.py's bounds (1 LSB / 1 code /
1e-3 relative) and composed within 4 LSB.  A failure names the case, the pixel, its dir^2 in ulps from 2^-15 and the
branch the oracle took there.  The test prints, per case and kernel, the near-threshold pixel count and how many pixels
fast math moved by more than 1 LSB."""
import math

import numpy as np
import pytest

from tests import easu_direction as ed
from tests import kernel_ledger as kl

pytestmark = pytest.mark.gpu

SHARP = 0.8
SCALES = (0.77, 0.9)


def _tag(fmt):
    return fmt if fmt in (ed.BGRA8, ed.RGB10A2, ed.BGRX8) else None


def _unorm(fmt):
    return ed.RGB10A2 if fmt == ed.RGB10A2 else ed.RGBA8


def _dtype(fmt):
    import torch
    return {ed.RGBA16F: torch.float16, ed.RGBA32F: torch.float32}.get(fmt, torch.uint8)


def _np_dtype(fmt):
    return {ed.RGBA16F: np.float16, ed.RGBA32F: np.float32}.get(fmt, np.uint8)


def _place(arr, fmt, where, dev):
    """'tma': pitch-aligned device image; 'tight': packed rows (odd width: no TMA box); 'array': CUDA array"""
    import torch
    import openvr_fsr_b200 as ovr
    if where == "tma":
        return ovr.to_image(arr, dev)
    t = torch.from_numpy(arr).to(dev)
    return t if where == "tight" else ovr.ArrayImage(arr.shape[1], arr.shape[0], fmt).upload(t)


def _host(d):
    import openvr_fsr_b200 as ovr
    return (d.download() if isinstance(d, ovr.ArrayImage) else d).cpu().numpy()


def _units(a, fmt):
    from openvr_fsr_b200 import synth
    return synth.unpack_rgb10a2(a)[..., :3] if fmt == ed.RGB10A2 else a[..., :3].astype(np.int64)


def _compare(label, got, want, fmt, mode, composed, dir2, zro, stats):
    """assert the bound; record the near-threshold count and the fast-math error in stats[label]"""
    assert got.shape == want.shape, (label, got.shape, want.shape)
    ulps = ed.ulps_from_threshold(dir2)

    def where(y, x):
        return (f"pixel (x={x}, y={y}): dir^2 {int(ulps[y, x]):+d} ulps from 2^-15, oracle "
                f"{'zro (dir = (1, dir.y))' if zro[y, x] else 'normalised dir / |dir|'}")

    if mode == "strict":
        bad = np.argwhere((np.ascontiguousarray(got).view(np.uint8) != np.ascontiguousarray(want).view(np.uint8))
                          .reshape(got.shape[0], got.shape[1], -1).any(axis=-1))
        assert len(bad) == 0, f"{label}: {len(bad)} pixels differ from the oracle, first at {where(*bad[0])}"
        return
    if fmt in (ed.RGBA16F, ed.RGBA32F):
        g, w = got[..., :3].astype(np.float64), want[..., :3].astype(np.float64)
        err = np.abs(g - w) / np.maximum(1.0, np.abs(w))
        err = np.where(np.isfinite(err), err, np.inf).max(axis=-1)
        y, x = np.unravel_index(np.argmax(err), err.shape)
        stats[label] = (float(err.max()), int((err > 1e-3).sum()))
        assert err.max() <= 1e-3, f"{label}: relative error {err.max():.3g} > 1e-3 at {where(y, x)}"
        return
    d = np.abs(_units(got, fmt) - _units(want, fmt)).max(axis=-1)
    y, x = np.unravel_index(np.argmax(d), d.shape)
    stats[label] = (int(d.max()), int((d > 1).sum()))
    bound = 4 if composed else 1
    assert d.max() <= bound, f"{label}: {int((d > 1).sum())} pixels beyond 1, max {int(d.max())} > {bound} at {where(y, x)}"


def _one_launch(fn):
    """run fn(); the library must have launched exactly one kernel for it (the instantiation each layout selects is
    recorded and checked by test_gpu_variant_matrix.py, whose sizes and placements these follow)"""
    import openvr_fsr_b200 as ovr
    n0 = ovr.kernel_launches()
    out = fn()
    assert ovr.kernel_launches() == n0 + 1, f"{ovr.kernel_launches() - n0} launches"
    return out


def _setup(name, scale):
    from oracle import pyoracle as po
    fmt, iw, ih, case_scale, _, _, _, min_near = ed.CASES[name]
    src = ed.case_source(name)
    ow, oh = po.output_size(iw, ih, scale)
    return fmt, iw, ih, ow, oh, src, (min_near if scale == case_scale else 0)


def _report(name, scale, mode, near, stats):
    print(f"\n{name} scale {scale} {mode}: {near[0]} pixels within 2 ulps of 2^-15 ({near[1]} zro, {near[2]} normalised)")
    for label, (mx, beyond) in sorted(stats.items()):
        print(f"  {label}: fast max {mx:.3g}, {beyond} pixels beyond the per-pass bound" if isinstance(mx, float)
              else f"  {label}: fast max {mx}, {beyond} pixels moved by more than 1")


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("name", sorted(ed.CASES))
def test_plain_dispatch_on_the_threshold(cuda, name, scale, mode):
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    fmt, iw, ih, ow, oh, src, min_near = _setup(name, scale)
    mm = ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST
    uc = po.upscale_constants(0, True, iw, ih, ow, oh, radius=2.0)  # every group inside: the filter at every pixel
    _, dir2, zro = ed.easu(src, fmt, uc.words(), ow, oh)
    near = ed.near_threshold(dir2, zro)
    assert near[0] >= min_near, f"{name}: {near[0]} near-threshold pixels at scale {scale}, promised {min_near}"
    packed = fmt not in (ed.RGBA16F, ed.RGBA32F)
    layouts = ([("tma", ["pitched"])] if packed else []) + [("tight", ["pitched"]), ("array", ["pitched", "array"])]
    stats, failures = {}, []
    for fout in (_unorm(fmt), ed.RGBA16F, ed.RGBA32F):
        want = po.easu(src, ow, oh, uc, out_dtype=_np_dtype(fout), src_fmt=_tag(fmt), dst_fmt=_tag(fout))
        for where, kinds in layouts:
            s = _place(src, fmt, where, cuda)
            for kind in kinds:
                d = ovr.ArrayImage(ow, oh, fout) if kind == "array" else ovr.alloc_image(ow, oh, _dtype(fout), cuda)

                def run():
                    ovr.fsr_easu(s, d, uc.words(), mm, src_fmt=None if where == "array" else _tag(fmt),
                                 dst_fmt=None if kind == "array" else _tag(fout))
                    return _host(d)
                got = _one_launch(run)
                label = f"{name} {where}->{kind} {kl.FORMAT_NAMES[fout]}"
                try:
                    _compare(label, got, want, fout, mode, False, dir2, zro, stats)
                except AssertionError as e:
                    failures.append(str(e))
    _report(name, scale, mode, near, stats)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("name", sorted(ed.CASES))
def test_paired_context_on_the_threshold(cuda, name, scale, mode):
    """PostProcessor with a UNORM output: paired EASU + RCAS, both eyes (the second eye a shifted copy)"""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    fmt, iw, ih, ow, oh, src, _ = _setup(name, scale)
    unorm = _unorm(fmt)
    eyes = [src, np.ascontiguousarray(np.roll(src, 3, axis=1))]
    stats, failures = {}, []
    wheres = (["tma"] if fmt not in (ed.RGBA16F, ed.RGBA32F) else []) + ["tight", "array"]
    for where in wheres:
        pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=scale, sharpness=SHARP, radius=2.0,
                                          mathMode=ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST))
        srcs = [_place(e, fmt, where, cuda) for e in eyes]
        if where == "array":
            dsts = [ovr.ArrayImage(ow, oh, unorm) for _ in eyes]
            pp.apply_pair_into(srcs[0], srcs[1], dsts[0], dsts[1])
            got = [_host(d) for d in dsts]
        else:
            got = [t.cpu().numpy() for t in pp.apply_pair(srcs[0], srcs[1], fmt=_tag(fmt))]
        torch.cuda.synchronize()
        pp.close()
        for e in (0, 1):
            uc = po.upscale_constants(e, True, iw, ih, ow, oh, radius=2.0)
            sc = po.sharpen_constants(e, True, ow, oh, radius=2.0, sharpness=SHARP)
            _, dir2, zro = ed.easu(eyes[e], fmt, uc.words(), ow, oh)
            want = po.rcas(po.easu(eyes[e], ow, oh, uc, src_fmt=_tag(fmt), dst_fmt=_tag(unorm)), sc,
                           src_fmt=_tag(unorm), dst_fmt=_tag(unorm))
            try:
                _compare(f"{name} paired {where} eye {e}", got[e], want, unorm, mode, True, dir2, zro, stats)
            except AssertionError as err:
                failures.append(str(err))
    _, dir2, zro = ed.easu(src, fmt, po.upscale_constants(0, True, iw, ih, ow, oh, radius=2.0).words(), ow, oh)
    _report(name, scale, mode, ed.near_threshold(dir2, zro), stats)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("tw", [60, 72])
@pytest.mark.parametrize("name", sorted(ed.CASES))
def test_fused_on_the_threshold(cuda, name, tw, mode):
    """the fused EASU -> RCAS kernel; its 72-column tile at out->in about 0.9 wide and 0.64 tall"""
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    fmt, iw, ih, _, _, src, _ = _setup(name, 0.77)
    if tw == 60:
        ow, oh = po.output_size(iw, ih, 0.77)
    else:
        ow, oh = math.ceil(iw / 0.898), math.ceil(ih / 0.635)
    mid = _unorm(fmt)
    uc = po.upscale_constants(0, True, iw, ih, ow, oh, radius=2.0)
    sc = po.sharpen_constants(0, True, ow, oh, radius=2.0, sharpness=SHARP)
    _, dir2, zro = ed.easu(src, fmt, uc.words(), ow, oh)
    want = po.rcas(po.easu(src, ow, oh, uc, src_fmt=_tag(fmt), dst_fmt=_tag(mid)), sc, src_fmt=_tag(mid), dst_fmt=_tag(mid))
    stats, failures = {}, []
    wheres = ["tma", "tight"] if fmt not in (ed.RGBA16F, ed.RGBA32F) else ["tight"]
    for where in wheres:
        s = _place(src, fmt, where, cuda)
        d = ovr.alloc_image(ow, oh, _dtype(mid), cuda)

        def run():
            ovr.fsr_fused(s, d, uc.words(), sc.words(), ovr.MATH_STRICT if mode == "strict" else ovr.MATH_FAST,
                          src_fmt=_tag(fmt), dst_fmt=_tag(mid))
            return _host(d)
        got = _one_launch(run)
        try:
            _compare(f"{name} fused TW={tw} {where}", got, want, mid, mode, True, dir2, zro, stats)
        except AssertionError as err:
            failures.append(str(err))
    _report(f"{name} fused", f"{ow}x{oh}", mode, ed.near_threshold(dir2, zro), stats)
    assert not failures, "\n".join(failures)
