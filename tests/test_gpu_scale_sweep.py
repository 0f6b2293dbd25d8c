"""The stateless resampling dispatches against the oracle across the whole out->in scale range, set separately per axis.

Every other parity test draws its scale from about ten render scales (out/in 1.07x to 2x, the same in x and y).  Here
each axis gets its own ratio: a slight shrink up to the launcher's refusal, 1.0-1.07x densely, 1.07-2x in steps of
0.05, 2.5x, 3x, 4x and 8x, anisotropic pairs (1.02x by 3x, 1.9x by 1.05x, ...), and the decision boundaries of the
launchers' tile sizing from test_resample_footprint_host.py, one float32 ulp of c0 on each side (the dispatches take
any constant words, so c0 is set directly there, on extents whose ratio matches it: Bilinear() positions itself from
the extents, the tile from c0, and the two agree only when the constants describe the images; NVScaler's kScale
boundaries 0.5 and 1 use real extents, one source texel either side).  Images are long and thin (12288 x 40 and 40 x 12288 outputs) so that
tiles sit beyond x = 8192 (and y = 8192), where float32 source positions round differently, while the oracle stays
cheap.  The radius mask is a circle whose edge crosses the long axis, so every image has filtered and bilinear groups.

Kernels: EASU (then RCAS on its output), the fused EASU->RCAS kernel, NVScaler (including kScale < 0.5, where the
config's tuning words are all zero, as NVScalerUpdateConfig leaves them) and the CAS upscale.  Packed sources run with
both loaders: a 16-byte aligned pitch (TMA) and a pitch that is not (plain loads); RGBA16F / RGBA32F sources and float
targets run too.  Strict math is bit for bit (the sign of zero included), fast math within the variant matrix's bounds.
Every case either matches the oracle or is refused with OVRFSR_ERR_UNSUPPORTED; the refused shapes are the same for
both loaders and are exactly those the host statement of the launchers' rule refuses."""
import os
import time
from collections import defaultdict

import numpy as np
import pytest

from tests import kernel_ledger as kl
from tests import test_resample_footprint_host as fp
from tests.test_gpu_variant_matrix import _check, _content, _dtype, _np_dtype, _tag

pytestmark = pytest.mark.gpu

F = np.float32
LONG, SHORT = 12288, 40
SHARP = 0.8
NTHREADS = max(1, min(16, os.cpu_count() or 1))

# out/in ratio per axis: a shrink down to the refusal, 1.0-1.07 densely, 1.07-2 by 0.05, then 2.5, 3, 4, 8
RATIOS = ([1 / 1.07, 1 / 1.06, 1 / 1.05, 1 / 1.03, 1 / 1.01] + [1.0, 1.002, 1.005, 1.01, 1.02, 1.03, 1.04, 1.05, 1.06, 1.07]
          + [round(1.1 + 0.05 * i, 2) for i in range(19)] + [2.5, 3.0, 4.0, 8.0])
ANISO = [(1.02, 3.0), (1.9, 1.05), (3.0, 1.02), (1.05, 1.9), (8.0, 1.0), (1.0, 8.0), (1 / 1.05, 2.0), (2.0, 1 / 1.05)]
SOURCES = [kl.RGBA8, kl.RGB10A2, kl.RGBA16F, kl.BGRA8, kl.RGBA32F]
STATS = defaultdict(lambda: [0, 0])            # (kernel, loader) -> [matched, refused]
OUTCOME = defaultdict(lambda: defaultdict(set))  # (kernel, case) -> loader -> {refused?}
T0 = {}


# ---- shapes ----------------------------------------------------------------------------------------------------------
class Shape:
    """one case: output and source size, and optionally c0 words set straight from a host boundary (per axis)"""

    def __init__(self, name, ow, oh, iw, ih, c0x=None, c0y=None):
        self.name, self.ow, self.oh, self.iw, self.ih, self.c0x, self.c0y = name, ow, oh, iw, ih, c0x, c0y


def _insize(out, ratio):
    return max(1, int(round(out / ratio)))


def ratio_shapes():
    out = []
    for i, r in enumerate(RATIOS):
        other = RATIOS[(7 * i + 3) % len(RATIOS)]
        out.append(Shape(f"x{r:.4g}/y{other:.4g} wide", LONG, SHORT, _insize(LONG, r), _insize(SHORT, other)))
        out.append(Shape(f"x{other:.4g}/y{r:.4g} tall", SHORT, LONG, _insize(SHORT, other), _insize(LONG, r)))
    for rx, ry in ANISO:
        out.append(Shape(f"x{rx:.4g}/y{ry:.4g} wide", LONG, SHORT, _insize(LONG, rx), _insize(SHORT, ry)))
        out.append(Shape(f"x{rx:.4g}/y{ry:.4g} tall", SHORT, LONG, _insize(SHORT, rx), _insize(LONG, ry)))
    return out


def boundary_shapes(kernel):
    """one case on each side of every boundary of this kernel's launcher (the host test's boundary_c0): the long axis
    gets c0 straight from the boundary, with extents whose ratio agrees with it (fp.consistent_extents); the short axis
    a ratio from RATIOS"""
    xs, ys = fp.boundary_c0(kernel)
    out = []
    for i, c in enumerate(xs + ys):
        n, src = fp.consistent_extents(c, limit=LONG + 64)[-1]
        other = RATIOS[(5 * i + 1) % len(RATIOS)]
        if i < len(xs):
            out.append(Shape(f"c0x={c!r}/y{other:.4g} wide", n, SHORT, src, _insize(SHORT, other), c0x=c))
        else:
            out.append(Shape(f"x{other:.4g}/c0y={c!r} tall", SHORT, n, _insize(SHORT, other), src, c0y=c))
    return out


# ---- constants: a radius circle across the long axis, c0 overrides ------------------------------------------------
def _circle(s):
    """centre words and radius (squared) that make groups 0.35-0.9 of the long axis inside"""
    if s.ow >= s.oh:
        cx, cy, r = int(0.625 * s.ow), s.oh // 2, int(0.275 * s.ow)
    else:
        cx, cy, r = s.ow // 2, int(0.625 * s.oh), int(0.275 * s.oh)
    return [cx, cy, cx, cy], r


def _f2u(v):
    return int(np.array([v], dtype=F).view(np.uint32)[0])


def upscale_words(s):
    """(oracle UpscaleConstants, SharpenConstants) for the shape, with the circle and any c0 override"""
    from oracle import pyoracle as po
    uc = po.upscale_constants(0, True, s.iw, s.ih, s.ow, s.oh)
    sc = po.sharpen_constants(0, True, s.ow, s.oh, sharpness=SHARP)
    centre, r = _circle(s)
    for k in (uc, sc):
        for i in range(4):
            k.imageCentre[i] = centre[i]
        k.radius[0], k.radius[1] = r, r * r
    for axis, c in ((0, s.c0x), (1, s.c0y)):
        if c is not None:
            uc.const0[axis] = _f2u(c)
            uc.const0[axis + 2] = _f2u(F(F(0.5) * F(c) - F(0.5)))
    return uc, sc


def nis_config(s):
    """the oracle's NISConfig for the shape (tuning words zero below kScale 0.5, like the reference), with the circle"""
    from oracle import pyoracle as po
    cfg, ok = po.nis_config(False, 0, True, s.iw, s.ih, s.ow, s.oh, sharpness=SHARP)
    centre, r = _circle(s)
    for i in range(4):
        cfg.imageCentre[i] = centre[i]
    cfg.radius[0], cfg.radius[1] = r, r * r
    return cfg, ok


def _kscale(cfg):
    raw = np.frombuffer(bytes(cfg), dtype=F)
    return raw[12], raw[13]


# ---- images ------------------------------------------------------------------------------------------------------
def _place(arr, fmt, loader, dev):
    """'tma': a pitch-aligned device image; 'plain': a 4-byte format's rows padded to a pitch that is not a multiple of
    16 bytes (float sources have no TMA variant: their rows are packed)"""
    import torch
    import openvr_fsr_b200 as ovr
    if loader == "tma":
        return ovr.to_image(arr, dev)
    if fmt not in kl.PACKED32:
        return torch.from_numpy(arr).to(dev)
    h, w = arr.shape[:2]
    pad = next(p for p in range(1, 4) if ((w + p) * 4) % 16)
    t = torch.zeros((h, w + pad, 4), dtype=_dtype(fmt), device=dev)
    t[:, :w].copy_(torch.from_numpy(arr))
    return t[:, :w]


def _loaders(fmt):
    return ("tma", "plain") if fmt in kl.PACKED32 else ("plain",)


def _status(fn):
    """None on success, else the library status"""
    from openvr_fsr_b200 import _lib as L
    try:
        fn()
        return None
    except L.OvrFsrError as e:
        return e.status


def _record(kernel, loader, name, status):
    from openvr_fsr_b200 import _lib as L
    assert status in (None, L.ERR_UNSUPPORTED), f"{kernel} {name} [{loader}]: status {status}"
    STATS[(kernel, loader)][status is not None] += 1
    OUTCOME[(kernel, name)][loader].add(status is not None)


def _loader_mismatches(kernel):
    """cases of `kernel` whose two loaders were not both refused or both run"""
    return [name for (k, name), by in OUTCOME.items() if k == kernel and len(set().union(*by.values())) > 1]


def _modes():
    import openvr_fsr_b200 as ovr
    return (("strict", ovr.MATH_STRICT), ("fast", ovr.MATH_FAST))


def _targets(fmt, i):
    if fmt == kl.RGB10A2:
        return [kl.RGB10A2, (kl.RGBA16F, kl.RGBA32F)[i % 2]]
    return [kl.RGBA8, (kl.RGBA16F, kl.RGBA32F)[i % 2]]


# ---- runners -----------------------------------------------------------------------------------------------------
def run_easu(shapes, dev):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    fails = []
    for i, s in enumerate(shapes):
        fmt = SOURCES[i % len(SOURCES)]
        src = _content(fmt, s.iw, s.ih, 100 + i)
        uc, sc = upscale_words(s)
        c0x, c0y = np.frombuffer(bytes(uc.const0), dtype=F)[:2]
        for fout in _targets(fmt, i):
            want = None
            for loader in _loaders(fmt):
                expect_ok = fp.easu_layout(c0x, c0y, loader == "tma") is not None
                img = _place(src, fmt, loader, dev)
                for mode, mm in _modes():
                    dst = ovr.alloc_image(s.ow, s.oh, _dtype(fout), dev)
                    st = _status(lambda: ovr.fsr_easu(img, dst, uc.words(), mm, src_fmt=_tag(fmt), dst_fmt=_tag(fout)))
                    torch.cuda.synchronize()
                    _record("easu", loader, s.name, st)
                    if (st is None) != expect_ok:
                        fails.append(f"easu {s.name} [{loader}]: status {st}, host rule expects {'success' if expect_ok else 'refusal'}")
                    if st is not None:
                        continue
                    if want is None:
                        want = po.easu(src, s.ow, s.oh, uc, out_dtype=_np_dtype(fout), src_fmt=_tag(fmt), dst_fmt=_tag(fout),
                                       nthreads=NTHREADS)
                    msg, _ = _check(dst.cpu().numpy(), want, fout, mode, False)
                    if msg:
                        fails.append(f"easu {mode} {s.name} {kl.FORMAT_NAMES[fmt]}->{kl.FORMAT_NAMES[fout]} [{loader}]: {msg}")
            # RCAS on the upscaled image (the oracle's, so that each pass is held to its own bound)
            if want is not None and fout != kl.RGBA32F:
                rw = po.rcas(want, sc, out_dtype=_np_dtype(fout), src_fmt=_tag(fout), dst_fmt=_tag(fout), nthreads=NTHREADS)
                mid = ovr.to_image(want, dev)
                for mode, mm in _modes():
                    dst = ovr.alloc_image(s.ow, s.oh, _dtype(fout), dev)
                    ovr.fsr_rcas(mid, dst, sc.words(), mm, src_fmt=_tag(fout), dst_fmt=_tag(fout))
                    msg, _ = _check(dst.cpu().numpy(), rw, fout, mode, False)
                    if msg:
                        fails.append(f"rcas {mode} after easu {s.name} -> {kl.FORMAT_NAMES[fout]}: {msg}")
    return fails


def run_fused(shapes, dev):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    fails = []
    for i, s in enumerate(shapes):
        fmt = SOURCES[i % len(SOURCES)]
        fout = kl.RGB10A2 if fmt == kl.RGB10A2 else kl.RGBA8
        src = _content(fmt, s.iw, s.ih, 200 + i)
        uc, sc = upscale_words(s)
        c0x, c0y = np.frombuffer(bytes(uc.const0), dtype=F)[:2]
        want = None
        for loader in _loaders(fmt):
            expect_ok = fp.fused_layout(c0x, c0y, loader == "tma") is not None
            img = _place(src, fmt, loader, dev)
            for mode, mm in _modes():
                dst = ovr.alloc_image(s.ow, s.oh, _dtype(fout), dev)
                st = _status(lambda: ovr.fsr_fused(img, dst, uc.words(), sc.words(), mm, src_fmt=_tag(fmt), dst_fmt=_tag(fout)))
                torch.cuda.synchronize()
                _record("fused", loader, s.name, st)
                if (st is None) != expect_ok:
                    fails.append(f"fused {s.name} [{loader}]: status {st}, host rule expects {'success' if expect_ok else 'refusal'}")
                if st is not None:
                    continue
                if want is None:
                    mid = po.easu(src, s.ow, s.oh, uc, src_fmt=_tag(fmt), dst_fmt=_tag(fout), nthreads=NTHREADS)
                    want = po.rcas(mid, sc, src_fmt=_tag(fout), dst_fmt=_tag(fout), nthreads=NTHREADS)
                msg, _ = _check(dst.cpu().numpy(), want, fout, mode, True)
                if msg:
                    fails.append(f"fused {mode} {s.name} {kl.FORMAT_NAMES[fmt]} [{loader}]: {msg}")
    return fails


def run_nis(shapes, dev):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    fails = []
    for i, s in enumerate(shapes):
        fmt = SOURCES[i % len(SOURCES)]
        fout = _targets(fmt, i)[i % 2]
        src = _content(fmt, s.iw, s.ih, 300 + i)
        cfg, _ = nis_config(s)
        kx, ky = _kscale(cfg)
        expect_ok = fp.nis_accepts(kx, ky)
        want = None
        for loader in _loaders(fmt):
            img = _place(src, fmt, loader, dev)
            for mode, mm in _modes():
                dst = ovr.alloc_image(s.ow, s.oh, _dtype(fout), dev)
                st = _status(lambda: ovr.nis_scaler(img, dst, bytes(cfg), mm, src_fmt=_tag(fmt), dst_fmt=_tag(fout)))
                torch.cuda.synchronize()
                _record("nis", loader, s.name, st)
                if (st is None) != expect_ok:
                    fails.append(f"nis {s.name} [{loader}]: status {st}, kScale ({kx!r}, {ky!r})")
                if st is not None:
                    continue
                if want is None:
                    want = po.nis_scaler(src, s.ow, s.oh, cfg, out_dtype=_np_dtype(fout), src_fmt=_tag(fmt), dst_fmt=_tag(fout),
                                         nthreads=NTHREADS)
                msg, _ = _check(dst.cpu().numpy(), want, fout, mode, False)
                if msg:
                    fails.append(f"nis {mode} {s.name} kScale ({kx!r}, {ky!r}) {kl.FORMAT_NAMES[fmt]}->{kl.FORMAT_NAMES[fout]} "
                                 f"[{loader}]: {msg}")
    return fails


def run_cas(shapes, dev):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    fails = []
    for i, s in enumerate(shapes):
        fmt = SOURCES[i % len(SOURCES)]
        fout = _targets(fmt, i)[i % 2]
        src = _content(fmt, s.iw, s.ih, 400 + i)
        kc = po.cas_setup(SHARP, 1.0, s.iw, s.ih, s.ow, s.oh)
        expect_ok = s.ow >= s.iw and s.oh >= s.ih  # the CAS upscale refuses a shrink in either axis
        want = None
        for loader in _loaders(fmt):
            img = _place(src, fmt, loader, dev)
            for mode, mm in _modes():
                dst = ovr.alloc_image(s.ow, s.oh, _dtype(fout), dev)
                st = _status(lambda: ovr.cas(img, dst, kc.words(), False, mm, src_fmt=_tag(fmt), dst_fmt=_tag(fout)))
                torch.cuda.synchronize()
                _record("cas", loader, s.name, st)
                if (st is None) != expect_ok:
                    fails.append(f"cas {s.name} [{loader}]: status {st}")
                if st is not None:
                    continue
                if want is None:
                    want = po.cas(src, s.ow, s.oh, kc, False, out_dtype=_np_dtype(fout), src_fmt=_tag(fmt), dst_fmt=_tag(fout),
                                  nthreads=NTHREADS)
                msg, _ = _check(dst.cpu().numpy(), want, fout, mode, False)
                if msg:
                    fails.append(f"cas {mode} {s.name} {kl.FORMAT_NAMES[fmt]}->{kl.FORMAT_NAMES[fout]} [{loader}]: {msg}")
    return fails


# ---- tests -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev(cuda):
    T0.setdefault("t", time.monotonic())
    return cuda


def test_easu_and_rcas_across_scales(dev):
    fails = run_easu(ratio_shapes() + boundary_shapes("easu"), dev)
    fails += [f"easu {n}: refused with one loader only" for n in _loader_mismatches("easu")]
    assert not fails, f"{len(fails)} failures:\n" + "\n".join(fails[:40])


def test_fused_across_scales(dev):
    fails = run_fused(ratio_shapes() + boundary_shapes("fused"), dev)
    fails += [f"fused {n}: refused with one loader only" for n in _loader_mismatches("fused")]
    assert not fails, f"{len(fails)} failures:\n" + "\n".join(fails[:40])


def test_nis_scaler_across_scales(dev):
    """the ratio shapes, and kScale on each side of the range NVScalerUpdateConfig accepts: 1 (in = out) and 0.5
    (in = out / 2), each with one source texel more and one less.  kScale comes from the image extents here, never set
    by hand: the chroma tap positions itself from kDstNorm and the source extent, the tile from kScale, so the two agree
    only when the constants describe the images (as the library's config does)"""
    edge = []
    for i, (name, iw) in enumerate((("1", LONG), ("0.5", LONG // 2))):
        for d in (-1, 0, 1):
            other = RATIOS[(3 * i + d + 8) % len(RATIOS)]
            edge.append(Shape(f"kScaleX~{name}{d:+d} wide", LONG, SHORT, iw + d, _insize(SHORT, other)))
            edge.append(Shape(f"kScaleY~{name}{d:+d} tall", SHORT, LONG, _insize(SHORT, other), iw + d))
    fails = run_nis(ratio_shapes() + edge, dev)
    fails += [f"nis {n}: refused with one loader only" for n in _loader_mismatches("nis")]
    assert not fails, f"{len(fails)} failures:\n" + "\n".join(fails[:40])


def test_cas_upscale_across_scales(dev):
    fails = run_cas(ratio_shapes(), dev)
    assert not fails, f"{len(fails)} failures:\n" + "\n".join(fails[:40])


# ---- the context path at render scales no other test uses ------------------------------------------------------
CTX_SCALES = [0.2, 0.3, 0.45, 0.49, 0.5, 0.51, 0.93, 0.97, 0.99, 0.999, 2.0, 3.0]
CTX_W, CTX_H = 97, 61
PROJ, RADIUS = (0.42, 0.47, 0.58, 0.53), 0.4


def _ctx_expected(path, src, eye, one_eye, ow, oh):
    """the oracle of the context's state for one eye (strict math, debug off)"""
    from oracle import pyoracle as po
    from tests import srtm_oracle as so
    if path == "nis":
        cfg, ok = po.nis_config(False, eye, one_eye, CTX_W, CTX_H, ow, oh, proj=PROJ, radius=RADIUS, sharpness=SHARP)
        if not ok:
            # NVScalerUpdateConfig leaves every tuning word zero outside kScale [0.5, 1] (kEps = 0 included), and the
            # context dispatches that config as the reference does: the oracle runs the same words
            assert not any(bytes(cfg)[:48]), "tuning words of a refused NVScalerUpdateConfig"
        return po.nis_scaler(src, ow, oh, cfg, nthreads=NTHREADS), ok
    uc = po.upscale_constants(eye, one_eye, CTX_W, CTX_H, ow, oh, proj=PROJ, radius=RADIUS)
    sc = po.sharpen_constants(eye, one_eye, ow, oh, proj=PROJ, radius=RADIUS, sharpness=SHARP)
    if path == "srtm":
        mid = so.easu(src, ow, oh, uc, out_dtype=np.float16, srtm_in=True, nthreads=NTHREADS)
        return so.rcas(mid, sc, out_dtype=np.uint8, srtm_out=True, nthreads=NTHREADS), True
    return po.rcas(po.easu(src, ow, oh, uc, nthreads=NTHREADS), sc, nthreads=NTHREADS), True


@pytest.mark.parametrize("shared", [False, True], ids=["one_eye", "shared"])
@pytest.mark.parametrize("path", ["fsr", "fused", "nis", "srtm"])
def test_context_at_render_scales_no_other_test_uses(dev, path, shared):
    """PostProcessor at render scales below 0.5 (set_config accepts any scale > 0), just below 1, and above 1 (the output
    is the input times the scale there): every eye equals the oracle of that state.  NIS below a render scale of 0.5
    (and at 3.0) runs the all-zero tuning config; NIS above 1 is NVScaler at kScale = 1 / scale.  The fused kernel runs
    exactly where the host rule has a layout for the tile (one launch per eye), and the two dispatches elsewhere."""
    import torch
    import openvr_fsr_b200 as ovr
    fmt = kl.RGBA16F if path == "srtm" else kl.RGBA8
    fails, zero_tuning, fused_where = [], [], []
    for scale in CTX_SCALES:
        ow, oh = ovr.output_size(CTX_W, CTX_H, scale)
        pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, useNis=path == "nis", renderScale=scale, sharpness=SHARP,
                                          radius=RADIUS, projCentre=PROJ, fusedFsr=path == "fused", srtm=path == "srtm",
                                          mathMode=ovr.MATH_STRICT))
        try:
            for eye in ((0,) if shared else (0, 1)):
                src = _content(fmt, CTX_W, CTX_H, 500 + eye + int(1000 * scale))
                bounds = ovr.TextureBounds(0.0, 0.0, 0.5, 1.0) if shared else None
                img = ovr.to_image(src, dev)
                n0 = ovr.kernel_launches()
                got = pp.apply(eye, img, bounds=bounds).cpu().numpy()
                torch.cuda.synchronize()
                launches = ovr.kernel_launches() - n0
                want, ok = _ctx_expected(path, src, eye, not shared, ow, oh)
                if not ok:
                    zero_tuning.append(scale)
                msg, _ = _check(got, want, kl.RGBA8, "strict", False)
                if msg:
                    fails.append(f"{path} scale {scale} eye {eye}{' shared' if shared else ''}: {msg}")
                if path == "fused":
                    c0 = pp.upscale_constants(eye)[:2].view(F)
                    expect = fp.fused_layout(c0[0], c0[1], True) is not None
                    if launches != (1 if expect else 2):
                        fails.append(f"fused scale {scale} eye {eye}: {launches} launches, host rule expects "
                                     f"{'the fused kernel' if expect else 'the two dispatches'}")
                    fused_where.append((scale, launches == 1))
        finally:
            pp.close()
    if path == "nis":
        assert sorted(set(zero_tuning)) == [0.2, 0.3, 0.45, 0.49, 3.0], zero_tuning
    if path == "fused":
        print("\nfused kernel per render scale:", sorted(set(fused_where)))
        assert any(f for _, f in fused_where) and not all(f for _, f in fused_where), "both outcomes are exercised"
    assert not fails, "\n".join(fails)


def test_sweep_statistics(dev):
    """prints how many cases each kernel and loader matched and how many it refused (run after the sweeps above)"""
    print("\ncases matched / refused per kernel and loader (each case: strict and fast math):")
    for (kernel, loader), (ok, refused) in sorted(STATS.items()):
        print(f"  {kernel:6s} {loader:6s} matched {ok:4d}  refused {refused:4d}")
    print(f"module wall time: {time.monotonic() - T0['t']:.1f} s")
