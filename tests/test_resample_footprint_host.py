"""Every tap of every resampling kernel lies inside the source tile its CTA loads, at every scale the launchers accept.

The kernels read their shared source tiles without bound checks (EASU's 12-tap window, NVScaler's 6x6 window), or clamp
an index into the tile (the bilinear copy outside the radius, NVScaler's window origin and chroma tap).  A tile one texel
short gives a wrong colour, not a fault, so it is checked here on the CPU, without the kernels: this module restates in
numpy float32 the launchers' tile sizing and refusal rules (csrc/kernels.inc) and each kernel's source positions, every
operation rounded as the device rounds it (mul_add_unfused = a rounded multiply then a rounded add, snap_subtexel's x256
is exact, (float)p / rad is an IEEE divide), and asserts, per axis and for every output pixel:

  * each tap is a texel of the tile its CTA loaded, without any of the tile clamps changing the index (a clamp to the
    image edge is allowed: the tile already holds the image-clamped texels);
  * a launcher refuses exactly the shapes whose tile its kernels cannot hold (72 columns, 40 rows for EASU, the
    113 KB budget of the fused kernel), and which shapes it refuses does not depend on the source loader (TMA box or
    plain loads);
  * NVScaler accepts every kScale in (0, 1] (its fixed 40 x 31 tile holds all of them) and nothing else -- the range
    NVScalerUpdateConfig accepts; the legacy CAS upscale's fixed 72 x 36 tile holds every out->in step <= 1.

The constants come from the library's own host functions (ovrfsr_make_upscale_constants, ovrfsr_make_nis_config,
ovrfsr_cas_setup).  Sweeps: every output extent 1-1024 at a dense set of ratios; extents up to 16384 at ratios on each
decision boundary of a launcher (one ulp of c0 each side); ratios where (N-1)*c0 is within a few ulps of an integer.
Positions far from the origin round differently, which is where a one-texel slop matters.

test_gpu_scale_sweep.py runs the same boundaries on the device and checks that the dispatches refuse exactly what
`easu_layout` / `fused_layout` / `nis_accepts` refuse here."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

F = np.float32
ROOT = Path(__file__).resolve().parents[1]

# ---- kernel geometry (fsr_kernels.cuh, fsr_fused.cuh, nis_kernels.cuh, cas_kernels.cuh) ---------------------------
TILE_W, TILE_H = 64, 32                 # EASU / fused / CAS output tile of one CTA
FUSED_EW, FUSED_EH = TILE_W + 2, TILE_H + 2
EASU_MAX_COLS, EASU_MAX_ROWS = 72, 8 * 5  # widest compiled row stride; 8 warps x kEasuRowsPerThread decode rows
EASU_MAX_SMEM, FUSED_MAX_SMEM = 120 * 1024, 113 * 1024
FUSED_MS = 67
NIS_BW, NIS_BH, NIS_TILE_W, NIS_TILE_H = 32, 24, 40, 31
CAS_TW, CAS_TH = 72, 36


# ---- device arithmetic ---------------------------------------------------------------------------------------------
def mul_add_unfused(a, b, c):
    """__fadd_rn(__fmul_rn(a, b), c) on float32 arrays"""
    return (F(a) * F(b)).astype(F) + F(c)


def snap_subtexel(s):
    """floorf(fmaf(s, 256, 0.5)) / 256: s*256 is exact, so the fma is one rounded add"""
    return np.floor(s * F(256) + F(0.5)) * F(1.0 / 256.0)


def ifloor(x):
    return np.floor(x).astype(np.int64)


def clampi(v, lo, hi):
    return np.minimum(np.maximum(v, lo), hi)


def easu_pos(p, scale, offs):
    return mul_add_unfused(np.asarray(p).astype(F), scale, offs)


def nis_pos(p, scale):
    """mul_add_unfused(0.5f + (float)p, kScale, -0.5f)"""
    return mul_add_unfused(F(0.5) + np.asarray(p).astype(F), scale, F(-0.5))


def ceil_tile(n, c0):
    """(int)ceilf(n * c0) with n an int constant of the launcher (c0 a float32 scalar or array)"""
    return np.ceil(F(n) * np.asarray(c0, dtype=F)).astype(np.int64)


# ---- the launchers' tile sizing and refusal rules (csrc/kernels.inc) ------------------------------------------------
def easu_tile(c0x, c0y):
    """launch_easu: source extent of one 64 x 32 output tile"""
    tw = (ceil_tile(TILE_W - 1, c0x) + 5 + 3) & ~3
    th = ceil_tile(TILE_H - 1, c0y) + 5
    return tw, th


def fused_tile(c0x, c0y):
    """launch_fsr_fused: source extent of the 66 x 34 first-pass region"""
    tw = (ceil_tile(FUSED_EW - 1, c0x) + 5 + 3) & ~3
    th = ceil_tile(FUSED_EH - 1, c0y) + 5
    return tw, th


def _stride(cols):
    return 60 if cols <= 60 else 72


def easu_layout(c0x, c0y, tma_able):
    """(TMA, row stride) the EASU launcher runs, or None when it refuses.  tma_able: a 4-byte source whose base and pitch
    are 16-byte aligned.  The TMA variant keeps 4 alignment columns; where they do not fit, plain loads run instead."""
    tw, th = easu_tile(c0x, c0y)
    for tma in ((True, False) if tma_able else (False,)):
        cols = tw + 4 if tma else tw
        stride = _stride(cols)
        if cols <= EASU_MAX_COLS and th <= EASU_MAX_ROWS and stride * th * 32 <= EASU_MAX_SMEM:
            return tma, stride
    return None


def fused_smem(tw, th, tma):
    stride = _stride(tw + 4 if tma else tw)
    tiles = (stride * th * (16 * 2 + 4) + 127) & ~127
    mid = (FUSED_MS * FUSED_EH * 16 + 127) & ~127
    return tiles + mid + ((tw + 4) * th * 4 if tma else 0)


def fused_layout(c0x, c0y, tma_able):
    """(TMA, row stride) the fused launcher runs, or None when it refuses (the context then runs the two dispatches)"""
    tw, th = fused_tile(c0x, c0y)
    for tma in ((True, False) if tma_able else (False,)):
        cols = tw + 4 if tma else tw
        if cols <= EASU_MAX_COLS and th <= EASU_MAX_ROWS and fused_smem(tw, th, tma) <= FUSED_MAX_SMEM:
            return tma, _stride(cols)
    return None


def nis_accepts(k_scale_x, k_scale_y):
    """fill_nis_args: NVScaler's fixed tile is sized for the range NVScalerUpdateConfig accepts"""
    return bool(0 < k_scale_x <= 1 and 0 < k_scale_y <= 1)


# ---- constants from the library's host functions ------------------------------------------------------------------
def _lib():
    from openvr_fsr_b200 import _lib as L
    return L


_CFG = {}


def _cfg():
    if "c" not in _CFG:
        import openvr_fsr_b200 as ovr
        _CFG["c"] = ovr.Config(fsrEnabled=True, renderScale=0.75, sharpness=0.8, radius=0.5).to_c()
    return _CFG["c"]


def easu_consts(in_w, in_h, out_w, out_h):
    """FsrEasuCon words as the library builds them: (c0x, c0y, c0z, c0w, radW, radH) as float32"""
    w = (C.c_uint32 * 24)()
    _lib().lib().ovrfsr_make_upscale_constants(w, C.byref(_cfg()), 0, 1, in_w, in_h, out_w, out_h)
    c0 = np.array(w[0:4], dtype=np.uint32).view(F)
    return c0[0], c0[1], c0[2], c0[3], F(w[22]), F(w[23])


def nis_consts(in_w, in_h, out_w, out_h):
    """NVScalerUpdateConfig as the library builds it: (kScaleX, kScaleY, kDstNormX, kDstNormY, ok)"""
    buf = C.create_string_buffer(256)
    ok = _lib().lib().ovrfsr_make_nis_config(C.cast(buf, C.c_void_p), C.byref(_cfg()), 0, 0, 1, in_w, in_h, out_w, out_h)
    f = np.frombuffer(buf.raw, dtype=F)
    return f[12], f[13], f[14], f[15], bool(ok)


def cas_consts(in_w, in_h, out_w, out_h):
    w = (C.c_uint32 * 8)()
    _lib().lib().ovrfsr_cas_setup(w, 0.8, 1.0, in_w, in_h, out_w, out_h)
    c0 = np.array(w[0:4], dtype=np.uint32).view(F)
    return c0[0], c0[1], c0[2], c0[3]


# ---- per-axis footprint checks, vectorised over the pixels of many cases ----------------------------------------
class Axis:
    """a batch of 1-D cases: output extent n, source extent src, out->in step c0 and offset cz (EASU / CAS), the
    Bilinear() divisor rad, NVScaler's kScale and kDstNorm.  One row of every array per case."""

    def __init__(self, n, src, c0=None, cz=None, rad=None, kscale=None, dnorm=None):
        self.n = np.asarray(n, dtype=np.int64)
        self.src = np.asarray(src, dtype=np.int64)
        self.c0, self.cz, self.rad = (None if v is None else np.asarray(v, dtype=F) for v in (c0, cz, rad))
        self.kscale, self.dnorm = (None if v is None else np.asarray(v, dtype=F) for v in (kscale, dnorm))

    def pixels(self, step):
        """(case index, pixel coordinate) of the first and last pixel of every `step`-aligned run of output pixels of
        every case.  Each source position here is monotone non-decreasing in the pixel coordinate (a rounded multiply
        by a positive step then a rounded add, an IEEE divide by a positive extent, the 1/256 snap and floor all are),
        so within a tile, a 16-pixel group or an NVScaler block -- all unions of such runs -- every tap's offset from
        the tile origin is extreme at a run's end: checking the run ends is checking every pixel."""
        runs = (self.n + step - 1) // step
        idx = np.repeat(np.arange(len(self.n)), runs)
        first = (np.arange(int(runs.sum()), dtype=np.int64) - (np.cumsum(runs) - runs)[idx]) * step
        last = np.minimum(first + step - 1, self.n[idx] - 1)
        return np.concatenate([idx, idx]), np.concatenate([first, last])


def _report(bad, ax, idx, p, what):
    """assertion text naming the first few failing cases"""
    cases = np.unique(idx[bad])
    lines = []
    for c in cases[:6]:
        first = p[bad & (idx == c)][0]
        lines.append(f"  n={ax.n[c]} src={ax.src[c]} c0={ax.c0[c] if ax.c0 is not None else ax.kscale[c]!r} first pixel {first}")
    return f"{what}: {len(cases)} case(s), {int(bad.sum())} pixel(s)\n" + "\n".join(lines)


def _holds(tile_col, tile_x0, extent_img, want_img):
    """the tile column `tile_col` (its texel is image column clamp(x0 + col)) holds image column clamp(want)"""
    return clampi(tile_x0 + tile_col, 0, extent_img - 1) == clampi(want_img, 0, extent_img - 1)


def _bilinear_taps(p, rad, src):
    """easu_bilinear_axis / NVScaler's DirectCopy position: floor of the snapped sample position"""
    u = p.astype(F) / rad
    return ifloor(snap_subtexel(mul_add_unfused(u, src.astype(F), F(-0.5))))


def check_easu_axis(ax, tile, sizes, tma, fused=False):
    """EASU (or the fused kernel's first pass) along one axis.  tile: output tile extent (64 in x, 32 in y); sizes[i]:
    the launcher's tile extent of case i (tw or th); tma: the TMA variant's 4-aligned origin (x only).  Returns a list
    of failure descriptions."""
    idx_all, p_all = ax.pixels(16)
    fails = []
    # a pixel belongs to its own tile and, in the fused kernel, to the ring of the neighbour whose region reaches it
    owners = [(np.ones_like(p_all, dtype=bool), 0)]
    if fused:
        owners += [((p_all % tile == tile - 1) & (p_all + 1 < ax.n[idx_all]), 1), ((p_all % tile == 0) & (p_all > 0), -1)]
    for sel, shift in owners:
        idx, p = idx_all[sel], p_all[sel]
        c0, cz, size, src = ax.c0[idx], ax.cz[idx], sizes[idx], ax.src[idx]
        o0 = ((p + shift) // tile) * tile
        s0 = ifloor(easu_pos(o0 - 1 if fused else o0, c0, cz)) - 1
        x0 = (s0 & ~3) if tma else s0
        cols = size + 4 if tma else size
        f = ifloor(easu_pos(p, c0, cz)) - x0
        # the 12 taps at -1..+2 and the features at 0..+1 (computed for tile columns 1..cols-2)
        bad = (f - 1 < 0) | (f + 2 > cols - 1)
        if bad.any():
            fails.append(_report(bad, ax, idx, p, f"{'fused' if fused else 'EASU'} filter window outside the tile"))
        if not fused:
            # one-colour group footprint (easu_flat_group): f of the group's first pixel .. f + 1 of its last
            g0 = (p // 16) * 16
            g1 = np.minimum(g0 + 15, ax.n[idx] - 1)
            a = ifloor(easu_pos(g0, c0, cz)) - x0
            b = ifloor(easu_pos(g1, c0, cz)) + 1 - x0
            bad = (a < 0) | (b > cols - 1)
            if bad.any():
                fails.append(_report(bad, ax, idx, p, "EASU one-colour group footprint outside the tile"))
        # Bilinear() outside the radius: clamps into the tile; the clamp must only ever stand for the image edge
        b0 = _bilinear_taps(p, ax.rad[idx], src)
        for tap in (b0, b0 + 1):
            bad = ~_holds(clampi(tap - x0, 0, cols - 1), x0, src, tap)
            if bad.any():
                fails.append(_report(bad, ax, idx, p, "bilinear tap changed by the tile clamp"))
    return fails


def check_nis_axis(ax, block, tile_max):
    """NVScaler along one axis: block = 32 (x) / 24 (y) output pixels, tile_max = kNisTileW / kNisTileH"""
    idx, p = ax.pixels(block)
    ks, dn, src = ax.kscale[idx], ax.dnorm[idx], ax.src[idx]
    b0 = (p // block) * block
    t0 = ifloor(nis_pos(b0, ks)) - 2
    ext = np.minimum(tile_max, ifloor(nis_pos(b0 + block - 1, ks)) - 2 - t0 + 7)  # tw / th of the block
    fails = []
    w = ifloor(nis_pos(p, ks)) - 2 - t0  # window origin px / pyOff before its clamp to [0, tile_max - 6]
    bad = (w < 0) | (w + 5 > ext - 1) | (w > tile_max - 6)
    if bad.any():
        fails.append(_report(bad, ax, idx, p, "NVScaler 6x6 window outside the loaded tile"))
    # the interpolated edge map reads window positions 2..3, computed for tile positions in [2, ext - 2)
    bad = (w + 2 < 2) | (w + 3 >= ext - 2)
    if bad.any():
        fails.append(_report(bad, ax, idx, p, "NVScaler edge-map read outside the computed band"))
    # the chroma tap: SampleLevel at (dst + 0.5) * kDstNorm, clamped into the loaded tile
    t = (p.astype(F) + F(0.5)) * dn
    c = ifloor(snap_subtexel(mul_add_unfused(t, src.astype(F), F(-0.5))))
    for tap in (c, c + 1):
        col = clampi(tap - t0, 0, ext - 1)
        bad = ~_holds(col, t0, src, tap)
        if bad.any():
            fails.append(_report(bad, ax, idx, p, "NVScaler chroma tap changed by the tile clamp"))
    return fails


def check_cas_axis(ax, tile, fixed):
    """CAS upscale along one axis: the fixed 72 x 36 tile from one texel before f of the tile's first pixel"""
    idx, p = ax.pixels(16)
    c0, cz = ax.c0[idx], ax.cz[idx]
    s0 = ifloor(easu_pos((p // tile) * tile, c0, cz)) - 1
    f = ifloor(easu_pos(p, c0, cz)) - s0
    bad = (f - 1 < 0) | (f + 2 > fixed - 1)
    return [_report(bad, ax, idx, p, "CAS window outside the tile")] if bad.any() else []


# ---- case generation -----------------------------------------------------------------------------------------------
DENSE_C0 = sorted({round(v, 4) for v in np.concatenate([
    1.0 / np.array([1.002, 1.01, 1.02, 1.04, 1.07, 1.15, 1.3, 1.5, 1.9, 2.5, 3.0, 4.0, 8.0]),
    [1.0, 1.01, 1.03, 1.05, 1.06, 1.0635, 1.09, 1.12, 1.15], np.linspace(0.2, 0.9, 6)])})


def _ulps(v, k):
    """v and the k float32 neighbours on each side"""
    out = [F(v)]
    lo = hi = F(v)
    for _ in range(k):
        lo, hi = np.nextafter(lo, F(-1)), np.nextafter(hi, F(2))
        out += [lo, hi]
    return out


def largest_c0(n, k):
    """the largest float32 c0 with ceil(n * c0) <= k: where a tile extent ceil(n * c0) + ... steps"""
    v = F(k / n)
    while int(np.ceil(F(n) * v)) > k:
        v = np.nextafter(v, F(0))
    while int(np.ceil(F(n) * np.nextafter(v, F(2)))) <= k:
        v = np.nextafter(v, F(2))
    return v


def boundary_c0(kernel=None):
    """(x values, y values) of c0 on each decision boundary of a launcher, +- 1 ulp.  EASU: the tile crosses 56 / 60 /
    64 / 68 / 72 columns (the 60- and 72-column strides with and without the TMA variant's 4 alignment columns, the
    refusal) and 40 rows.  Fused: the same columns, and every tile height at which a (stride, loader) layout leaves the
    113 KB budget.  kernel=None: both, and kScale 0.5 and 1 (NVScaler)."""
    xs, ys = set(), set()
    for kern, n_x, n_y in (("easu", TILE_W - 1, TILE_H - 1), ("fused", FUSED_EW - 1, FUSED_EH - 1)):
        if kernel not in (None, kern):
            continue
        for k in (51, 55, 59, 63, 67):
            xs |= set(_ulps(largest_c0(n_x, k), 1))
        if kern == "easu":
            ys |= set(_ulps(largest_c0(n_y, EASU_MAX_ROWS - 5), 1))
        else:
            for tw in (56, 60, 64, 68, 72):
                for tma in (False, True):
                    fit = [th for th in range(6, EASU_MAX_ROWS + 1) if fused_smem(tw, th, tma) <= FUSED_MAX_SMEM]
                    ys |= set(_ulps(largest_c0(n_y, max(fit) - 5), 1))
            ys |= set(_ulps(largest_c0(n_y, EASU_MAX_ROWS - 5), 1))
    if kernel is None:
        xs |= set(_ulps(F(1.0), 1)) | set(_ulps(F(0.5), 1))
    return sorted(xs), sorted(ys)


def _pairs_dense():
    """(in, out) pairs: every out extent 1-1024 at each DENSE_C0 step, plus exact ratios p/q whose (N-1)*c0 lands on or
    next to an integer"""
    pairs = set()
    for c0 in DENSE_C0:
        for n in range(1, 1025):
            pairs.add((max(1, int(round(n * c0))), n))
    for q in (7, 31, 33, 63, 65):
        for pnum in range(max(1, q // 4), q + 5):
            for m in range(1, 1024 // q + 1):
                pairs.add((pnum * m, q * m))
                pairs.add((pnum * m + 1, q * m + 1))
    return sorted(pairs)


LARGE = (2047, 4096, 8193, 12000, 16384)


def _pairs_boundary():
    """(in, out) pairs of large extents whose out->in step sits on a launcher boundary: in / out = k / n, and one
    extent either side"""
    pairs = set()
    for n, ks in ((TILE_W - 1, range(44, 70)), (FUSED_EW - 1, range(44, 70)), (TILE_H - 1, range(20, 37)),
                  (FUSED_EH - 1, range(15, 37))):
        for k in ks:
            for m in (16384 // n, 8192 // n, 193):
                for d in (-1, 0, 1):
                    pairs.add((k * m, n * m + d))
    for out in LARGE:
        pairs.add((out, out))
        pairs.add((out // 2, out))
    for out in range(8000, 16385, 251):  # in / out within about 1e-4 of 1, far from the origin
        pairs.add((out - 1, out))
    return sorted(p for p in pairs if p[0] >= 1 and 1 <= p[1] <= 16384)


def _easu_axis(pairs):
    c = [easu_consts(i, i, o, o) for i, o in pairs]
    return Axis([o for _, o in pairs], [i for i, _ in pairs], [v[0] for v in c], [v[2] for v in c], [v[4] for v in c])


def consistent_extents(c0, limit=16384):
    """(out, in) extents whose ratio in / out is c0 to within a few ulps: c0 near k / q for one of the launchers'
    denominators q, and out a multiple of q.  The bilinear copy positions itself from the image extents, the tile from
    c0, so (as in the library's constants) the two must agree"""
    for q in (63, 31, 65, 33, 1, 2):
        k = int(round(float(c0) * q))
        if k and abs(float(c0) * q - k) < 1e-4:
            ms = sorted({1, 2, 3, limit // (2 * q), limit // q - 1, limit // q})
            return [(q * m, k * m) for m in ms if 1 <= q * m <= limit]
    raise AssertionError(f"{c0!r} is not near a ratio of small integers")


def _synthetic_axis(c0s):
    """cases built from c0 directly (the stateless dispatches take any constant words): one ulp around a boundary"""
    rows = [(n, src, F(c0), F(F(0.5) * F(c0) - F(0.5))) for c0 in c0s for n, src in consistent_extents(c0)]
    return Axis([r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], [r[3] for r in rows],
                [F(r[0]) for r in rows])


def _check_easu_family(ax, fused):
    """every accepted case, with each loader the launcher may run for it"""
    fails = []
    tile_fn = fused_tile if fused else easu_tile
    for axis_name, tile in (("x", TILE_W), ("y", TILE_H)):
        sizes = tile_fn(ax.c0, ax.c0)[0 if axis_name == "x" else 1]
        for tma in ((False, True) if axis_name == "x" else (False,)):
            ok = sizes + (4 if tma else 0) <= EASU_MAX_COLS if axis_name == "x" else sizes <= EASU_MAX_ROWS
            sub = Axis(ax.n[ok], ax.src[ok], ax.c0[ok], ax.cz[ok], ax.rad[ok])
            if len(sub.n):
                fails += [f"[{axis_name}, {'TMA' if tma else 'plain'}] {m}"
                          for m in check_easu_axis(sub, tile, sizes[ok], tma, fused)]
    return fails


# ---- tests ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib(built_lib):
    return built_lib


@pytest.mark.parametrize("fused", [False, True], ids=["easu", "fused"])
def test_easu_taps_inside_tile_dense(lib, fused):
    fails = _check_easu_family(_easu_axis(_pairs_dense()), fused)
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("fused", [False, True], ids=["easu", "fused"])
def test_easu_taps_inside_tile_at_boundaries(lib, fused):
    ax = _easu_axis(_pairs_boundary())
    xs, ys = boundary_c0()
    syn = _synthetic_axis(sorted(set(xs) | set(ys)))
    fails = _check_easu_family(ax, fused) + _check_easu_family(syn, fused)
    assert not fails, "\n".join(fails)


def _nis_axis(pairs):
    rows = []
    for i, o in pairs:
        ks, _, dn, _, _ = nis_consts(i, i, o, o)
        if nis_accepts(ks, ks):
            rows.append((o, i, ks, dn))
    return Axis([r[0] for r in rows], [r[1] for r in rows], kscale=[r[2] for r in rows], dnorm=[r[3] for r in rows])


def test_nis_taps_inside_tile(lib):
    pairs = [p for p in _pairs_dense() + _pairs_boundary() if p[0] <= p[1]]
    ax = _nis_axis(pairs)
    # kScale values straight from the boundary, one ulp each side, at large extents (kDstNorm = 1 / out)
    rows = [(n, max(1, int(round(n * float(k)))), k, F(F(1) / F(n))) for k in _ulps(F(1.0), 2) + _ulps(F(0.5), 2) + [F(0.1)]
            for n in LARGE if 0 < k <= 1]
    syn = Axis([r[0] for r in rows], [r[1] for r in rows], kscale=[r[2] for r in rows], dnorm=[r[3] for r in rows])
    fails = []
    for a in (ax, syn):
        fails += [f"[x] {m}" for m in check_nis_axis(a, NIS_BW, NIS_TILE_W)]
        fails += [f"[y] {m}" for m in check_nis_axis(a, NIS_BH, NIS_TILE_H)]
    assert not fails, "\n".join(fails)


def test_cas_upscale_taps_inside_tile(lib):
    pairs = [p for p in _pairs_dense() + _pairs_boundary() if p[0] <= p[1]]  # the CAS upscale refuses a shrink
    c = [cas_consts(i, i, o, o) for i, o in pairs]
    ax = Axis([o for _, o in pairs], [i for i, _ in pairs], [v[0] for v in c], [v[2] for v in c])
    fails = check_cas_axis(ax, TILE_W, CAS_TW) + check_cas_axis(ax, TILE_H, CAS_TH)
    assert not fails, "\n".join(fails)


def test_refusal_is_capacity_and_not_the_loader(lib):
    """each launcher refuses exactly where no compiled layout holds the tile, with either loader"""
    c0s = sorted(set(boundary_c0()[0]) | set(boundary_c0()[1]) | {F(v) for v in DENSE_C0})
    for c0x in c0s:
        for c0y in c0s:
            tw, th = easu_tile(c0x, c0y)
            holds = tw <= EASU_MAX_COLS and th <= EASU_MAX_ROWS
            for tma_able in (False, True):
                lay = easu_layout(c0x, c0y, tma_able)
                assert (lay is not None) == holds, (c0x, c0y, tma_able, tw, th)
                if lay:
                    cols = tw + 4 if lay[0] else tw
                    assert cols <= lay[1] and lay[1] * th * 32 <= EASU_MAX_SMEM
            fw, fh = fused_tile(c0x, c0y)
            holds = fw <= EASU_MAX_COLS and fh <= EASU_MAX_ROWS and fused_smem(fw, fh, False) <= FUSED_MAX_SMEM
            for tma_able in (False, True):
                assert (fused_layout(c0x, c0y, tma_able) is not None) == holds, (c0x, c0y, tma_able, fw, fh)
    # the thresholds themselves: EASU takes every out->in step up to 67/63 in x and 35/31 in y, and nothing beyond
    x_max = max(c for c in c0s if easu_layout(c, F(1), True))
    y_max = max(c for c in c0s if easu_layout(F(1), c, True))
    assert int(np.ceil(F(63) * x_max)) == 67 and int(np.ceil(F(63) * np.nextafter(x_max, F(2)))) == 68
    assert int(np.ceil(F(31) * y_max)) == 35 and int(np.ceil(F(31) * np.nextafter(y_max, F(2)))) == 36
    # NVScaler: the library's own config for a shrink carries kScale > 1, which the dispatch refuses
    ks, _, _, _, ok = nis_consts(101, 100, 100, 100)
    assert ks > 1 and not ok and not nis_accepts(ks, F(1))
    ks, _, _, _, ok = nis_consts(100, 100, 100, 100)
    assert ks == 1 and ok and nis_accepts(ks, ks)
    ks, _, _, _, ok = nis_consts(20, 20, 100, 100)  # render scale 0.2: zero tuning words, still dispatched
    assert not ok and nis_accepts(ks, ks)


def test_launcher_source_states_these_rules():
    """the formulas restated above are the ones in csrc/kernels.inc and the kernels' headers: a change there must come
    with the same change here (and a run of this sweep)"""
    src = (ROOT / "openvr_fsr_b200/csrc/kernels.inc").read_text()
    nis = (ROOT / "openvr_fsr_b200/csrc/nis_kernels.cuh").read_text()
    fsr = (ROOT / "openvr_fsr_b200/csrc/fsr_kernels.cuh").read_text()
    cas = (ROOT / "openvr_fsr_b200/csrc/cas_kernels.cuh").read_text()
    squash = lambda s: re.sub(r"\s+", " ", s)  # noqa: E731
    src, nis, fsr, cas = map(squash, (src, nis, fsr, cas))
    for needle in ("const int tw = ((int)ceilf((kTileW - 1) * a.c0x) + 5 + 3) & ~3;",
                   "const int th = (int)ceilf((kTileH - 1) * a.c0y) + 5;",
                   "a.tileW = ((int)ceilf((kFusedEW - 1) * a.c0x) + 5 + 3) & ~3;",
                   "a.tileH = (int)ceilf((kFusedEH - 1) * a.c0y) + 5;",
                   "const int stride = cols <= 60 ? 60 : 72;",
                   "constexpr int kEasuMaxSmem = 120 * 1024;",
                   "constexpr int kFusedMaxSmem = 113 * 1024;",
                   "return c.kScaleX > 0.f && c.kScaleX <= 1.f && c.kScaleY > 0.f && c.kScaleY <= 1.f;"):
        assert needle in src, needle
    for needle in ("const int tw = min(W, (int)floorf(srcX1) - 2 - tx0 + 7), th = min(kNisTileH, (int)floorf(srcY1) - 2 - ty0 + 7);",
                   "constexpr int kNisTileW = 40, kNisTileH = 31;", "constexpr int kNisBW = 32;",
                   "constexpr int kNisScalerBH = 24;"):
        assert needle in nis, needle
    for needle in ("constexpr int kTileW = 64;", "constexpr int kTileH = 32;", "constexpr int kEasuRowsPerThread = 5;",
                   "return mul_add_unfused((float)p, scale, offs);"):
        assert needle in fsr, needle
    assert "constexpr int kCasTW = 72, kCasTH = 36;" in cas
