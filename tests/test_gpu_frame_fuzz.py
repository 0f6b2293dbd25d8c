"""Seeded random frame sequences through one PostProcessor, every context feature at once, against the oracle.

Each seed drives one context through FRAMES frames.  Before each frame it draws state changes: set_config (render
scale, sharpness, radius, debug tint, projection centre, output format, math mode, fused kernel, SRTM, SRTM_NIS, FINITE,
PERCEPTUAL, NIS, sometimes a pass-through), set_sharpness (0, 1 or between) / clear_sharpness, set_focus / clear_focus
and set_focus_radius / clear_focus_radius per eye (the ends of both ranges included), a new input size (outputs on or
next to multiples of 16 / 32 / 64, tiny inputs, one side above 1000), the layout (one eye per texture, or both side by
side), the source format (RGBA8, BGRA8, BGRX8, RGB10A2, RGBA16F, RGBA32F, RGB32F, 2x / 4x MSAA; a change between a
UNORM and a float format changes the plan without a set_config) and the entry point (apply, apply_pair, apply_into to a
tensor or a CUDA array, apply_pair_into, apply_host; CUDA-array sources; an sRGB-encoded output goes into an RGBA8
destination with or without OVRFSR_FORMAT_SRGB_BIT).  Every frame has new content: natural texture with one-colour
rectangles on and off the 16x16 group grid and across the border, flat in two channels only, flat RGB under varying
alpha, and (float sources) HDR, negative and signed-zero texels and one-colour HDR blocks on the group grid where the
frame's bound covers them.  Strict frames, and fast frames with FINITE, may also carry infinities and NaNs (one channel
or three; FP16 0x7c00 / 0xfc00 / 0x7e00 / 0x7c01, FP32 NaNs with payloads; one-colour +inf and NaN blocks on the group
grid) and FP32 texels beyond 65504; fast frames without FINITE stay finite (DESIGN section 3: no bound exists there).

The context carries state from frame to frame: its outputs, the paired intermediate, the focus block, the intermediate's
format.  So every output a frame returned is filled with a sentinel byte pattern as soon as it has been compared, before
the next frame changes anything (a context's output keeps its storage while nothing resets it), and caller-owned
destinations hold the sentinel when the call runs: a pixel that no kernel writes shows up as the sentinel, a stale
intermediate as last frame's content.

The expected output is the oracle's, a pure function of the frame's effective state: a focus is the projection centre
of its eye, a radius override its radius, a sharpness override (which survives set_config and the layout reset) its
sharpness; a shared texture with unequal radii selects per 16x16 group (NIS: per block) between the oracle's
all-inside and all-outside passes (test_gpu_focus_radius.py); the fused kernel gives the two-pass chain; MSAA sources
the oracle's resolve (oracle/frontend.py).  The plan -- each pass's map bits, the intermediate's format, the pairing,
the fused kernel and the sRGB-encoded output -- is tests/perceptual_oracle.py's ctx_plan, the one statement that
tests/test_plan_host.py pins to make_plan: a float source whose passes have bits goes through that file's passes with
them, a UNORM source through the plain oracle.  apply and apply_pair must return OVRFSR_FORMAT_SRGB_BIT exactly when
the plan encodes sRGB.

Strict math is compared bit for bit (NaN against NaN by class).  Fast math, per pass, the bounds of each feature's own
tests: <= 1 LSB / code into a UNORM target (test_gpu_variant_matrix.py); test_gpu_float_signed.check into a float
target, its footprint term taken on finite_in(source) with FINITE (test_gpu_finite.py); with the tone map and no
PERCEPTUAL, 4 codes into RGBA8 / RGB10A2 and 2e-3 in tone-mapped space into a float target (test_gpu_srtm.py,
test_gpu_nis_srtm.py), also after two passes, as test_gpu_srtm.py measured the context; with PERCEPTUAL,
test_gpu_perceptual._fast_check: 4 codes into RGBA8, 2e-3 (relative above 1) into a float target in the pass's filter
domain (the store maps undone).  Two passes (EASU -> intermediate -> RCAS): <= 4 LSB into a UNORM target, and through
a UNORM intermediate at a sharpness above 0.8 the bound RCAS's amplification of the intermediate's last bit gives
(_paired_lsb: up to 8 LSB at sharpness 1); the share of channels beyond 1 LSB (through a UNORM intermediate: beyond 1
LSB plus that bound's excess over 4, so 5 at sharpness 1) is held below 1e-4 per seed and over the session (a single
small frame has too few channels for that share; with 192 seeds, three fast seeds whose paired frames ran at sharpness
0.93 to 1 had 1.0e-4 to 1.8e-4 of their channels beyond 1 LSB on an H100, the same last-bit differences amplified).  Into a float target the other files have no bound; this file introduces one: 4x the per-pass bound of
test_gpu_float_signed.check (4e-3), the factor between the per-pass and composed UNORM bounds (RCAS amplifies a
last-bit difference of the intermediate: up to 0.00195, 4 FP16 ulps just below 1, measured on an H100), with PERCEPTUAL
in the filter domain.  Into an sRGB-encoded RGBA8 target no bound exists elsewhere; this file proposes 8 codes, the
composed UNORM bound doubled for the sRGB encode's slope (12.92 below 0.0031), and prints the share of channels beyond
2 codes.

A failure names the seed, the frame, the whole effective state and the first wrong pixel, with its 16x16 group's role
(inside the circle, one-colour footprint / window, outside next to an inside group).  RCAS's window rule compares the
texels after the pass's read maps (pq.read_map), as the kernel's one-colour test does.  The last test asserts that the
session reached each coverage category and prints the counters, the fast-math maxima and the wall time; it reads the
counters the sequence tests left in this process (as test_gpu_variant_matrix.py does), so it fails when selected alone
or run in another worker than the sequences.

OVRFSR_FRAME_FUZZ_SEEDS sets the number of strict seeds (default 48; a third as many fast-math seeds run beside them),
OVRFSR_FRAME_FUZZ_FRAMES the frames per seed (default 12)."""
import dataclasses
import os
import time
from collections import Counter, defaultdict

import numpy as np
import pytest

from tests import finite_rule as fin
from tests import perceptual_oracle as pq
from tests import test_gpu_easu_flat as ef
from tests import test_gpu_float_signed as fs
from tests import test_gpu_focus_radius as fr
from tests import test_gpu_perceptual as tp
from tests import test_gpu_rcas_flat as rf
from tests import test_gpu_srtm as ts
from tests import test_gpu_variant_matrix as vm

pytestmark = pytest.mark.gpu

N_STRICT = int(os.environ.get("OVRFSR_FRAME_FUZZ_SEEDS", "48"))
N_FAST = max(1, N_STRICT // 3)
FRAMES = int(os.environ.get("OVRFSR_FRAME_FUZZ_FRAMES", "12"))
NT = os.cpu_count() or 1

RGBA8, BGRA8, RGBA16F, RGBA32F, RGB10A2, BGRX8, RGB32F, AUTO = 0, 1, 2, 3, 4, 5, 6, -1
NAMES = {RGBA8: "RGBA8", BGRA8: "BGRA8", RGBA16F: "RGBA16F", RGBA32F: "RGBA32F", RGB10A2: "RGB10A2", BGRX8: "BGRX8",
         RGB32F: "RGB32F", AUTO: "AUTO"}
FORMATS = [RGBA8, BGRA8, BGRX8, RGB10A2, RGBA16F, RGBA32F, RGB32F]
FLOATS = (RGBA16F, RGBA32F, RGB32F)
MSAA_FORMATS = (RGBA8, RGB10A2, RGBA16F, RGBA32F)
SCALES = [0.5, 0.59, 0.67, 0.75, 0.77, 0.83, 0.91, 1.0, 1.3, 1.5]
RADII = [0.0, 0.2, 0.45, 0.7, 2.0, 4.0]
ENTRIES = ["apply", "apply_pair", "apply_into", "apply_pair_into", "apply_host"]
SHARED = ((0.0, 0.0, 0.5, 1.0), (0.5, 0.0, 1.0, 1.0))  # TextureBounds of the two eyes of a shared texture
MAX_OUT = (640, 420)  # most outputs stay within this, so the CPU oracle stays cheap
SRGB_BIT = 0x100      # OVRFSR_FORMAT_SRGB_BIT
# infinities and NaNs (test_gpu_float_nonfinite.py): +inf, -inf, quiet NaN, signalling NaN / NaNs with payloads
NONFINITE = {RGBA16F: (np.uint16, (0x7c00, 0xfc00, 0x7e00, 0x7c01)),
             RGBA32F: (np.uint32, (0x7f800000, 0xff800000, 0x7fc00000, 0x7f800001, 0xff800001, 0x7fc00001, 0xffc00000,
                                   0x7fa5a5a5))}
NONFINITE[RGB32F] = NONFINITE[RGBA32F]

STATE = {"t0": None, "seeds": 0, "frames": 0, "cov": Counter(), "maxima": defaultdict(float), "beyond": [0, 0],
         "beyond_srgb": [0, 0]}


# ---- state ---------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Frame:
    """the effective state of one frame"""
    cfg: object
    foci: list
    radii: list
    one: bool           # one eye per texture (else both side by side in one texture)
    fmt: int            # API source format
    samples: int        # > 1: MSAA source
    entry: str
    src_array: bool
    dst_array: bool
    size: tuple         # (w, h) of each texture
    tight: bool         # device sources with packed rows (plain loads) rather than pitch-aligned ones (TMA)
    sharp: object = None      # set_sharpness override, None after clear_sharpness
    dst_srgb: bool = False    # caller-owned RGBA8 destinations tagged OVRFSR_FORMAT_SRGB_BIT

    def out_format(self):
        o = self.cfg.outputFormat
        return (RGB10A2 if self.fmt == RGB10A2 else RGBA8) if o == AUTO else o

    def strict(self):
        import openvr_fsr_b200 as ovr
        return self.cfg.mathMode == ovr.MATH_STRICT

    def fsr(self):
        return not self.cfg.useNis

    def upscale(self):
        return self.cfg.renderScale != 1.0

    def plan(self):
        """(easu, rcas, nis bits, intermediate dtype or None, paired, fused tried, sRGB output): pq.ctx_plan"""
        return pq.ctx_plan(self.cfg.to_c().flags, self.cfg.useNis, self.upscale(), self.fmt, self.out_format())

    def bits(self):
        """the map bits of every pass that runs, OR-ed"""
        easu_b, rcas_b, nis_b = self.plan()[:3]
        return nis_b if self.cfg.useNis else (rcas_b | (easu_b if self.upscale() else 0))

    def paired(self):
        return self.plan()[4]

    def fused(self):
        return self.plan()[5] and not (self.src_array or self.dst_array)

    def srgb(self):
        return self.plan()[6]

    def sharpness(self):
        return self.cfg.sharpness if self.sharp is None else self.sharp

    def proj(self):
        p = list(self.cfg.projCentre)
        for e in (0, 1):
            if self.foci[e] is not None:
                p[2 * e:2 * e + 2] = self.foci[e]
        return tuple(p)

    def radius(self, eye):
        return self.cfg.radius if self.radii[eye] is None else self.radii[eye]

    def describe(self):
        c = self.cfg
        easu_b, rcas_b, nis_b, mid, paired, _, srgb = self.plan()
        return (f"entry={self.entry} layout={'one eye per texture' if self.one else 'shared texture'} "
                f"source={NAMES[self.fmt]}{f' x{self.samples} MSAA' if self.samples > 1 else ''}"
                f"{' (CUDA array)' if self.src_array else ''}{' -> CUDA array' if self.dst_array else ''}"
                f"{' (tagged sRGB)' if self.dst_srgb else ''} size={self.size} "
                f"config(fsrEnabled={c.fsrEnabled}, useNis={c.useNis}, renderScale={c.renderScale}, sharpness={c.sharpness:.3f}, "
                f"radius={c.radius}, debugMode={c.debugMode}, projCentre={tuple(round(v, 3) for v in c.projCentre)}, "
                f"outputFormat={NAMES[c.outputFormat]}, mathMode={'strict' if self.strict() else 'fast'}, fusedFsr={c.fusedFsr}, "
                f"srtm={c.srtm}, srtmNis={c.srtmNis}, finite={c.finite}, perceptual={c.perceptual}) "
                f"sharpness override={'none' if self.sharp is None else f'{self.sharp:.3f}'} foci={self.foci} "
                f"radii={self.radii} plan(bits easu={easu_b} rcas={rcas_b} nis={nis_b}, "
                f"intermediate={'output format' if mid is None else np.dtype(mid).name}, paired={paired}, "
                f"fused={self.fused()}, sRGB output={srgb})")


def _draw_config(rng, math, cur=None):
    import openvr_fsr_b200 as ovr
    mm = {"strict": ovr.MATH_STRICT, "fast": ovr.MATH_FAST}.get(math)
    if cur is not None and rng.random() < 0.5:  # one field changes: the transitions between allocations and kernels
        field = str(rng.choice(["srtm", "srtmNis", "finite", "perceptual", "fusedFsr", "outputFormat", "renderScale",
                                "radius", "debugMode", "useNis"] + (["mathMode"] if math == "mixed" else [])))
        new = {"srtm": lambda: not cur.srtm, "srtmNis": lambda: not cur.srtmNis, "finite": lambda: not cur.finite,
               "perceptual": lambda: not cur.perceptual, "fusedFsr": lambda: not cur.fusedFsr,
               "debugMode": lambda: not cur.debugMode,
               "useNis": lambda: not cur.useNis, "outputFormat": lambda: int(rng.choice([AUTO, RGBA16F, RGBA32F])),
               "renderScale": lambda: float(rng.choice(SCALES)), "radius": lambda: float(rng.choice(RADII)),
               "mathMode": lambda: ovr.MATH_FAST if cur.mathMode == ovr.MATH_STRICT else ovr.MATH_STRICT}[field]()
        cfg = dataclasses.replace(cur, fsrEnabled=True, **{field: new})
    else:
        cfg = ovr.Config(fsrEnabled=bool(rng.random() > 0.04), useNis=bool(rng.random() < 0.2),
                         renderScale=float(rng.choice(SCALES)), sharpness=float(rng.uniform(0.0, 1.0)),
                         radius=float(rng.choice(RADII)), debugMode=bool(rng.random() < 0.3),
                         projCentre=tuple(float(v) for v in rng.uniform(0.3, 0.7, 4)),
                         outputFormat=int(rng.choice([AUTO, AUTO, RGBA16F, RGBA32F])),
                         mathMode=mm if mm is not None else int(rng.choice([ovr.MATH_STRICT, ovr.MATH_FAST])),
                         fusedFsr=bool(rng.random() < 0.35), srtm=bool(rng.random() < 0.3),
                         srtmNis=bool(rng.random() < 0.4), finite=bool(rng.random() < 0.45),
                         perceptual=bool(rng.random() < 0.3))
    if cfg.useNis and cfg.renderScale > 1.0:  # NVScaler upscales only
        cfg = dataclasses.replace(cfg, useNis=False)
    return cfg


def _draw_point(rng):
    return tuple(float(rng.choice([0.0, 1.0, rng.uniform(0, 1), rng.uniform(0, 1)])) for _ in range(2))


def _draw_size(rng, scale, one):
    """(w, h) of each texture: mostly so that the output lands on or next to a multiple of 16, 32 or 64"""
    from oracle import pyoracle as po
    r = rng.random()
    if r < 0.1:
        w, h = int(rng.integers(1, 17)), int(rng.integers(1, 17))
        return (w, h) if one else (max(1, w // 2), h)
    if r < 0.16:
        long, short = int(rng.integers(1001, 1400)), int(rng.integers(4, 48))
        w, h = (long, short) if rng.random() < 0.5 else (short, long)
        return (w, h) if one else (max(1, w // 2), h)
    size = []
    for limit in MAX_OUT:
        m = int(rng.choice([16, 32, 64]))
        target = max(1, m * int(rng.integers(1, limit // m + 1)) + int(rng.choice([-1, 0, 0, 1])))
        size.append(target)
    # the input whose output is the target, where one exists (output_size truncates)
    ow, oh = size
    tw = ow if one else ow // 2 * 2
    best = None
    for w in range(max(1, int(tw * scale / (1 if one else 2)) - 2), int(tw * scale / (1 if one else 2)) + 3):
        for h in range(max(1, int(oh * scale) - 2), int(oh * scale) + 3):
            got = po.output_size(w if one else 2 * w, h, scale)
            d = abs(got[0] - tw) + abs(got[1] - oh)
            if best is None or d < best[0]:
                best = (d, w, h)
    return best[1], best[2]


# ---- content -------------------------------------------------------------------------------------------------------
def _content(rng, fmt, w, h, ow, oh, extras, nonfinite=(), beyond=False):
    """(h, w, 4) source ((h, w, 3) for RGB32F) of API format fmt, painted for the output grid of an ow x oh output.
    extras: None, 'signed' (HDR, negative and +-0 texels), 'scrgb' (HDR up to 7.5 and small negatives), 'hdr'
    (HDR >= 0); with extras, also one-colour HDR blocks on the group grid.  nonfinite (float formats): the infinity /
    NaN bit patterns to place, in one channel or three and as one-colour blocks on the group grid.  beyond (FP32
    formats): texels from 6.6e4 to 1e6, negative ones too unless extras is 'hdr', sparse and as one-colour blocks"""
    from openvr_fsr_b200 import synth
    val = synth.natural_f32(w, h, int(rng.integers(1 << 30))).astype(np.float64)
    alpha = np.ones((h, w))
    sx, sy = w / ow, h / oh
    delta = 1.0 / 1023 if fmt == RGB10A2 else 1.0 / 255

    def block(k):
        """source rectangle around a k x k block of output groups: their EASU footprints and their RCAS windows"""
        gx, gy = int(rng.integers(0, (ow + 15) // 16)), int(rng.integers(0, (oh + 15) // 16))
        return (int(np.floor((16 * gx - 3) * sx)) - 2, int(np.ceil((16 * (gx + k) + 2) * sx)) + 2,
                int(np.floor((16 * gy - 3) * sy)) - 2, int(np.ceil((16 * (gy + k) + 2) * sy)) + 2)

    # EASU's source position of an output pixel (easu_pos, con0 of FsrEasuCon); at scale 1 RCAS reads the source itself
    easu = (w, h) != (ow, oh)
    con = [(np.float32(n) / np.float32(o), np.float32(0.5) * (np.float32(n) / np.float32(o)) - np.float32(0.5))
           for n, o in ((w, ow), (h, oh))]

    def fk(p, axis):
        """first source texel of output pixel p's f / g / j / k"""
        return int(np.floor(ef._pos(p, *con[axis]))) if easu else p

    def edge():
        """a one-colour rectangle around a group's RCAS window, one of whose sides lands on the last texel of the
        group's EASU footprint (f .. k) or of the taps behind the window (so that exactly the ring row / column
        differs), or one texel to either side of it: the footprint and window rules tested at their ends"""
        g = (int(rng.integers(0, (ow + 15) // 16)), int(rng.integers(0, (oh + 15) // 16)))
        size = (ow, oh)
        lo = [fk(16 * g[a] - 1, a) - (1 if easu else 0) - 2 for a in (0, 1)]
        hi = [fk(16 * g[a] + 16, a) + (2 if easu else 0) + 2 for a in (0, 1)]
        a, far, d = int(rng.integers(0, 2)), bool(rng.integers(0, 2)), int(rng.integers(-1, 2))
        last = min(16 * g[a] + 15, size[a] - 1)
        if rng.random() < 0.5:  # the footprint's last / first texel
            end = fk(last, a) + (1 if easu else 0) if far else fk(16 * g[a], a)
        else:  # the window: everything but the far / near ring differs... from the ring on
            end = fk(last, a) + (2 if easu else 0) if far else fk(16 * g[a], a) - (1 if easu else 0)
        if far:
            hi[a] = end + d
        else:
            lo[a] = end - d
        return lo[0], hi[0], lo[1], hi[1]

    for _ in range(int(rng.integers(3, 10))):
        kind = str(rng.choice(["block", "block", "block", "edge", "edge", "edge", "off", "border", "two", "alpha",
                               "black"]))
        if kind == "edge":
            x0, x1, y0, y1 = edge()
        elif kind in ("block", "two", "alpha"):
            x0, x1, y0, y1 = block(int(rng.integers(1, 4)))
        elif kind == "off":
            x0, y0 = int(rng.integers(-4, max(1, w))), int(rng.integers(-4, max(1, h)))
            x1, y1 = x0 + int(rng.integers(2, 48)), y0 + int(rng.integers(2, 48))
        else:  # over the border (black: zeros next to RCAS's zero ring)
            x0, x1, y0, y1 = block(int(rng.integers(1, 3)))
            side = int(rng.integers(0, 4))
            x0, x1, y0, y1 = [(-5, x1, y0, y1), (x0, w + 5, y0, y1), (x0, x1, -5, y1), (x0, x1, y0, h + 5)][side]
        xs, ys = slice(max(x0, 0), min(x1, w - 1) + 1), slice(max(y0, 0), min(y1, h - 1) + 1)
        if xs.start >= xs.stop or ys.start >= ys.stop:
            continue
        val[ys, xs] = 0.0 if kind == "black" else rng.uniform(0.02, 0.98, 3)
        if kind == "two":  # flat in two channels only
            hh, ww = ys.stop - ys.start, xs.stop - xs.start
            val[ys, xs, int(rng.integers(0, 3))] += delta * (np.add.outer(np.arange(hh), np.arange(ww)) % 2)
        if kind == "alpha" or (kind == "black" and rng.random() < 0.5):  # one RGB under varying alpha
            alpha[ys, xs] = rng.uniform(0, 1, (ys.stop - ys.start, xs.stop - xs.start))
    if fmt in FLOATS and extras:
        hit = rng.random((h, w)) < 0.015
        hdr = {"signed": [2.0, 7.5, 250.0, 4000.0], "scrgb": [1.5, 3.0, 7.5], "hdr": [2.0, 7.5, 250.0, 1000.0]}[extras]
        val[hit] = rng.choice(hdr, size=(int(hit.sum()), 3))
        if extras in ("signed", "scrgb"):
            hit = rng.random((h, w)) < 0.01
            val[hit] = rng.choice([-0.25, -0.5] + ([-2.0] if extras == "signed" else []), size=(int(hit.sum()), 3))
            x0, y0 = int(rng.integers(0, w)), int(rng.integers(0, h))
            val[y0:y0 + 20, x0:x0 + 20] = -0.0  # by assignment: a -0 block
            x0, y0 = int(rng.integers(0, w)), int(rng.integers(0, h))
            z = val[y0:y0 + 20, x0:x0 + 20]
            val[y0:y0 + 20, x0:x0 + 20] = np.where(rng.random(z.shape) < 0.5, -0.0, 0.0)
    def on_grid():
        """the in-image part of a block around output groups (block), its colour channels"""
        x0, x1, y0, y1 = block(int(rng.integers(1, 3)))
        return slice(max(y0, 0), min(y1, h - 1) + 1), slice(max(x0, 0), min(x1, w - 1) + 1), slice(0, 3)
    grid = []  # one-colour blocks on the group grid, painted last so that no sparse texel breaks them: (where, rgb)
    if fmt in FLOATS and extras:
        grid += [(on_grid(), rng.choice(hdr, 3)) for _ in range(int(rng.integers(0, 3)))]
    if beyond and fmt in (RGBA32F, RGB32F):
        sign = 1.0 if extras == "hdr" else rng.choice([-1.0, 1.0], (h, w, 3))
        big = rng.uniform(6.6e4, 1e6, (h, w, 3)) * sign
        hit = rng.random((h, w)) < 0.01
        val[hit] = big[hit]
        grid += [(on_grid(), rng.uniform(6.6e4, 1e6)) for _ in range(int(rng.integers(1, 3)))]
    out = np.ascontiguousarray(val.astype(np.float32)) if fmt == RGB32F else rf._encode(val, alpha, fmt, rng)
    for where, rgb in grid:
        out[where] = rgb
    if nonfinite and fmt in FLOATS:
        ut = NONFINITE[fmt][0]
        pats = np.array(nonfinite, dtype=ut)
        u = out.view(ut)  # bit patterns: payloads and signalling NaNs survive
        ys, xs = np.nonzero(rng.random((h, w)) < 0.004)
        three = rng.random(len(ys)) < 0.5
        u[ys[~three], xs[~three], rng.integers(0, 3, int((~three).sum()))] = rng.choice(pats, int((~three).sum()))
        u[ys[three], xs[three], :3] = rng.choice(pats, (int(three.sum()), 3))
        for where, rgb in grid:  # the blocks stay one colour
            out[where] = rgb
        blocks = [p for p in pats if p in (0x7c00, 0x7f800000) or np.isnan(np.array(p, ut).view(out.dtype))]
        for _ in range(int(rng.integers(1, 3))):  # one colour: +inf or a NaN
            u[on_grid()] = rng.choice(blocks)
    return out


def _msaa(rng, img, n):
    """(h, w * n, 4) samples: the image's texel in every sample, another texel in a fifth of the samples"""
    raw = np.repeat(img, n, axis=1)
    alt = np.repeat(np.roll(img, (3, 7), axis=(0, 1)), n, axis=1)
    hit = rng.random(raw.shape[:2]) < 0.2
    raw[hit] = alt[hit]
    return np.ascontiguousarray(raw)


def _effective(src, fmt, samples):
    """(what the passes read, its oracle format tag): the resolved MSAA image, the RGBA32F copy of an RGB32F source"""
    from oracle import frontend
    if samples > 1:
        src = frontend.resolve_msaa(src, samples, fmt)
    if fmt == RGB32F:
        return np.concatenate([src, np.ones(src.shape[:2] + (1,), np.float32)], -1), None
    return src, (fmt if fmt in (BGRA8, RGB10A2, BGRX8) else None)


# ---- the oracle ----------------------------------------------------------------------------------------------------
def _out_dtype(fmt):
    return {RGBA16F: np.float16, RGBA32F: np.float32}.get(fmt, np.uint8)


def _want(st, src, stag, eye, one):
    """the oracle's output of one texture (eye `eye` of a one-eye layout, or the shared texture) and, for FSR, what the
    coverage counters and the failure message need: (output, info)"""
    from oracle import pyoracle as po
    cfg = st.cfg
    h, w = src.shape[:2]
    scale = cfg.renderScale
    ow, oh = po.output_size(w, h, scale)
    proj = st.proj()
    rs = (st.radius(eye),) * 2 if one else (st.radius(0), st.radius(1))
    rsq = [po.upscale_constants(0, True, w, h, ow, oh, radius=r).radius[1] for r in rs]
    ofmt = st.out_format()
    odt, otag = _out_dtype(ofmt), (RGB10A2 if ofmt == RGB10A2 else None)
    easu_b, rcas_b, nis_b, mid_dt = st.plan()[:4]
    kw = dict(proj=proj, sharpness=st.sharpness(), debug=cfg.debugMode)
    if cfg.useNis:
        sharpen = scale == 1.0

        def run(c):
            if nis_b:  # a float source: the checker's pass with the plan's bits
                if sharpen:
                    return pq.nis_sharpen(src, c, odt, nis_b, nthreads=NT)
                return pq.nis_scaler(src, ow, oh, c, odt, nis_b, nthreads=NT)
            if sharpen:
                return po.nis_sharpen(src, c, out_dtype=odt, nthreads=NT, src_fmt=stag, dst_fmt=otag)
            return po.nis_scaler(src, ow, oh, c, out_dtype=odt, nthreads=NT, src_fmt=stag, dst_fmt=otag)
        nis = lambda r: po.nis_config(sharpen, eye, one, w, h, ow, oh, radius=r, **kw)[0]  # noqa: E731
        if rs[0] == rs[1]:
            return run(nis(rs[0])), {"nis": True}
        m = fr._mask((oh, ow), 32, 32 if sharpen else 24, list(nis(0.5).imageCentre), *rsq)
        return fr._select(m, run(fr._all(nis(0.5), True)), run(fr._all(nis(0.5), False))), {"nis": True, "unequal": True}
    # the intermediate: the plan's float format for mapped values, else the output's format
    mtag = otag if mid_dt is None else None
    mid_dt = odt if mid_dt is None else mid_dt
    uc = lambda r: po.upscale_constants(eye, one, w, h, ow, oh, proj=proj, radius=r)  # noqa: E731
    sc = lambda r: po.sharpen_constants(eye, one, ow, oh, radius=r, **kw)  # noqa: E731

    def easu(c):
        if easu_b:
            return pq.easu(src, ow, oh, c, mid_dt, easu_b, nthreads=NT)
        return po.easu(src, ow, oh, c, out_dtype=mid_dt, nthreads=NT, src_fmt=stag, dst_fmt=mtag)

    def rcas(mid, c):
        if rcas_b:  # a float source or a float intermediate (a UNORM intermediate gets no bits)
            return pq.rcas(mid, c, odt, rcas_b, nthreads=NT)
        return po.rcas(mid, c, out_dtype=odt, nthreads=NT, src_fmt=stag if scale == 1.0 else mtag, dst_fmt=otag)
    centre = list(sc(0.5).imageCentre)
    m = fr._mask((oh, ow), 16, 16, centre, *rsq)
    if rs[0] == rs[1]:
        mid = easu(uc(rs[0])) if scale != 1.0 else src
        out = rcas(mid, sc(rs[0]))
    else:
        mid = fr._select(m, easu(fr._all(uc(0.5), True)), easu(fr._all(uc(0.5), False))) if scale != 1.0 else src
        out = fr._select(m, rcas(mid, fr._all(sc(0.5), True)), rcas(mid, fr._all(sc(0.5), False)))
    info = {"nis": False, "unequal": rs[0] != rs[1], "inside": m[::16, ::16], "src": src, "src_fmt": _code(src, stag),
            "mid": mid, "mid_fmt": _code(mid, mtag if scale != 1.0 else stag), "rcas_bits": rcas_b,
            "easu_words": uc(0.5).words() if scale != 1.0 else None, "ow": ow, "oh": oh}
    return out, info


def _code(a, tag):
    """the format an oracle array with format tag `tag` holds"""
    return tag if tag is not None else {np.float16: RGBA16F, np.float32: RGBA32F}.get(np.dtype(a.dtype).type, RGBA8)


# ---- group roles (numpy mirrors of the kernels' footprint and window rules) -------------------------------------------
def _roles(info):
    """per-group arrays (gy, gx): inside, EASU one-colour footprint (UNORM sources: the only ones EASU tests), RCAS
    one-colour window (of the texels after RCAS's read maps), outside with an inside 4-neighbour"""
    inside = info["inside"]
    easu_flat = np.zeros_like(inside)
    rcas_flat = np.zeros_like(inside)
    if info["easu_words"] is not None and info["src_fmt"] not in (RGBA16F, RGBA32F):
        key = rf._rgb_bits(info["src"], info["src_fmt"])
        h, w = key.shape[:2]
        for (gx, gy), (x0, x1, y0, y1) in ef._footprints(info["easu_words"], info["ow"], info["oh"]).items():
            if inside[gy, gx]:
                xs, ys = np.clip(np.arange(x0, x1 + 1), 0, w - 1), np.clip(np.arange(y0, y1 + 1), 0, h - 1)
                fp = key[np.ix_(ys, xs)]
                easu_flat[gy, gx] = (fp == fp[0, 0]).all()
    mid, read = info["mid"], info["rcas_bits"] & pq.READ_BITS
    h, w = mid.shape[:2]
    key = np.zeros((h + 18, w + 18, 3), np.int64)  # zeros outside the image, as Texture2D.Load reads there
    if read:
        # the kernel's one-colour test compares the texels after its read maps; the device's maps return one NaN
        m = pq.read_map(mid, read)
        key[1:h + 1, 1:w + 1] = rf._rgb_bits(np.where(np.isnan(m), np.float32(np.nan), m), RGBA32F)
    else:
        key[1:h + 1, 1:w + 1] = rf._rgb_bits(mid, info["mid_fmt"])
    for gy, gx in zip(*np.nonzero(inside)):
        win = key[gy * 16:gy * 16 + 18, gx * 16:gx * 16 + 18]
        rcas_flat[gy, gx] = (win == win[1, 1]).all()
    pad = np.pad(inside, 1)
    nbr = ~inside & (pad[:-2, 1:-1] | pad[2:, 1:-1] | pad[1:-1, :-2] | pad[1:-1, 2:])
    return inside, easu_flat, rcas_flat, nbr


def _role_of(info, roles, y, x):
    if info["nis"]:
        return "NIS block (32-pixel)"
    inside, easu_flat, rcas_flat, nbr = roles
    gy, gx = y // 16, x // 16
    if inside[gy, gx]:
        what = ["inside the circle"]
        if info["easu_words"] is not None:
            what.append("EASU footprint one colour (easu_flat_group)" if easu_flat[gy, gx] else "EASU filtered")
        what.append("RCAS window one colour (rcas_flat_group)" if rcas_flat[gy, gx] else "RCAS filtered")
        # the paired path: which outside neighbours' intermediate this group reads, and the RCAS CTA's skip
        pad = np.pad(inside, 1)
        out_nb = [n for n, (dy, dx) in zip(("left", "right", "top", "bottom"), ((0, -1), (0, 1), (-1, 0), (1, 0)))
                  if not pad[gy + 1 + dy, gx + 1 + dx]]
        if out_nb:
            what.append("outside neighbours " + "/".join(out_nb))
        tile = inside[gy // 2 * 2:gy // 2 * 2 + 2, gx // 4 * 4:gx // 4 * 4 + 4]
        what.append(f"RCAS tile ({gx // 4}, {gy // 2}) group row {gy % 2}, inside groups per row "
                    f"{[int(r.sum()) for r in tile]}")
        return ", ".join(what)
    return "outside the circle" + (", next to an inside group" if nbr[gy, gx] else "")


# ---- comparison ----------------------------------------------------------------------------------------------------
def _bad_strict(got, want):
    if got.dtype.kind == "f":
        bits = {2: np.uint16, 4: np.uint32}[got.dtype.itemsize]
        return (got.view(bits) != want.view(bits)) & ~(np.isnan(got) & np.isnan(want))
    return got != want


def _compare(st, got, want, src):
    """(None or a description, per-pixel bad mask or None, fast-math error, maxima key)"""
    ofmt = st.out_format()
    if got.shape != want.shape or got.dtype != want.dtype:
        return f"shape / dtype {got.shape} {got.dtype} != {want.shape} {want.dtype}", None, 0.0, None
    if st.strict():
        bad = _bad_strict(got, want)
        return (None if not bad.any() else f"strict: {int(bad.sum())} words differ"), bad, 0.0, None
    easu_b, rcas_b, nis_b = st.plan()[:3]
    bits = st.bits()
    store = nis_b if st.cfg.useNis else rcas_b  # the last pass's bits
    tone, perc, finite = bits & (pq.SRTM_IN | pq.SRTM_OUT), bits & pq.PERCEPTUAL_IN, bits & pq.FINITE_IN
    two = st.fsr() and st.upscale()  # two passes
    maps = "+".join(n for n, b in (("srtm", tone), ("finite", finite), ("perceptual", perc)) if b)
    key = (f"{'nis' if st.cfg.useNis else 'fsr'}{' ' + maps if maps else ''}{' (composed)' if two else ''} -> "
           f"{NAMES[ofmt]}{' (sRGB)' if st.srgb() else ''}")
    if ofmt in (RGBA8, RGB10A2):
        d = np.abs(vm._units(got, ofmt) - vm._units(want, ofmt))
        if st.srgb():
            # one pass: test_gpu_perceptual._fast_check; two: the bound this file proposes (module docstring)
            lim = 8 if two else 4
            if two:
                STATE["beyond_srgb"][0] += int((d > 2).sum())
                STATE["beyond_srgb"][1] += d.size
        else:
            comp = two or tone  # two passes, or the tone map's G after RCAS / NIS
            lim = _paired_lsb(st.sharpness()) if st.paired() else 4 if comp else 1
            if comp:
                # 1 LSB, plus what RCAS's amplification adds to the paired bound above its 4 LSB (_paired_lsb)
                STATE["beyond"][0] += int((d > (lim - 3 if st.paired() else 1)).sum())
                STATE["beyond"][1] += d.size
        err = float(d.max())
        return (None if err <= lim else f"fast: max {err:.0f} > {lim}"), d > lim, err, key
    if perc:
        # test_gpu_perceptual._fast_check in the filter domain (the store maps undone), 2e-3 per pass, relative
        # above 1; two passes: 4e-3, the bound this file introduces for two passes into a float target
        lim = 4e-3 if two else 2e-3
        g, w = (tp._fast_domain(a, store, ofmt).astype(np.float64) for a in (got, want))
        same = (g == w) | (np.isnan(g) & np.isnan(w))
        with np.errstate(invalid="ignore"):
            rel = np.where(same, 0.0, np.abs(g - w) / np.maximum(1.0, np.abs(w)))
        rel = np.where(np.isnan(rel), np.inf, rel)  # a NaN on one side only, or infinities that differ
        err = float(rel.max())
        return (None if err <= lim else f"fast: filter-domain error {err:.3g} > {lim}"), rel > lim, err, key
    if tone:
        err, same = ts._tone_err(got, want)
        g, w = ts._f64(got), ts._f64(want)
        bad = (np.abs(g - w) > 2e-3) | (np.isnan(g) != np.isnan(w))
        return (None if same and err <= 2e-3 else f"fast: tone-mapped error {err:.3g} > 2e-3 (NaN classes agree: {same})"), \
            bad, err, key
    fsrc = src if (src is not None and src.dtype.kind == "f") else None  # the footprint term is for float sources
    if fsrc is not None and finite:
        fsrc = fin.finite_in(fsrc)  # what the first pass filters (test_gpu_finite.py)
    msg, err = fs.check(got, want, ofmt, "fast", two, fsrc)
    # two passes into a float target: the bound this file introduces (module docstring), 4x the per-pass bound
    lim = 4e-3 if two else 1e-3
    if err <= lim:
        return None, None, err, key
    g, w = got.astype(np.float64), want.astype(np.float64)
    bad = ~np.isclose(g, w, rtol=lim, atol=lim, equal_nan=True)
    return msg or f"fast: error {err:.3g} > {lim}", bad, err, key


def _paired_lsb(sharpness):
    """the fast bound of EASU -> UNORM intermediate -> RCAS: RCAS's own 1 LSB plus the intermediate's 1 LSB as RCAS
    amplifies it.  RCAS's output is (L (b + d + f + h) + e) / (4 L + 1) with a lobe L in [-0.1875 s, 0] and
    s = exp2(-(2 - 2 sharpness)) (FsrRcasCon), so one LSB in each of its five taps moves it by up to
    (1 + 4 |L|) / (1 - 4 |L|): 3.6 LSB at test_gpu_variant_matrix.py's sharpness 0.8, whose measured 4 LSB this keeps,
    and 7 LSB at sharpness 1, where an H100 gave 5 (strict/23 frame 6 of the mixed-math seeds, set_sharpness(1))"""
    lobe = 4 * 0.1875 * 2.0 ** -(2 - 2 * min(max(sharpness, 0.0), 1.0))
    return max(4, int(1 + (1 + lobe) / (1 - lobe)))


# ---- one frame -----------------------------------------------------------------------------------------------------
def _sentinel(frame):
    return 0xA5 if frame % 2 == 0 else 0x5A


def _poison(t, byte):
    import torch
    import openvr_fsr_b200 as ovr
    if isinstance(t, ovr.ArrayImage):
        dt = t._dtype()
        es = torch.empty((), dtype=dt).element_size()
        fill = torch.full((t.height, t.width, 4 * es), byte, dtype=torch.uint8, device=t.device).view(dt)
        t.upload(fill)
        return t
    t.view(torch.uint8).fill_(byte)
    return t


def _is_sentinel(a, byte):
    return bool((np.ascontiguousarray(a).view(np.uint8) == byte).all())


def _host(t):
    import openvr_fsr_b200 as ovr
    return np.ascontiguousarray((t.download() if isinstance(t, ovr.ArrayImage) else t).cpu().numpy())


def _api_fmt(fmt):
    return fmt if fmt in (BGRA8, RGB10A2, BGRX8, RGB32F) else None


def _run_frame(pp, st, texs, dev, byte, keep):
    """submit one frame (both eyes) through st.entry.  texs: the numpy textures (one per eye, or the shared one).
    Returns ([(eye label, output tensor / array / host tensor, sentinel expected, owned by the context)], the sources,
    OVRFSR_FORMAT_SRGB_BIT of the returned format for apply / apply_pair, else None);
    keep: the caller's objects to free after the frame"""
    import torch
    import openvr_fsr_b200 as ovr
    fmt, ofmt = st.fmt, st.out_format()
    w, h = texs[0].shape[1] // max(st.samples, 1), texs[0].shape[0]
    ow, oh = ovr.output_size(w, h, st.cfg.renderScale)
    bounds = [ovr.TextureBounds()] * 2 if st.one else [ovr.TextureBounds(*b) for b in SHARED]
    afmt = _api_fmt(fmt)
    dfmt = RGB10A2 if ofmt == RGB10A2 else (RGBA8 | SRGB_BIT) if st.dst_srgb else None
    if st.entry == "apply_host":
        srcs = [torch.from_numpy(t).pin_memory() for t in texs]
        dsts = [_poison(torch.empty((oh, ow, 4), dtype=vm._dtype(ofmt)).pin_memory(), byte) for _ in range(2)]
        torch.cuda.synchronize()
        for e in (0, 1):
            pp.apply_host(e, srcs[e], dsts[e], bounds[e], fmt=afmt, dst_fmt=dfmt)
        torch.cuda.synchronize()
        keep += srcs
        return [(f"eye {e}", dsts[e], False, False) for e in (0, 1)], srcs, None
    if st.src_array:
        srcs = [ovr.ArrayImage(t.shape[1], t.shape[0], fmt).upload(torch.from_numpy(t).to(dev)) for t in texs]
        keep += srcs
    elif fmt == RGB32F or st.tight:
        srcs = [torch.from_numpy(t).to(dev) for t in texs]  # tight rows: plain loads
    else:
        srcs = [ovr.to_image(t, dev) for t in texs]  # pitch-aligned: TMA loads
    if not st.one:
        srcs = [srcs[0], srcs[0]]
    res = []
    if st.entry in ("apply_into", "apply_pair_into"):
        if st.dst_array:
            dsts = [_poison(ovr.ArrayImage(ow, oh, ofmt), byte) for _ in range(2)]
            keep += dsts
        else:
            dsts = [_poison(ovr.alloc_image(ow, oh, vm._dtype(ofmt), dev), byte) for _ in range(2)]
        torch.cuda.synchronize()
        if st.dst_array and st.dst_srgb:  # the tag is the image's; cleared again before anything downloads it
            for d in dsts:
                d.image.format |= SRGB_BIT
        if st.entry == "apply_into":
            outs = [pp.apply_into(e, srcs[e], dsts[e], bounds[e], fmt=afmt, dst_fmt=dfmt) for e in (0, 1)]
        else:
            outs = list(pp.apply_pair_into(srcs[0], srcs[1], dsts[0], dsts[1], bounds[0], fmt=afmt, dst_fmt=dfmt))
        torch.cuda.synchronize()
        if st.dst_array:
            for d in dsts:
                d.image.format &= ~SRGB_BIT
        if not st.cfg.fsrEnabled:
            assert all(o is s for o, s in zip(outs, srcs)), "pass-through returns the source"
            return [(f"eye {e}", dsts[e], True, False) for e in (0, 1)], srcs, None
        assert all(o is d for o, d in zip(outs, dsts))
        # a shared texture is processed by the first call of a frame; the second writes nothing
        return [(f"eye {e}", dsts[e], not st.one and e == 1, False) for e in (0, 1)], srcs, None
    if st.entry == "apply":
        outs = [pp.apply(e, srcs[e], bounds[e], fmt=afmt, samples=st.samples) for e in (0, 1)]
    else:
        outs = list(pp.apply_pair(srcs[0], srcs[1], bounds[0], fmt=afmt))
    torch.cuda.synchronize()
    if not st.cfg.fsrEnabled:
        assert all(o is s for o, s in zip(outs, srcs)), "pass-through returns the source"
        return [], srcs, None
    if not st.one:
        assert outs[0].data_ptr() == outs[1].data_ptr()
        outs = outs[:1]
    return [(f"eye {e}" if st.one else "shared", o, False, True) for e, o in enumerate(outs)], srcs, \
        pp.last_output_format & SRGB_BIT


def _count(st, info, roles, cov):
    if info["nis"]:
        return
    inside, easu_flat, rcas_flat, nbr = roles
    if not st.fused():  # the two dispatches ran (the fused kernel has no one-colour paths)
        if info["easu_words"] is not None and info["src_fmt"] not in (RGBA16F, RGBA32F):
            cov["EASU one-colour inside groups"] += int((inside & easu_flat).sum())
            cov["EASU filtered inside groups"] += int((inside & ~easu_flat).sum())
        cov["RCAS one-colour inside groups"] += int((inside & rcas_flat).sum())
        if info["rcas_bits"]:
            after = "after EASU" if info["easu_words"] is not None else "RCAS alone"
            cov[f"RCAS one-colour inside groups with map bits, {after}"] += int((inside & rcas_flat).sum())
        cov["RCAS filtered inside groups"] += int((inside & ~rcas_flat).sum())
    if st.paired() and not st.fused():
        cov["paired: outside groups next to inside ones"] += int(nbr.sum())


def _frame_sequence(kind, seed, dev):
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    STATE["t0"] = STATE["t0"] or time.monotonic()
    rng = np.random.default_rng([7919, 0 if kind == "strict" else 1, seed])
    math = "fast" if kind == "fast" else ("mixed" if seed % 4 == 3 else "strict")
    cfg = _draw_config(rng, math)
    cfg = dataclasses.replace(cfg, fsrEnabled=True)
    beyond0 = list(STATE["beyond"])
    pp = ovr.PostProcessor(cfg)
    cov = STATE["cov"]
    foci, radii, sharp = [None, None], [None, None], None
    one, fmt = bool(rng.random() < 0.75), int(rng.choice(FORMATS))
    size = _draw_size(rng, cfg.renderScale, one)
    live = None  # (size, format, layout) the context last ran a frame with, None after a reset
    pending = set()  # set_config transitions on a live context not yet followed by a frame
    try:
        for i in range(FRAMES):
            byte = _sentinel(i)
            changed = []
            # -- state changes --------------------------------------------------------------------------------------
            if i > 0 and rng.random() < 0.3:
                new = _draw_config(rng, math, cfg)
                if live is not None:
                    for f in ("srtm", "srtmNis", "finite", "perceptual", "fusedFsr", "outputFormat"):
                        if getattr(new, f) != getattr(cfg, f):
                            pending.add(f)
                pp.set_config(new)
                cfg, live = new, None
                changed.append("set_config")
                if rng.random() < 0.5:
                    size = _draw_size(rng, cfg.renderScale, one)
            for e in (0, 1):
                r = rng.random()
                if r < 0.3:
                    foci[e] = _draw_point(rng)
                    pp.set_focus(e, *foci[e])
                    changed.append(f"set_focus({e}, {foci[e]})")
                elif r < 0.4:
                    foci[e] = None
                    pp.clear_focus(e)
                    changed.append(f"clear_focus({e})")
                r = rng.random()
                if r < 0.3:
                    radii[e] = float(rng.choice([0.0, 4.0, rng.uniform(0, 4)] + RADII))
                    pp.set_focus_radius(e, radii[e])
                    changed.append(f"set_focus_radius({e}, {radii[e]:.3f})")
                elif r < 0.4:
                    radii[e] = None
                    pp.clear_focus_radius(e)
                    changed.append(f"clear_focus_radius({e})")
            focus_change = any(c.startswith(("set_focus", "clear_focus")) for c in changed)
            # the sharpness override: late-latched, kept across set_config and reset
            r, sharp_change = rng.random(), None
            if r < 0.15:
                sharp, sharp_change = float(rng.choice([0.0, 1.0, rng.uniform(0, 1)])), "set"
                pp.set_sharpness(sharp)
                changed.append(f"set_sharpness({sharp:.3f})")
            elif r < 0.25:
                sharp, sharp_change = None, "clear"
                pp.clear_sharpness()
                changed.append("clear_sharpness()")
            if i > 0 and rng.random() < 0.12:
                one = not one
                if live is not None:
                    pp.reset()  # the layout is read when the context (re)creates its resources
                    live = None
                    changed.append("reset (layout)")
                size = _draw_size(rng, cfg.renderScale, one)
            if i > 0 and rng.random() < 0.25:
                size = _draw_size(rng, cfg.renderScale, one)
            if i > 0 and rng.random() < 0.15:
                fmt = int(rng.choice(FORMATS))
            # -- entry point and I/O ---------------------------------------------------------------------------------
            entries = [e for e in ENTRIES if (e != "apply_host" or (one and fmt != RGB32F and cfg.fsrEnabled))]
            entry = str(rng.choice(entries))
            samples = int(rng.choice([2, 4])) if entry == "apply" and fmt in MSAA_FORMATS and rng.random() < 0.15 else 1
            src_array = entry != "apply_host" and samples == 1 and fmt != RGB32F and rng.random() < 0.25
            dst_array = entry in ("apply_into", "apply_pair_into") and rng.random() < 0.35
            st = Frame(cfg, list(foci), list(radii), one, fmt, samples, entry, src_array, dst_array, size,
                       samples > 1 or rng.random() < 0.3, sharp)
            st.dst_srgb = entry in ("apply_into", "apply_pair_into") and st.srgb() and rng.random() < 0.5
            bits = st.bits()
            # -- content ---------------------------------------------------------------------------------------------
            w, h = size
            tw = w if one else 2 * w
            ow, oh = po.output_size(tw, h, cfg.renderScale)
            ofmt = st.out_format()
            tone = bits & (pq.SRTM_IN | pq.SRTM_OUT)
            if st.strict():
                extras = "signed"
            elif tone:
                extras = "hdr"  # the tone map's domain: fast math has no bound on negative texels through G
            elif ofmt in (RGBA16F, RGBA32F) or bits & pq.PERCEPTUAL_IN:
                extras = "scrgb"
            else:
                extras = None
            # infinities, NaNs and FP32 texels beyond 65504: strict frames, and fast frames whose passes get FINITE
            # (fast math without it has no bound there; with the tone map only +inf and NaNs stay in its domain)
            hold = fmt in FLOATS and (st.strict() or bits & pq.FINITE_IN)
            nonfinite = ()
            if hold and rng.random() < 0.6:
                nonfinite = tuple(p for p in NONFINITE[fmt][1]
                                  if st.strict() or not tone or p not in (0xfc00, 0xff800000))
            beyond = hold and fmt != RGBA16F and rng.random() < 0.5
            texs = [_content(rng, fmt, tw, h, ow, oh, extras, nonfinite, beyond) for _ in range(2 if one else 1)]
            if samples > 1:
                texs = [_msaa(rng, t, samples) for t in texs]
            # -- coverage of the transitions -------------------------------------------------------------------------
            if cfg.fsrEnabled:
                if live is not None and (live[0] != size or live[1] != fmt):
                    cov["size / format change on a live context"] += 1
                if live is not None and focus_change:
                    cov[f"focus / radius change on a live context: {entry}"] += 1
                if live is not None and sharp_change:
                    cov[f"sharpness {sharp_change} on a live context: {entry}"] += 1
                if live is not None and live[0] == size and (live[1] in FLOATS) != (fmt in FLOATS) and \
                        (cfg.perceptual or cfg.srtm or cfg.srtmNis):
                    cov["UNORM <-> float source change at the same size on a live context with PERCEPTUAL or SRTM"] += 1
                for f in pending:
                    cov[f"{f} transition on a live context"] += 1
                pending.clear()
            # -- run and compare -------------------------------------------------------------------------------------
            keep = []
            outs, _, tag = _run_frame(pp, st, texs, dev, byte, keep)
            if cfg.fsrEnabled:
                live = (size, fmt, one)
                cov[f"source {NAMES[fmt]}"] += 1
                cov[f"math {'strict' if st.strict() else 'fast'}"] += 1
                cov[f"entry {entry}"] += 1
                if samples > 1:
                    cov["MSAA source"] += 1
                if src_array:
                    cov["CUDA-array source"] += 1
                if dst_array:
                    cov["CUDA-array destination"] += 1
                if tone:
                    cov["SRTM_NIS frames" if st.cfg.useNis else "SRTM frames"] += 1
                if bits & pq.FINITE_IN:
                    cov["FINITE frames"] += 1
                if bits & pq.PERCEPTUAL_IN:
                    cov["PERCEPTUAL frames"] += 1
                if st.srgb():
                    cov["sRGB-encoded outputs"] += 1
                if st.dst_srgb:
                    cov["tagged sRGB destination"] += 1
                if nonfinite:
                    cov["non-finite texels with FINITE" if bits & pq.FINITE_IN else
                        "non-finite texels in strict without FINITE"] += 1
                if beyond and (ofmt == RGBA16F or st.plan()[3] == np.float16):
                    cov["FP32 texels beyond 65504 into an FP16 intermediate or output"] += 1
                if st.fused():
                    cov["fused frames"] += 1
                    if bits & pq.FINITE_IN:
                        cov["fused frames with FINITE"] += 1
                if st.cfg.useNis:
                    cov["NIS frames"] += 1
            else:
                cov["pass-through frames"] += 1
            failures = []
            if tag is not None and bool(tag) != st.srgb():
                failures.append(f"the returned format {'carries' if tag else 'lacks'} OVRFSR_FORMAT_SRGB_BIT, but the "
                                f"plan {'encodes' if st.srgb() else 'does not encode'} sRGB")
            wants = {}
            for label, out, expect_sentinel, ctx_owned in outs:
                got = _host(out)
                if expect_sentinel:
                    if not _is_sentinel(got, byte):
                        failures.append(f"{label}: a call that writes nothing changed its destination")
                    continue
                eye = 0 if label == "shared" or not one else int(label[-1])
                src, stag = _effective(texs[eye if one else 0], fmt, samples)
                if (eye, one) not in wants:
                    wants[eye, one] = _want(st, src, stag, eye if one else 0, one)
                want, info = wants[eye, one]
                roles = None if info["nis"] else _roles(info)
                if roles is not None:
                    _count(st, info, roles, cov)
                if info.get("unequal"):
                    cov["shared texture with unequal radii"] += 1
                msg, bad, err, key = _compare(st, got, want, src)
                if key is not None:
                    STATE["maxima"][key] = max(STATE["maxima"][key], err)
                if msg:
                    where = ""
                    if bad is not None and bad.any():
                        y, x = (int(v) for v in np.argwhere(bad.reshape(bad.shape[0], bad.shape[1], -1).any(-1))[0])
                        g, wv = got[y, x], want[y, x]
                        where = (f"; first wrong pixel (x={x}, y={y}): got {g.tolist()} want {wv.tolist()}"
                                 f"{' (the sentinel)' if _is_sentinel(g, byte) else ''}; 16x16 group ({x // 16}, {y // 16}) "
                                 "by the oracle's rules: "
                                 f"{_role_of(info, roles, y, x)}")
                    failures.append(f"{label}: {msg}{where}")
            assert not failures, (f"seed {kind}/{seed} frame {i} ({' '.join(changed) or 'no state change'}): "
                                  + "; ".join(failures) + f"\n  state: {st.describe()}")
            # -- poison what the frame returned, before anything of the next frame ------------------------------------
            for _, out, _, _ in outs:
                _poison(out, byte)
            torch.cuda.synchronize()
            for a in keep:
                if isinstance(a, ovr.ArrayImage):
                    a.release()
                    a.close()
            STATE["frames"] += 1
    finally:
        pp.close()
    STATE["seeds"] += 1
    n_beyond, n = STATE["beyond"][0] - beyond0[0], STATE["beyond"][1] - beyond0[1]
    assert n_beyond <= 1e-4 * n, f"seed {kind}/{seed}: fast composed: {n_beyond} of {n} channels beyond 1 LSB"


@pytest.mark.parametrize("fmt", [RGBA16F, RGBA32F])
def test_nis_sharpen_reads_its_texel_through_the_bilinear_tap(cuda, fmt):
    """Found by the sequences below (strict seed 34, NIS at scale 1 on an RGB32F eye): NVSharpen reads each output's
    own texel through a bilinear tap with weights 1 and 0, which adds the zero-weighted neighbours -- so a -0 texel
    left of a positive one reads as +0.  The kernel read the texel alone and kept -0 (-0 where the oracle has +0 at
    (16, 16) of this 32x32 crop of that frame: a -0 block next to natural texels and a 7.5 impulse).  Strict, stateless
    and through the context."""
    import torch
    import openvr_fsr_b200 as ovr
    from oracle import pyoracle as po
    rgb = np.load(os.path.join(os.path.dirname(__file__), "golden", "nis_sharpen_signed_zero.npz"))["rgb"]
    h, w = rgb.shape[:2]
    src = np.concatenate([rgb, np.ones((h, w, 1), np.float32)], -1).astype(_out_dtype(fmt))
    cfg, ok = po.nis_config(True, 0, True, w, h, w, h, radius=2.0, sharpness=0.277)
    assert ok
    want = po.nis_sharpen(src, cfg, out_dtype=np.float32)
    assert np.signbit(src[16, 16, :3]).all() and not np.signbit(want[16, 16, :3]).any() and (want[16, 16, :3] == 0).all()
    out = torch.empty((h, w, 4), dtype=torch.float32, device=cuda)
    ovr.nis_sharpen(torch.from_numpy(src).to(cuda), out, bytes(cfg), ovr.MATH_STRICT)
    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, useNis=True, renderScale=1.0, sharpness=0.277, radius=2.0,
                                      outputFormat=RGBA32F, mathMode=ovr.MATH_STRICT))
    ctx = pp.apply(0, torch.from_numpy(src).to(cuda))
    torch.cuda.synchronize()
    for what, got in (("dispatch", out.cpu().numpy()), ("context", ctx.cpu().numpy())):
        bad = _bad_strict(np.ascontiguousarray(got), want)
        assert not bad.any(), f"{what}: {int(bad.sum())} words differ, first at {np.argwhere(bad)[0].tolist()}"
    pp.close()


SEEDS = [("strict", i) for i in range(N_STRICT)] + [("fast", i) for i in range(N_FAST)]


@pytest.mark.parametrize("kind,seed", SEEDS, ids=[f"{k}-{s}" for k, s in SEEDS])
def test_frame_sequence(cuda, kind, seed):
    _frame_sequence(kind, seed, cuda)


REQUIRED = ["EASU one-colour inside groups", "EASU filtered inside groups", "RCAS one-colour inside groups",
            "RCAS filtered inside groups", "paired: outside groups next to inside ones", "shared texture with unequal radii",
            "size / format change on a live context", "srtm transition on a live context",
            "fusedFsr transition on a live context", "outputFormat transition on a live context", "math strict",
            "math fast", "MSAA source", "CUDA-array source", "CUDA-array destination", "SRTM frames", "SRTM_NIS frames",
            "FINITE frames", "PERCEPTUAL frames", "sRGB-encoded outputs", "tagged sRGB destination",
            "srtmNis transition on a live context", "finite transition on a live context",
            "perceptual transition on a live context",
            "UNORM <-> float source change at the same size on a live context with PERCEPTUAL or SRTM",
            "non-finite texels with FINITE",
            "non-finite texels in strict without FINITE", "fused frames with FINITE",
            "RCAS one-colour inside groups with map bits, after EASU",
            "RCAS one-colour inside groups with map bits, RCAS alone"] + \
    [f"focus / radius change on a live context: {e}" for e in ENTRIES] + \
    [f"sharpness {c} on a live context: {e}" for c in ("set", "clear") for e in ENTRIES] + \
    [f"source {NAMES[f]}" for f in FORMATS]


def test_frame_fuzz_coverage(cuda):
    """runs last: every category reached by the sequences above"""
    cov = STATE["cov"]
    print(f"\nframe fuzz: {STATE['seeds']} seeds, {STATE['frames']} frames")
    for k in sorted(cov):
        print(f"  {k}: {cov[k]}")
    print("fast-math maxima (LSB / code; float targets: error in units of the bound, scaled to 1e-3; SRTM without "
          "PERCEPTUAL: tone-mapped; PERCEPTUAL: relative error in the filter domain):")
    for k, v in sorted(STATE["maxima"].items()):
        print(f"  {k}: {v:.3g}")
    n_beyond, n = STATE["beyond"]
    print(f"fast composed UNORM channels beyond 1 LSB (paired: beyond 1 + the excess of _paired_lsb over 4): "
          f"{n_beyond} of {n}")
    n2, n8 = STATE["beyond_srgb"]
    print(f"fast composed sRGB RGBA8 channels beyond 2 codes: {n2} of {n8}"
          f"{f' ({n2 / n8:.2e})' if n8 else ''}")
    if STATE["t0"] is not None:
        print(f"wall time: {time.monotonic() - STATE['t0']:.1f} s")
    missing = [k for k in REQUIRED if cov[k] == 0]
    assert STATE["frames"], "no frame sequence ran"
    assert not missing, "never reached: " + ", ".join(missing)
    assert n_beyond <= 1e-4 * n, f"fast composed: {n_beyond} of {n} channels beyond 1 LSB"
