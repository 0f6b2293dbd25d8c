"""Dev bench: per-launch time of the stateless EASU dispatch at C2 (1683x1869 -> 2244x2492 RGBA8, radius 2.0) on
natural, textured and uniform-noise content, strict and fast math (CUDA events, back to back on one stream, 8 distinct
pitch-aligned sources cycled).  EASU's time follows the content: inside groups whose footprint has one colour skip the
filter, and tiles without a group that needs it skip the feature stage.  The share of such groups is printed beside
the time (numpy mirror of the footprint rule).  OVRFSR_LIB=<path> measures another build of the library."""
import os, sys, statistics
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import openvr_fsr_b200 as ovr
from openvr_fsr_b200 import synth
from oracle import pyoracle as po

IW, IH, OW, OH = 1683, 1869, 2244, 2492
REPS = int(os.environ.get("REPS", "40"))


def flat_share(img, words):
    """share of 16x16 groups whose f/g/j/k footprint has one RGB (radius 2.0: every group is inside)"""
    f = lambda i: np.array([words[i]], dtype=np.uint32).view(np.float32)[0]  # noqa: E731
    c0x, c0y, c0z, c0w = f(0), f(1), f(2), f(3)
    pos = lambda p, s, o: np.floor(np.float32(np.float32(p) * s) + o).astype(np.int64)  # noqa: E731
    gx = np.arange((OW + 15) // 16) * 16
    gy = np.arange((OH + 15) // 16) * 16
    x0, x1 = pos(gx, c0x, c0z), pos(np.minimum(gx + 15, OW - 1), c0x, c0z) + 1
    y0, y1 = pos(gy, c0y, c0w), pos(np.minimum(gy + 15, OH - 1), c0y, c0w) + 1
    key = img[..., :3].astype(np.int64) @ np.array([1, 256, 65536])
    n = 0
    for a, b in zip(y0, y1):
        rows = key[np.clip(np.arange(a, b + 1), 0, IH - 1)]
        for c, d in zip(x0, x1):
            blk = rows[:, np.clip(np.arange(c, d + 1), 0, IW - 1)]
            n += bool((blk == blk[0, 0]).all())
    return n / (len(gx) * len(gy))


def main():
    dev = torch.device("cuda:0")
    dst = ovr.alloc_image(OW, OH, torch.uint8, dev)
    uc = po.upscale_constants(0, True, IW, IH, OW, OH, radius=2.0)
    words = uc.words()
    gens = {"natural": synth.natural_rgba8, "textured": synth.textured_rgba8, "uniform": synth.uniform_rgba8}
    out = []
    for name, gen in gens.items():
        base = gen(IW, IH, 1)
        share = flat_share(base, words)
        pool = [ovr.to_image(np.ascontiguousarray(np.roll(base, 37 * i, axis=0)), dev) for i in range(8)]
        for mm, mname in ((ovr.MATH_STRICT, "strict"), (ovr.MATH_FAST, "fast")):
            for i in range(16):
                ovr.fsr_easu(pool[i % 8], dst, words, mm)
            marks = []
            for _ in range(REPS):
                for i in range(8):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(); ovr.fsr_easu(pool[i], dst, words, mm); e1.record(); marks.append((e0, e1))
            torch.cuda.synchronize()
            t = [a.elapsed_time(b) * 1e3 for a, b in marks]
            out.append(f"{name} {mname}: EASU {statistics.mean(t):6.1f} us (median {statistics.median(t):6.1f}), "
                       f"one-colour groups {share:.1%}")
    print(os.environ.get("OVRFSR_LIB", "current"))
    print("\n".join(out))


if __name__ == "__main__":
    main()
