"""Dev bench: per-launch time of the stateless RCAS dispatch at C2 (2244x2492 RGBA8 -> RGBA8, radius 2.0) on natural,
textured and uniform-noise content, strict and fast math (CUDA events, back to back on one stream, 8 distinct
pitch-aligned intermediates cycled).  Each scene goes once through fsr_easu to give the intermediates RCAS sees in the
two-pass path.  RCAS's time follows the content: inside groups whose cross window (the group plus a 1-texel ring) has
one RGB store their first pixel's value instead of filtering every pixel.  The share of such groups is printed beside
the time (numpy mirror of the window rule on the downloaded intermediate).  OVRFSR_LIB=<path> measures another build."""
import os, sys, statistics
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import openvr_fsr_b200 as ovr
from openvr_fsr_b200 import synth
from oracle import pyoracle as po

IW, IH, OW, OH = 1683, 1869, 2244, 2492
REPS = int(os.environ.get("REPS", "40"))


def flat_share(img):
    """share of 16x16 groups whose 18x18 window (zeros outside the image) has one RGB (radius 2.0: all inside)"""
    key = np.zeros((OH + 18, OW + 18), np.int64)
    key[1:OH + 1, 1:OW + 1] = img[..., :3].astype(np.int64) @ np.array([1, 256, 65536])
    n = total = 0
    for gy in range(0, OH, 16):
        for gx in range(0, OW, 16):
            win = key[gy:gy + 18, gx:gx + 18]
            n += bool((win == win[1, 1]).all())
            total += 1
    return n / total


def main():
    dev = torch.device("cuda:0")
    dst = ovr.alloc_image(OW, OH, torch.uint8, dev)
    uc = po.upscale_constants(0, True, IW, IH, OW, OH, radius=2.0)
    sc = po.sharpen_constants(0, True, OW, OH, radius=2.0, sharpness=0.9)
    words, rwords = uc.words(), sc.words()
    gens = {"natural": synth.natural_rgba8, "textured": synth.textured_rgba8, "uniform": synth.uniform_rgba8}
    out = []
    for name, gen in gens.items():
        base = gen(IW, IH, 1)
        pool = []
        for i in range(8):
            mid = ovr.alloc_image(OW, OH, torch.uint8, dev)
            ovr.fsr_easu(ovr.to_image(np.ascontiguousarray(np.roll(base, 37 * i, axis=0)), dev), mid, words,
                         ovr.MATH_STRICT)
            pool.append(mid)
        torch.cuda.synchronize()
        share = flat_share(pool[0].cpu().numpy())
        for mm, mname in ((ovr.MATH_STRICT, "strict"), (ovr.MATH_FAST, "fast")):
            for i in range(16):
                ovr.fsr_rcas(pool[i % 8], dst, rwords, mm)
            marks = []
            for _ in range(REPS):
                for i in range(8):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(); ovr.fsr_rcas(pool[i], dst, rwords, mm); e1.record(); marks.append((e0, e1))
            torch.cuda.synchronize()
            t = [a.elapsed_time(b) * 1e3 for a, b in marks]
            out.append(f"{name} {mname}: RCAS {statistics.mean(t):6.1f} us (median {statistics.median(t):6.1f}), "
                       f"one-colour windows {share:.1%}")
    print(os.environ.get("OVRFSR_LIB", "current"))
    print("\n".join(out))


if __name__ == "__main__":
    main()
