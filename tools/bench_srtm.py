"""Dev bench: what OVRFSR_FLAG_SRTM (AMD's reversible tone map around EASU and RCAS) costs on linear RGBA16F eyes.

Workloads: C2-shaped (1683x1869 -> 2244x2492, renderScale 0.75) and C3a-shaped (2244x2492 -> 2917x3239, renderScale
1.3) RGBA16F eyes from synth.natural_rgba16f (peak 4).  Flag off and on, strict and fast math, radius 2.0 (every group
filtered) and 0.5 (the reference default).
  per launch : the stateless dispatches at the ctx's shapes -- EASU float -> intermediate (off: RGBA8, the ctx's
               intermediate for an RGBA8 output; on: F on read into RGBA16F) and RCAS intermediate -> RGBA8 (on: G on
               store); median of --reps windows of --launches launches, CUDA events
  pairs/s    : PostProcessor.apply_pair, RGBA8 output (on: two plain dispatches through an RGBA16F intermediate; off:
               the paired dispatches through RGBA8), median of --reps windows of --passes pairs
The card's name, power limit and SM clocks are read in the same call and printed with the numbers.
usage: python tools/bench_srtm.py [--json out.json]"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
SHAPES = {"C2": (1683, 1869, 0.75), "C3a": (2244, 2492, 1.3)}
SHARP = 0.9


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def timed(fn, n, reps, stream):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(n):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / n)  # us per call
    return statistics.median(ts), min(ts), max(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--passes", type=int, default=30)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--json")
    args = ap.parse_args()
    sys.path.insert(0, str(ROOT))
    import numpy as np
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    dev = torch.device("cuda:0")
    main_s = torch.cuda.current_stream(dev)
    out = {"card_before": card(), "per_launch_us": {}, "pairs_s": {}}
    for shape, (w, h, scale) in SHAPES.items():
        left = synth.natural_rgba16f(w, h, 1)
        right = np.ascontiguousarray(np.roll(left, 16, axis=1))
        tl, tr = ovr.to_image(left, dev), ovr.to_image(right, dev)
        ow, oh = ovr.output_size(w, h, scale)
        mids = {False: ovr.alloc_image(ow, oh, torch.uint8, dev), True: ovr.alloc_image(ow, oh, torch.float16, dev)}
        fin = ovr.alloc_image(ow, oh, torch.uint8, dev)
        for radius in (2.0, 0.5):
            cfg = ovr.Config(fsrEnabled=True, renderScale=scale, sharpness=SHARP, radius=radius)
            uc = ovr.make_upscale_constants(cfg, 0, True, w, h, ow, oh)
            sc = ovr.make_sharpen_constants(cfg, 0, True, ow, oh)
            for mode, mm in (("strict", ovr.MATH_STRICT), ("fast", ovr.MATH_FAST)):
                for on in (False, True):
                    tag = f"{shape}/r{radius}/{mode}/{'on' if on else 'off'}"
                    mid = mids[on]
                    e = timed(lambda: ovr.fsr_easu(tl, mid, uc, mm, srtm_in=on), args.launches, args.reps, main_s)
                    r = timed(lambda: ovr.fsr_rcas(mid, fin, sc, mm, srtm_out=on), args.launches, args.reps, main_s)
                    out["per_launch_us"][tag] = {"easu": e, "rcas": r}
                    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, renderScale=scale, sharpness=SHARP, radius=radius,
                                                      mathMode=mm, srtm=on))
                    t = timed(lambda: pp.apply_pair(tl, tr, stream=main_s), args.passes, args.reps, main_s)
                    pp.close()
                    out["pairs_s"][tag] = {"median": 1e6 / t[0], "min": 1e6 / t[2], "max": 1e6 / t[1]}
                    print(f"{tag:24s} EASU {e[0]:7.1f} us  RCAS {r[0]:7.1f} us  apply_pair {1e6 / t[0]:7.0f} pairs/s", flush=True)
    out["card_after"] = card()
    print(f"card before: {out['card_before']}\ncard after:  {out['card_after']}")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
