"""Dev bench: what OVRFSR_FLAG_SRTM (AMD's reversible tone map around EASU and RCAS) and OVRFSR_FLAG_SRTM_NIS (the same
map around NVScaler / NVSharpen) cost on linear RGBA16F eyes.

FSR workloads: C2-shaped (1683x1869 -> 2244x2492, renderScale 0.75) and C3a-shaped (2244x2492 -> 2917x3239, renderScale
1.3) RGBA16F eyes from synth.natural_rgba16f (peak 4).  Flag off and on, strict and fast math, radius 2.0 (every group
filtered) and 0.5 (the reference default).
  per launch : the stateless dispatches at the ctx's shapes -- EASU float -> intermediate (off: RGBA8, the ctx's
               intermediate for an RGBA8 output; on: F on read into RGBA16F) and RCAS intermediate -> RGBA8 (on: G on
               store); median of --reps windows of --launches launches, CUDA events
  pairs/s    : PostProcessor.apply_pair, RGBA8 output (on: two plain dispatches through an RGBA16F intermediate; off:
               the paired dispatches through RGBA8), median of --reps windows of --passes pairs
NIS workloads: C4-shaped RGBA16F eyes (1512x1680 -> 2016x2240, NVScaler at renderScale 0.75; NVSharpen at renderScale 1
on the same eyes), same flag / math / radius arms: per launch = the stateless NIS dispatch RGBA16F -> RGBA8 (on: F on
read and G on store), pairs/s = PostProcessor.apply_pair with useNis, RGBA8 output.
Overshoot (oracle, CPU, printed only): NVScaler output channels above the maximum of their 6x6 source window (and above
1.5 x that maximum), in linear light, on a quarter-size C4 eye at peak 4 and 1000, radius 2.0, RGBA32F output, flag off
and on.
The card's name, power limit and SM clocks are read in the same call and printed with the numbers.
usage: python tools/bench_srtm.py [--only fsr|nis|overshoot] [--json out.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
SHAPES = {"C2": (1683, 1869, 0.75), "C3a": (2244, 2492, 1.3)}
NIS_SHAPE = (1512, 1680)  # C4
NIS_PATHS = {"scaler": 0.75, "sharpen": 1.0}
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


def nis_arms(args, out, dev, main_s):
    """NVScaler / NVSharpen at C4, RGBA16F -> RGBA8, OVRFSR_FLAG_SRTM_NIS off and on"""
    import numpy as np
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    w, h = NIS_SHAPE
    left = synth.natural_rgba16f(w, h, 1)
    right = np.ascontiguousarray(np.roll(left, 16, axis=1))
    tl, tr = ovr.to_image(left, dev), ovr.to_image(right, dev)
    for path, scale in NIS_PATHS.items():
        ow, oh = ovr.output_size(w, h, scale)
        fin = ovr.alloc_image(ow, oh, torch.uint8, dev)
        for radius in (2.0, 0.5):
            cfg = ovr.Config(fsrEnabled=True, useNis=True, renderScale=scale, sharpness=SHARP, radius=radius)
            ncfg, ok = ovr.make_nis_config(cfg, scale == 1.0, 0, True, w, h, ow, oh)
            assert ok
            fn = ovr.nis_scaler if scale != 1.0 else ovr.nis_sharpen
            for mode, mm in (("strict", ovr.MATH_STRICT), ("fast", ovr.MATH_FAST)):
                for on in (False, True):
                    tag = f"C4/nis_{path}/r{radius}/{mode}/{'on' if on else 'off'}"
                    k = timed(lambda: fn(tl, fin, ncfg, mm, srtm_in=on, srtm_out=on), args.launches, args.reps, main_s)
                    out["per_launch_us"][tag] = {"nis": k}
                    pp = ovr.PostProcessor(ovr.Config(fsrEnabled=True, useNis=True, renderScale=scale, sharpness=SHARP,
                                                      radius=radius, mathMode=mm, srtmNis=on))
                    t = timed(lambda: pp.apply_pair(tl, tr, stream=main_s), args.passes, args.reps, main_s)
                    pp.close()
                    out["pairs_s"][tag] = {"median": 1e6 / t[0], "min": 1e6 / t[2], "max": 1e6 / t[1]}
                    print(f"{tag:32s} NIS {k[0]:7.1f} us  apply_pair {1e6 / t[0]:7.0f} pairs/s", flush=True)


def nis_overshoot():
    """NVScaler output channels (linear light, RGBA32F) above the maximum of the same channel over the 6x6 source window
    the pass reads (rows / columns floor(src) - 2 .. floor(src) + 3, clamped), flag off and on, from the oracle"""
    import numpy as np
    from scipy.ndimage import maximum_filter
    from openvr_fsr_b200 import synth
    from oracle import pyoracle as po
    sys.path.insert(0, str(ROOT / "tests"))
    import srtm_oracle as so
    w, h = NIS_SHAPE[0] // 4, NIS_SHAPE[1] // 4
    ow, oh = po.output_size(w, h, 0.75)
    cfg, ok = po.nis_config(False, 0, True, w, h, ow, oh, radius=2.0, sharpness=SHARP)
    assert ok
    res = {}
    for peak in (4.0, 1000.0):
        src = synth.natural_rgba16f(w, h, 5, peak=peak).astype(np.float32)
        # window max at texel i over i - 2 .. i + 3 (edge texels repeated: the sampler's clamp)
        wmax = np.stack([maximum_filter(src[..., c], size=6, origin=-1, mode="nearest") for c in range(3)], -1)
        fy = np.clip(np.floor((np.arange(oh) + 0.5) * (h / oh) - 0.5).astype(int), 0, h - 1)
        fx = np.clip(np.floor((np.arange(ow) + 0.5) * (w / ow) - 0.5).astype(int), 0, w - 1)
        bound = wmax[fy][:, fx]
        row = {"channels": int(ow * oh * 3)}
        for on in (False, True):
            s = src.copy()
            if on:
                s[..., :3] = so.srtm(s[..., :3])
            o = po.nis_scaler(np.ascontiguousarray(s), ow, oh, cfg, out_dtype=np.float32, nthreads=os.cpu_count() or 1)[..., :3]
            if on:
                o = so.srtm(o, inverse=True)
            row["on" if on else "off"] = {"above": int((o > bound).sum()), "above_1.5x": int((o > 1.5 * bound).sum()),
                                          "below_zero": int((o < 0).sum()), "max": float(o.max())}
        res[f"peak {peak:g}"] = row
        print(f"NVScaler overshoot, peak {peak:g}: {row}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--passes", type=int, default=30)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--only", choices=["fsr", "nis", "overshoot"])
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
    if args.only in (None, "overshoot"):
        out["nis_overshoot"] = nis_overshoot()
    if args.only in (None, "nis"):
        nis_arms(args, out, dev, main_s)
    for shape, (w, h, scale) in (SHAPES.items() if args.only in (None, "fsr") else ()):
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
