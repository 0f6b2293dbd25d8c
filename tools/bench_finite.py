"""Dev bench: what OVRFSR_FLAG_FINITE (finite-in on every float texel read, finite-out on every float pixel stored) costs
on RGBA16F eyes, flag off against flag on, alternated window by window in one call, strict and fast math.

Workloads (synth.natural_rgba16f, peak 4: finite content, so both arms compute the same pixels):
  C3a      2244x2492 -> 2917x3239 (renderScale 1.3), EASU + RCAS into RGBA8: the paired plan.  Per launch: the stateless
           EASU RGBA16F -> RGBA8 (on: finite-in and finite-out; RCAS reads the UNORM intermediate and gets no bits, so it
           is not timed).  Radius 2.0 (every group filtered) and 0.5 (the reference default).
  C3b      2915x3240 at renderScale 1, RCAS alone, RGBA16F out.  Per launch: the stateless RCAS RGBA16F -> RGBA16F
           (on: both bits).  Radius 2.0 and 0.5.
  C4       1512x1680, NVScaler at renderScale 0.75 and NVSharpen at renderScale 1, RGBA16F -> RGBA8.  Per launch: the
           stateless NIS dispatch (on: both bits).  Radius 2.0 and 0.5.
  pairs/s  PostProcessor.apply_pair of the same shape, radius and output with Config.finite off and on.
Per-launch times are the median of --reps windows of --launches launches (CUDA events); pairs/s the median of --reps
windows of --passes pairs.  The card's name, power limit and SM clocks are read in the same call and printed with the
numbers.
usage: python tools/bench_finite.py [--only c3a|c3b|c4] [--json out.json]"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
SHARP = 0.9


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def ab(fns, n, reps, stream):
    """{arm: (median, min, max) us per call}: the arms' windows alternate, so drift lands on both"""
    import torch
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(n):
                fn()
            e1.record(stream)
            torch.cuda.synchronize()
            ts[k].append(e0.elapsed_time(e1) * 1e3 / n)
    return {k: (statistics.median(v), min(v), max(v)) for k, v in ts.items()}


def run(args, out, dev, stream, name, w, h, scale, out_dtype, kind):
    import numpy as np
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    left = synth.natural_rgba16f(w, h, 1)
    right = np.ascontiguousarray(np.roll(left, 16, axis=1))
    tl, tr = ovr.to_image(left, dev), ovr.to_image(right, dev)
    ow, oh = ovr.output_size(w, h, scale)
    dst = ovr.alloc_image(ow, oh, out_dtype, dev)
    ofmt = {torch.uint8: ovr.FORMAT_AUTO, torch.float16: ovr.FORMAT_RGBA16F}[out_dtype]
    for radius in (2.0, 0.5):
        base = dict(fsrEnabled=True, renderScale=scale, sharpness=SHARP, radius=radius, outputFormat=ofmt, useNis=kind.startswith("nis"))
        cfg = ovr.Config(**base)
        if kind == "easu":
            k = ovr.make_upscale_constants(cfg, 0, True, w, h, ow, oh)
            fn = ovr.fsr_easu
        elif kind == "rcas":
            k = ovr.make_sharpen_constants(cfg, 0, True, ow, oh)
            fn = ovr.fsr_rcas
        else:
            k, ok = ovr.make_nis_config(cfg, scale == 1.0, 0, True, w, h, ow, oh)
            assert ok
            fn = ovr.nis_scaler if scale != 1.0 else ovr.nis_sharpen
        for mode, mm in (("strict", ovr.MATH_STRICT), ("fast", ovr.MATH_FAST)):
            tag = f"{name}/{kind}/r{radius}/{mode}"
            per = ab({on: (lambda on=on: fn(tl, dst, k, mm, finite_in=on, finite_out=on)) for on in (False, True)},
                     args.launches, args.reps, stream)
            pps = {on: ovr.PostProcessor(ovr.Config(**base, mathMode=mm, finite=on)) for on in (False, True)}
            pair = ab({on: (lambda on=on: pps[on].apply_pair(tl, tr, stream=stream)) for on in (False, True)},
                      args.passes, args.reps, stream)
            for pp in pps.values():
                pp.close()
            for on in (False, True):
                arm = f"{tag}/{'on' if on else 'off'}"
                out["per_launch_us"][arm] = per[on]
                out["pairs_s"][arm] = {"median": 1e6 / pair[on][0], "min": 1e6 / pair[on][2], "max": 1e6 / pair[on][1]}
            print(f"{tag:28s} {kind} off {per[False][0]:7.1f} us  on {per[True][0]:7.1f} us ({per[True][0] / per[False][0] - 1:+.1%})"
                  f"  apply_pair off {1e6 / pair[False][0]:6.0f}  on {1e6 / pair[True][0]:6.0f} pairs/s", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--passes", type=int, default=30)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--only", choices=["c3a", "c3b", "c4"])
    ap.add_argument("--json")
    args = ap.parse_args()
    sys.path.insert(0, str(ROOT))
    import torch
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev)
    out = {"card_before": card(), "per_launch_us": {}, "pairs_s": {}}
    work = {
        "c3a": [("C3a", 2244, 2492, 1.3, torch.uint8, "easu")],
        "c3b": [("C3b", 2915, 3240, 1.0, torch.float16, "rcas")],
        "c4": [("C4", 1512, 1680, 0.75, torch.uint8, "nis_scaler"), ("C4", 1512, 1680, 1.0, torch.uint8, "nis_sharpen")],
    }
    for key, items in work.items():
        if args.only in (None, key):
            for item in items:
                run(args, out, dev, stream, *item)
    out["card_after"] = card()
    print(f"card before: {out['card_before']}\ncard after:  {out['card_after']}")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
