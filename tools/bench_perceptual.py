"""Dev bench: what OVRFSR_FLAG_PERCEPTUAL (P on every float texel read, P^-1 and the sRGB encode on every pixel stored)
costs on RGBA16F eyes, flag off against flag on, alternated window by window in one call, strict and fast math.

Workloads (synth.natural_rgba16f, linear light):
  C2       1683x1869 -> 2244x2492 (renderScale 0.75), FSR into RGBA8.  Off: the paired plan (EASU writes the outside
           groups, RCAS the inside ones); on: EASU into an RGBA16F intermediate, then RCAS (the SRTM plan).
  C3a      2244x2492 -> 2917x3239 (renderScale 1.3), the same two plans.
  C4       1512x1680, NVScaler at renderScale 0.75 and NVSharpen at renderScale 1, RGBA16F -> RGBA8.
Per launch: the stateless dispatch of each pass as the context runs it (off: no bits, EASU into RGBA8; on: EASU with
perceptual-in into RGBA16F, RCAS with perceptual-out from it; NIS with both), the median of --reps windows of
--launches launches (CUDA events).  pairs/s: PostProcessor.apply_pair with Config.perceptual off and on, and a third
arm, the float-output workaround: RGBA16F output without the flag.  Radius 2.0 (every group filtered) and 0.5 (the
reference default).  The card's name, power limit and SM clocks are read in the same call and printed with the
numbers.
usage: python tools/bench_perceptual.py [--only c2|c3a|c4] [--json out.json]"""
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


def run(args, out, dev, stream, name, w, h, scale, kind):
    import numpy as np
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import synth
    left = synth.natural_rgba16f(w, h, 1)
    right = np.ascontiguousarray(np.roll(left, 16, axis=1))
    tl, tr = ovr.to_image(left, dev), ovr.to_image(right, dev)
    ow, oh = ovr.output_size(w, h, scale)
    d8 = ovr.alloc_image(ow, oh, torch.uint8, dev)
    d16 = ovr.alloc_image(ow, oh, torch.float16, dev)
    for radius in (2.0, 0.5):
        base = dict(fsrEnabled=True, renderScale=scale, sharpness=SHARP, radius=radius, useNis=kind != "fsr")
        cfg = ovr.Config(**base)
        for mode, mm in (("strict", ovr.MATH_STRICT), ("fast", ovr.MATH_FAST)):
            tag = f"{name}/{kind}/r{radius}/{mode}"
            if kind == "fsr":
                uc = ovr.make_upscale_constants(cfg, 0, True, w, h, ow, oh)
                sc = ovr.make_sharpen_constants(cfg, 0, True, ow, oh)
                per = ab({"off": lambda: ovr.fsr_easu(tl, d8, uc, mm),
                          "on": lambda: ovr.fsr_easu(tl, d16, uc, mm, perceptual_in=True)}, args.launches, args.reps, stream)
                rc = ab({"off": lambda: ovr.fsr_rcas(d8, d8, sc, mm),
                         "on": lambda: ovr.fsr_rcas(d16, d8, sc, mm, perceptual_out=True)}, args.launches, args.reps, stream)
                out["per_launch_us"][f"{tag}/rcas"] = rc
            else:
                k, ok = ovr.make_nis_config(cfg, scale == 1.0, 0, True, w, h, ow, oh)
                assert ok
                fn = ovr.nis_scaler if scale != 1.0 else ovr.nis_sharpen
                per = ab({"off": lambda: fn(tl, d8, k, mm),
                          "on": lambda: fn(tl, d8, k, mm, perceptual_in=True, perceptual_out=True)}, args.launches, args.reps, stream)
            out["per_launch_us"][f"{tag}/{'easu' if kind == 'fsr' else kind}"] = per
            arms = {"off": dict(), "on": dict(perceptual=True), "rgba16f_out": dict(outputFormat=ovr.FORMAT_RGBA16F)}
            pps = {a: ovr.PostProcessor(ovr.Config(**base, mathMode=mm, **kw)) for a, kw in arms.items()}
            pair = ab({a: (lambda a=a: pps[a].apply_pair(tl, tr, stream=stream)) for a in arms}, args.passes, args.reps, stream)
            for pp in pps.values():
                pp.close()
            out["pairs_s"][tag] = {a: 1e6 / pair[a][0] for a in arms}
            line = f"{tag:26s} {'easu' if kind == 'fsr' else kind} off {per['off'][0]:7.1f} us on {per['on'][0]:7.1f} us " \
                   f"({per['on'][0] / per['off'][0] - 1:+.1%})"
            if kind == "fsr":
                line += f"  rcas off {rc['off'][0]:6.1f} on {rc['on'][0]:6.1f} us"
            line += "  pairs/s " + "  ".join(f"{a} {1e6 / pair[a][0]:5.0f}" for a in arms)
            print(line, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--passes", type=int, default=30)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--only", choices=["c2", "c3a", "c4"])
    ap.add_argument("--json")
    args = ap.parse_args()
    sys.path.insert(0, str(ROOT))
    import torch
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev)
    out = {"card_before": card(), "per_launch_us": {}, "pairs_s": {}}
    work = {
        "c2": [("C2", 1683, 1869, 0.75, "fsr")],
        "c3a": [("C3a", 2244, 2492, 1.3, "fsr")],
        "c4": [("C4", 1512, 1680, 0.75, "nis_scaler"), ("C4", 1512, 1680, 1.0, "nis_sharpen")],
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
