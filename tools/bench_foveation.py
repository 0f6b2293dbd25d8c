"""Dev bench: what a gaze-following radius mask (ovrfsr_set_focus, ovrfsr_set_focus_radius) costs and buys at C2
(stereo 1683x1869 -> 2244x2492 RGBA8, strict FSR EASU+RCAS, the bench.py scene).  Pairs/s with the focus off, set once
(static) and moved before every frame (moving), at radius 0.3, 0.5 and 2.0; and with a per-eye radius override equal
to the config radius, set once with no focus (radius_static), or changed before every frame -- both eyes alternating
0.3 / 0.5, out of phase -- with the focus moving too (radius_moving); and with a sharpness override
(ovrfsr_set_sharpness) and no focus or radius override, equal to the config sharpness and set once (sharp_static), or
alternated 0.9 / 0.6 before every frame (sharp_moving).  Two drivers:
  pair     : one caller stream, both eyes per PostProcessor.apply_pair call
  streams4 : two contexts (frames in flight), one stream per eye -- bench.py's default driver
Each arm is the median of --reps timed windows of --passes passes over a pool of 8 distinct pairs (CUDA events on
the caller stream, everything joined before the end event).  The focus cost per apply is the radius-2.0 difference
between 'static' and 'off' (at radius 2.0 every group is filtered whatever the centre, so only the copy differs).

A/B: --lib PATH (repeatable) runs each library in its own child process, alternated --rounds times; a library without
ovrfsr_set_focus (an older build) runs the 'off' arms only, one without ovrfsr_set_focus_radius skips the radius_* arms,
one without ovrfsr_set_sharpness the sharp_* arms.  The card's name, power limit and SM clock are read in the same
call and printed with the numbers.
usage: python tools/bench_foveation.py [--lib A.so --lib B.so] [--rounds 2] [--json out.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
IN_W, IN_H, SCALE, SHARP, POOL = 1683, 1869, 0.75, 0.9, 8
RADII = (0.3, 0.5, 2.0)
FOCUS = ("off", "static", "moving", "radius_static", "radius_moving", "sharp_static", "sharp_moving")
DRIVERS = ("pair", "streams4")


def gaze(i):
    """a saccade-like path over the central part of the eye texture: a new point every frame"""
    return 0.3 + 0.4 * ((i * 0.37) % 1.0), 0.3 + 0.4 * ((i * 0.61) % 1.0)


def child(args):
    sys.path.insert(0, str(ROOT))
    import numpy as np
    import torch
    import openvr_fsr_b200 as ovr
    from openvr_fsr_b200 import _lib as L, synth
    dev = torch.device("cuda:0")
    has_focus = hasattr(L.lib(), "ovrfsr_set_focus")
    has_radius = hasattr(L.lib(), "ovrfsr_set_focus_radius")
    has_sharp = hasattr(L.lib(), "ovrfsr_set_sharpness")
    base_l, base_r = synth.stereo_pair("natural", IN_W, IN_H, 1)
    pool = [(ovr.to_image(np.roll(base_l, 37 * i, axis=0), dev), ovr.to_image(np.roll(base_r, 37 * i, axis=0), dev))
            for i in range(POOL)]
    main = torch.cuda.current_stream(dev)
    res = {}
    for radius in RADII:
        for driver in DRIVERS:
            cfg = ovr.Config(fsrEnabled=True, renderScale=SCALE, sharpness=SHARP, radius=radius, mathMode=ovr.MATH_STRICT)
            n_ctx = 1 if driver == "pair" else 2
            pps = [ovr.PostProcessor(cfg) for _ in range(n_ctx)]
            streams = [[main, main]] if driver == "pair" else [[torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)] for _ in pps]
            for focus in FOCUS:
                if ((focus != "off" and not has_focus) or (focus.startswith("radius") and not has_radius) or
                        (focus.startswith("sharp") and not has_sharp)):
                    continue
                for p in pps:
                    if focus in ("off", "radius_static", "sharp_static", "sharp_moving") and has_focus:
                        p.clear_focus(0), p.clear_focus(1)
                    if focus.startswith("sharp"):
                        p.clear_focus_radius(0), p.clear_focus_radius(1)
                        p.set_sharpness(SHARP)
                    if focus == "static":
                        p.set_focus(0, 0.45, 0.55), p.set_focus(1, 0.55, 0.55)
                    elif focus == "radius_static":
                        p.set_focus_radius(0, radius), p.set_focus_radius(1, radius)

                def run(passes, frame0):
                    for s in (x for pair in streams for x in pair if x is not main):
                        s.wait_stream(main)
                    for i in range(frame0, frame0 + passes * POOL):
                        p, (sl, sr), (l, r) = pps[i % n_ctx], streams[i % n_ctx], pool[i % POOL]
                        if focus in ("moving", "radius_moving"):
                            p.set_focus(0, *gaze(i)), p.set_focus(1, *gaze(i + 1))
                        if focus == "radius_moving":
                            p.set_focus_radius(0, (0.3, 0.5)[i % 2]), p.set_focus_radius(1, (0.5, 0.3)[i % 2])
                        if focus == "sharp_moving":
                            p.set_sharpness((SHARP, 0.6)[i % 2])
                        if driver == "pair":
                            p.apply_pair(l, r, stream=sl)
                        else:
                            p.apply(0, l, stream=sl), p.apply(1, r, stream=sr)
                    for s in (x for pair in streams for x in pair if x is not main):
                        main.wait_stream(s)

                run(2, 0)  # warm-up: lazy init, module loads
                torch.cuda.synchronize()
                rates = []
                for rep in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(main)
                    run(args.passes, 1000 * (rep + 1))
                    e1.record(main)
                    torch.cuda.synchronize()
                    rates.append(args.passes * POOL / (e0.elapsed_time(e1) * 1e-3))
                res[f"{driver}/r{radius}/{focus}"] = {"pairs_s": statistics.median(rates), "min": min(rates), "max": max(rates)}
            for p in pps:
                p.close()
    print(json.dumps({"lib": os.environ.get("OVRFSR_LIB", "in-tree"), "has_focus": has_focus, "has_radius": has_radius,
                      "has_sharp": has_sharp, "arms": res}))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="libovrfsr.so to measure (repeatable); default the in-tree build")
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the libraries")
    ap.add_argument("--passes", type=int, default=8, help="passes over the 8-pair pool per timed window")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", help="write every child result and the card readings here")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    libs = args.lib or [str(ROOT / "openvr_fsr_b200" / "libovrfsr.so")]
    out = {"card_before": card(), "runs": []}
    for rnd in range(args.rounds):
        for lib in libs:
            r = subprocess.run([sys.executable, __file__, "--child", "--passes", str(args.passes), "--reps", str(args.reps)],
                               env={**os.environ, "OVRFSR_LIB": lib}, capture_output=True, text=True, check=True)
            run = json.loads(r.stdout.strip().splitlines()[-1])
            run["round"], run["card_after"] = rnd, card()
            out["runs"].append(run)
            print(f"round {rnd} {lib} ({run['card_after']})")
            for k, v in run["arms"].items():
                print(f"  {k:26s} {v['pairs_s']:8.0f} pairs/s  (min {v['min']:.0f}, max {v['max']:.0f})")
            a = run["arms"]
            for d in DRIVERS:
                if f"{d}/r2.0/static" in a:
                    per_apply_us = (1e6 / a[f"{d}/r2.0/static"]["pairs_s"] - 1e6 / a[f"{d}/r2.0/off"]["pairs_s"]) / 2
                    print(f"  {d}: focus cost per apply at radius 2.0 (static - off) {per_apply_us:+.2f} us")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
