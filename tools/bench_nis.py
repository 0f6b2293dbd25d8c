"""Dev/measurement tool: per-eye device time of the NIS alternate path at BASELINE.json configs[3] (C4: 1512x1680 ->
2016x2240, sharpness 0.9, NVScaler only) and of NVSharpen at 2016x2240.  CUDA events on the launch stream, no sync
inside the loop.  Both kernels skip the directional filters of pixels whose interpolated edge weights are all zero, so
their time depends on the CONTENT: measured on the natural scene (1-2 % of the texels carry an edge), the textured one
(about a third) and uniform noise (84 %: nothing to skip).  The *_ctx arms time the kernels of the ctx path, with and
without the latched block of ovrfsr_set_sharpness (torch.profiler, per launch).
usage: python tools/bench_nis.py [--math fast|strict]"""
import argparse, json, statistics, sys
from pathlib import Path
import numpy as np, torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import openvr_fsr_b200 as ovr
from openvr_fsr_b200 import synth

ap = argparse.ArgumentParser(); ap.add_argument("--math", default="strict"); ap.add_argument("--reps", type=int, default=20)
a = ap.parse_args()
mode = ovr.MATH_STRICT if a.math == "strict" else ovr.MATH_FAST
dev = torch.device("cuda:0")
iw, ih, scale = 1512, 1680, 0.75
ow, oh = ovr.output_size(iw, ih, scale)
out = {}
GEN = {"natural": synth.natural_rgba8, "textured": synth.textured_rgba8, "uniform": synth.uniform_rgba8}
for content, radius in (("natural", 2.0), ("natural", 0.5), ("textured", 2.0), ("uniform", 2.0), ("uniform", 0.5)):
    gen, sfx = GEN[content], ("" if content == "natural" else "_" + content)
    cfg = ovr.Config(fsrEnabled=True, useNis=True, renderScale=scale, sharpness=0.9, radius=radius)
    scfg, _ = ovr.make_nis_config(cfg, False, 0, True, iw, ih, ow, oh)
    shcfg, _ = ovr.make_nis_config(cfg, True, 0, True, ow, oh, ow, oh)
    pool = [ovr.to_image(np.roll(gen(iw, ih, 1), 31 * i, axis=0), dev) for i in range(8)]
    big = [ovr.to_image(np.roll(gen(ow, oh, 2), 31 * i, axis=0), dev) for i in range(4)]
    dst = ovr.alloc_image(ow, oh, torch.uint8, dev)
    for name, fn, srcs, c, nbytes in (("nvscaler", ovr.nis_scaler, pool, scfg, iw * ih * 4 + ow * oh * 4),
                                      ("nvsharpen", ovr.nis_sharpen, big, shcfg, 2 * ow * oh * 4)):
        for s in srcs: fn(s, dst, c, mode)
        torch.cuda.synchronize()
        marks = []
        for _ in range(a.reps):
            for s in srcs:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); fn(s, dst, c, mode); e1.record(); marks.append((e0, e1))
        torch.cuda.synchronize()
        ms = statistics.mean(x.elapsed_time(y) for x, y in marks[len(marks) // 4:])
        out[f"{name}_r{radius}{sfx}"] = {"ms_per_eye": ms, "GBps_algorithmic": nbytes / ms / 1e6, "eye_pairs_per_s_1gpu": 500.0 / ms}

# The ctx path with and without the latched block (a sharpness override equal to the config's makes the kernels read
# their mask and sharpness words from the block the apply's 64-byte copy refreshes): kernel time per launch from
# torch.profiler, so the copy itself is not counted.  Natural scene, radius 2.0 and 0.5.
def ctx_kernel_us(cfg, srcs, latched):
    pp = ovr.PostProcessor(cfg)
    if latched:
        pp.set_sharpness(cfg.sharpness)
    for s in srcs: pp.apply(0, s)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            for s in srcs: pp.apply(0, s)
        torch.cuda.synchronize()
    pp.close()
    times = [e.time_range.elapsed_us() for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "nis_" in e.name]
    return statistics.median(times), len(times)


for radius in (2.0, 0.5):
    for name, sc, srcs in (("nvscaler", scale, [ovr.to_image(np.roll(synth.natural_rgba8(iw, ih, 1), 31 * i, axis=0), dev) for i in range(8)]),
                           ("nvsharpen", 1.0, [ovr.to_image(np.roll(synth.natural_rgba8(ow, oh, 2), 31 * i, axis=0), dev) for i in range(4)])):
        cfg = ovr.Config(fsrEnabled=True, useNis=True, renderScale=sc, sharpness=0.9, radius=radius, mathMode=mode)
        for latched in (False, True):
            us, n = ctx_kernel_us(cfg, srcs, latched)
            out[f"{name}_ctx{'_latched' if latched else ''}_r{radius}"] = {"us_per_launch_median": us, "launches": n}
print(json.dumps({"workload": "C4 1512x1680->2016x2240 RGBA8 NIS sharpness 0.9", "math": a.math, **out}))
