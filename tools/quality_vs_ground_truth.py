"""How far the hybrid frame is from the ground truth: the deferred combine's FINAL output against the indirect path tracer's, compared on
the device with hr_image_compare.

    python tools/quality_vs_ground_truth.py [--width 1920 --height 1080 --tris 262144] [--samples 256 --bounces 2] [--frames 8]
                                            [--sweep reflections.filter_iterations=0,1,2,3,4] [--sweep shadows.filter_iterations=0,4]

The scene, camera, light and sky are bench.py's (arcade, the nave view).  The path tracer (trace_indirect = 1, max_ray_bounces =
--bounces) accumulates --samples renders once.  For each point of the sweeps (every combination of their values; no sweep: the default
parameters) the hybrid chain (device G-buffer, shadows, AO at half resolution, DDGI, reflections at half resolution, deferred with
the synthetic split-sum BRDF LUT, pyhr.brdf_lut, so that the reflections reach it) is created afresh and renders a static sequence of --frames frames; after each frame one JSON line gives mse, relmse, psnr and ssim of
the deferred output against the path tracer's, the wall time of the hr_image_compare call (CUDA events; it includes the call's
stream synchronisation) and the frame's stage times (hr_pass_stage_times).  A last line gives the compare kernels' device time
(torch.profiler, mean over 20 calls) and the path tracer's time per sample, with the GPU name and power limit read in the same run.
The numbers describe the bias and noise of this hybrid frame against this path tracer, quirks both reproduce included (DESIGN.md §6);
they are not a verdict on the reference.  Fails when there is no GPU.  Writes nothing.
"""
import argparse
import itertools
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "hybrid-rendering_b200"))

from bench import CAM_POS, CAM_TGT, LIGHT_ROT_X, SKY  # noqa: E402

PASSES = ("shadows", "ao", "ddgi", "reflections", "deferred")


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def parse_sweep(specs):
    """["pass.param=v1,v2", ...] -> [(pass, param, [values])]"""
    out = []
    for s in specs:
        key, vals = s.split("=", 1)
        p, name = key.split(".", 1)
        if p not in PASSES:
            raise SystemExit(f"--sweep {s}: pass must be one of {PASSES}")
        out.append((p, name, [float(v) if "." in v else int(v) for v in vals.split(",")]))
    return out


def hybrid_chain(pyhr, ctx, W, H, point):
    """fresh passes (a fresh DDGI pass too: hr_pass_reset_history does not restart its probe grid), bench.py's parameters, then the
    point's overrides"""
    P = {"shadows": pyhr.Pass(ctx, "shadows", W, H, 0), "ao": pyhr.Pass(ctx, "ao", W, H, 1), "ddgi": pyhr.DDGIPass(ctx, W, H, 0),
         "reflections": pyhr.ReflectionsPass(ctx, W, H, 1), "deferred": pyhr.DeferredPass(ctx, W, H)}
    P["ddgi"].params.probe_distance, P["ddgi"].params.normal_bias = 4.2, 0.5
    for k in range(3):
        P["ddgi"].params.sky_color[k] = P["reflections"].params.sky_color[k] = P["deferred"].params.env_color[k] = SKY[k]
    for (p, name), v in point.items():
        if not hasattr(P[p].params, name):
            raise SystemExit(f"--sweep: {p} has no parameter {name}")
        setattr(P[p].params, name, v)
    return P


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--samples", type=int, default=256, help="path tracer renders accumulated")
    ap.add_argument("--bounces", type=int, default=2, help="path tracer max_ray_bounces (trace_indirect = 1)")
    ap.add_argument("--frames", type=int, default=8, help="hybrid frames per sweep point (static camera)")
    ap.add_argument("--sweep", action="append", default=[], help="pass.param=v1,v2,... (repeatable; the points are all combinations)")
    args = ap.parse_args()
    sweeps = parse_sweep(args.sweep)
    import torch
    import pyhr
    if not torch.cuda.is_available():
        raise SystemExit("quality_vs_ground_truth: no CUDA device")
    torch.cuda.set_device(0)
    gpu = gpu_info()
    W, H = args.width, args.height
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    ctx.set_brdf_lut(pyhr.brdf_lut())  # without a LUT the deferred combine's indirect specular term, the reflections' share, is 0
    ctx.build_scene(pyhr.SynthScene(pyhr.SCENE_ARCADE, args.tris))
    ctx.gbuffer_create(W, H)
    ctx.set_profiling(True)
    stream = torch.cuda.current_stream().cuda_stream
    light = pyhr.default_light(rot_x_deg=LIGHT_ROT_X)

    pt = pyhr.PathTracerPass(ctx, W, H)
    pt.params.trace_indirect, pt.params.max_ray_bounces = 1, args.bounces
    for k in range(3):
        pt.params.sky_color[k] = SKY[k]
    f0 = pyhr.make_frame(CAM_POS, CAM_TGT, W, H, light=light)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.samples):
        pt.render(f0, stream)
    e1.record()
    torch.cuda.synchronize()
    pt_ms = e0.elapsed_time(e1) / args.samples
    pt.stage_times()

    points = [dict(zip([(p, n) for p, n, _ in sweeps], combo)) for combo in itertools.product(*[v for _, _, v in sweeps])]
    for point in points:
        P = hybrid_chain(pyhr, ctx, W, H, point)
        f = None
        for i in range(args.frames):
            f = pyhr.make_frame(CAM_POS, CAM_TGT, W, H, prev=f, num_frames=i, light=light)
            ctx.gbuffer_render(f.ping_pong, f, stream=stream)
            P["shadows"].render(f, stream)
            P["ao"].render(f, stream)
            P["ddgi"].render(f, pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5)), stream)
            P["reflections"].render(f, P["ddgi"], stream)
            P["deferred"].render(f, P["shadows"], P["ao"], P["reflections"], P["ddgi"], stream)
            stages = {k: dict(p.stage_times()) for k, p in P.items()}
            c0, c1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            c0.record()
            s = ctx.compare(P["deferred"], pt, stream=stream)
            c1.record()
            c1.synchronize()
            r = pyhr.compare_finish(s)
            print(json.dumps({"point": {f"{p}.{n}": v for (p, n), v in point.items()}, "frame": i, "mse": r.mse, "relmse": r.relmse,
                              "psnr": r.psnr, "ssim": r.ssim, "mean_abs": r.mean_abs, "max_abs": r.max_abs, "pixels": r.pixels,
                              "nonfinite_test": r.nonfinite_test, "nonfinite_ref": r.nonfinite_ref, "compare_call_us": round(c0.elapsed_time(c1) * 1e3, 1),
                              "stage_ms": {k: {n: round(v, 4) for n, v in st.items()} for k, st in stages.items()}}), flush=True)
        last = P["deferred"]
        if point is not points[-1]:
            for p in P.values():
                p.destroy()

    # the compare kernels' device time, in a profiled window of its own
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        ctx.compare(last, pt, stream=stream)
    torch.cuda.synchronize()
    n = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            ctx.compare(last, pt, stream=stream)
        torch.cuda.synchronize()
    durations = {}
    for e in prof.events():
        if "k_compare" in e.name and e.device_type == DeviceType.CUDA:
            durations.setdefault("k_compare_total" if "k_compare_total" in e.name else "k_compare", []).append(e.time_range.end - e.time_range.start)
    us = {k: float(np.mean(v)) for k, v in durations.items()}  # the profiler may drop a record: the mean over those it kept
    bytes_read = 2 * W * H * 8
    print(json.dumps({"gpu": gpu, "width": W, "height": H, "triangles": args.tris, "samples": args.samples, "bounces": args.bounces,
                      "path_tracer_ms_per_sample": round(pt_ms, 3), "compare_kernel_us": {k: round(v, 2) for k, v in us.items()},
                      "compare_kernels_recorded": {k: len(v) for k, v in durations.items()},
                      "compare_read_gb_per_s": round(bytes_read / (us.get("k_compare", float("nan")) * 1e-6) / 1e9, 1)}), flush=True)
    for p in P.values():
        p.destroy()
    pt.destroy()
    ctx.close()


if __name__ == "__main__":
    main()
