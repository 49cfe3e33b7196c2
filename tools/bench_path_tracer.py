"""Ground-truth path tracer cost per sample, mode 0 (the reference as written) against trace_indirect = 1 at several max_ray_bounces.

    python tools/bench_path_tracer.py [--width 3840 --height 2160 --tris 262144] [--samples 8] [--warmup 3] [--rounds 2]

The scene, camera, light and sky are bench.py's config 3 (arcade, 262 144 triangles, 4K).  Every form renders `samples` progressive
samples after `warmup` untimed ones, timed with CUDA events; the forms are alternated over `rounds` rounds and each form's best round is
reported.  Rays are the pass's own counters (hr_pass_get_stats: primary + shadow + bounce rays).  Prints one JSON line with the GPU
name and power limit read in the same run.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "hybrid-rendering_b200"))

from bench import CAM_POS, CAM_TGT, LIGHT_ROT_X, SKY  # noqa: E402

FORMS = [(0, 2), (1, 1), (1, 2), (1, 4), (1, 8)]  # (trace_indirect, max_ray_bounces)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--samples", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    import pyhr
    if not torch.cuda.is_available():
        raise SystemExit("bench_path_tracer: no CUDA device")
    torch.cuda.set_device(0)
    W, H = args.width, args.height
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    sc = pyhr.SynthScene(pyhr.SCENE_ARCADE, args.tris)
    ctx.build_scene(sc)
    f = pyhr.make_frame(CAM_POS, CAM_TGT, W, H, light=pyhr.default_light(rot_x_deg=LIGHT_ROT_X))
    stream = torch.cuda.current_stream().cuda_stream
    pt = pyhr.PathTracerPass(ctx, W, H)
    for k in range(3):
        pt.params.sky_color[k] = SKY[k]
    best = {}
    for _ in range(args.rounds):
        for ti, B in FORMS:
            pt.params.trace_indirect, pt.params.max_ray_bounces = ti, B
            pt.reset_history()
            for _ in range(args.warmup):
                pt.render(f, stream)
            pt.stats(stream)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.samples):
                pt.render(f, stream)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.samples
            st = pt.stats(stream)
            rays = (st.rays_primary + st.rays_secondary) / args.samples
            key = f"mode{ti}_B{B}"
            if key not in best or ms < best[key]["ms_per_sample"]:
                best[key] = {"trace_indirect": ti, "max_ray_bounces": B, "ms_per_sample": round(ms, 4), "rays_per_sample": rays,
                             "mrays_per_s": round(rays / 1e6 / (ms / 1e3), 1)}
    pt.destroy()
    ctx.close()
    print(json.dumps({"gpu": gpu_info(), "width": W, "height": H, "triangles": args.tris, "samples": args.samples, "rounds": args.rounds,
                      "forms": list(best.values())}))


if __name__ == "__main__":
    main()
