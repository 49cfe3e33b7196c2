"""DDGI cost on one GPU, this build against a baseline checkout: the stage times of the world-1 DDGI render (Ray Trace, Probe Update,
Sample Probe Grid) on the config-4 grid (arcade, 262 144 triangles, 4K, probe_distance 4.2: 16 x 8 x 32 = 4096 probes x 256 rays),
and `bench.py --config 4 --gpus 1` frames/s with the dumped final outputs compared between the two builds.

    python tools/bench_ddgi_sharded.py --baseline DIR [--rounds 2] [--frames 20] [--steps 20]

DIR is a built checkout of the commit to compare against.  The two builds run alternately, `rounds` times each, every run in a
process of its own; the GPU name and power limit are read in the same run.  Prints one JSON line.  Dumps go to a temporary directory.
The multi-GPU legs (the atlas store and wait per rank) need several GPUs and are not measured here.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def stage_times(root, frames):
    """one process: the DDGI pass of config 4 alone, profiled; mean ms per stage over `frames` renders after 3 untimed ones"""
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "hybrid-rendering_b200"))
    import torch
    import pyhr
    from bench import CAM_POS, CAM_TGT, LIGHT_ROT_X, SKY
    W, H = 3840, 2160
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    ctx.build_scene(pyhr.SynthScene(pyhr.SCENE_ARCADE, 262144))
    ctx.gbuffer_create(W, H)
    light = pyhr.default_light(rot_x_deg=LIGHT_ROT_X)
    f = pyhr.make_frame(CAM_POS, CAM_TGT, W, H, light=light)
    ctx.gbuffer_render(0, f)
    dd = pyhr.DDGIPass(ctx, W, H, 0)
    dd.params.probe_distance, dd.params.normal_bias = 4.2, 0.5
    for k in range(3):
        dd.params.sky_color[k] = SKY[k]
    for i in range(3):
        dd.render(f, pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5)))
    torch.cuda.synchronize()
    ctx.set_profiling(True)
    for i in range(frames):
        dd.render(f, pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5)))
    torch.cuda.synchronize()
    t = {k: round(v, 4) for k, v in dd.stage_times()}
    u = dd.uniforms()
    out = dict(stages_ms=t, probes=u.probe_counts[0] * u.probe_counts[1] * u.probe_counts[2], rays_per_probe=u.rays_per_probe)
    dd.destroy()
    ctx.close()
    return out


def bench_config4(root, steps, dump):
    cmd = [sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--config", "4", "--steps", str(steps), "--warmup", "5", "--no-cpu-baseline",
           "--no-extras", "--dump-outputs", dump]
    r = subprocess.run(cmd, cwd=root, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"{' '.join(cmd)} failed:\n{r.stdout[-3000:]}")
    return json.loads(lines[-1])


def same_dumps(a, b):
    import numpy as np
    names = sorted(n for n in os.listdir(a) if n.endswith(".npy"))
    if names != sorted(n for n in os.listdir(b) if n.endswith(".npy")):
        return False
    return all(np.array_equal(np.load(os.path.join(a, n)), np.load(os.path.join(b, n))) for n in names)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline", help="a built checkout of the commit to compare against")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--stage-times-of", metavar="ROOT", help=argparse.SUPPRESS)  # one measurement process
    args = ap.parse_args()
    if args.stage_times_of:
        print(json.dumps(stage_times(args.stage_times_of, args.frames)))
        return
    builds = {"this": ROOT, "baseline": os.path.abspath(args.baseline)} if args.baseline else {"this": ROOT}
    res = {"gpu": gpu_info(), "rounds": []}
    with tempfile.TemporaryDirectory() as tmp:
        for k in range(args.rounds):
            rnd = {}
            for name, root in builds.items():
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--stage-times-of", root, "--frames", str(args.frames)], stdout=subprocess.PIPE,
                                   stderr=subprocess.STDOUT, text=True)
                lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
                if r.returncode != 0 or not lines:
                    raise RuntimeError(f"stage times of {root} failed:\n{r.stdout[-3000:]}")
                dump = os.path.join(tmp, f"{name}{k}")
                b = bench_config4(root, args.steps, dump)
                rnd[name] = dict(json.loads(lines[-1]), config4=b)
                print(f"round {k} {name}: {rnd[name]['stages_ms']}, config 4 {b.get('value')} {b.get('unit')}", file=sys.stderr, flush=True)
            if "baseline" in builds:
                rnd["config4_outputs_identical"] = same_dumps(os.path.join(tmp, f"this{k}"), os.path.join(tmp, f"baseline{k}"))
            res["rounds"].append(rnd)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
