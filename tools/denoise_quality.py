"""How close each denoise chain's FINAL output is to a converged reference of its own signal (hr_reference_render), compared on the
device with hr_image_compare.

    python tools/denoise_quality.py [--width 1920 --height 1080 --tris 262144] [--samples 1024] [--frames 16] [--effects shadows,ao,reflections]

The scene, camera, light and sky are bench.py's (arcade, the nave view), with a static camera.  For each effect and each case of the
sweeps (filter_iterations 0..4 for shadows and reflections, spp 1 / 2 / 4, scale FULL / HALF; every other parameter at its default,
shadows and reflections at FULL and AO at HALF) a fresh pass renders --frames frames.  After frame 2, every later power of two and the
last frame (the reflections' GI terms are off on the first frame), the reference is restarted and rendered with --samples rays per pixel
of that frame's signal (for reflections: with the DDGI atlas of that frame), and one JSON line gives mse, psnr and ssim of FINAL against
it and the reference's noise floor: the mean of STDERR^2 over the image.  A row whose floor is not at least 10x below the measured mse is not
reported: its "mse" and the other metrics are null and "refused" says why.  A last line gives each reference kernel's rays per second
(CUDA events around the render, rays from hr_pass_get_stats) with the GPU name and power limit read in the same run.  A shadows FINAL at
full resolution is RG16F: its r channel is copied into an R16F image first.  Fails when there is no GPU.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "hybrid-rendering_b200"))

from bench import CAM_POS, CAM_TGT, LIGHT_ROT_X, SKY  # noqa: E402

BENCH_SCALE = {"shadows": 0, "ao": 1, "reflections": 0}


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def cases(effect):
    out = [{"filter_iterations": i} for i in range(5)] if effect != "ao" else []
    out += [{"spp": s} for s in (1, 2, 4)]
    out += [{"scale": s} for s in (0, 1)]
    return out


def checkpoints(frames):
    c, k = {frames}, 2
    while k <= frames:
        c.add(k)
        k *= 2
    return sorted(x for x in c if x <= frames)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--samples", type=int, default=1024, help="reference rays per pixel")
    ap.add_argument("--frames", type=int, default=16, help="frames of the denoise chain (history length)")
    ap.add_argument("--effects", default="shadows,ao,reflections")
    args = ap.parse_args()
    import torch
    import pyhr
    if not torch.cuda.is_available():
        raise SystemExit("denoise_quality: no CUDA device")
    torch.cuda.set_device(0)
    gpu = gpu_info()
    W, H = args.width, args.height
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    ctx.build_scene(pyhr.SynthScene(pyhr.SCENE_ARCADE, args.tris))
    ctx.gbuffer_create(W, H)
    stream = torch.cuda.current_stream().cuda_stream
    light = pyhr.default_light(rot_x_deg=LIGHT_ROT_X)
    rates = {}
    for effect in args.effects.split(","):
        for case in cases(effect):
            scale = case.get("scale", BENCH_SCALE[effect])
            ddgi = None
            if effect == "reflections":
                tgt = pyhr.ReflectionsPass(ctx, W, H, scale)
                ddgi = pyhr.DDGIPass(ctx, W, H, 0)
                ddgi.params.probe_distance, ddgi.params.normal_bias = 4.2, 0.5
                for k in range(3):
                    tgt.params.sky_color[k] = ddgi.params.sky_color[k] = SKY[k]
            else:
                tgt = pyhr.Pass(ctx, effect, W, H, scale)
            for k, v in case.items():
                if k != "scale":
                    setattr(tgt.params, k, v)
            ref = pyhr.ReferencePass(tgt)
            f = None
            for i in range(args.frames):
                f = pyhr.make_frame(CAM_POS, CAM_TGT, W, H, prev=f, num_frames=i, light=light)
                ctx.gbuffer_render(f.ping_pong, f, stream=stream)
                if ddgi:
                    ddgi.render(f, pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5)), stream)
                tgt.render(f, ddgi, stream) if ddgi else tgt.render(f, stream)
                if i + 1 not in checkpoints(args.frames):
                    continue
                # a reference of this frame's signal: the reflections' DDGI terms read the atlas DDGI wrote this frame, which changes from
                # frame to frame, so the reference restarts and is rendered again at every checkpoint
                ref.reset_history()
                ref.stats(stream)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                left = args.samples
                while left:
                    n = min(left, 256)
                    ref.render(f, n, ddgi=ddgi, stream=stream)
                    left -= n
                e1.record()
                e1.synchronize()
                st = ref.stats(stream)
                rates.setdefault(effect, []).append((st.rays_primary + st.rays_secondary) / (e0.elapsed_time(e1) * 1e-3))
                se = ref.download(pyhr.REFERENCE_OUT_STDERR).view(np.float16).astype(np.float64)
                floor = float(np.mean((se[..., :3] if se.ndim == 3 else se) ** 2))
                test = tgt.output(100)
                keep = None
                if effect == "shadows" and test.format != ref.output(pyhr.REFERENCE_OUT_MEAN).format:
                    a = tgt.download(100).view(np.float16)[..., 0].copy()  # RG16F (visibility, variance): the visibility alone
                    keep = torch.from_numpy(a.view(np.int16)).cuda()
                    test = pyhr.hr_image(keep.data_ptr(), W, H, ref.output(pyhr.REFERENCE_OUT_MEAN).format)
                r = pyhr.compare_finish(ctx.compare(test, ref, stream=stream))
                row = {"effect": effect, "case": case, "scale": scale, "frames": i + 1, "samples": args.samples, "noise_floor": floor}
                if not floor * 10 <= r.mse:
                    row.update({"mse": None, "psnr": None, "ssim": None, "refused": f"noise floor {floor:.3g} is not 10x below mse {r.mse:.3g}"})
                else:
                    row.update({"mse": r.mse, "psnr": r.psnr, "ssim": r.ssim})
                print(json.dumps(row), flush=True)
                del keep
            for p in (ref, tgt) + ((ddgi,) if ddgi else ()):
                p.destroy()
    print(json.dumps({"gpu": gpu, "width": W, "height": H, "triangles": args.tris, "samples": args.samples,
                      "reference_rays_per_s": {k: float(np.median(v)) for k, v in rates.items()}}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
