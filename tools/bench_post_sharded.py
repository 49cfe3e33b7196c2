"""Sharded post-processing and path tracer: path-tracer cost per sample (mode 0, and trace_indirect = 1 at max_ray_bounces 8) and
TAA + tone map per frame, at N = 1 and at the N GPUs of the run.

    torchrun --nproc-per-node N tools/bench_post_sharded.py [--width 3840 --height 2160 --tris 262144] [--samples 4] [--frames 20]
    python tools/bench_post_sharded.py          # N = 1 only

The scene, camera, light and sky are bench.py's config 3 (arcade, 262 144 triangles, 4K).  Rank 0 first runs the whole sequence on an
unsharded context (N = 1) while the other ranks wait; then every rank runs the same sequence sharded (hr_shard_init: the path tracer's
interleaved chunks with the push to the peers, TAA and tone map by bands with the NCCL gathers).  Every timing is CUDA events around
`samples` / `frames` renders after untimed warm-up ones.  After the timings the sequence restarts the accumulation and the TAA history
and renders a fixed number of frames; the device checksums of the gathered finals of every rank are printed against N = 1.  Prints one
JSON line (rank 0) with the GPU name and power limit read in the same run.  Writes nothing.
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


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def run(ctx, sc, W, H, args, stream, barrier):
    """the measured sequence; identical on every rank and at every N"""
    import torch
    import pyhr
    ctx.set_bluenoise(*pyhr.blue_noise())
    ctx.build_scene(sc)
    ctx.gbuffer_create(W, H)
    light = pyhr.default_light(rot_x_deg=LIGHT_ROT_X)
    f = pyhr.make_frame(CAM_POS, CAM_TGT, W, H, light=light)
    f = pyhr.make_frame(CAM_POS, CAM_TGT, W, H, prev=f, num_frames=1, light=light)
    j = pyhr.taa_jitter(1, W, H)
    f.ubo.current_prev_jitter[0], f.ubo.current_prev_jitter[1] = float(j[0]), float(j[1])
    ctx.gbuffer_render(0, f, 0, 0, stream)
    ctx.gbuffer_render(1, f, 0, 0, stream)
    de, taa, tm, pt = pyhr.DeferredPass(ctx, W, H), pyhr.TAAPass(ctx, W, H), pyhr.TonemapPass(ctx, W, H), pyhr.PathTracerPass(ctx, W, H)
    for k in range(3):
        de.params.env_color[k] = pt.params.sky_color[k] = SKY[k]
    taa.params.reset_every_frame = 0

    def timed(fn, n, warm):
        for _ in range(warm):
            fn()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return round(e0.elapsed_time(e1) / n, 4)

    out = {}
    de.render(f, None, None, None, None, stream)

    def post():
        taa.render(f, de, stream)
        tm.render(taa, stream)

    out["taa_tonemap_ms_per_frame"] = timed(post, args.frames, 3)
    for key, ti, B in (("path_tracer_mode0_ms_per_sample", 0, 2), ("path_tracer_indirect_B8_ms_per_sample", 1, 8)):
        pt.params.trace_indirect, pt.params.max_ray_bounces = ti, B
        pt.reset_history()
        out[key] = timed(lambda: pt.render(f, stream), args.samples, 2)
    # checksums: a fixed sequence after restarting the accumulation and the history
    pt.reset_history()
    for _ in range(3):
        pt.render(f, stream)
    taa.reset_history()
    for _ in range(3):
        post()
    out["checksums"] = {"path_tracer": pt.checksum(100, stream=stream), "taa": taa.checksum(100, stream=stream), "tonemap": tm.checksum(100, stream=stream)}
    torch.cuda.synchronize()
    for p in (de, taa, tm, pt):
        p.destroy()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--samples", type=int, default=4)
    ap.add_argument("--frames", type=int, default=20)
    args = ap.parse_args()
    import torch
    import pyhr
    if not torch.cuda.is_available():
        raise SystemExit("bench_post_sharded: no CUDA device")
    rank, world, local_rank = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))

    def barrier():
        if dist is not None:
            dist.barrier()

    W, H = args.width, args.height
    sc = pyhr.SynthScene(pyhr.SCENE_ARCADE, args.tris)
    stream = torch.cuda.current_stream().cuda_stream
    one = None
    if rank == 0:
        ctx = pyhr.Context(local_rank)
        one = run(ctx, sc, W, H, args, stream, lambda: None)
        ctx.close()
    barrier()
    line = {"gpu": gpu_info(), "width": W, "height": H, "triangles": args.tris, "samples": args.samples, "frames": args.frames, "n1": one}
    if world > 1:
        uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            uid.copy_(torch.frombuffer(bytearray(pyhr.shard_unique_id()), dtype=torch.uint8))
        dist.broadcast(uid, 0)
        ctx = pyhr.Context(local_rank)
        ctx.shard_init(rank, world, bytes(uid.cpu().numpy().tobytes()))
        mine = run(ctx, sc, W, H, args, stream, barrier)
        ctx.shard_shutdown()
        ctx.close()
        gathered = [None] * world
        dist.all_gather_object(gathered, mine)
        if rank == 0:
            line[f"n{world}"] = gathered[0]
            line["checksums_match_n1"] = all(g["checksums"] == one["checksums"] for g in gathered)
        dist.destroy_process_group()
    else:
        line["multi_gpu"] = "multi-GPU scaling not measured (one GPU)"
    if rank == 0:
        print(json.dumps(line))


if __name__ == "__main__":
    main()
