"""CPU, gloo world 2 / 3: the cooperative multi-sample (spp > 1) ray trace restated on the oracle (DESIGN.md §9).  Each rank traces an
arbitrary, frame-varying share of the count image's mask rows (4 image rows each) — what k_ray_trace_shared<MODE, true> does with the
cost-balanced partition — and the shares are exchanged so that every rank holds the complete count image (k_rt_push).  The
denoise stages then run on band +- halo with the history of each rank valid on its own band only; the result must equal the
whole-image oracle bit for bit.
"""
import os

import numpy as np
import pytest

import oracle as O
import pyhr
from test_sharding_cpu import _coop_bounds, _gather_bands, shard_rows

W, H = 256, 144


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
        tri, _ = sc.world_triangles()
        osc = O.Scene(tri, brute=True)
        bn = pyhr.blue_noise()
        ref_sh, ref_ao = O.ShadowsOracle(W, H, 0, spp=2), O.AOOracle(W, H, 1, spp=2)
        sh, ao = O.ShadowsOracle(W, H, 0, spp=2), O.AOOracle(W, H, 1, spp=2)
        sh.band = shard_rows(sh.H, rank, world)
        ao.band = shard_rows(ao.H, rank, world)
        L = O.lib()
        trace = {"sh": L.orc_shadows_ray_trace_spp, "ao": L.orc_ao_ray_trace_spp}
        state = {}

        def cooperative(name, o):
            """the oracle's whole-image trace, then only this rank's share of the mask rows kept, then the shares exchanged"""
            def run(*args):
                trace[name](*args)
                bd = state["bounds"]
                r0, r1 = 4 * bd[rank], min(4 * bd[rank + 1], o.H)
                rng = np.random.default_rng(7 * state["frame"] + rank)
                keep = o.count[r0:r1].copy()
                o.count[:] = rng.integers(0, 255, size=o.count.shape, dtype=np.uint8)  # rows of the other ranks: never traced here
                o.count[r0:r1] = keep
                for r in range(world):
                    a, b = 4 * bd[r], min(4 * bd[r + 1], o.H)
                    t = torch.from_numpy(np.ascontiguousarray(o.count[a:b]))
                    dist.broadcast(t, src=r)
                    o.count[a:b] = t.numpy()
            return run

        f, prev = None, O.zero_gbuf_mips(W, H)
        for i in range(5):
            dx = 0.0 if i < 2 else 0.08 * (i - 1)
            dy = 0.0 if i < 2 else 0.3 * (i - 1)  # vertical motion: history taps cross the band borders
            f = pyhr.make_frame((dx, 14 + dy, 34), (dx, 3 - dy, 0), W, H, prev=f, num_frames=i)
            cur = O.GBufMips(pyhr.write_gbuffer(sc, f, W, H))
            ref_sh.render(osc, cur, prev, f, bn)
            ref_ao.render(osc, cur, prev, f, bn)
            pp = f.ping_pong
            if i > 0:  # distributed history: rows owned by the peers are fetched from them before the reprojection
                sh.prev_image[:] = _gather_bands(dist, sh.prev_image, sh.H, rank, world)
                sh.moments[1 - pp][:] = _gather_bands(dist, sh.moments[1 - pp], sh.H, rank, world)
                ao.color[1 - pp][:] = _gather_bands(dist, ao.color[1 - pp], ao.H, rank, world)
                ao.length[1 - pp][:] = _gather_bands(dist, ao.length[1 - pp], ao.H, rank, world)
            state["frame"] = i
            for name, o, fn in (("sh", sh, "orc_shadows_ray_trace_spp"), ("ao", ao, "orc_ao_ray_trace_spp")):
                state["bounds"] = _coop_bounds((o.H + 3) // 4, world, i)
                setattr(L, fn, cooperative(name, o))
                try:
                    o.render(osc, cur, prev, f, bn)
                finally:
                    setattr(L, fn, trace[name])
            prev = cur
            if not (np.array_equal(sh.count, ref_sh.count) and np.array_equal(ao.count, ref_ao.count)):
                q.put(f"rank {rank} frame {i}: exchanged count image is not the complete count image")
                return
            for o, arrs in ((sh, (sh.prev_image, sh.moments[pp])), (ao, (ao.color[pp], ao.length[pp]))):
                for a in arrs:
                    o._poison(a, 0)  # a rank keeps the history of its own band only
            b0, b1 = sh.band
            a0, a1 = ao.band
            u0, u1 = a0 << 1, (ao.final.shape[0] if a1 >= ao.H else a1 << 1)
            checks = (("shadows final", sh.final[b0:b1], ref_sh.final[b0:b1]), ("prev_image", sh.prev_image[b0:b1], ref_sh.prev_image[b0:b1]),
                      ("moments", sh.moments[pp][b0:b1], ref_sh.moments[pp][b0:b1]), ("ao colour", ao.color[pp][a0:a1], ref_ao.color[pp][a0:a1]),
                      ("ao length", ao.length[pp][a0:a1], ref_ao.length[pp][a0:a1]), ("ao final", ao.final[u0:u1], ref_ao.final[u0:u1]))
            for name, a, b in checks:
                if not np.array_equal(a, b):
                    q.put(f"rank {rank} frame {i}: {name} (own band) differs from the unsharded result")
                    return
        q.put("ok")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_cooperative_count_trace_and_distributed_history_gloo(world):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 613) % 2000 + world
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p_ in procs:
        p_.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p_ in procs:
        p_.join(60)
    assert res == ["ok"] * world, res
