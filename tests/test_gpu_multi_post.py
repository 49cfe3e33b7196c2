"""Sharding of the ground-truth path tracer, TAA and the tone map (DESIGN.md §9): gathered N-rank results must be BIT-IDENTICAL to
the single-GPU result.

* test_path_tracer_linked_*: N ranks emulated on one GPU (one hr_ctx and one stream per rank) and linked with hr_shard_link_local:
  every rank traces the 8-row chunks c % world == rank of the whole image and pushes them into every peer's image, so every rank's
  FINAL is complete after its render.  The primary hit and path hash images are valid on the rank's own chunks.
* test_taa_tonemap_emulation: N ranks emulated with hr_shard_config only; every rank resolves / maps its band and the test moves the
  bands (what the gather does) through hr_pass_download / hr_pass_upload.
* test_nccl_post_chain_matches_single: one process per GPU (hr_shard_init), the whole frame chain; needs >= 2 GPUs.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import oracle as O  # noqa: F401  (path setup)
import pyhr
from test_gpu_multi import merge_bands
from test_textures_cpu import textured_scene

pytestmark = pytest.mark.gpu

SKY = (0.3, 0.4, 0.6)
HR_ERR_UNSUPPORTED = -5
PT_MODES = {"mode0": (0, 2), "indirect_B4": (1, 4)}  # (trace_indirect, max_ray_bounces)


def own_rows(H, rank, world):
    """rows of the 8-row chunks c with c % world == rank"""
    return np.array([y for y in range(H) if (y // 8) % world == rank], np.int64)


def pt_frame(i, W, H):
    return pyhr.make_frame((0.05 * i, 14.0, 34.0), (0.0, 3.0 - 0.1 * i, 0.0), W, H, num_frames=i)


def _pt_rank(scene, textures, W, H, ti, B, rank=0, world=1):
    c = pyhr.Context(0)
    s = c.build_scene(scene)
    if textures is not None:
        c.set_textures(s, *textures)
    if world > 1:
        c.shard_config(rank, world)
    p = pyhr.PathTracerPass(c, W, H)
    p.params.sky_color[0], p.params.sky_color[1], p.params.sky_color[2] = SKY
    p.params.trace_indirect, p.params.max_ray_bounces = ti, B
    return c, p


def _linked_pt(scene, textures, W, H, ti, B, world):
    ref = _pt_rank(scene, textures, W, H, ti, B)
    ranks = [_pt_rank(scene, textures, W, H, ti, B, r, world) for r in range(world)]
    for r in range(world):
        for q in range(world):
            if q != r:
                ranks[r][1].link_local(q, ranks[q][1])
    return ref, ranks


def _close(ref, ranks):
    for c, p in [ref] + ranks:
        p.destroy()
    for c, p in [ref] + ranks:
        c.close()


def run_linked_path_tracer(scene, textures, W, H, world, ti, B, n=8, reset_at=6):
    """n renders with a restart of the accumulation (hr_pass_reset_history on every rank) before render `reset_at`"""
    ref, ranks = _linked_pt(scene, textures, W, H, ti, B, world)
    streams = [torch.cuda.Stream() for _ in range(world)]
    for c, p in [ref] + ranks:
        p.stats()
    for i in range(n):
        if i == reset_at:
            for c, p in [ref] + ranks:
                p.reset_history()
        f = pt_frame(i, W, H)
        ref[1].render(f)
        for (c, p), st in zip(ranks, streams):
            p.render(f, st.cuda_stream)
        torch.cuda.synchronize()
        want, want_prim = ref[1].download(100), ref[1].download(1)
        want_hash = ref[1].download(2) if ti else None
        s_ref = ref[1].stats()
        assert s_ref.rays_primary == W * H
        primary, secondary = 0, 0
        for r, (c, p) in enumerate(ranks):
            what = f"world={world} rank {r} render {i}"
            assert np.array_equal(p.download(100), want), f"{what}: FINAL differs from the single-GPU image"
            rows = own_rows(H, r, world)
            assert np.array_equal(p.download(1)[rows], want_prim[rows]), f"{what}: primary hits differ on the own chunks"
            if ti:
                assert np.array_equal(p.download(2)[rows], want_hash[rows]), f"{what}: path hashes differ on the own chunks"
            s = p.stats()
            assert s.rays_primary == W * len(rows), f"{what}: {s.rays_primary} primary rays, own rows {len(rows)}"
            primary += s.rays_primary
            secondary += s.rays_secondary
        assert (primary, secondary) == (s_ref.rays_primary, s_ref.rays_secondary), f"world={world} render {i}: ray counts do not sum"
    _close(ref, ranks)


@pytest.fixture(scope="module")
def shadows_scene():
    return pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)


@pytest.mark.parametrize("mode", list(PT_MODES))
@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_path_tracer_linked_bit_identical(shadows_scene, world, mode):
    ti, B = PT_MODES[mode]
    run_linked_path_tracer(shadows_scene, None, 256, 144, world, ti, B)


@pytest.mark.parametrize("mode", list(PT_MODES))
def test_path_tracer_linked_textured(mode):
    """the TEX instantiations take the chunk mapping too"""
    sc, asc, textures, bindings = textured_scene()
    ti, B = PT_MODES[mode]
    run_linked_path_tracer(asc, (textures, bindings), 192, 112, 3, ti, B, n=4, reset_at=3)


@pytest.mark.parametrize("W,H,world", [(250, 141, 3), (64, 16, 3)], ids=["250x141_w3", "64x16_w3"])
def test_path_tracer_linked_edge_shapes(shadows_scene, W, H, world):
    """a ragged height, and more ranks than chunks: rank 2 of 64x16 owns no chunk and still publishes its tick (no rank times out)"""
    run_linked_path_tracer(shadows_scene, None, W, H, world, 1, 4, n=4, reset_at=3)


def test_path_tracer_odd_width_gather_refused(shadows_scene):
    """the chunk push copies texel pairs: an odd width is refused while the gather is on and changes nothing; with the gather off
    every rank traces its own chunks"""
    W, H, world = 251, 64, 2
    ref, ranks = _linked_pt(shadows_scene, None, W, H, 0, 2, world)
    f = pt_frame(0, W, H)
    for c, p in ranks:
        assert p.lib.hr_path_tracer_render(p.h, C.byref(f), C.byref(p.params), None) == HR_ERR_UNSUPPORTED
        with pytest.raises(pyhr.HrError):
            p.output(100)  # nothing was rendered
    for c, p in ranks:
        c.shard_set_gather(0)
    streams = [torch.cuda.Stream() for _ in range(world)]
    for i in range(2):
        f = pt_frame(i, W, H)
        ref[1].render(f)
        for (c, p), st in zip(ranks, streams):
            p.render(f, st.cuda_stream)
        torch.cuda.synchronize()
        want = ref[1].download(100)
        for r, (c, p) in enumerate(ranks):
            rows = own_rows(H, r, world)
            assert np.array_equal(p.download(100)[rows], want[rows]), f"rank {r} render {i}: own chunks differ"
    _close(ref, ranks)


# ---- TAA + tone map: bands on complete inputs ---------------------------------------------------------------------------------
TW, TH = 256, 144


def taa_frames(n, pan_from=2, vertical=0.35):
    """test_gpu_multi.frames with the TAA jitter applied (vertical pan: reprojected history taps cross band edges)"""
    f, prev_j = None, np.zeros(2, np.float32)
    for i in range(n):
        dx = 0.0 if i < pan_from else 0.05 * (i - pan_from + 1)
        dy = 0.0 if i < pan_from else vertical * (i - pan_from + 1)
        f = pyhr.make_frame((dx, 14.0 + dy, 34.0), (dx, 3.0 - dy, 0.0), TW, TH, prev=f, num_frames=i)
        j = pyhr.taa_jitter(i, TW, TH)
        pyhr.apply_jitter(f, j, prev_j)
        prev_j = j
        yield i, f


def _post_rank(sc, reset_every_frame, rank=0, world=1):
    c = pyhr.Context(0)
    c.set_bluenoise(*pyhr.blue_noise())
    c.build_scene(sc)
    c.gbuffer_create(TW, TH)
    if world > 1:
        c.shard_config(rank, world)
    de, taa, tm = pyhr.DeferredPass(c, TW, TH), pyhr.TAAPass(c, TW, TH), pyhr.TonemapPass(c, TW, TH)
    de.params.env_color[0], de.params.env_color[1], de.params.env_color[2] = SKY
    taa.params.reset_every_frame, taa.params.sharpen = reset_every_frame, 1
    return c, de, taa, tm


@pytest.mark.parametrize("reset_every_frame", [0, 1])
@pytest.mark.parametrize("world", [2, 3, 5])
def test_taa_tonemap_emulation(world, reset_every_frame):
    """The single-GPU deferred combine of shadows, AO, reflections and DDGI is the input.  Every rank holds it whole (the input pass's
    gather, restored with hr_pass_upload), resolves its band of TAA and maps its band; the merged bands equal the single-GPU TAA and
    tone-map images bit for bit every frame, and the merged TAA output is every rank's history of the next frame."""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ref = _post_rank(sc, reset_every_frame)
    rc = ref[0]
    sh, ao, rf, dd = pyhr.Pass(rc, "shadows", TW, TH, 0), pyhr.Pass(rc, "ao", TW, TH, 1), pyhr.ReflectionsPass(rc, TW, TH, 1), pyhr.DDGIPass(rc, TW, TH, 0)
    dd.params.probe_distance, dd.params.normal_bias = 4.0, 1.0
    for P in (dd.params, rf.params):
        P.sky_color[0], P.sky_color[1], P.sky_color[2] = SKY
    ranks = [_post_rank(sc, reset_every_frame, r, world) for r in range(world)]
    for i, f in taa_frames(7):
        g = pyhr.write_gbuffer(sc, f, TW, TH)
        rc.gbuffer_upload(f.ping_pong, g)
        sh.render(f)
        ao.render(f)
        dd.render(f, pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5)))
        rf.render(f, dd)
        ref[1].render(f, sh, ao, rf, dd)
        ref[2].render(f, ref[1])
        ref[3].render(ref[2])
        deferred = ref[1].download(100)
        for c, de, taa, tm in ranks:
            c.gbuffer_upload(f.ping_pong, g)
            de.render(f)
            de.upload(100, deferred)  # the gathered input
            taa.render(f, de)
            tm.render(taa)
        merged = merge_bands([r[2].download(100) for r in ranks], TH, world)
        assert np.array_equal(merged, ref[2].download(100)), f"TAA differs (world={world}, frame {i})"
        merged8 = merge_bands([r[3].download(100) for r in ranks], TH, world)
        assert np.array_equal(merged8, ref[3].download(100)), f"tone map differs (world={world}, frame {i})"
        for r in ranks:  # the TAA gather: next frame's history is complete on every rank
            r[2].upload(100, merged)
    # world > 1 without the gather: refused, the output is unchanged
    c, de, taa, tm = ranks[0]
    before = taa.download(100)
    c.shard_set_gather(0)
    assert taa.lib.hr_taa_render(taa.h, C.byref(f), C.byref(taa.params), de.h, None) == HR_ERR_UNSUPPORTED
    assert np.array_equal(taa.download(100), before)
    for p in (sh, ao, rf, dd):
        p.destroy()
    for c, de, taa, tm in [ref] + ranks:
        for p in (de, taa, tm):
            p.destroy()
        c.close()


# ---- one process per GPU: the whole frame chain ------------------------------------------------------------------------------------
def _chain(c, W, H):
    sh, ao, rf, dd = pyhr.Pass(c, "shadows", W, H, 0), pyhr.Pass(c, "ao", W, H, 1), pyhr.ReflectionsPass(c, W, H, 1), pyhr.DDGIPass(c, W, H, 0)
    de, taa, tm = pyhr.DeferredPass(c, W, H), pyhr.TAAPass(c, W, H), pyhr.TonemapPass(c, W, H)
    pt0, pt1 = pyhr.PathTracerPass(c, W, H), pyhr.PathTracerPass(c, W, H)
    dd.params.probe_distance, dd.params.normal_bias = 4.0, 1.0
    for P in (dd.params, rf.params, pt0.params, pt1.params):
        P.sky_color[0], P.sky_color[1], P.sky_color[2] = SKY
    de.params.env_color[0], de.params.env_color[1], de.params.env_color[2] = SKY
    taa.params.reset_every_frame = 0
    pt1.params.trace_indirect, pt1.params.max_ray_bounces = 1, 4
    return [sh, ao, rf, dd, de, taa, tm, pt0, pt1]


def _run_chain(c, sharded, W, H):
    P = _chain(c, W, H)
    sh, ao, rf, dd, de, taa, tm, pt0, pt1 = P
    outs = []
    for i, f in taa_frames(5):
        if sharded:
            c.gbuffer_render_sharded(f.ping_pong, f)
        else:
            c.gbuffer_render(f.ping_pong, f)
        sh.render(f)
        ao.render(f)
        dd.render(f, pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5)))
        rf.render(f, dd)
        de.render(f, sh, ao, rf, dd)
        taa.render(f, de)
        tm.render(taa)
        pt0.render(f)
        pt1.render(f)
        outs.append([p.download(100) for p in (de, taa, tm, pt0, pt1)])
    for p in P:
        p.destroy()
    return outs


def _nccl_chain_worker(rank, world, uid, result_dir):
    import torch
    torch.cuda.set_device(rank)
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    c = pyhr.Context(rank)
    c.set_bluenoise(*pyhr.blue_noise())
    c.build_scene(sc)
    c.gbuffer_create(TW, TH)
    c.shard_init(rank, world, uid)
    outs = _run_chain(c, True, TW, TH)
    np.savez(os.path.join(result_dir, f"chain{rank}.npz"), **{f"f{i}_{j}": a for i, o in enumerate(outs) for j, a in enumerate(o)})
    c.shard_shutdown()
    c.close()


def test_nccl_post_chain_matches_single(tmp_path):
    """sharded G-buffer, shadows, AO, DDGI, reflections, deferred, TAA, tone map and the path tracer in both modes: every rank's
    gathered finals equal the single-GPU images bit for bit"""
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    uid = pyhr.shard_unique_id()
    mp.spawn(_nccl_chain_worker, args=(world, uid, str(tmp_path)), nprocs=world, join=True)
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    c = pyhr.Context(0)
    c.set_bluenoise(*pyhr.blue_noise())
    c.build_scene(sc)
    c.gbuffer_create(TW, TH)
    ref = _run_chain(c, False, TW, TH)
    c.close()
    names = ("deferred", "TAA", "tone map", "path tracer mode 0", "path tracer indirect")
    for r in range(world):
        d = np.load(os.path.join(str(tmp_path), f"chain{r}.npz"))
        for i, o in enumerate(ref):
            for j, a in enumerate(o):
                assert np.array_equal(d[f"f{i}_{j}"], a), f"rank {r} frame {i}: {names[j]} differs from the single-GPU result"
