"""Cooperative multi-sample (spp > 1) ray trace on linked ranks (DESIGN.md §9): every rank traces its cost-balanced share of the
WHOLE count image (shadows, AO) or its interleaved 8-row chunks (reflections) and pushes it to the peers, so each ray of a frame is
traced once.  Every output must stay BIT-IDENTICAL to the single-GPU result.

N ranks are emulated on one GPU (one hr_ctx per rank, hr_shard_config + hr_shard_link_local, one CUDA stream per rank: linked ranks
wait for each other inside a frame); test_nccl_* is the one-process-per-GPU run and needs >= 2 GPUs.
"""
import os
import re

import numpy as np
import pytest
import torch

import oracle as O  # noqa: F401  (path setup)
import pyhr
from test_gpu_multi import AO, H, SH, W, frames, merge_bands
from test_gpu_ragged import kernels_launched

pytestmark = pytest.mark.gpu

RF = dict(rt=0, temporal=1, atrous=2, moments=4, final=100)
SKY = (0.3, 0.4, 0.6)


def _ctx(sc, rank=0, world=1, W=W, H=H, textures=None):
    c = pyhr.Context(0)
    c.set_bluenoise(*pyhr.blue_noise())
    s = c.build_scene(sc)
    if textures is not None:
        c.set_textures(s, *textures)
    c.gbuffer_create(W, H)
    if world > 1:
        c.shard_config(rank, world)
    return c


def _link(passes):
    for r, p in enumerate(passes):
        for q, o in enumerate(passes):
            if q != r:
                p.link_local(q, o)


def _refl(c, scale, spp):
    p = pyhr.ReflectionsPass(c, W, H, scale)
    p.params.sky_color[0], p.params.sky_color[1], p.params.sky_color[2] = SKY
    p.params.spp = spp
    return p


def _ddgi(c):
    d = pyhr.DDGIPass(c, W, H, 0)
    d.params.probe_distance, d.params.normal_bias = 4.0, 1.0
    d.params.sky_color[0], d.params.sky_color[1], d.params.sky_color[2] = SKY
    return d


def _close(ctxs, passes):
    for p in passes:
        p.destroy()
    for c in ctxs:
        c.close()


class Group:
    """the world-1 reference and `world` linked emulated ranks of the shadows and AO passes"""

    def __init__(self, sc, world, sh_scale, ao_scale, spp, W=W, H=H):
        self.world, self.W, self.H = world, W, H
        self.ref = _ctx(sc, W=W, H=H)
        self.ctxs = [_ctx(sc, r, world, W, H) for r in range(world)]
        self.sh = [pyhr.Pass(c, "shadows", W, H, sh_scale) for c in [self.ref] + self.ctxs]
        self.ao = [pyhr.Pass(c, "ao", W, H, ao_scale) for c in [self.ref] + self.ctxs]
        for p in self.sh + self.ao:
            p.params.spp = spp
        _link(self.sh[1:])
        _link(self.ao[1:])
        self.streams = [torch.cuda.Stream() for _ in range(world)]

    def render(self, f, g, passes=("sh", "ao")):
        self.ref.gbuffer_upload(f.ping_pong, g)
        for c, st in zip(self.ctxs, self.streams):
            c.gbuffer_upload(f.ping_pong, g, st.cuda_stream)
        for name in passes:
            ps = getattr(self, name)
            ps[0].render(f)
            for p, st in zip(ps[1:], self.streams):
                p.render(f, st.cuda_stream)
        torch.cuda.synchronize()

    def close(self):
        _close([self.ref] + self.ctxs, self.sh + self.ao)


def _check_shadows_ao(g, f, sh_h, ao_h, sh_scale, ao_scale, what=""):
    tag = f"(world={g.world}, frame {f.num_frames}{what})"
    for name, ps in (("shadows", g.sh), ("ao", g.ao)):
        ref = ps[0].download(0)
        for r, p in enumerate(ps[1:]):  # the count image is complete on every rank, not only band +- the ray-trace halo
            assert np.array_equal(p.download(0), ref), f"{name} count image of rank {r} differs {tag}"
    for name, which, shift in (("prev", SH["prev"], 0), ("moments", SH["moments"], 0), ("temporal", SH["temporal"], 0), ("final", SH["final"], sh_scale)):
        merged = merge_bands([p.download(which) for p in g.sh[1:]], sh_h, g.world, shift if name == "final" else 0)
        assert np.array_equal(merged, g.sh[0].download(which)), f"shadows {name} differs {tag}"
    for name, which, shift in (("temporal", AO["temporal"], 0), ("length", AO["length"], 0), ("final", AO["final"], ao_scale)):
        merged = merge_bands([p.download(which) for p in g.ao[1:]], ao_h, g.world, shift if name == "final" else 0)
        assert np.array_equal(merged, g.ao[0].download(which)), f"ao {name} differs {tag}"


# 1366x768: count rows of 5464 bytes per mask row, not a multiple of 16, so the push copies a byte-wise head and tail
COUNT_CASES = [pytest.param(w, s, a, spp, W, H, id=f"{w}-{s}-{a}-{spp}") for w in (2, 5, 8) for s, a in ((0, 1), (0, 0), (1, 1)) for spp in (2, 4)]
COUNT_CASES += [pytest.param(w, 0, 0, 2, 1366, 768, id=f"1366x768-{w}") for w in (3, 8)]


@pytest.mark.parametrize("world,sh_scale,ao_scale,spp,W,H", COUNT_CASES)
def test_count_image_cooperative_trace_bit_identical(world, sh_scale, ao_scale, spp, W, H):
    """shadows + AO at spp > 1 on linked ranks, vertical pan (reprojection crosses band edges): complete count image on every rank,
    merged bands of prev_image / moments / temporal / history length / final equal to world 1 over 8 frames"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    g = Group(sc, world, sh_scale, ao_scale, spp, W, H)
    try:
        for f in frames(8, pan_from=2, vertical=0.35, W=W, H=H):
            g.render(f, pyhr.write_gbuffer(sc, f, W, H))
            _check_shadows_ao(g, f, H >> sh_scale, H >> ao_scale, sh_scale, ao_scale)
    finally:
        g.close()


@pytest.mark.parametrize("spp", [2, 4])
@pytest.mark.parametrize("world", [3, 8])
def test_no_ray_traced_twice(world, spp):
    """per frame and pass, the primary (and, for reflections, secondary) rays of all ranks add up to the world-1 count: no halo row
    is traced on two ranks"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    g = Group(sc, world, 0, 1, spp)
    rf = [_refl(c, 1, spp) for c in [g.ref] + g.ctxs]
    _link(rf[1:])
    try:
        for f in frames(5, pan_from=2, vertical=0.35):
            gb = pyhr.write_gbuffer(sc, f, W, H)
            g.render(f, gb)
            for p, st in zip([rf[0]] + rf[1:], [None] + g.streams):
                p.render(f, None, st.cuda_stream if st else 0)
            torch.cuda.synchronize()
            for name, ps, fields in (("shadows", g.sh, ("rays_primary",)), ("ao", g.ao, ("rays_primary",)), ("reflections", rf, ("rays_primary", "rays_secondary"))):
                stats = [p.stats() for p in ps]
                for fld in fields:
                    want, got = getattr(stats[0], fld), sum(getattr(s, fld) for s in stats[1:])
                    assert want > 0 and got == want, f"{name} {fld}: ranks traced {got}, world 1 traced {want} (world={world}, frame {f.num_frames})"
    finally:
        _close([], rf)
        g.close()


REFL_CASES = [(w, s, spp, None) for w in (2, 3, 8) for s in (0, 1) for spp in (2, 4)] + [(3, 1, 2, "ddgi"), (3, 0, 2, "textures"), (8, 1, 4, "textures")]


@pytest.mark.parametrize("world,scale,spp,extra", REFL_CASES)
def test_reflections_spp_cooperative_trace_bit_identical(world, scale, spp, extra):
    """reflections at spp > 1 on linked ranks (interleaved chunks of the multi-sample K12): each rank's band of every stage and the
    merged final output equal world 1; one case reads a DDGI atlas, two run the textured (TEX) multi-sample instantiation"""
    if extra == "textures":
        from test_textures_cpu import textured_scene
        _, sc, textures, bindings = textured_scene()
        tex = (textures, bindings)
    else:
        sc, tex = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST), None
    ctxs = [_ctx(sc, textures=tex)] + [_ctx(sc, r, world, textures=tex) for r in range(world)]
    rf = [_refl(c, scale, spp) for c in ctxs]
    dd = [_ddgi(c) for c in ctxs] if extra == "ddgi" else [None] * len(ctxs)
    _link(rf[1:])
    streams = [None] + [torch.cuda.Stream() for _ in range(world)]
    ph = H >> scale
    try:
        for i, f in enumerate(frames(7, pan_from=2, vertical=0.35)):
            for c, p, d, st in zip(ctxs, rf, dd, streams):
                s = st.cuda_stream if st else 0
                c.gbuffer_render(f.ping_pong, f, stream=s)
                if d is not None:
                    d.render(f, pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5)), s)
                p.render(f, d, s)
            torch.cuda.synchronize()
            for name, which, shift in (("ray trace", RF["rt"], 0), ("temporal", RF["temporal"], 0), ("moments", RF["moments"], 0), ("a-trous", RF["atrous"], 0),
                                       ("final", RF["final"], scale)):
                merged = merge_bands([p.download(which) for p in rf[1:]], ph, world, shift if name == "final" else 0)
                assert np.array_equal(merged, rf[0].download(which)), f"reflections {name} differs (world={world}, spp={spp}, frame {f.num_frames})"
    finally:
        _close(ctxs, rf + [d for d in dd if d is not None])


@pytest.mark.parametrize("world", [3, 5])
def test_spp_changes_on_linked_ranks(world):
    """spp 1, 2, 4, 1, 2 on consecutive frames of linked ranks: the mask / count image is complete on every rank and every pass's
    merged outputs equal world 1 on every frame"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    g = Group(sc, world, 0, 1, 1)
    rf = [_refl(c, 1, 1) for c in [g.ref] + g.ctxs]
    _link(rf[1:])
    try:
        for spp, f in zip((1, 2, 4, 1, 2), frames(5, pan_from=1, vertical=0.35)):
            for p in g.sh + g.ao + rf:
                p.params.spp = spp
            g.render(f, pyhr.write_gbuffer(sc, f, W, H))
            for p, st in zip(rf, [None] + g.streams):
                p.render(f, None, st.cuda_stream if st else 0)
            torch.cuda.synchronize()
            _check_shadows_ao(g, f, H, H >> 1, 0, 1, f", spp={spp}")
            for name, which, shift in (("ray trace", RF["rt"], 0), ("temporal", RF["temporal"], 0), ("final", RF["final"], 1)):
                merged = merge_bands([p.download(which) for p in rf[1:]], H >> 1, world, shift if name == "final" else 0)
                assert np.array_equal(merged, rf[0].download(which)), f"reflections {name} differs (world={world}, spp={spp}, frame {f.num_frames})"
    finally:
        _close([], rf)
        g.close()


@pytest.mark.parametrize("world", [3, 8])
def test_spp_without_denoise_count_image_complete(world):
    """denoise = 0 at spp 2: the final output is the count image, complete and equal to world 1 on every rank"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    g = Group(sc, world, 0, 1, 2)
    for p in g.sh + g.ao:
        p.params.denoise = 0
    try:
        for f in frames(4, pan_from=1, vertical=0.35):
            g.render(f, pyhr.write_gbuffer(sc, f, W, H))
            for name, ps in (("shadows", g.sh), ("ao", g.ao)):
                ref = ps[0].download(100)
                assert ref.dtype == np.uint8 and ref.max() > 0
                for r, p in enumerate(ps[1:]):
                    assert np.array_equal(p.download(100), ref), f"{name} final (count image) of rank {r} differs (world={world}, frame {f.num_frames})"
    finally:
        g.close()


def test_cost_balancing_above_1024_mask_rows():
    """64 x 4320 (1080 mask rows), the lower half of the rows almost all sky: after the first frame's uniform split the partition
    follows the measured cost.  The uniform split hands the sky rank ~7 % of the traced rays; balanced on cost, each rank traces
    a large share.  The bar is 25 %: a sky warp costs a few cycles against thousands for a traced one, so balancing the cost gives
    each rank close to half the rays."""
    TW, TH = 64, 4320
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    g = Group(sc, 2, 0, 0, 2, TW, TH)
    try:
        f = None
        for i in range(4):
            f = pyhr.make_frame((0.0, 10.0, 34.0), (0.0, 6.0, 0.0), TW, TH, prev=f, num_frames=i)
            g.render(f, pyhr.write_gbuffer(sc, f, TW, TH), passes=("sh",))
            for name, which in (("count", 0), ("final", 100)):
                ref = g.sh[0].download(which)
                for r, p in enumerate(g.sh[1:]):
                    got = p.download(which)
                    if name == "final":
                        b, e = pyhr.shard_rows(TH, r, 2)
                        got, ref_r = got[b:e], ref[b:e]
                    else:
                        ref_r = ref
                    assert np.array_equal(got, ref_r), f"{name} of rank {r} differs (frame {i})"
            rays = [p.stats().rays_primary for p in g.sh]
            assert sum(rays[1:]) == rays[0]
            share = min(rays[1:]) / rays[0]
            if i == 0:
                assert share < 0.15, f"frame 0 (uniform split): the sky rank traced {share:.1%} of the rays — the scene does not test balancing"
            else:
                assert share >= 0.25, f"frame {i}: a rank traced only {share:.1%} of the rays (cost balancing not effective above 1024 mask rows)"
    finally:
        g.close()


@pytest.mark.parametrize("kind", ["shadows", "ao", "reflections"])
def test_launch_count_linked_spp2_trace_kernel(kind):
    """hr_ctx_launch_count over a linked spp = 2 pair equals the kernels torch.profiler records, and the ray trace among them is
    the cooperative multi-sample one"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctxs = [_ctx(sc, r, 2) for r in range(2)]
    if kind == "reflections":
        ps = [_refl(c, 1, 2) for c in ctxs]
    else:
        ps = [pyhr.Pass(c, kind, W, H, 0 if kind == "shadows" else 1) for c in ctxs]
        for p in ps:
            p.params.spp = 2
    _link(ps)
    streams = [torch.cuda.Stream() for _ in range(2)]
    fr = list(frames(12, pan_from=1, vertical=0.35))
    gbs = [pyhr.write_gbuffer(sc, f, W, H) for f in fr]
    state = {"i": 0, "launches": 0}

    def one():  # one frame of the pair (kernels_launched may run it more than once: each call renders the next frame)
        i = state["i"]
        state["i"] += 1
        before = sum(c.launch_count() for c in ctxs)
        for c, st in zip(ctxs, streams):
            c.gbuffer_upload(fr[i].ping_pong, gbs[i], st.cuda_stream)  # + the mip build
        torch.cuda.synchronize()
        for p, st in zip(ps, streams):
            if kind == "reflections":
                p.render(fr[i], None, st.cuda_stream)
            else:
                p.render(fr[i], st.cuda_stream)
        state["launches"] = sum(c.launch_count() for c in ctxs) - before
        torch.cuda.synchronize()

    try:
        one()  # first frame: history clears, peer mapping
        names = kernels_launched(one)
        assert len(names) == state["launches"], f"{kind}: {state['launches']} launches counted, {len(names)} kernels recorded: {names}"
        # shadows / AO: the cooperative trace in its count form, k_ray_trace_shared<MODE, true> however the name is (de)mangled
        coop = r"k_ray_trace_shared(<[^,>]*, ?(true|\(bool\)1)>|ILi\dELb1E)" if kind != "reflections" else "reflections_ray_trace"
        assert any(re.search(coop, n) for n in names), names
    finally:
        _close(ctxs, ps)


def _nccl_worker(rank, world, uid, result_dir):
    import torch
    torch.cuda.set_device(rank)
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    c = pyhr.Context(rank)
    c.set_bluenoise(*pyhr.blue_noise())
    c.build_scene(sc)
    c.gbuffer_create(W, H)
    c.shard_init(rank, world, uid)
    sh, ao, rf = pyhr.Pass(c, "shadows", W, H, 0), pyhr.Pass(c, "ao", W, H, 1), _refl(c, 1, 2)
    sh.params.spp = ao.params.spp = 2
    outs = []
    for f in frames(6, vertical=0.35):
        c.gbuffer_render(f.ping_pong, f)
        sh.render(f)
        ao.render(f)
        rf.render(f, None)
        outs.append((sh.download(0), sh.download(100), ao.download(100), rf.download(100), sh.download(SH["prev"]), ao.download(AO["temporal"]),
                     rf.download(RF["temporal"])))
    np.savez(os.path.join(result_dir, f"rank{rank}.npz"), **{f"f{i}_{j}": a for i, o in enumerate(outs) for j, a in enumerate(o)})
    for p in (sh, ao, rf):
        p.destroy()
    c.shard_shutdown()
    c.close()


def test_nccl_spp2_matches_single(tmp_path):
    """one process per GPU, shadows + AO + reflections at spp 2: count image and gathered final outputs complete and equal to world 1 on
    every rank, history bands equal"""
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    uid = pyhr.shard_unique_id()
    mp.spawn(_nccl_worker, args=(world, uid, str(tmp_path)), nprocs=world, join=True)
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    c = _ctx(sc)
    sh, ao, rf = pyhr.Pass(c, "shadows", W, H, 0), pyhr.Pass(c, "ao", W, H, 1), _refl(c, 1, 2)
    sh.params.spp = ao.params.spp = 2
    ref = []
    for f in frames(6, vertical=0.35):
        c.gbuffer_render(f.ping_pong, f)
        sh.render(f)
        ao.render(f)
        rf.render(f, None)
        ref.append((sh.download(0), sh.download(100), ao.download(100), rf.download(100), sh.download(SH["prev"]), ao.download(AO["temporal"]),
                    rf.download(RF["temporal"])))
    band_h = {4: H, 5: H >> 1, 6: H >> 1}  # history images stay distributed: each rank holds its own band
    for r in range(world):
        d = np.load(os.path.join(str(tmp_path), f"rank{r}.npz"))
        for i, o in enumerate(ref):
            for j, a in enumerate(o):
                got = d[f"f{i}_{j}"]
                if j in band_h:
                    b, e = pyhr.shard_rows(band_h[j], r, world)
                    assert np.array_equal(got[b:e], a[b:e]), f"rank {r} frame {i} image {j}: own band differs from the single-GPU result"
                else:
                    assert np.array_equal(got, a), f"rank {r} frame {i} image {j} differs from the single-GPU result"
    _close([c], [sh, ao, rf])
