"""BVH traversal on the GPU against the oracle's brute-force loop, on adversarial geometry and rays (bvh_cases.py).

The bit-exact claim of every ray-traced pass rests on the box test being conservative: whatever the tree, a box that holds a
triangle the ray hits in (t_min, t_max) must be entered.  These tests check that claim directly with hr_trace_any /
hr_trace_closest (any flag, t, primitive and barycentrics compared bit for bit) under both tree builders, through the
packet walk of the G-buffer producer and through the shadows / AO ray-trace kernels.
"""
import numpy as np
import pytest

import bvh_cases as B
import oracle as O
import pyhr
from bvh_gpu import SoupShading, array_scene, bad_entries, build, chain_rays, check_scene, compare, gpu_trace, switches

pytestmark = pytest.mark.gpu

TOPOLOGIES = {"ploc": 1, "karras": 0}  # hr_debug_set(3, q)
HR_ERR_UNSUPPORTED = -5


@pytest.fixture(scope="module")
def ctx():
    c = pyhr.Context(0)
    c.set_bluenoise(*pyhr.blue_noise())
    yield c
    c.close()


# ---------------------------------------------------------------------------------------------- hr_trace_* against brute force
@pytest.mark.parametrize("topology", sorted(TOPOLOGIES))
@pytest.mark.parametrize("scene", sorted(B.SCENES))
def test_trace_matches_bruteforce(ctx, scene, topology):
    tri = B.SCENES[scene]()
    with switches(ctx.lib, k3=TOPOLOGIES[topology]):
        report, hits = check_scene(ctx, tri)
    assert hits > 0
    assert not bad_entries(report), f"{scene} / {topology}: rays that differ from brute force (any, closest) per family: {bad_entries(report)}"


@pytest.mark.parametrize("topology", sorted(TOPOLOGIES))
def test_chain_at_the_depth_limit(ctx, topology):
    n = B.MAX_DEPTH + 1
    tri = B.chain(n)
    with switches(ctx.lib, k3=TOPOLOGIES[topology]):
        rc, h, _ = build(ctx, tri)
        ctx.check(rc, "hr_scene_build")
        try:
            depth = ctx.scene_info(h).depth
            if topology == "ploc":
                assert depth == B.MAX_DEPTH, "PLOC builds the chain one merge per level"
            assert depth <= B.MAX_DEPTH
            ctx.check(ctx.lib.hr_scene_set_current(ctx.h, h), "hr_scene_set_current")
            rays, x = chain_rays(n)
            a, t, p, uv = gpu_trace(ctx, rays)
            assert np.array_equal(p, np.arange(n, dtype=np.uint32)), f"closest primitive along the chain: {p.tolist()}"
            assert np.array_equal(t, x) and np.all(a == 1)
            ba, bc, _ = compare(ctx, O.Scene(tri, brute=True), np.concatenate([rays, B.aimed(tri, np.random.default_rng(3), 2000, 5.0)]))
            assert ba == 0 and bc == 0
        finally:
            ctx.lib.hr_scene_destroy(h)


def test_too_deep_chain_is_refused_and_the_context_still_works(ctx):
    tri = B.chain(B.MAX_DEPTH + 2)
    with switches(ctx.lib, k3=1):
        rc, h, _ = build(ctx, tri)
    assert rc == HR_ERR_UNSUPPORTED, rc
    assert "deeper than the traversal stack" in ctx.lib.hr_last_error(ctx.h).decode()
    report, hits = check_scene(ctx, B.grid(8), n=1000)
    assert hits > 0 and not bad_entries(report), bad_entries(report)


# ---------------------------------------------------------------------------------------------- the packet and per-pass walks
GB_W, GB_H = 160, 96
# (scene, camera position relative to the scene's centre, in scene extents); a 4x4 roof over part of the scene casts the
# shadows and occludes the AO rays
PASS_CASES = {
    "grid_off2e4_near": ("grid_off2e4", (0.3, 1.2, 1.1)),
    "grid_off2e4_far": ("grid_off2e4", (1.5, 3.0, 4.0)),
    "duplicates": ("duplicates", (0.4, 1.0, 1.2)),
    "grid_off1e5": ("grid_off1e5", (-0.5, 0.8, 1.3)),
}


def with_roof(tri):
    lo, _ = B.scene_bounds(tri)
    return np.concatenate([tri, B.grid(4, (float(lo[0]) + 2.0, float(lo[1]) + 1.5, float(lo[2]) + 2.0))])


@pytest.mark.parametrize("case", sorted(PASS_CASES))
def test_gbuffer_shadows_ao_walks_match_the_oracle(case):
    """hr_gbuffer_render (packet closest-hit walk) bit for bit against orc_gbuffer, then the shadows and AO visibility masks
    (per-lane walk) against the oracle, under both tree builders"""
    scene, rel = PASS_CASES[case]
    tri = with_roof(B.SCENES[scene]())
    lo, hi = B.scene_bounds(tri)
    ext = float((hi - lo).max())
    c = 0.5 * (lo + hi)
    cam = tuple(float(v) for v in c + np.array(rel) * ext)
    tgt = tuple(float(v) for v in c)
    light = pyhr.default_light(rot_x_deg=35.0, rot_y_deg=20.0)
    bn = pyhr.blue_noise()
    asc = array_scene(tri)
    ss = O.ShadingScene(SoupShading(tri, asc), brute=True)
    ctx = pyhr.Context(0)
    try:
        ctx.set_bluenoise(*bn)
        ctx.gbuffer_create(GB_W, GB_H)
        failures = []
        for topology in sorted(TOPOLOGIES):
            with switches(ctx.lib, k3=TOPOLOGIES[topology]):
                h = ctx.build_scene(asc)
            try:
                f0 = pyhr.make_frame(cam, tgt, GB_W, GB_H, light=light)
                f = pyhr.make_frame(cam, tgt, GB_W, GB_H, prev=f0, num_frames=1, light=light)
                ctx.gbuffer_render(f.ping_pong, f)
                ref = O.gbuffer_render(ss, f, GB_W, GB_H)
                for which, want in ((0, ref.depth), (1, ref.gb1), (2, ref.gb2), (3, ref.gb3)):
                    if not np.array_equal(ctx.gbuffer_download(f.ping_pong, 0, which, GB_W, GB_H), want):
                        failures.append(f"{topology}: G-buffer image {which}")
                assert np.mean(ref.depth < 1.0) > 0.005, "the camera sees the scene"
                cur = O.GBufMips(ref)
                osh, oao = O.ShadowsOracle(GB_W, GB_H, 0), O.AOOracle(GB_W, GB_H, 0)
                osh.render(ss.scene, cur, O.zero_gbuf_mips(GB_W, GB_H), f, bn)
                oao.render(ss.scene, cur, O.zero_gbuf_mips(GB_W, GB_H), f, bn)
                ctx.gbuffer_upload(f.ping_pong, ref)
                sh, ao = pyhr.Pass(ctx, "shadows", GB_W, GB_H, 0), pyhr.Pass(ctx, "ao", GB_W, GB_H, 0)
                try:
                    sh.render(f)
                    ao.render(f)
                    if not np.array_equal(sh.download(0), osh.mask):
                        failures.append(f"{topology}: shadow mask")
                    if not np.array_equal(ao.download(0), oao.mask):
                        failures.append(f"{topology}: AO mask")
                finally:
                    sh.destroy()
                    ao.destroy()
            finally:
                ctx.lib.hr_scene_destroy(h)
        assert not failures, f"{case}: {failures}"
    finally:
        ctx.close()
