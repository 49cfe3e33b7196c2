"""The non-default BVH builder must produce the same bit-exact visibility masks as the oracle:
  * hr_debug_set(3, 0): Karras radix-tree topology instead of the default PLOC agglomerative build (hit results must not
    depend on the BVH topology)."""
import numpy as np
import pytest

import oracle as O
import pyhr

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dbg_key,dbg_val,dbg_default", [(3, 0, 1)], ids=["lbvh-topology"])
@pytest.mark.parametrize("scene_kind,tris,W,H,cam", [
    (pyhr.SCENE_SHADOWS_TEST, 0, 256, 144, ((0.0, 14.0, 34.0), (0.0, 3.0, 0.0))),
    (pyhr.SCENE_ARCADE, 30000, 200, 104, ((0.0, 9.0, -4.0), (2.0, 7.0, 60.0))),  # width not a multiple of 16: a partial last CTA
])
def test_variant_masks_bit_exact(scene_kind, tris, W, H, cam, dbg_key, dbg_val, dbg_default):
    sc = pyhr.SynthScene(scene_kind, tris)
    tri, _ = sc.world_triangles()
    osc = O.Scene(tri, brute=sc.n_tris <= 4096)
    bn = pyhr.blue_noise()
    ctx = pyhr.Context(0)
    try:
        ctx.lib.hr_debug_set(dbg_key, dbg_val)
        ctx.set_bluenoise(*bn)
        scene = ctx.build_scene(sc)
        info = ctx.scene_info(scene)
        assert 1 <= info.depth <= 63, "tree height is reported and within the traversal stack (HR_BVH_MAX_DEPTH)"
        assert info.depth >= int(np.ceil(np.log2(max(info.n_triangles, 2) / 4.0))) - 1
        ctx.gbuffer_create(W, H)
        sh, ao = pyhr.Pass(ctx, "shadows", W, H, 0), pyhr.Pass(ctx, "ao", W, H, 0)
        sh.params.denoise = ao.params.denoise = 0
        osh, oao = O.ShadowsOracle(W, H, 0), O.AOOracle(W, H, 0)
        osh.params.denoise = oao.params.denoise = 0
        f = None
        light = pyhr.default_light(rot_x_deg=25.0) if scene_kind == pyhr.SCENE_ARCADE else None
        for i in range(3):
            f = pyhr.make_frame(cam[0], cam[1], W, H, prev=f, num_frames=i, light=light)
            g = pyhr.write_gbuffer(sc, f, W, H)
            ctx.gbuffer_upload(f.ping_pong, g)
            sh.render(f)
            ao.render(f)
            cur = O.GBufMips(g)
            osh.render(osc, cur, cur, f, bn)
            oao.render(osc, cur, cur, f, bn)
            assert np.array_equal(sh.download(0), osh.mask), f"frame {i}: shadows mask (variant {dbg_key}={dbg_val})"
            assert np.array_equal(ao.download(0), oao.mask), f"frame {i}: AO mask (variant {dbg_key}={dbg_val})"
            assert osh.mask.any() and oao.mask.any()
        sh.destroy()
        ao.destroy()
    finally:
        ctx.lib.hr_debug_set(dbg_key, dbg_default)
        ctx.close()
