"""spp > 1 (SURVEY.md §8d configs 4-5; NOT in the reference): `spp` rays per pixel with sample index num_frames * spp + s, an
8-bit image of unoccluded-ray counts instead of the 1-bit mask, visibility = count / spp in the temporal stage.

This mode runs the COUNT forms of the 1-spp kernels (k_ray_trace<MODE, true>, k_temporal<MODE, PEER, true>); the ray counts must be
exact against the oracle and the denoised images within the same tolerances as the 1-spp chains.
"""
import numpy as np
import pytest

import oracle as O
import pyhr

pytestmark = pytest.mark.gpu

W, H = 256, 144


def f16(a):
    return np.ascontiguousarray(a).view(np.float16).astype(np.float32)


def rmse(a, b):
    return float(np.sqrt(np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)))


def check_counts(i, sh, ao, osh, oao):
    """one spp > 1 frame of both chains against the oracle: counts, tile flags and history lengths exact, images within the 1-spp bars"""
    # counts are decisions of the deterministic chain: exact
    assert np.array_equal(sh.download(0), osh.count), f"frame {i}: shadows ray counts not exact"
    assert np.array_equal(ao.download(0), oao.count), f"frame {i}: AO ray counts not exact"
    assert np.array_equal(sh.download(6), osh.tile_flags), f"frame {i}: shadows tile classification differs in {np.count_nonzero(sh.download(6) != osh.tile_flags)} tiles"
    assert np.array_equal(ao.download(6), oao.tile_flags), f"frame {i}: AO tile classification differs in {np.count_nonzero(ao.download(6) != oao.tile_flags)} tiles"
    assert np.array_equal(f16(sh.download(4))[..., 2], O.h2f(osh.cur_moments)[..., 2]), f"frame {i}: history length"
    assert np.array_equal(f16(ao.download(4)), O.h2f(oao.cur_length)), f"frame {i}: AO history length"
    for which, ref, mx in ((1, osh.temporal, 2e-3), (2, osh.atrous_out, 4e-3), (100, osh.final, 4e-3)):
        c, o = f16(sh.download(which)), O.h2f(ref)
        assert rmse(c, o) <= 1e-3 and np.abs(c - o).max() <= mx, f"frame {i} shadows image {which}: rmse {rmse(c, o)} max {np.abs(c - o).max()}"
    for which, ref, mx in ((1, oao.temporal, 2e-3), (2, oao.blur[1], 4e-3), (100, oao.final, 4e-3)):
        c, o = f16(ao.download(which)), O.h2f(ref)
        assert rmse(c, o) <= 1e-3 and np.abs(c - o).max() <= mx, f"frame {i} AO image {which}: rmse {rmse(c, o)} max {np.abs(c - o).max()}"


@pytest.mark.parametrize("spp", [2, 4])
def test_spp_counts_exact_and_denoise_within_tolerance(spp):
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    tri, _ = sc.world_triangles()
    osc = O.Scene(tri, brute=True)
    bn = pyhr.blue_noise()
    ctx = pyhr.Context(0)
    try:
        ctx.set_bluenoise(*bn)
        ctx.build_scene(sc)
        ctx.gbuffer_create(W, H)
        sh, ao = pyhr.Pass(ctx, "shadows", W, H, 0), pyhr.Pass(ctx, "ao", W, H, 1)
        sh.params.spp = ao.params.spp = spp
        osh, oao = O.ShadowsOracle(W, H, 0, spp=spp), O.AOOracle(W, H, 1, spp=spp)
        f, prev = None, O.zero_gbuf_mips(W, H)
        for i in range(5):
            dx = 0.0 if i < 3 else 0.05 * (i - 2)
            f = pyhr.make_frame((dx, 14.0, 34.0), (dx, 3.0, 0.0), W, H, prev=f, num_frames=i)
            g = pyhr.write_gbuffer(sc, f, W, H)
            ctx.gbuffer_upload(f.ping_pong, g)
            sh.render(f)
            ao.render(f)
            cur = O.GBufMips(g)
            osh.render(osc, cur, prev, f, bn)
            oao.render(osc, cur, prev, f, bn)
            prev = cur
            check_counts(i, sh, ao, osh, oao)
        assert osh.count.max() == spp and oao.count.max() == spp
        sh.destroy()
        ao.destroy()
    finally:
        ctx.close()


def test_spp_sharded_emulation_matches_single():
    """spp > 1 on a sharded rank (band-local count image + recompute halo): each rank's band of the count image and of the denoised
    output equals the single-GPU result bit for bit (2 emulated ranks, history bands exchanged by the test)."""
    W, H = 128, 96
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)

    def mk(rank=0, world=1):
        c = pyhr.Context(0)
        c.set_bluenoise(*pyhr.blue_noise())
        c.build_scene(sc)
        c.gbuffer_create(W, H)
        if world > 1:
            c.shard_config(rank, world)
        sh = pyhr.Pass(c, "shadows", W, H, 0)
        sh.params.spp = 2
        return c, sh

    ref, ranks = mk(), [mk(r, 2) for r in range(2)]
    f = None
    for i in range(4):
        f = pyhr.make_frame((0.05 * i, 14.0, 34.0), (0.0, 3.0, 0.0), W, H, prev=f, num_frames=i)
        g = pyhr.write_gbuffer(sc, f, W, H)
        for c, sh in [ref] + ranks:
            c.gbuffer_upload(f.ping_pong, g)
            sh.render(f)
        for which in (0, 5, 4, 100):  # count image, prev_image, moments, final
            full = ref[1].download(which)
            parts = [r[1].download(which) for r in ranks]
            merged = full.copy()
            for r in range(2):
                b, e = pyhr.shard_rows(H, r, 2)
                merged[b:e] = parts[r][b:e]
            assert np.array_equal(merged, full), f"frame {i} image {which}"
            if which in (5, 4):
                for r in ranks:
                    r[1].upload(which, merged)
    for c, sh in [ref] + ranks:
        sh.destroy()
        c.close()


@pytest.mark.parametrize("spp", [2, 4])
def test_reflections_spp_matches_oracle(spp):
    """reflections with spp > 1 (SURVEY.md §8d): GGX lobe averaged over spp directions; ray length of sample 0 exact, colours and the
    denoised chain within the 1-spp tolerances."""
    from test_gpu_gi_refl import close, f16
    W, H = 192, 112
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    bn = pyhr.blue_noise()
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*bn)
    ctx.build_scene(sc)
    ctx.gbuffer_create(W, H)
    rf = pyhr.ReflectionsPass(ctx, W, H, 0)
    rf.params.spp = spp
    rf.params.sky_color[0], rf.params.sky_color[1], rf.params.sky_color[2] = 0.3, 0.4, 0.6
    orf = O.ReflectionsOracle(W, H, 0, rf.params)
    f, prev_g = None, O.zero_gbuf_mips(W, H)
    for i in range(3):
        f = pyhr.make_frame((0.05 * i, 14.0, 34.0), (0.0, 3.0, 0.0), W, H, prev=f, num_frames=i)
        g = pyhr.write_gbuffer(sc, f, W, H)
        ctx.gbuffer_upload(f.ping_pong, g)
        cur_g = O.GBufMips(g)
        rf.render(f, None)
        orf.render(ss, cur_g, prev_g, f, bn, None)
        prev_g = cur_g
        rt_c, rt_o = f16(rf.download(0)), O.h2f(orf.rt)
        assert np.array_equal(rt_c[..., 3], rt_o[..., 3]), f"frame {i}: ray length of sample 0 not exact"
        close(rt_c[..., :3], rt_o[..., :3], f"frame {i} ray trace", 1e-3, 0.02)
        close(f16(rf.download(100)), O.h2f(orf.final), f"frame {i} final")
    s = rf.stats()
    assert s.rays_primary > W * H  # more than one ray per traced GGX pixel
    rf.destroy()
    ctx.close()


def test_per_spp_scrambling_table_slot_is_used():
    """hr_bluenoise_set_slot (BlueNoiseSpp, src/blue_noise.cpp:9-19): a 2-spp shadows pass reads the table of slot 1 once it is set —
    its count image equals the oracle's run with that table (and differs from the run with the 1-spp table)."""
    W, H = 128, 96
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    tri, _ = sc.world_triangles()
    osc = O.Scene(tri, brute=False)
    sobol, sr1 = pyhr.blue_noise(1234)
    _, sr2 = pyhr.blue_noise(99)
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(sobol, sr1)
    ctx.set_bluenoise_slot(1, sr2)
    ctx.build_scene(sc)
    ctx.gbuffer_create(W, H)
    sh = pyhr.Pass(ctx, "shadows", W, H, 0)
    sh.params.spp = 2
    sh.params.denoise = 0
    f = pyhr.make_frame((0.0, 14.0, 34.0), (0.0, 3.0, 0.0), W, H)
    g = pyhr.write_gbuffer(sc, f, W, H)
    ctx.gbuffer_upload(f.ping_pong, g)
    sh.render(f)
    got = sh.download(0)
    cur = O.GBufMips(g)
    want = {}
    for name, sr in (("slot", sr2), ("base", sr1)):
        o = O.ShadowsOracle(W, H, 0, spp=2)
        o.params.denoise = 0
        o.render(osc, cur, cur, f, (sobol, sr))
        want[name] = o.count.copy()
    assert np.array_equal(got, want["slot"])
    assert not np.array_equal(want["slot"], want["base"])
    sh.destroy()
    ctx.close()
