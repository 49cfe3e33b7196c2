"""GPU parity at ragged frame sizes and non-default filter parameters.

The library picks a different kernel or edge path from the pass size and the filter parameters: an odd pass width or
phi_normal != 32 sends the a-trous stages of shadows and reflections to their scalar kernels (k_atrous_tiled, k_refl_atrous),
radius 2 or steps >= 16 to k_atrous_naive, an AO blur radius above 8 to the v1 k_ao_blur, a full-resolution frame that is not
exactly twice the coarse mip to k_upsample_v2, a one-column frame to k_upsample_scalar / k_upsample_vec4; sizes that are not
multiples of 8 leave partial 8x4 ray-trace groups, partial 8x8 tiles and partial warps everywhere.  Any odd window width gives an
odd-width half-resolution pass (1366x768 -> 683x384), so these are paths a user meets first.

Every stage is compared with the CPU oracle under the bars of the aligned-size tests, reused unchanged: check_all
(test_gpu_parity) for small frames, check_all_large / bounded (test_gpu_config_sizes) at about 1 Mpx, close (test_gpu_gi_refl) for
DDGI and reflections, same_halves and the tone-map rule (widened/test_gpu_taa_tonemap), the path-tracer bars
(widened/test_gpu_trace_ground_truth).  test_fallback_kernel_launched proves, with torch.profiler, that each case runs the kernel
it is meant to cover.  Run with -s to print the largest RMSE / max-abs error of every stage per case.
"""
import re

import numpy as np
import pytest
import torch

import oracle as O
import pyhr
from test_gpu_config_sizes import check_all_large
from test_gpu_gi_refl import close
from test_gpu_multi import AO, RF, SH, merge_bands
from test_gpu_parity import check_all, f16, rmse
from widened.test_gpu_taa_tonemap import same_halves, u16
from widened.test_gpu_trace_ground_truth import compare as compare_path_traced

pytestmark = pytest.mark.gpu

SKY = (0.3, 0.4, 0.6)
CAM_SHADOWS_TEST = ((0.0, 14.0, 34.0), (0.0, 3.0, 0.0))
CAM_ARCADE = ((0.0, 9.0, -4.0), (2.0, 7.0, 60.0))
# 250x141: W % 8 = 2, H % 4 = 1, half res 125x70 (odd width, not 2x), quarter 62x35; 251x144: odd width at full res;
# 7x3: smaller than one 8x4 group, mips collapse to 1; 1x1: one column, the only way to the scalar upsample kernels
SIZES = [(250, 141), (251, 144), (7, 3), (1, 1)]


def frames(W, H, n, pan_from=3, vertical=0.0, cam=CAM_SHADOWS_TEST, light=None):
    """static camera, then a lateral pan of 0.05 / frame; `vertical` adds a vertical pan so history taps cross the bottom edge"""
    (px, py, pz), (tx, ty, tz) = cam
    f = None
    for i in range(n):
        dx = 0.0 if i < pan_from else 0.05 * (i - pan_from + 1)
        dy = 0.0 if i < pan_from else vertical * (i - pan_from + 1)
        f = pyhr.make_frame((px + dx, py + dy, pz), (tx + dx, ty - dy, tz), W, H, prev=f, num_frames=i, light=light)
        yield i, f


class Worst:
    """largest RMSE and max-abs difference of each stage over a case's frames (printed with -s)"""

    def __init__(self, case):
        self.case, self.d = case, {}

    def add(self, stage, got, want):
        a, b = np.asarray(got, np.float64), np.asarray(want, np.float64)
        e, m = rmse(a, b), float(np.abs(a - b).max())
        r0, m0 = self.d.get(stage, (0.0, 0.0))
        self.d[stage] = (max(r0, e), max(m0, m))

    def report(self):
        print(f"\n[{self.case}] rmse / max-abs: " + ", ".join(f"{k} {r:.1e} / {m:.1e}" for k, (r, m) in self.d.items()))


def new_context(sc, W, H):
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    ctx.build_scene(sc)
    ctx.gbuffer_create(W, H)
    zero = pyhr.GBufferHost(W, H)  # the history slot starts as zeros, like the oracle's
    ctx.gbuffer_upload(0, zero)
    ctx.gbuffer_upload(1, zero)
    return ctx


def same_gbuffer(ctx, f, ref: O.GBufMips, W, H):
    """the device G-buffer producer and its mips 1 and 2 are the oracle's bits; the frame is not all sky (1x1 and 7x3 included)"""
    assert (ref.levels[0][4] != 1.0).any(), f"{W}x{H}: the camera sees no geometry"
    for mip in range(3):
        _, _, gb2, gb3, depth = ref.levels[mip]
        for which, arr in ((0, depth), (2, gb2), (3, gb3)):
            assert np.array_equal(ctx.gbuffer_download(f.ping_pong, mip, which, W, H), arr), f"{W}x{H}: device G-buffer image {which} of mip {mip} differs"


def set_params(dst_list, params):
    for k, v in (params or {}).items():
        for P in dst_list:
            setattr(P, k, v)


# ---------------------------------------------------------------------------------------------- shadows + AO
def measure_sh_ao(w, sh, ao, osh, oao):
    w.add("sh temporal", f16(sh.download(1)), O.h2f(osh.temporal))
    w.add("sh a-trous", f16(sh.download(2)), O.h2f(osh.atrous_out))
    w.add("sh prev_image", f16(sh.download(5)), O.h2f(osh.prev_image))
    w.add("sh final", f16(sh.download(100)), O.h2f(osh.final))
    w.add("ao temporal", f16(ao.download(1)), O.h2f(oao.temporal))
    w.add("ao blur", f16(ao.download(2)), O.h2f(oao.blur[1]))
    w.add("ao final", f16(ao.download(100)), O.h2f(oao.final))


def run_shadows_ao(case, W, H, sh_scale, ao_scale, sh_params=None, ao_params=None, n=5, vertical=0.0, scene=pyhr.SCENE_SHADOWS_TEST, tris=0,
                   cam=CAM_SHADOWS_TEST, light=None, check=check_all, pan_from=3):
    sc = pyhr.SynthScene(scene, tris)
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    bn = pyhr.blue_noise()
    ctx = new_context(sc, W, H)
    sh, ao = pyhr.Pass(ctx, "shadows", W, H, sh_scale), pyhr.Pass(ctx, "ao", W, H, ao_scale)
    osh, oao = O.ShadowsOracle(W, H, sh_scale), O.AOOracle(W, H, ao_scale)
    set_params([sh.params, osh.params], sh_params)
    set_params([ao.params, oao.params], ao_params)
    w = Worst(case)
    prev_g = O.zero_gbuf_mips(W, H)
    for i, f in frames(W, H, n, pan_from, vertical, cam, light):
        ctx.gbuffer_render(f.ping_pong, f)
        cur_g = O.GBufMips(O.gbuffer_render(ss, f, W, H))
        same_gbuffer(ctx, f, cur_g, W, H)
        sh.render(f)
        ao.render(f)
        osh.render(ss.scene, cur_g, prev_g, f, bn)
        oao.render(ss.scene, cur_g, prev_g, f, bn)
        prev_g = cur_g
        if check is check_all:
            check_all(i, sh, ao, osh, oao, [])
        else:
            check(i, sh, ao, osh, oao)
        measure_sh_ao(w, sh, ao, osh, oao)
    w.report()
    sh.destroy()
    ao.destroy()
    ctx.close()
    return w


@pytest.mark.parametrize("scale", [0, 1, 2])
@pytest.mark.parametrize("W,H", SIZES)
def test_shadows_ao_ragged_sizes(W, H, scale):
    """both chains at the same scale; 3 static + 2 panning frames, the half-resolution case pans vertically too"""
    run_shadows_ao(f"shadows+ao {W}x{H} scale {scale}", W, H, scale, scale, vertical=0.35 if scale == 1 else 0.0)


def test_shadows_ao_display_size_half_res():
    """1366x768: shadows, AO (and reflections, below) at half resolution 683x384, an odd-width pass of 262 k pixels"""
    run_shadows_ao("shadows+ao 1366x768 scale 1", 1366, 768, 1, 1, n=3, pan_from=2, scene=pyhr.SCENE_ARCADE, tris=20000, cam=CAM_ARCADE,
                   light=pyhr.default_light(rot_x_deg=25.0), check=check_all_large)


SH_PARAMS = {
    "radius2": dict(radius=2),
    "phi_normal16": dict(phi_normal=16.0),
    "iter6_fb5": dict(filter_iterations=6, feedback_iteration=5),  # steps 16 and 32
    "iter1_fb0": dict(filter_iterations=1, feedback_iteration=0),  # the fed-back iteration is the last one: filtered, then copied
    "iter4_fb7": dict(filter_iterations=4, feedback_iteration=7),  # never fed back: the history image keeps its contents
    "iter0": dict(filter_iterations=0),
}


@pytest.mark.parametrize("case", list(SH_PARAMS))
def test_shadows_parameters(case):
    """6 frames, so each frame's fed-back image is the next frame's temporal history; prev_image compared every frame"""
    run_shadows_ao(f"shadows {case} 256x144", 256, 144, 0, 1, sh_params=SH_PARAMS[case], n=6)


@pytest.mark.parametrize("case", ["radius2", "phi_normal16"])
def test_shadows_parameters_ragged(case):
    run_shadows_ao(f"shadows {case} 250x141", 250, 141, 0, 1, sh_params=SH_PARAMS[case], n=6, vertical=0.35)


@pytest.mark.parametrize("blur_radius", [1, 8, 9, 16])
def test_ao_blur_radius(blur_radius):
    """8 is the largest radius of k_ao_blur_v2; 9..16 run the v1 kernel"""
    run_shadows_ao(f"ao blur_radius {blur_radius} 256x144", 256, 144, 0, 1, ao_params=dict(blur_radius=blur_radius), n=6)


# ---------------------------------------------------------------------------------------------- DDGI + reflections
def run_gi_refl(case, W, H, scale, with_ddgi, params=None, n=5, pan_from=3, vertical=0.0, scene=pyhr.SCENE_SHADOWS_TEST, tris=0, cam=CAM_SHADOWS_TEST,
                light=None):
    """test_gpu_gi_refl.run at any size and scale (DDGI sampled at the reflections' scale), fed by the device G-buffer producer"""
    sc = pyhr.SynthScene(scene, tris)
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    bn = pyhr.blue_noise()
    ctx = new_context(sc, W, H)
    mn, mx = sc.bounds()
    dd = pyhr.DDGIPass(ctx, W, H, scale) if with_ddgi else None
    rf = pyhr.ReflectionsPass(ctx, W, H, scale)
    for P in ([dd.params] if dd else []) + [rf.params]:
        P.sky_color[0], P.sky_color[1], P.sky_color[2] = SKY
    set_params([rf.params], params)  # the reflections oracle reads the same parameter block
    odd = None
    if dd:
        dd.params.probe_distance = 4.0 if scene == pyhr.SCENE_SHADOWS_TEST else 12.0
        dd.params.normal_bias = 1.0
        odd = O.DDGIOracle(W, H, scale, dd.params, mn, mx)
    orf = O.ReflectionsOracle(W, H, scale, rf.params)
    w = Worst(case)
    prev_g = O.zero_gbuf_mips(W, H)
    for i, f in frames(W, H, n, pan_from, vertical, cam, light):
        ctx.gbuffer_render(f.ping_pong, f)
        cur_g = O.GBufMips(O.gbuffer_render(ss, f, W, H))
        same_gbuffer(ctx, f, cur_g, W, H)
        if dd:
            rot = pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))
            dd.render(f, rot)
            odd.render(ss, cur_g, f, rot)
            if i == 0:
                assert bytes(dd.uniforms()) == bytes(odd.u), "DDGIUniforms differ"
            dird_c = dd.download(1).view(np.uint16)
            assert np.array_equal(dird_c, odd.dirdepth.reshape(dird_c.shape)), f"frame {i}: probe ray direction / hit distance not exact"
            close(f16(dd.download(0)), O.h2f(odd.radiance).reshape(-1, odd.u.rays_per_probe, 4), f"frame {i} ddgi radiance", 2e-3, 0.05)
            close(f16(dd.download(2)), O.h2f(odd.cur_irr), f"frame {i} irradiance atlas")
            close(f16(dd.download(3)), O.h2f(odd.cur_dep), f"frame {i} depth atlas", 2e-3, 0.05)
            close(f16(dd.download(4)), O.h2f(odd.sample), f"frame {i} ddgi sample")
            w.add("ddgi irradiance", f16(dd.download(2)), O.h2f(odd.cur_irr))
            w.add("ddgi sample", f16(dd.download(4)), O.h2f(odd.sample))
        rf.render(f, dd)
        orf.render(ss, cur_g, prev_g, f, bn, odd)
        prev_g = cur_g
        rt_c, rt_o = f16(rf.download(0)), O.h2f(orf.rt)
        assert np.array_equal(rt_c[..., 3], rt_o[..., 3]), f"frame {i}: reflection ray length (hit / miss / t) not exact"
        close(rt_c[..., :3], rt_o[..., :3], f"frame {i} reflections ray trace", 1e-3, 0.02)
        w.add("rt", rt_c[..., :3], rt_o[..., :3])
        if not rf.params.denoise:
            continue
        assert np.array_equal(rf.download(6), orf.tile_flags), f"frame {i}: reflections tile classification"
        mo_c, mo_o = f16(rf.download(4)), O.h2f(orf.cur_moments)
        assert np.array_equal(mo_c[..., 2], mo_o[..., 2]), f"frame {i}: reflections history length"
        for name, got, want in (("temporal", f16(rf.download(1)), O.h2f(orf.cur_temporal)), ("moments", mo_c, mo_o),
                                ("a-trous", f16(rf.download(2)), O.h2f(orf.atrous_out)), ("final", f16(rf.download(100)), O.h2f(orf.final))):
            close(got, want, f"frame {i} reflections {name}")
            w.add(name, got, want)
    w.report()
    rf.destroy()
    if dd:
        dd.destroy()
    ctx.close()
    return float(rt_o[..., :3].mean()), float((rt_o[..., 3] > 0).mean())


@pytest.mark.parametrize("scale", [0, 1])
@pytest.mark.parametrize("W,H", SIZES)
def test_ddgi_reflections_ragged_sizes(W, H, scale):
    """DDGI + reflections reading its atlas; 250x141 on the arcade scene, where every reflection lobe occurs"""
    kw = dict(vertical=0.35 if scale == 1 else 0.0)
    if (W, H) == (250, 141):
        kw.update(scene=pyhr.SCENE_ARCADE, tris=20000, cam=CAM_ARCADE, light=pyhr.default_light(rot_x_deg=25.0), vertical=0.2 if scale == 1 else 0.0)
    mean, hit_frac = run_gi_refl(f"ddgi+reflections {W}x{H} scale {scale}", W, H, scale, True, **kw)
    if (W, H) == (250, 141):
        assert mean > 0.01 and hit_frac > 0.2


def test_reflections_display_size_half_res():
    """1366x768 reflections at half resolution; `close` is also the rule of the 4K reflections test"""
    run_gi_refl("reflections 1366x768 scale 1", 1366, 768, 1, False, n=3, pan_from=2, scene=pyhr.SCENE_ARCADE, tris=20000, cam=CAM_ARCADE,
                light=pyhr.default_light(rot_x_deg=25.0))


REFL_PARAMS = {
    "iter0": (dict(filter_iterations=0), False),
    "iter1": (dict(filter_iterations=1), False),
    "iter5": (dict(filter_iterations=5), False),  # steps 1..16
    "phi_normal16": (dict(phi_normal=16.0), False),
    "blur_as_input_fb0": (dict(blur_as_input=1, feedback_iteration=0), False),  # history = a-trous iteration 0 of the last frame
    "blur_as_input_fb2": (dict(blur_as_input=1, feedback_iteration=2), False),
    "approx0_ddgi": (dict(approximate_with_ddgi=0), True),
    "approx1_ddgi": (dict(approximate_with_ddgi=1), True),
}


@pytest.mark.parametrize("case", list(REFL_PARAMS))
def test_reflections_parameters(case):
    params, with_ddgi = REFL_PARAMS[case]
    run_gi_refl(f"reflections {case} 256x144", 256, 144, 0, with_ddgi, params=params, n=6)


def test_reflections_phi_normal_ragged():
    run_gi_refl("reflections phi_normal16 250x141", 250, 141, 0, False, params=dict(phi_normal=16.0), n=6, vertical=0.2)


# ---------------------------------------------------------------------------------------------- full-resolution post chain
@pytest.mark.parametrize("W,H", [(250, 141), (251, 144)])
def test_post_chain_ragged(W, H):
    """deferred combine over the device's own pass outputs, TAA over it (bit-exact), tone map, and the path tracer"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    ctx = new_context(sc, W, H)
    sh, ao, rf, de = pyhr.Pass(ctx, "shadows", W, H, 0), pyhr.Pass(ctx, "ao", W, H, 1), pyhr.ReflectionsPass(ctx, W, H, 1), pyhr.DeferredPass(ctx, W, H)
    rf.params.sky_color[0], rf.params.sky_color[1], rf.params.sky_color[2] = SKY
    de.params.env_color[0], de.params.env_color[1], de.params.env_color[2] = SKY
    taa, tm = pyhr.TAAPass(ctx, W, H), pyhr.TonemapPass(ctx, W, H)
    taa.params.reset_every_frame = 0  # the history feeds the next frame
    otaa = O.TAAOracle(W, H, reset_every_frame=0)
    w = Worst(f"post chain {W}x{H}")
    prev_j = np.zeros(2, np.float32)
    for i, f in frames(W, H, 5, pan_from=2):
        j = pyhr.taa_jitter(i, W, H)
        assert np.array_equal(j, O.taa_jitter(i, W, H))
        pyhr.apply_jitter(f, j, prev_j)
        prev_j = j
        ctx.gbuffer_render(f.ping_pong, f)
        sh.render(f)
        ao.render(f)
        rf.render(f, None)
        de.render(f, sh, ao, rf, None)
        g = pyhr.GBufferHost(W, H)  # the combine's inputs as the device holds them: no upstream tolerance leaks in
        g.gb1 = ctx.gbuffer_download(f.ping_pong, 0, 1, W, H)
        g.gb2 = ctx.gbuffer_download(f.ping_pong, 0, 2, W, H)
        g.gb3 = ctx.gbuffer_download(f.ping_pong, 0, 3, W, H)
        g.depth = ctx.gbuffer_download(f.ping_pong, 0, 0, W, H)
        want = f16(O.deferred(g, f, shadow=sh.download(100), ao=ao.download(100), reflections=rf.download(100), env=SKY))
        got = f16(de.download(100))
        assert got.shape == want.shape == (H, W, 4)
        w.add("deferred", got[..., :3], want[..., :3])
        assert rmse(got[..., :3], want[..., :3]) <= 1e-3, f"frame {i}: deferred RMSE {rmse(got[..., :3], want[..., :3])}"
        assert np.abs(got[..., :3] - want[..., :3]).max() <= 2e-2
        assert (got[..., 3] == 1.0).all()
        cur = u16(de.download(100))
        taa.render(f, de)
        want_taa = otaa.render(f, cur, g.depth, u16(g.gb2))
        got_taa = u16(taa.download(100))
        assert same_halves(got_taa, want_taa), f"frame {i}: TAA: {np.count_nonzero(got_taa != want_taa)} of {got_taa.size} halves differ"
        assert same_halves(u16(taa.download(0)), otaa.img[1 - f.ping_pong]), f"frame {i}: TAA history image"
        tm.render(taa)
        got8, want8 = tm.download(100), O.tonemap(got_taa)
        d = np.abs(got8.astype(np.int16) - want8.astype(np.int16))
        assert got8.shape == (H, W, 4) and d.max() <= 1 and np.mean(d == 0) >= 0.995, f"frame {i}: tone map max diff {d.max()}, identical {np.mean(d == 0):.4f}"
    w.report()
    pt = pyhr.PathTracerPass(ctx, W, H)
    pt.params.sky_color[0], pt.params.sky_color[1], pt.params.sky_color[2] = SKY
    opt = O.PathTracerOracle(W, H, sky=SKY)
    f = pyhr.make_frame(*CAM_SHADOWS_TEST, W, H)
    for i in range(3):
        pt.render(f)
        want = opt.render(ss, f)
        assert np.array_equal(pt.download(1), opt.prim), f"sample {i}: primary hits differ in {np.count_nonzero(pt.download(1) != opt.prim)} pixels"
        compare_path_traced(f16(pt.download(100)), f16(want), f"{W}x{H} sample {i}")
    for p in (pt, tm, taa, de, rf, sh, ao):
        p.destroy()
    ctx.close()


# ---------------------------------------------------------------------------------------------- sharding at a ragged height
def _linked_ranks(make, world):
    ref = make(0, 1)
    ranks = [make(r, world) for r in range(world)]
    for r in range(world):
        for q in range(world):
            if q != r:
                for a, b in zip(ranks[r][1:], ranks[q][1:]):
                    a.link_local(q, b)
    return ref, ranks


def test_peer_history_ragged_non_default_parameters():
    """test_gpu_multi.test_peer_history_emulation_bit_identical at 250x141, world 3, shadows radius 2 with 6 iterations (halos derived
    from those) and AO blur_radius 12: every rank's band of every image is the single-rank image bit for bit"""
    W, H, world = 250, 141, 3
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)

    def make(rank, world):
        c = pyhr.Context(0)
        c.set_bluenoise(*pyhr.blue_noise())
        c.build_scene(sc)
        c.gbuffer_create(W, H)
        if world > 1:
            c.shard_config(rank, world)
        sh, ao = pyhr.Pass(c, "shadows", W, H, 0), pyhr.Pass(c, "ao", W, H, 1)
        sh.params.radius, sh.params.filter_iterations, sh.params.feedback_iteration = 2, 6, 1
        ao.params.blur_radius = 12
        return c, sh, ao

    ref, ranks = _linked_ranks(make, world)
    streams = [torch.cuda.Stream() for _ in range(world)]
    sh_h, ao_h = H, O.pass_size(W, H, 1)[1]
    for _, f in frames(W, H, 7, pan_from=2, vertical=0.35):
        g = pyhr.write_gbuffer(sc, f, W, H)
        ref[0].gbuffer_upload(f.ping_pong, g)
        ref[1].render(f)
        ref[2].render(f)
        for (c, sh, ao), st in zip(ranks, streams):
            c.gbuffer_upload(f.ping_pong, g, st.cuda_stream)
        for (c, sh, ao), st in zip(ranks, streams):
            sh.render(f, st.cuda_stream)
        for (c, sh, ao), st in zip(ranks, streams):
            ao.render(f, st.cuda_stream)
        torch.cuda.synchronize()
        for r in ranks:
            assert np.array_equal(r[1].download(0), ref[1].download(0)), f"shadows mask differs (frame {f.num_frames})"
            assert np.array_equal(r[2].download(0), ref[2].download(0)), f"ao mask differs (frame {f.num_frames})"
        for name, which in (("prev", SH["prev"]), ("moments", SH["moments"]), ("a-trous", SH["atrous"]), ("final", SH["final"])):
            merged = merge_bands([r[1].download(which) for r in ranks], sh_h, world)
            assert np.array_equal(merged, ref[1].download(which)), f"shadows {name} differs (frame {f.num_frames})"
        for name, which, shift in (("temporal", AO["temporal"], 0), ("length", AO["length"], 0), ("blur", AO["blur"], 0), ("final", AO["final"], 1)):
            merged = merge_bands([r[2].download(which) for r in ranks], ao_h, world, shift)
            assert np.array_equal(merged, ref[2].download(which)), f"ao {name} differs (frame {f.num_frames})"
    for c, sh, ao in [ref] + ranks:
        sh.destroy()
        ao.destroy()
    for c, sh, ao in [ref] + ranks:
        c.close()


def test_peer_history_reflections_ragged_half_res():
    """the reflections emulation of test_gpu_multi at 250x141, half resolution (125x70), world 3, vertical pan"""
    W, H, world, scale = 250, 141, 3, 1
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)

    def make(rank, world):
        c = pyhr.Context(0)
        c.set_bluenoise(*pyhr.blue_noise())
        c.build_scene(sc)
        c.gbuffer_create(W, H)
        if world > 1:
            c.shard_config(rank, world)
        p = pyhr.ReflectionsPass(c, W, H, scale)
        p.params.sky_color[0], p.params.sky_color[1], p.params.sky_color[2] = SKY
        return c, p

    ref, ranks = _linked_ranks(make, world)
    streams = [torch.cuda.Stream() for _ in range(world)]
    ph = O.pass_size(W, H, scale)[1]
    for _, f in frames(W, H, 7, pan_from=2, vertical=0.35):
        g = pyhr.write_gbuffer(sc, f, W, H)
        ref[0].gbuffer_upload(f.ping_pong, g)
        ref[1].render(f, None)
        for (c, p), st in zip(ranks, streams):
            c.gbuffer_upload(f.ping_pong, g, st.cuda_stream)
        for (c, p), st in zip(ranks, streams):
            p.render(f, None, st.cuda_stream)
        torch.cuda.synchronize()
        for name, which, shift in (("ray trace", RF["rt"], 0), ("temporal", RF["temporal"], 0), ("moments", RF["moments"], 0), ("a-trous", RF["atrous"], 0),
                                   ("final", RF["final"], scale)):
            merged = merge_bands([r[1].download(which) for r in ranks], ph, world, shift)
            assert np.array_equal(merged, ref[1].download(which)), f"reflections {name} differs (frame {f.num_frames})"
    for c, p in [ref] + ranks:
        p.destroy()
    for c, p in [ref] + ranks:
        c.close()


# ---------------------------------------------------------------------------------------------- which kernel ran
def _kernel_names(run):
    """demangled names of the kernels launched while `run` executes (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    return {e.name for e in prof.events()}


def _launched(names, kernel):
    """`kernel` is among the names, matched up to its template / argument list: k_refl_atrous does not match k_refl_atrous_v2"""
    pat = re.compile(r"(?<![\w])" + re.escape(kernel) + r"[<(]")
    return any(pat.search(n) for n in names)


def _one_frame(kind, W, H, scale, params=None):
    """one frame of one pass on a fresh context; returns the kernels its render launched"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    p = pyhr.ReflectionsPass(ctx, W, H, scale) if kind == "reflections" else pyhr.Pass(ctx, kind, W, H, scale)
    set_params([p.params], params)
    f = pyhr.make_frame(*CAM_SHADOWS_TEST, W, H)
    ctx.gbuffer_render(f.ping_pong, f)
    torch.cuda.synchronize()
    names = _kernel_names(lambda: p.render(f, None) if kind == "reflections" else p.render(f))
    p.destroy()
    ctx.close()
    return names


# (case of the parity tests above, (pass, W, H, scale, parameters), kernel that must run, kernels that must not): every fallback kernel
# of the dispatch.  The feedback bookkeeping (history copies, blur_as_input) launches no kernel of its own; its parity is compared above.
COVERAGE = [
    ("shadows 251x144 (odd pass width)", ("shadows", 251, 144, 0, None), "k_atrous_tiled", ["k_atrous_v3", "k_atrous_v3s"]),
    ("shadows 250x141 half res (125 wide)", ("shadows", 250, 141, 1, None), "k_atrous_tiled", ["k_atrous_v3", "k_atrous_v3s"]),
    ("shadows phi_normal 16", ("shadows", 256, 144, 0, dict(phi_normal=16.0)), "k_atrous_tiled", ["k_atrous_v3", "k_atrous_v3s"]),
    ("shadows radius 2", ("shadows", 256, 144, 0, dict(radius=2)), "k_atrous_naive", ["k_atrous_v3", "k_atrous_tiled"]),
    ("shadows 6 iterations (steps 16, 32)", ("shadows", 256, 144, 0, dict(filter_iterations=6, feedback_iteration=5)), "k_atrous_naive", []),
    ("AO blur_radius 9", ("ao", 256, 144, 1, dict(blur_radius=9)), "k_ao_blur", ["k_ao_blur_v2"]),
    ("AO blur_radius 16", ("ao", 256, 144, 1, dict(blur_radius=16)), "k_ao_blur", ["k_ao_blur_v2"]),
    ("shadows 250x141 half res (141 != 2 x 70)", ("shadows", 250, 141, 1, None), "k_upsample_v2", ["k_upsample_2x"]),
    ("AO 251x144 half res (251 != 2 x 125)", ("ao", 251, 144, 1, None), "k_upsample_v2", ["k_upsample_2x"]),
    ("AO 250x141 quarter res", ("ao", 250, 141, 2, None), "k_upsample_v2", ["k_upsample_2x"]),
    ("shadows 1x1 half res (one column)", ("shadows", 1, 1, 1, None), "k_upsample_scalar", ["k_upsample_v2", "k_upsample_2x"]),
    ("AO 1x1 half res (one column)", ("ao", 1, 1, 1, None), "k_upsample_scalar", ["k_upsample_v2", "k_upsample_2x"]),
    ("reflections 251x144 (odd pass width)", ("reflections", 251, 144, 0, None), "k_refl_atrous", ["k_refl_atrous_v2", "k_refl_atrous_tma"]),
    ("reflections 250x141 half res (125 wide)", ("reflections", 250, 141, 1, None), "k_refl_atrous", ["k_refl_atrous_v2", "k_refl_atrous_tma"]),
    ("reflections phi_normal 16", ("reflections", 256, 144, 0, dict(phi_normal=16.0)), "k_refl_atrous", ["k_refl_atrous_v2", "k_refl_atrous_tma"]),
    ("reflections 1x1 half res (one column)", ("reflections", 1, 1, 1, None), "k_upsample_vec4", []),
    # the defaults at an aligned size, so that a matcher that matched everything would be caught
    ("shadows defaults 256x144", ("shadows", 256, 144, 1, None), "k_atrous_v3", ["k_atrous_tiled", "k_atrous_naive", "k_upsample_v2"]),
    ("AO defaults 256x144", ("ao", 256, 144, 1, None), "k_ao_blur_v2", ["k_ao_blur", "k_upsample_v2"]),
    ("reflections defaults 256x144", ("reflections", 256, 144, 0, None), "k_refl_atrous_v2", ["k_refl_atrous"]),
]


@pytest.mark.parametrize("case,setup,kernel,absent", COVERAGE, ids=[c[0] for c in COVERAGE])
def test_fallback_kernel_launched(case, setup, kernel, absent):
    """the case above launches the kernel it is meant to cover (separate from the parity tests, so a profiler problem cannot hide a
    parity result); no hr_debug_set switch is touched"""
    names = _one_frame(*setup)
    kernels = sorted(n for n in names if n.startswith("void ") or re.search(r"\bk_\w+[<(]", n))
    assert _launched(names, kernel), f"{case}: {kernel} not launched; kernels: {kernels}"
    for k in absent:
        assert not _launched(names, k), f"{case}: {k} launched; kernels: {kernels}"
    print(f"\n[{case}] launched {kernel}")
