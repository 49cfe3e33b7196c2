"""Deferred shading combine (SURVEY.md §8 f2, deferred.frag:146-205) and the IBL specular term of the reflections hit shading
(reflections_ray_trace.rchit:97-104) with the synthetic split-sum LUT standing in for textures/brdf_lut.bin.

The end-to-end image metric VERDICT r1 asked for: all four passes -> combine, CUDA vs oracle, RMSE / PSNR of the final image.
"""
import numpy as np
import pytest

import oracle as O
import pyhr

W, H = 192, 112
SKY = (0.3, 0.4, 0.6)


def f16(a):
    return np.ascontiguousarray(a).view(np.float16).astype(np.float32)


@pytest.fixture(scope="module")
def lut():
    return pyhr.brdf_lut(64)


def test_brdf_lut_is_the_split_sum_table(lut):
    t = f16(lut)
    assert t.shape == (512, 512, 2) and np.isfinite(t).all()
    # smooth surface seen head-on: scale -> 1, bias -> 0; grazing smooth: bias grows (Fresnel); rough: scale drops
    assert t[2, 510, 0] > 0.95 and t[2, 510, 1] < 0.02
    assert t[2, 5, 1] > 0.3
    assert t[500, 510, 0] < 0.7
    assert (t >= 0).all() and (t[..., 0] + t[..., 1] <= 1.05).all()


def test_oracle_deferred_limits(lut):
    """no inputs bound, black environment, light along the normal of a plane: Lo = direct term only, > 0 where lit, 0 on unlit sides"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    f = pyhr.make_frame((0.0, 14.0, 34.0), (0.0, 3.0, 0.0), W, H)
    g = pyhr.write_gbuffer(sc, f, W, H)
    a = f16(O.deferred(g, f))
    assert np.isfinite(a).all() and (a[..., 3] == 1.0).all()
    floor = (f16(g.gb3)[..., 2] == 0.0) & (g.depth != 1.0)
    assert a[floor][:, :3].min() > 0.0                       # the floor faces the light
    b = f16(O.deferred(g, f, shadow=np.zeros((H, W), np.uint16)))  # visibility 0 everywhere: direct term gone, no environment => black
    assert np.abs(b[..., :3]).max() == 0.0
    # render_skybox (deferred_shading.cpp:69): the pixels the G-buffer left at its clear depth show the environment, alpha 1
    sky = g.depth == 1.0
    assert sky.any() and np.abs(a[sky][:, :3]).max() == 0.0
    c = f16(O.deferred(g, f, env=SKY, brdf_lut=lut))
    assert np.allclose(c[sky][:, :3], np.float16(SKY).astype(np.float32)) and (c[sky][:, 3] == 1.0).all()
    assert (c[floor][:, :3] >= a[floor][:, :3] - 1e-3).all() and c[floor][:, :3].mean() > a[floor][:, :3].mean()


def full_frame_then_combine(lut, light=None, cmp=None, frames=4):
    """shadows + AO + DDGI + reflections (with IBL specular) -> deferred combine over `frames` frames; every input compared elsewhere, here
    the combined image: RMSE <= 1e-3 (PSNR >= 60 dB at peak 1), and the reflections pass with the IBL term within its own tolerance.
    cmp(got, want, name, r, m): the rule for both images when they may hold inf and NaN (test_gpu_lights.SameClassThenClose); the
    combined image's RMSE and max-abs bars are then relative to max(1, |reference|)"""
    from test_gpu_gi_refl import close
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    bn = pyhr.blue_noise()
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*bn)
    ctx.set_brdf_lut(lut)
    ctx.build_scene(sc)
    ctx.gbuffer_create(W, H)
    mn, mx = sc.bounds()
    sh, ao = pyhr.Pass(ctx, "shadows", W, H, 0), pyhr.Pass(ctx, "ao", W, H, 1)
    dd, rf, de = pyhr.DDGIPass(ctx, W, H, 0), pyhr.ReflectionsPass(ctx, W, H, 1), pyhr.DeferredPass(ctx, W, H)
    dd.params.probe_distance, dd.params.normal_bias = 4.0, 1.0
    for P in (dd.params, rf.params):
        P.sky_color[0], P.sky_color[1], P.sky_color[2] = SKY
    de.params.env_color[0], de.params.env_color[1], de.params.env_color[2] = SKY
    osh, oao = O.ShadowsOracle(W, H, 0), O.AOOracle(W, H, 1)
    odd = O.DDGIOracle(W, H, 0, dd.params, mn, mx)
    orf = O.ReflectionsOracle(W, H, 1, rf.params)
    orf.brdf_lut = lut
    f, prev_g = None, O.zero_gbuf_mips(W, H)
    for i in range(frames):
        f = pyhr.make_frame((0.05 * max(0, i - 2), 14.0, 34.0), (0.0, 3.0, 0.0), W, H, prev=f, num_frames=i, light=light)
        ctx.gbuffer_render(f.ping_pong, f)
        g = O.gbuffer_render(ss, f, W, H)
        cur_g = O.GBufMips(g)
        rot = pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))
        sh.render(f); ao.render(f); dd.render(f, rot); rf.render(f, dd)
        de.render(f, sh, ao, rf, dd)
        osh.render(ss.scene, cur_g, prev_g, f, bn)
        oao.render(ss.scene, cur_g, prev_g, f, bn)
        odd.render(ss, cur_g, f, rot)
        orf.render(ss, cur_g, prev_g, f, bn, odd)
        prev_g = cur_g
        (cmp or close)(f16(rf.download(0))[..., :3], O.h2f(orf.rt)[..., :3], f"frame {i} reflections ray trace with IBL specular", 1e-3, 0.02)
        ref = f16(O.deferred(g, f, shadow=osh.final, ao=oao.final, reflections=orf.final, gi=odd.sample, env=SKY, brdf_lut=lut))
        got = f16(de.download(100))
        if cmp:
            cmp(got[..., :3], ref[..., :3], f"frame {i} combined image", 1e-3, 2e-2)
        else:
            err = float(np.sqrt(np.mean((got[..., :3] - ref[..., :3]) ** 2)))
            assert err <= 1e-3, f"frame {i}: combined image RMSE {err}"
            assert np.abs(got[..., :3] - ref[..., :3]).max() <= 2e-2
        assert (got[..., 3] == 1.0).all()
    assert f16(rf.download(0))[..., :3].mean() > 0.0
    for p in (sh, ao, dd, rf, de):
        p.destroy()
    ctx.close()


@pytest.mark.gpu
def test_full_frame_all_passes_then_combine_matches_oracle(lut):
    full_frame_then_combine(lut)


# light_cases: point, spot (smoothstep band, equal and reversed cone angles), a coloured sun, the overhead sun (no shadow ray: the
# combine shows the environment and the indirect terms only)
LIGHT_CASES = ["point_high", "point_low", "spot_band", "spot_hard_edge", "spot_reversed", "colored", "sun_overhead"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LIGHT_CASES)
def test_full_frame_then_combine_under_light(lut, case):
    """the raster light form of deferred.cu (built with FMA contraction, 1 / dot(tl, tl) for 1 / d^2) against the oracle's"""
    import light_cases as LC
    full_frame_then_combine(lut, LC.light(LC.BY_ID[case]))


@pytest.mark.gpu
def test_full_frame_then_combine_point_overflow(lut):
    """the 1e5 point light of light_cases.point_overflow: inf and NaN texels in the same places on the device and in the oracle
    (201 NaN in the oracle's frame 0).  Frame 0 only: from frame 1 the combine reads the device's own K21 sample, where a few
    hundred texels are inf on one side and the NaN guard's value on the other (test_gpu_lights.test_ddgi_reflections_point_overflow)"""
    import light_cases as LC
    from test_gpu_lights import SameClassThenClose
    cmp = SameClassThenClose()
    full_frame_then_combine(lut, LC.light(LC.BY_ID["point_overflow"]), cmp, frames=1)
    cmp.report("point_overflow")
