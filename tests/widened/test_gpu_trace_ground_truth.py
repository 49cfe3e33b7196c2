"""GPU parity of the ground-truth path tracer (SURVEY.md §8 f4) through the C ABI: hr_path_tracer_render vs oracle/orc_path_trace.cpp.
Bars: the primitive hit by every primary ray identical (the ray generation and the traversal are bit-specified); the accumulated
RGBA16F image within the colour tolerance of the other shaded stages (RMSE <= 1e-3, max <= 2e-2: a flipped shadow ray at a
silhouette is a full-scale difference in one pixel, so a handful of outliers are budgeted separately)."""
import numpy as np
import pytest

import light_cases as LC
import oracle as O
import pyhr

pytestmark = pytest.mark.gpu

W, H = 192, 112
SKY = (0.3, 0.4, 0.6)


def f16(a):
    return np.ascontiguousarray(a).view(np.float16).astype(np.float32)


def compare(got, want, what):
    d = np.abs(got[..., :3] - want[..., :3])
    outliers = d.max(-1) > 2e-2
    assert np.mean(outliers) <= 2e-3, f"{what}: {np.count_nonzero(outliers)} pixels differ by more than 2e-2"
    e = float(np.sqrt(np.mean(d[~outliers].astype(np.float64) ** 2)))
    assert e <= 1e-3, f"{what}: RMSE {e}"
    assert np.all(got[..., 3] == 1.0)


# the default sun, a point light, and the spot / overhead-sun / horizon-sun / coloured cases of light_cases.py (the soft shadow-ray form
# of the direct term: the smoothstep band, the NaN tangent of the overhead sun, N.Wi just below 0, Li per channel)
LIGHT_KW = [{}, dict(type=1, position=(4.0, 12.0, 6.0), radius=0.5, intensity=300.0)] + [LC.BY_ID[c].kw for c in ("spot_band", "sun_overhead", "sun_horizon", "colored")]


@pytest.mark.parametrize("light_kw", LIGHT_KW)
def test_path_tracer_matches_the_oracle(light_kw):
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    ctx.build_scene(sc)
    pt = pyhr.PathTracerPass(ctx, W, H)
    pt.params.sky_color[0], pt.params.sky_color[1], pt.params.sky_color[2] = SKY
    opt = O.PathTracerOracle(W, H, sky=SKY)
    light = pyhr.default_light(**light_kw)
    f = pyhr.make_frame((0.0, 14.0, 34.0), (0.0, 3.0, 0.0), W, H, light=light)
    pt.stats()
    n_hit = 0
    for i in range(4):
        pt.render(f)
        want = opt.render(ss, f)
        assert np.array_equal(pt.download(1), opt.prim), f"sample {i}: primary hits differ in {np.count_nonzero(pt.download(1) != opt.prim)} pixels"
        compare(f16(pt.download(100)), f16(want), f"sample {i}")
        n_hit += int(np.count_nonzero(opt.prim != 0xFFFFFFFF))
    st = pt.stats()
    assert st.rays_primary == 4 * W * H and st.renders == 4
    assert n_hit <= st.rays_secondary <= 2 * n_hit  # every hit traces the sky shadow ray, the ones facing the light its shadow ray too
    # restart_accumulation(): the image is replaced by sample 0 again
    first = O.PathTracerOracle(W, H, sky=SKY)
    first.render(ss, f)
    pt.reset_history()
    opt.restart_accumulation()
    pt.render(f)
    opt.render(ss, f)
    compare(f16(pt.download(100)), f16(first.final), "after restart")
    # the reference tone-maps the ground-truth image directly (tone_map.cpp:106-125)
    tm = pyhr.TonemapPass(ctx, W, H)
    tm.render(pt)
    got, want8 = tm.download(100), O.tonemap(np.ascontiguousarray(pt.download(100)).view(np.uint16))
    d = np.abs(got.astype(np.int16) - want8.astype(np.int16))
    assert d.max() <= 1 and np.mean(d == 0) >= 0.995
    # roughness multiplier and a moved camera change the image; parity holds there too
    pt.params.roughness_multiplier = 0.5
    opt.roughness_multiplier = 0.5
    f2 = pyhr.make_frame((3.0, 10.0, 30.0), (0.0, 3.0, 0.0), W, H, light=light)
    pt.reset_history()
    opt.restart_accumulation()
    pt.render(f2)
    compare(f16(pt.download(100)), f16(opt.render(ss, f2)), "moved camera, roughness x 0.5")
    assert np.array_equal(pt.download(1), opt.prim)
    for p in (pt, tm):
        p.destroy()
    ctx.close()
