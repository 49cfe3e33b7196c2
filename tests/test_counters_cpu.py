"""The oracle's side of the counter cases (counter_cases.py), on the CPU.

- The blue-noise sample index is (num_frames * spp + s) mod 256 over the unsigned counter: with a static camera the mask or count
  image at frame N equals the one at N mod 256, also where num_frames * spp + s passes 2^31 or num_frames passes 2^32.
- Sensitivity: at spp 41 a temporal stage that multiplied by the rounded reciprocal 1 / spp instead of dividing would flag other
  AO tiles than the oracle, so the exact tile-flag comparison of the GPU case tells the two formulas apart.
- The history length saturates: 32 on every frame from 31 on in a long static run.
"""
import ctypes as C

import numpy as np
import pytest

import counter_cases as K
import oracle as O
import pyhr


@pytest.fixture(scope="module")
def scene():
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    return O.ShadingScene(sc, brute=sc.n_tris <= 4096)


def _static(ss, W, H, num_frames):
    f = pyhr.make_frame(*K.CAM, W, H, num_frames=num_frames)
    return f, O.GBufMips(O.gbuffer_render(ss, f, W, H))


def _visibility(ss, kind, spp, num_frames, W, H):
    """the ray-trace result of a shadows or AO pass at scale 0 without denoising: the bit mask (spp 1) or the count image"""
    f, g = _static(ss, W, H, num_frames)
    o = O.ShadowsOracle(W, H, 0, spp=spp) if kind == "shadows" else O.AOOracle(W, H, 0, spp=spp)
    o.params.denoise = 0
    o.render(ss.scene, g, g, f, pyhr.blue_noise())
    return (o.mask if spp == 1 else o.count).copy()


@pytest.mark.parametrize("kind", ["shadows", "ao"])
@pytest.mark.parametrize("spp,n", K.MOD256, ids=[f"spp{s}-{n}" for s, n in K.MOD256])
def test_sample_index_wraps_mod_256(spp, n, kind, scene):
    W, H = (128, 72) if spp > 1 else (256, 144)
    got, want = _visibility(scene, kind, spp, n, W, H), _visibility(scene, kind, spp, n % 256, W, H)
    assert np.array_equal(got, want), f"{kind} spp {spp}: frame {n} differs from frame {n % 256}"
    # the table entry really depends on the index: the neighbouring frame differs
    assert not np.array_equal(want, _visibility(scene, kind, spp, (n + 1) % 256, W, H))


def test_reflections_sample_index_wraps_mod_256(scene):
    """K12's GGX sample index at spp 4 across num_frames * 4 = 2^31"""
    W, H, spp, n = 128, 72, 4, 2**29 + 3
    out = []
    for nf in (n, n % 256):
        f, g = _static(scene, W, H, nf)
        P = pyhr.hr_reflections_params()
        pyhr.load_product().hr_reflections_default_params(C.byref(P))
        P.spp, P.denoise = spp, 0
        P.sky_color[0], P.sky_color[1], P.sky_color[2] = 0.3, 0.4, 0.6
        o = O.ReflectionsOracle(W, H, 0, P)
        o.render(scene, g, g, f, pyhr.blue_noise(), None)
        out.append(o.rt.copy())
    assert (O.h2f(out[0])[..., 3] > 0).mean() > 0.2, "too few reflection rays hit: the case does not test the GGX index"
    assert np.array_equal(out[0], out[1])


def _ao_frame0(ss, spp, W=256, H=144):
    f, g = _static(ss, W, H, 0)
    o = O.AOOracle(W, H, 1, spp=spp)
    o.render(ss.scene, g, O.zero_gbuf_mips(W, H), f, pyhr.blue_noise())
    return o, g.levels[1][4][:o.H, :o.W]


@pytest.mark.parametrize("spp", [41, 47])
def test_reciprocal_multiply_flags_other_ao_tiles(spp, scene):
    """frame 0 (alpha = 1, so o0 = visibility): flags from count / spp reproduce the oracle's exactly, flags from
    count * (1 / spp) do not"""
    o, depth = _ao_frame0(scene, spp)
    geo, f32 = depth != 1.0, np.float32
    cnt = o.count.astype(f32)
    exact = K.tile_any(geo & (cnt / f32(spp) < 1))
    recip = K.tile_any(geo & (cnt * (f32(1) / f32(spp)) < 1))
    assert np.array_equal(exact, o.tile_flags.astype(bool)), "the division's emulation does not reproduce the oracle's flags"
    differ = int((recip != exact).sum())
    print(f"\nspp {spp}: oracle flags {int(exact.sum())} of {exact.size} AO tiles, reciprocal multiply {int(recip.sum())}, {differ} differ")
    assert differ > 0
    assert K.full_count_tiles(o.count, depth, o.cur_length.view(np.float16).astype(np.float32), spp) >= differ


def test_spp3_reaches_an_open_window(scene):
    """spp 3 (a 17x17 window mean of 867 / 867 that a reciprocal multiply does not give as 1): the shadows case has open windows"""
    f, g = _static(scene, 256, 144, 0)
    o = O.ShadowsOracle(256, 144, 0, spp=3)
    o.params.denoise = 0
    o.render(scene.scene, g, g, f, pyhr.blue_noise())
    assert K.open_windows(o.count, 3) > 100
    f32 = np.float32
    assert f32(867) * (f32(1) / f32(867)) != 1.0 and f32(867) / f32(867) == 1.0


def test_history_length_saturates_in_the_long_run(scene):
    """K.LONG_STATIC static frames at 64x48: every geometry pixel's history length is min(32, frame + 1), in K3 and K9"""
    W, H = 64, 48
    bn = pyhr.blue_noise()
    osh, oao = O.ShadowsOracle(W, H, 0), O.AOOracle(W, H, 0)
    prev_g = O.zero_gbuf_mips(W, H)
    for i, f in K.frames(W, H, K.LONG_STATIC):
        g = O.GBufMips(O.gbuffer_render(scene, f, W, H))
        osh.render(scene.scene, g, prev_g, f, bn)
        oao.render(scene.scene, g, prev_g, f, bn)
        prev_g = g
        geo = g.levels[0][4] != 1.0
        want = min(K.HIST_CAP, i + 1)
        for name, ln in (("shadows", O.h2f(osh.cur_moments)[..., 2]), ("ao", O.h2f(oao.cur_length))):
            assert (ln[geo] == want).all(), f"frame {i}: {name} history length {np.unique(ln[geo])}, want {want}"
            assert (ln[~geo] == 0).all()
