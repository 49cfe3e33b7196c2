"""The converged references' CPU restatement (oracle/orc_reference.cpp) against closed forms and its own sample split.

The hand-built scenes use view_proj_inverse = identity, so pixel (x, y) at depth d sits at world ((x + 0.5) / W * 2 - 1,
(y + 0.5) / H * 2 - 1, d): a plane z = 0.5 facing +z."""
import numpy as np
import pytest

import oracle as O
import oracle_reference as R
import pyhr

W, H = 16, 12


def _box(lo, hi):
    """12 triangles of the closed axis-aligned box [lo, hi]^3, (12, 9) float32"""
    v = np.array([[x, y, z] for x in (lo, hi) for y in (lo, hi) for z in (lo, hi)], np.float32)
    faces = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    tris = []
    for a, b, c, d in faces:
        tris += [v[[a, b, c]].reshape(9), v[[a, c, d]].reshape(9)]
    return np.array(tris, np.float32)


def _quad(x0, x1, y0, y1, z):
    a, b, c, d = (x0, y0, z), (x1, y0, z), (x1, y1, z), (x0, y1, z)
    return np.array([a + b + c, a + c + d], np.float32)


def _plane_gbuffer(roughness=0.5):
    g = pyhr.GBufferHost(W, H)
    g.depth[:] = 0.5
    g.gb2[:] = 0
    g.gb2[..., 0] = np.float16(0.0).view(np.uint16)  # octahedral (0, 0) = +z
    g.gb2[..., 1] = np.float16(0.0).view(np.uint16)
    g.gb3[:] = 0
    g.gb3[..., 0] = np.float16(roughness).view(np.uint16)
    return O.GBufMips(g, 1)


def _frame(light_dir=(0.0, 0.0, 1.0), radius=0.1):
    f = pyhr.hr_frame()
    for i in range(4):
        f.ubo.view_proj_inverse[5 * i] = 1.0
    f.ubo.light.data0[0], f.ubo.light.data0[1], f.ubo.light.data0[2], f.ubo.light.data0[3] = (*light_dir, 1.0)
    f.ubo.light.data1[3] = radius
    f.ubo.light.data3[0] = 0.0  # directional
    return f


def test_plane_normal_is_up():
    e = np.zeros(2, np.float32)
    out = np.empty(3, np.float32)
    O.lib().orc_oct_decode(O.p(e), 1, O.p(out))
    assert out.tolist() == [0.0, 0.0, 1.0]


def _count(tris, kind, frame, n, p0, p1=0.0, k0=0):
    sc = O.Scene(tris)
    c = np.zeros((H, W), np.uint32)
    return R.reference_mask(sc, _plane_gbuffer(), frame, kind, p0, p1, k0, n, c)


def test_ao_of_an_unoccluded_plane_is_one():
    far = _quad(100, 101, 100, 101, -50)  # one triangle far below: nothing above the plane
    assert (_count(far, "ao", _frame(), 64, 7.0, 0.3) == 64).all()


def test_ao_inside_a_closed_box_is_zero():
    assert (_count(_box(-2.0, 2.0), "ao", _frame(), 64, 7.0, 0.3) == 0).all()


def test_shadows_with_the_light_below_the_horizon_are_zero():
    far = _quad(100, 101, 100, 101, -50)
    assert (_count(far, "shadows", _frame(light_dir=(0.0, 0.0, -1.0)), 64, 0.5) == 0).all()


def test_shadows_behind_a_symmetric_edge_are_one_half():
    x = 7
    px = np.float32((x + 0.5) / W * 2 - 1)
    occ = _quad(-10.0, float(px), -10.0, 10.0, 2.0)  # covers world x < px at z = 2: the edge halves the light's disk at pixel column x
    N = 4096
    c = _count(occ, "shadows", _frame(radius=0.2), N, 0.5)
    m, se = R.mean_and_stderr(c, N)
    assert (c[:, x + 2:] == N).all() and (c[:, :x - 1] == 0).all()
    assert np.all(np.abs(m[:, x] - 0.5) <= 4 * np.sqrt(0.25 / N)), m[:, x]


@pytest.mark.parametrize("kind", ["shadows", "ao"])
def test_sample_split_is_invariant(kind):
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    tri, _ = sc.world_triangles()
    osc = O.Scene(tri)
    Wt, Ht = 40, 24
    f = pyhr.make_frame((0, 14, 34), (0, 3, 0), Wt, Ht)
    g = O.GBufMips(pyhr.write_gbuffer(sc, f, Wt, Ht), 1)
    p0, p1 = (0.5, 0.0) if kind == "shadows" else (7.0, 0.3)
    whole = R.reference_mask(osc, g, f, kind, p0, p1, 0, 256, np.zeros((Ht, Wt), np.uint32))
    split = np.zeros((Ht, Wt), np.uint32)
    R.reference_mask(osc, g, f, kind, p0, p1, 0, 64, split)
    R.reference_mask(osc, g, f, kind, p0, p1, 64, 192, split)
    assert np.array_equal(whole, split)
    assert 0 < whole.sum() < 256 * Wt * Ht  # neither all occluded nor all visible


def test_mirror_reflections_have_zero_stderr_and_equal_one_k12_ray():
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ss = O.ShadingScene(sc)
    Wt, Ht = 32, 20
    f = pyhr.make_frame((0, 14, 34), (0, 3, 0), Wt, Ht)
    gh = pyhr.write_gbuffer(sc, f, Wt, Ht)
    gh.gb3[..., 0] = np.float16(0.02).view(np.uint16)
    g = O.GBufMips(gh, 1)
    prm = pyhr.hr_reflections_params()
    prm.bias, prm.trim, prm.gi_intensity, prm.rough_ddgi_intensity = 0.5, 0.8, 0.5, 0.5
    prm.sky_color[0], prm.sky_color[1], prm.sky_color[2] = 0.3, 0.5, 0.9
    N = 37
    acc = R.reference_reflections(ss, g, f, prm, 0, N, np.zeros((Ht, Wt, 6), np.float64))
    m, se = R.mean_and_stderr(acc, N)
    k12 = np.zeros((Ht, Wt, 4), np.uint16)
    sky = np.array(prm.sky_color[:], np.float32)
    bn = pyhr.blue_noise()
    gc = g.c(0)
    O.lib().orc_reflections_ray_trace(ss.h, O.C.byref(gc), O.C.byref(f), prm.bias, prm.trim, 0, 0, prm.gi_intensity, prm.rough_ddgi_intensity, O.p(sky),
                                      O.p(bn[0]), O.p(bn[1]), None, None, None, O.p(k12))
    surf = gh.depth != 1.0
    assert surf.any()
    assert (se[surf] == 0).all()
    assert np.array_equal(m[surf].astype(np.float16), O.h2f(k12)[..., :3][surf].astype(np.float16))


@pytest.mark.parametrize("kind", ["shadows", "ao"])
def test_the_blue_noise_mean_of_256_frames_lies_within_the_bound(kind):
    """the bound test_gpu_reference.py holds the device to, checked on the oracle: 256 frames of the one-ray mask (one blue-noise
    period, static camera) against a 4096-sample reference"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    osc = O.Scene(sc.world_triangles()[0])
    Wt, Ht = 64, 48
    frames = [pyhr.make_frame((0, 14, 34), (0, 3, 0), Wt, Ht, num_frames=i) for i in range(256)]
    g = O.GBufMips(pyhr.write_gbuffer(sc, frames[0], Wt, Ht), 1)
    p0, p1 = (0.5, 0.0) if kind == "shadows" else (7.0, 0.3)
    bn = pyhr.blue_noise()
    bnm = R.blue_noise_mean(osc, g, frames, kind, p0, p1, bn)
    N = 4096
    p, se = R.mean_and_stderr(R.reference_mask(osc, g, frames[0], kind, p0, p1, 0, N, np.zeros((Ht, Wt), np.uint32)), N)
    surf = g.levels[0][4] != 1.0
    err = float(np.sqrt(np.mean((bnm - p)[surf] ** 2)))
    bound = R.blue_noise_bound(p[surf], se[surf], 256)
    assert err <= bound, (err, bound)
    assert err > 0  # the blue noise is not the reference's random stream
