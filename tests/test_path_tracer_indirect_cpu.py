"""The path tracer's indirect mode (hr_path_tracer_params.trace_indirect = 1, DESIGN.md §7) on the CPU: its oracle
(oracle/orc_path_trace_indirect.cpp) against closed forms computed independently in numpy (tests/pt_indirect.py), and the properties the
estimator must have whatever the scene: B = 1 is mode 0 (oracle/orc_path_trace.cpp) bit for bit, more bounces never darken a sample, a convex object has no
indirect light."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
import pyhr
import pt_indirect as PI

SKY = (0.3, 0.4, 0.6)
FW, FH, F_SAMPLES, F_INTENSITY = 64, 48, 64, 4.0
FURNACE_MATERIALS = [(0.8, 0.7, 0.0), (0.8, 0.1, 1.0)]  # (grey albedo, roughness, metallic)


def f16(a):
    return np.ascontiguousarray(a).view(np.float16).astype(np.float32)


@pytest.fixture(scope="module")
def sphere():
    return PI.icosphere(4)  # 5120 triangles, radius 10


@pytest.fixture(scope="module")
def furnace_values():
    return {m: PI.furnace_expected(m[0], m[1], m[2], F_INTENSITY, 10.0, (1, 2, 3, 4, 8), n_mu=128, n_phi=256) for m in FURNACE_MATERIALS}


def furnace_frame(W, H):
    light = pyhr.default_light(type=1, position=(0.0, 0.0, 0.0), radius=0.0, intensity=F_INTENSITY, color=(1.0, 1.0, 1.0))
    return pyhr.make_frame((0.0, 0.0, 0.0), (1.0, 0.3, 0.2), W, H, light=light)


def test_default_params_keep_the_reference():
    p = pyhr.hr_path_tracer_params()
    p.trace_indirect = 7
    pyhr.load_product().hr_path_tracer_default_params(C.byref(p))
    assert p.trace_indirect == 0 and p.max_ray_bounces == 2
    assert pyhr.hr_path_tracer_params.trace_indirect.offset == 20 and C.sizeof(pyhr.hr_path_tracer_params) == 24  # appended after sky_color


def test_quadrature_is_converged():
    for m in FURNACE_MATERIALS:
        a = PI.furnace_expected(m[0], m[1], m[2], F_INTENSITY, 10.0, (1, 8), n_mu=128, n_phi=256)
        b = PI.furnace_expected(m[0], m[1], m[2], F_INTENSITY, 10.0, (1, 8), n_mu=256, n_phi=512)
        assert all(abs(a[k] / b[k] - 1.0) < 1e-4 for k in a)
    # B = 1 at normal incidence has a closed form: metallic 1, roughness 0.1 -> D_ggx clamps to 1, G = 1, F = F0: f = F0 / 4
    assert PI.furnace_expected(0.8, 0.1, 1.0, 4.0, 10.0, (1,))[1] == pytest.approx(0.8 / 4.0 * 4.0 / 100.0, rel=1e-12)


@pytest.mark.parametrize("material", FURNACE_MATERIALS, ids=["diffuse_r0.7", "metal_r0.1"])
@pytest.mark.parametrize("bounces", [1, 2, 3, 4, 8])
def test_closed_sphere_furnace(sphere, furnace_values, material, bounces):
    """inward-facing sphere, point light of radius 0 and camera at its centre: the image mean is L_B(0) of the 1-D recursion"""
    mesh = PI.MeshScene(*sphere, (material[0],) * 3, material[1], material[2])
    ss = O.ShadingScene(mesh)
    f = furnace_frame(FW, FH)
    o = PI.IndirectPathTracerOracle(FW, FH, max_ray_bounces=bounces, sky=SKY)
    for i in range(F_SAMPLES):
        img = f16(o.render(ss, f))
        if i == 0:
            assert img[..., :3].max() < 0.9  # the per-sample clamp at RADIANCE_CLAMP_COLOR does not bind
            assert np.all(o.prim != 0xFFFFFFFF)
    want = furnace_values[material][bounces]
    got = float(img[..., :3].astype(np.float64).mean())
    assert abs(got / want - 1.0) <= 0.01, f"B={bounces}: image mean {got}, recursion {want}"
    # the sky contributes exactly 0: every sky shadow ray hits the wall
    dark = PI.IndirectPathTracerOracle(FW, FH, max_ray_bounces=bounces, sky=(0.0, 0.0, 0.0))
    lit = PI.IndirectPathTracerOracle(FW, FH, max_ray_bounces=bounces, sky=SKY)
    assert np.array_equal(dark.render(ss, f), lit.render(ss, f))


def cube_mesh():
    return PI.MeshScene(*PI.cube(), (0.7, 0.5, 0.3), 0.4, 0.3)


def cube_frames(W, H):
    light = pyhr.default_light(type=1, position=(3.0, 9.0, 7.0), radius=0.5, intensity=120.0)
    return [pyhr.make_frame((1.5, 4.0, 8.0), (0.0, 1.0, 0.0), W, H, light=light), pyhr.make_frame((-6.0, 5.0, 5.0), (0.0, 1.0, 0.0), W, H)]


def check_convex_paths(prim, hash_, what):
    """every path has one segment.  It ends in a miss, or (a GGX half vector far from N reflects Wo below the face) below the horizon"""
    hit = prim != 0xFFFFFFFF
    miss = PI.one_segment_hash(prim)
    horizon = PI.fnv1a(PI.fnv1a(PI.FNV_BASIS, prim), PI.END_HORIZON).astype(np.uint32)
    assert np.all((hash_ == miss) | (hit & (hash_ == horizon))), f"{what}: a bounce ray hit the convex object"
    assert np.count_nonzero(hash_[hit] == miss[hit]) >= 0.9 * np.count_nonzero(hit), what


def test_convex_object_has_no_indirect_light():
    """a bounce leaves a convex object's face through the face's upper half space: B = 4 renders B = 1 bit for bit, and no bounce ray hits"""
    ss = O.ShadingScene(cube_mesh())
    W, H = 96, 64
    for f in cube_frames(W, H):
        o1 = PI.IndirectPathTracerOracle(W, H, max_ray_bounces=1, sky=SKY)
        o4 = PI.IndirectPathTracerOracle(W, H, max_ray_bounces=4, sky=SKY)
        for i in range(3):
            assert np.array_equal(o1.render(ss, f), o4.render(ss, f)), f"sample {i}"
            check_convex_paths(o4.prim, o4.hash, f"sample {i}")
            assert np.count_nonzero(o4.prim != 0xFFFFFFFF) > 0.1 * W * H


@pytest.fixture(scope="module")
def shadows_scene():
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    return sc, O.ShadingScene(sc, brute=True)


LIGHTS = [{}, dict(type=1, position=(4.0, 12.0, 6.0), radius=0.5, intensity=300.0)]


@pytest.mark.parametrize("light_kw", LIGHTS, ids=["directional", "point"])
def test_more_bounces_never_darken_the_first_sample(shadows_scene, light_kw):
    sc, ss = shadows_scene
    W, H = 64, 36
    f = pyhr.make_frame((0, 14, 34), (0, 3, 0), W, H, light=pyhr.default_light(**light_kw))
    imgs, hashes = [], []
    for B in (1, 2, 3, 4):
        o = PI.IndirectPathTracerOracle(W, H, max_ray_bounces=B, sky=SKY)
        imgs.append(f16(o.render(ss, f))[..., :3])
        hashes.append(o.hash.copy())
    for a, b in zip(imgs, imgs[1:]):
        assert np.all(b >= a)
    assert imgs[3].mean() > imgs[0].mean()
    # B = 1: one vertex, then the max-bounces end code; longer paths extend it
    hit = (o.prim != 0xFFFFFFFF)
    want1 = np.where(hit, PI.fnv1a(PI.fnv1a(PI.FNV_BASIS, o.prim), PI.END_MAX_BOUNCES), PI.fnv1a(PI.FNV_BASIS, PI.END_MISS)).astype(np.uint32)
    assert np.array_equal(hashes[0], want1)
    assert np.mean(hashes[3] != hashes[0]) > 0.3


@pytest.mark.parametrize("light_kw", LIGHTS, ids=["directional", "point"])
def test_one_vertex_is_mode_0_bit_for_bit(shadows_scene, light_kw):
    sc, ss = shadows_scene
    W, H = 64, 36
    f = pyhr.make_frame((0, 14, 34), (0, 3, 0), W, H, light=pyhr.default_light(**light_kw))
    m0 = O.PathTracerOracle(W, H, max_ray_bounces=1, sky=SKY)
    m1 = PI.IndirectPathTracerOracle(W, H, max_ray_bounces=1, sky=SKY)
    for i in range(3):
        assert np.array_equal(m0.render(ss, f), m1.render(ss, f)), f"sample {i}"
        assert np.array_equal(m0.prim, m1.prim)
    assert m1.secondary_rays > 0
