"""GPU parity of the path tracer's indirect mode (hr_path_tracer_params.trace_indirect = 1, DESIGN.md §7) through the C ABI against
oracle/orc_path_trace_indirect.cpp.  Bars: the primary primitive and the path hash (HR_PATH_TRACER_OUT_PATH_HASH: every segment's primitive
and the end code) equal the oracle's in every pixel and sample, because the lobe choice, the directions, the horizon tests and the
bounce rays follow the deterministic chain; colours within the bars of test_gpu_trace_ground_truth.py; rays_secondary equal to the
oracle's count of shadow plus bounce rays.  The closed-sphere furnace and the convex cube run again on the device against the numpy
values of tests/pt_indirect.py."""
import ctypes as C

import numpy as np
import pytest

import light_cases as LC
import oracle as O
import pyhr
import pt_indirect as PI
from test_gpu_trace_ground_truth import compare
from test_path_tracer_indirect_cpu import (F_INTENSITY, F_SAMPLES, FH, FURNACE_MATERIALS, FW, LIGHTS, SKY, check_convex_paths, cube_frames, cube_mesh,
                                           f16, furnace_frame)
from test_textures_cpu import textured_scene

pytestmark = pytest.mark.gpu


def set_params(pt, B, trace_indirect=1, roughness_multiplier=1.0):
    pt.params.sky_color[0], pt.params.sky_color[1], pt.params.sky_color[2] = SKY
    pt.params.max_ray_bounces, pt.params.trace_indirect, pt.params.roughness_multiplier = B, trace_indirect, roughness_multiplier


def run_parity(ctx, ss, frames, W, H, B, samples, roughness_multiplier=1.0, what=""):
    pt = pyhr.PathTracerPass(ctx, W, H)
    set_params(pt, B, roughness_multiplier=roughness_multiplier)
    opt = PI.IndirectPathTracerOracle(W, H, max_ray_bounces=B, roughness_multiplier=roughness_multiplier, sky=SKY)
    pt.stats()
    for i in range(samples):
        f = frames[i % len(frames)]
        pt.render(f)
        want = opt.render(ss, f)
        assert np.array_equal(pt.download(1), opt.prim), f"{what} sample {i}: primary hits differ in {np.count_nonzero(pt.download(1) != opt.prim)} pixels"
        got_hash = pt.download(2)
        assert np.array_equal(got_hash, opt.hash), f"{what} sample {i}: paths differ in {np.count_nonzero(got_hash != opt.hash)} pixels"
        compare(f16(pt.download(100)), f16(want), f"{what} sample {i}")
    st = pt.stats()
    assert st.renders == samples and st.rays_primary == samples * W * H, what
    assert st.rays_secondary == opt.secondary_rays, f"{what}: {st.rays_secondary} secondary rays, the oracle traced {opt.secondary_rays}"
    pt.destroy()
    return opt


@pytest.fixture(scope="module")
def shadows():
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    ctx.build_scene(sc)
    yield ctx, ss
    ctx.close()


# the spot / overhead-sun / horizon-sun / coloured cases of light_cases.py after the two of the CPU tests
LIGHT_CASES = ["spot_band", "sun_overhead", "sun_horizon", "colored"]
LIGHTS = LIGHTS + [LC.BY_ID[c].kw for c in LIGHT_CASES]
LIGHT_IDS = ["directional", "point"] + LIGHT_CASES


@pytest.mark.parametrize("size", [(192, 112), (251, 141)], ids=["192x112", "251x141"])
@pytest.mark.parametrize("light_kw", LIGHTS, ids=LIGHT_IDS)
@pytest.mark.parametrize("B", [2, 4])
def test_indirect_matches_the_oracle(shadows, size, light_kw, B):
    ctx, ss = shadows
    W, H = size
    light = pyhr.default_light(**light_kw)
    frames = [pyhr.make_frame((0.0, 14.0, 34.0), (0.0, 3.0, 0.0), W, H, light=light)]
    opt = run_parity(ctx, ss, frames, W, H, B, 4, what=f"{W}x{H} B={B}")
    assert opt.secondary_rays > 4 * np.count_nonzero(opt.prim != 0xFFFFFFFF)  # the bounces were traced


@pytest.mark.parametrize("roughness_multiplier", [0.0, 0.5])
def test_indirect_roughness_multiplier(shadows, roughness_multiplier):
    """0: the as-written D_ggx is 0 everywhere, every specular sample ends the path (its pdf is not positive)"""
    ctx, ss = shadows
    W, H = 192, 112
    light = pyhr.default_light(type=1, position=(4.0, 12.0, 6.0), radius=0.5, intensity=300.0)
    frames = [pyhr.make_frame((3.0, 10.0, 30.0), (0.0, 3.0, 0.0), W, H, light=light)]
    run_parity(ctx, ss, frames, W, H, 4, 3, roughness_multiplier=roughness_multiplier, what=f"roughness x {roughness_multiplier}")


def test_indirect_with_material_textures():
    """the TEX instantiation: textures change albedo, roughness, metallic (the lobe choice) and the normal (the directions)"""
    sc, asc, textures, bindings = textured_scene()
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    ss.set_textures(textures, bindings, asc.primitive_uvs(), asc.primitive_tangent_frames())
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    scene = ctx.build_scene(asc)
    ctx.set_textures(scene, textures, bindings)
    W, H = 192, 112
    frames = [pyhr.make_frame((0.05 * i, 14.0, 34.0), (0.0, 3.0, 0.0), W, H) for i in range(3)]
    run_parity(ctx, ss, frames, W, H, 3, 3, what="textured")
    ctx.close()


def test_furnace_and_convex_on_the_device():
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    tris, vn = PI.icosphere(4)
    for m in FURNACE_MATERIALS:
        want = PI.furnace_expected(m[0], m[1], m[2], F_INTENSITY, 10.0, (1, 2, 3, 4, 8), n_mu=128, n_phi=256)
        mesh = PI.MeshScene(tris, vn, (m[0],) * 3, m[1], m[2])
        ctx.build_scene(mesh.array_scene)
        ss = O.ShadingScene(mesh)
        f = furnace_frame(FW, FH)
        for B in (1, 2, 3, 4, 8):
            pt = pyhr.PathTracerPass(ctx, FW, FH)
            set_params(pt, B)
            for i in range(F_SAMPLES):
                pt.render(f)
                if i == 0 and B == 8:  # the device walks the oracle's paths in the closed sphere too
                    opt = PI.IndirectPathTracerOracle(FW, FH, max_ray_bounces=B, sky=SKY)
                    opt.render(ss, f)
                    assert np.array_equal(pt.download(2), opt.hash)
            got = float(f16(pt.download(100))[..., :3].astype(np.float64).mean())
            assert abs(got / want[B] - 1.0) <= 0.01, f"material {m} B={B}: image mean {got}, recursion {want[B]}"
            pt.destroy()
    # convex cube: B = 4 renders B = 1 bit for bit, no bounce ray hits
    ctx.build_scene(cube_mesh().array_scene)
    W, H = 96, 64
    for f in cube_frames(W, H):
        p1, p4 = pyhr.PathTracerPass(ctx, W, H), pyhr.PathTracerPass(ctx, W, H)
        set_params(p1, 1)
        set_params(p4, 4)
        for i in range(3):
            p1.render(f)
            p4.render(f)
            assert np.array_equal(p1.download(100), p4.download(100)), f"sample {i}"
            check_convex_paths(p4.download(1), p4.download(2), f"device sample {i}")
        p1.destroy()
        p4.destroy()
    ctx.close()


def test_one_vertex_is_mode_0_and_restart(shadows):
    ctx, ss = shadows
    W, H = 192, 112
    f = pyhr.make_frame((0.0, 14.0, 34.0), (0.0, 3.0, 0.0), W, H, light=pyhr.default_light(type=1, position=(4.0, 12.0, 6.0), radius=0.5, intensity=300.0))
    m0, m1 = pyhr.PathTracerPass(ctx, W, H), pyhr.PathTracerPass(ctx, W, H)
    set_params(m0, 1, trace_indirect=0)
    set_params(m1, 1)
    m0.stats()
    m1.stats()
    for i in range(3):
        m0.render(f)
        m1.render(f)
        assert np.array_equal(m0.download(100), m1.download(100)), f"sample {i}"
    s0, s1 = m0.stats(), m1.stats()
    assert (s0.rays_primary, s0.rays_secondary) == (s1.rays_primary, s1.rays_secondary)  # the same rays
    # hr_pass_reset_history restarts the accumulation in mode 1: the image is sample 0 again
    set_params(m1, 3)
    m1.reset_history()
    m1.render(f)
    first = PI.IndirectPathTracerOracle(W, H, max_ray_bounces=3, sky=SKY)
    want = first.render(ss, f)
    assert np.array_equal(m1.download(2), first.hash)
    compare(f16(m1.download(100)), f16(want), "after restart")
    m0.destroy()
    m1.destroy()


def test_invalid_parameters_are_refused(shadows):
    ctx, ss = shadows
    W, H = 64, 48
    f = pyhr.make_frame((0.0, 14.0, 34.0), (0.0, 3.0, 0.0), W, H)
    pt = pyhr.PathTracerPass(ctx, W, H)
    lib = pt.lib

    def rc(B, ti):
        set_params(pt, B, trace_indirect=ti)
        return lib.hr_path_tracer_render(pt.h, C.byref(f), C.byref(pt.params), None)

    for B, ti in ((2, 2), (2, -1), (32, 1), (0, 1), (0, 0)):
        assert rc(B, ti) == -1, (B, ti)  # HR_ERR_INVALID_ARG
        assert rc(2, 1) == 0  # the next valid render succeeds
    assert rc(32, 0) == 0 and rc(31, 1) == 0  # mode 0 validates as before; 31 vertices is the limit
    ref = PI.IndirectPathTracerOracle(W, H, max_ray_bounces=2, sky=SKY)
    pt.reset_history()
    assert rc(2, 1) == 0
    ref.render(ss, f)
    assert np.array_equal(pt.download(2), ref.hash)
    pt.destroy()
