"""Parameter cases shared by tests/test_gpu_parameters.py (device vs oracle) and tests/test_param_sensitivity_cpu.py (the oracle
reacts to each case).  Numbers and names only, no GPU.

A continuous case changes ONE parameter of one pass away from its default, so that a kernel that ignores the parameter, inverts
it, or reads its neighbour in the parameter block (alpha 0.01 in three passes, moments_alpha 0.2 in two, bias 0.5 in shadows and
reflections, power 1.2 in shadows and AO, sigma_depth and DDGI gi_intensity 1) renders something the oracle does not.  `stage` is
where the parameter acts: the sensitivity test requires the oracle's image there to move by at least 10x a bar (RMSE or max-abs)
the GPU test applies to it.  The GPU test compares every stage of the chain, not only that one.

The layout cases change the DDGI probe grid (rays_per_probe, irradiance_oct_size, depth_oct_size) to the extremes the API accepts;
probe_distance keeps the oracle's rays per frame near the default test's 867 probes x 256 rays.
"""
from collections import namedtuple

import pyhr

SIZE = (256, 144)  # even widths, phi_normal 32, radius 1: the fast default a-trous / blur kernels run

# name -> scene kind, triangles, camera (position, target), default_light overrides (None: the synthetic frame's light);
# the cameras and lights of test_gpu_ragged
SCENES = {
    "shadows_test": (pyhr.SCENE_SHADOWS_TEST, 0, ((0.0, 14.0, 34.0), (0.0, 3.0, 0.0)), None),
    "arcade": (pyhr.SCENE_ARCADE, 20000, ((0.0, 9.0, -4.0), (2.0, 7.0, 60.0)), dict(rot_x_deg=25.0)),
    # the arcade plus one triangle beyond its lower corner (test_gpu_parameters.arcade_lifted_grid): no wall or floor on a probe plane
    "arcade_lifted": (pyhr.SCENE_ARCADE, 20000, ((0.0, 9.0, -4.0), (2.0, 7.0, 60.0)), dict(rot_x_deg=25.0)),
}


def scene_kw(name):
    """the scene keywords of test_gpu_ragged's runners"""
    kind, tris, cam, light = SCENES[name]
    return dict(scene=kind, tris=tris, cam=cam, light=pyhr.default_light(**light) if light else None)

# stage -> (RMSE bar, max-abs bar) of the GPU comparison.  DDGI and reflections: test_gpu_gi_refl.close (relative to
# max(1, |reference|)), shadows and AO: test_gpu_parity.check_all (absolute; it bounds the shadows' final image by RMSE only).
BARS = {
    "ddgi radiance": (2e-3, 0.05), "ddgi irradiance": (1e-3, 6e-3), "ddgi depth": (2e-3, 0.05), "ddgi sample": (1e-3, 6e-3),
    "rt": (1e-3, 0.02), "temporal": (1e-3, 6e-3), "moments": (1e-3, 6e-3), "a-trous": (1e-3, 6e-3), "final": (1e-3, 6e-3),
    "sh temporal": (1e-3, 2e-3), "sh a-trous": (1e-3, 4e-3), "ao temporal": (1e-3, 2e-3), "ao blur": (1e-3, 4e-3), "ao final": (1e-3, 4e-3),
}
RELATIVE = {"ddgi radiance", "ddgi irradiance", "ddgi depth", "ddgi sample", "rt", "temporal", "moments", "a-trous", "final"}

# kind: "shadows" / "ao" (one run of both chains, shadows at scale 0, AO at scale 1, like test_shadows_parameters),
# "reflections" (scale 0), "ddgi" (DDGI sampled at the reflections' scale 0, reflections reading it).
# ddgi: the reflections read a DDGI pass; lut: the synthetic BRDF LUT is set (IBL specular term); kernels: what the profiler
# must see the pass launch (the fast kernels, not the fallbacks test_gpu_ragged covers).
Case = namedtuple("Case", "id kind params frames scene stage kernels ddgi lut", defaults=(False, False))

SH_KERNELS = ("k_atrous_v3",)
AO_KERNELS = ("k_ao_blur_v2",)
RF_KERNELS = ("k_refl_atrous_tma", "k_refl_atrous_v2")


def _sh(name, value, stage):
    return Case(f"shadows {name} {value}", "shadows", {name: value}, 6, "shadows_test", stage, SH_KERNELS)


def _ao(name, value, stage):
    return Case(f"ao {name} {value}", "ao", {name: value}, 6, "shadows_test", stage, AO_KERNELS)


def _rf(name, value, stage, ddgi=False, lut=False):
    return Case(f"reflections {name} {value}", "reflections", {name: value}, 6, "arcade" if ddgi else "shadows_test", stage, RF_KERNELS, ddgi, lut)


def _dd(name, value, stage, frames=5):
    return Case(f"ddgi {name} {value}", "ddgi", {name: value}, frames, "arcade", stage, RF_KERNELS, True)


# The temporal stages blend with max(alpha, 1 / history length): over 6 frames an alpha or moments_alpha below 1/6 acts like the
# default, so those cases go above it.  The a-trous depth weight is the reference's exp(-exp(-|dz| / sigma_depth)), bounded to
# [1/e, 1]: sigma_depth moves the filtered image by a few 1e-3 RMSE at most, and its cases are held to the max-abs bar.
CONTINUOUS = [
    _sh("bias", 0.05, "sh temporal"), _sh("bias", 2.0, "sh temporal"),
    _sh("alpha", 0.6, "sh temporal"),
    _sh("moments_alpha", 0.8, "sh a-trous"),
    _sh("phi_visibility", 2.0, "sh a-trous"), _sh("phi_visibility", 40.0, "sh a-trous"),
    _sh("sigma_depth", 0.25, "sh a-trous"), _sh("sigma_depth", 4.0, "sh a-trous"),
    _sh("power", 1.0, "sh a-trous"), _sh("power", 3.0, "sh a-trous"),  # the last a-trous iteration raises to `power`
    _ao("ray_length", 0.5, "ao temporal"), _ao("ray_length", 30.0, "ao temporal"),
    _ao("bias", 0.05, "ao temporal"), _ao("bias", 1.0, "ao temporal"),
    _ao("alpha", 0.6, "ao temporal"),
    _ao("power", 3.0, "ao final"),  # applied by the upsample only: AO runs at scale 1
    _rf("bias", 0.1, "rt"), _rf("bias", 1.5, "rt"),
    _rf("trim", 0.3, "rt"), _rf("trim", 1.0, "rt"),  # 1.0: the GGX sample's E.y reaches the grazing limit
    _rf("gi_intensity", 2.0, "rt", ddgi=True),
    _rf("rough_ddgi_intensity", 2.0, "rt", ddgi=True),
    _rf("sample_gi", 0, "rt", ddgi=True),
    _rf("alpha", 0.6, "temporal"),
    _rf("moments_alpha", 0.8, "moments"),
    _rf("phi_color", 2.0, "a-trous"), _rf("phi_color", 50.0, "a-trous"),
    _rf("sigma_depth", 0.1, "a-trous"), _rf("sigma_depth", 10.0, "a-trous"),
    _rf("ibl_indirect_specular_intensity", 1.0, "rt", ddgi=True, lut=True),  # the IBL term is added where sample_gi reads DDGI
    _dd("visibility_test", 0, "ddgi sample"),
    _dd("infinite_bounces", 0, "ddgi radiance"),
    _dd("infinite_bounce_intensity", 0.5, "ddgi radiance"),
    _dd("hysteresis", 0.0, "ddgi irradiance"), _dd("hysteresis", 0.5, "ddgi irradiance"),
    _dd("hysteresis", 1.0, "ddgi irradiance", frames=16),  # the default 0.98 drifts 2 % a frame from the first frame's atlas
    _dd("depth_sharpness", 1.0, "ddgi depth"), _dd("depth_sharpness", 200.0, "ddgi depth"),
    _dd("normal_bias", 0.0, "ddgi sample"),
    _dd("recursive_energy_preservation", 0.5, "ddgi sample"),  # scales every sample_irradiance (K21, K18's bounce, K12's rough lobe)
    _dd("gi_intensity", 2.5, "ddgi sample"),
]


def _layout(rays, irr, dep, probe_distance, what, scene="arcade", frames=4):
    return Case(f"ddgi layout {rays} rays {irr}/{dep} ({what})", "ddgi",
                dict(rays_per_probe=rays, irradiance_oct_size=irr, depth_oct_size=dep, probe_distance=probe_distance), frames, scene, None, RF_KERNELS, True)


# arcade bounds 60 x 28.5 x 128: probe_distance 2 -> 32 x 16 x 66 probes, 4 -> 17 x 9 x 34, 8 -> 9 x 5 x 18, 14 -> 6 x 4 x 11.
# One ray per probe leaves most depth texels at zero variance, so nearly every probe fails K21's Chebyshev test and sits at the
# 1e-6 weight floor (1e-6^3 / 0.04 after the < 0.2 rule).  On the arcade the floor (and the walls at the bounds) lie on probe planes: the trilinear
# weight of the probes above it is clamp(P.y / step, 0, 1) with P.y reconstructed from depth to within a few 1e-6, 0 on one side
# and ~1e-6 on the other, and that ~1e-6 alone decides whether a visible probe above outweighs the floored ones (RMSE 0.047 between
# the device and the oracle at frame 0, pixels flipping between 0 and a full probe value).  This layout therefore runs with one
# more triangle 0.7 beyond the scene's lower corner, which moves every probe plane off the floor and walls; the other layouts keep
# them on the planes.  It stops after the three static frames: on the first panning frame the same tie between a visible probe and
# the floored ones still flips one pixel (0.019 in three channels, RMSE inside the bar), more texels than bounded allows.
LAYOUTS = [
    _layout(1, 2, 2, 2.0, "4-thread K19 blocks, gutter loop longer than the block, one ray per probe", scene="arcade_lifted", frames=3),
    _layout(33, 6, 14, 4.0, "partial warp in K18, sides that are not powers of two"),
    _layout(257, 16, 32, 8.0, "K18 loops above 256 threads, 1024-thread depth blocks"),
    _layout(1024, 8, 16, 14.0, "the ray maximum: every shared staging slot"),
]


def ids(cases):
    return [c.id for c in cases]
