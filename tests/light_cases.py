"""Light cases shared by tests/test_gpu_lights.py and the other GPU tests that take a light (device vs oracle), and by
tests/test_light_sensitivity_cpu.py (the oracle reacts to each case).  Numbers and names only, no GPU.

The light is hr_frame.ubo.light (lighting.glsl's Light: direction + intensity, position + radius, colour, type + cone cosines),
built by pyhr.default_light(**kw) + make_frame.  Three pieces of device code evaluate it: the soft shadow-ray form
(det_math.cuh fetch_light_properties_shadow: the shadows mask, the path tracer's direct term), the hard form with Li
(rt_shade.cu fetch_light_properties_hard: K12 reflection hits, K18 probe rays) and the raster form inline in deferred.cu.
A case moves the light to a place where one of them can go wrong: each light type, the cone's smoothstep band and its
degenerate forms, the soft disk near a point light, the sun at the zenith / horizon / below, a coloured light, non-finite
radiance, and a light that changes under a static camera.

`twin` is the case the sensitivity test requires the oracle to tell apart from this one at each of its `stages` (by at least
10x the GPU bar there, or in 1 % of the mask bits): so a device that evaluated the case as its twin would fail the GPU comparison.
"""
from collections import namedtuple

import pyhr

SIZE = (256, 144)
# name -> scene kind, triangles, camera (position, target): the scenes and cameras of test_gpu_ragged
SCENES = {
    "shadows_test": (pyhr.SCENE_SHADOWS_TEST, 0, ((0.0, 14.0, 34.0), (0.0, 3.0, 0.0))),
    "arcade": (pyhr.SCENE_ARCADE, 20000, ((0.0, 9.0, -4.0), (2.0, 7.0, 60.0))),
}

POINT, SPOT = 1, 2
HIGH = dict(position=(2.0, 12.0, 6.0), radius=2.5, intensity=500.0)   # test_gpu_parity.test_point_and_spot_lights
LOW = dict(position=(0.0, 0.25, 4.0), radius=0.5)                       # 0.25 above the floor, in front of the camera
DOWN = dict(rot_x_deg=0.0, rot_y_deg=0.0)                               # data0 = (0, 1, 0): a spot pointing down


def _moving(i):
    """turns 4 degrees a frame about the vertical; a point light at the sun's place in the sky for frames 0-2, a spot from
    frame 3 (the camera stays still: only the light changes the temporal stages' and the DDGI hysteresis' inputs)"""
    kw = dict(rot_x_deg=20.0, rot_y_deg=4.0 * i, position=(2.0 + 0.5 * i, 12.0, 6.0), radius=2.5, intensity=500.0, cone_inner_deg=25.0,
              cone_outer_deg=40.0)
    kw["type"] = POINT if i < 3 else SPOT
    return kw


# kw: default_light overrides, or a callable frame -> overrides; stages: where the sensitivity test looks ("mask": the
# shadows ray-trace bits, "sh temporal": the shadows' temporal stage, "rt": the K12 colours, "deferred": the combine's direct
# term, the shadows pass's output times direct_lighting)
Light = namedtuple("Light", "id kw scene twin stages")

CASES = [
    # ---- sun (directional): data0 = -(R_y R_x (0, -1, 0))
    Light("sun_default", {}, "shadows_test", "sun_below", ("mask",)),
    # data0 = (-0, 1, -0): soft_shadow_dir's tangent is normalize(cross(data0, (0, 1, 0))) = normalize(0) = NaN (lighting.glsl:40)
    Light("sun_overhead", dict(rot_x_deg=0.0, rot_y_deg=0.0), "shadows_test", "sun_near_overhead", ("mask",)),
    Light("sun_near_overhead", dict(rot_x_deg=0.01, rot_y_deg=0.0), "shadows_test", "sun_overhead", ("mask",)),
    Light("sun_horizon", dict(rot_x_deg=90.0), "shadows_test", "sun_grazing", ("mask",)),  # data0.y = -4.4e-8: N.Wi on the floor just below 0
    Light("sun_grazing", dict(rot_x_deg=89.5), "shadows_test", "sun_horizon", ("mask",)),  # att > 0 close to 0 on every floor pixel
    Light("sun_below", dict(rot_x_deg=180.0), "shadows_test", "sun_default", ("mask",)),   # att = 0 everywhere
    Light("sun_hard", dict(radius=0.0), "shadows_test", "sun_wide", ("sh temporal",)),
    Light("sun_wide", dict(radius=0.5), "shadows_test", "sun_hard", ("sh temporal",)),
    # ---- point: 1 / d^2
    Light("point_high", dict(type=POINT, **HIGH, **DOWN), "shadows_test", "spot_band", ("mask",)),
    Light("point_low", dict(type=POINT, **LOW, intensity=20.0), "shadows_test", "point_high", ("deferred",)),  # radius / dist > 1 near the light
    # ---- spot: smoothstep(cos_outer, cos_inner, dot(Wi, data0)) / d^2
    Light("spot_band", dict(type=SPOT, **HIGH, **DOWN, cone_inner_deg=20.0, cone_outer_deg=35.0), "shadows_test", "point_high",
          ("mask", "rt", "deferred")),
    # (x - e0) / 0: +-inf, NaN exactly on the edge; the clamp takes both to [0, 1]
    Light("spot_hard_edge", dict(type=SPOT, **HIGH, **DOWN, cone_inner_deg=30.0, cone_outer_deg=30.0), "shadows_test", "spot_band", ("deferred",)),
    Light("spot_reversed", dict(type=SPOT, **HIGH, **DOWN, cone_inner_deg=35.0, cone_outer_deg=20.0), "shadows_test", "spot_band", ("mask",)),
    Light("spot_away", dict(type=SPOT, **HIGH, rot_x_deg=180.0, rot_y_deg=0.0, cone_inner_deg=20.0, cone_outer_deg=35.0), "shadows_test",
          "spot_band", ("deferred",)),  # pointing up: att = 0 everywhere
    # ---- colour, intensity, non-finite, a changing light
    Light("colored", dict(color=(1.0, 0.25, 0.0625)), "shadows_test", "sun_default", ("deferred",)),
    Light("intensity_zero", dict(intensity=0.0), "shadows_test", "sun_default", ("deferred",)),  # att excludes intensity: rays still traced
    Light("point_overflow", dict(type=POINT, **LOW, intensity=1e5), "shadows_test", "point_low", ("rt",)),  # saturates fp16
    Light("moving", _moving, "shadows_test", "point_high", ("sh temporal",)),
    # ---- on the 20 000-triangle arcade, where every reflection lobe and the DDGI grid see the light
    Light("arcade_spot_band", dict(type=SPOT, position=(2.0, 20.0, 30.0), radius=1.0, intensity=2000.0, **DOWN, cone_inner_deg=20.0,
                                   cone_outer_deg=35.0), "arcade", "arcade_point_low", ("mask",)),
    Light("arcade_point_low", dict(type=POINT, position=(2.0, 0.25, 20.0), radius=0.5, intensity=20.0), "arcade", "arcade_spot_band", ("mask",)),
    Light("arcade_moving", _moving, "arcade", "arcade_spot_band", ("sh temporal",)),
]
BY_ID = {c.id: c for c in CASES}


def light(case, i=0):
    """the case's light descriptor at frame i"""
    kw = case.kw(i) if callable(case.kw) else case.kw
    return pyhr.default_light(**kw)


def light_arg(case):
    """what test_gpu_ragged.frames takes: one descriptor, or frame -> descriptor for a changing light"""
    return (lambda i: light(case, i)) if callable(case.kw) else light(case)


def scene_kw(case):
    """the scene keywords of test_gpu_ragged's runners"""
    kind, tris, cam = SCENES[case.scene]
    return dict(scene=kind, tris=tris, cam=cam, light=light_arg(case))


def ids(cases):
    return [c.id for c in cases]
