"""Camera cases shared by tests/test_gpu_camera.py (device vs oracle under camera motion) and tests/test_camera_sensitivity_cpu.py
(the oracle reacts to each case).  Numbers, names and host geometry only, no GPU.

Every other moving test pans the camera by 0.05 world units a frame under hrs_make_frame's fixed projection (60 degrees, near 1,
far 1000, up +Y): the image moves by a fraction of a pixel.  A case here moves it the ways a user does: yaw, pitch and roll in
place, dolly, a fast pan that carries history across the left edge, an orbit that disoccludes the background behind the
cylinders, a zoom, narrow and wide fields of view, other near / far planes, a near plane that clips geometry, and a cut with and
without hr_pass_reset_history.  Each path is 2 static frames (the history gets length), then N_FRAMES - 2 moving ones.

`targets` are the reprojection branches the case must reach, "kernel:branch", as the oracle's reproject() records them
(oracle.ReprojectCodes, ORC_RP_* in oracle/orc_glsl.h) in that kernel's temporal stage (K3 shadows at full resolution, K9 AO at
half resolution, K14 reflections), in at least MIN_PIXELS pixels on some frame that reads history: "out" history out of frame,
"trunc" a history_coord_floor component in (-1, 0) (ivec2() truncates it to 0 where floor gives -1), "sumw" some taps valid but
sumw < 0.01, "fallback" the 3x3 fallback valid, "invalid" no history.  Every case's K14 also reaches both the virtual-point and
the motion-vector reprojection.
`twins` are the wrong inputs the sensitivity test requires the oracle to tell apart: "zbp" the AO blur given z_buffer_params
[0], [1] in place of [2], [3]; "delta" K14 with a non-zero camera_delta; "mv0" the temporal stage with zero motion vectors.
"""
from collections import namedtuple

import numpy as np

import pyhr

SIZE = (256, 144)
N_FRAMES = 7
MIN_PIXELS = 20
SCENES = {
    "shadows_test": (pyhr.SCENE_SHADOWS_TEST, 0, ((0.0, 14.0, 34.0), (0.0, 3.0, 0.0))),
    "arcade": (pyhr.SCENE_ARCADE, 20000, ((0.0, 9.0, -4.0), (2.0, 7.0, 60.0))),
}
Pose = namedtuple("Pose", "pos target up fovy_deg near far")


def pose(pos, target, up=(0.0, 1.0, 0.0), fovy_deg=60.0, near=1.0, far=1000.0):
    return Pose(tuple(float(x) for x in pos), tuple(float(x) for x in target), tuple(float(x) for x in up), float(fovy_deg), float(near), float(far))


def _rot(axis, deg):
    """rotation matrix about a unit axis (Rodrigues), float64"""
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    t = np.radians(deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * (K @ K)


def _moving(i):
    """how far frame i is into the motion: 0 for the 2 static frames, then 1, 2, ..."""
    return max(0, i - 1)


def _base(scene):
    p, t = SCENES[scene][2]
    return np.array(p), np.array(t)


def yaw(deg, scene="shadows_test"):
    def path(i):
        p, t = _base(scene)
        return pose(p, p + _rot((0, 1, 0), deg * _moving(i)) @ (t - p))
    return path


def pitch(deg, scene="shadows_test"):
    def path(i):
        p, t = _base(scene)
        right = np.cross(t - p, (0, 1, 0))
        return pose(p, p + _rot(right, deg * _moving(i)) @ (t - p))
    return path


def roll(deg):
    def path(i):
        p, t = _base("shadows_test")
        return pose(p, t, up=_rot(t - p, deg * _moving(i)) @ np.array([0.0, 1.0, 0.0]))
    return path


def dolly(step):
    """step world units a frame along the view direction (> 0: in)"""
    def path(i):
        p, t = _base("shadows_test")
        d = (t - p) / np.linalg.norm(t - p)
        return pose(p + step * _moving(i) * d, t)
    return path


def pan(step, **proj):
    """a lateral pan of `step` world units a frame along +x (< 0: leftward), under the projection `proj`"""
    def path(i):
        p, t = _base("shadows_test")
        dx = np.array([step * _moving(i), 0.0, 0.0])
        return pose(p + dx, t + dx, **proj)
    return path


def orbit(deg, scene="shadows_test"):
    def path(i):
        p, t = _base(scene)
        return pose(t + _rot((0, 1, 0), deg * _moving(i)) @ (p - t), t)
    return path


def zoom(fov0, fov1):
    def path(i):
        p, t = _base("shadows_test")
        k = _moving(i) / (N_FRAMES - 2)
        return pose(p, t, fovy_deg=fov0 + (fov1 - fov0) * k)
    return path


def near_clip(i):
    """near plane 4 units from a camera 2 units above the floor and 4-8 units from the middle cylinder and the slab: the near plane
    cuts the floor at the bottom of the image and the cylinder; a slow pan"""
    dx = 0.05 * _moving(i)
    return pose((dx, 2.0, 16.0), (dx, 2.0, 0.0), near=4.0)


def cut(at, scene="shadows_test"):
    """the base camera, then from frame `at` the opposite side of the target (mirrored through the target's vertical axis, looking
    back), then a slow pan.  Every point the new camera sees is also in front of the old one (the scene ends before it): large,
    finite motion vectors (test_camera_sensitivity_cpu.test_cut_motion_vectors)"""
    def path(i):
        p, t = _base(scene)
        if i >= at:
            p = np.array([2 * t[0] - p[0], p[1], 2 * t[2] - p[2]])
            p[0] += 0.05 * (i - at)
        return pose(p, t)
    return path


Case = namedtuple("Case", "id path scene resets targets twins")

CASES = [
    Case("yaw_slow", yaw(0.5), "shadows_test", (), ("K3:out", "K3:trunc", "K3:invalid"), ("mv0", "delta")),
    Case("yaw_fast", yaw(6.0), "shadows_test", (), ("K3:out", "K3:trunc", "K3:invalid", "K9:out"), ("mv0", "delta")),
    Case("pitch_fast", pitch(-8.0), "shadows_test", (), ("K3:out", "K3:trunc", "K3:fallback", "K3:invalid", "K9:fallback"), ("mv0",)),
    Case("roll", roll(5.0), "shadows_test", (), ("K3:out", "K3:trunc", "K3:invalid"), ("mv0",)),
    Case("dolly_in", dolly(3.0), "shadows_test", (), ("K3:fallback", "K3:invalid", "K14:fallback"), ("mv0",)),
    Case("dolly_out", dolly(-3.0), "shadows_test", (), ("K3:out", "K3:trunc", "K3:fallback", "K3:invalid"), ("mv0",)),
    Case("pan_fast_left", pan(-1.0), "shadows_test", (), ("K3:out", "K3:trunc", "K3:sumw", "K3:fallback", "K3:invalid", "K14:sumw"), ("mv0",)),
    Case("orbit", orbit(5.0), "shadows_test", (), ("K3:out", "K3:trunc", "K3:fallback", "K3:invalid"), ("mv0",)),
    Case("zoom", zoom(60.0, 40.0), "shadows_test", (), ("K14:trunc",), ("mv0", "delta")),
    Case("fov20", pan(0.5, fovy_deg=20.0), "shadows_test", (), ("K3:out", "K3:fallback", "K3:invalid"), ("mv0",)),
    Case("fov100", pan(0.5, fovy_deg=100.0), "shadows_test", (), ("K3:out", "K3:invalid"), ("mv0",)),
    Case("near0.1_far100", pan(0.05, near=0.1, far=100.0), "shadows_test", (), (), ("zbp",)),
    Case("near4_far5000", pan(0.05, near=4.0, far=5000.0), "shadows_test", (), ("K14:trunc",), ("zbp",)),
    Case("near_clip", near_clip, "shadows_test", (), ("K3:out", "K3:invalid"), ("zbp",)),
    Case("cut", cut(3), "shadows_test", (), ("K3:out", "K3:trunc", "K3:fallback", "K3:invalid", "K9:fallback", "K14:fallback"), ("mv0",)),
    Case("cut_reset_odd", cut(3), "shadows_test", (3,), ("K3:trunc",), ()),
    Case("cut_reset_even", cut(4), "shadows_test", (4,), ("K3:trunc",), ()),
    # ---- on the 20 000-triangle arcade
    Case("arcade_orbit", orbit(5.0, "arcade"), "arcade", (), ("K3:out", "K3:trunc", "K3:fallback", "K3:invalid", "K14:sumw"), ("mv0",)),
    Case("arcade_pitch_fast", pitch(-8.0, "arcade"), "arcade", (), ("K3:out", "K3:trunc", "K3:fallback", "K3:invalid", "K14:sumw"), ("mv0",)),
    Case("arcade_cut", cut(3, "arcade"), "arcade", (), ("K3:out", "K3:trunc", "K3:invalid"), ()),  # after the cut the pan is sub-pixel: mv0 changes nothing
]
BY_ID = {c.id: c for c in CASES}


def ids(cases):
    return [c.id for c in cases]


def frames(case, W, H, light=None, n=N_FRAMES):
    """(i, hr_frame) along the case's path, each frame's prev the frame before (a cut included: no first_frame)"""
    f = None
    for i in range(n):
        ps = case.path(i)
        f = pyhr.make_frame(ps.pos, ps.target, W, H, prev=f, num_frames=i, light=light, up=ps.up, fovy_deg=ps.fovy_deg, near=ps.near, far=ps.far)
        yield i, f


def scene_kw(case):
    kind, tris, _ = SCENES[case.scene]
    return dict(scene=kind, tris=tris)


def motion(gb2):
    """the G-buffer's motion vectors (prev_uv - cur_uv) from gb2 (uint16 halves, z and w), float64"""
    return np.ascontiguousarray(gb2[..., 2:4]).view(np.float16).astype(np.float64)
