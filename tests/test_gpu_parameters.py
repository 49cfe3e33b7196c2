"""GPU parity at non-default parameter VALUES: the DDGI probe layouts the API accepts, one continuous parameter at a time in every
pass (param_cases.py), and the DDGI probe grid's lifecycle (re-initialisation, refused parameters, scene replacement).

Every stage is compared with the CPU oracle under the bars of the aligned-size tests, reused unchanged through test_gpu_ragged's
runners: `close` (test_gpu_gi_refl) for DDGI and reflections with DDGIUniforms bytes, probe ray directions / hit distances,
reflection ray lengths, tile flags and history lengths exact; check_all (test_gpu_parity) for shadows and AO.
test_param_sensitivity_cpu.py shows that the oracle moves by at least 10x one of those bars at each continuous case, so a kernel that
ignored a parameter or read its neighbour would fail here.  test_fast_kernels_launched proves, with torch.profiler, that these
cases run the default kernels, not the fallbacks test_gpu_ragged covers.  Run with -s to print the largest RMSE / max-abs error of
every stage per case.
"""
import ctypes as C
import re

import numpy as np
import pytest

import oracle as O
import param_cases as PC
import pyhr
from test_gpu_config_sizes import check_all_large
from test_gpu_gi_refl import close, f16
from test_gpu_parity import check_all
from test_gpu_ragged import CAM_ARCADE, CAM_SHADOWS_TEST, SKY, Worst, _launched, _one_frame, check_ddgi, run_gi_refl, run_shadows_ao, set_params

pytestmark = pytest.mark.gpu

W, H = PC.SIZE
HR_ERR_INVALID_ARG, HR_ERR_NOT_READY, HR_ERR_UNSUPPORTED = -1, -4, -5


# Cases held to test_gpu_config_sizes.bounded (check_all_large) instead of check_all, with the reason.  Shadows phi_visibility 40,
# frame 3 (the first panning frame): one a-trous texel of the 73 728 is 4.9e-3 off (bar 4e-3), RMSE 2.9e-5.  Fed the device's own
# temporal output, the oracle's a-trous chain matches every kernel form (k_atrous_v3, k_atrous_tiled, k_atrous_naive with expf) to
# one fp16 ulp; the texel comes from the temporal inputs, which differ by up to 2.4e-4 (inside their own bar) at freshly
# disoccluded, near-zero-variance pixels, where the luminance weight exp(-|dl| / (phi * sqrt(var))) amplifies an ulp: bounded's rule.
BOUNDED = {"shadows phi_visibility 40.0"}


def by_kind(*kinds):
    return [c for c in PC.CONTINUOUS if c.kind in kinds]


# ---------------------------------------------------------------------------------------------- continuous parameters
@pytest.mark.parametrize("case", by_kind("shadows", "ao"), ids=PC.ids(by_kind("shadows", "ao")))
def test_shadows_ao_parameter(case):
    """shadows at scale 0 and AO at scale 1, like test_shadows_parameters: 3 static + 3 panning frames"""
    kw = dict(sh_params=case.params) if case.kind == "shadows" else dict(ao_params=case.params)
    run_shadows_ao(case.id, W, H, 0, 1, n=case.frames, check=check_all_large if case.id in BOUNDED else check_all, **kw, **PC.scene_kw(case.scene))


@pytest.mark.parametrize("case", by_kind("reflections"), ids=PC.ids(by_kind("reflections")))
def test_reflections_parameter(case):
    run_gi_refl(case.id, W, H, 0, case.ddgi, params=case.params, n=case.frames, lut=pyhr.brdf_lut(64) if case.lut else None, **PC.scene_kw(case.scene))


@pytest.mark.parametrize("case", by_kind("ddgi"), ids=PC.ids(by_kind("ddgi")))
def test_ddgi_parameter(case):
    """default layout, 5 frames: hysteresis and the infinite bounce act from the second frame on; the reflections read the atlas"""
    run_gi_refl(case.id, W, H, 0, True, ddgi_params=case.params, n=case.frames, **PC.scene_kw(case.scene))


# ---------------------------------------------------------------------------------------------- probe layouts
@pytest.mark.parametrize("case", PC.LAYOUTS, ids=PC.ids(PC.LAYOUTS))
def test_ddgi_layout(case):
    """whole atlases (gutters and outer border included), the sample and the reflections chain, whose rough lobe samples the atlas
    (approximate_with_ddgi = 1, the default)"""
    kw = PC.scene_kw(case.scene)
    if case.scene == "arcade_lifted":  # see param_cases.LAYOUTS
        kw["scene"] = arcade_lifted_grid()
    run_gi_refl(case.id, W, H, 0, True, ddgi_params=case.params, n=case.frames, **kw)


# ---------------------------------------------------------------------------------------------- grid lifecycle
def _render_rc(dd, f, rot, params):
    return dd.lib.hr_ddgi_render(dd.h, C.byref(f), C.byref(params), np.ascontiguousarray(rot, np.float32).ctypes.data, None)


def _uniforms_rc(dd):
    u = pyhr.hr_ddgi_uniforms()
    return dd.lib.hr_ddgi_get_uniforms(dd.h, C.byref(u)), u


def test_ddgi_layout_switch_mid_sequence():
    """the layout changes at frame 3: the grid re-initialises with first-frame semantics (zero atlases, no hysteresis, no infinite
    bounce), compared with a new oracle from that frame on; the reflections history goes on"""
    def hook(i, f, rot, dd, odd, fresh):
        if i != 3:
            return odd
        set_params([dd.params], dict(rays_per_probe=33, irradiance_oct_size=6, depth_oct_size=14, probe_distance=8.0))
        return fresh()
    run_gi_refl("ddgi layout switch at frame 3", W, H, 0, True, n=6, ddgi_hook=hook, **PC.scene_kw("arcade"))


def test_ddgi_continuous_switch_mid_sequence():
    """hysteresis and depth_sharpness change at frame 2 and again at frame 4: applied every frame, the grid is kept"""
    def hook(i, f, rot, dd, odd, fresh):
        if i == 2:
            set_params([dd.params], dict(hysteresis=0.5, depth_sharpness=5.0))
        if i == 4:
            set_params([dd.params], dict(hysteresis=0.9))
        return odd  # shares dd.params: it refreshes its uniforms every frame, like the device
    run_gi_refl("ddgi hysteresis switch at frames 2 and 4", W, H, 0, True, n=6, ddgi_hook=hook, **PC.scene_kw("arcade"))


REJECTED = [("rays_per_probe", 0), ("rays_per_probe", 1025), ("irradiance_oct_size", 1), ("irradiance_oct_size", 17), ("depth_oct_size", 1),
            ("depth_oct_size", 33), ("probe_distance", 0.0), ("probe_distance", -1.0), ("probe_distance", float("nan"))]


def test_ddgi_rejected_values():
    """out-of-range values are refused with HR_ERR_INVALID_ARG before anything changes: the grid and its uniforms stay, and the
    next frame with valid parameters matches the oracle that never saw the refused calls"""
    def hook(i, f, rot, dd, odd, fresh):
        if i != 2:
            return odd
        before = bytes(_uniforms_rc(dd)[1])
        for k, v in REJECTED:
            bad = pyhr.hr_ddgi_params.from_buffer_copy(dd.params)
            setattr(bad, k, v)
            assert _render_rc(dd, f, rot, bad) == HR_ERR_INVALID_ARG, f"{k} = {v} accepted"
            rc, u = _uniforms_rc(dd)
            assert rc == 0 and bytes(u) == before, f"{k} = {v}: the grid changed"
        return odd
    run_gi_refl("ddgi rejected values at frame 2", W, H, 0, True, n=4, ddgi_hook=hook, **PC.scene_kw("arcade"))


def test_ddgi_too_many_probes_leaves_no_grid():
    """a probe_distance that gives more than 2^20 probes returns HR_ERR_UNSUPPORTED after the old grid was freed: the pass must
    hold no grid then (hr_ddgi_get_uniforms: HR_ERR_NOT_READY, a host-only check made before anything runs on the device again),
    and the next render with the previous, valid parameters initialises a new grid with first-frame semantics"""
    def hook(i, f, rot, dd, odd, fresh):
        if i != 2:
            return odd
        for pd in (0.1, 1e-30):  # 602 x 287 x 1282 probes; a ratio above INT_MAX, which does not convert to int
            bad = pyhr.hr_ddgi_params.from_buffer_copy(dd.params)
            bad.probe_distance = pd
            assert _render_rc(dd, f, rot, bad) == HR_ERR_UNSUPPORTED, f"probe_distance {pd}"
            assert _uniforms_rc(dd)[0] == HR_ERR_NOT_READY, f"probe_distance {pd}: the pass still reports the freed grid"
        return fresh()
    run_gi_refl("ddgi too many probes at frame 2", W, H, 0, True, n=4, ddgi_hook=hook, **PC.scene_kw("arcade"))


def test_ddgi_scene_replacement():
    """destroy the scene and build one with other bounds: the pass re-initialises its grid whether or not the new scene got the
    old one's address, and every DDGI output equals a fresh oracle's.  Then the reflections read that grid."""
    bn = pyhr.blue_noise()
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*bn)
    ctx.gbuffer_create(W, H)
    zero = pyhr.GBufferHost(W, H)
    ctx.gbuffer_upload(0, zero)
    ctx.gbuffer_upload(1, zero)
    dd, rf = pyhr.DDGIPass(ctx, W, H, 0), pyhr.ReflectionsPass(ctx, W, H, 0)
    for P in (dd.params, rf.params):
        P.sky_color[0], P.sky_color[1], P.sky_color[2] = SKY
    dd.params.probe_distance, dd.params.normal_bias = 12.0, 1.0
    w = Worst("ddgi scene replacement")
    f, handle, reused = None, None, None
    prev_g = O.zero_gbuf_mips(W, H)  # the device's other G-buffer slot: the previous frame, whichever scene it showed
    for n_scene, (kind, tris, cam, light) in enumerate(((pyhr.SCENE_SHADOWS_TEST, 0, CAM_SHADOWS_TEST, None),
                                                       (pyhr.SCENE_ARCADE, 20000, CAM_ARCADE, pyhr.default_light(rot_x_deg=25.0)))):
        sc = pyhr.SynthScene(kind, tris)
        ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
        if handle is not None:
            old = handle.value
            assert ctx.lib.hr_scene_destroy(handle) == 0
            handle = ctx.build_scene(sc)
            reused = handle.value == old
        else:
            handle = ctx.build_scene(sc)
        odd = O.DDGIOracle(W, H, 0, dd.params, *sc.bounds())
        orf = O.ReflectionsOracle(W, H, 0, rf.params)
        for k in range(3):
            i = 3 * n_scene + k
            f = pyhr.make_frame(*cam, W, H, prev=f, num_frames=i, light=light)
            ctx.gbuffer_render(f.ping_pong, f)
            cur_g = O.GBufMips(O.gbuffer_render(ss, f, W, H))
            rot = pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))
            dd.render(f, rot)
            odd.render(ss, cur_g, f, rot)
            check_ddgi(i, dd, odd, w)
            if n_scene == 1:
                rf.render(f, dd)
                orf.render(ss, cur_g, prev_g, f, bn, odd)
                close(f16(rf.download(0))[..., :3], O.h2f(orf.rt)[..., :3], f"frame {i} reflections ray trace", 1e-3, 0.02)
                close(f16(rf.download(100)), O.h2f(orf.final), f"frame {i} reflections final")
            prev_g = cur_g
    w.report()
    print(f"the new scene {'reused' if reused else 'did not reuse'} the destroyed scene's address")
    rf.destroy()
    dd.destroy()
    ctx.lib.hr_scene_destroy(handle)
    ctx.close()


# ---------------------------------------------------------------------------------------------- a wide atlas
class BoxScene(pyhr.ArrayScene):
    """an axis-aligned box as explicit arrays, with the SynthScene interface oracle.ShadingScene reads"""

    def __init__(self, lo, hi, albedo=(0.8, 0.7, 0.6), roughness=0.5):
        lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
        V, I = [], []
        for axis in range(3):
            for side in (0, 1):
                n = np.zeros(3, np.float32)
                n[axis] = 1.0 if side else -1.0
                u, v = (axis + 1) % 3, (axis + 2) % 3
                base = len(V)
                for a, b in ((0, 0), (1, 0), (1, 1), (0, 1)):
                    p = np.where(np.arange(3) == axis, (hi if side else lo), 0.0).astype(np.float32)
                    p[u], p[v] = (hi[u] if a else lo[u]), (hi[v] if b else lo[v])
                    t = np.zeros(3, np.float32)
                    t[u] = 1.0
                    bt = np.cross(n, t).astype(np.float32)
                    V.append(np.concatenate([p, [1], [a, b, 0, 0], n, [0], t, [0], bt, [0]]))
                quad = [0, 1, 2, 0, 2, 3] if side else [0, 2, 1, 0, 3, 2]  # counter-clockwise seen from outside
                I += [base + q for q in quad]
        ident = (C.c_float * 16)(*np.eye(4, dtype=np.float32).reshape(16))
        mat = pyhr.hr_material((C.c_float * 4)(*albedo, 1.0), (C.c_float * 4)(), roughness, 0.0)
        super().__init__(np.array(V, np.float32), np.array(I, np.uint32), [pyhr.hr_instance(ident, 0, len(I), 0, 0)], [mat])
        self.n_materials = 1
        tri = self.V[self.I, :3].reshape(-1, 9)
        self._tri, self._nrm = np.ascontiguousarray(tri, np.float32), np.ascontiguousarray(self.V[self.I, 8:11].reshape(-1, 9), np.float32)
        self._lo, self._hi = tri.reshape(-1, 3).min(0), tri.reshape(-1, 3).max(0)

    def world_triangles(self):
        return self._tri, np.zeros(self.n_tris, np.uint32)

    def world_normals(self):
        return self._nrm, np.zeros(self.n_tris, np.uint32)

    def materials_array(self):
        return self.mats

    def bounds(self):
        return self._lo.astype(np.float32), self._hi.astype(np.float32)


class SoupScene(pyhr.ArrayScene):
    """a world-space triangle soup (tri (n, 9), vertex normals (n, 9), material per triangle) as explicit arrays, one instance per
    material with the identity transform, with the SynthScene interface oracle.ShadingScene reads"""

    def __init__(self, tri, nrm, mat, materials):
        order = np.argsort(mat, kind="stable")
        tri, nrm, mat = np.asarray(tri, np.float32)[order], np.asarray(nrm, np.float32)[order], np.asarray(mat)[order]
        n = len(tri)
        V = np.zeros((3 * n, 20), np.float32)
        V[:, 0:3], V[:, 3] = tri.reshape(-1, 3), 1.0
        V[:, 8:11], V[:, 12], V[:, 17] = nrm.reshape(-1, 3), 1.0, 1.0
        ident = (C.c_float * 16)(*np.eye(4, dtype=np.float32).reshape(16))
        inst, self._inst = [], np.zeros(n, np.uint32)
        for m in np.unique(mat):
            lo, hi = np.searchsorted(mat, m), np.searchsorted(mat, m, side="right")
            self._inst[lo:hi] = len(inst)
            inst.append(pyhr.hr_instance(ident, 3 * lo, 3 * (hi - lo), 0, int(m)))
        super().__init__(V, np.arange(3 * n, dtype=np.uint32), inst, list(materials))
        self._tri, self._mat = np.ascontiguousarray(tri), np.ascontiguousarray(mat, np.uint32)
        w = nrm.reshape(-1, 3)  # normalize(mat3(model) * normal) with the identity, in hr_scene_build's arithmetic
        ln = np.sqrt((w[:, 0] * w[:, 0] + w[:, 1] * w[:, 1]) + w[:, 2] * w[:, 2]).astype(np.float32)
        il = np.where(ln > 0, np.float32(1.0) / np.where(ln > 0, ln, 1).astype(np.float32), np.float32(0.0)).astype(np.float32)
        self._nrm = np.ascontiguousarray((w * il[:, None]).astype(np.float32).reshape(-1, 9))
        pts = tri.reshape(-1, 3)
        self._lo, self._hi = pts.min(0), pts.max(0)

    def world_triangles(self):
        return self._tri, self._inst

    def world_normals(self):
        return self._nrm, self._mat

    def materials_array(self):
        return self.mats

    def bounds(self):
        return self._lo.astype(np.float32), self._hi.astype(np.float32)


def arcade_lifted_grid():
    """the arcade scene plus one triangle 0.7 below, left of and behind its floor's corner, out of view: the probe grid starts there,
    so neither the floor nor the walls at the scene's bounds lie on a probe plane"""
    sc = pyhr.SynthScene(pyhr.SCENE_ARCADE, 20000)
    tri, _ = sc.world_triangles()
    nrm, mat = sc.world_normals()
    extra = np.array([[-30.7, -0.7, -8.7, -29.7, -0.7, -7.7, -29.7, -0.7, -8.7]], np.float32)
    up = np.array([[0.0, 1.0, 0.0] * 3], np.float32)
    return SoupScene(np.concatenate([tri, extra]), np.concatenate([nrm, up]), np.concatenate([mat, [0]]), sc.materials_array())


def test_ddgi_wide_atlas():
    """a 400 x 40 x 1 slab with probe_distance 1: 402 x 42 x 3 probes in one atlas row, a depth atlas 303 914 texels wide, where
    K21 / K12's texel addressing (an approximate reciprocal of the width) is furthest from the oracle's exact division.  The camera
    looks at the end of the slab that the last atlas columns hold."""
    box = BoxScene((-200.0, -20.0, -0.5), (200.0, 20.0, 0.5))
    u = O.ddgi_uniforms_from(pyhr.hr_ddgi_params(probe_distance=1.0, irradiance_oct_size=8, depth_oct_size=16, rays_per_probe=16), *box.bounds())
    assert list(u.probe_counts) == [402, 42, 3] and u.depth_texture_width == 303914
    run_gi_refl("ddgi wide atlas", W, H, 0, True, n=3, scene=box, cam=((185.0, 16.0, 14.0), (185.0, 16.0, 0.0)),
                ddgi_params=dict(probe_distance=1.0, rays_per_probe=16))


# ---------------------------------------------------------------------------------------------- which kernel ran
PROFILED = by_kind("shadows", "ao", "reflections")


FALLBACKS = {"shadows": ("k_atrous_tiled", "k_atrous_naive"), "ao": ("k_ao_blur",), "reflections": ("k_refl_atrous",)}


@pytest.mark.parametrize("case", PROFILED, ids=PC.ids(PROFILED))
def test_fast_kernels_launched(case):
    """the parameter cases keep phi_normal 32, radius 1 and even widths: the default kernels run and none of the fallbacks
    test_gpu_ragged covers (separate from the parity tests, so a profiler problem cannot hide a parity result)"""
    for _ in range(2):  # a profiled cycle that holds no kernel record at all is a profiler failure, not a kernel choice: profile again
        names = _one_frame(case.kind, W, H, 1 if case.kind == "ao" else 0, case.params)
        kernels = sorted(n for n in names if re.search(r"\bk_\w+[<(]", n))
        if kernels:
            break
    for k in case.kernels:
        assert _launched(names, k), f"{case.id}: {k} not launched; kernels: {kernels}"
    for k in FALLBACKS[case.kind]:
        assert not _launched(names, k), f"{case.id}: {k} launched; kernels: {kernels}"
    print(f"\n[{case.id}] launched {', '.join(case.kernels)}")
