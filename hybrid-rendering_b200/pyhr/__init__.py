"""pyhr — thin ctypes binding over the C ABI (include/hr_api.h) and the synthetic-input library (host/synth.h).

Used by tests/ and bench.py only; the product is the C ABI + CUDA kernels.  PyTorch appears solely as a provider of
device memory / streams where a caller wants to hand device pointers to the ABI.  There is no CPU fallback: loading
or initialising fails loudly when the CUDA library or a GPU is missing.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
PKG_ROOT = os.path.dirname(_HERE)
BUILD_DIR = os.path.join(PKG_ROOT, "build")
LIB_PRODUCT = os.path.join(BUILD_DIR, "libhr_b200.so")
LIB_SYNTH = os.path.join(BUILD_DIR, "libhr_synth.so")

c_float_p = C.POINTER(C.c_float)
c_u8_p = C.POINTER(C.c_uint8)
c_u16_p = C.POINTER(C.c_uint16)
c_u32_p = C.POINTER(C.c_uint32)


# ---------------------------------------------------------------------------------------------- ABI structs
class hr_light(C.Structure):
    _fields_ = [("data0", C.c_float * 4), ("data1", C.c_float * 4), ("data2", C.c_float * 4), ("data3", C.c_float * 4)]


class hr_ubo(C.Structure):
    _fields_ = [("view_inverse", C.c_float * 16), ("proj_inverse", C.c_float * 16), ("view_proj_inverse", C.c_float * 16),
                ("prev_view_proj", C.c_float * 16), ("view_proj", C.c_float * 16), ("cam_pos", C.c_float * 4),
                ("current_prev_jitter", C.c_float * 4), ("light", hr_light)]


class hr_frame(C.Structure):
    _fields_ = [("ubo", hr_ubo), ("num_frames", C.c_uint32), ("ping_pong", C.c_int32), ("first_frame", C.c_int32),
                ("z_buffer_params", C.c_float * 4), ("camera_delta", C.c_float * 3), ("frame_time", C.c_float)]


class hr_vertex(C.Structure):
    _fields_ = [("position", C.c_float * 4), ("tex_coord", C.c_float * 4), ("normal", C.c_float * 4), ("tangent", C.c_float * 4),
                ("bitangent", C.c_float * 4)]


class hr_material(C.Structure):
    _fields_ = [("albedo", C.c_float * 4), ("emissive", C.c_float * 4), ("roughness", C.c_float), ("metallic", C.c_float), ("_pad", C.c_float * 2)]


class hr_instance(C.Structure):
    _fields_ = [("model", C.c_float * 16), ("first_index", C.c_uint32), ("index_count", C.c_uint32), ("base_vertex", C.c_uint32),
                ("material_idx", C.c_uint32)]


class hr_texture(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32), ("srgb", C.c_int32), ("data", C.c_void_p)]


class hr_material_textures(C.Structure):
    _fields_ = [("albedo", C.c_int32), ("normal", C.c_int32), ("roughness", C.c_int32), ("roughness_channel", C.c_int32), ("metallic", C.c_int32),
                ("metallic_channel", C.c_int32), ("emissive", C.c_int32)]


class hr_scene_info(C.Structure):
    _fields_ = [("n_triangles", C.c_uint64), ("n_nodes", C.c_uint64), ("bounds_min", C.c_float * 3), ("bounds_max", C.c_float * 3),
                ("build_ms", C.c_float), ("depth", C.c_uint32)]


class hr_gbuffer_desc(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("gb1", C.c_void_p), ("gb2", C.c_void_p), ("gb3", C.c_void_p), ("depth", C.c_void_p)]


class hr_image(C.Structure):
    _fields_ = [("data", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("format", C.c_int32)]


class hr_shadows_params(C.Structure):
    _fields_ = [("bias", C.c_float), ("alpha", C.c_float), ("moments_alpha", C.c_float), ("phi_visibility", C.c_float), ("phi_normal", C.c_float),
                ("sigma_depth", C.c_float), ("power", C.c_float), ("radius", C.c_int32), ("filter_iterations", C.c_int32),
                ("feedback_iteration", C.c_int32), ("denoise", C.c_int32), ("spp", C.c_int32)]


class hr_ao_params(C.Structure):
    _fields_ = [("ray_length", C.c_float), ("bias", C.c_float), ("alpha", C.c_float), ("power", C.c_float), ("blur_radius", C.c_int32),
                ("denoise", C.c_int32), ("spp", C.c_int32)]


class hr_pass_stats(C.Structure):
    _fields_ = [("rays_primary", C.c_uint64), ("rays_secondary", C.c_uint64), ("tiles_total", C.c_uint64), ("tiles_denoise", C.c_uint64),
                ("pixels_total", C.c_uint64), ("renders", C.c_uint64)]


class hrs_light_desc(C.Structure):
    _fields_ = [("type", C.c_int32), ("rot_y_deg", C.c_float), ("rot_x_deg", C.c_float), ("position", C.c_float * 3), ("radius", C.c_float),
                ("intensity", C.c_float), ("color", C.c_float * 3), ("cone_inner_deg", C.c_float), ("cone_outer_deg", C.c_float)]


HR_FMT = {1: ("<u4", 1), 2: ("<f2", 1), 3: ("<f2", 2), 4: ("<f2", 4), 5: ("u1", 1), 6: ("u1", 4)}  # hr_format -> (dtype, channels)

# every symbol include/hr_api.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "hr_init", "hr_shutdown", "hr_last_error", "hr_version", "hr_bluenoise_set", "hr_scene_build", "hr_scene_destroy", "hr_scene_set_current",
    "hr_scene_get_info", "hr_scene_rebuild", "hr_trace_any", "hr_trace_closest", "hr_gbuffer_create", "hr_gbuffer_upload",
    "hr_gbuffer_stage_upload", "hr_gbuffer_commit_staged", "hr_pass_download_async", "hr_pass_download_rows_async",
    "hr_gbuffer_copy_from_device", "hr_gbuffer_bind_device", "hr_gbuffer_download", "hr_shadows_default_params", "hr_shadows_create",
    "hr_shadows_render", "hr_ao_default_params", "hr_ao_create", "hr_ao_render", "hr_pass_output", "hr_pass_download", "hr_pass_reset_history",
    "hr_pass_destroy", "hr_pass_upload", "hr_ctx_set_profiling", "hr_pass_stage_times", "hr_debug_set", "hr_ctx_launch_count", "hr_shard_config", "hr_shard_rows", "hr_shard_unique_id", "hr_shard_init", "hr_shard_shutdown", "hr_shard_set_gather", "hr_shard_halo_rows", "hr_shard_link_local",
    "hr_ddgi_default_params", "hr_ddgi_create", "hr_ddgi_render", "hr_ddgi_get_uniforms", "hr_reflections_default_params", "hr_reflections_create",
    "hr_reflections_render", "hr_pass_get_stats", "hr_pass_output_checksum", "hr_gbuffer_render", "hr_gbuffer_render_sharded", "hr_brdf_lut_set", "hr_deferred_create", "hr_deferred_render", "hr_gbuffer_stage_render", "hr_bluenoise_set_slot",
    "hr_taa_default_params", "hr_taa_jitter", "hr_taa_create", "hr_taa_render", "hr_tonemap_default_params", "hr_tonemap_create", "hr_tonemap_render", "hr_path_tracer_default_params", "hr_path_tracer_create", "hr_path_tracer_render", "hr_scene_set_textures",
]

_product = None
_synth = None


def load_product():
    """dlopen the CUDA library.  Raises (never falls back) if it has not been built."""
    global _product
    if _product is None:
        if not os.path.exists(LIB_PRODUCT):
            raise RuntimeError(f"{LIB_PRODUCT} not found: build it with `make -C {PKG_ROOT}` (no CPU fallback exists)")
        lib = C.CDLL(LIB_PRODUCT)
        lib.hr_last_error.restype = C.c_char_p
        lib.hr_last_error.argtypes = [C.c_void_p]
        lib.hr_ctx_launch_count.restype = C.c_uint64
        lib.hr_ctx_launch_count.argtypes = [C.c_void_p]
        _product = lib
    return _product


def load_synth():
    global _synth
    if _synth is None:
        if not os.path.exists(LIB_SYNTH):
            raise RuntimeError(f"{LIB_SYNTH} not found: build it with `make -C {PKG_ROOT}`")
        lib = C.CDLL(LIB_SYNTH)
        lib.hrs_scene_create.restype = C.c_void_p
        lib.hrs_scene_create.argtypes = [C.c_int, C.c_int, C.c_uint32]
        lib.hrs_scene_destroy.argtypes = [C.c_void_p]
        lib.hrs_scene_counts.argtypes = [C.c_void_p] + [C.POINTER(C.c_uint64)] * 4
        for n in ("hrs_scene_vertices", "hrs_scene_indices", "hrs_scene_instances", "hrs_scene_materials"):
            getattr(lib, n).restype = C.c_void_p
            getattr(lib, n).argtypes = [C.c_void_p]
        lib.hrs_scene_bounds.argtypes = [C.c_void_p, c_float_p, c_float_p]
        lib.hrs_scene_world_triangles.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.hrs_scene_world_normals.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.hrs_default_light.argtypes = [C.POINTER(hrs_light_desc)]
        lib.hrs_make_frame.argtypes = [C.POINTER(hr_frame), c_float_p, c_float_p, C.c_int, C.c_int, C.POINTER(hrs_light_desc), C.POINTER(hr_frame), C.c_uint32]
        lib.hrs_make_frame_ex.argtypes = [C.POINTER(hr_frame), c_float_p, c_float_p, c_float_p, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int,
                                          C.POINTER(hrs_light_desc), C.POINTER(hr_frame), C.c_uint32]
        lib.hrs_write_gbuffer.argtypes = [C.c_void_p, C.POINTER(hr_frame), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.hrs_blue_noise.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p]
        _synth = lib
    return _synth


class HrError(RuntimeError):
    pass


def shard_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    rc = load_product().hr_shard_unique_id(buf)
    if rc != 0:
        raise HrError(f"hr_shard_unique_id failed ({rc}): {load_product().hr_last_error(None).decode()}")
    return buf.raw


def shard_halo_rows(kind, radius=1, filter_iterations=4, blur_radius=5):
    """(denoise_halo, ray_trace_halo) of a sharded rank for the given pass parameters (hr_shard_halo_rows; pure, no GPU)"""
    k = {"shadows": 1, "ao": 2, "reflections": 3}[kind]
    a, b = C.c_int(), C.c_int()
    rc = load_product().hr_shard_halo_rows(k, int(radius), int(filter_iterations), int(blur_radius), C.byref(a), C.byref(b))
    if rc != 0:
        raise ValueError(f"hr_shard_halo_rows: {rc}")
    return a.value, b.value


def shard_rows(H, rank, world):
    b, e = C.c_int(), C.c_int()
    load_product().hr_shard_rows(H, rank, world, C.byref(b), C.byref(e))
    return b.value, e.value


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# ---------------------------------------------------------------------------------------------- synthetic inputs
SCENE_SINGLE_TRIANGLE, SCENE_GROUND_PLANE, SCENE_SHADOWS_TEST, SCENE_ARCADE = 0, 1, 2, 3


class SynthScene:
    def __init__(self, kind, target_tris=0, seed=7):
        self.lib = load_synth()
        self.h = self.lib.hrs_scene_create(kind, target_tris, seed)
        if not self.h:
            raise HrError("hrs_scene_create failed")
        c = [C.c_uint64() for _ in range(4)]
        self.lib.hrs_scene_counts(self.h, *[C.byref(x) for x in c])
        self.n_vertices, self.n_indices, self.n_instances, self.n_materials = [int(x.value) for x in c]
        self.n_tris = self.n_indices // 3

    def __del__(self):
        try:
            if self.h:
                self.lib.hrs_scene_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def raw(self):
        """(vertices_ptr, indices_ptr, instances_ptr, materials_ptr) host pointers valid while self lives."""
        L = self.lib
        return (L.hrs_scene_vertices(self.h), L.hrs_scene_indices(self.h), L.hrs_scene_instances(self.h), L.hrs_scene_materials(self.h))

    def world_triangles(self):
        tri = np.empty((self.n_tris, 9), np.float32)
        inst = np.empty(self.n_tris, np.uint32)
        self.lib.hrs_scene_world_triangles(self.h, _ptr(tri), _ptr(inst))
        return tri, inst

    def world_normals(self):
        nrm = np.empty((self.n_tris, 9), np.float32)
        mat = np.empty(self.n_tris, np.uint32)
        self.lib.hrs_scene_world_normals(self.h, _ptr(nrm), _ptr(mat))
        return nrm, mat

    def materials_array(self):
        n = self.n_materials
        buf = (hr_material * n).from_address(self.lib.hrs_scene_materials(self.h))
        return buf

    def bounds(self):
        mn = (C.c_float * 3)()
        mx = (C.c_float * 3)()
        self.lib.hrs_scene_bounds(self.h, mn, mx)
        return np.array(mn[:], np.float32), np.array(mx[:], np.float32)


class ArrayScene:
    """hr_scene_build arguments held as arrays (vertices (n, 20) float32 = dw::Vertex, uint32 indices, [hr_instance], [hr_material]): has the
    attributes Context.build_scene reads.  Tests use it to change a procedural scene's texture coordinates."""

    def __init__(self, vertices, indices, instances, materials):
        self.V = np.ascontiguousarray(vertices, np.float32)
        self.I = np.ascontiguousarray(indices, np.uint32)
        self.inst = (hr_instance * len(instances))(*instances)
        self.mats = (hr_material * len(materials))(*materials)
        self.n_vertices, self.n_indices, self.n_instances, self.n_materials = len(self.V), len(self.I), len(instances), len(materials)
        self.n_tris = self.n_indices // 3

    def raw(self):
        return (self.V.ctypes.data, self.I.ctypes.data, C.addressof(self.inst), C.addressof(self.mats))

    def primitive_tangent_frames(self):
        """(n_tris, 18): world-space unit tangents of the three corners, then their bitangents, as hr_scene_build keeps them (normalize(mat3(model) * t))"""
        out = []
        for it in self.inst:
            M = np.array(it.model[:], np.float32).reshape(4, 4).T
            idx = self.I[it.first_index: it.first_index + it.index_count // 3 * 3].astype(np.int64) + it.base_vertex
            rows = []
            for col in (12, 16):  # tangent, bitangent of dw::Vertex
                a = self.V[idx, col:col + 3]
                w = np.empty_like(a)
                for r in range(3):
                    w[:, r] = (M[r, 0] * a[:, 0] + M[r, 1] * a[:, 1]) + M[r, 2] * a[:, 2]
                ln = np.sqrt((w[:, 0] * w[:, 0] + w[:, 1] * w[:, 1]) + w[:, 2] * w[:, 2]).astype(np.float32)
                il = np.where(ln > 0, np.float32(1.0) / np.where(ln > 0, ln, 1).astype(np.float32), np.float32(0.0)).astype(np.float32)
                rows.append((w * il[:, None]).astype(np.float32).reshape(-1, 9))
            out.append(np.concatenate(rows, 1))
        return np.ascontiguousarray(np.concatenate(out), np.float32)

    def primitive_uvs(self):
        """(n_tris, 6): texture coordinates of the three corners in hr_scene_build's primitive order (instances in order, triangles in index order)"""
        out = []
        for it in self.inst:
            idx = self.I[it.first_index: it.first_index + it.index_count // 3 * 3].astype(np.int64) + it.base_vertex
            out.append(self.V[idx, 4:6].reshape(-1, 6))
        return np.ascontiguousarray(np.concatenate(out), np.float32)


def default_light(**kw):
    l = hrs_light_desc()
    load_synth().hrs_default_light(C.byref(l))
    for k, v in kw.items():
        if isinstance(v, (tuple, list)):
            for i, x in enumerate(v):
                getattr(l, k)[i] = x
        else:
            setattr(l, k, v)
    return l


def make_frame(cam_pos, cam_target, W, H, prev=None, num_frames=0, light=None, up=(0.0, 1.0, 0.0), fovy_deg=60.0, near=1.0, far=1000.0):
    """hrs_make_frame_ex: look_at(cam_pos, cam_target, up), perspective(fovy_deg, W / H, near, far); the defaults are hrs_make_frame's camera"""
    f = hr_frame()
    p = (C.c_float * 3)(*cam_pos)
    t = (C.c_float * 3)(*cam_target)
    u = (C.c_float * 3)(*up)
    load_synth().hrs_make_frame_ex(C.byref(f), p, t, u, fovy_deg, near, far, W, H, C.byref(light) if light is not None else None,
                                   C.byref(prev) if prev is not None else None, num_frames)
    return f


class GBufferHost:
    """mip-0 G-buffer in host memory in the reference's formats."""

    def __init__(self, W, H, pinned=False):
        self.W, self.H = W, H
        if pinned:
            import torch
            self._t = [torch.empty((H, W, 4), dtype=torch.uint8).pin_memory(), torch.empty((H, W, 4), dtype=torch.int16).pin_memory(),
                       torch.empty((H, W, 4), dtype=torch.int16).pin_memory(), torch.empty((H, W), dtype=torch.float32).pin_memory()]
            self.gb1 = self._t[0].numpy()
            self.gb2 = self._t[1].numpy().view(np.uint16)
            self.gb3 = self._t[2].numpy().view(np.uint16)
            self.depth = self._t[3].numpy()
        else:
            self.gb1 = np.zeros((H, W, 4), np.uint8)
            self.gb2 = np.zeros((H, W, 4), np.uint16)
            self.gb3 = np.zeros((H, W, 4), np.uint16)
            self.depth = np.zeros((H, W), np.float32)

    def desc(self):
        return hr_gbuffer_desc(self.W, self.H, _ptr(self.gb1), _ptr(self.gb2), _ptr(self.gb3), _ptr(self.depth))

    def nbytes(self):
        return self.gb1.nbytes + self.gb2.nbytes + self.gb3.nbytes + self.depth.nbytes


def write_gbuffer(scene: SynthScene, frame: hr_frame, W, H, out: GBufferHost = None, pinned=False):
    g = out if out is not None else GBufferHost(W, H, pinned)
    load_synth().hrs_write_gbuffer(scene.h, C.byref(frame), W, H, _ptr(g.gb1), _ptr(g.gb2), _ptr(g.gb3), _ptr(g.depth))
    return g


def blue_noise(seed=1234):
    sobol = np.empty((256, 4), np.uint8)
    sr = np.empty((128, 128, 4), np.uint8)
    load_synth().hrs_blue_noise(seed, _ptr(sobol), _ptr(sr))
    return sobol, sr


# ---------------------------------------------------------------------------------------------- product wrappers
class Context:
    def __init__(self, device=0):
        self.lib = load_product()
        h = C.c_void_p()
        rc = self.lib.hr_init(device, C.byref(h))
        if rc != 0:
            raise HrError(f"hr_init failed ({rc}): {self.lib.hr_last_error(None).decode()}")
        self.h = h
        self._keep = []

    def check(self, rc, what=""):
        if rc != 0:
            raise HrError(f"{what} failed ({rc}): {self.lib.hr_last_error(self.h).decode()}")

    def close(self):
        if self.h:
            self.lib.hr_shutdown(self.h)
            self.h = None

    def set_bluenoise_slot(self, slot, sr):
        """scrambling / ranking table of sample-count slot `slot` (log2 spp), src/blue_noise.cpp:9-19"""
        self.check(self.lib.hr_bluenoise_set_slot(self.h, slot, _ptr(np.ascontiguousarray(sr))), "hr_bluenoise_set_slot")

    def set_brdf_lut(self, lut):
        lut = np.ascontiguousarray(lut, np.uint16)
        assert lut.shape == (512, 512, 2)
        self.check(self.lib.hr_brdf_lut_set(self.h, _ptr(lut)), "hr_brdf_lut_set")

    def set_bluenoise(self, sobol, sr):
        self.check(self.lib.hr_bluenoise_set(self.h, _ptr(np.ascontiguousarray(sobol)), _ptr(np.ascontiguousarray(sr))), "hr_bluenoise_set")

    def build_scene(self, s: SynthScene):
        v, i, inst, m = s.raw()
        out = C.c_void_p()
        self.check(self.lib.hr_scene_build(self.h, C.c_void_p(v), C.c_size_t(s.n_vertices), C.c_void_p(i), C.c_size_t(s.n_indices), C.c_void_p(inst),
                                           C.c_size_t(s.n_instances), C.c_void_p(m), C.c_size_t(s.n_materials), C.byref(out)), "hr_scene_build")
        self.check(self.lib.hr_scene_set_current(self.h, out), "hr_scene_set_current")
        return out

    def set_textures(self, scene, textures, bindings):
        """hr_scene_set_textures: textures = [(uint8 array (H, W) / (H, W, C), srgb)], bindings = one dict per material with the keys of
        hr_material_textures (missing keys: -1 / channel 0).  textures = [] removes them."""
        keep = [np.ascontiguousarray(a, np.uint8) for a, _ in textures]
        tx = (hr_texture * max(1, len(textures)))()
        for i, (a, (_, srgb)) in enumerate(zip(keep, textures)):
            tx[i] = hr_texture(a.shape[1], a.shape[0], 1 if a.ndim == 2 else a.shape[2], int(bool(srgb)), a.ctypes.data)
        bd = (hr_material_textures * max(1, len(bindings)))()
        for i, b in enumerate(bindings):
            bd[i] = hr_material_textures(b.get("albedo", -1), b.get("normal", -1), b.get("roughness", -1), b.get("roughness_channel", 0), b.get("metallic", -1),
                                         b.get("metallic_channel", 0), b.get("emissive", -1))
        self.check(self.lib.hr_scene_set_textures(scene, tx, C.c_size_t(len(textures)), bd, C.c_size_t(len(bindings))), "hr_scene_set_textures")

    def scene_info(self, scene):
        info = hr_scene_info()
        self.check(self.lib.hr_scene_get_info(scene, C.byref(info)), "hr_scene_get_info")
        return info

    def gbuffer_create(self, W, H):
        self.check(self.lib.hr_gbuffer_create(self.h, W, H), "hr_gbuffer_create")

    def gbuffer_upload(self, slot, g: GBufferHost, stream=0):
        d = g.desc()
        self.check(self.lib.hr_gbuffer_upload(self.h, slot, C.byref(d), C.c_void_p(stream)), "hr_gbuffer_upload")

    def gbuffer_stage_upload(self, g: GBufferHost):
        """Start the PCIe copy of the NEXT frame's (pinned) G-buffer on the library's upload stream; returns immediately."""
        d = g.desc()
        self.check(self.lib.hr_gbuffer_stage_upload(self.h, C.byref(d)), "hr_gbuffer_stage_upload")

    def gbuffer_commit_staged(self, slot, stream=0):
        self.check(self.lib.hr_gbuffer_commit_staged(self.h, slot, C.c_void_p(stream)), "hr_gbuffer_commit_staged")

    def gbuffer_copy_from_device(self, slot, desc: hr_gbuffer_desc, stream=0):
        self.check(self.lib.hr_gbuffer_copy_from_device(self.h, slot, C.byref(desc), C.c_void_p(stream)), "hr_gbuffer_copy_from_device")

    def gbuffer_bind_device(self, slot, desc: hr_gbuffer_desc, stream=0):
        self.check(self.lib.hr_gbuffer_bind_device(self.h, slot, C.byref(desc), C.c_void_p(stream)), "hr_gbuffer_bind_device")

    def gbuffer_render(self, slot, frame, row0=0, row1=0, stream=0):
        """device G-buffer producer (hr_gbuffer_render): primary-visibility ray cast of the current scene into `slot`"""
        self.check(self.lib.hr_gbuffer_render(self.h, slot, C.byref(frame), row0, row1, C.c_void_p(stream)), "hr_gbuffer_render")

    def gbuffer_stage_render(self, frame):
        """start the NEXT frame's G-buffer ray cast on the library's side stream (hr_gbuffer_stage_render); commit with gbuffer_commit_staged"""
        self.check(self.lib.hr_gbuffer_stage_render(self.h, C.byref(frame)), "hr_gbuffer_stage_render")

    def gbuffer_render_sharded(self, slot, frame, halo_rows=48, stream=0):
        self.check(self.lib.hr_gbuffer_render_sharded(self.h, slot, C.byref(frame), halo_rows, C.c_void_p(stream)), "hr_gbuffer_render_sharded")

    def gbuffer_download(self, slot, mip, which, W, H):
        w, h = W, H
        for _ in range(mip):
            w, h = max(w // 2, 1), max(h // 2, 1)
        if which == 0:
            a = np.empty((h, w), np.float32)
        elif which == 1:
            a = np.empty((h, w, 4), np.uint8)
        else:
            a = np.empty((h, w, 4), np.uint16)
        self.check(self.lib.hr_gbuffer_download(self.h, slot, mip, which, _ptr(a), C.c_size_t(a.nbytes)), "hr_gbuffer_download")
        return a

    def shard_set_gather(self, on):
        self.check(self.lib.hr_shard_set_gather(self.h, int(on)), "hr_shard_set_gather")

    def shard_config(self, rank, world):
        self.check(self.lib.hr_shard_config(self.h, rank, world), "hr_shard_config")

    def shard_init(self, rank, world, unique_id: bytes):
        buf = C.create_string_buffer(unique_id, 128)
        self.check(self.lib.hr_shard_init(self.h, rank, world, buf), "hr_shard_init")

    def shard_shutdown(self):
        self.lib.hr_shard_shutdown(self.h)

    def launch_count(self):
        return int(self.lib.hr_ctx_launch_count(self.h))

    def set_profiling(self, on):
        self.lib.hr_ctx_set_profiling(self.h, int(on))


class Pass:
    def __init__(self, ctx: Context, kind, W, H, scale):
        self.ctx, self.kind, self.lib = ctx, kind, ctx.lib
        h = C.c_void_p()
        create = {"shadows": self.lib.hr_shadows_create, "ao": self.lib.hr_ao_create}[kind]
        ctx.check(create(ctx.h, W, H, scale, C.byref(h)), f"hr_{kind}_create")
        self.h = h
        if kind == "shadows":
            self.params = hr_shadows_params()
            self.lib.hr_shadows_default_params(C.byref(self.params))
        else:
            self.params = hr_ao_params()
            self.lib.hr_ao_default_params(C.byref(self.params))

    def render(self, frame: hr_frame, stream=0):
        fn = {"shadows": self.lib.hr_shadows_render, "ao": self.lib.hr_ao_render}[self.kind]
        self.ctx.check(fn(self.h, C.byref(frame), C.byref(self.params), C.c_void_p(stream)), f"hr_{self.kind}_render")

    def output(self, which):
        img = hr_image()
        self.ctx.check(self.lib.hr_pass_output(self.h, which, C.byref(img)), "hr_pass_output")
        return img

    def download(self, which, stream=0, out=None):
        img = self.output(which)
        dt, ch = HR_FMT[img.format]
        shape = (img.height, img.width) if ch == 1 else (img.height, img.width, ch)
        a = out if out is not None else np.empty(shape, np.dtype(dt))
        self.ctx.check(self.lib.hr_pass_download(self.h, which, _ptr(a), C.c_size_t(a.nbytes), C.c_void_p(stream)), "hr_pass_download")
        return a

    def download_rows_async(self, which, row0, row1, out, stream=0):
        """rows [row0,row1) of the image into `out` (pinned, exactly that many rows), no synchronisation"""
        self.ctx.check(self.lib.hr_pass_download_rows_async(self.h, which, row0, row1, _ptr(out), C.c_size_t(out.nbytes), C.c_void_p(stream)),
                       "hr_pass_download_rows_async")
        return out

    def link_local(self, rank, peer):
        """same-process peer history: rank `rank`'s band of this pass's history lives in `peer` (hr_shard_link_local)"""
        self.ctx.check(self.lib.hr_shard_link_local(self.h, rank, peer.h), "hr_shard_link_local")

    def download_async(self, which, out, stream=0):
        """Enqueue the device -> host copy on `stream` without synchronising (out: pinned array of the image's size)."""
        self.ctx.check(self.lib.hr_pass_download_async(self.h, which, _ptr(out), C.c_size_t(out.nbytes), C.c_void_p(stream)), "hr_pass_download_async")
        return out

    def upload(self, which, a, stream=0):
        a = np.ascontiguousarray(a)
        self.ctx.check(self.lib.hr_pass_upload(self.h, which, _ptr(a), C.c_size_t(a.nbytes), C.c_void_p(stream)), "hr_pass_upload")

    def stage_times(self):
        names = (C.c_char_p * 32)()
        ms = (C.c_float * 32)()
        n = C.c_int()
        self.ctx.check(self.lib.hr_pass_stage_times(self.h, names, ms, 32, C.byref(n)), "hr_pass_stage_times")
        return [(names[i].decode(), float(ms[i])) for i in range(n.value)]

    def reset_history(self):
        self.lib.hr_pass_reset_history(self.h)

    def stats(self, stream=0):
        """work done since the previous call (rays) / by the last render (tiles): hr_pass_get_stats"""
        s = hr_pass_stats()
        self.ctx.check(self.lib.hr_pass_get_stats(self.h, C.byref(s), C.c_void_p(stream)), "hr_pass_get_stats")
        return s

    def checksum(self, which=100, row0=0, row1=0, stream=0):
        """device-side order-independent checksum of an output image (rows [row0,row1), default whole image)"""
        v = C.c_uint64()
        self.ctx.check(self.lib.hr_pass_output_checksum(self.h, which, row0, row1, C.byref(v), C.c_void_p(stream)), "hr_pass_output_checksum")
        return int(v.value)

    def destroy(self):
        if self.h:
            self.lib.hr_pass_destroy(self.h)
            self.h = None


class hr_ddgi_uniforms(C.Structure):
    _fields_ = [("grid_start_position", C.c_float * 3), ("grid_step", C.c_float * 3), ("probe_counts", C.c_int32 * 3), ("max_distance", C.c_float),
                ("depth_sharpness", C.c_float), ("hysteresis", C.c_float), ("normal_bias", C.c_float), ("energy_preservation", C.c_float),
                ("irradiance_probe_side_length", C.c_int32), ("irradiance_texture_width", C.c_int32), ("irradiance_texture_height", C.c_int32),
                ("depth_probe_side_length", C.c_int32), ("depth_texture_width", C.c_int32), ("depth_texture_height", C.c_int32),
                ("rays_per_probe", C.c_int32), ("visibility_test", C.c_int32)]


class hr_ddgi_params(C.Structure):
    _fields_ = [("infinite_bounces", C.c_int32), ("infinite_bounce_intensity", C.c_float), ("rays_per_probe", C.c_int32), ("visibility_test", C.c_int32),
                ("probe_distance", C.c_float), ("recursive_energy_preservation", C.c_float), ("irradiance_oct_size", C.c_int32), ("depth_oct_size", C.c_int32),
                ("hysteresis", C.c_float), ("depth_sharpness", C.c_float), ("normal_bias", C.c_float), ("gi_intensity", C.c_float), ("sky_color", C.c_float * 3)]


class hr_reflections_params(C.Structure):
    _fields_ = [("bias", C.c_float), ("trim", C.c_float), ("sample_gi", C.c_int32), ("approximate_with_ddgi", C.c_int32), ("gi_intensity", C.c_float),
                ("rough_ddgi_intensity", C.c_float), ("ibl_indirect_specular_intensity", C.c_float), ("alpha", C.c_float), ("moments_alpha", C.c_float),
                ("blur_as_input", C.c_int32), ("phi_color", C.c_float), ("phi_normal", C.c_float), ("sigma_depth", C.c_float), ("radius", C.c_int32),
                ("filter_iterations", C.c_int32), ("feedback_iteration", C.c_int32), ("denoise", C.c_int32), ("sky_color", C.c_float * 3), ("spp", C.c_int32)]


class hr_deferred_params(C.Structure):
    _fields_ = [("env_color", C.c_float * 3)]


def brdf_lut(samples=128):
    """synthetic stand-in for textures/brdf_lut.bin: 512 x 512 RG16F split-sum LUT (host/synth.cpp::hrs_brdf_lut)"""
    a = np.empty((512, 512, 2), np.uint16)
    L = load_synth()
    L.hrs_brdf_lut.argtypes = [C.c_int, C.c_void_p]
    L.hrs_brdf_lut(samples, _ptr(a))
    return a


def rotation_matrix(angle, axis):
    """glm::mat4_cast(glm::angleAxis(angle, normalize(axis))) as 16 column-major floats (ddgi.cpp:788)"""
    ax = np.asarray(axis, np.float64)
    ax = ax / np.linalg.norm(ax)
    c, s, t = np.cos(angle), np.sin(angle), 1.0 - np.cos(angle)
    x, y, z = ax
    R = np.array([[t * x * x + c, t * x * y - s * z, t * x * z + s * y], [t * x * y + s * z, t * y * y + c, t * y * z - s * x],
                  [t * x * z - s * y, t * y * z + s * x, t * z * z + c]])
    M = np.eye(4)
    M[:3, :3] = R
    return np.ascontiguousarray(M.T.reshape(16), np.float32)  # column-major


class DDGIPass(Pass):
    def __init__(self, ctx: Context, W, H, scale=0):
        self.ctx, self.kind, self.lib = ctx, "ddgi", ctx.lib
        h = C.c_void_p()
        ctx.check(self.lib.hr_ddgi_create(ctx.h, W, H, scale, C.byref(h)), "hr_ddgi_create")
        self.h = h
        self.params = hr_ddgi_params()
        self.lib.hr_ddgi_default_params(C.byref(self.params))

    def render(self, frame: hr_frame, rot16, stream=0):
        rot16 = np.ascontiguousarray(rot16, np.float32)
        self.ctx.check(self.lib.hr_ddgi_render(self.h, C.byref(frame), C.byref(self.params), _ptr(rot16), C.c_void_p(stream)), "hr_ddgi_render")

    def uniforms(self):
        u = hr_ddgi_uniforms()
        self.ctx.check(self.lib.hr_ddgi_get_uniforms(self.h, C.byref(u)), "hr_ddgi_get_uniforms")
        return u


class ReflectionsPass(Pass):
    def __init__(self, ctx: Context, W, H, scale=1):
        self.ctx, self.kind, self.lib = ctx, "reflections", ctx.lib
        h = C.c_void_p()
        ctx.check(self.lib.hr_reflections_create(ctx.h, W, H, scale, C.byref(h)), "hr_reflections_create")
        self.h = h
        self.params = hr_reflections_params()
        self.lib.hr_reflections_default_params(C.byref(self.params))

    def render(self, frame: hr_frame, ddgi: DDGIPass = None, stream=0):
        self.ctx.check(self.lib.hr_reflections_render(self.h, C.byref(frame), C.byref(self.params), ddgi.h if ddgi is not None else None, C.c_void_p(stream)),
                       "hr_reflections_render")


class DeferredPass(Pass):
    """deferred shading combine (hr_deferred_*): consumes the four pass outputs + G-buffer"""

    def __init__(self, ctx: Context, W, H):
        self.ctx, self.kind, self.lib = ctx, "deferred", ctx.lib
        h = C.c_void_p()
        ctx.check(self.lib.hr_deferred_create(ctx.h, W, H, C.byref(h)), "hr_deferred_create")
        self.h = h
        self.params = hr_deferred_params()

    def render(self, frame: hr_frame, shadows=None, ao=None, reflections=None, ddgi=None, stream=0):
        hs = [x.h if x is not None else None for x in (shadows, ao, reflections, ddgi)]
        self.ctx.check(self.lib.hr_deferred_render(self.h, C.byref(frame), C.byref(self.params), hs[0], hs[1], hs[2], hs[3], C.c_void_p(stream)), "hr_deferred_render")


class hr_taa_params(C.Structure):
    _fields_ = [("feedback_min", C.c_float), ("feedback_max", C.c_float), ("sharpen", C.c_int32), ("reset_every_frame", C.c_int32)]


class hr_tonemap_params(C.Structure):
    _fields_ = [("exposure", C.c_float), ("single_channel", C.c_int32)]


def taa_jitter(num_frames, W, H):
    """TemporalAA::update (hr_taa_jitter): (x, y) jitter of frame num_frames; pure host function"""
    out = (C.c_float * 2)()
    L = load_product()
    L.hr_taa_jitter.restype = None
    L.hr_taa_jitter.argtypes = [C.c_uint32, C.c_int, C.c_int, C.POINTER(C.c_float)]
    L.hr_taa_jitter(num_frames, W, H, out)
    return np.array(out[:], np.float32)


def apply_jitter(frame, current, previous, first_frame=None):
    """What HybridRendering::update_uniforms does with the TAA jitter (main.cpp:941-957) to an hr_frame built without it:
    projection' = translate(current) * projection, hence view_proj' = J * view_proj, view_proj_inverse' = view_proj_inverse * J^-1,
    proj_inverse' = proj_inverse * J^-1, prev_view_proj' = J * prev_view_proj (not on the first frame), current_prev_jitter = (current, previous).
    Same arithmetic as hr::TemporalAA::apply_jitter (host/hybrid_rendering.h)."""
    def mat(a):
        return np.array(a[:], np.float32).reshape(4, 4).T  # column-major -> M[r, c]

    def put(a, M):
        a[:] = [float(v) for v in np.ascontiguousarray(M.T, np.float32).reshape(-1)]

    J, Ji = np.eye(4, dtype=np.float32), np.eye(4, dtype=np.float32)
    J[0, 3], J[1, 3] = current[0], current[1]
    Ji[0, 3], Ji[1, 3] = -current[0], -current[1]
    u = frame.ubo
    put(u.view_proj, J @ mat(u.view_proj))
    put(u.view_proj_inverse, mat(u.view_proj_inverse) @ Ji)
    put(u.proj_inverse, mat(u.proj_inverse) @ Ji)
    if not (frame.first_frame if first_frame is None else first_frame):
        put(u.prev_view_proj, J @ mat(u.prev_view_proj))
    u.current_prev_jitter[0], u.current_prev_jitter[1], u.current_prev_jitter[2], u.current_prev_jitter[3] = [float(v) for v in (current[0], current[1], previous[0], previous[1])]
    return frame


class TAAPass(Pass):
    """temporal anti-aliasing (hr_taa_*): resolves another pass's final output against its own previous output"""

    def __init__(self, ctx: Context, W, H):
        self.ctx, self.kind, self.lib = ctx, "taa", ctx.lib
        h = C.c_void_p()
        ctx.check(self.lib.hr_taa_create(ctx.h, W, H, C.byref(h)), "hr_taa_create")
        self.h = h
        self.params = hr_taa_params()
        self.lib.hr_taa_default_params(C.byref(self.params))

    def render(self, frame: hr_frame, input_pass, stream=0):
        self.ctx.check(self.lib.hr_taa_render(self.h, C.byref(frame), C.byref(self.params), input_pass.h, C.c_void_p(stream)), "hr_taa_render")


class TonemapPass(Pass):
    """tone map (hr_tonemap_*): exposure + ACES + gamma -> RGBA8"""

    def __init__(self, ctx: Context, W, H):
        self.ctx, self.kind, self.lib = ctx, "tonemap", ctx.lib
        h = C.c_void_p()
        ctx.check(self.lib.hr_tonemap_create(ctx.h, W, H, C.byref(h)), "hr_tonemap_create")
        self.h = h
        self.params = hr_tonemap_params()
        self.lib.hr_tonemap_default_params(C.byref(self.params))

    def render(self, input_pass, stream=0):
        self.ctx.check(self.lib.hr_tonemap_render(self.h, C.byref(self.params), input_pass.h, C.c_void_p(stream)), "hr_tonemap_render")


class hr_path_tracer_params(C.Structure):
    _fields_ = [("max_ray_bounces", C.c_int32), ("roughness_multiplier", C.c_float), ("sky_color", C.c_float * 3), ("trace_indirect", C.c_int32)]


class PathTracerPass(Pass):
    """ground-truth progressive path tracer (hr_path_tracer_*); reset_history() = restart_accumulation().  params.trace_indirect = 1 traces
    the indirect bounces up to params.max_ray_bounces path vertices (0, the default, is the reference as written); download(2) is then the
    path hash (HR_PATH_TRACER_OUT_PATH_HASH)"""

    def __init__(self, ctx: Context, W, H):
        self.ctx, self.kind, self.lib = ctx, "path_tracer", ctx.lib
        h = C.c_void_p()
        ctx.check(self.lib.hr_path_tracer_create(ctx.h, W, H, C.byref(h)), "hr_path_tracer_create")
        self.h = h
        self.params = hr_path_tracer_params()
        self.lib.hr_path_tracer_default_params(C.byref(self.params))

    def render(self, frame: hr_frame, stream=0):
        self.ctx.check(self.lib.hr_path_tracer_render(self.h, C.byref(frame), C.byref(self.params), C.c_void_p(stream)), "hr_path_tracer_render")
