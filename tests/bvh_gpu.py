"""Device BVH helpers shared by the GPU BVH tests: triangle soups as scenes, hr_trace_* against the oracle's brute-force
loop over every bvh_cases ray family, the process-wide topology switch, and the rays along bvh_cases.chain."""
import ctypes as C

import numpy as np

import bvh_cases as B
import oracle as O
import pyhr

# Rays from 1e4 scene extents away are compared on the any-hit result only.  At that range Moeller-Trumbore's own rounding
# moves a hit sideways by about 2e-4 of the extent: a ray that crosses a shared edge just inside one triangle is also
# reported as hitting its neighbour at the same t, outside the neighbour's padded box (2^-16 of the extent).  The walk then
# returns the triangle the ray really crosses and brute force the lower-numbered neighbour (one ray in a few thousand,
# measured on an H100).  Closest hits are compared bit for bit up to 1e3 extents.
FAR_RAYS = ("aimed_10000x",)


def array_scene(tri):
    """(n, 9) soup -> pyhr.ArrayScene: one dw::Vertex per corner (position, face normal), identity instance, one material"""
    tri = np.ascontiguousarray(tri, np.float32)
    n = len(tri)
    V = np.zeros((3 * n, 20), np.float32)
    V[:, 0:3] = tri.reshape(-1, 3)
    V[:, 3] = 1.0
    v = tri.reshape(-1, 3, 3).astype(np.float64)
    nrm = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
    ln = np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm = np.where(ln > 0, nrm / np.where(ln > 0, ln, 1), [0.0, 1.0, 0.0])
    V[:, 8:11] = np.repeat(nrm, 3, 0)
    V[:, 12] = 1.0   # tangent
    V[:, 18] = 1.0   # bitangent
    inst = pyhr.hr_instance()
    for k in (0, 5, 10, 15):
        inst.model[k] = 1.0
    inst.first_index, inst.index_count, inst.base_vertex, inst.material_idx = 0, 3 * n, 0, 0
    mat = pyhr.hr_material()
    mat.albedo[:] = (0.7, 0.6, 0.5, 1.0)
    mat.roughness, mat.metallic = 0.4, 0.0
    return pyhr.ArrayScene(V, np.arange(3 * n, dtype=np.uint32), [inst], [mat])


class SoupShading:
    """the attributes oracle.ShadingScene reads from a synthetic scene, for a triangle soup"""

    def __init__(self, tri, asc):
        self.tri = np.ascontiguousarray(tri, np.float32)
        self.asc = asc
        self.n_materials = 1

    def world_triangles(self):
        return self.tri, np.zeros(len(self.tri), np.uint32)

    def world_normals(self):
        return np.ascontiguousarray(self.asc.V[:, 8:11].reshape(-1, 9)), np.zeros(len(self.tri), np.uint32)

    def materials_array(self):
        return self.asc.mats


def gpu_trace(ctx, rays):
    import torch
    n = len(rays)
    dr = torch.from_numpy(np.ascontiguousarray(rays, np.float32)).cuda()
    out_any = torch.empty(n, dtype=torch.int32, device="cuda")
    out_t = torch.empty(n, dtype=torch.float32, device="cuda")
    out_p = torch.empty(n, dtype=torch.int32, device="cuda")
    out_uv = torch.empty((n, 2), dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    L = ctx.lib
    ctx.check(L.hr_trace_any(ctx.h, C.c_void_p(dr.data_ptr()), C.c_size_t(n), C.c_void_p(out_any.data_ptr()), C.c_void_p(st)), "hr_trace_any")
    ctx.check(L.hr_trace_closest(ctx.h, C.c_void_p(dr.data_ptr()), C.c_size_t(n), C.c_void_p(out_t.data_ptr()), C.c_void_p(out_p.data_ptr()),
                                 C.c_void_p(out_uv.data_ptr()), C.c_void_p(st)), "hr_trace_closest")
    torch.cuda.synchronize()
    return out_any.cpu().numpy().view(np.uint32), out_t.cpu().numpy(), out_p.cpu().numpy().view(np.uint32), out_uv.cpu().numpy()


def compare(ctx, osc, rays):
    """number of rays whose any flag differs, and whose closest hit (t, primitive, u, v) differs in any bit"""
    a, t, p, uv = gpu_trace(ctx, rays)
    ra = osc.trace_any(rays)
    rt, rp, ruv = osc.trace_closest(rays)
    bad_any = int(np.count_nonzero(a != ra))
    bad_cl = int(np.count_nonzero((p != rp) | (t.view(np.uint32) != rt.view(np.uint32)) | np.any(uv.view(np.uint32) != ruv.view(np.uint32), 1)))
    return bad_any, bad_cl, (rt, rp)


def build(ctx, tri):
    asc = array_scene(tri)
    v, i, inst, m = asc.raw()
    out = C.c_void_p()
    rc = ctx.lib.hr_scene_build(ctx.h, C.c_void_p(v), C.c_size_t(asc.n_vertices), C.c_void_p(i), C.c_size_t(asc.n_indices), C.c_void_p(inst),
                                C.c_size_t(asc.n_instances), C.c_void_p(m), C.c_size_t(asc.n_materials), C.byref(out))
    return rc, out, asc


def check_scene(ctx, tri, seed=0, n=3000):
    """every ray family (and its interval-end rays) through hr_trace_*: {family: (any mismatches, closest mismatches)}"""
    rc, h, _ = build(ctx, tri)
    ctx.check(rc, "hr_scene_build")
    try:
        ctx.check(ctx.lib.hr_scene_set_current(ctx.h, h), "hr_scene_set_current")
        osc = O.Scene(tri, brute=True)
        report, hits = {}, 0
        for name, rays in B.ray_families(tri, seed=seed, n=n).items():
            ba, bc, (rt, rp) = compare(ctx, osc, rays)
            if name in FAR_RAYS:
                bc = 0  # any-hit only, see FAR_RAYS
            report[name] = (ba, bc)
            hit = rp != 0xFFFFFFFF
            hits += int(hit.sum())
            ba, bc, _ = compare(ctx, osc, B.interval_ends(rays, rt, hit))
            report[name + "+ends"] = (ba, 0 if name in FAR_RAYS else bc)
        return report, hits
    finally:
        ctx.lib.hr_scene_destroy(h)


def bad_entries(report):
    return {k: v for k, v in report.items() if any(v)}


class switches:
    """process-wide hr_debug_set switches, restored to the given defaults on exit"""

    def __init__(self, lib, **kv):
        self.lib, self.kv = lib, {int(k[1:]): v for k, v in kv.items()}
        self.defaults = {3: 1}

    def __enter__(self):
        for k, v in self.kv.items():
            self.lib.hr_debug_set(k, v)
        return self

    def __exit__(self, *exc):
        for k in self.kv:
            self.lib.hr_debug_set(k, self.defaults[k])
        return False


def chain_rays(n):
    """rays along the chain's line from x = 0; t_min between triangle k - 1 and k makes triangle k the closest hit, so the walk
    enters both children of every node on the path to the deepest leaf and keeps one pending entry per level on its stack"""
    x = 2.0 ** np.arange(n)
    rays = np.zeros((n, 8), np.float32)
    rays[:, 0:3] = (0.0, 0.25, 0.25)
    rays[:, 4:7] = (1.0, 0.0, 0.0)
    rays[:, 3] = 0.75 * x
    rays[:, 7] = B.T_FAR
    return rays, x.astype(np.float32)
