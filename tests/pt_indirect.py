"""Scenes and closed forms for the path tracer's indirect mode (hr_path_tracer_params.trace_indirect = 1).  TEST INFRASTRUCTURE ONLY.

* `MeshScene`: a triangle soup with one material, buildable both on the device (`.array_scene`, hr_scene_build) and in the oracle
  (`O.ShadingScene(mesh)`): the world positions and the renormalised vertex normals are computed exactly as hr_scene_build does.
* `icosphere` (inward-facing, smooth normals) and `cube` (flat normals).
* `furnace_expected`: the pixel value of the closed-sphere furnace, by quadrature of evaluate_uber_brdf as written (brdf.glsl:130-142,
  guards included) in float64, independent of the oracle and the kernel.
* `IndirectPathTracerOracle`: the host sequencing of `O.PathTracerOracle` around oracle/orc_path_trace_indirect.cpp.
"""
import ctypes as C

import numpy as np

import oracle as O
import pyhr

FNV_BASIS, FNV_PRIME = 2166136261, 16777619
END_MISS, END_HORIZON, END_MAX_BOUNCES = 0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFFD


def fnv1a(h, w):
    """one word of the path hash (HR_PATH_TRACER_OUT_PATH_HASH) on uint32 arrays"""
    return ((np.asarray(h, np.uint64) ^ np.asarray(w, np.uint64)) * np.uint64(FNV_PRIME)) & np.uint64(0xFFFFFFFF)


def one_segment_hash(prim):
    """the hash of a path that ends with a miss right after its primary hit (a primary miss: no primitive, then the miss code)"""
    prim = np.asarray(prim, np.uint32)
    hit = fnv1a(fnv1a(FNV_BASIS, prim), END_MISS)
    return np.where(prim == 0xFFFFFFFF, fnv1a(FNV_BASIS, END_MISS), hit).astype(np.uint32)


class IndirectPathTracerOracle:
    """GroundTruthPathTracer::render host sequencing (frame counter, two images, ping-pong) with trace_indirect = 1.  .prim: the last render's
    primary primitives; .hash: its path hashes (HR_PATH_TRACER_OUT_PATH_HASH); .secondary_rays: shadow + bounce rays of every render so far."""

    def __init__(self, W, H, max_ray_bounces=2, roughness_multiplier=1.0, sky=(0.0, 0.0, 0.0)):
        L = O.lib()
        if not L.orc_path_trace_indirect.argtypes:
            P, I, U, F = C.c_void_p, C.c_int, C.c_uint32, C.c_float
            L.orc_path_trace_indirect.argtypes = [P, P, I, I, U, U, F, P, P, P, P, P, P]
        self.W, self.H = W, H
        self.img = [np.zeros((H, W, 4), np.uint16), np.zeros((H, W, 4), np.uint16)]
        self.prim = np.full((H, W), 0xFFFFFFFF, np.uint32)
        self.hash = np.zeros((H, W), np.uint32)
        self._rays = np.zeros(1, np.uint64)
        self.frame_idx, self.ping_pong = 0, 0
        self.max_ray_bounces, self.roughness_multiplier, self.sky = max_ray_bounces, roughness_multiplier, np.asarray(sky, np.float32)

    @property
    def secondary_rays(self):
        return int(self._rays[0])

    def restart_accumulation(self):
        self.frame_idx = 0

    def render(self, ss, frame):
        if self.frame_idx == 0:
            self.ping_pong = 0
        r, w = self.ping_pong, 1 - self.ping_pong
        O.lib().orc_path_trace_indirect(ss.h, C.byref(frame), self.W, self.H, self.frame_idx, self.max_ray_bounces, self.roughness_multiplier,
                                        O.p(self.sky), O.p(self.img[r]), O.p(self.img[w]), O.p(self.prim), O.p(self.hash), O.p(self._rays))
        self.frame_idx += 1
        self.ping_pong = 1 - self.ping_pong
        self.final = self.img[w]
        return self.final


class MeshScene:
    """tris (n, 3, 3) positions, vnorm (n, 3, 3) vertex normals, one material (albedo rgb, roughness, metallic)"""

    def __init__(self, tris, vnorm, albedo, roughness, metallic):
        tris = np.ascontiguousarray(tris, np.float32)
        vnorm = np.ascontiguousarray(vnorm, np.float32)
        n = tris.shape[0]
        V = np.zeros((3 * n, 20), np.float32)
        V[:, 0:3] = tris.reshape(-1, 3)
        V[:, 3] = 1.0
        V[:, 8:11] = vnorm.reshape(-1, 3)
        V[:, 12] = 1.0  # tangent / bitangent: unused without normal maps
        V[:, 17] = 1.0
        inst = pyhr.hr_instance()
        for i in range(16):
            inst.model[i] = 1.0 if i % 5 == 0 else 0.0
        inst.first_index, inst.index_count, inst.base_vertex, inst.material_idx = 0, 3 * n, 0, 0
        mat = pyhr.hr_material()
        mat.albedo[0], mat.albedo[1], mat.albedo[2], mat.albedo[3] = albedo[0], albedo[1], albedo[2], 1.0
        mat.roughness, mat.metallic = roughness, metallic
        self.array_scene = pyhr.ArrayScene(V, np.arange(3 * n, dtype=np.uint32), [inst], [mat])
        self._mats = (pyhr.hr_material * 1)(mat)
        self.n_tris, self.n_materials = n, 1
        # hr_scene_build with an identity model: positions unchanged, normals renormalised as normalize(mat3(model) * n) in float32
        v = vnorm.reshape(-1, 3)
        ln = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]).astype(np.float32)
        il = (np.float32(1.0) / ln).astype(np.float32)
        self._tri = tris.reshape(n, 9)
        self._nrm = np.ascontiguousarray((v * il[:, None]).astype(np.float32).reshape(n, 9))

    # the SynthScene methods O.ShadingScene reads
    def world_triangles(self):
        return self._tri, np.zeros(self.n_tris, np.uint32)

    def world_normals(self):
        return self._nrm, np.zeros(self.n_tris, np.uint32)

    def materials_array(self):
        return self._mats


def icosphere(subdivisions=4, radius=10.0):
    """(tris, vnorm) of an icosphere with 20 * 4^subdivisions triangles, wound and shaded to face its centre"""
    t = (1.0 + 5.0 ** 0.5) / 2.0
    verts = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    verts = [np.array(v, np.float64) / np.linalg.norm(v) for v in verts]
    faces = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
             (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    for _ in range(subdivisions):
        cache, nf = {}, []

        def mid(a, b):
            k = (min(a, b), max(a, b))
            if k not in cache:
                m = verts[a] + verts[b]
                verts.append(m / np.linalg.norm(m))
                cache[k] = len(verts) - 1
            return cache[k]
        for a, b, c in faces:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = nf
    P = np.array(verts)
    F = np.array(faces)[:, ::-1]  # inward winding
    tris = (P[F] * radius).astype(np.float32)
    vnorm = (-P[F]).astype(np.float32)
    return tris, vnorm


def cube(half=2.0, center=(0.0, 1.0, 0.0)):
    """(tris, vnorm) of an axis-aligned cube with one flat normal per face"""
    c = np.asarray(center, np.float64)
    tris, nrm = [], []
    for axis in range(3):
        for s in (-1.0, 1.0):
            n = np.zeros(3)
            n[axis] = s
            u, v = np.zeros(3), np.zeros(3)
            u[(axis + 1) % 3], v[(axis + 2) % 3] = 1.0, 1.0
            q = [c + half * (n + a * u + b * v) for a, b in ((-1, -1), (1, -1), (1, 1), (-1, 1))]
            for tri in ((q[0], q[1], q[2]), (q[0], q[2], q[3])):
                tris.append(tri if s > 0 else tri[::-1])
                nrm.append((n, n, n))
    return np.array(tris, np.float32), np.array(nrm, np.float32)


# ---- closed-sphere furnace -----------------------------------------------------------------------------------------------------------
def uber_brdf(cd, F0, roughness, cos_o, cos_i, phi):
    """evaluate_uber_brdf (brdf.glsl:130-142) as written, float64, Wo = (sin o, 0, cos o), Wi = (sin i cos phi, sin i sin phi, cos i), N = z"""
    so, si = np.sqrt(np.maximum(1.0 - cos_o ** 2, 0.0)), np.sqrt(np.maximum(1.0 - cos_i ** 2, 0.0))
    wo = np.stack(np.broadcast_arrays(so, 0.0 * so, cos_o), -1)
    wi = np.stack(np.broadcast_arrays(si * np.cos(phi), si * np.sin(phi), cos_i), -1)
    h = wo + wi
    h = h / np.linalg.norm(h, axis=-1, keepdims=True)
    NdotL, NdotV, NdotH = np.maximum(wi[..., 2], 0.0), np.maximum(wo[..., 2], 0.0), np.maximum(h[..., 2], 0.0)
    VdotH = np.maximum(np.sum(wi * h, -1), 0.0)
    F = F0 + (1.0 - F0) * (1.0 - VdotH) ** 5
    a2 = (roughness * roughness) ** 2
    denom = NdotH * NdotH * (a2 - 1.0) + 1.0
    D = a2 / np.maximum(1e-4, np.pi * denom * denom)
    k = (roughness + 1.0) ** 2 / 8.0
    G1 = lambda x: x / np.maximum(1e-4, x * (1.0 - k) + k)  # noqa: E731
    spec = D * (G1(NdotL) * G1(NdotV)) / np.maximum(1e-4, 4.0 * NdotL * NdotV)
    return (1.0 - F) * (cd / np.pi) + F * spec


def furnace_expected(albedo, roughness, metallic, intensity, radius, bounces, n_mu=256, n_phi=512):
    """L_B(0) of L_1(o) = f(o, N) I / r^2, L_B(o) = L_1(o) + int f(o, wi) L_{B-1}(i) cos i dwi for B in `bounces` (grey albedo): the pixel
    value of the closed sphere with a point light at its centre seen from the centre.  Every chord leaves and meets the sphere at the
    same angle to the normal, so the radiance leaving a wall point depends only on its angle."""
    F0 = 0.04 * (1.0 - metallic) + albedo * metallic
    cd = albedo * (1.0 - F0) * (1.0 - metallic)
    x, w = np.polynomial.legendre.leggauss(n_mu)
    mu, wmu = 0.5 * (x + 1.0), 0.5 * w                       # cos i in (0, 1)
    phi = (np.arange(n_phi) + 0.5) * (2.0 * np.pi / n_phi)
    cos_o = np.concatenate([[1.0], mu])                      # row 0: the primary vertex, seen at normal incidence
    L1 = uber_brdf(cd, F0, roughness, cos_o, 1.0, 0.0) * intensity / radius ** 2
    K = np.empty((len(cos_o), n_mu))
    for j, co in enumerate(cos_o):
        f = uber_brdf(cd, F0, roughness, co, mu[:, None], phi[None, :])
        K[j] = f.sum(1) * (2.0 * np.pi / n_phi) * mu * wmu
    out, L = {}, L1.copy()
    for b in range(1, max(bounces) + 1):
        if b > 1:
            L = L1 + K @ L[1:]
        if b in bounces:
            out[b] = float(L[0])
    return out
