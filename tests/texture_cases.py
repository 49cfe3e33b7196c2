"""Material-texture edge cases for the TEX instantiations of the hit-shading kernels (tests/test_gpu_textured_kernels.py) and their
sensitivity check on the CPU (tests/test_texture_sensitivity_cpu.py).

Every case is the shadows-test geometry turned into a triangle soup (every triangle has its own three vertices, so a triangle's texture
coordinates can be set alone), with its own texture coordinates, textures and bindings, built as
  * `asc`, a pyhr.ArrayScene for hr_scene_build, and
  * `sc`, a stand-in for pyhr.SynthScene with the same primitives, instances and materials, for oracle.ShadingScene.
The textures hold independent random texels: picking the wrong texel, channel or decode moves a result by far more than the bars.

  far_uv         texture coordinates offset by integers (+-4096, -8191), of magnitude 1e5 .. 1e7 (u * W - 0.5 keeps few fraction bits)
                 and with |u * W| >= 2^31, where the float -> int conversion saturates and x0 + 1 wraps to INT_MIN
  texel_borders  one constant coordinate on all three corners of a triangle, at texel borders and centres of NPOT textures, nudged by
                 one ulp either way: the interpolated coordinate lands within an ulp of the border, on either side
  sizes          1x1, 1xN, Nx1, 3x5, 7x13, 33x17 and 16384x1 (the widest image hr_scene_set_textures accepts)
  big_offset     an 8193x8192 one-channel image first, so every other texture's TexDesc::offset (in texels) is above 2^26
  many           300 textures and 300 materials on 300+ instances: texture and material indices above 255
  channels       1-, 2- and 4-channel images, sRGB on 1- and 2-channel images too, roughness / metallic channels 0..3 (alpha is never
                 sRGB-decoded), roughness texels 0..26 around the MIN_ROUGHNESS clamp (0.1 * 255 = 25.5)
  normal_maps    normal maps at both call sites, a material bound to a normal map only (material_at_hit's early return), and
                 corners whose tangent is zero (hr_scene_build normalises it to 0)
  untextured     the same soup without textures: the untextured instantiations under the same comparisons
"""
import ctypes as C
import re

import numpy as np

import pyhr
from test_assets import synth_arrays

CASES = ["far_uv", "texel_borders", "sizes", "big_offset", "many", "channels", "normal_maps", "untextured"]


class CaseScene:
    """what oracle.ShadingScene and oracle.gbuffer_render read from a pyhr.SynthScene, for a soup with its own instances and materials"""

    def __init__(self, synth, prim_inst, prim_mat, materials):
        self.synth = synth
        self.prim_inst, self.prim_mat = np.ascontiguousarray(prim_inst, np.uint32), np.ascontiguousarray(prim_mat, np.uint32)
        self.mats = (pyhr.hr_material * len(materials))(*materials)
        self.n_materials = len(materials)
        self.n_tris = synth.n_tris

    def world_triangles(self):
        tri, _ = self.synth.world_triangles()
        return tri, self.prim_inst.copy()

    def world_normals(self):
        nrm, _ = self.synth.world_normals()
        return nrm, self.prim_mat.copy()

    def materials_array(self):
        return self.mats

    def bounds(self):
        return self.synth.bounds()


class Case:
    def __init__(self, name, sc, asc, textures, bindings):
        self.name, self.sc, self.asc, self.textures, self.bindings = name, sc, asc, textures, bindings

    def vuv(self):
        return self.asc.primitive_uvs()

    def vtb(self):
        return self.asc.primitive_tangent_frames()


def _soup(split=1):
    """the shadows-test scene as a triangle soup; split > 1 cuts every instance into pieces of `split` triangles (one instance each)"""
    synth = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    V, I, insts, mats = synth_arrays(synth)
    rows, new_insts = [], []
    n = 0
    for it in insts:
        idx = I[it.first_index: it.first_index + it.index_count // 3 * 3].astype(np.int64) + it.base_vertex
        rows.append(V[idx])
        step = 3 * split if split > 1 else len(idx)
        for a in range(0, len(idx), step):
            c = min(step, len(idx) - a)
            new_insts.append(pyhr.hr_instance((C.c_float * 16)(*it.model[:]), n + a, c, 0, it.material_idx))
        n += len(idx)
    Vs = np.ascontiguousarray(np.concatenate(rows), np.float32)
    return synth, Vs, np.arange(len(Vs), dtype=np.uint32), new_insts, mats


def _planar(V):
    V[:, 4] = V[:, 0] / 4.0 + V[:, 1] / 8.0
    V[:, 5] = V[:, 2] / 4.0 + V[:, 1] / 8.0


def _finish(name, synth, V, I, insts, mats, textures, bindings):
    asc = pyhr.ArrayScene(V, I, insts, mats)
    prim_inst = np.concatenate([np.full(it.index_count // 3, k) for k, it in enumerate(insts)])
    prim_mat = np.concatenate([np.full(it.index_count // 3, it.material_idx) for it in insts])
    return Case(name, CaseScene(synth, prim_inst, prim_mat, mats), asc, textures, bindings)


def _bind_cycle(n_materials, n_textures, rng, normal=None):
    """bindings that use every texture: albedo / roughness / metallic from different textures, all four channels"""
    out = []
    for k in range(n_materials):
        b = dict(albedo=int(rng.integers(0, n_textures)))
        if k % 3 != 2:
            b.update(roughness=int(rng.integers(0, n_textures)), roughness_channel=k % 4)
        if k % 2 == 0:
            b.update(metallic=int(rng.integers(0, n_textures)), metallic_channel=(k + 1) % 4)
        if normal is not None and k % 4 == 1:
            b.update(normal=normal)
        out.append(b)
    return out


def build(name, seed=0):
    rng = np.random.default_rng(seed + 17 * CASES.index(name))
    rnd = lambda *shape: rng.integers(0, 256, shape, dtype=np.uint8)  # noqa: E731
    synth, V, I, insts, mats = _soup(split=6 if name == "many" else 1)
    _planar(V)
    if name == "untextured":
        return _finish(name, synth, V, I, insts, mats, [], [])
    if name == "far_uv":
        # per instance: an integer offset, a huge coordinate, or one past 2^31 texels
        shifts = [(4096.0, -4096.0), (-8191.0, 4096.0), (1e5, 2e5), (3e6, -1e6), (1e7, 7e6), (-4e7, 9e7), (2.5e8, -3e8)]
        prim_of_inst = np.concatenate([np.full(it.index_count, k) for k, it in enumerate(insts)])
        for k in range(len(insts)):
            su, sv = shifts[k % len(shifts)]
            rows = prim_of_inst == k
            V[rows, 4] += np.float32(su)
            V[rows, 5] += np.float32(sv)
        textures = [(rnd(13, 7, 4), True), (rnd(17, 33, 4), False), (rnd(64, 64), False), (rnd(5, 3, 2), False)]
        return _finish(name, synth, V, I, insts, mats, textures, _bind_cycle(len(mats), len(textures), rng))
    if name == "texel_borders":
        textures = [(rnd(5, 3, 4), True), (rnd(13, 7, 4), False), (rnd(17, 33, 4), True)]
        n_tri = len(V) // 3
        cand = []
        for (img, _) in textures:
            h, w = img.shape[:2]
            for n in (w, h):
                for k in range(-n, 2 * n + 1):
                    for c in (k / n, (k + 0.5) / n):
                        f = np.float32(c)
                        cand += [f, np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))]
        cand = np.array(cand, np.float32)
        uv = cand[rng.integers(0, len(cand), (n_tri, 2))]
        V[:, 4] = np.repeat(uv[:, 0], 3)
        V[:, 5] = np.repeat(uv[:, 1], 3)
        return _finish(name, synth, V, I, insts, mats, textures, _bind_cycle(len(mats), len(textures), rng))
    if name == "sizes":
        textures = [(rnd(1, 1, 4), True), (rnd(9, 1, 4), False), (rnd(1, 11, 4), True), (rnd(5, 3, 4), False), (rnd(13, 7, 4), True),
                    (rnd(17, 33, 4), False), (rnd(1, 16384, 4), True)]
        V[:, 4] *= np.float32(3.0)  # several wraps of every image across a triangle
        return _finish(name, synth, V, I, insts, mats, textures, _bind_cycle(len(mats), len(textures), rng))
    if name == "big_offset":
        textures = [(rnd(8192, 8193), False), (rnd(13, 7, 4), True), (rnd(17, 33, 4), False), (rnd(9, 1, 2), False)]
        bindings = _bind_cycle(len(mats), len(textures) - 1, rng)
        for b in bindings:  # the small textures, indices 1..3, carry the colours; texture 0 is bound as one material's roughness
            for k in ("albedo", "roughness", "metallic"):
                if k in b:
                    b[k] += 1
        bindings[0].update(roughness=0, roughness_channel=0)
        return _finish(name, synth, V, I, insts, mats, textures, bindings)
    if name == "many":
        n = 300
        base = list(mats)
        mats = []
        for k in range(n):
            m = pyhr.hr_material.from_buffer_copy(base[k % len(base)])
            m.albedo[0] = float(rng.uniform(0.1, 0.9))
            mats.append(m)
        for k, it in enumerate(insts):  # instance k -> material k (mod n), then the highest indices first
            it.material_idx = (n - 1 - k) % n
        textures = [(rnd(int(rng.integers(1, 9)), int(rng.integers(1, 9)), 4), bool(k % 2)) for k in range(n)]
        bindings = []
        for k in range(n):
            t = (k * 7 + 256) % n  # indices above 255 for most materials
            bindings.append(dict(albedo=t, roughness=(t + 1) % n, roughness_channel=k % 4, metallic=(n - 1 - k), metallic_channel=(k + 2) % 4))
        return _finish(name, synth, V, I, insts, mats, textures, bindings)
    if name == "channels":
        rough1 = rng.integers(0, 27, (6, 5), dtype=np.uint8)  # 0..26: on both sides of MIN_ROUGHNESS * 255
        rough4 = rnd(7, 3, 4)
        rough4[..., :] = rng.integers(0, 27, (7, 3, 4))
        textures = [(rnd(5, 7), True), (rnd(3, 9, 2), True), (rnd(11, 4, 4), True), (rough1, False), (rnd(4, 6, 2), False), (rough4, True), (rnd(9, 5, 4), False)]
        bindings = []
        for k in range(len(mats)):
            b = dict(albedo=(0, 1, 2, 6)[k % 4])  # sRGB 1-, 2- and 4-channel images and a linear one
            b.update(roughness=(3, 4, 5, 6)[k % 4], roughness_channel=k % 4)
            b.update(metallic=(6, 5, 4, 2, 1, 0)[k % 6], metallic_channel=(k // 2) % 4)
            bindings.append(b)
        return _finish(name, synth, V, I, insts, mats, textures, bindings)
    if name == "normal_maps":
        nm = rnd(16, 16, 4)
        nm[..., 2] = rng.integers(160, 256, (16, 16))  # mostly facing out, like real maps
        nm2 = rnd(7, 13, 4)
        nm2[..., 2] = rng.integers(140, 256, (7, 13))
        textures = [(rnd(13, 7, 4), True), (nm, False), (nm2, False), (rnd(5, 3, 4), False)]
        bindings = []
        for k in range(len(mats)):
            if k % 4 == 0:
                bindings.append(dict(normal=1 + (k // 4) % 2))  # normal map only: material_at_hit returns early
            elif k % 4 == 1:
                bindings.append(dict(albedo=0, normal=2, roughness=3, roughness_channel=1))
            elif k % 4 == 2:
                bindings.append(dict(albedo=0, normal=1, metallic=3, metallic_channel=3))
            else:
                bindings.append(dict(roughness=3, roughness_channel=0))
        # a real tangent frame that varies per corner, and one corner of every 7th triangle with a zero tangent (normalised to 0)
        V[:, 12:15] = np.stack([np.ones(len(V)), 0.3 * np.sin(V[:, 0]), 0.2 * np.cos(V[:, 2])], -1)
        V[:, 16:19] = np.stack([0.2 * np.cos(V[:, 0]), 0.1 * np.sin(V[:, 2]), np.ones(len(V))], -1)
        V[::21, 12:15] = 0.0
        return _finish(name, synth, V, I, insts, mats, textures, bindings)
    raise KeyError(name)


# ---- instantiation ledger ------------------------------------------------------------------------------------------------------------
# Every instantiation of a hit-shading kernel that a launch site in rt_shade.cu, gbuffer.cu or reference.cu can select, and the test case
# that launches it and compares its output with the oracle.  test_hit_shading_ledger_cpu.py holds this table to the launch sites (a new
# instantiation fails there until a comparing test is named for it); test_gpu_textured_kernels.py proves with torch.profiler that each
# named case launches its instantiation.
HIT_SHADING_KERNELS = ("k_gbuffer_render", "k_ddgi_ray_trace", "k_reflections_ray_trace", "k_path_trace", "k_reference_reflections", "k_reference_mask")
_TEXTURED = "test_gpu_textured_kernels.py::test_textured_kernels_match_the_oracle[channels]"
_PLAIN = "test_gpu_textured_kernels.py::test_textured_kernels_match_the_oracle[untextured]"
HIT_SHADING = {
    "k_gbuffer_render<true>": _TEXTURED,
    "k_gbuffer_render<false>": _PLAIN,
    "k_ddgi_ray_trace<true>": _TEXTURED,
    "k_ddgi_ray_trace<false>": _PLAIN,
    "k_reflections_ray_trace<true, 8, true, true>": _TEXTURED,      # spp > 1
    "k_reflections_ray_trace<false, 18, true, true>": _TEXTURED,    # spp 1 with the DDGI terms
    "k_reflections_ray_trace<false, 24, true, false>": _TEXTURED,   # spp 1 without them
    "k_reflections_ray_trace<true, 8, false, true>": _PLAIN,
    "k_reflections_ray_trace<false, 18, false, true>": _PLAIN,
    "k_reflections_ray_trace<false, 24, false, false>": _PLAIN,
    "k_path_trace<true, true>": _TEXTURED,
    "k_path_trace<true, false>": _TEXTURED,
    "k_path_trace<false, true>": _PLAIN,
    "k_path_trace<false, false>": _PLAIN,
    "k_reference_reflections<true, true>": _TEXTURED,
    "k_reference_reflections<true, false>": _TEXTURED,
    "k_reference_reflections<false, true>": _PLAIN,
    "k_reference_reflections<false, false>": _PLAIN,
    "k_reference_mask<0>": "test_gpu_reference.py::test_mask_counts_equal_the_oracle",
    "k_reference_mask<1>": "test_gpu_reference.py::test_mask_counts_equal_the_oracle",
}
# position of the TEX template argument of each kernel (k_reference_mask has none)
_TEX_ARG = {"k_gbuffer_render": 0, "k_ddgi_ray_trace": 0, "k_reflections_ray_trace": 2, "k_path_trace": 0, "k_reference_reflections": 0}


def textured(inst):
    """whether an instantiation spelled like a HIT_SHADING key is a TEX = true one"""
    name, args = inst.rstrip(">").split("<")
    return [a.strip() for a in args.split(",")][_TEX_ARG[name]] == "true"


def instantiations(text):
    """the hit-shading instantiations named in `text`, spelled like the HIT_SHADING keys: launch sites `k_x<args><<<`, function-pointer
    selections `k_x<args>` followed by `;`, `:` or `)`, and demangled kernel names `k_x<args>(...)` as torch.profiler reports them"""
    out = set()
    for m in re.finditer(r"\b(" + "|".join(HIT_SHADING_KERNELS) + r")<([^<>]*)>\s*(?:<<<|[;:()])", text):
        out.add(f"{m.group(1)}<{', '.join(a.strip() for a in m.group(2).split(','))}>")
    return out
