"""Material textures (scene_descriptor_set.glsl:180-218 fetch_albedo / fetch_roughness / fetch_metallic; hr_scene_set_textures) on the CPU:
  * the oracle's sampler (oracle/orc_shading.h::Texture2D: mip 0, bilinear, REPEAT, sRGB decode before filtering) against closed forms;
  * the PRODUCT's device functions (hybrid-rendering_b200/csrc/tex_px.cuh, what the TEX kernel instantiations call) built for the host
    (tests/hostemu) against the oracle, bit for bit, for the sampler and for the material fetch at hit points;
  * the oracle's G-buffer and path tracer with textures bound (the GPU parity test of the kernels: tests/widened/test_gpu_with_material_textures.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle as O
import pyhr
from test_assets import synth_arrays

HERE = os.path.dirname(os.path.abspath(__file__))


class TexDesc(C.Structure):
    _fields_ = [("offset", C.c_uint32), ("width", C.c_int32), ("height", C.c_int32), ("srgb", C.c_int32)]


class MatTex(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("albedo", "normal", "roughness", "roughness_channel", "metallic", "metallic_channel", "emissive", "_pad")]


def emu():
    so = os.path.join(HERE, "hostemu", "_build", "libhostemu.so")
    if not os.path.exists(so):
        subprocess.run(["make", "-C", os.path.join(HERE, "hostemu")], check=True, stdout=subprocess.DEVNULL)
    L = C.CDLL(so)
    P, I = C.c_void_p, C.c_int
    L.emu_tex_sample.argtypes = [P, P, I, P, I, P, C.c_size_t, P]
    L.emu_material_at_hit.argtypes = [P, P, I, P, P, P, P, P, P, C.c_size_t, P, P, P]
    L.emu_normal_at_hit.argtypes = [P, P, I, P, P, P, P, P, P, P, C.c_size_t, I, P]
    return L


def srgb_lut():
    """the 256-entry table the library uploads (hr_api.cu) = the oracle's decode: read it back through the oracle by sampling texel centres"""
    ramp = np.arange(256, dtype=np.uint8).reshape(1, 256)
    uv = np.stack([(np.arange(256) + 0.5) / 256.0, np.full(256, 0.5)], -1)
    return np.ascontiguousarray(O.texture_sample(ramp, True, uv)[:, 0])


def pack(textures):
    """what hr_scene_set_textures builds: RGBA8 texels of every texture + descriptors (component fill (r, 0, 0, 255) / (r, g, 0, 255))"""
    texels, desc = [], (TexDesc * len(textures))()
    off = 0
    for i, (a, srgb) in enumerate(textures):
        a = np.ascontiguousarray(a, np.uint8)
        h, w = a.shape[:2]
        c = 1 if a.ndim == 2 else a.shape[2]
        rgba = np.zeros((h, w, 4), np.uint32)
        rgba[..., 3] = 255
        rgba[..., :c] = a.reshape(h, w, c)
        texels.append((rgba[..., 0] | (rgba[..., 1] << 8) | (rgba[..., 2] << 16) | (rgba[..., 3] << 24)).astype(np.uint32).reshape(-1))
        desc[i] = TexDesc(off, w, h, int(srgb))
        off += w * h
    return np.ascontiguousarray(np.concatenate(texels)), desc


def test_sampler_closed_forms():
    img = np.array([[[0, 0, 0, 255], [255, 0, 0, 255]], [[0, 255, 0, 255], [0, 0, 255, 0]]], np.uint8)  # 2 x 2
    # texel centres return the texels; the image centre is the average of all four; REPEAT: uv + integers changes nothing; (0, 0) is the corner
    # shared by the four wrapped texels
    c = O.texture_sample(img, False, [(0.25, 0.25), (0.75, 0.25), (0.25, 0.75), (0.75, 0.75), (0.5, 0.5), (0.0, 0.0), (1.25, -0.75), (-3.75, 7.25)])
    assert np.allclose(c[0], (0, 0, 0, 1)) and np.allclose(c[1], (1, 0, 0, 1)) and np.allclose(c[2], (0, 1, 0, 1)) and np.allclose(c[3], (0, 0, 1, 0))
    assert np.allclose(c[4], (0.25, 0.25, 0.25, 0.75)) and np.allclose(c[5], (0.25, 0.25, 0.25, 0.75))
    assert np.array_equal(c[6], c[0]) and np.array_equal(c[7], c[0])
    # sRGB: decode BEFORE filtering (the mean of decoded black and white = 0.5, not decode(mean)); alpha stays linear; known value of byte 188
    bw = np.array([[[0, 0, 0, 128], [255, 255, 255, 128]]], np.uint8)
    s = O.texture_sample(bw, True, [(0.5, 0.5), (0.25, 0.5)])
    assert np.allclose(s[0, :3], 0.5) and np.isclose(s[0, 3], 128 / 255.0) and np.allclose(s[1, :3], 0.0)
    lut = srgb_lut()
    assert lut[0] == 0.0 and lut[255] == 1.0 and np.isclose(lut[188], 0.5029, atol=2e-4) and np.isclose(lut[10], 10 / 255.0 / 12.92, rtol=1e-6) and np.all(np.diff(lut) > 0)
    # 1- and 2-channel images read (r, 0, 0, 1) / (r, g, 0, 1)
    g = np.array([[100, 200]], np.uint8)
    assert np.allclose(O.texture_sample(g, False, [(0.25, 0.5)])[0], (100 / 255.0, 0, 0, 1))
    rg = np.array([[[100, 50], [200, 150]]], np.uint8)
    assert np.allclose(O.texture_sample(rg, False, [(0.75, 0.5)])[0], (200 / 255.0, 150 / 255.0, 0, 1))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_device_sampler_equals_the_oracle_bit_for_bit(seed):
    rng = np.random.default_rng(seed)
    r = lambda *shape: rng.integers(0, 256, shape, dtype=np.uint8)  # noqa: E731
    textures = [(r(5, 7, 4), True), (r(16, 16), False), (r(3, 2, 2), False), (r(1, 1, 4), True), (r(64, 33, 4), False),
                # 1 x N, N x 1, NPOT sizes, the widest accepted image; sRGB on 1- and 2-channel images
                (r(9, 1, 4), False), (r(1, 11, 4), True), (r(5, 3, 4), True), (r(13, 7), True), (r(17, 33, 2), True), (r(1, 16384, 4), False)]
    texels, desc = pack(textures)
    lut = srgb_lut()
    L = emu()
    base = rng.uniform(-3, 4, (4000, 2))
    borders = []
    for img, _ in textures:  # texel borders and centres of every size, and their float neighbours on both sides
        h, w = img.shape[:2]
        for n in (w, h):
            c = np.concatenate([np.arange(-n, 2 * n + 1) / n, (np.arange(-n, 2 * n + 1) + 0.5) / n]).astype(np.float32)
            borders.append(np.concatenate([c, np.nextafter(c, np.float32(-np.inf)), np.nextafter(c, np.float32(np.inf))]))
    borders = np.concatenate(borders)
    uv = np.concatenate([base, rng.uniform(-1e4, 1e4, (200, 2)),
                         np.stack(np.meshgrid(np.arange(-8, 9) / 7.0, np.arange(-8, 9) / 5.0), -1).reshape(-1, 2),          # exact texel borders of the 7 x 5 image
                         np.stack(np.meshgrid((np.arange(-8, 9) + 0.5) / 16.0, (np.arange(-8, 9) + 0.5) / 16.0), -1).reshape(-1, 2),
                         rng.choice(borders, (3000, 2)),
                         base[:600] + np.array([[4096.0, -4096.0]]), base[600:1200] + np.array([[-8191.0, 8191.0]]),                 # integer offsets
                         rng.uniform(1e5, 1e7, (400, 2)) * rng.choice([-1.0, 1.0], (400, 2)),                                      # few fraction bits
                         rng.uniform(2.2e9, 1e12, (300, 2)) * rng.choice([-1.0, 1.0], (300, 2)),                                    # |u W| >= 2^31 for W >= 1
                         rng.uniform(1.4e5, 1e8, (300, 2)) * rng.choice([-1.0, 1.0], (300, 2))]).astype(np.float32)                # >= 2^31 for the 16384-wide image
    for ti, (img, srgb) in enumerate(textures):
        want = O.texture_sample(img, srgb, uv)
        got = np.empty_like(want)
        L.emu_tex_sample(O.p(texels), desc, len(textures), O.p(lut), ti, O.p(uv), len(uv), O.p(got))
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"texture {ti}: {np.count_nonzero(got != want)} components differ"


def textured_scene(seed=0):
    """the shadows-test scene with planar texture coordinates (u, v) = (x, z) / 4 + y / 8 on every vertex, four textures and bindings on half of
    the materials: albedo (sRGB RGBA), a packed roughness (.g) / metallic (.b) image as glTF uses it, a grey roughness map"""
    rng = np.random.default_rng(seed)
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    V, I, insts, mats = synth_arrays(sc)
    V[:, 4] = V[:, 0] / 4.0 + V[:, 1] / 8.0
    V[:, 5] = V[:, 2] / 4.0 + V[:, 1] / 8.0
    asc = pyhr.ArrayScene(V, I, insts, mats)
    yy, xx = np.mgrid[0:32, 0:32]
    checker = np.zeros((32, 32, 4), np.uint8)
    checker[..., 0] = np.where((xx // 4 + yy // 4) % 2, 230, 40)
    checker[..., 1] = (xx * 8) % 256
    checker[..., 2] = rng.integers(0, 256, (32, 32))
    checker[..., 3] = 255
    orm = rng.integers(0, 256, (16, 8, 4), dtype=np.uint8)
    orm[..., 1] = rng.integers(0, 256, (16, 8))          # roughness in .g: values below MIN_ROUGHNESS * 255 exercise the clamp
    grey = rng.integers(0, 256, (8, 8), dtype=np.uint8)
    bumps = np.zeros((16, 16, 4), np.uint8)  # tangent-space normals tilted up to ~35 degrees, blue (z) dominant like real normal maps
    bumps[..., 0] = 128 + (60 * np.sin(xx[:16, :16] * 0.9)).astype(int)
    bumps[..., 1] = 128 + (60 * np.cos(yy[:16, :16] * 0.7)).astype(int)
    bumps[..., 2] = 230
    bumps[..., 3] = 255
    textures = [(checker, True), (orm, False), (grey, False), (rng.integers(0, 256, (4, 4, 4), dtype=np.uint8), True), (bumps, False)]
    bindings = []
    for k in range(sc.n_materials):
        b = {}
        if k % 5 == 0 or k == 1:
            b.update(normal=4)
        if k % 2 == 0:
            b.update(albedo=0 if k % 4 == 0 else 3)
        if k % 3 == 0:
            b.update(roughness=1, roughness_channel=1, metallic=1, metallic_channel=2)
        elif k % 3 == 1:
            b.update(roughness=2, roughness_channel=0)
        bindings.append(b)
    return sc, asc, textures, bindings


def test_device_material_fetch_equals_the_oracle_bit_for_bit():
    sc, asc, textures, bindings = textured_scene()
    ss = O.ShadingScene(sc, brute=True)
    vuv = asc.primitive_uvs()
    ss.set_textures(textures, bindings, vuv, asc.primitive_tangent_frames())
    rng = np.random.default_rng(3)
    n = 6000
    prim = rng.integers(0, sc.n_tris, n).astype(np.uint32)
    bu = rng.random(n).astype(np.float32)
    bv = (rng.random(n).astype(np.float32) * (1.0 - bu)).astype(np.float32)
    bary = np.stack([bu, bv], -1)
    want = O.fetch_material(ss, prim, bary)
    # the product function starts from the constants fetch_surface computed (roughness already clamped to MIN_ROUGHNESS) and overrides them
    _, _, insts, mats = synth_arrays(sc)
    _, prim_mat = sc.world_normals()
    prim_mat = np.ascontiguousarray(prim_mat, np.uint32)
    albedo = np.array([[mats[m].albedo[0], mats[m].albedo[1], mats[m].albedo[2]] for m in prim_mat[prim]], np.float32)
    rough = np.array([max(mats[m].roughness, 0.1) for m in prim_mat[prim]], np.float32)
    metal = np.array([mats[m].metallic for m in prim_mat[prim]], np.float32)
    texels, desc = pack(textures)
    mt = (MatTex * len(bindings))()
    for i, b in enumerate(bindings):
        mt[i] = MatTex(b.get("albedo", -1), b.get("normal", -1), b.get("roughness", -1), b.get("roughness_channel", 0), b.get("metallic", -1), b.get("metallic_channel", 0), -1, 0)
    lut = srgb_lut()
    emu().emu_material_at_hit(O.p(texels), desc, len(textures), O.p(lut), mt, O.p(vuv), O.p(prim_mat), O.p(prim), O.p(bary), n, O.p(albedo), O.p(rough), O.p(metal))
    got = np.concatenate([albedo, rough[:, None], metal[:, None]], 1)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # something was actually textured, the roughness clamp fired, and unbound materials kept their constants
    ss0 = O.ShadingScene(sc, brute=True)
    base = O.fetch_material(ss0, prim, bary)
    bound = np.array([any(k in bindings[m] for k in ("albedo", "roughness", "metallic")) for m in prim_mat[prim]])
    assert np.array_equal(want[~bound], base[~bound]) and np.mean(np.any(want[bound] != base[bound], axis=1)) > 0.9
    assert want[:, 3].min() == np.float32(0.1) and want[:, 3].max() > 0.9


def test_device_normal_map_fetch_equals_the_oracle_bit_for_bit():
    """fetch_normal / get_normal_from_map: both call sites — the hit shaders' (tangent passed as bitangent, rchit:134) and the G-buffer pass's (real
    frame, g_buffer.frag:100) — host build of csrc/tex_px.cuh::normal_at_hit vs the oracle, plus closed forms"""
    sc, asc, textures, bindings = textured_scene()
    ss = O.ShadingScene(sc, brute=True)
    vuv, vtb = asc.primitive_uvs(), asc.primitive_tangent_frames()
    ss.set_textures(textures, bindings, vuv, vtb)
    rng = np.random.default_rng(5)
    n = 5000
    prim = rng.integers(0, sc.n_tris, n).astype(np.uint32)
    bu = rng.random(n).astype(np.float32)
    bary = np.stack([bu, (rng.random(n).astype(np.float32) * (1.0 - bu)).astype(np.float32)], -1)
    _, prim_mat = sc.world_normals()
    prim_mat = np.ascontiguousarray(prim_mat, np.uint32)
    plain = O.ShadingScene(sc, brute=True)
    n_interp = O.fetch_normal(plain, prim, bary)  # no textures: the interpolated unit normal
    assert np.allclose(np.linalg.norm(n_interp, axis=1), 1.0, atol=1e-6)
    texels, desc = pack(textures)
    mt = (MatTex * len(bindings))()
    for i, b in enumerate(bindings):
        mt[i] = MatTex(b.get("albedo", -1), b.get("normal", -1), b.get("roughness", -1), b.get("roughness_channel", 0), b.get("metallic", -1), b.get("metallic_channel", 0), -1, 0)
    lut = srgb_lut()
    mapped = np.array(["normal" in bindings[m] for m in prim_mat[prim]])
    assert mapped.any() and (~mapped).any()
    for quirk in (1, 0):
        want = O.fetch_normal(ss, prim, bary, hit_shader=bool(quirk))
        got = n_interp.copy()
        emu().emu_normal_at_hit(O.p(texels), desc, len(textures), O.p(lut), mt, O.p(vuv), O.p(vtb), O.p(prim_mat), O.p(prim), O.p(bary), n, quirk, O.p(got))
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        assert np.array_equal(want[~mapped], n_interp[~mapped])                         # materials without a normal map keep the interpolated normal
        assert np.allclose(np.linalg.norm(want, axis=1), 1.0, atol=1e-6)
        tilt = np.degrees(np.arccos(np.clip(np.sum(want[mapped] * n_interp[mapped], axis=1), -1, 1)))
        assert tilt.max() < 50.0 and tilt.mean() > 3.0                                 # the map tilts the normal, moderately (blue-dominant texels)
    a, b = O.fetch_normal(ss, prim, bary, True), O.fetch_normal(ss, prim, bary, False)
    assert not np.array_equal(a[mapped], b[mapped])                                     # the two call sites differ (the rchit quirk is real)
    # a flat map (128, 128, 255) leaves the normal where it is up to the quantisation of 128 / 255 (0.3 degrees)
    flat = np.zeros((2, 2, 4), np.uint8)
    flat[...] = (128, 128, 255, 255)
    ss.set_textures([(flat, False)], [dict(normal=0)] * sc.n_materials, vuv, vtb)
    f = O.fetch_normal(ss, prim, bary, False)
    assert np.degrees(np.arccos(np.clip(np.sum(f * n_interp, axis=1), -1, 1))).max() < 0.5


def test_oracle_gbuffer_and_path_tracer_see_the_textures():
    W, H = 96, 54
    sc, asc, textures, bindings = textured_scene()
    plain, tex = O.ShadingScene(sc, brute=True), O.ShadingScene(sc, brute=True)
    tex.set_textures(textures, bindings, asc.primitive_uvs(), asc.primitive_tangent_frames())
    f = pyhr.make_frame((0, 14, 34), (0, 3, 0), W, H)
    g0, g1 = O.gbuffer_render(plain, f, W, H), O.gbuffer_render(tex, f, W, H)
    # geometry channels identical (depth, motion vectors, curvature — it uses the interpolated normal —, mesh id, linear z); material channels differ:
    # GB1 (albedo, metallic), GB3.x (roughness), and the encoded normal where a normal map is bound
    assert np.array_equal(g0.depth, g1.depth) and np.array_equal(g0.gb2[..., 2:], g1.gb2[..., 2:]) and np.array_equal(g0.gb3[..., 1:], g1.gb3[..., 1:])
    hit = g0.depth != 1.0
    _, _, insts0, _ = synth_arrays(sc)
    has_nmap = np.array(["normal" in bindings[it.material_idx] for it in insts0])
    mid0 = np.clip(g1.gb3[..., 2].view(np.float16).astype(np.int64), 0, len(insts0) - 1)
    nm_px = hit & has_nmap[mid0]
    assert nm_px.any() and np.mean(np.any(g0.gb2[..., :2][nm_px] != g1.gb2[..., :2][nm_px], axis=-1)) > 0.9
    assert np.array_equal(g0.gb2[..., :2][hit & ~nm_px], g1.gb2[..., :2][hit & ~nm_px])
    assert np.mean(np.any(g0.gb1[hit] != g1.gb1[hit], axis=-1)) > 0.3 and np.any(g0.gb3[..., 0] != g1.gb3[..., 0])
    # fetch_roughness clamps TEXTURED roughness to MIN_ROUGHNESS (fp16 of 0.1); pixels of materials without a roughness map keep their constant
    _, _, insts, _ = synth_arrays(sc)
    mesh_id = g1.gb3[..., 2].view(np.float16).astype(np.int64)
    has_rough = np.array([bindings[it.material_idx].get("roughness", -1) >= 0 for it in insts])
    r0, r1 = g0.gb3[..., 0].view(np.float16).astype(np.float32), g1.gb3[..., 0].view(np.float16).astype(np.float32)
    mapped = hit & has_rough[np.clip(mesh_id, 0, len(insts) - 1)]
    assert mapped.any() and r1[mapped].min() >= 0.0999 and np.array_equal(r1[hit & ~mapped], r0[hit & ~mapped])
    # the checker pattern of texture 0 is visible in the floor's albedo: both of its red levels occur (sRGB-decoded: 40 -> 0.021, 230 -> 0.791)
    red = g1.gb1[..., 0][hit]
    assert np.any(np.abs(red.astype(int) - round(0.0212 * 255)) <= 2) and np.any(np.abs(red.astype(int) - round(0.7913 * 255)) <= 2)
    p0, p1 = O.PathTracerOracle(W, H, sky=(0.3, 0.4, 0.6)), O.PathTracerOracle(W, H, sky=(0.3, 0.4, 0.6))
    a, b = p0.render(plain, f), p1.render(tex, f)
    assert np.array_equal(p0.prim, p1.prim) and not np.array_equal(a, b)
    tex.set_textures([], [], np.zeros((0, 6), np.float32))  # removing them restores the constants
    assert np.array_equal(O.gbuffer_render(tex, f, W, H).gb1, g0.gb1)


@pytest.mark.parametrize("case", ["far_uv", "texel_borders", "sizes", "many", "channels", "normal_maps"])
def test_device_fetch_on_the_edge_cases_equals_the_oracle(case):
    """material_at_hit and normal_at_hit (both call sites) of the host build against the oracle on the scenes of texture_cases.py:
    coordinates far from the origin and on texel borders, every size, 300 textures and materials, channels 0..3, normal maps with zero
    tangents; bit for bit, NaNs compared by class"""
    import texture_cases as TC
    c = TC.build(case)
    ss = O.ShadingScene(c.sc, brute=True)
    vuv, vtb = c.vuv(), c.vtb()
    ss.set_textures(c.textures, c.bindings, vuv, vtb)
    rng = np.random.default_rng(11)
    n = 8000
    prim = rng.integers(0, c.sc.n_tris, n).astype(np.uint32)
    bu = rng.random(n).astype(np.float32)
    bary = np.stack([bu, (rng.random(n).astype(np.float32) * (1.0 - bu)).astype(np.float32)], -1)
    bary[:50] = 0.0  # exactly on corner 0, where some tangents are zero
    want = O.fetch_material(ss, prim, bary)
    mats = c.sc.materials_array()
    prim_mat = c.sc.prim_mat
    albedo = np.array([[mats[m].albedo[0], mats[m].albedo[1], mats[m].albedo[2]] for m in prim_mat[prim]], np.float32)
    rough = np.array([max(mats[m].roughness, 0.1) for m in prim_mat[prim]], np.float32)
    metal = np.array([mats[m].metallic for m in prim_mat[prim]], np.float32)
    texels, desc = pack(c.textures)
    mt = (MatTex * len(c.bindings))()
    for i, b in enumerate(c.bindings):
        mt[i] = MatTex(b.get("albedo", -1), b.get("normal", -1), b.get("roughness", -1), b.get("roughness_channel", 0), b.get("metallic", -1), b.get("metallic_channel", 0), -1, 0)
    lut = srgb_lut()
    L = emu()
    L.emu_material_at_hit(O.p(texels), desc, len(c.textures), O.p(lut), mt, O.p(vuv), O.p(prim_mat), O.p(prim), O.p(bary), n, O.p(albedo), O.p(rough), O.p(metal))
    got = np.concatenate([albedo, rough[:, None], metal[:, None]], 1)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    if case == "channels":  # the roughness clamp fired and let values above it through
        assert (want[:, 3] == np.float32(0.1)).any() and (want[:, 3] > np.float32(0.1)).any()
    plain = O.ShadingScene(c.sc, brute=True)
    n_interp = O.fetch_normal(plain, prim, bary)
    for quirk in (1, 0):
        want = O.fetch_normal(ss, prim, bary, hit_shader=bool(quirk))
        got = n_interp.copy()
        L.emu_normal_at_hit(O.p(texels), desc, len(c.textures), O.p(lut), mt, O.p(vuv), O.p(vtb), O.p(prim_mat), O.p(prim), O.p(bary), n, quirk, O.p(got))
        nan_w, nan_g = np.isnan(want), np.isnan(got)
        assert np.array_equal(nan_w, nan_g)
        assert np.array_equal(got[~nan_g].view(np.uint32), want[~nan_w].view(np.uint32))
