"""Scene / asset ingestion (SURVEY.md §8 f3, hybrid-rendering_b200/host/assets.{h,cpp}): CPU tests.

The reference reads its inputs through assimp and stb_image (external/dwSampleFramework/src/mesh.cpp:244-613, src/vk.cpp:136-190,
src/blue_noise.cpp:5-33); neither library nor any asset is in /root/reference, so the loaders are checked against files this test
writes itself with independent encoders (Python's zlib for the deflate streams, struct / json for the containers) and against the
procedural scenes exported to OBJ / glTF and read back bit for bit."""
import base64
import ctypes as C
import json
import os
import struct
import zlib

import numpy as np
import pytest

import pyhr
from pyhr import assets as A


# ---------------------------------------------------------------------------------------------- encoders used by the tests
def _png_chunk(tag, body):
    return struct.pack(">I", len(body)) + tag + body + struct.pack(">I", zlib.crc32(tag + body) & 0xFFFFFFFF)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)


def _filter_rows(rows, bpp, cycle):
    """rows: list of bytes (one scanline each); filter type of row y = cycle[y % len(cycle)]"""
    out = bytearray()
    prev = bytes(len(rows[0])) if rows else b""
    for y, row in enumerate(rows):
        ft = cycle[y % len(cycle)]
        out.append(ft)
        for i, v in enumerate(row):
            a = row[i - bpp] if i >= bpp else 0
            b = prev[i]
            c = prev[i - bpp] if i >= bpp else 0
            pred = [0, a, b, (a + b) >> 1, _paeth(a, b, c)][ft]
            out.append((v - pred) & 0xFF)
        prev = row
    return bytes(out)


def _pack_row(samples, depth):
    """samples: 1-D array of channel-interleaved sample values of one row"""
    if depth == 8:
        return bytes(int(v) for v in samples)
    if depth == 16:
        return b"".join(struct.pack(">H", int(v)) for v in samples)
    bits = "".join(format(int(v), f"0{depth}b") for v in samples)
    bits += "0" * (-len(bits) % 8)
    return bytes(int(bits[i:i + 8], 2) for i in range(0, len(bits), 8))


def write_png(path, samples, ctype, depth, cycle=(0, 1, 2, 3, 4), interlace=False, level=6, plte=None, trns=None, split_idat=1):
    """samples: (H, W, C) integer array of raw sample values (palette indices for colour type 3)"""
    H, W, Cn = samples.shape
    bpp = max(1, depth * Cn // 8)
    if not interlace:
        raw = _filter_rows([_pack_row(samples[y].reshape(-1), depth) for y in range(H)], bpp, cycle)
    else:
        raw = b""
        for x0, y0, dx, dy in [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]:
            sub = samples[y0::dy, x0::dx]
            if sub.shape[0] == 0 or sub.shape[1] == 0:
                continue
            raw += _filter_rows([_pack_row(sub[y].reshape(-1), depth) for y in range(sub.shape[0])], bpp, cycle)
    z = zlib.compress(raw, level)
    body = b"\x89PNG\r\n\x1a\n" + _png_chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, ctype, 0, 0, 1 if interlace else 0))
    if plte is not None:
        body += _png_chunk(b"PLTE", bytes(plte))
    if trns is not None:
        body += _png_chunk(b"tRNS", bytes(trns))
    body += _png_chunk(b"tEXt", b"Comment\x00written by tests/test_assets.py")
    n = max(1, len(z) // split_idat)
    for i in range(0, len(z), n):
        body += _png_chunk(b"IDAT", z[i:i + n])
    body += _png_chunk(b"IEND", b"")
    with open(path, "wb") as f:
        f.write(body)


def write_hdr(path, rgbe, rle):
    H, W, _ = rgbe.shape
    out = b"#?RADIANCE\n# made by tests\nFORMAT=32-bit_rle_rgbe\nEXPOSURE=1.0\n\n" + f"-Y {H} +X {W}\n".encode()
    for y in range(H):
        if not rle:
            out += rgbe[y].tobytes()
            continue
        out += bytes([2, 2, W >> 8, W & 255])
        for c in range(4):
            row = rgbe[y, :, c]
            x = 0
            while x < W:
                run = 1
                while x + run < W and run < 127 and row[x + run] == row[x]:
                    run += 1
                if run >= 3:
                    out += bytes([128 + run, int(row[x])])
                    x += run
                else:
                    lit = min(W - x, 5)
                    out += bytes([lit]) + bytes(int(v) for v in row[x:x + lit])
                    x += lit
    with open(path, "wb") as f:
        f.write(out)


def _f(v):
    return repr(float(np.float32(v)))


def synth_arrays(sc):
    v, i, inst, m = sc.raw()
    V = np.frombuffer((C.c_float * (20 * sc.n_vertices)).from_address(v), np.float32).reshape(-1, 20).copy()
    I = np.frombuffer((C.c_uint32 * sc.n_indices).from_address(i), np.uint32).copy()
    insts = [pyhr.hr_instance.from_buffer_copy(x) for x in (pyhr.hr_instance * sc.n_instances).from_address(inst)]  # copies, not views
    mats = [pyhr.hr_material.from_buffer_copy(x) for x in (pyhr.hr_material * sc.n_materials).from_address(m)]
    return V, I, insts, mats


def export_obj(sc, directory, name="scene"):
    """one OBJ object per synthetic instance (its vertices in object space), one MTL entry per material"""
    V, I, insts, mats = synth_arrays(sc)
    with open(os.path.join(directory, name + ".mtl"), "w") as f:
        for k, m in enumerate(mats):
            f.write(f"newmtl m{k}\nKd {_f(m.albedo[0])} {_f(m.albedo[1])} {_f(m.albedo[2])}\nPr {_f(m.roughness)}\nPm {_f(m.metallic)}\n\n")
    with open(os.path.join(directory, name + ".obj"), "w") as f:
        f.write(f"# exported by tests/test_assets.py\nmtllib {name}.mtl\n")
        nv = 0
        for k, it in enumerate(insts):
            idx = I[it.first_index: it.first_index + it.index_count].astype(np.int64) + it.base_vertex
            f.write(f"o inst{k}\nusemtl m{it.material_idx}\n")
            for vi in idx:
                f.write(f"v {_f(V[vi, 0])} {_f(V[vi, 1])} {_f(V[vi, 2])}\nvn {_f(V[vi, 8])} {_f(V[vi, 9])} {_f(V[vi, 10])}\n")
            for t in range(len(idx) // 3):
                a = nv + 3 * t + 1
                f.write(f"f {a}//{a} {a + 1}//{a + 1} {a + 2}//{a + 2}\n")
            nv += len(idx)
    return os.path.join(directory, name + ".obj"), [np.array(it.model[:], np.float32) for it in insts]


def export_gltf(sc, directory, name="scene", glb=False, arrays=None):
    """one glTF mesh with one primitive per synthetic instance; binary buffer with POSITION / NORMAL / uint32 indices"""
    V, I, insts, mats = arrays if arrays is not None else synth_arrays(sc)
    blob = bytearray()
    views, accessors, prims = [], [], []

    def add(data, target):
        while len(blob) % 4:
            blob.append(0)
        views.append(dict(buffer=0, byteOffset=len(blob), byteLength=len(data), target=target))
        blob.extend(data)
        return len(views) - 1

    for it in insts:
        idx = I[it.first_index: it.first_index + it.index_count].astype(np.int64) + it.base_vertex
        used = np.unique(idx)
        remap = {int(u): k for k, u in enumerate(used)}
        pos, nrm = V[used, 0:3].astype("<f4"), V[used, 8:11].astype("<f4")
        local = np.array([remap[int(i)] for i in idx], "<u4")
        a0 = len(accessors)
        accessors.append(dict(bufferView=add(pos.tobytes(), 34962), componentType=5126, count=len(used), type="VEC3", min=pos.min(0).tolist(), max=pos.max(0).tolist()))
        accessors.append(dict(bufferView=add(nrm.tobytes(), 34962), componentType=5126, count=len(used), type="VEC3"))
        accessors.append(dict(bufferView=add(local.tobytes(), 34963), componentType=5125, count=len(local), type="SCALAR"))
        prims.append(dict(attributes=dict(POSITION=a0, NORMAL=a0 + 1), indices=a0 + 2, material=int(it.material_idx), mode=4))
    doc = dict(asset=dict(version="2.0", generator="tests/test_assets.py"), scene=0, scenes=[dict(nodes=[0])], nodes=[dict(mesh=0)],
               meshes=[dict(name="scene", primitives=prims)], accessors=accessors, bufferViews=views,
               materials=[dict(name=f"m{k}", pbrMetallicRoughness=dict(baseColorFactor=[float(m.albedo[0]), float(m.albedo[1]), float(m.albedo[2]), 1.0],
                                                                         metallicFactor=float(m.metallic), roughnessFactor=float(m.roughness)))
                          for k, m in enumerate(mats)])
    models = [np.array(it.model[:], np.float32) for it in insts]
    if glb:
        doc["buffers"] = [dict(byteLength=len(blob))]
        js = json.dumps(doc).encode()
        js += b" " * (-len(js) % 4)
        while len(blob) % 4:
            blob.append(0)
        total = 12 + 8 + len(js) + 8 + len(blob)
        path = os.path.join(directory, name + ".glb")
        with open(path, "wb") as f:
            f.write(b"glTF" + struct.pack("<II", 2, total) + struct.pack("<II", len(js), 0x4E4F534A) + js + struct.pack("<II", len(blob), 0x004E4942) + bytes(blob))
        return path, models
    doc["buffers"] = [dict(uri=name + ".bin", byteLength=len(blob))]
    with open(os.path.join(directory, name + ".bin"), "wb") as f:
        f.write(bytes(blob))
    path = os.path.join(directory, name + ".gltf")
    with open(path, "w") as f:
        json.dump(doc, f)
    return path, models


def export_world_baked_glb(sc, directory, name="baked"):
    """export with the instances' model matrices applied by the exporter (same arithmetic as hr_scene_build), so ONE instance of the
    loaded mesh with an identity model reproduces the procedural scene's primitive order and mesh ids"""
    V, I, insts, mats = synth_arrays(sc)
    done = np.zeros(len(V), bool)
    for it in insts:
        M = np.array(it.model[:], np.float32).reshape(4, 4).T
        idx = np.unique(I[it.first_index: it.first_index + it.index_count].astype(np.int64) + it.base_vertex)
        assert not done[idx].any(), "instances share vertices: the in-place bake would transform them twice"
        done[idx] = True
        p = V[idx, 0:3].copy()
        for r in range(3):
            V[idx, r] = ((M[r, 0] * p[:, 0] + M[r, 1] * p[:, 1]) + M[r, 2] * p[:, 2]) + M[r, 3]
        it.model[:] = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1]
    path, _ = export_gltf(sc, directory, name=name, glb=True, arrays=(V, I, insts, mats))
    return path


# ---------------------------------------------------------------------------------------------- images
@pytest.mark.parametrize("level", [0, 1, 9])
def test_png_rgba8_all_filters_and_deflate_block_types(tmp_path, level):
    """level 0 = stored blocks, small images = fixed Huffman, larger = dynamic Huffman; filter types 0-4 cycle over the rows"""
    rng = np.random.default_rng(level)
    for W, H in [(7, 5), (128, 128)]:
        img = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
        img[H // 2:, :, :] = (np.arange(W)[None, :, None] * 2 + np.arange(H - H // 2)[:, None, None]) & 255  # compressible part
        p = tmp_path / f"rgba_{W}_{level}.png"
        write_png(p, img, 6, 8, level=level, split_idat=3)
        got = A.image_load(p)
        assert got.shape == (H, W, 4) and np.array_equal(got, img)
        assert np.array_equal(A.image_load(p, flip_vertical=True), img[::-1])
        assert np.array_equal(A.image_load(data=open(p, "rb").read()), img)


def test_png_colour_types_bit_depths_and_stb_channel_rules(tmp_path):
    rng = np.random.default_rng(3)
    H, W = 9, 13
    # RGB -> RGBA with alpha 255 (vk.cpp:163-168)
    rgb = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    write_png(tmp_path / "rgb.png", rgb, 2, 8)
    got = A.image_load(tmp_path / "rgb.png")
    assert got.shape == (H, W, 4) and np.array_equal(got[..., :3], rgb) and np.all(got[..., 3] == 255)
    # RGB + tRNS colour key: matching pixels get alpha 0
    rgb[2, 3] = (10, 20, 30)
    write_png(tmp_path / "rgbk.png", rgb, 2, 8, trns=[0, 10, 0, 20, 0, 30])
    got = A.image_load(tmp_path / "rgbk.png")
    want_a = np.where(np.all(rgb == (10, 20, 30), axis=-1), 0, 255)
    assert np.array_equal(got[..., 3], want_a)
    # grey 8 -> 1 channel; grey + alpha -> 2 channels
    g = rng.integers(0, 256, (H, W, 1), dtype=np.uint8)
    write_png(tmp_path / "g.png", g, 0, 8)
    assert np.array_equal(A.image_load(tmp_path / "g.png"), g)
    ga = rng.integers(0, 256, (H, W, 2), dtype=np.uint8)
    write_png(tmp_path / "ga.png", ga, 4, 8)
    assert np.array_equal(A.image_load(tmp_path / "ga.png"), ga)
    # 16-bit samples keep their high byte
    r16 = rng.integers(0, 65536, (H, W, 4), dtype=np.uint16)
    write_png(tmp_path / "r16.png", r16, 6, 16)
    assert np.array_equal(A.image_load(tmp_path / "r16.png"), (r16 >> 8).astype(np.uint8))
    # low bit depths: grey values are scaled to 0..255, rows are padded to whole bytes
    for depth in (1, 2, 4):
        gl = rng.integers(0, 1 << depth, (H, W, 1), dtype=np.uint8)
        write_png(tmp_path / f"g{depth}.png", gl, 0, depth)
        assert np.array_equal(A.image_load(tmp_path / f"g{depth}.png"), gl * (255 // ((1 << depth) - 1)))
    # palette (4-bit indices) with tRNS: RGBA out
    plte = rng.integers(0, 256, (16, 3), dtype=np.uint8)
    trns = rng.integers(0, 256, 5, dtype=np.uint8)
    pi = rng.integers(0, 16, (H, W, 1), dtype=np.uint8)
    write_png(tmp_path / "pal.png", pi, 3, 4, plte=plte.reshape(-1).tolist(), trns=trns.tolist())
    got = A.image_load(tmp_path / "pal.png")
    alpha = np.concatenate([trns, np.full(11, 255, np.uint8)])
    assert np.array_equal(got[..., :3], plte[pi[..., 0]]) and np.array_equal(got[..., 3], alpha[pi[..., 0]])


def test_png_adam7_interlace(tmp_path):
    rng = np.random.default_rng(5)
    for W, H in [(1, 1), (3, 2), (9, 9), (33, 17)]:
        img = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
        write_png(tmp_path / "i.png", img, 6, 8, interlace=True)
        assert np.array_equal(A.image_load(tmp_path / "i.png"), img)
    g1 = rng.integers(0, 2, (11, 19, 1), dtype=np.uint8)
    write_png(tmp_path / "i1.png", g1, 0, 1, interlace=True)
    assert np.array_equal(A.image_load(tmp_path / "i1.png"), g1 * 255)


def test_png_writer_round_trips_and_is_a_valid_zlib_stream(tmp_path):
    """hra_image_save_png: read back by our decoder AND taken apart independently (chunk CRCs, Python's zlib on the IDAT stream)"""
    rng = np.random.default_rng(8)
    for shape in [(5, 7), (3, 4, 2), (300, 301, 3), (17, 9, 4)]:  # the RGB case spans several 65535-byte stored blocks
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        p = tmp_path / "w.png"
        A.image_save_png(p, img)
        got = A.image_load(p)
        c = 1 if img.ndim == 2 else img.shape[2]
        want = img.reshape(img.shape[0], img.shape[1], c)
        if c == 3:
            assert got.shape[2] == 4 and np.array_equal(got[..., :3], want) and np.all(got[..., 3] == 255)
        else:
            assert np.array_equal(got, want)
        data = open(p, "rb").read()
        assert data[:8] == b"\x89PNG\r\n\x1a\n"
        pos, idat = 8, b""
        while pos < len(data):
            n = struct.unpack(">I", data[pos:pos + 4])[0]
            tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
            assert struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(tag + body) & 0xFFFFFFFF
            if tag == b"IHDR":
                assert struct.unpack(">IIBBBBB", body) == (img.shape[1], img.shape[0], 8, {1: 0, 2: 4, 3: 2, 4: 6}[c], 0, 0, 0)
            if tag == b"IDAT":
                idat += body
            pos += 12 + n
        raw = zlib.decompress(idat)  # checks the stored-block framing and the adler32
        stride = img.shape[1] * c
        assert len(raw) == (stride + 1) * img.shape[0] and all(raw[(stride + 1) * y] == 0 for y in range(img.shape[0]))
        assert raw[1:stride + 1] == want[0].tobytes()
    with pytest.raises(pyhr.HrError, match="cannot write"):
        A.image_save_png(tmp_path / "no_such_dir" / "x.png", np.zeros((2, 2), np.uint8))


def test_png_errors(tmp_path):
    img = np.zeros((4, 4, 4), np.uint8)
    write_png(tmp_path / "ok.png", img, 6, 8)
    data = open(tmp_path / "ok.png", "rb").read()
    with pytest.raises(pyhr.HrError, match="not a PNG"):
        A.image_load(data=b"JFIF" + data)
    bad = bytearray(data)
    k = bad.index(b"IDAT") + 12
    bad[k] ^= 0xFF
    with pytest.raises(pyhr.HrError):
        A.image_load(data=bytes(bad[:k + 2]) + bytes(20))
    with pytest.raises(pyhr.HrError, match="cannot read"):
        A.image_load(tmp_path / "missing.png")


def test_bluenoise_directory_like_the_reference(tmp_path):
    """file names of src/blue_noise.cpp:5-19; RGB tables come back RGBA; missing higher-spp tables are reported, not invented"""
    rng = np.random.default_rng(9)
    sobol = rng.integers(0, 256, (1, 256, 4), dtype=np.uint8)
    write_png(tmp_path / "sobol_256_4d.png", sobol, 6, 8)
    tables = {}
    for s in (0, 1, 3):
        t = rng.integers(0, 256, (128, 128, 3), dtype=np.uint8)  # Heitz's files are RGB
        tables[s] = t
        write_png(tmp_path / f"scrambling_ranking_128x128_2d_{1 << s}spp.png", t, 2, 8)
    so, sr, mask = A.bluenoise_load(tmp_path)
    assert mask == 0b1011
    assert np.array_equal(so, sobol[0])
    for s, t in tables.items():
        assert np.array_equal(sr[s, ..., :3], t) and np.all(sr[s, ..., 3] == 255)
    # these arrays are what hr_bluenoise_set / hr_bluenoise_set_slot take: same shapes as the substitute tables
    so2, sr2 = pyhr.blue_noise()
    assert so.shape == so2.shape and sr[0].shape == sr2.shape and so.dtype == so2.dtype
    os.remove(tmp_path / "scrambling_ranking_128x128_2d_1spp.png")
    with pytest.raises(pyhr.HrError, match="1spp"):
        A.bluenoise_load(tmp_path)
    write_png(tmp_path / "scrambling_ranking_128x128_2d_1spp.png", tables[0][:64], 2, 8)
    with pytest.raises(pyhr.HrError, match="expected 128 x 128"):
        A.bluenoise_load(tmp_path)


def test_brdf_lut_raw_file(tmp_path):
    so = pyhr.load_synth()
    so.hrs_brdf_lut.argtypes = [C.c_int, C.c_void_p]
    lut = np.zeros((512, 512, 2), np.uint16)
    so.hrs_brdf_lut(16, lut.ctypes.data)
    lut.tofile(tmp_path / "brdf_lut.bin")
    assert np.array_equal(A.brdf_lut_load(tmp_path / "brdf_lut.bin"), lut)
    lut[:100].tofile(tmp_path / "short.bin")
    with pytest.raises(pyhr.HrError, match="expected"):
        A.brdf_lut_load(tmp_path / "short.bin")


def test_hdr_rgbe_flat_and_rle(tmp_path):
    rng = np.random.default_rng(11)
    H, W = 6, 40
    rgbe = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    rgbe[..., 3] = rng.integers(120, 136, (H, W))
    rgbe[1, 5:30, :] = rgbe[1, 5, :]  # runs
    rgbe[2, :, 3] = 0                 # zero exponent -> black
    want = np.zeros((H, W, 4), np.float32)
    scale = np.ldexp(np.float32(1.0), rgbe[..., 3].astype(np.int32) - 136).astype(np.float32)
    for c in range(3):
        want[..., c] = np.where(rgbe[..., 3] != 0, rgbe[..., c].astype(np.float32) * scale, 0.0)
    want[..., 3] = 1.0
    for rle in (False, True):
        write_hdr(tmp_path / "e.hdr", rgbe, rle)
        got = A.image_loadf(tmp_path / "e.hdr")
        assert got.shape == (H, W, 4) and np.array_equal(got, want)
        assert np.array_equal(A.image_loadf(tmp_path / "e.hdr", flip_vertical=True), want[::-1])
    # constant environment colour: a uniform map returns its colour whatever the row weights
    uni = np.zeros((8, 16, 4), np.uint8)
    uni[...] = (64, 128, 32, 129)  # (0.25, 0.5, 0.125) * 2^(129-136+8)... mantissa / 256 * 2^(e-128)
    write_hdr(tmp_path / "u.hdr", uni, True)
    c = A.environment_constant(tmp_path / "u.hdr")
    assert np.allclose(c, (64 / 128.0, 128 / 128.0, 32 / 128.0), rtol=1e-6)


# ---------------------------------------------------------------------------------------------- meshes
OBJ_TEXT = """# two groups, two materials, a quad, negative indices, a face without normals
mtllib cube.mtl
o first
v 0 0 0
v 1 0 0
v 1 1 0
v 0 1 0
vt 0 0
vt 1 0
vt 1 1
vt 0 1
vn 0 0 1
usemtl red
f 1/1/1 2/2/1 3/3/1 4/4/1
g second
v 0 0 1
v 1 0 1
v 0 1 1
usemtl shiny
f -3 -2 -1
usemtl red
f 5 7 6
"""
MTL_TEXT = """newmtl red
Kd 0.8 0.1 0.2
Ke 5 5 5
d 0.5
map_Kd textures\\red albedo.png
map_Bump bump.png
newmtl shiny
Kd 0.25 0.5 0.75
Pr 0.125
Pm 1
"""


def test_obj_mtl_loader(tmp_path):
    (tmp_path / "cube.obj").write_text(OBJ_TEXT)
    (tmp_path / "cube.mtl").write_text(MTL_TEXT)
    m = A.Mesh(tmp_path / "cube.obj")
    sub = m.submeshes()
    # sub-meshes: (first, red) quad -> 2 triangles; (second, shiny) 1 triangle; (second, red) 1 triangle
    assert [s["index_count"] for s in sub] == [6, 3, 3]
    assert [s["base_index"] for s in sub] == [0, 6, 9]
    assert [s["vertex_count"] for s in sub] == [4, 3, 3]
    assert [s["mat_idx"] for s in sub] == [0, 1, 0]  # materials in first-use order, re-used by later sub-meshes (mesh.cpp:511-513)
    assert m.n_materials == 2
    mats = m.materials()
    assert np.allclose(mats[0]["albedo"], (0.8, 0.1, 0.2, 0.5)) and mats[0]["roughness"] == 1.0 and mats[0]["metallic"] == 0.0
    assert mats[0]["emissive"][:3] == (0.0, 0.0, 0.0)  # the reference never reads the constant (mesh.cpp:455)
    assert np.allclose(mats[1]["albedo"][:3], (0.25, 0.5, 0.75)) and mats[1]["roughness"] == 0.125 and mats[1]["metallic"] == 1.0
    assert m.texture(0, A.TEX_ALBEDO) == str(tmp_path / "textures/red albedo.png")  # '\\' -> '/', spaces kept (mesh.cpp:352)
    assert m.texture(0, A.TEX_NORMAL) == str(tmp_path / "bump.png") and m.texture(1, A.TEX_ALBEDO) == ""
    V, I = m.vertices(), m.indices()
    assert V.shape == (10, 20)
    # triangulation: fan over the quad, base vertex folded into the indices
    assert I.tolist() == [0, 1, 2, 0, 2, 3, 4, 5, 6, 7, 8, 9]
    assert np.array_equal(V[:4, 0:3], [[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]])
    assert np.array_equal(V[:4, 3], [0, 0, 0, 0]) and np.array_equal(V[4:7, 3], [1, 1, 1])  # position.w = material index
    assert np.array_equal(V[:4, 4:6], [[0, 1], [1, 1], [1, 0], [0, 0]])  # aiProcess_FlipUVs
    assert np.array_equal(V[:4, 8:11], [[0, 0, 1]] * 4)
    # tangent frame from the (flipped) UVs: orthonormal, right-handed with the normal
    t, b, n = V[:4, 12:15], V[:4, 16:19], V[:4, 8:11]
    assert np.allclose(np.abs(t), [[1, 0, 0]] * 4) and np.allclose(np.abs(b), [[0, 1, 0]] * 4)
    assert np.all(np.einsum("ij,ij->i", np.cross(n, t), b) > 0)
    # generated normals for the faces without vn: (0,0,1) for 5-6-7 (ccw seen from +z) and the opposite winding's (0,0,-1)
    assert np.allclose(V[4:7, 8:11], [[0, 0, 1]] * 3) and np.allclose(V[7:10, 8:11], [[0, 0, -1]] * 3)
    mn, mx = m.extents()
    assert np.array_equal(mn, [0, 0, 0]) and np.array_equal(mx, [1, 1, 1])
    assert sub[1]["min_extents"] == (0.0, 0.0, 1.0) and sub[1]["max_extents"] == (1.0, 1.0, 1.0)


def _tiny_gltf(tmp_path, embed):
    """one mesh, two primitives: (a) float positions + normals + tangents + ushort indices in an interleaved (strided) view,
    (b) positions only, normalised ubyte UVs, no indices, no material"""
    blob = bytearray()
    # primitive a: interleaved position (12) normal (12) tangent (16) = stride 40, 4 vertices
    pa = np.array([[0, 0, 0], [2, 0, 0], [2, 2, 0], [0, 2, 0]], "<f4")
    na = np.array([[0, 0, 1]] * 4, "<f4")
    ta = np.array([[1, 0, 0, -1]] * 4, "<f4")
    for k in range(4):
        blob += pa[k].tobytes() + na[k].tobytes() + ta[k].tobytes()
    ia_off = len(blob)
    blob += np.array([0, 1, 2, 0, 2, 3], "<u2").tobytes()
    pb_off = len(blob)
    pb = np.array([[0, 0, 5], [1, 0, 5], [0, 1, 5]], "<f4")
    blob += pb.tobytes()
    uv_off = len(blob)
    blob += bytes([0, 0, 255, 0, 0, 255]) + bytes(2)
    views = [dict(buffer=0, byteOffset=0, byteLength=160, byteStride=40), dict(buffer=0, byteOffset=ia_off, byteLength=12),
             dict(buffer=0, byteOffset=pb_off, byteLength=36), dict(buffer=0, byteOffset=uv_off, byteLength=6)]
    acc = [dict(bufferView=0, byteOffset=0, componentType=5126, count=4, type="VEC3"), dict(bufferView=0, byteOffset=12, componentType=5126, count=4, type="VEC3"),
           dict(bufferView=0, byteOffset=24, componentType=5126, count=4, type="VEC4"), dict(bufferView=1, componentType=5123, count=6, type="SCALAR"),
           dict(bufferView=2, componentType=5126, count=3, type="VEC3"), dict(bufferView=3, componentType=5121, normalized=True, count=3, type="VEC2")]
    doc = dict(asset=dict(version="2.0"), buffers=[dict(byteLength=len(blob))], bufferViews=views, accessors=acc,
               images=[dict(uri="tex/base%20color.png")], textures=[dict(source=0)],
               materials=[dict(name="unused"), dict(name="gold", pbrMetallicRoughness=dict(baseColorFactor=[1.0, 0.75, 0.25, 1.0], roughnessFactor=0.5,
                                                                                            baseColorTexture=dict(index=0)), emissiveFactor=[9, 9, 9])],
               meshes=[dict(primitives=[dict(attributes=dict(POSITION=0, NORMAL=1, TANGENT=2), indices=3, material=1),
                                        dict(attributes=dict(POSITION=4, TEXCOORD_0=5))])],
               nodes=[dict(mesh=0, translation=[100, 0, 0])], scenes=[dict(nodes=[0])], scene=0)
    if embed:
        doc["buffers"][0]["uri"] = "data:application/octet-stream;base64," + base64.b64encode(bytes(blob)).decode()
    else:
        doc["buffers"][0]["uri"] = "tiny.bin"
        (tmp_path / "tiny.bin").write_bytes(bytes(blob))
    p = tmp_path / ("tiny_embed.gltf" if embed else "tiny.gltf")
    p.write_text(json.dumps(doc, indent=1).replace("gold", "g\\u006fld"))
    return p


@pytest.mark.parametrize("embed", [False, True])
def test_gltf_loader(tmp_path, embed):
    m = A.Mesh(_tiny_gltf(tmp_path, embed))
    sub = m.submeshes()
    assert [s["index_count"] for s in sub] == [6, 3] and [s["vertex_count"] for s in sub] == [4, 3]
    assert [s["mat_idx"] for s in sub] == [0, 1]  # first-use order: "gold" is local material 0, the importer's default material 1
    mats = m.materials()
    assert np.allclose(mats[0]["albedo"], (1.0, 0.75, 0.25, 1.0)) and mats[0]["roughness"] == 0.5 and mats[0]["metallic"] == 1.0  # metallicFactor defaults to 1
    assert mats[0]["emissive"][:3] == (0.0, 0.0, 0.0)
    assert np.allclose(mats[1]["albedo"], (1, 1, 1, 1)) and mats[1]["roughness"] == 1.0
    assert m.texture(0, A.TEX_ALBEDO).endswith("tex/base%20color.png")
    V, I = m.vertices(), m.indices()
    assert I.tolist() == [0, 1, 2, 0, 2, 3, 4, 5, 6]
    assert np.array_equal(V[:4, 0:3], [[0, 0, 0], [2, 0, 0], [2, 2, 0], [0, 2, 0]])  # node translation NOT applied (mesh.cpp:283-291)
    assert np.array_equal(V[:4, 8:11], [[0, 0, 1]] * 4)
    # bitangent = cross(n, t) * w = (0,1,0) * -1; then the reference flips the TANGENT when the frame is left-handed (mesh.cpp:553-556)
    assert np.array_equal(V[:4, 16:19], [[0, -1, 0]] * 4) and np.array_equal(V[:4, 12:15], [[-1, 0, 0]] * 4)
    assert np.array_equal(V[4:7, 0:3], [[0, 0, 5], [1, 0, 5], [0, 1, 5]])
    assert np.allclose(V[4:7, 4:6], [[0, 0], [1, 0], [0, 1]])  # importer flip + aiProcess_FlipUVs cancel
    assert np.allclose(V[4:7, 8:11], [[0, 0, 1]] * 3)          # generated
    assert np.array_equal(V[4:7, 3], [1, 1, 1])


def test_gltf_errors(tmp_path):
    (tmp_path / "bad.gltf").write_text('{"asset": {"version": "2.0"}, "meshes": [')
    with pytest.raises(pyhr.HrError, match="JSON syntax"):
        A.Mesh(tmp_path / "bad.gltf")
    (tmp_path / "nobuf.gltf").write_text(json.dumps(dict(asset=dict(version="2.0"), buffers=[dict(uri="gone.bin", byteLength=36)],
                                                         bufferViews=[dict(buffer=0, byteLength=36)], accessors=[dict(bufferView=0, componentType=5126, count=3, type="VEC3")],
                                                         meshes=[dict(primitives=[dict(attributes=dict(POSITION=0))])])))
    with pytest.raises(pyhr.HrError, match="gone.bin"):
        A.Mesh(tmp_path / "nobuf.gltf")
    (tmp_path / "gone.bin").write_bytes(bytes(20))
    with pytest.raises(pyhr.HrError, match="past the end"):
        A.Mesh(tmp_path / "nobuf.gltf")
    with pytest.raises(pyhr.HrError, match="unsupported mesh format"):
        A.Mesh(tmp_path / "scene.fbx")


# ---------------------------------------------------------------------------------------------- scenes
def test_scene_tables_like_ray_traced_scene(tmp_path):
    (tmp_path / "cube.obj").write_text(OBJ_TEXT)
    (tmp_path / "cube.mtl").write_text(MTL_TEXT)
    a = A.Mesh(tmp_path / "cube.obj")
    b = A.Mesh(_tiny_gltf(tmp_path, True))
    ident = np.eye(4, dtype=np.float32)
    shift = np.eye(4, dtype=np.float32)
    shift[:3, 3] = (10, 20, 30)
    sc = A.AssetScene([(a, ident.T.reshape(-1)), (b, ident.T.reshape(-1)), (a, shift.T.reshape(-1))])
    # meshes are stored once (ray_traced_scene.cpp:283-297); one draw per (instance, sub-mesh) in order = mesh id (g_buffer.cpp:141-175)
    assert sc.n_vertices == a.n_vertices + b.n_vertices and sc.n_indices == a.n_indices + b.n_indices and sc.n_materials == 4
    inst = sc.instances()
    assert len(inst) == 3 + 2 + 3
    assert [i["first_index"] for i in inst] == [0, 6, 9, 12, 18, 0, 6, 9]
    assert [i["base_vertex"] for i in inst] == [0, 0, 0, 10, 10, 0, 0, 0]
    assert [i["material_idx"] for i in inst] == [0, 1, 0, 2, 3, 0, 1, 0]
    assert inst[5]["model"][12:15] == (10.0, 20.0, 30.0)
    tri, pid = sc.world_triangles()
    assert tri.shape == (4 + 3 + 4, 9) and pid.tolist() == [0, 0, 1, 2, 3, 3, 4, 5, 5, 6, 7]
    assert np.array_equal(tri[7].reshape(3, 3), tri[0].reshape(3, 3) + (10, 20, 30))


def test_scene_material_textures(tmp_path):
    """hra_scene_finalize decodes every image the materials reference once and produces hr_scene_set_textures' arguments: albedo sRGB, glTF's
    packed roughness (.g) / metallic (.b) image, OBJ maps on channel 0; files that cannot be decoded fall back to the constant with a warning"""
    rng = np.random.default_rng(12)
    (tmp_path / "textures").mkdir()
    red = rng.integers(0, 256, (4, 6, 3), dtype=np.uint8)
    write_png(tmp_path / "textures" / "red albedo.png", red, 2, 8)
    (tmp_path / "cube.obj").write_text(OBJ_TEXT)
    (tmp_path / "cube.mtl").write_text(MTL_TEXT + "map_Ns rough.png\nmap_Ka rough.png\nmap_Kd photo.jpg\n")
    rough = rng.integers(0, 256, (8, 8, 1), dtype=np.uint8)
    write_png(tmp_path / "rough.png", rough, 0, 8)
    gl = _tiny_gltf(tmp_path, True)  # "gold" references tex/base%20color.png (missing)
    a, b = A.Mesh(tmp_path / "cube.obj"), A.Mesh(gl)
    ident = np.eye(4, dtype=np.float32).reshape(-1)
    sc = A.AssetScene([(a, ident), (b, ident), (a, ident)])
    textures, bindings, warnings = sc.textures()
    assert len(bindings) == sc.n_materials == 4
    # "red": albedo = the RGB file as RGBA, sRGB; bump.png (normal map) is missing -> -1 + warning
    assert bindings[0]["albedo"] == 0 and textures[0][1] is True and np.array_equal(textures[0][0][..., :3], red) and np.all(textures[0][0][..., 3] == 255)
    assert bindings[0]["normal"] == -1 and "bump.png" in warnings
    # "shiny": roughness and metallic share one decoded grey image (channel 0 for OBJ), linear; its map_Kd is a JPEG -> constant + warning
    assert bindings[1]["roughness"] == bindings[1]["metallic"] == 1 and bindings[1]["roughness_channel"] == bindings[1]["metallic_channel"] == 0
    assert textures[1][1] is False and np.array_equal(textures[1][0], rough[..., 0]) and bindings[1]["albedo"] == -1 and "photo.jpg: not a PNG" in warnings
    # glTF materials: channels 1 / 2; the missing base colour image falls back to the constant
    assert bindings[2]["albedo"] == -1 and "base%20color.png" in warnings and bindings[2]["roughness_channel"] == 1 and bindings[2]["metallic_channel"] == 2
    assert bindings[3] == dict(albedo=-1, normal=-1, roughness=-1, roughness_channel=1, metallic=-1, metallic_channel=2, emissive=-1)
    assert len(textures) == 2  # every image decoded once although the mesh is instanced twice


@pytest.mark.parametrize("fmt", ["obj", "gltf", "glb"])
def test_procedural_scene_round_trip_is_bit_exact(tmp_path, fmt):
    """export the shadows-test scene, read it back through the loaders and the scene tables: the world-space triangle soup that
    hr_scene_build would see equals the synthetic scene's bit for bit (so every parity result carries over to loaded assets)"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    path, models = export_obj(sc, tmp_path) if fmt == "obj" else export_gltf(sc, tmp_path, glb=(fmt == "glb"))
    mesh = A.Mesh(path)
    assert mesh.n_submeshes == sc.n_instances
    tri_ref, inst_ref = sc.world_triangles()
    # the export wrote one sub-mesh per synthetic instance; instance k of the asset scene draws the whole mesh with model k, so
    # keep the triangles of sub-mesh k of instance k
    asc = A.AssetScene([(mesh, models[k]) for k in range(sc.n_instances)])
    tri, pid = asc.world_triangles()
    n_sub = mesh.n_submeshes
    keep = (pid // n_sub) == (pid % n_sub)
    assert np.array_equal(tri[keep].view(np.uint32), tri_ref.view(np.uint32))
    # materials: constants survive the trip (the per-mesh material table is in first-use order)
    _, _, insts, mats = synth_arrays(sc)
    lm = mesh.materials()
    for k, s in enumerate(mesh.submeshes()):
        src = mats[insts[k].material_idx]
        assert np.allclose(lm[s["mat_idx"]]["albedo"][:3], src.albedo[:3], rtol=0, atol=0)
        assert lm[s["mat_idx"]]["roughness"] == src.roughness and lm[s["mat_idx"]]["metallic"] == src.metallic


def test_world_baked_export_reproduces_primitive_order_and_mesh_ids(tmp_path):
    """the fixture of tests/widened/test_gpu_scene_assets.py: one identity instance of the loaded file = the procedural scene"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    mesh = A.Mesh(export_world_baked_glb(sc, tmp_path))
    asc = A.AssetScene([(mesh, np.eye(4, dtype=np.float32).reshape(-1))])
    tri_ref, inst_ref = sc.world_triangles()
    tri, inst = asc.world_triangles()
    assert np.array_equal(tri.view(np.uint32), tri_ref.view(np.uint32)) and np.array_equal(inst, inst_ref)


def test_loaders_reject_corrupted_files_without_crashing(tmp_path):
    """robustness of the parsers: random byte flips, truncations and splices of valid PNG / HDR / OBJ / glTF / GLB files either load
    or fail with an error message (the same campaign ran 2 500 cases under AddressSanitizer + UBSan clean while this was written)"""
    import random
    rnd = random.Random(20260923)
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (9, 13, 4), dtype=np.uint8)
    write_png(tmp_path / "a.png", img, 6, 8)
    write_png(tmp_path / "b.png", img[..., :1] % 16, 3, 4, plte=list(range(48)), trns=[1, 2, 3])
    write_png(tmp_path / "c.png", img, 6, 8, interlace=True)
    rgbe = rng.integers(0, 256, (6, 40, 4), dtype=np.uint8)
    write_hdr(tmp_path / "e.hdr", rgbe, True)
    (tmp_path / "cube.obj").write_text(OBJ_TEXT)
    (tmp_path / "cube.mtl").write_text(MTL_TEXT)
    seeds = [tmp_path / "a.png", tmp_path / "b.png", tmp_path / "c.png", tmp_path / "e.hdr", tmp_path / "cube.obj", _tiny_gltf(tmp_path, True), _tiny_gltf(tmp_path, False),
             export_gltf(pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST), tmp_path, glb=True)[0]]
    loaded = failed = 0
    for _ in range(240):
        src = rnd.choice(seeds)
        data = bytearray(open(src, "rb").read())
        mode = rnd.random()
        if mode < 0.6:
            for _ in range(rnd.choice([1, 1, 2, 4, 16])):
                data[rnd.randrange(len(data))] = rnd.randrange(256)
        elif mode < 0.8:
            data = data[:rnd.randrange(1, len(data))]
        else:
            i = rnd.randrange(len(data))
            data[i:i + rnd.randrange(1, 8)] = bytes(rnd.randrange(256) for _ in range(rnd.randrange(0, 12)))
        out = tmp_path / ("fz" + os.path.splitext(str(src))[1])
        out.write_bytes(bytes(data))
        try:
            if out.suffix == ".png":
                A.image_load(out)
            elif out.suffix == ".hdr":
                A.image_loadf(out)
            else:
                A.Mesh(out)
            loaded += 1
        except pyhr.HrError as e:
            assert str(e)
            failed += 1
    assert loaded + failed == 240 and failed > 40
    # a header that claims a huge image over a tiny data stream is refused before anything of that size is allocated
    big = bytearray(open(tmp_path / "a.png", "rb").read())
    big[16:24] = struct.pack(">II", 16000, 16000)
    with pytest.raises(pyhr.HrError, match="too short"):
        A.image_load(data=bytes(big))


def test_png_encode_decode_property(tmp_path):
    """hypothesis: any 8-bit image of 1-4 channels survives hra_image_save_png -> hra_image_load (RGB comes back with alpha 255), and
    any image written by the independent test encoder with any filter cycle / deflate level / interlacing decodes to itself"""
    from hypothesis import given, settings, strategies as st
    from hypothesis.extra import numpy as hnp

    @settings(max_examples=40, deadline=None)
    @given(hnp.arrays(np.uint8, st.tuples(st.integers(1, 24), st.integers(1, 24), st.integers(1, 4))))
    def ours(img):
        p = tmp_path / "h.png"
        A.image_save_png(p, img)
        got = A.image_load(p)
        if img.shape[2] == 3:
            assert np.array_equal(got[..., :3], img) and np.all(got[..., 3] == 255)
        else:
            assert np.array_equal(got, img)

    @settings(max_examples=40, deadline=None)
    @given(hnp.arrays(np.uint8, st.tuples(st.integers(1, 20), st.integers(1, 20), st.just(4))), st.lists(st.integers(0, 4), min_size=1, max_size=5), st.integers(0, 9),
           st.booleans(), st.integers(1, 4))
    def theirs(img, cycle, level, interlace, split):
        p = tmp_path / "t.png"
        write_png(p, img, 6, 8, cycle=tuple(cycle), interlace=interlace, level=level, split_idat=split)
        assert np.array_equal(A.image_load(p), img)

    ours()
    theirs()


@pytest.mark.parametrize("fmt", ["obj", "gltf", "glb"])
def test_scene_material_indices_are_in_range(tmp_path, fmt):
    """hr_scene_build refuses an instance whose material_idx is not below n_materials: neither the scene tables of loaded meshes (each
    mesh's sub-mesh indices offset by its first material, meshes instanced more than once) nor the synthetic scenes produce one"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    path, models = export_obj(sc, tmp_path) if fmt == "obj" else export_gltf(sc, tmp_path, glb=(fmt == "glb"))
    (tmp_path / "cube.obj").write_text(OBJ_TEXT)
    (tmp_path / "cube.mtl").write_text(MTL_TEXT)
    mesh, cube = A.Mesh(path), A.Mesh(tmp_path / "cube.obj")
    ident = np.eye(4, dtype=np.float32).reshape(-1)
    asc = A.AssetScene([(cube, ident), (mesh, models[0]), (cube, ident), (mesh, models[1])])
    idx = [i["material_idx"] for i in asc.instances()]
    assert asc.n_materials == cube.n_materials + mesh.n_materials and max(idx) == asc.n_materials - 1 and min(idx) == 0
    for kind in (pyhr.SCENE_SHADOWS_TEST, pyhr.SCENE_ARCADE):
        s = pyhr.SynthScene(kind, 2000)
        _, _, insts, mats = synth_arrays(s)
        assert max(it.material_idx for it in insts) < len(mats)
