"""CPU tests of the drop-in boundary: the shared library loads, exports every symbol include/hr_api.h declares, and fails
loudly (no CPU fallback) when there is no GPU.  No compute calls are made here."""
import ctypes as C
import os
import re

import pytest

import pyhr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HR_ERR_INVALID_ARG = -1


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "hr_api.h")).read()
    return sorted(set(re.findall(r"HR_API\s+[\w\s\*]+?\b(hr_\w+)\s*\(", src)))


def test_header_and_binding_agree():
    assert declared_symbols() == sorted(pyhr.ABI_SYMBOLS)


def test_library_exports_every_declared_symbol():
    lib = pyhr.load_product()
    for name in declared_symbols():
        assert hasattr(lib, name), f"{name} is declared in hr_api.h but not exported"


def test_asset_library_exports_every_declared_symbol():
    """include/hr_assets.h is the boundary of libhr_assets.so (dw::Mesh::load / Image::create_from_file / BlueNoise / RayTracedScene tables)"""
    from pyhr import assets
    src = open(os.path.join(ROOT, "include", "hr_assets.h")).read()
    names = sorted(set(re.findall(r"HR_API\s+[\w\s\*]+?\b(hra_\w+)\s*\(", src)))
    assert len(names) >= 25, names
    lib = assets.load_assets()
    for name in names:
        assert hasattr(lib, name), f"{name} is declared in hr_assets.h but not exported"
    assert C.sizeof(assets.hra_submesh) == 5 * 4 + 6 * 4


def test_struct_layouts_match_the_reference():
    assert C.sizeof(pyhr.hr_ubo) == 416          # struct UBO, src/common.h:161-179 (5 mat4 + 2 vec4 + Light)
    assert C.sizeof(pyhr.hr_light) == 64         # src/common.h:106-111
    assert C.sizeof(pyhr.hr_vertex) == 80        # dw::Vertex, mesh.h:16-23
    assert C.sizeof(pyhr.hr_instance) == 80
    assert C.sizeof(pyhr.hr_material) == 48


def test_version_and_defaults_without_gpu():
    lib = pyhr.load_product()
    assert lib.hr_version() == 100
    p = pyhr.hr_shadows_params()
    lib.hr_shadows_default_params(C.byref(p))     # src/ray_traced_shadows.h:50-115
    assert (p.bias, p.radius, p.filter_iterations, p.feedback_iteration, p.denoise) == (0.5, 1, 4, 1, 1)
    assert abs(p.alpha - 0.01) < 1e-9 and abs(p.moments_alpha - 0.2) < 1e-7 and p.phi_visibility == 10.0 and p.phi_normal == 32.0
    a = pyhr.hr_ao_params()
    lib.hr_ao_default_params(C.byref(a))          # src/ray_traced_ao.h:51-110
    assert (a.ray_length, a.blur_radius, a.denoise) == (7.0, 4, 1) and abs(a.bias - 0.3) < 1e-7 and abs(a.power - 1.2) < 1e-7
    assert p.spp == 1 and a.spp == 1             # one ray per pixel like the reference; > 1 is the SURVEY.md §8d extension


def test_shard_rows_partition():
    lib = pyhr.load_product()
    for H in (2160, 1080, 540, 270, 144, 36):
        for world in (1, 2, 4, 8):
            rows = []
            for r in range(world):
                b, e = C.c_int(), C.c_int()
                assert lib.hr_shard_rows(H, r, world, C.byref(b), C.byref(e)) == 0
                assert (b.value % 8 == 0 or b.value == H) and (e.value % 8 == 0 or e.value == H)
                rows.append((b.value, e.value))
            assert rows[0][0] == 0 and rows[-1][1] == H
            assert all(rows[i][1] == rows[i + 1][0] for i in range(world - 1))
            sizes = [e - b for b, e in rows]
            assert max(sizes) - min(sizes) <= 8 + (-H) % 8  # bands differ by at most one 8-row tile (+ a partial last tile)


def test_debug_set_rejects_undefined_keys_and_values():
    """hr_debug_set touches no device: removed keys and values a key does not define are refused, every defined value is taken"""
    lib = pyhr.load_product()
    try:
        for key in (0, 2, 4, 5, 7, 8, 9, 10, 11, 12, 13):
            assert lib.hr_debug_set(key, 0) == HR_ERR_INVALID_ARG and lib.hr_debug_set(key, 1) == HR_ERR_INVALID_ARG, key
        for key, value in ((6, 1), (6, 4), (1, 2), (3, 2), (1, -1), (3, -1), (6, -1), (1, 4), (6, 5)):
            assert lib.hr_debug_set(key, value) == HR_ERR_INVALID_ARG, (key, value)
        for key, values in ((1, (0, 1, 3)), (3, (0, 1)), (6, (0, 2, 3))):
            for value in values:
                assert lib.hr_debug_set(key, value) == 0, (key, value)
    finally:
        for key, default in ((1, 3), (3, 1), (6, 3)):
            assert lib.hr_debug_set(key, default) == 0


def test_init_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(pyhr.HrError, match="no CUDA device"):
        pyhr.Context(0)
