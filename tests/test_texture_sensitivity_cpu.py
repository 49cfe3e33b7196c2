"""Would the textured-kernel tests notice a wrong sampler?  For every case of texture_cases.py, wrong twins of the oracle's inputs stand
for the mistakes a kernel could make, and each twin must move an output tests/test_gpu_textured_kernels.py compares by far more than
its bar.  That output is the G-buffer, compared bit for bit: a twin must change at least 10 hit pixels of its material images
(albedo / metallic, roughness) or of the encoded normal.
  * texels rolled by one texel (np.roll): the wrong texel;
  * the channels of every multi-channel image permuted: the wrong channel;
  * every sRGB flag flipped: the wrong decode;
  * the u and v columns of the texture coordinates swapped;
  * the tangent passed as the bitangent at the G-buffer's call site (fetch_normal's hit_shader flipped), on the case with normal maps.
The first four twins are also held to the reflections ray trace (K12, spp 1, no DDGI terms), whose colours the GPU test compares with
`close(1e-3, 0.02)`: on the right G-buffer, the twin's hit shading must move the colours by 10x that bar (RMSE >= 1e-2 or a pixel
>= 0.2).  The opposite flip at the hit shaders' call site (the real bitangent where they pass the tangent) cannot be built from the
oracle's inputs; a kernel making it fails the GPU test's K12 comparison.  Clamp-for-repeat and nearest-for-bilinear mistakes also fail
the GPU tests and the host-build comparison of test_textures_cpu.py."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
import pyhr
import texture_cases as TC

W, H = 96, 56
MIN_PIXELS = 10
TEXTURED = [c for c in TC.CASES if c != "untextured"]


def gbuffer(case, textures, bindings, vuv, vtb):
    ss = O.ShadingScene(case.sc, brute=True)
    ss.set_textures(textures, bindings, vuv, vtb)
    f = pyhr.make_frame((0.0, 14.0, 34.0), (0.0, 3.0, 0.0), W, H, num_frames=0)
    return O.gbuffer_render(ss, f, W, H)


def differing_pixels(a, b):
    hit = a.depth != 1.0
    d = np.any(a.gb1 != b.gb1, -1) | (a.gb3[..., 0] != b.gb3[..., 0]) | np.any(a.gb2[..., :2] != b.gb2[..., :2], -1)
    return int(np.count_nonzero(d & hit))


def twins(case):
    vuv, vtb = case.vuv(), case.vtb()
    tx, b = case.textures, case.bindings
    yield "texels rolled", [(np.roll(a, 1, axis=1), s) for a, s in tx], b, vuv, vtb
    yield "channels permuted", [(np.roll(a, 1, axis=2) if a.ndim == 3 else a, s) for a, s in tx], b, vuv, vtb
    yield "sRGB flipped", [(a, not s) for a, s in tx], b, vuv, vtb
    yield "u and v swapped", tx, b, np.ascontiguousarray(vuv[:, [1, 0, 3, 2, 5, 4]]), vtb
    if any("normal" in x for x in b):
        bent = vtb.copy()
        bent[:, 9:18] = vtb[:, 0:9]
        yield "tangent as bitangent", tx, b, vuv, bent


@pytest.mark.parametrize("case", TEXTURED)
def test_each_wrong_twin_moves_the_gbuffer(case):
    c = TC.build(case)
    right = gbuffer(c, c.textures, c.bindings, c.vuv(), c.vtb())
    for name, tx, b, vuv, vtb in twins(c):
        n = differing_pixels(right, gbuffer(c, tx, b, vuv, vtb))
        assert n >= MIN_PIXELS, f"{case}: {name} changes only {n} G-buffer pixels"


def k12_colours(case, textures, bindings, vuv, vtb, g, f, bn):
    ss = O.ShadingScene(case.sc, brute=True)
    ss.set_textures(textures, bindings, vuv, vtb)
    P = pyhr.hr_reflections_params()
    pyhr.load_product().hr_reflections_default_params(C.byref(P))
    P.sky_color[0], P.sky_color[1], P.sky_color[2] = 0.3, 0.4, 0.6
    P.denoise = 0
    orf = O.ReflectionsOracle(W, H, 0, P)
    orf.render(ss, O.GBufMips(g), O.zero_gbuf_mips(W, H), f, bn, None)
    return O.h2f(orf.rt)[..., :3]


@pytest.mark.parametrize("case", TEXTURED)
def test_each_wrong_twin_moves_the_reflections(case):
    c = TC.build(case)
    f = pyhr.make_frame((0.0, 14.0, 34.0), (0.0, 3.0, 0.0), W, H, num_frames=0)
    g = gbuffer(c, c.textures, c.bindings, c.vuv(), c.vtb())
    bn = pyhr.blue_noise()
    right = k12_colours(c, c.textures, c.bindings, c.vuv(), c.vtb(), g, f, bn)
    for name, tx, b, vuv, vtb in twins(c):
        if name == "tangent as bitangent":
            continue
        d = np.abs(k12_colours(c, tx, b, vuv, vtb, g, f, bn) - right) / np.maximum(1.0, np.abs(right))
        e = float(np.sqrt(np.mean(d.astype(np.float64) ** 2)))
        assert e >= 1e-2 or d.max() >= 0.2, f"{case}: {name} moves the K12 colours by rmse {e:.1e}, max {d.max():.1e}"
