"""ctypes binding of the converged references' CPU restatement (oracle/orc_reference.cpp).  TEST INFRASTRUCTURE ONLY.

The accumulators follow the device's (hr_reference_render): shadows / AO add unoccluded rays to a uint32 image, reflections add
float64 (sum r, g, b, sum of squares r, g, b) per pixel.  mean_and_stderr turns them into the untransformed MEAN and STDERR.
"""
import ctypes as C

import numpy as np

import oracle as O

_bound = False


def _lib():
    global _bound
    L = O.lib()
    if not _bound:
        P, I, F, U = C.c_void_p, C.c_int, C.c_float, C.c_uint32
        L.orc_reference_mask.argtypes = [P, P, P, I, F, F, U, I, I, I, P]
        L.orc_reference_reflections.argtypes = [P, P, P, F, F, I, I, F, F, P, P, P, P, P, F, U, I, I, I, P]
        _bound = True
    return L


def reference_mask(scene: "O.Scene", g: "O.GBufMips", frame, kind, p0, p1, k0, n, count, row0=0, row1=None):
    """count += unoccluded rays of samples k0 .. k0 + n - 1 of K1 (kind "shadows": p0 = bias) or K7 (kind "ao": p0 = ray length,
    p1 = bias) on rows [row0, row1) of mip 0 of g"""
    assert count.dtype == np.uint32 and count.flags.c_contiguous
    gc = g.c(0)
    _lib().orc_reference_mask(scene.h, C.byref(gc), C.byref(frame), 1 if kind == "ao" else 0, p0, p1, k0, n, row0, g.size(0)[1] if row1 is None else row1,
                              O.p(count))
    return count


def reference_reflections(ss: "O.ShadingScene", g: "O.GBufMips", frame, prm, k0, n, acc, sample_gi=0, approx=0, ddgi=None, brdf_lut=None, row0=0, row1=None):
    """acc += K12's clamped samples k0 .. k0 + n - 1 (prm: pyhr.hr_reflections_params; ddgi: an O.DDGIOracle that rendered this frame)"""
    assert acc.dtype == np.float64 and acc.flags.c_contiguous
    gc = g.c(0)
    sky = np.array(prm.sky_color[:], np.float32)
    _lib().orc_reference_reflections(ss.h, C.byref(gc), C.byref(frame), prm.bias, prm.trim, sample_gi, approx, prm.gi_intensity, prm.rough_ddgi_intensity, O.p(sky),
                                     C.byref(ddgi.u) if ddgi is not None else None, O.p(ddgi.cur_irr) if ddgi is not None else None,
                                     O.p(ddgi.cur_dep) if ddgi is not None else None, O.p(brdf_lut) if brdf_lut is not None else None,
                                     prm.ibl_indirect_specular_intensity, k0, n, row0, g.size(0)[1] if row1 is None else row1, O.p(acc))
    return acc


def mean_and_stderr(acc_or_count, N):
    """(mean, stderr) in float64: a count image (Bernoulli samples) or a (H, W, 6) reflections accumulator; stderr = sqrt(s^2 / N) with the
    unbiased sample variance, 0 for N = 1"""
    a = np.asarray(acc_or_count, np.float64)
    s, q = (a, a) if a.ndim == 2 else (a[..., :3], a[..., 3:])
    m = s / N
    if N < 2:
        return m, np.zeros_like(m)
    var = np.maximum(0.0, (q - s * m) / (N - 1))
    return m, np.sqrt(var / N)


def unpack_mask(words, W, H):
    """K1 / K7 mask words (ceil(H / 4), ceil(W / 8)) -> (H, W) bits: bit (y % 4) * 8 + x % 8 of word (y / 4, x / 8)"""
    words = np.asarray(words, np.uint32)
    y, x = np.mgrid[0:H, 0:W]
    return (words[y // 4, x // 8] >> ((y % 4) * 8 + x % 8).astype(np.uint32)) & 1


def blue_noise_mean(scene: "O.Scene", g: "O.GBufMips", frames, kind, p0, p1, bn):
    """the mean over `frames` (hr_frame list, one per blue-noise sample index) of the oracle's K1 / K7 mask bits"""
    W, H = g.size(0)
    gc = g.c(0)
    acc = np.zeros((H, W), np.float64)
    mask = np.zeros(((H + 3) // 4, (W + 7) // 8), np.uint32)
    L = O.lib()
    for f in frames:
        if kind == "ao":
            L.orc_ao_ray_trace(scene.h, C.byref(gc), C.byref(f), p0, p1, O.p(bn[0]), O.p(bn[1]), O.p(mask))
        else:
            L.orc_shadows_ray_trace(scene.h, C.byref(gc), C.byref(f), p0, O.p(bn[0]), O.p(bn[1]), O.p(mask))
        acc += unpack_mask(mask, W, H)
    return acc / len(frames)


def blue_noise_bound(p, se, n):
    """what the mean of n one-ray masks may differ from the reference by, as an RMS over the pixels: the error of n independent samples
    of a Bernoulli(p) variable, sqrt(p (1 - p) / n), plus the reference's own standard error.  The blue noise's n = 256 samples are
    stratified, so they do not do worse than independent samples."""
    return float(np.sqrt(np.mean(p * (1 - p) / n + se ** 2)))
