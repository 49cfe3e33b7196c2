"""The host restatement of hr_image_compare (image_compare.py) on the CPU: against an independent float64 formulation
(scipy.ndimage.correlate1d, mode "nearest", the continuous Gaussian), known answers, row splits, the exact fixed-point sums, and the
library's pure host functions hr_compare_sums_add / hr_compare_finish (called in libhr_b200.so, no device needed) against add / finish.
"""
import math

import numpy as np
import pytest
from scipy.ndimage import correlate1d

import image_compare as IC
import measurement_hooks as MH
import pyhr

FORMATS = [IC.FMT_RGBA16F, IC.FMT_RGBA8, IC.FMT_RG16F, IC.FMT_R16F]


def random_image(rng, fmt, W, H, lo=-0.25, hi=1.5):
    """a device image of format fmt with smooth structure plus noise (values outside [0, 1] included for the fp16 formats)"""
    if fmt == IC.FMT_RGBA8:
        return rng.integers(0, 256, size=(H, W, 4), dtype=np.uint8)
    C = {IC.FMT_R16F: 1, IC.FMT_RG16F: 2, IC.FMT_RGBA16F: 4}[fmt]
    y, x = np.mgrid[0:H, 0:W]
    base = 0.5 + 0.4 * np.sin(x[..., None] * 0.3 + np.arange(C) * 1.1) * np.cos(y[..., None] * 0.2)
    a = np.clip(base + rng.normal(0, 0.2, size=(H, W, C)), lo, hi).astype(np.float16).view(np.uint16)
    return a[..., 0] if C == 1 else a


def perturb(rng, img, fmt):
    """a second image near the first: the test image of a comparison"""
    if fmt == IC.FMT_RGBA8:
        return np.clip(img.astype(np.int32) + rng.integers(-20, 21, size=img.shape), 0, 255).astype(np.uint8)
    f = img.view(np.float16).astype(np.float32)
    return (f + rng.normal(0, 0.05, size=f.shape).astype(np.float32)).astype(np.float16).view(np.uint16)


def float64_metrics(test, ref, fmt, eps=0.01, c1=1e-4, c2=9e-4):
    """the metrics in float64, written independently: scipy's separable correlation with edge-nearest taps"""
    t, r = (IC.channels(a, fmt).astype(np.float64) for a in (test, ref))
    d = t - r
    C = t.shape[2]

    def lum(c):
        k = np.clip(c, 0.0, 1.0)
        if C == 1:
            return k[..., 0]
        return 0.299 * k[..., 0] + 0.587 * k[..., 1] + (0.114 * k[..., 2] if C == 3 else 0.0)

    g = np.exp(-np.arange(-5, 6, dtype=np.float64) ** 2 / (2 * 1.5**2))
    g /= g.sum()

    def blur(a):
        return correlate1d(correlate1d(a, g, axis=1, mode="nearest"), g, axis=0, mode="nearest")

    yt, yr = lum(t), lum(r)
    mt, mr = blur(yt), blur(yr)
    vt, vr, cv = blur(yt * yt) - mt * mt, blur(yr * yr) - mr * mr, blur(yt * yr) - mt * mr
    ssim = ((2 * mt * mr + c1) * (2 * cv + c2)) / ((mt * mt + mr * mr + c1) * (vt + vr + c2))
    return dict(mse=np.mean(d * d), relmse=np.mean(d * d / (r * r + eps)), mean_abs=np.mean(np.abs(d)), max_abs=np.abs(d).max(), ssim=ssim.mean())


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("W,H", [(64, 48), (37, 23), (5, 3)])
def test_restatement_agrees_with_float64(fmt, W, H):
    rng = np.random.default_rng(W * 100 + H + fmt)
    ref = random_image(rng, fmt, W, H)
    test = perturb(rng, ref, fmt)
    got = IC.finish(IC.sums(test, ref, fmt))
    want = float64_metrics(test, ref, fmt)
    assert got["pixels"] == W * H
    for k in ("mse", "relmse", "mean_abs", "max_abs"):
        assert abs(got[k] - want[k]) <= 1e-6 * abs(want[k]), f"{k}: {got[k]!r} vs float64 {want[k]!r}"
    assert abs(got["ssim"] - want["ssim"]) <= 1e-5, f"ssim {got['ssim']!r} vs float64 {want['ssim']!r}"
    assert 0.0 < got["ssim"] < 1.0


@pytest.mark.parametrize("fmt", FORMATS)
def test_identical_images(fmt):
    rng = np.random.default_rng(fmt)
    a = random_image(rng, fmt, 41, 29)
    s = IC.sums(a, a, fmt)
    assert (s["sq"], s["abs"], s["rel"], s["max_abs_err"]) == (0, 0, 0, 0)
    assert s["ssim"] == s["pixels"] << 32, "ssim of an image with itself is not exactly 1"
    f = IC.finish(s)
    assert f["mse"] == 0.0 and f["ssim"] == 1.0 and f["psnr"] == math.inf


@pytest.mark.parametrize("fmt", [IC.FMT_RGBA16F, IC.FMT_RG16F, IC.FMT_R16F])
def test_constant_offset(fmt):
    """ref in [0.25, 0.5) on the fp16 grid, test = ref + k: every d is exactly k, so mse = k^2 and mean_abs = k exactly"""
    rng = np.random.default_rng(11)
    C = {IC.FMT_R16F: 1, IC.FMT_RG16F: 2, IC.FMT_RGBA16F: 4}[fmt]
    r = (0.25 + rng.integers(0, 256, size=(19, 33, C)) / 1024.0).astype(np.float16)
    for k in (0.125, 0.0625, 0.5):
        t = (r.astype(np.float32) + k).astype(np.float16)
        assert np.array_equal(t.astype(np.float32) - r.astype(np.float32), np.full(r.shape, k, np.float32))
        ti, ri = (x.view(np.uint16)[..., 0] if C == 1 else x.view(np.uint16) for x in (t, r))
        f = IC.finish(IC.sums(ti, ri, fmt))
        assert f["mse"] == k * k and f["mean_abs"] == k and f["max_abs"] == k
        assert f["psnr"] == 10.0 * math.log10(1.0 / (k * k))


@pytest.mark.parametrize("fmt", FORMATS)
def test_swap_keeps_mse_and_ssim(fmt):
    rng = np.random.default_rng(7 + fmt)
    a = random_image(rng, fmt, 30, 26)
    b = perturb(rng, a, fmt)
    s, w = IC.sums(a, b, fmt), IC.sums(b, a, fmt)
    for k in ("pixels", "sq", "abs", "ssim", "max_abs_err"):
        assert s[k] == w[k], k


def test_non_finite_pixels_are_left_out():
    rng = np.random.default_rng(5)
    a = random_image(rng, IC.FMT_RGBA16F, 23, 17)
    b = perturb(rng, a, IC.FMT_RGBA16F)
    a[3, 4, 1] = 0x7C00   # +inf in the test image
    b[3, 4, 0] = 0x7E00   # and NaN in the reference at the same pixel
    b[9, 0, 2] = 0xFC00   # -inf in the reference
    a[16, 22, 3] = 0x7E00  # NaN in alpha: ignored
    s = IC.sums(a, b, IC.FMT_RGBA16F)
    assert (s["pixels"], s["nonfinite_test"], s["nonfinite_ref"]) == (23 * 17 - 2, 1, 2)
    f = IC.finish(s)
    assert all(math.isfinite(f[k]) for k in ("mse", "relmse", "mean_abs", "max_abs", "ssim"))


@pytest.mark.parametrize("fmt", FORMATS)
def test_row_splits_add_up(fmt):
    rng = np.random.default_rng(100 + fmt)
    W, H = 29, 53
    a = random_image(rng, fmt, W, H)
    b = perturb(rng, a, fmt)
    T = IC.pixel_terms(a, b, fmt)
    whole = IC.sums(a, b, fmt, terms=T)
    for k in (2, 3, 7):
        cuts = MH.random_cuts(rng, H, k)
        acc = IC.zero()
        for r0, r1 in zip(cuts[:-1], cuts[1:]):
            if r1 > r0:
                acc = IC.add(acc, IC.sums(a, b, fmt, r0, r1, terms=T))
        assert acc == whole, f"split at {cuts}"


def test_fixed_point_terms():
    """round-to-nearest-even(x * 2^32) against exact rational arithmetic, at ties, the clamp and NaN"""
    from fractions import Fraction
    xs = np.array([0.0, -0.0, 2.0**-33, 3 * 2.0**-33, 5 * 2.0**-33, -3 * 2.0**-33, 1.0, -1.0, 0.1, -0.7, 1e-12, 2.0**40 + 2.0**17,
                   2.0**63, 2.0**70, -2.0**90, np.inf, -np.inf, np.nan, 1.7e10], np.float32)
    for x in xs:
        if math.isnan(x):
            want = 0
        else:
            v = Fraction(min(max(float(x), -2.0**63), 2.0**63)) * 2**32
            fl = math.floor(v)
            want = fl + 1 if v - fl > Fraction(1, 2) or (v - fl == Fraction(1, 2) and fl % 2) else fl
        assert IC.fixed_sum(np.array([x], np.float32)) == want, x
    rng = np.random.default_rng(1)
    v = (rng.normal(0, 1, 5000) * 10.0 ** rng.integers(-9, 6, 5000)).astype(np.float32)
    assert IC.fixed_sum(v) == sum(IC.fixed_sum(np.array([x], np.float32)) for x in v)


def _as_struct(d):
    s = pyhr.hr_compare_sums()
    s.pixels, s.nonfinite_test, s.nonfinite_ref = d["pixels"], d["nonfinite_test"], d["nonfinite_ref"]
    for name, k in (("sq_err", "sq"), ("abs_err", "abs"), ("rel_err", "rel"), ("ssim", "ssim")):
        v = d[k] % IC.U128
        getattr(s, name)[0], getattr(s, name)[1] = v & (2**64 - 1), v >> 64
    s.max_abs_err = d["max_abs_err"]
    return s


def _as_dict(s):
    return dict(pixels=s.pixels, nonfinite_test=s.nonfinite_test, nonfinite_ref=s.nonfinite_ref, sq=s.sq(), abs=s.abs(), rel=s.rel(), ssim=s.ssim_sum(),
                max_abs_err=s.max_abs_err)


def test_library_sums_add_and_finish():
    """hr_compare_sums_add and hr_compare_finish of libhr_b200.so equal add / finish: carries out of the low 64 bits, negative SSIM sums
    and their crossing of 0, sums past 2^64, the max, no pixel summed"""
    rng = np.random.default_rng(9)
    M = 2**64 - 1

    def big(bits):
        return int.from_bytes(rng.bytes(16), "little") >> (128 - bits)

    cases = [IC.zero()]
    for i in range(200):
        d = dict(pixels=int(rng.integers(0, 2**40)), nonfinite_test=int(rng.integers(0, 100)), nonfinite_ref=int(rng.integers(0, 100)),
                 max_abs_err=int(np.float32(rng.uniform(0, 4)).view(np.uint32)))
        for k in ("sq", "abs", "rel"):
            d[k] = [M - big(20), big(94), big(50)][i % 3]
        d["ssim"] = [-big(70), big(70), -1, M][i % 4]
        cases.append(d)
    acc_py, acc_c = IC.zero(), pyhr.hr_compare_sums()
    for d in cases:
        acc_py = IC.add(acc_py, d)
        pyhr.sums_add(acc_c, _as_struct(d))
        assert _as_dict(acc_c) == acc_py
        for s in (d, acc_py):
            got, want = pyhr.compare_finish(_as_struct(s)), IC.finish(s)
            for k, v in want.items():
                g = getattr(got, k)
                assert g == v or (isinstance(v, float) and math.isnan(v) and math.isnan(g)), f"{k}: library {g!r}, restatement {v!r}"
    assert acc_py["ssim"] < 0 or any(d["ssim"] < 0 for d in cases)
    p = pyhr.compare_default_params()
    assert (p.relmse_eps, p.ssim_c1, p.ssim_c2) == (np.float32(0.01), np.float32(1e-4), np.float32(9e-4))
