"""Host restatement of hr_image_compare (include/hr_api.h, "Image comparison"): the per-pixel terms in float32 numpy in the kernel's
operation order, the 128-bit fixed-point sums as Python integers, hr_compare_sums_add and hr_compare_finish.  No GPU and no CUDA
library needed; the CPU checks of this file are tests/test_image_compare_cpu.py, the device comparison tests/test_gpu_image_compare.py.
"""
import math

import numpy as np

F = np.float32
R = 5  # window radius: 11 taps
U128 = 1 << 128
FMT_R16F, FMT_RG16F, FMT_RGBA16F, FMT_RGBA8 = 2, 3, 4, 6
CHANNELS = {FMT_R16F: 1, FMT_RG16F: 2, FMT_RGBA16F: 3, FMT_RGBA8: 3}
QNAN_H = 0x7E00
FIELDS = ("pixels", "nonfinite_test", "nonfinite_ref", "sq", "abs", "rel", "ssim", "max_abs_err")


def gaussian_window(sigma=1.5):
    """the 11 float32 weights: each in double, normalised by their sum (in tap order), then rounded"""
    g = [math.exp(-float(k * k) / (2.0 * sigma * sigma)) for k in range(-R, R + 1)]
    s = 0.0
    for v in g:
        s += v
    return np.array([v / s for v in g], F)


WINDOW = gaussian_window()


def channels(img, fmt):
    """device image ((H, W) uint16, (H, W, 2 | 4) uint16 holding fp16 bits, or (H, W, 4) uint8) -> (H, W, C) float32"""
    a = np.asarray(img)
    if fmt == FMT_RGBA8:
        return a[..., :3].astype(F) / F(255)
    h = a.view(np.float16).astype(F)
    if fmt == FMT_R16F:
        return h.reshape(h.shape[0], h.shape[1], 1)
    return h[..., :CHANNELS[fmt]]


def luminance(c):
    k = np.clip(c, F(0), F(1)).astype(F)
    if c.shape[2] == 1:
        return k[..., 0]
    c2 = k[..., 2] if c.shape[2] == 3 else np.zeros_like(k[..., 0])
    return (F(0.299) * k[..., 0] + F(0.587) * k[..., 1]) + F(0.114) * c2


def pixel_terms(test, ref, fmt, params=(0.01, 1e-4, 9e-4)):
    """per-pixel terms of the whole image: dict of (H, W) arrays ae, se, rel, ssim (float32), max_d (largest channel |d|), fin_t,
    fin_r, ok (bool).  Terms at left-out pixels are meaningless (masked by ok)"""
    eps, c1, c2 = (F(p) for p in params)
    t, r = channels(test, fmt), channels(ref, fmt)
    H, W, C = t.shape
    fin_t, fin_r = np.isfinite(t).all(2), np.isfinite(r).all(2)
    ok = fin_t & fin_r
    with np.errstate(all="ignore"):
        d = t - r
        se, ae, rl = (np.zeros((H, W), F) for _ in range(3))
        for k in range(C):
            dk = d[..., k]
            d2 = dk * dk
            se = se + d2
            ae = ae + np.abs(dk)
            rl = rl + d2 / (r[..., k] * r[..., k] + eps)
        se, ae, rl = se / F(C), ae / F(C), rl / F(C)
        max_d = np.abs(d).max(2)
        yt = np.where(ok, luminance(np.where(ok[..., None], t, F(0))), F(0)).astype(F)
        yr = np.where(ok, luminance(np.where(ok[..., None], r, F(0))), F(0)).astype(F)
        # rows first: taps along x clamped to the image
        pt, pr = np.pad(yt, ((0, 0), (R, R)), mode="edge"), np.pad(yr, ((0, 0), (R, R)), mode="edge")
        hq = [np.zeros((H, W), F) for _ in range(5)]
        for k in range(2 * R + 1):
            u, v, w = pt[:, k:k + W], pr[:, k:k + W], WINDOW[k]
            hq[0] = hq[0] + w * u
            hq[1] = hq[1] + w * v
            hq[2] = hq[2] + w * (u * u)
            hq[3] = hq[3] + w * (v * v)
            hq[4] = hq[4] + w * (u * v)
        # then columns, taps along y clamped to the image
        m = [np.zeros((H, W), F) for _ in range(5)]
        for j in range(5):
            p = np.pad(hq[j], ((R, R), (0, 0)), mode="edge")
            for k in range(2 * R + 1):
                m[j] = m[j] + WINDOW[k] * p[k:k + H, :]
        mt, mr = m[0], m[1]
        vt, vr, cv = m[2] - mt * mt, m[3] - mr * mr, m[4] - mt * mr
        ss = (((F(2) * mt) * mr + c1) * (F(2) * cv + c2)) / (((mt * mt + mr * mr) + c1) * ((vt + vr) + c2))
    return dict(ae=ae, se=se, rel=rl, ssim=ss.astype(F), max_d=max_d, fin_t=fin_t, fin_r=fin_r, ok=ok)


def fixed_terms(x):
    """round-to-nearest-even(x * 2^32) of float32 x clamped to [-2^63, 2^63], NaN -> 0, as integer-valued float32"""
    x = np.asarray(x, F)
    with np.errstate(invalid="ignore"):
        x = np.where(np.isnan(x), F(0), np.clip(x, F(-2.0**63), F(2.0**63))).astype(F)
    return np.rint(x * F(2.0**32)).astype(F)


def fixed_sum(x):
    """exact integer sum of fixed_terms(x): mantissas grouped by exponent (int64 per group, < 2^24 each)"""
    y = fixed_terms(x).ravel()
    if y.size == 0:
        return 0
    m, e = np.frexp(y)
    mi = (m * F(2.0**24)).astype(np.int64)
    sh = e.astype(np.int64) - 24
    total = 0
    for s in np.unique(sh):
        part = int(mi[sh == s].sum())
        total += part << int(s) if s >= 0 else part >> int(-s)  # exact: every term of a negative-shift group is an integer
    return total


def sums(test, ref, fmt, row0=0, row1=0, params=(0.01, 1e-4, 9e-4), terms=None):
    """hr_compare_sums of rows [row0, row1) (row1 <= 0: the whole image) as a dict of Python integers (sq, abs, rel mod 2^128,
    ssim signed)"""
    T = terms if terms is not None else pixel_terms(test, ref, fmt, params)
    H = T["ok"].shape[0]
    if row1 <= 0:
        row0, row1 = 0, H
    sl = slice(row0, row1)
    ok = T["ok"][sl]
    mx = T["max_d"][sl][ok]
    return dict(pixels=int(ok.sum()), nonfinite_test=int((~T["fin_t"][sl]).sum()), nonfinite_ref=int((~T["fin_r"][sl]).sum()),
                sq=fixed_sum(T["se"][sl][ok]) % U128, abs=fixed_sum(T["ae"][sl][ok]) % U128, rel=fixed_sum(T["rel"][sl][ok]) % U128,
                ssim=fixed_sum(T["ssim"][sl][ok]), max_abs_err=int(mx.max().view(np.uint32)) if mx.size else 0)


def add(a, b):
    """hr_compare_sums_add"""
    out = {k: a[k] + b[k] for k in ("pixels", "nonfinite_test", "nonfinite_ref")}
    for k in ("sq", "abs", "rel"):
        out[k] = (a[k] + b[k]) % U128
    s = (a["ssim"] + b["ssim"]) % U128
    out["ssim"] = s - U128 if s >> 127 else s
    out["max_abs_err"] = max(a["max_abs_err"], b["max_abs_err"])
    return out


def zero():
    return dict.fromkeys(FIELDS, 0)


def finish(s):
    """hr_compare_finish: each mean (double)(sum) * 2^-32 / (double)pixels (the integer rounded once); psnr = 10 log10(1 / mse)"""
    n = float(s["pixels"])

    def mean(v):
        return float(v) * 2.0**-32 / n if n else math.nan

    mse = mean(s["sq"])
    return dict(mse=mse, rmse=math.sqrt(mse) if mse == mse else math.nan,
                psnr=math.inf if mse == 0.0 else (10.0 * math.log10(1.0 / mse) if mse == mse else math.nan),
                relmse=mean(s["rel"]), mean_abs=mean(s["abs"]), max_abs=float(np.uint32(s["max_abs_err"]).view(F)), ssim=mean(s["ssim"]),
                pixels=s["pixels"], nonfinite_test=s["nonfinite_test"], nonfinite_ref=s["nonfinite_ref"])


def error_map(T, row0, row1, before):
    """what hr_image_compare leaves in an error map that held `before` ((H, W, 4) uint16): rows [row0, row1) get (ae, se, rel, ssim) in
    fp16 (quiet NaNs at left-out pixels), the other rows are unchanged"""
    out = before.copy()
    q = np.stack([T["ae"], T["se"], T["rel"], T["ssim"]], 2)[row0:row1]
    with np.errstate(over="ignore", invalid="ignore"):
        h = q.astype(np.float16).view(np.uint16)
    h = np.where(T["ok"][row0:row1, :, None], h, np.uint16(QNAN_H))
    out[row0:row1] = h
    return out
