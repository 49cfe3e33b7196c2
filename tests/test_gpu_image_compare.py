"""hr_image_compare on the device against the host restatement (image_compare.py): the integer sums exactly, in every accepted format,
at 1x1 to 3840x2160, on random fp16 bits (negatives, values above 1, subnormals, NaN, +-inf) and on images that differ in one pixel at
each corner; the error map in the range's rows only; row splits on one GPU and the bands of emulated linked ranks adding up to the
whole image's sums; refused calls changing nothing; a real frame (deferred combine against the path tracer); the launch counter.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import image_compare as IC
import measurement_hooks as MH
import pyhr
from test_gpu_launch_count import check_counted
from test_gpu_ragged import CAM_SHADOWS_TEST, SKY, _linked_ranks, frames, new_context

pytestmark = pytest.mark.gpu

FORMATS = [IC.FMT_RGBA16F, IC.FMT_RGBA8, IC.FMT_RG16F, IC.FMT_R16F]
SIZES = [(1, 1), (7, 3), (250, 141), (1366, 768), (3840, 2160)]
HR_ERR_INVALID_ARG, HR_ERR_UNSUPPORTED = -1, -5


def random_bits(rng, fmt, W, H, special=0.02):
    """a host image of format fmt: fp16 values around [-0.5, 1.5] with a `special` share of arbitrary bit patterns (subnormals, NaN,
    +-inf, huge values); RGBA8 random bytes"""
    if fmt == IC.FMT_RGBA8:
        return rng.integers(0, 256, size=(H, W, 4), dtype=np.uint8)
    C_ = {IC.FMT_R16F: 1, IC.FMT_RG16F: 2, IC.FMT_RGBA16F: 4}[fmt]
    a = rng.normal(0.5, 0.5, size=(H, W, C_)).astype(np.float16).view(np.uint16)
    m = rng.random(a.shape) < special
    a[m] = rng.integers(0, 1 << 16, size=int(m.sum()), dtype=np.uint16)
    sub = rng.random(a.shape) < special / 2
    a[sub] = rng.integers(1, 1024, size=int(sub.sum()), dtype=np.uint16) | (rng.integers(0, 2, size=int(sub.sum()), dtype=np.uint16) << 15)
    return a[..., 0] if C_ == 1 else a


def near(rng, a, fmt):
    """the test image: `a` with noise (special patterns of `a` kept, a few new ones)"""
    if fmt == IC.FMT_RGBA8:
        return np.clip(a.astype(np.int32) + rng.integers(-12, 13, size=a.shape), 0, 255).astype(np.uint8)
    f = a.view(np.float16).astype(np.float32)
    with np.errstate(all="ignore"):
        b = (f + rng.normal(0, 0.03, size=f.shape).astype(np.float32)).astype(np.float16).view(np.uint16)
    m = rng.random(b.shape) < 0.005
    b[m] = rng.integers(0, 1 << 16, size=int(m.sum()), dtype=np.uint16)
    return b


def device(a):
    """a host image on the device (the tensor keeps the memory alive)"""
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8 if a.dtype == np.uint8 else np.int16)).cuda()


def himg(t, fmt, W, H):
    return pyhr.hr_image(t.data_ptr(), W, H, fmt)


def as_dict(s):
    return dict(pixels=s.pixels, nonfinite_test=s.nonfinite_test, nonfinite_ref=s.nonfinite_ref, sq=s.sq(), abs=s.abs(), rel=s.rel(), ssim=s.ssim_sum(),
                max_abs_err=s.max_abs_err)


@pytest.fixture(scope="module")
def ctx():
    c = pyhr.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("W,H", SIZES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_exact_sums(ctx, fmt, W, H):
    rng = np.random.default_rng(W * 7 + H * 3 + fmt)
    ref = random_bits(rng, fmt, W, H)
    test = near(rng, ref, fmt)
    dt, dr = device(test), device(ref)
    T = IC.pixel_terms(test, ref, fmt)
    want = IC.sums(test, ref, fmt, terms=T)
    got = as_dict(ctx.compare(himg(dt, fmt, W, H), himg(dr, fmt, W, H)))
    assert got == want, f"{W}x{H} format {fmt}: device {got}, restatement {want}"
    if fmt != IC.FMT_RGBA8 and W * H > 100:
        assert want["nonfinite_test"] > 0 and want["nonfinite_ref"] > 0 and want["ssim"] < want["pixels"] << 32
    # non-default parameters
    p = pyhr.hr_compare_params(0.25, 0.0, 0.5)
    got = as_dict(ctx.compare(himg(dt, fmt, W, H), himg(dr, fmt, W, H), params=p))
    assert got == IC.sums(test, ref, fmt, params=(p.relmse_eps, p.ssim_c1, p.ssim_c2))


@pytest.mark.parametrize("W,H", [(1, 1), (7, 3), (250, 141), (1366, 768)])
@pytest.mark.parametrize("fmt", FORMATS)
def test_one_pixel_at_each_corner(ctx, fmt, W, H):
    """identical images but for one pixel at a corner: the clamped SSIM taps; the image with itself: ssim exactly 1"""
    rng = np.random.default_rng(5 + fmt)
    ref = random_bits(rng, fmt, W, H, special=0.0)
    dr = device(ref)
    same = ctx.compare(himg(dr, fmt, W, H), himg(dr, fmt, W, H))
    assert same.sq() == 0 and same.ssim_sum() == same.pixels << 32 == (W * H) << 32
    assert pyhr.compare_finish(same).psnr == float("inf")
    for y, x in ((0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1)):
        test = ref.copy()
        test[y, x] = (255 - test[y, x]) if fmt == IC.FMT_RGBA8 else np.float16(3.0).view(np.uint16) - test[y, x] % 7
        got = as_dict(ctx.compare(himg(device(test), fmt, W, H), himg(dr, fmt, W, H)))
        assert got == IC.sums(test, ref, fmt), f"{W}x{H} format {fmt}: corner ({x}, {y})"
        assert got["sq"] > 0


@pytest.mark.parametrize("W,H", [(7, 3), (250, 141), (1366, 768)])
def test_error_map(ctx, W, H):
    """the range's rows get the restatement's terms in fp16 (NaNs at left-out pixels); the other rows keep what they held"""
    fmt = IC.FMT_RGBA16F
    rng = np.random.default_rng(W + H)
    ref = random_bits(rng, fmt, W, H)
    test = near(rng, ref, fmt)
    dt, dr = device(test), device(ref)
    T = IC.pixel_terms(test, ref, fmt)
    before = rng.integers(0, 1 << 16, size=(H, W, 4), dtype=np.uint16)
    for r0, r1 in ((0, 0), (0, H), (1, H - 1), (H // 2, H // 2 + 1), (H - 1, H), (2, 2)):
        em = device(before)
        got = ctx.compare(himg(dt, fmt, W, H), himg(dr, fmt, W, H), r0, r1, error_map=himg(em, IC.FMT_RGBA16F, W, H))
        a = em.cpu().numpy().view(np.uint16)
        want = IC.error_map(T, *((0, H) if r1 <= 0 else (r0, r1)), before)
        assert np.array_equal(a, want), f"{W}x{H} rows [{r0}, {r1}): error map differs at {np.argwhere(a != want)[:5].tolist()}"
        assert as_dict(got) == IC.sums(test, ref, fmt, r0, r1, terms=T)


@pytest.mark.parametrize("fmt", FORMATS)
def test_row_splits_add_up(ctx, fmt):
    W, H = 1366, 768
    rng = np.random.default_rng(40 + fmt)
    ref = random_bits(rng, fmt, W, H)
    test = near(rng, ref, fmt)
    dt, dr = device(test), device(ref)
    whole = ctx.compare(himg(dt, fmt, W, H), himg(dr, fmt, W, H))
    assert as_dict(whole) == IC.sums(test, ref, fmt)
    for k in (2, 3, 5, 9):
        cuts = MH.random_cuts(rng, H, k)
        acc = pyhr.hr_compare_sums()
        for r0, r1 in zip(cuts[:-1], cuts[1:]):
            part = ctx.compare(himg(dt, fmt, W, H), himg(dr, fmt, W, H), r0, r1) if r1 > r0 else pyhr.hr_compare_sums()
            pyhr.sums_add(acc, part)
        assert as_dict(acc) == as_dict(whole), f"split at {cuts}"


@pytest.mark.parametrize("world", [2, 3])
def test_linked_ranks_bands_add_up(world):
    """linked shadows + AO ranks feed each rank's deferred combine; their bands are gathered into every rank's image (what the
    gather does across GPUs); each rank compares its band hr_shard_rows with the single-GPU path tracer image, and the sums,
    added with hr_compare_sums_add, equal the single-GPU comparison"""
    W, H = 250, 141
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)

    def make(rank, world):
        c = pyhr.Context(0)
        c.set_bluenoise(*pyhr.blue_noise())
        c.build_scene(sc)
        c.gbuffer_create(W, H)
        if world > 1:
            c.shard_config(rank, world)
        return c, pyhr.Pass(c, "shadows", W, H, 0), pyhr.Pass(c, "ao", W, H, 0)

    ref, ranks = _linked_ranks(make, world)
    des = [pyhr.DeferredPass(c, W, H) for c, *_ in [ref] + ranks]
    for d in des:
        d.params.env_color[0], d.params.env_color[1], d.params.env_color[2] = SKY
    pt = pyhr.PathTracerPass(ref[0], W, H)
    pt.params.sky_color[0], pt.params.sky_color[1], pt.params.sky_color[2] = SKY
    streams = [torch.cuda.Stream() for _ in range(world)]
    for i, f in frames(W, H, 3, pan_from=2):
        ref[0].gbuffer_render(f.ping_pong, f)
        ref[1].render(f)
        ref[2].render(f)
        des[0].render(f, ref[1], ref[2], None, None)
        pt.render(f)
        for (c, sh, ao), st in zip(ranks, streams):
            c.gbuffer_render(f.ping_pong, f, stream=st.cuda_stream)
        for (c, sh, ao), st in zip(ranks, streams):
            sh.render(f, st.cuda_stream)
        for (c, sh, ao), st in zip(ranks, streams):
            ao.render(f, st.cuda_stream)
        for (c, sh, ao), d, st in zip(ranks, des[1:], streams):
            d.render(f, sh, ao, None, None, st.cuda_stream)
        torch.cuda.synchronize()
        bands = [pyhr.shard_rows(H, r, world) for r in range(world)]
        full = np.concatenate([des[1 + r].download(100)[b0:b1] for r, (b0, b1) in enumerate(bands)])
        assert np.array_equal(full, des[0].download(100)), f"frame {i}: the ranks' bands are not the single-GPU frame"
        for d in des[1:]:
            d.upload(100, full)
        want = ref[0].compare(des[0], pt)
        acc = pyhr.hr_compare_sums()
        for r, (b0, b1) in enumerate(bands):
            pyhr.sums_add(acc, ranks[r][0].compare(des[1 + r], pt.output(100), b0, b1))
        assert as_dict(acc) == as_dict(want), f"frame {i} world {world}: the bands' sums do not add up"
        assert as_dict(want) == IC.sums(des[0].download(100), pt.download(100), IC.FMT_RGBA16F)
    for p in des + [pt]:
        p.destroy()
    for c, sh, ao in [ref] + ranks:
        sh.destroy()
        ao.destroy()
        c.close()


def test_refusals_change_nothing(ctx):
    W, H = 64, 32
    rng = np.random.default_rng(3)
    a, b = random_bits(rng, IC.FMT_RGBA16F, W, H), random_bits(rng, IC.FMT_RGBA16F, W, H)
    da, db = device(a), device(b)
    u32, u8 = torch.zeros((H, W), dtype=torch.int32, device="cuda"), torch.zeros((H, W), dtype=torch.uint8, device="cuda")
    small = device(a[:H - 1])
    em_bits = rng.integers(0, 1 << 16, size=(H, W, 4), dtype=np.uint16)
    em = device(em_bits)
    big = device(np.concatenate([b, b]))  # 2H rows: images placed inside it overlap without leaving the allocation
    good = pyhr.compare_default_params()
    t, r, m = himg(da, IC.FMT_RGBA16F, W, H), himg(db, IC.FMT_RGBA16F, W, H), himg(em, IC.FMT_RGBA16F, W, H)
    lib = ctx.lib
    sentinel = pyhr.hr_compare_sums()
    C.memset(C.byref(sentinel), 0xA5, C.sizeof(sentinel))

    def call(test, ref_, params, row0, row1, out, emap):
        return lib.hr_image_compare(ctx.h, test and C.byref(test), ref_ and C.byref(ref_), params and C.byref(params), row0, row1, out and C.byref(out),
                                    emap and C.byref(emap), C.c_void_p(0))

    cases = [
        ("null test", (None, r, good, 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("null ref", (t, None, good, 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("null params", (t, r, None, 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("null out", (t, r, good, 0, 0, False, m), HR_ERR_INVALID_ARG),
        ("null data", (pyhr.hr_image(None, W, H, IC.FMT_RGBA16F), r, good, 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("height mismatch", (himg(small, IC.FMT_RGBA16F, W, H - 1), r, good, 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("width mismatch", (pyhr.hr_image(da.data_ptr(), W - 1, H, IC.FMT_RGBA16F), r, good, 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("format mismatch", (pyhr.hr_image(da.data_ptr(), W, H, IC.FMT_RG16F), r, good, 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("zero size", (pyhr.hr_image(da.data_ptr(), 0, H, IC.FMT_RGBA16F), pyhr.hr_image(db.data_ptr(), 0, H, IC.FMT_RGBA16F), good, 0, 0, True, m),
         HR_ERR_INVALID_ARG),
        ("unknown format", (pyhr.hr_image(da.data_ptr(), W, H, 9), pyhr.hr_image(db.data_ptr(), W, H, 9), good, 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("R32_UINT", (pyhr.hr_image(u32.data_ptr(), W, H, 1), pyhr.hr_image(u32.data_ptr(), W, H, 1), good, 0, 0, True, m), HR_ERR_UNSUPPORTED),
        ("R8_UINT", (pyhr.hr_image(u8.data_ptr(), W, H, 5), pyhr.hr_image(u8.data_ptr(), W, H, 5), good, 0, 0, True, m), HR_ERR_UNSUPPORTED),
        ("row0 < 0", (t, r, good, -1, 5, True, m), HR_ERR_INVALID_ARG),
        ("row1 > H", (t, r, good, 0, H + 1, True, m), HR_ERR_INVALID_ARG),
        ("row1 < row0", (t, r, good, 7, 3, True, m), HR_ERR_INVALID_ARG),
        ("row0 > H", (t, r, good, H + 1, H + 2, True, m), HR_ERR_INVALID_ARG),
        ("negative eps", (t, r, pyhr.hr_compare_params(-0.01, 1e-4, 9e-4), 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("negative c1", (t, r, pyhr.hr_compare_params(0.01, -1e-4, 9e-4), 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("negative c2", (t, r, pyhr.hr_compare_params(0.01, 1e-4, -9e-4), 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("NaN c2", (t, r, pyhr.hr_compare_params(0.01, 1e-4, float("nan")), 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("inf eps", (t, r, pyhr.hr_compare_params(float("inf"), 1e-4, 9e-4), 0, 0, True, m), HR_ERR_INVALID_ARG),
        ("error map size", (t, r, good, 0, 0, True, pyhr.hr_image(em.data_ptr(), W, H - 1, IC.FMT_RGBA16F)), HR_ERR_INVALID_ARG),
        ("error map format", (t, r, good, 0, 0, True, pyhr.hr_image(em.data_ptr(), W, H, IC.FMT_RG16F)), HR_ERR_INVALID_ARG),
        ("error map data", (t, r, good, 0, 0, True, pyhr.hr_image(None, W, H, IC.FMT_RGBA16F)), HR_ERR_INVALID_ARG),
        ("error map is the test image", (t, r, good, 0, 0, True, t), HR_ERR_INVALID_ARG),
        ("error map overlaps ref", (t, pyhr.hr_image(big.data_ptr(), W, H, IC.FMT_RGBA16F), good, 0, 0, True,
                                    pyhr.hr_image(big.data_ptr() + 8 * W * (H // 2), W, H, IC.FMT_RGBA16F)), HR_ERR_INVALID_ARG),
        ("error map ends in test", (pyhr.hr_image(big.data_ptr() + 8 * W * (H - 1), W, H, IC.FMT_RGBA16F), pyhr.hr_image(db.data_ptr(), W, H, IC.FMT_RGBA16F),
                                    good, 0, 0, True, pyhr.hr_image(big.data_ptr(), W, H, IC.FMT_RGBA16F)), HR_ERR_INVALID_ARG),
    ]
    for what, (tt, rr, pp, r0, r1, has_out, mm), code in cases:
        out = pyhr.hr_compare_sums()
        C.memmove(C.byref(out), C.byref(sentinel), C.sizeof(out))
        n0 = ctx.launch_count()
        assert call(tt, rr, pp, r0, r1, out if has_out else None, mm) == code, what
        torch.cuda.synchronize()
        assert bytes(out) == bytes(sentinel), f"{what}: out was written"
        assert np.array_equal(em.cpu().numpy().view(np.uint16), em_bits), f"{what}: the error map was written"
        for buf, bits in ((da, a), (db, b), (big, np.concatenate([b, b]))):
            assert np.array_equal(buf.cpu().numpy().view(np.uint16), bits), f"{what}: an input image was written"
        assert ctx.launch_count() == n0, f"{what}: kernels launched"
    # the accepted neighbours of the refused calls
    assert call(t, r, pyhr.hr_compare_params(0.0, 0.0, 0.0), 0, 0, sentinel, None) == 0
    assert call(t, r, good, H, H, sentinel, m) == 0 and sentinel.pixels == 0 and sentinel.sq() == 0


def test_real_frame(ctx):
    """the hybrid chain (shadows, AO, DDGI, reflections, deferred with a BRDF LUT, so the reflections reach it) against the indirect path
    tracer on the shadows-test scene: finite results within plausible bounds; the deferred frame with itself: ssim exactly 1, mse 0"""
    W, H = 256, 144
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    c = new_context(sc, W, H)
    c.set_brdf_lut(pyhr.brdf_lut(64))  # the deferred combine adds the reflections (its indirect specular term) only with a LUT
    sh, ao, dd, rf, de = (pyhr.Pass(c, "shadows", W, H, 0), pyhr.Pass(c, "ao", W, H, 1), pyhr.DDGIPass(c, W, H, 0), pyhr.ReflectionsPass(c, W, H, 1),
                          pyhr.DeferredPass(c, W, H))
    pt = pyhr.PathTracerPass(c, W, H)
    for P in (dd.params, rf.params, pt.params):
        P.sky_color[0], P.sky_color[1], P.sky_color[2] = SKY
    de.params.env_color[0], de.params.env_color[1], de.params.env_color[2] = SKY
    dd.params.probe_distance = 4.0
    pt.params.trace_indirect = 1
    f = None
    for i in range(8):
        f = pyhr.make_frame(*CAM_SHADOWS_TEST, W, H, prev=f, num_frames=i)
        c.gbuffer_render(f.ping_pong, f)
        sh.render(f)
        ao.render(f)
        dd.render(f, pyhr.rotation_matrix(0.3 + i, (0.2, 1.0, -0.4)))
        rf.render(f, dd)
        de.render(f, sh, ao, rf, dd)
        pt.render(f)
    em = torch.zeros((H, W, 4), dtype=torch.int16, device="cuda")
    s = c.compare(de, pt, error_map=himg(em, IC.FMT_RGBA16F, W, H))
    r = pyhr.compare_finish(s)
    assert s.pixels == W * H and s.nonfinite_test == 0 and s.nonfinite_ref == 0
    assert 0.0 < r.mse < 1.0 and 0.0 < r.psnr < 100.0 and -1.0 < r.ssim < 1.0 and 0.0 < r.relmse and 0.0 < r.max_abs
    assert as_dict(s) == IC.sums(de.download(100), pt.download(100), IC.FMT_RGBA16F)
    assert np.isfinite(em.cpu().numpy().view(np.float16).astype(np.float32)[..., [0, 2, 3]]).all()
    same = c.compare(de, de)
    assert same.ssim_sum() == same.pixels << 32 and same.sq() == 0 and pyhr.compare_finish(same).ssim == 1.0
    de_no_rf = pyhr.DeferredPass(c, W, H)
    de_no_rf.params.env_color[0], de_no_rf.params.env_color[1], de_no_rf.params.env_color[2] = SKY
    de_no_rf.render(f, sh, ao, None, dd)
    assert c.compare(de, de_no_rf).sq() > 0, "the reflections do not reach the deferred frame"
    for p in (de_no_rf, pt, de, rf, dd, ao, sh):
        p.destroy()
    c.close()


def test_launch_count(ctx):
    """two kernels per comparison of a non-empty range (the per-tile sums, their total), none for an empty range"""
    W, H = 250, 141
    rng = np.random.default_rng(8)
    a, b = random_bits(rng, IC.FMT_RGBA16F, W, H), random_bits(rng, IC.FMT_RGBA16F, W, H)
    da, db = device(a), device(b)
    t, r = himg(da, IC.FMT_RGBA16F, W, H), himg(db, IC.FMT_RGBA16F, W, H)
    for r0, r1, n in ((0, 0, 2), (5, 6, 2), (7, 7, 0), (H, H, 0)):
        before = ctx.launch_count()
        ctx.compare(t, r, r0, r1)
        assert ctx.launch_count() - before == n, (r0, r1)
        check_counted([ctx], lambda: ctx.compare(t, r, r0, r1), f"hr_image_compare rows [{r0}, {r1})")
