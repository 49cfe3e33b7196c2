"""GPU: the converged references (hr_reference_create / hr_reference_render) against their CPU restatement and their targets.

Shadows and AO follow the deterministic chain, so their counts (seen through MEAN = count / N at sample counts whose quotients
fp16 keeps apart) equal the oracle's bit for bit; reflections colours are compared with the K12 parity tolerance of
test_gpu_gi_refl.py (RMSE 1e-3, max-abs 6e-3 relative to max(1, |reference|))."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
import oracle_reference as R
import pyhr

pytestmark = pytest.mark.gpu

SKY = (0.3, 0.4, 0.6)
CAM = ((0.0, 14.0, 34.0), (0.0, 3.0, 0.0))


def f16(a):
    return np.ascontiguousarray(a).view(np.float16).astype(np.float32)


def close(a, b, name, r=1e-3, m=6e-3):
    assert a.shape == b.shape, name
    d = np.abs(a - b) / np.maximum(1.0, np.abs(b))
    e = float(np.sqrt(np.mean(d.astype(np.float64) ** 2)))
    assert e <= r and d.max() <= m, f"{name}: rmse {e}, max {d.max()}"


class Rig:
    def __init__(self, W, H, scene=pyhr.SCENE_SHADOWS_TEST):
        self.W, self.H = W, H
        self.sc = pyhr.SynthScene(scene)
        self.bn = pyhr.blue_noise()
        self.ctx = pyhr.Context(0)
        self.ctx.set_bluenoise(*self.bn)
        self.ctx.build_scene(self.sc)
        self.ctx.gbuffer_create(W, H)
        self.f = None
        self.n = 0

    def frame(self, gbuf_edit=None):
        self.f = pyhr.make_frame(*CAM, self.W, self.H, prev=self.f, num_frames=self.n)
        self.n += 1
        self.g = pyhr.write_gbuffer(self.sc, self.f, self.W, self.H)
        if gbuf_edit:
            gbuf_edit(self.g)
        self.ctx.gbuffer_upload(self.f.ping_pong, self.g)
        return self.f

    def close(self):
        self.ctx.close()


def mask_params(kind, bias):
    P = pyhr.hr_shadows_params() if kind == "shadows" else pyhr.hr_ao_params()
    L = pyhr.load_product()
    (L.hr_shadows_default_params if kind == "shadows" else L.hr_ao_default_params)(C.byref(P))
    P.bias = bias
    P.denoise = 0  # MEAN without the FINAL's power: count / N
    return P


def target(rig, kind, scale=0):
    if kind == "reflections":
        t = pyhr.ReflectionsPass(rig.ctx, rig.W, rig.H, scale)
        t.params.sky_color[0], t.params.sky_color[1], t.params.sky_color[2] = SKY
        return t
    return pyhr.Pass(rig.ctx, kind, rig.W, rig.H, scale)


@pytest.mark.parametrize("size", [(64, 48), (97, 53), (7, 3), (1, 1)])
@pytest.mark.parametrize("kind", ["shadows", "ao"])
@pytest.mark.parametrize("bias", [0.05, 0.5])
def test_mask_counts_equal_the_oracle(size, kind, bias):
    W, H = size
    rig = Rig(W, H)
    osc = O.Scene(rig.sc.world_triangles()[0])
    t = target(rig, kind)
    ref = pyhr.ReferencePass(t)
    P = mask_params(kind, bias)
    p0, p1 = (P.bias, 0.0) if kind == "shadows" else (P.ray_length, P.bias)
    count, N = np.zeros((H, W), np.uint32), 0
    O.take_ray_counts()  # drain the oracle's counters
    for n in (3, 29, 64):  # three renders of one frame: the accumulation and the sample index carry over
        f = rig.frame() if N == 0 else rig.f
        ref.render(f, n, params=P)
        R.reference_mask(osc, O.GBufMips(rig.g, 1), f, kind, p0, p1, N, n, count)
        N += n
        m, se = R.mean_and_stderr(count, N)
        sky = rig.g.depth == 1.0
        want = np.where(sky, 1.0 if kind == "ao" else 0.0, m).astype(np.float32).astype(np.float16)
        got = ref.download(pyhr.REFERENCE_OUT_MEAN).view(np.float16)
        assert np.array_equal(got, want), f"{kind} {size} N={N}: counts differ from the oracle"
        np.testing.assert_allclose(f16(ref.download(pyhr.REFERENCE_OUT_STDERR)), np.where(sky, 0.0, se), atol=1e-3)
    st = ref.stats()
    assert (st.rays_primary, st.rays_secondary) == O.take_ray_counts(), "rays traced differ from the oracle's"
    ref.destroy()
    t.destroy()
    rig.close()


@pytest.mark.parametrize("kind", ["shadows", "ao"])
def test_mask_split_and_rows_are_exact(kind):
    rig = Rig(64, 48)
    t = target(rig, kind)
    a, b, c = pyhr.ReferencePass(t), pyhr.ReferencePass(t), pyhr.ReferencePass(t)
    P = mask_params(kind, 0.3)
    f = rig.frame()
    a.render(f, 256, params=P)
    b.render(f, 64, params=P)
    b.render(f, 192, params=P)
    c.render(f, 256, params=P, row0=10, row1=30)
    ma, mb, mc = (x.download(pyhr.REFERENCE_OUT_MEAN).view(np.uint16) for x in (a, b, c))
    assert np.array_equal(ma, mb)
    assert np.array_equal(mc[10:30], ma[10:30])
    assert (mc[:10] == 0).all() and (mc[30:] == 0).all()
    for x in (a, b, c):
        x.destroy()
    t.destroy()
    rig.close()


def _edit_roughness(g):
    """left third mirror (0.02), right third DDGI branch (0.9), the middle as the scene has it"""
    W = g.W
    g.gb3[:, : W // 3, 0] = np.float16(0.02).view(np.uint16)
    g.gb3[:, 2 * W // 3:, 0] = np.float16(0.9).view(np.uint16)


@pytest.mark.parametrize("with_ddgi", [False, True])
def test_reflections_equal_the_oracle_and_k12(with_ddgi):
    W, H = 96, 56
    rig = Rig(W, H)
    ss = O.ShadingScene(rig.sc)
    t = target(rig, "reflections")
    ref = pyhr.ReferencePass(t)
    dd = pyhr.DDGIPass(rig.ctx, W, H, 0) if with_ddgi else None
    odd = None
    if dd:
        dd.params.probe_distance, dd.params.normal_bias = 4.0, 1.0
        dd.params.sky_color[0], dd.params.sky_color[1], dd.params.sky_color[2] = SKY
        mn, mx = rig.sc.bounds()
        odd = O.DDGIOracle(W, H, 0, dd.params, mn, mx)
    for i in range(3):
        f = rig.frame(_edit_roughness)
        if dd:
            rot = pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))
            dd.render(f, rot)
            odd.render(ss, O.GBufMips(rig.g, 1), f, rot)
        t.render(f, dd)
    gi = 1 if with_ddgi else 0
    N = 48
    ref.render(f, N, ddgi=dd)
    acc = R.reference_reflections(ss, O.GBufMips(rig.g, 1), f, t.params, 0, N, np.zeros((H, W, 6), np.float64), sample_gi=gi, approx=gi, ddgi=odd)
    m, se = R.mean_and_stderr(acc, N)
    got = f16(ref.download(pyhr.REFERENCE_OUT_MEAN))
    sky = rig.g.depth == 1.0
    close(got[..., :3], np.where(sky[..., None], 0.0, m).astype(np.float32), "reflections MEAN")
    assert (got[..., 3] == 1.0).all()
    close(f16(ref.download(pyhr.REFERENCE_OUT_STDERR))[..., :3], se.astype(np.float32), "reflections STDERR")
    # mirror and DDGI-branch pixels do not depend on the sample: STDERR 0 and MEAN = this frame's K12 output
    rough = f16(rig.g.gb3)[..., 0]
    det = ~sky & ((rough < 0.05) | ((rough > 0.75) & with_ddgi))
    assert det.any()
    assert (f16(ref.download(pyhr.REFERENCE_OUT_STDERR))[det][:, :3] == 0).all()
    k12 = f16(t.download(0))[..., :3]  # HR_REFLECTIONS_OUT_RAY_TRACE
    assert np.array_equal(got[..., :3][det], k12[det])
    # rows [10, 30) alone equal the whole render's rows bit for bit; the other rows are untouched
    c = pyhr.ReferencePass(t)
    c.render(f, N, ddgi=dd, row0=10, row1=30)
    mc = c.download(pyhr.REFERENCE_OUT_MEAN).view(np.uint16)
    assert np.array_equal(mc[10:30], ref.download(pyhr.REFERENCE_OUT_MEAN).view(np.uint16)[10:30])
    assert (mc[:10] == 0).all() and (mc[30:] == 0).all()
    c.destroy()
    # split invariance of the float64 sums, seen through the fp16 MEAN (the sums themselves are not an output)
    b = pyhr.ReferencePass(t)
    b.render(f, 16, ddgi=dd)
    b.render(f, 32, ddgi=dd)
    np.testing.assert_allclose(f16(b.download(pyhr.REFERENCE_OUT_MEAN)), got, rtol=1e-3, atol=1e-4)
    for x in (b, ref, t) + ((dd,) if dd else ()):
        x.destroy()
    rig.close()


@pytest.mark.parametrize("kind", ["shadows", "ao", "reflections"])
@pytest.mark.parametrize("scale", [0, 1, 2])
def test_final_equals_mean_at_sky_pixels(kind, scale):
    rig = Rig(96, 56)
    t = target(rig, kind, scale)
    ref = pyhr.ReferencePass(t)
    for _ in range(3):
        f = rig.frame()
        t.render(f)
    ref.render(f, 4)
    sky = rig.g.depth == 1.0
    assert sky.any()
    fin = f16(t.download(100))
    mean = f16(ref.download(pyhr.REFERENCE_OUT_MEAN))
    if kind == "shadows" and fin.ndim == 3:
        fin = fin[..., 0]  # RG16F (visibility, variance) at full resolution
    if kind == "reflections":
        fin, mean = fin[..., :3], mean[..., :3]
    assert np.array_equal(fin[sky], mean[sky])
    ref.destroy()
    t.destroy()
    rig.close()


def test_reset_restarts_and_refusals_change_nothing():
    rig = Rig(32, 24)
    t = target(rig, "ao")
    ref = pyhr.ReferencePass(t)
    f = rig.frame()
    ref.render(f, 8)
    first = ref.download(pyhr.REFERENCE_OUT_MEAN).copy()
    ref.render(f, 8)
    ref.reset_history()
    ref.render(f, 8)
    assert np.array_equal(ref.download(pyhr.REFERENCE_OUT_MEAN), first)
    L = rig.ctx.lib
    before = ref.download(pyhr.REFERENCE_OUT_MEAN).copy()
    P = t.params
    bad_nan = mask_params("ao", 0.3)
    bad_nan.ray_length = float("nan")

    def call(r=ref.h, fr=C.byref(f), prm=C.byref(P), samples=8, row0=0, row1=0):
        return L.hr_reference_render(r, fr, prm, None, samples, row0, row1, None)

    for rc in (call(samples=0), call(samples=65537), call(row0=-1), call(row0=10, row1=5), call(row1=25), call(r=None), call(fr=None), call(prm=None),
               call(prm=C.byref(bad_nan))):
        assert rc == -1
    assert np.array_equal(ref.download(pyhr.REFERENCE_OUT_MEAN), before)
    # rows other than those of the first render since the reset
    rr = pyhr.ReferencePass(t)
    rr.render(f, 4, row0=4, row1=12)
    mr = rr.download(pyhr.REFERENCE_OUT_MEAN).copy()
    assert L.hr_reference_render(rr.h, C.byref(f), C.byref(P), None, 4, 0, 0, None) == -1
    assert L.hr_reference_render(rr.h, C.byref(f), C.byref(P), None, 4, 4, 12, None) == 0
    rr.reset_history()
    rr.render(f, 4)  # after a reset any rows
    rr.destroy()
    # a DDGI pass of another context
    other = Rig(32, 24)
    odd = pyhr.DDGIPass(other.ctx, 32, 24, 0)
    assert L.hr_reference_render(ref.h, C.byref(f), C.byref(P), odd.h, 8, 0, 0, None) == -1
    assert np.array_equal(ref.download(pyhr.REFERENCE_OUT_MEAN), before)
    odd.destroy()
    other.close()
    # another kind of target
    h = C.c_void_p()
    dd = pyhr.DDGIPass(rig.ctx, 32, 24, 0)
    assert L.hr_reference_create(dd.h, C.byref(h)) == -1
    assert L.hr_reference_create(None, C.byref(h)) == -1
    # the sample counter stops at 2^32 - 1 (a sky pixel: no rays, so the 65536 renders are cheap)
    small = Rig(1, 1)
    ts = target(small, "ao")
    rs = pyhr.ReferencePass(ts)
    fs = small.frame(lambda g: g.depth.fill(1.0))
    n = 0
    while n + 65536 <= 0xFFFFFFFF:
        assert L.hr_reference_render(rs.h, C.byref(fs), C.byref(ts.params), None, 65536, 0, 0, None) == 0
        n += 65536
    assert L.hr_reference_render(rs.h, C.byref(fs), C.byref(ts.params), None, 0xFFFFFFFF - n, 0, 0, None) == 0
    before = rs.download(pyhr.REFERENCE_OUT_MEAN).copy()
    assert L.hr_reference_render(rs.h, C.byref(fs), C.byref(ts.params), None, 1, 0, 0, None) == -1
    assert np.array_equal(rs.download(pyhr.REFERENCE_OUT_MEAN), before)
    for x in (rs, ts, ref, t, dd):
        x.destroy()
    small.close()
    rig.close()


@pytest.mark.parametrize("kind", ["shadows", "ao"])
def test_blue_noise_mean_of_256_frames_lies_within_the_bound(kind):
    """With a static camera, the mean of one blue-noise period (256 frames) of the pass's own one-ray masks lies within the bound derived
    from the CPU oracle's reference (oracle_reference.blue_noise_bound, checked on the oracle by test_reference_cpu.py)."""
    W, H = 64, 48
    rig = Rig(W, H)
    osc = O.Scene(rig.sc.world_triangles()[0])
    t = target(rig, kind)
    t.params.denoise = 0  # output 0 is the frame's mask
    ref = pyhr.ReferencePass(t)
    P = mask_params(kind, t.params.bias)
    p0, p1 = (P.bias, 0.0) if kind == "shadows" else (P.ray_length, P.bias)
    acc = np.zeros((H, W), np.float64)
    for i in range(256):
        f = pyhr.make_frame(*CAM, W, H, num_frames=i)  # static: the same view, blue-noise sample index i
        if i == 0:
            rig.g = pyhr.write_gbuffer(rig.sc, f, W, H)
            rig.ctx.gbuffer_upload(0, rig.g)
            rig.ctx.gbuffer_upload(1, rig.g)
            ref.render(f, 4096, params=P)
        t.render(f)
        acc += R.unpack_mask(t.download(0), W, H)
    N = 4096
    p, se = R.mean_and_stderr(R.reference_mask(osc, O.GBufMips(rig.g, 1), f, kind, p0, p1, 0, N, np.zeros((H, W), np.uint32)), N)
    surf = rig.g.depth != 1.0
    bound = R.blue_noise_bound(p[surf], se[surf], 256)
    err = float(np.sqrt(np.mean((acc / 256 - f16(ref.download(pyhr.REFERENCE_OUT_MEAN)))[surf] ** 2)))
    assert err <= bound, (err, bound)
    ref.destroy()
    t.destroy()
    rig.close()


@pytest.mark.parametrize("with_ddgi", [False, True])
def test_textured_scene_equals_the_oracle(with_ddgi):
    """material textures bound: the TEX instantiations of the reflections reference against the oracle, and the mask counts"""
    from test_textures_cpu import textured_scene
    W, H = 96, 56
    sc, asc, textures, bindings = textured_scene()
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    ss.set_textures(textures, bindings, asc.primitive_uvs(), asc.primitive_tangent_frames())
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    scene = ctx.build_scene(asc)
    ctx.set_textures(scene, textures, bindings)
    ctx.gbuffer_create(W, H)
    rf = pyhr.ReflectionsPass(ctx, W, H, 0)
    rf.params.sky_color[0], rf.params.sky_color[1], rf.params.sky_color[2] = SKY
    dd = pyhr.DDGIPass(ctx, W, H, 0) if with_ddgi else None
    odd = None
    if dd:
        dd.params.probe_distance, dd.params.normal_bias = 4.0, 1.0
        dd.params.sky_color[0], dd.params.sky_color[1], dd.params.sky_color[2] = SKY
        mn, mx = sc.bounds()
        odd = O.DDGIOracle(W, H, 0, dd.params, mn, mx)
    f = None
    for i in range(3):
        f = pyhr.make_frame(*CAM, W, H, prev=f, num_frames=i)
        ctx.gbuffer_render(f.ping_pong, f)
        g = O.gbuffer_render(ss, f, W, H)
        if dd:
            rot = pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))
            dd.render(f, rot)
            odd.render(ss, O.GBufMips(g, 1), f, rot)
        rf.render(f, dd)
    ref = pyhr.ReferencePass(rf)
    N = 32
    ref.render(f, N, ddgi=dd)
    gi = 1 if with_ddgi else 0
    acc = R.reference_reflections(ss, O.GBufMips(g, 1), f, rf.params, 0, N, np.zeros((H, W, 6), np.float64), sample_gi=gi, approx=gi, ddgi=odd)
    m, se = R.mean_and_stderr(acc, N)
    sky = g.depth == 1.0
    close(f16(ref.download(pyhr.REFERENCE_OUT_MEAN))[..., :3], np.where(sky[..., None], 0.0, m).astype(np.float32), "textured reflections MEAN")
    close(f16(ref.download(pyhr.REFERENCE_OUT_STDERR))[..., :3], se.astype(np.float32), "textured reflections STDERR")
    osc = ss.scene
    for kind in ("shadows", "ao"):
        t = pyhr.Pass(ctx, kind, W, H, 0)
        mr = pyhr.ReferencePass(t)
        P = mask_params(kind, 0.3)
        p0, p1 = (P.bias, 0.0) if kind == "shadows" else (P.ray_length, P.bias)
        mr.render(f, 40, params=P)
        cnt = R.reference_mask(osc, O.GBufMips(g, 1), f, kind, p0, p1, 0, 40, np.zeros((H, W), np.uint32))
        want = np.where(sky, 1.0 if kind == "ao" else 0.0, cnt / 40.0).astype(np.float32).astype(np.float16)
        assert np.array_equal(mr.download(pyhr.REFERENCE_OUT_MEAN).view(np.float16), want), f"textured scene: {kind} counts differ"
        mr.destroy()
        t.destroy()
    for x in (ref, rf) + ((dd,) if dd else ()):
        x.destroy()
    ctx.close()
