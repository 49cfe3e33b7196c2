"""Every hit-shading kernel instantiation against the oracle, on the material-texture edge cases of tests/texture_cases.py.

Each case runs through the C ABI at 96x56 and 128x72 with brute-force oracle scenes, under the bars the untextured tests use:
  * the G-buffer producer: all four images and the mips bit for bit;
  * the reflections ray trace (K12) in all three forms at scales 0 and 1: spp 1 without the DDGI terms, spp 1 with sample_gi /
    approximate_with_ddgi, spp 2 (with the DDGI terms) and 4 (without); ray lengths exact, colours within `close`, and the temporal, a-trous and upsample stages
    downstream under the bars of test_gpu_gi_refl.py;
  * the DDGI probe ray trace (K18): directions and hit distances exact, radiance within `close`;
  * the path tracer in both modes: primary hits (and in the indirect mode the path hashes) exact, images under the widened bars;
  * the reflections reference with both GI settings: MEAN and STDERR against the oracle's.
The whole case runs under torch.profiler, which proves that it launched the instantiations texture_cases.HIT_SHADING names it for.
Rebinding (no normal map, then the first one, a rebuild with them bound, another set, none) and the refused material tables are tested
at the end.
Run with -s to print the worst RMSE / max-abs error of every stage per case.
"""
import ctypes as C

import numpy as np
import pytest

import oracle as O
import oracle_reference as R
import pt_indirect as PI
import pyhr
import texture_cases as TC
from test_gpu_gi_refl import close
from test_gpu_ragged import Worst, kernels_launched
from widened.test_gpu_trace_ground_truth import compare as compare_path_traced

pytestmark = pytest.mark.gpu

SIZES = [(96, 56), (128, 72)]
W, H = SIZES[0]
SKY = (0.3, 0.4, 0.6)
# (label, spp, with DDGI, scale): the three K12 forms, each at scales 0 and 1
REFLECTIONS = [("k12 spp1", 1, False, 0), ("k12 spp1", 1, False, 1), ("k12 gi", 1, True, 0), ("k12 gi", 1, True, 1),
               ("k12 spp2", 2, True, 0), ("k12 spp2", 2, True, 1), ("k12 spp4", 4, False, 0), ("k12 spp4", 4, False, 1)]
N_FRAMES = 2  # the DDGI terms are forced off on a pass's first frame


def f16(a):
    return np.ascontiguousarray(a).view(np.float16).astype(np.float32)


def frame_at(i, prev, W=W, H=H):
    return pyhr.make_frame((0.05 * i, 14.0, 34.0), (0.0, 3.0, 0.0), W, H, prev=prev, num_frames=i)


def oracle_scene(case):
    ss = O.ShadingScene(case.sc, brute=True)
    if case.textures:
        ss.set_textures(case.textures, case.bindings, case.vuv(), case.vtb())
    return ss


def run_case(case, worst, W, H):
    ss = oracle_scene(case)
    bn = pyhr.blue_noise()
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*bn)
    scene = ctx.build_scene(case.asc)
    if case.textures:
        ctx.set_textures(scene, case.textures, case.bindings)
    ctx.gbuffer_create(W, H)
    zero = pyhr.GBufferHost(W, H)
    ctx.gbuffer_upload(0, zero)
    ctx.gbuffer_upload(1, zero)
    mn, mx = case.sc.bounds()
    dd = pyhr.DDGIPass(ctx, W, H, 0)
    dd.params.probe_distance, dd.params.normal_bias = 4.0, 1.0
    dd.params.sky_color[0], dd.params.sky_color[1], dd.params.sky_color[2] = SKY
    odd = O.DDGIOracle(W, H, 0, dd.params, mn, mx)
    rfs = []
    for label, spp, gi, scale in REFLECTIONS:
        rf = pyhr.ReflectionsPass(ctx, W, H, scale)
        rf.params.spp = spp
        rf.params.sky_color[0], rf.params.sky_color[1], rf.params.sky_color[2] = SKY
        rfs.append((f"{label} scale {scale}", gi, rf, O.ReflectionsOracle(W, H, scale, rf.params)))
    pt = pyhr.PathTracerPass(ctx, W, H)
    pt.params.sky_color[0], pt.params.sky_color[1], pt.params.sky_color[2] = SKY
    opt = O.PathTracerOracle(W, H, sky=SKY)
    f, prev_g, frames = None, O.zero_gbuf_mips(W, H), []
    for i in range(N_FRAMES):
        f = frame_at(i, f, W, H)
        frames.append(f)
        # G-buffer producer: bit for bit, mips included
        ctx.gbuffer_render(f.ping_pong, f)
        g = O.gbuffer_render(ss, f, W, H)
        for which, want in ((0, g.depth), (1, g.gb1), (2, g.gb2), (3, g.gb3)):
            got = ctx.gbuffer_download(f.ping_pong, 0, which, W, H)
            assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8)), \
                f"{case.name} frame {i}: G-buffer image {which}, {np.count_nonzero(got != want)} values differ"
        cur_g = O.GBufMips(g)
        for mip in (1, 2):
            _, _, r2, r3, rd = cur_g.levels[mip]
            for which, want in ((0, rd), (2, r2), (3, r3)):
                assert np.array_equal(ctx.gbuffer_download(f.ping_pong, mip, which, W, H), want), f"{case.name} frame {i}: G-buffer mip {mip} image {which}"
        # K18
        rot = pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))
        dd.render(f, rot)
        odd.render(ss, cur_g, f, rot)
        dird = dd.download(1).view(np.uint16)
        assert np.array_equal(dird, odd.dirdepth.reshape(dird.shape)), f"{case.name} frame {i}: probe ray direction / hit distance"
        rad_c, rad_o = f16(dd.download(0)), O.h2f(odd.radiance).reshape(-1, odd.u.rays_per_probe, 4)
        worst.add("k18 radiance", rad_c, rad_o)
        close(rad_c, rad_o, f"{case.name} frame {i} ddgi radiance", 2e-3, 0.05)
        # K12 in its three forms, and the denoise chain downstream
        for name, gi, rf, orf in rfs:
            what = f"{case.name} {W}x{H} frame {i} {name}"
            rf.render(f, dd if gi else None)
            orf.render(ss, cur_g, prev_g, f, bn, odd if gi else None)
            rt_c, rt_o = f16(rf.download(0)), O.h2f(orf.rt)
            assert np.array_equal(rt_c[..., 3], rt_o[..., 3]), f"{what}: reflection ray length"
            worst.add(name, rt_c[..., :3], rt_o[..., :3])
            close(rt_c[..., :3], rt_o[..., :3], f"{what} ray trace", 1e-3, 0.02)
            assert np.array_equal(rf.download(6), orf.tile_flags), f"{what}: tile classification"
            close(f16(rf.download(1)), O.h2f(orf.cur_temporal), f"{what} temporal")
            mo_c, mo_o = f16(rf.download(4)), O.h2f(orf.cur_moments)
            assert np.array_equal(mo_c[..., 2], mo_o[..., 2]), f"{what}: history length"
            close(mo_c, mo_o, f"{what} moments")
            worst.add(name + " a-trous", f16(rf.download(2)), O.h2f(orf.atrous_out))
            close(f16(rf.download(2)), O.h2f(orf.atrous_out), f"{what} a-trous")
            worst.add(name + " final", f16(rf.download(100)), O.h2f(orf.final))
            close(f16(rf.download(100)), O.h2f(orf.final), f"{what} final")
        prev_g = cur_g
        # path tracer, the reference as written
        pt.render(f)
        want = opt.render(ss, f)
        assert np.array_equal(pt.download(1), opt.prim), f"{case.name} frame {i}: path tracer primary hits"
        worst.add("path tracer", f16(pt.download(100))[..., :3], f16(want)[..., :3])
        compare_path_traced(f16(pt.download(100)), f16(want), f"{case.name} frame {i} path tracer")
    # path tracer, indirect mode (3 path vertices): primary hits and path hashes exact, images under the same bars
    pti = pyhr.PathTracerPass(ctx, W, H)
    pti.params.sky_color[0], pti.params.sky_color[1], pti.params.sky_color[2] = SKY
    pti.params.max_ray_bounces, pti.params.trace_indirect = 3, 1
    opti = PI.IndirectPathTracerOracle(W, H, max_ray_bounces=3, sky=SKY)
    for i, fr in enumerate(frames):
        pti.render(fr)
        want = opti.render(ss, fr)
        assert np.array_equal(pti.download(1), opti.prim), f"{case.name} indirect sample {i}: primary hits"
        assert np.array_equal(pti.download(2), opti.hash), f"{case.name} indirect sample {i}: paths differ in {np.count_nonzero(pti.download(2) != opti.hash)} pixels"
        worst.add("path tracer indirect", f16(pti.download(100))[..., :3], f16(want)[..., :3])
        compare_path_traced(f16(pti.download(100)), f16(want), f"{case.name} indirect sample {i}")
    pti.destroy()
    # the reflections reference, with and without the DDGI terms, on the last frame's G-buffer
    g_last = O.GBufMips(g, 1)
    for name, gi, rf, orf in rfs:
        if rf.params.spp != 1 or orf.scale != 0:
            continue
        ref = pyhr.ReferencePass(rf)
        n = 16
        ref.render(f, n, ddgi=dd if gi else None)
        acc = R.reference_reflections(ss, g_last, f, rf.params, 0, n, np.zeros((H, W, 6), np.float64), sample_gi=int(gi), approx=int(gi), ddgi=odd if gi else None)
        m, se = R.mean_and_stderr(acc, n)
        sky = g.depth == 1.0
        got = f16(ref.download(pyhr.REFERENCE_OUT_MEAN))
        worst.add(f"reference {name}", got[..., :3], np.where(sky[..., None], 0.0, m))
        close(got[..., :3], np.where(sky[..., None], 0.0, m).astype(np.float32), f"{case.name} reference {name} MEAN")
        close(f16(ref.download(pyhr.REFERENCE_OUT_STDERR))[..., :3], se.astype(np.float32), f"{case.name} reference {name} STDERR")
        ref.destroy()
    for _, _, rf, _ in rfs:
        rf.destroy()
    pt.destroy()
    dd.destroy()
    ctx.close()


@pytest.mark.parametrize("case", TC.CASES)
def test_textured_kernels_match_the_oracle(case):
    c = TC.build(case)
    got = set()
    for w, h in SIZES:
        worst = Worst(f"{case} {w}x{h}")
        got |= TC.instantiations("\n".join(kernels_launched(lambda: run_case(c, worst, w, h))))
        worst.report()
    # the ledger names one case per instantiation; every textured case runs the same stages, so it launches all the TEX ones
    mine = {k for k, v in TC.HIT_SHADING.items() if v.startswith("test_gpu_textured_kernels.py::") and TC.textured(k) == (case != "untextured")}
    assert len(mine) == 9 and mine <= got, f"{case}: instantiations this case did not launch: {sorted(mine - got)}"
    if case != "untextured":  # a scene with textures never reaches an untextured hit-shading kernel
        assert all(TC.textured(k) for k in got if not k.startswith("k_reference_mask")), sorted(got)


@pytest.mark.parametrize("kind", ["shadows", "ao"])
def test_ledger_mask_references_launch(kind):
    """the k_reference_mask instantiations are compared with the oracle by test_gpu_reference.py; prove that the named case launches them"""
    import test_gpu_reference as T
    want = {k for k, v in TC.HIT_SHADING.items() if v == "test_gpu_reference.py::test_mask_counts_equal_the_oracle" and k.endswith(("<0>", "<1>")[kind == "ao"])}
    assert len(want) == 1
    names = kernels_launched(lambda: T.test_mask_counts_equal_the_oracle((64, 48), kind, 0.05))
    assert want <= TC.instantiations("\n".join(names))


def test_rebinding_textures():
    """hr_scene_set_textures without a normal map, then with one (the first upload of the tangent frames), then another set, then none;
    then hr_scene_rebuild: every state renders the G-buffer and K12 (spp 1, no DDGI) of the oracle with the same bindings"""
    c = TC.build("normal_maps")
    other = TC.build("channels")
    ctx = pyhr.Context(0)
    bn = pyhr.blue_noise()
    ctx.set_bluenoise(*bn)
    scene = ctx.build_scene(c.asc)
    ctx.gbuffer_create(W, H)
    zero = pyhr.GBufferHost(W, H)
    ctx.gbuffer_upload(0, zero)
    ctx.gbuffer_upload(1, zero)
    rf = pyhr.ReflectionsPass(ctx, W, H, 0)
    rf.params.sky_color[0], rf.params.sky_color[1], rf.params.sky_color[2] = SKY
    rf.params.denoise = 0
    no_normal = [{k: v for k, v in b.items() if k != "normal"} for b in c.bindings]
    # "rebuilt": hr_scene_rebuild while the normal-map set is bound (a per-frame TLAS rebuild), rendered without binding again: the
    # textures, the tangent frames and the material table must survive it
    states = [("no normal map", c.textures, no_normal), ("normal maps", c.textures, c.bindings), ("rebuilt", c.textures, c.bindings),
              ("another set", other.textures, other.bindings), ("none", [], [])]
    f = None
    for i, (label, textures, bindings) in enumerate(states):
        if label == "rebuilt":
            ctx.check(ctx.lib.hr_scene_rebuild(scene, None), "hr_scene_rebuild")
        else:
            ctx.set_textures(scene, textures, bindings)
        ss = O.ShadingScene(c.sc, brute=True)
        if textures:
            ss.set_textures(textures, bindings, c.vuv(), c.vtb())
        f = frame_at(i, f)
        ctx.gbuffer_render(f.ping_pong, f)
        g = O.gbuffer_render(ss, f, W, H)
        for which, want in ((0, g.depth), (1, g.gb1), (2, g.gb2), (3, g.gb3)):
            got = ctx.gbuffer_download(f.ping_pong, 0, which, W, H)
            assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8)), f"{label}: G-buffer image {which}"
        orf = O.ReflectionsOracle(W, H, 0, rf.params)
        rf.reset_history()
        rf.render(f, None)
        orf.render(ss, O.GBufMips(g), O.zero_gbuf_mips(W, H), f, bn, None)
        rt_c, rt_o = f16(rf.download(0)), O.h2f(orf.rt)
        assert np.array_equal(rt_c[..., 3], rt_o[..., 3]), f"{label}: reflection ray length"
        close(rt_c[..., :3], rt_o[..., :3], f"{label} ray trace", 1e-3, 0.02)
    rf.destroy()
    ctx.close()


def _build(ctx, asc, n_materials=None):
    v, i, inst, m = asc.raw()
    out = C.c_void_p()
    nm = asc.n_materials if n_materials is None else n_materials
    rc = ctx.lib.hr_scene_build(ctx.h, C.c_void_p(v), C.c_size_t(asc.n_vertices), C.c_void_p(i), C.c_size_t(asc.n_indices), C.c_void_p(inst),
                                C.c_size_t(asc.n_instances), C.c_void_p(m) if nm else None, C.c_size_t(nm), C.byref(out))
    return rc, out


def test_material_index_out_of_range_is_refused():
    """hr_scene_build refuses an instance whose material_idx is not below n_materials (no scene comes back, nothing is rendered);
    without materials the index is not read and the scene is legal, but every render that shades hits refuses it"""
    c = TC.build("untextured")
    ctx = pyhr.Context(0)
    for bad in (c.asc.n_materials, c.asc.n_materials + 255, 0xFFFFFFFF):
        keep = c.asc.inst[5].material_idx
        c.asc.inst[5].material_idx = bad
        rc, out = _build(ctx, c.asc)
        assert rc == -1 and not out.value, (bad, rc)  # HR_ERR_INVALID_ARG
        assert b"material_idx" in ctx.lib.hr_last_error(ctx.h)
        c.asc.inst[5].material_idx = keep
    rc, out = _build(ctx, c.asc)
    assert rc == 0 and out.value
    ctx.check(ctx.lib.hr_scene_destroy(out))
    # no materials: legal, any material_idx; the shading renders refuse the scene, the path tracer included
    c.asc.inst[5].material_idx = 1000
    rc, out = _build(ctx, c.asc, n_materials=0)
    assert rc == 0 and out.value
    ctx.check(ctx.lib.hr_scene_set_current(ctx.h, out))
    ctx.set_bluenoise(*pyhr.blue_noise())
    ctx.gbuffer_create(W, H)
    pt = pyhr.PathTracerPass(ctx, W, H)
    f = frame_at(0, None)
    with pytest.raises(pyhr.HrError, match="without materials"):
        pt.render(f)
    assert pt.stats().renders == 0
    pt.destroy()
    ctx.check(ctx.lib.hr_scene_destroy(out))
    ctx.close()
