"""Every temporal stage under every camera case of camera_cases.py against the CPU oracle: yaw, pitch, roll, dolly, a fast pan
across the left edge, an orbit, a zoom, fields of view 20 and 100, near / far 0.1 / 100 and 4 / 5000, a near plane that clips
geometry, and a cut with and without hr_pass_reset_history (on an odd and an even frame).

The runners and bars are test_gpu_ragged's, unchanged: shadows + AO under check_all (masks, tile flags and history lengths
exact), DDGI + reflections with the DDGIUniforms bytes, probe rays, reflection ray lengths, tile flags and history lengths exact
and the images under `close`; every frame also checks the four G-buffer images (gb2, gb3 and depth at every mip, gb1 at mip 0).
Beyond the chained comparison, each temporal stage is compared in isolation: the oracle's temporal stage is fed the device's
previous-frame history images, and its a-trous, AO blur and upsample stages the device's own input to that stage, so an error
in one kernel is told apart from ulps carried down the chain.  Each case also asserts, from the frames' motion vectors, that it
reaches the reprojection situations it targets (camera_cases.reprojection_counts; printed with -s).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import camera_cases as CC
import oracle as O
import pyhr
from test_gpu_gi_refl import close
from test_gpu_multi import AO, SH, merge_bands
from test_gpu_parity import check_all, f16, rmse
from test_gpu_ragged import SKY, Worst, new_context, run_gi_refl, run_shadows_ao
from widened.test_gpu_taa_tonemap import same_halves, u16

pytestmark = pytest.mark.gpu

W, H = CC.SIZE
P = O.p


def _bounded(got, want, name, r, m):
    """check_all's bar of a stage: RMSE <= r and max-abs <= m"""
    e, d = rmse(got, want), float(np.abs(got - want).max())
    assert e <= r and d <= m, f"{name}: rmse {e:.2e} (bar {r}), max-abs {d:.2e} (bar {m})"


class Reach:
    """the reprojection branches a case reaches: the oracle's branch codes (O.ReprojectCodes) of the isolated K3, K9 and K14 stages,
    worst frame of each, over the frames that read history"""

    def __init__(self, case):
        self.case, self.n = case, {}

    def codes(self, kernel, i, W, H):
        """`with reach.codes("K3", i, W, H):` around that kernel's oracle stage"""
        reach = self

        class _Rec(O.ReprojectCodes):
            def __exit__(self, *exc):
                super().__exit__(*exc)
                if i and i not in reach.case.resets:
                    d = reach.n.setdefault(kernel, {})
                    for k, v in self.counts().items():
                        d[k] = max(d.get(k, 0), v)
        return _Rec(W, H)

    def check(self, kernels):
        print(f"\n[{self.case.id}] reprojection branch pixels: {self.n}")
        for t in self.case.targets:
            k, b = t.split(":")
            if k in kernels:
                got = self.n.get(k, {}).get(b, 0)
                assert got >= CC.MIN_PIXELS, f"{self.case.id}: {k} reaches '{b}' in {got} pixels only"
        if "K14" in kernels:
            for b in ("virtual", "motion"):
                assert self.n["K14"][b] >= CC.MIN_PIXELS, f"{self.case.id}: K14 reaches the {b} reprojection in {self.n['K14'][b]} pixels only"


def _first(case, i):
    return i == 0 or i in case.resets


# ---------------------------------------------------------------------------------------------- shadows + AO
def _sh_ao_isolated(case, reach):
    """before / after hooks: the cut's history reset, then every stage of both chains fed the device's own inputs (the previous
    frame's, or what after.hist holds: a planted history)"""
    hist = {}

    def before(i, f, passes, oracles):
        if i in case.resets:
            for p in passes:
                p.reset_history()
            for o in oracles:
                o.first = True

    def after(i, f, cur_g, prev_g, passes, oracles):
        sh, ao = passes
        osh, oao = oracles
        L = O.lib()
        # ---- shadows temporal (K3), fed the device's feedback image and moments of the previous frame
        gc, gp = cur_g.c(osh.scale), prev_g.c(osh.scale)
        shw, shh = osh.W, osh.H
        prev_img, prev_mom = hist["sh"] if "sh" in hist and i not in case.resets else (np.zeros((shh, shw, 2), np.uint16), np.zeros((shh, shw, 4), np.uint16))
        t, m, tf = np.zeros((shh, shw, 2), np.uint16), np.zeros((shh, shw, 4), np.uint16), np.zeros_like(osh.tile_flags)
        with reach.codes("K3", i, shw, shh):
            L.orc_shadows_temporal(C.byref(gc), C.byref(gp), P(np.ascontiguousarray(sh.download(0))), P(prev_img), P(prev_mom), C.byref(f), osh.params.alpha,
                                   osh.params.moments_alpha, P(t), P(m), P(tf))
        assert np.array_equal(sh.download(6), tf), f"frame {i}: isolated shadows tile flags"
        assert np.array_equal(f16(sh.download(4))[..., 2], O.h2f(m)[..., 2]), f"frame {i}: isolated shadows history length"
        _bounded(f16(sh.download(1)), O.h2f(t), f"frame {i}: isolated shadows temporal", 1e-3, 2e-3)
        # ---- shadows a-trous chain fed the device's temporal output and tile flags
        Q = osh.params
        src, dev_tf = np.ascontiguousarray(sh.download(1)), np.ascontiguousarray(sh.download(6))
        for it in range(Q.filter_iterations):
            dst = np.zeros((shh, shw, 2), np.uint16)
            L.orc_shadows_atrous(C.byref(gc), P(src), P(dev_tf), Q.radius, 1 << it, Q.phi_visibility, Q.phi_normal, Q.sigma_depth,
                                 Q.power if it == Q.filter_iterations - 1 else 0.0, P(dst))
            src = dst
        _bounded(f16(sh.download(2)), O.h2f(src), f"frame {i}: isolated shadows a-trous", 1e-3, 4e-3)
        hist["sh"] = (np.ascontiguousarray(sh.download(5)), np.ascontiguousarray(sh.download(4)))
        # ---- AO temporal (K9), fed the device's colour and length of the previous frame
        gc, gp = cur_g.c(oao.scale), prev_g.c(oao.scale)
        aw, ah = oao.W, oao.H
        prev_c, prev_l = hist["ao"] if "ao" in hist and i not in case.resets else (np.zeros((ah, aw), np.uint16), np.zeros((ah, aw), np.uint16))
        col, ln, tf = np.zeros((ah, aw), np.uint16), np.zeros((ah, aw), np.uint16), np.zeros_like(oao.tile_flags)
        with reach.codes("K9", i, aw, ah):
            L.orc_ao_temporal(C.byref(gc), C.byref(gp), P(np.ascontiguousarray(ao.download(0))), P(prev_c), P(prev_l), C.byref(f), oao.params.alpha, P(col), P(ln), P(tf))
        assert np.array_equal(ao.download(6), tf), f"frame {i}: isolated AO tile flags"
        assert np.array_equal(f16(ao.download(4)), O.h2f(ln)), f"frame {i}: isolated AO history length"
        _bounded(f16(ao.download(1)), O.h2f(col), f"frame {i}: isolated AO temporal", 1e-3, 2e-3)
        # ---- AO blur fed the device's temporal output and tile flags; the upsample fed the device's blur
        zbp = np.array(f.z_buffer_params[:], np.float32)
        dev_t, dev_tf = np.ascontiguousarray(ao.download(1)), np.ascontiguousarray(ao.download(6))
        b0, b1 = np.zeros((ah, aw), np.uint16), np.zeros((ah, aw), np.uint16)
        L.orc_ao_bilateral_blur(C.byref(gc), P(dev_t), P(dev_tf), P(zbp), 1, 0, oao.params.blur_radius, P(b0))
        L.orc_ao_bilateral_blur(C.byref(gc), P(b0), P(dev_tf), P(zbp), 0, 1, oao.params.blur_radius, P(b1))
        _bounded(f16(ao.download(2)), O.h2f(b1), f"frame {i}: isolated AO blur", 1e-3, 4e-3)
        up = np.zeros((oao.H0, oao.W0), np.uint16)
        L.orc_upsample_scalar(C.byref(cur_g.c(0)), C.byref(gc), P(np.ascontiguousarray(ao.download(2))), 1, 1.0, oao.params.power, P(up))
        _bounded(f16(ao.download(100)), O.h2f(up), f"frame {i}: isolated AO upsample", 1e-3, 4e-3)
        hist["ao"] = (np.ascontiguousarray(ao.download(1)), np.ascontiguousarray(ao.download(4)))

    after.hist = hist  # the history the isolated stages read next: {"sh" | "ao" | "rf": (image, aux)}; absent on a first frame
    return before, after


@pytest.mark.parametrize("case", CC.CASES, ids=CC.ids(CC.CASES))
def test_shadows_ao_under_camera(case):
    reach = Reach(case)
    before, after = _sh_ao_isolated(case, reach)
    run_shadows_ao(f"shadows+ao {case.id}", W, H, 0, 1, check=check_all, seq=CC.frames(case, W, H), before=before, after=after, **CC.scene_kw(case))
    reach.check(("K3", "K9"))


# ---------------------------------------------------------------------------------------------- DDGI + reflections
def _refl_isolated(case, reach):
    hist = {}

    def before(i, f, passes, oracles):
        if i in case.resets:  # the reflections pass; the DDGI grid keeps its probes (a cut does not move the scene)
            passes[1].reset_history()
            oracles[1].first = True

    def after(i, f, cur_g, prev_g, passes, oracles):
        dd, rf = passes
        odd, orf = oracles
        L, Q = O.lib(), rf.params
        gc, gp = cur_g.c(orf.scale), prev_g.c(orf.scale)
        # ---- K21 fed the device's own atlases of this frame
        sample = np.zeros((orf.H, orf.W, 4), np.uint16)
        L.orc_ddgi_sample_probe_grid(C.byref(gc), C.byref(f), C.byref(odd.u), P(np.ascontiguousarray(dd.download(2))), P(np.ascontiguousarray(dd.download(3))),
                                     dd.params.gi_intensity, P(sample))
        close(f16(dd.download(4)), O.h2f(sample), f"frame {i} isolated ddgi sample")
        rw, rh = orf.W, orf.H
        first = _first(case, i)
        z = np.zeros((rh, rw, 4), np.uint16)
        prev_t, prev_m = hist["rf"] if "rf" in hist and i not in case.resets else (z, z)
        approx = 1 if (Q.approximate_with_ddgi and dd is not None and not first) else 0
        t, m, tf = np.zeros_like(z), np.zeros_like(z), np.zeros_like(orf.tile_flags)
        with reach.codes("K14", i, rw, rh):
            L.orc_reflections_temporal(C.byref(gc), C.byref(gp), P(np.ascontiguousarray(rf.download(0))), P(prev_t), P(prev_m), C.byref(f), Q.alpha,
                                       Q.moments_alpha, approx, P(t), P(m), P(tf))
        assert np.array_equal(rf.download(6), tf), f"frame {i}: isolated reflections tile flags"
        mo = f16(rf.download(4))
        assert np.array_equal(mo[..., 2], O.h2f(m)[..., 2]), f"frame {i}: isolated reflections history length"
        close(f16(rf.download(1)), O.h2f(t), f"frame {i} isolated reflections temporal")
        close(mo, O.h2f(m), f"frame {i} isolated reflections moments")
        src, dev_tf = np.ascontiguousarray(rf.download(1)), np.ascontiguousarray(rf.download(6))
        for it in range(Q.filter_iterations):
            dst = np.zeros_like(z)
            L.orc_reflections_atrous(C.byref(gc), P(src), P(dev_tf), Q.radius, 1 << it, Q.phi_color, Q.phi_normal, Q.sigma_depth, approx, P(dst))
            src = dst
        close(f16(rf.download(2)), O.h2f(src), f"frame {i} isolated reflections a-trous")
        hist["rf"] = (np.ascontiguousarray(rf.download(1)), np.ascontiguousarray(rf.download(4)))

    after.hist = hist  # the history the isolated stages read next: {"sh" | "ao" | "rf": (image, aux)}; absent on a first frame
    return before, after


@pytest.mark.parametrize("case", CC.CASES, ids=CC.ids(CC.CASES))
def test_ddgi_reflections_under_camera(case):
    """near / far 0.1 / 100 found a K21 bug: it rebuilt P with fused products and an approximate reciprocal of w, where w cancels by
    ~100x near the far plane, and its sample exceeded `close` (max-abs 6.35e-3 against 6e-3 on the H100, a static frame).  K21 now
    rounds P as the reference does, and the case runs under the unchanged bar, K21 also compared alone on the device's atlases."""
    reach = Reach(case)
    before, after = _refl_isolated(case, reach)
    run_gi_refl(f"ddgi+reflections {case.id}", W, H, 0, True, seq=CC.frames(case, W, H), before=before, after=after, **CC.scene_kw(case))
    reach.check(("K14",))


# ---------------------------------------------------------------------------------------------- full-resolution post chain
POST = ["yaw_fast", "dolly_in", "cut", "near0.1_far100"]


@pytest.mark.parametrize("cid", POST)
def test_post_chain_under_camera(cid):
    """deferred combine over the device's pass outputs, TAA over it (reset_every_frame = 0, bit-exact), tone map (test_gpu_ragged's rule)"""
    case = CC.BY_ID[cid]
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    sh, ao, rf, de = pyhr.Pass(ctx, "shadows", W, H, 0), pyhr.Pass(ctx, "ao", W, H, 1), pyhr.ReflectionsPass(ctx, W, H, 1), pyhr.DeferredPass(ctx, W, H)
    rf.params.sky_color[0], rf.params.sky_color[1], rf.params.sky_color[2] = SKY
    de.params.env_color[0], de.params.env_color[1], de.params.env_color[2] = SKY
    taa, tm = pyhr.TAAPass(ctx, W, H), pyhr.TonemapPass(ctx, W, H)
    taa.params.reset_every_frame = 0
    otaa = O.TAAOracle(W, H, reset_every_frame=0)
    w = Worst(f"post chain {cid}")
    prev_j = np.zeros(2, np.float32)
    for i, f in CC.frames(case, W, H):
        j = pyhr.taa_jitter(i, W, H)
        pyhr.apply_jitter(f, j, prev_j)
        prev_j = j
        ctx.gbuffer_render(f.ping_pong, f)
        sh.render(f)
        ao.render(f)
        rf.render(f, None)
        de.render(f, sh, ao, rf, None)
        g = pyhr.GBufferHost(W, H)
        g.gb1 = ctx.gbuffer_download(f.ping_pong, 0, 1, W, H)
        g.gb2 = ctx.gbuffer_download(f.ping_pong, 0, 2, W, H)
        g.gb3 = ctx.gbuffer_download(f.ping_pong, 0, 3, W, H)
        g.depth = ctx.gbuffer_download(f.ping_pong, 0, 0, W, H)
        want = f16(O.deferred(g, f, shadow=sh.download(100), ao=ao.download(100), reflections=rf.download(100), env=SKY))
        got = f16(de.download(100))
        w.add("deferred", got[..., :3], want[..., :3])
        _bounded(got[..., :3], want[..., :3], f"frame {i}: deferred", 1e-3, 2e-2)
        cur = u16(de.download(100))
        taa.render(f, de)
        want_taa = otaa.render(f, cur, g.depth, u16(g.gb2))
        got_taa = u16(taa.download(100))
        assert same_halves(got_taa, want_taa), f"frame {i}: TAA: {np.count_nonzero(got_taa != want_taa)} of {got_taa.size} halves differ"
        assert same_halves(u16(taa.download(0)), otaa.img[1 - f.ping_pong]), f"frame {i}: TAA history image"
        tm.render(taa)
        got8, want8 = tm.download(100), O.tonemap(got_taa)
        d = np.abs(got8.astype(np.int16) - want8.astype(np.int16))
        assert d.max() <= 1 and np.mean(d == 0) >= 0.995, f"frame {i}: tone map max diff {d.max()}, identical {np.mean(d == 0):.4f}"
    w.report()
    for p in (tm, taa, de, rf, sh, ao):
        p.destroy()
    ctx.close()


@pytest.mark.parametrize("cid", ["fov20", "fov100", "near0.1_far100", "near4_far5000", "near_clip"])
def test_path_tracer_primary_hits_under_projection(cid):
    """the path tracer's primary rays come from the frame's inverse projection: its hits are the oracle's, exactly"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ss = O.ShadingScene(sc, brute=True)
    ctx = new_context(sc, W, H)
    pt = pyhr.PathTracerPass(ctx, W, H)
    pt.params.sky_color[0], pt.params.sky_color[1], pt.params.sky_color[2] = SKY
    opt = O.PathTracerOracle(W, H, sky=SKY)
    f = [f for _, f in CC.frames(CC.BY_ID[cid], W, H, n=3)][-1]
    for i in range(2):
        pt.render(f)
        opt.render(ss, f)
        prim = pt.download(1)
        assert np.array_equal(prim, opt.prim), f"sample {i}: primary hits differ in {np.count_nonzero(prim != opt.prim)} pixels"
        assert (prim != 0xFFFFFFFF).mean() > 0.2
    pt.destroy()
    ctx.close()


# ---------------------------------------------------------------------------------------------- sharding under motion
WORLD = 3


def _rank(sc, W, H, rank, world):
    c = pyhr.Context(0)
    c.set_bluenoise(*pyhr.blue_noise())
    c.build_scene(sc)
    c.gbuffer_create(W, H)
    zero = pyhr.GBufferHost(W, H)
    c.gbuffer_upload(0, zero)
    c.gbuffer_upload(1, zero)
    if world > 1:
        c.shard_config(rank, world)
    return c, pyhr.Pass(c, "shadows", W, H, 0), pyhr.Pass(c, "ao", W, H, 1)


def _ranks(sc, W, H):
    ranks = [_rank(sc, W, H, r, WORLD) for r in range(WORLD)]
    for r in range(WORLD):
        for q in range(WORLD):
            if q != r:
                for a, b in zip(ranks[r][1:], ranks[q][1:]):
                    a.link_local(q, b)
    return ranks


def _close_all(sets):
    everyone = [r for s in sets for r in s]
    for c, sh, ao in everyone:
        sh.destroy()
        ao.destroy()
    for c, sh, ao in everyone:
        c.close()


def _owner(rows, H):
    own = np.full(rows.shape, -1)
    for r in range(WORLD):
        b, e = pyhr.shard_rows(H, r, WORLD)
        own[(rows >= b) & (rows < e)] = r
    return own


def _bands_differ(ranks, ref, H):
    """the images whose ranks' bands, merged, differ from the single-rank image"""
    bad = []
    for name, which in (("prev", SH["prev"]), ("moments", SH["moments"]), ("a-trous", SH["atrous"]), ("final", SH["final"])):
        if not np.array_equal(merge_bands([r[1].download(which) for r in ranks], H, WORLD), ref[1].download(which)):
            bad.append(f"shadows {name}")
    ah = O.pass_size(1, H, 1)[1]
    for name, which, shift in (("temporal", AO["temporal"], 0), ("length", AO["length"], 0), ("blur", AO["blur"], 0), ("final", AO["final"], 1)):
        if not np.array_equal(merge_bands([r[2].download(which) for r in ranks], ah, WORLD, shift), ref[2].download(which)):
            bad.append(f"ao {name}")
    return bad


def _render(ranks, f, streams, gbuf):
    """one frame on every rank; gbuf(c, stream) fills the rank's G-buffer slot"""
    for (c, _, _), st in zip(ranks, streams):
        gbuf(c, st.cuda_stream)
    for (c, sh, _), st in zip(ranks, streams):
        sh.render(f, st.cuda_stream)
    for (c, _, ao), st in zip(ranks, streams):
        ao.render(f, st.cuda_stream)
    torch.cuda.synchronize()


def _row_reach(g, H):
    """rows the reprojection of this G-buffer's frame reaches from each pixel into the previous frame's G-buffer: max |motion.y| * H,
    + 2 for the bilinear footprint and the 3x3 fallback (0 when nothing has geometry)"""
    mv = CC.motion(g.gb2)
    geo = (g.depth != 1.0) & np.isfinite(mv).all(-1)
    return int(np.ceil(np.abs(mv[..., 1][geo] * H).max())) + 2 if geo.any() else 0


# pitch 16 degrees a frame: at 250x141 (bands of 48, 48 and 45 rows) some history rows lie on the non-adjacent rank (1 500 pixels over
# the sequence, from the oracle's motion vectors); pitch_fast's 8 degrees and the cut reach the neighbouring band only
MULTI = {"pitch_fast": CC.BY_ID["pitch_fast"], "cut": CC.BY_ID["cut"], "pitch_16": CC.Case("pitch_16", CC.pitch(-16.0), "shadows_test", (), (), ())}


@pytest.mark.parametrize("cid", list(MULTI))
def test_peer_history_under_motion(cid):
    """world 3 at 250x141, ranks emulated on one GPU, the G-buffer uploaded whole: every band of every shadows and AO image is the
    single-rank image bit for bit; on pitch_16 some pixel's history row (from the single-rank motion vectors) is on a non-adjacent rank"""
    W, H = 250, 141
    case = MULTI[cid]
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ref, ranks = _rank(sc, W, H, 0, 1), _ranks(sc, W, H)
    streams = [torch.cuda.Stream() for _ in range(WORLD)]
    non_adjacent = 0
    for i, f in CC.frames(case, W, H):
        g = pyhr.write_gbuffer(sc, f, W, H)
        ref[0].gbuffer_upload(f.ping_pong, g)
        ref[1].render(f)
        ref[2].render(f)
        _render(ranks, f, streams, lambda c, st: c.gbuffer_upload(f.ping_pong, g, st))
        mv = CC.motion(g.gb2)
        geo = (g.depth != 1.0) & np.isfinite(mv).all(-1)
        if i and geo.any():
            hist = np.floor((np.arange(H)[:, None] + mv[..., 1] * H)[geo]).astype(np.int64)
            src = _owner(np.broadcast_to(np.arange(H)[:, None], (H, W))[geo], H)
            inside = (hist >= 0) & (hist < H)
            non_adjacent += int(np.count_nonzero(inside & (np.abs(_owner(np.clip(hist, 0, H - 1), H) - src) > 1)))
        for r in ranks:
            assert np.array_equal(r[1].download(0), ref[1].download(0)), f"frame {i}: shadows mask differs"
            assert np.array_equal(r[2].download(0), ref[2].download(0)), f"frame {i}: AO mask differs"
        bad = _bands_differ(ranks, ref, H)
        assert not bad, f"frame {i}: {bad} differ"
    print(f"\n[{cid}] pixels whose history row is on a non-adjacent rank: {non_adjacent}")
    if cid == "pitch_16":
        assert non_adjacent > 0, "no history read reaches past the neighbouring band"
    _close_all([[ref], ranks])


def _recompute_halo():
    """full-resolution rows beyond its band a rank recomputes for these passes (shadows at full resolution, AO at half: twice its rows)"""
    return max(sum(pyhr.shard_halo_rows("shadows")), 2 * sum(pyhr.shard_halo_rows("ao")))


def test_sharded_gbuffer_halo_under_pitch():
    """hr_gbuffer_render_sharded's contract (hr_api.h): halo_rows must include the recompute halo and the reprojection reach.  World 3
    at 1366x768 (bands of 256 rows, so band +- halo leaves rows stale), fast pitch: the slot rendered at frame i is read as the
    previous G-buffer at frame i + 1, at rows up to frame i + 1's reach away, and the AO chain reads it at up to frame i's own reach,
    so frame i's halo = recompute halo + 8 + the larger of the two reaches, rounded up to 8.  With it every band of every image is the single-rank image bit for bit.  Negative controls: the recompute halo
    alone, and the 64 rows bench.py gives its lateral pan, must differ once the pitch starts."""
    W, H = 1366, 768
    case = CC.BY_ID["pitch_fast"]
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    seq = list(CC.frames(case, W, H))
    gbufs = [pyhr.write_gbuffer(sc, f, W, H) for _, f in seq]
    reach = [_row_reach(g, H) if i else 0 for (i, _), g in zip(seq, gbufs)]
    rec = _recompute_halo()
    # measured on the H100: with the recompute halo + frame i + 1's reach alone, the last frame (which no later frame reads) differed in
    # AO at halos 80 and 88; with 8 rows more and the larger of the two reaches every frame matches.  Which AO read needs the frame's
    # own reach is not pinned down here.
    halos = [-(-(rec + 8 + max(reach[i], reach[i + 1] if i + 1 < len(seq) else 0)) // 8) * 8 for i in range(len(seq))]
    ref = _rank(sc, W, H, 0, 1)
    legs = {"derived": _ranks(sc, W, H), "recompute only": _ranks(sc, W, H), "64 rows": _ranks(sc, W, H)}
    fixed = {"recompute only": -(-rec // 8) * 8, "64 rows": 64}
    streams = [torch.cuda.Stream() for _ in range(WORLD)]
    differs = {k: [] for k in fixed}
    for (i, f), g, halo in zip(seq, gbufs, halos):
        ref[0].gbuffer_upload(f.ping_pong, g)
        ref[1].render(f)
        ref[2].render(f)
        for name, ranks in legs.items():
            h = halo if name == "derived" else fixed[name]
            _render(ranks, f, streams, lambda c, st: c.gbuffer_render_sharded(f.ping_pong, f, h, st))
        bad = _bands_differ(legs["derived"], ref, H)
        assert not bad, f"frame {i}, halo {halo}: {bad} differ"
        for name in fixed:
            differs[name].append(_bands_differ(legs[name], ref, H))
    print(f"\n[1366x768 pitch_fast] recompute halo {rec}, reach per frame {reach}, derived halo per frame {halos}; images that differ per "
          f"frame: {differs}")
    assert max(halos) + 256 + max(halos) < H, "the derived halo leaves stale rows"
    for name in fixed:
        assert any(differs[name]), f"the {name} halo ({fixed[name]}) reproduces the single-rank images under a fast pitch"
    _close_all([[ref]] + list(legs.values()))
