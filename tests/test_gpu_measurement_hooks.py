"""The measurement hooks bench.py builds its headline numbers from, against host restatements (measurement_hooks.py) and the oracle.

- hr_pass_output_checksum: equal to the restatement of hr_api.h's formula over the downloaded bytes, for every output of every pass
  kind in every format (R32_UINT masks, R8_UINT tile flags and count images, R16F, RG16F, RGBA16F, RGBA8), at 256x144 and the ragged
  sizes, scales 0-2, spp 1 and > 1, and one 4K RGBA16F image (the grid-stride loop runs several times); whole images, single rows and
  random splits, which add up to the whole mod 2^64; bad row ranges.  Linked ranks emulated in one process: each rank's own rows add
  up to the single-GPU checksum; images complete on every rank (DDGI atlases, the path tracer's gathered output) equal it.
- hr_pass_get_stats: tiles_denoise = the non-zero flags of the (oracle-exact) tile-flag image, tiles_total / pixels_total from the
  rows the denoise stages covered (band +- hr_shard_halo_rows for sharded ranks), 0 / 0 / 0 after a render with denoise = 0, the
  counts of the last render only; ray counts equal to the oracle's (K1, K7, K12 primary and secondary, K18), accumulated until
  drained, summed over linked ranks, and drained in 64 bits past 2^32.
- hr_pass_stage_times: the documented stage list of each pass and parameter block; windows whose renders record different lists
  report every name once, in first-seen order; more than 1024 undrained renders.  Durations: finite and >= 0, nothing else.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import light_cases as LC
import measurement_hooks as MH
import oracle as O
import pyhr
from test_gpu_parity import check_all
from test_gpu_ragged import CAM_SHADOWS_TEST, SKY, _linked_ranks, frames, new_context, run_gi_refl, run_shadows_ao
from test_gpu_spp import check_counts

pytestmark = pytest.mark.gpu

SIZES = [(256, 144), (250, 141), (251, 144), (7, 3), (1, 1)]
SH_OUTS = {0: (0, 1, 2, 4, 5, 6, 100), 1: (0, 1, 2, 3, 4, 5, 6, 100)}  # by scale > 0: 3 = the full-resolution upsample
AO_OUTS = {0: (0, 1, 2, 4, 6, 100), 1: (0, 1, 2, 3, 4, 6, 100)}
RF_OUTS = {0: (0, 1, 2, 4, 6, 100), 1: (0, 1, 2, 3, 4, 6, 100)}


def _raw(p, which):
    """the output's bytes as the device holds them: (H, W) or (H, W, C) of 1-, 2- or 4-byte channels"""
    return np.ascontiguousarray(p.download(which))


def check_checksums(p, whichs, rng, what):
    """device checksum == restatement: whole image, every row of images up to 64 rows (6 random rows of taller ones), and a random
    3- and 5-way split whose device sums add up to the whole mod 2^64"""
    for which in whichs:
        a = _raw(p, which)
        H = a.shape[0]
        whole = MH.checksum(a)
        got = p.checksum(which)
        assert got == whole, f"{what}: checksum of output {which} ({a.dtype} {a.shape}) {got:#x}, restatement {whole:#x}"
        rows = range(H) if H <= 64 else sorted(set(int(y) for y in rng.integers(0, H, size=6)))
        for y in rows:
            assert p.checksum(which, y, y + 1) == MH.checksum(a, y, y + 1), f"{what}: output {which} row {y}"
        for k in (3, 5):
            cuts = MH.random_cuts(rng, H, k)
            parts = [p.checksum(which, a0, b0) for a0, b0 in zip(cuts[:-1], cuts[1:]) if b0 > a0]
            assert sum(parts) & MH.M64 == whole, f"{what}: output {which} split at {cuts} does not add up"


def counted(o, log):
    """make the oracle `o` log the (primary, secondary) rays each of its renders casts"""
    inner = o.render

    def render(*a, **k):
        O.take_ray_counts()
        r = inner(*a, **k)
        log.append(O.take_ray_counts())
        return r
    o.render = render


def check_tile_stats(s, p, o, W, H, what, row0=0, row1=None):
    """tiles_denoise = the device flags over the covered rows = the oracle's; tiles_total / pixels_total from those rows"""
    flags = p.download(6)
    want = MH.tile_counts(flags, W, H, row0, row1)
    got = (s.tiles_total, s.tiles_denoise, s.pixels_total)
    assert got == want, f"{what}: (tiles_total, tiles_denoise, pixels_total) {got}, restatement {want}"
    if o is not None:
        assert s.tiles_denoise == np.count_nonzero(o.tile_flags), f"{what}: the oracle flags {np.count_nonzero(o.tile_flags)} tiles"
    if row1 is None:
        assert (s.tiles_total, s.pixels_total) == (((W + 7) // 8) * ((H + 7) // 8), W * H)


# ---------------------------------------------------------------------------------------------- shadows + AO on one GPU
def _sh_ao_hooks(spp, scale, W, H, reset_at=2):
    rng = np.random.default_rng(W * 1000 + H + 17 * spp + scale)
    logs = ([], [])

    def before(i, f, passes, oracles):
        if i == 0:
            for o, log in zip(oracles, logs):
                o.spp = spp
                counted(o, log)
        if i == reset_at:
            for p in passes:
                p.reset_history()
            for o in oracles:
                o.first = True

    def after(i, f, cur_g, prev_g, passes, oracles):
        sh, ao = passes
        for p, o, log, name in zip(passes, oracles, logs, ("shadows", "ao")):
            what = f"{name} {W}x{H} scale {scale} spp {spp} frame {i}"
            s = p.stats()
            assert s.renders == 1
            assert (s.rays_primary, s.rays_secondary) == log[-1], f"{what}: device rays {(s.rays_primary, s.rays_secondary)}, oracle {log[-1]}"
            pw, ph = O.pass_size(W, H, scale)
            if o.params.denoise:
                check_tile_stats(s, p, o, pw, ph, what)
            else:
                assert (s.tiles_total, s.tiles_denoise, s.pixels_total) == (0, 0, 0), f"{what}: denoise off"
            outs = (SH_OUTS if name == "shadows" else AO_OUTS)[int(scale > 0)] if o.params.denoise else (0, 100)
            check_checksums(p, outs, rng, what)
    return before, after


@pytest.mark.parametrize("spp", [1, 3])
@pytest.mark.parametrize("scale", [0, 1, 2])
@pytest.mark.parametrize("W,H", SIZES)
def test_shadows_ao_hooks(W, H, scale, spp):
    """checksums of every output, tile and pixel counts and ray counts after every frame: 2 static frames, a reset, a pan"""
    before, after = _sh_ao_hooks(spp, scale, W, H)
    run_shadows_ao(f"hooks shadows+ao {W}x{H} scale {scale} spp {spp}", W, H, scale, scale, sh_params=dict(spp=spp), ao_params=dict(spp=spp), n=4,
                   pan_from=3, check=check_all if spp == 1 else check_counts, before=before, after=after)


@pytest.mark.parametrize("case", ["iter0", "spp41", "spp255"])
def test_shadows_ao_hooks_parameters(case):
    """filter_iterations 0 (the tile flags come from the temporal stage alone), and sample counts 41 and 255 with a vertical pan"""
    W, H = (250, 141) if case != "spp255" else (64, 45)
    spp = {"spp41": 41, "spp255": 255}.get(case, 1)
    sh_p, ao_p = dict(spp=spp), dict(spp=spp)
    if case == "iter0":
        sh_p["filter_iterations"] = 0
    before, after = _sh_ao_hooks(spp, 0, W, H)
    run_shadows_ao(f"hooks shadows+ao {case}", W, H, 0, 0, sh_params=sh_p, ao_params=ao_p, n=4, pan_from=3, vertical=0.35,
                   check=check_all if spp == 1 else check_counts, before=before, after=after)


@pytest.mark.parametrize("light", ["point_high", "point_low", "spot_band", "spot_away", "sun_below", "sun_grazing"])
def test_shadow_ray_counts_under_lights(light):
    """K1 traces no ray where the light's attenuation is 0 (outside a spot's cone, behind the surface): the counts still equal the
    oracle's, at spp 1 and 3"""
    case = LC.BY_ID[light]
    for spp in (1, 3):
        before, after = _sh_ao_hooks(spp, 0, 250, 141)
        run_shadows_ao(f"hooks lights {light} spp {spp}", 250, 141, 0, 0, sh_params=dict(spp=spp), ao_params=dict(spp=spp), n=2,
                       check=check_all if spp == 1 else check_counts, before=before, after=after, **LC.scene_kw(case))


# ---------------------------------------------------------------------------------------------- DDGI + reflections
# (reflections parameters, with DDGI, DDGI parameters, light case, the light reaches no hit point: no secondary ray in K12).  The sun
# straight below (rot_x 180 degrees) still lights the walls facing one way by a rounding-sized N.L > 0, so K12 casts shadow rays
# there, as the oracle does; a spot pointing up lights nothing.
REFL_CASES = {
    "spp1": (dict(spp=1), False, None, None, False),
    "spp3": (dict(spp=3), False, None, None, False),
    "spp1_ddgi": (dict(spp=1), True, None, None, False),
    "spp3_ddgi": (dict(spp=3), True, None, None, False),
    "ddgi_layout_33_rays": (dict(spp=1), True, dict(rays_per_probe=33, irradiance_oct_size=6, depth_oct_size=14), None, False),
    "sun_below_ddgi": (dict(spp=1), True, None, "sun_below", False),
    "spot_away_ddgi": (dict(spp=3), True, None, "spot_away", True),
    "half_res_iter1": (dict(spp=1, filter_iterations=1), True, None, None, False),
}


@pytest.mark.parametrize("case", list(REFL_CASES))
def test_ddgi_reflections_hooks(case):
    params, with_ddgi, ddgi_params, light, unlit = REFL_CASES[case]
    scale = 1 if case == "half_res_iter1" else 0
    W, H = 250, 141
    rng = np.random.default_rng(7)
    logs = {"ddgi": [], "refl": []}

    def before(i, f, passes, oracles):
        if i == 0:
            odd, orf = oracles
            counted(orf, logs["refl"])
            if odd is not None:
                counted(odd, logs["ddgi"])

    def after(i, f, cur_g, prev_g, passes, oracles):
        dd, rf = passes
        what = f"reflections {case} frame {i}"
        s = rf.stats()
        assert s.renders == 1
        assert (s.rays_primary, s.rays_secondary) == logs["refl"][-1], f"{what}: device rays {(s.rays_primary, s.rays_secondary)}, oracle {logs['refl'][-1]}"
        assert s.rays_primary > 0
        if unlit:
            assert s.rays_secondary == 0, f"{what}: the light reaches no surface, yet {s.rays_secondary} shadow rays"
        pw, ph = O.pass_size(W, H, scale)
        check_tile_stats(s, rf, oracles[1], pw, ph, what)
        check_checksums(rf, RF_OUTS[scale], rng, what)
        if dd is not None:
            d = dd.stats()
            u = dd.uniforms()
            probes = u.probe_counts[0] * u.probe_counts[1] * u.probe_counts[2]
            assert d.rays_primary == probes * u.rays_per_probe
            assert (d.rays_primary, d.rays_secondary) == logs["ddgi"][-1], f"ddgi {case} frame {i}: device {(d.rays_primary, d.rays_secondary)}, oracle {logs['ddgi'][-1]}"
            assert (d.tiles_total, d.tiles_denoise, d.pixels_total, d.renders) == (0, 0, 0, 1)
            check_checksums(dd, (0, 1, 2, 3, 4, 100), rng, f"ddgi {case} frame {i}")

    run_gi_refl(f"hooks {case}", W, H, scale, with_ddgi, params=params, n=3, pan_from=2, ddgi_params=ddgi_params,
                light=None if light is None else LC.light(LC.BY_ID[light]), before=before, after=after)


# ---------------------------------------------------------------------------------------------- the other passes, 4K, bad arguments
@pytest.mark.parametrize("W,H", [(250, 141), (7, 3), (1, 1)])
def test_post_and_path_tracer_checksums(W, H):
    """deferred (RGBA16F), TAA (both images), tone map (RGBA8), the path tracer (colour and R32_UINT primitives, the path hash with
    trace_indirect) and their ray counts"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    rng = np.random.default_rng(3)
    sh, ao, de = pyhr.Pass(ctx, "shadows", W, H, 0), pyhr.Pass(ctx, "ao", W, H, 1), pyhr.DeferredPass(ctx, W, H)
    taa, tm, pt = pyhr.TAAPass(ctx, W, H), pyhr.TonemapPass(ctx, W, H), pyhr.PathTracerPass(ctx, W, H)
    de.params.env_color[0], de.params.env_color[1], de.params.env_color[2] = SKY
    pt.params.sky_color[0], pt.params.sky_color[1], pt.params.sky_color[2] = SKY
    for i, f in frames(W, H, 3, pan_from=2):
        ctx.gbuffer_render(f.ping_pong, f)
        sh.render(f)
        ao.render(f)
        de.render(f, sh, ao, None, None)
        taa.render(f, de)
        tm.render(taa)
        pt.params.trace_indirect = i % 2
        pt.render(f)
        torch.cuda.synchronize()
        for p, outs, name in ((de, (100,), "deferred"), (taa, (0, 100), "taa"), (tm, (100,), "tonemap"), (pt, (0, 1, 100) + ((2,) if i % 2 else ()), "path tracer")):
            check_checksums(p, outs, rng, f"{name} {W}x{H} frame {i}")
        s = pt.stats()
        assert s.renders == 1 and s.rays_primary == W * H, f"path tracer: {s.rays_primary} primary rays for {W * H} pixels"
    for p in (pt, tm, taa, de, ao, sh):
        p.destroy()
    ctx.close()


def test_checksum_4k_rgba16f():
    """3840 x 2160 RGBA16F (8.3 M texels against 296 x 256 threads): the deferred combine of the 4K frame"""
    W, H = 3840, 2160
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    de = pyhr.DeferredPass(ctx, W, H)
    de.params.env_color[0], de.params.env_color[1], de.params.env_color[2] = SKY
    f = pyhr.make_frame(*CAM_SHADOWS_TEST, W, H)
    ctx.gbuffer_render(f.ping_pong, f)
    de.render(f, None, None, None, None)
    a = _raw(de, 100)
    assert a.shape == (H, W, 4) and len(np.unique(a.reshape(-1, 4), axis=0)) > 100
    whole = MH.checksum(a)
    assert de.checksum(100) == whole
    assert (de.checksum(100, 0, 1001) + de.checksum(100, 1001, H)) & MH.M64 == whole
    assert de.checksum(100, 2159, 2160) == MH.checksum(a, 2159, 2160)
    de.destroy()
    ctx.close()


def test_checksum_row_range_arguments():
    W, H = 250, 141
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    sh = pyhr.Pass(ctx, "shadows", W, H, 0)
    f = pyhr.make_frame(*CAM_SHADOWS_TEST, W, H)
    ctx.gbuffer_render(f.ping_pong, f)
    sh.render(f)
    v = C.c_uint64()

    def rc(which, r0, r1):
        return sh.lib.hr_pass_output_checksum(sh.h, which, r0, r1, C.byref(v), C.c_void_p(0))

    for which, h in ((100, H), (0, (H + 3) // 4), (6, (H + 7) // 8)):
        for r0, r1 in ((-1, 5), (0, h + 1), (7, 3), (h + 1, h + 2)):
            assert rc(which, r0, r1) == -1, f"output {which}: rows [{r0}, {r1}) accepted"  # HR_ERR_INVALID_ARG
        whole = sh.checksum(which)
        for r0, r1 in ((0, 0), (5, 0), (0, -3), (h - 1, -1)):
            assert rc(which, r0, r1) == 0 and v.value == whole, f"output {which}: row1 = {r1} is not the whole image"
        assert rc(which, 3, 3) == 0 and v.value == 0
        assert rc(which, h, h) == 0 and v.value == 0
    sh.destroy()
    ctx.close()


# ---------------------------------------------------------------------------------------------- tile counts: the last render only
@pytest.mark.parametrize("kind", ["shadows", "ao", "reflections"])
def test_tile_counts_describe_the_last_render(kind):
    """two renders across a cut, one stats call: the counts of the second; then denoise = 0 after a denoised render reports 0 / 0 / 0
    (the flags of the earlier render stay in the image)"""
    W, H = 250, 141
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    p = pyhr.ReflectionsPass(ctx, W, H, 0) if kind == "reflections" else pyhr.Pass(ctx, kind, W, H, 0)

    def render(f):
        ctx.gbuffer_render(f.ping_pong, f)
        p.render(f, None) if kind == "reflections" else p.render(f)

    a = pyhr.make_frame(*CAM_SHADOWS_TEST, W, H)
    b = pyhr.make_frame((0.0, 6.0, 2.0), (0.0, 0.0, 0.0), W, H, prev=a, num_frames=1)  # a cut: every history tap is rejected
    render(a)
    torch.cuda.synchronize()
    fa = np.count_nonzero(p.download(6))
    render(b)
    s = p.stats()
    fb = np.count_nonzero(p.download(6))
    assert fa != fb, "the two renders flag as many tiles: the case cannot tell them apart"
    assert s.renders == 2
    assert (s.tiles_total, s.tiles_denoise, s.pixels_total) == MH.tile_counts(p.download(6), W, H), f"{kind}: {fa} / {fb} flagged, stats {s.tiles_denoise}"
    assert fb > 0
    p.params.denoise = 0
    render(pyhr.make_frame(*CAM_SHADOWS_TEST, W, H, prev=b, num_frames=2))
    s = p.stats()
    assert (s.tiles_total, s.tiles_denoise, s.pixels_total) == (0, 0, 0), f"{kind} with denoise = 0: stats {s.tiles_total} / {s.tiles_denoise} / {s.pixels_total}"
    assert s.renders == 1 and s.rays_primary > 0
    p.destroy()
    ctx.close()


# ---------------------------------------------------------------------------------------------- ray counters: accumulation and the drain
def test_ray_counts_accumulate_until_drained():
    W, H = 250, 141
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    ao = pyhr.Pass(ctx, "ao", W, H, 0)
    ao.params.denoise = 0
    f = pyhr.make_frame(*CAM_SHADOWS_TEST, W, H)
    ctx.gbuffer_render(f.ping_pong, f)
    geo = int(np.count_nonzero(ctx.gbuffer_download(f.ping_pong, 0, 0, W, H) != 1.0))
    for spp, n in ((1, 3), (7, 2)):
        ao.params.spp = spp
        for _ in range(n):
            ao.render(f)
        s = ao.stats()
        assert (s.rays_primary, s.rays_secondary, s.renders) == (n * spp * geo, 0, n)
        s = ao.stats()
        assert (s.rays_primary, s.rays_secondary, s.renders) == (0, 0, 0), "a second drain reads what the first one took"
    ao.destroy()
    ctx.close()


def test_ray_counter_drain_past_2_pow_32():
    """AO at full resolution, 1920x1080, spp 255, 9 renders without a drain: 9 * 255 * (pixels on geometry) rays, more than 2^32, and
    each of the 32 counter slots passes 2^16"""
    W, H, spp, n = 1920, 1080, 255, 9
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    ao = pyhr.Pass(ctx, "ao", W, H, 0)
    ao.params.denoise, ao.params.spp = 0, spp
    f = pyhr.make_frame((0.0, 6.0, 2.0), (0.0, 0.0, 0.0), W, H)  # looking down at the floor: geometry in every pixel
    ctx.gbuffer_render(f.ping_pong, f)
    geo = int(np.count_nonzero(ctx.gbuffer_download(f.ping_pong, 0, 0, W, H) != 1.0))
    want = n * spp * geo
    assert want > 2**32 and want // 32 > 2**16
    ao.stats()
    for _ in range(n):
        ao.render(f)
    s = ao.stats()
    assert s.renders == n
    assert s.rays_primary == want, f"{s.rays_primary} rays counted, {want} traced ({s.rays_primary - want:+d}; 2^32 = {2**32})"
    ao.destroy()
    ctx.close()


# ---------------------------------------------------------------------------------------------- linked ranks
def _make_sh_ao(sc, W, H):
    def make(rank, world):
        c = pyhr.Context(0)
        c.set_bluenoise(*pyhr.blue_noise())
        c.build_scene(sc)
        c.gbuffer_create(W, H)
        if world > 1:
            c.shard_config(rank, world)
        return c, pyhr.Pass(c, "shadows", W, H, 0), pyhr.Pass(c, "ao", W, H, 1)
    return make


@pytest.mark.parametrize("world", [2, 3])
def test_linked_ranks_own_rows_add_up(world):
    """shadows (full resolution) and AO (half resolution, upsampled) on linked ranks at 250x141: each rank's checksum of its own rows
    of the final output, and of its band of the history images, sum to the single-GPU checksum; ray counts sum to the single-GPU
    count; the tile counts cover the band +- the denoise halo"""
    W, H = 250, 141
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ref, ranks = _linked_ranks(_make_sh_ao(sc, W, H), world)
    streams = [torch.cuda.Stream() for _ in range(world)]
    ao_h = O.pass_size(W, H, 1)[1]
    halo = {"shadows": pyhr.shard_halo_rows("shadows", 1, 4, 4)[0], "ao": pyhr.shard_halo_rows("ao", 1, 4, 4)[0]}
    for _, f in frames(W, H, 4, pan_from=2, vertical=0.35):
        g = pyhr.write_gbuffer(sc, f, W, H)
        ref[0].gbuffer_upload(f.ping_pong, g)
        ref[1].render(f)
        ref[2].render(f)
        for (c, sh, ao), st in zip(ranks, streams):
            c.gbuffer_upload(f.ping_pong, g, st.cuda_stream)
        for (c, sh, ao), st in zip(ranks, streams):
            sh.render(f, st.cuda_stream)
        for (c, sh, ao), st in zip(ranks, streams):
            ao.render(f, st.cuda_stream)
        torch.cuda.synchronize()
        for j, name, ph in ((1, "shadows", H), (2, "ao", ao_h)):
            rp = ref[j]
            s_ref = rp.stats()
            assert rp.checksum(100) == MH.checksum(_raw(rp, 100))
            scale = 0 if name == "shadows" else 1
            outs = [(100, scale)] + ([(5, 0), (4, 0)] if name == "shadows" else [(4, 0), (1, 0)])
            for which, shift in outs:
                parts = []
                for r in range(world):
                    a, b = MH.own_rows(ph, r, world, shift, H)
                    parts.append(ranks[r][j].checksum(which, a, b) if b > a else 0)
                assert sum(parts) & MH.M64 == rp.checksum(which), f"{name} output {which} frame {f.num_frames}: own rows do not add up (world {world})"
            prim = 0
            for r in range(world):
                p = ranks[r][j]
                s = p.stats()
                prim += s.rays_primary
                r0, r1 = MH.denoise_rows(ph, r, world, halo[name])
                pw = O.pass_size(W, H, scale)[0]
                assert (s.tiles_total, s.tiles_denoise, s.pixels_total) == MH.tile_counts(p.download(6), pw, ph, r0, r1), \
                    f"{name} rank {r}/{world} frame {f.num_frames}: rows [{r0}, {r1})"
            assert prim == s_ref.rays_primary, f"{name} frame {f.num_frames}: ranks trace {prim} rays, one GPU {s_ref.rays_primary}"
    for c, sh, ao in [ref] + ranks:
        sh.destroy()
        ao.destroy()
    for c, sh, ao in [ref] + ranks:
        c.close()


@pytest.mark.parametrize("world", [2, 3])
def test_linked_ranks_complete_outputs_match(world):
    """outputs complete on every linked rank: the path tracer's gathered frame (gather on) and the DDGI atlases; every rank's whole
    checksum equals the single-GPU one and the restatement, ray counts sum to the single-GPU counts.  With the gather off, the
    path tracer's own 8-row chunks of every rank add up to the single-GPU frame"""
    W, H = 250, 141
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    mn, mx = sc.bounds()

    def make(rank, world):
        c = pyhr.Context(0)
        c.set_bluenoise(*pyhr.blue_noise())
        c.build_scene(sc)
        c.gbuffer_create(W, H)
        if world > 1:
            c.shard_config(rank, world)
        pt, dd = pyhr.PathTracerPass(c, W, H), pyhr.DDGIPass(c, W, H, 0)
        pt.params.sky_color[0], pt.params.sky_color[1], pt.params.sky_color[2] = SKY
        dd.params.probe_distance = 4.0
        return c, pt, dd

    ref, ranks = _linked_ranks(make, world)
    streams = [torch.cuda.Stream() for _ in range(world)]
    for i, f in frames(W, H, 4, pan_from=2):
        gather = i < 2
        for c, *_ in ranks:
            c.shard_set_gather(int(gather))
        rot = pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))
        ref[0].gbuffer_render(f.ping_pong, f)
        ref[1].render(f)
        ref[2].render(f, rot)
        for (c, pt, dd), st in zip(ranks, streams):
            c.gbuffer_render(f.ping_pong, f, stream=st.cuda_stream)
        for (c, pt, dd), st in zip(ranks, streams):
            pt.render(f, st.cuda_stream)
        for (c, pt, dd), st in zip(ranks, streams):
            dd.render(f, rot, st.cuda_stream)
        torch.cuda.synchronize()
        want_pt = ref[1].checksum(100)
        assert want_pt == MH.checksum(_raw(ref[1], 100))
        if gather:
            for r in range(world):
                assert ranks[r][1].checksum(100) == want_pt, f"path tracer rank {r}/{world} frame {i}: gathered frame differs"
        else:
            chunks = [(y, min(y + 8, H)) for y in range(0, H, 8)]
            total = sum(ranks[(k % world)][1].checksum(100, a, b) for k, (a, b) in enumerate(chunks))
            assert total & MH.M64 == want_pt, f"path tracer frame {i}: the ranks' own chunks do not add up (world {world})"
        for which in (2, 3):
            want = ref[2].checksum(which)
            assert want == MH.checksum(_raw(ref[2], which))
            for r in range(world):
                assert ranks[r][2].checksum(which) == want, f"ddgi atlas {which} rank {r}/{world} frame {i}"
        for j in (1, 2):
            s_ref = ref[j].stats()
            got = [ranks[r][j].stats() for r in range(world)]
            assert sum(s.rays_primary for s in got) == s_ref.rays_primary
            assert sum(s.rays_secondary for s in got) == s_ref.rays_secondary
    for c, pt, dd in [ref] + ranks:
        pt.destroy()
        dd.destroy()
    for c, *_ in [ref] + ranks:
        c.close()


# ---------------------------------------------------------------------------------------------- stage timings
def _times(p):
    t = p.stage_times()
    for name, ms in t:
        assert math.isfinite(ms) and ms >= 0.0, f"stage {name}: {ms} ms"
    return [n for n, _ in t]


def _ctx_profiled(W, H, sc=None):
    sc = sc or pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    ctx.set_profiling(1)
    return ctx


SH_LISTS = [  # (pass, scale, params)
    ("shadows", 0, dict()), ("shadows", 1, dict()), ("shadows", 2, dict(filter_iterations=0)), ("shadows", 1, dict(filter_iterations=6, feedback_iteration=5)),
    ("shadows", 0, dict(denoise=0)), ("shadows", 1, dict(spp=3)), ("shadows", 1, dict(spp=3, denoise=0)),
    ("ao", 0, dict()), ("ao", 1, dict()), ("ao", 2, dict(spp=5)), ("ao", 1, dict(denoise=0)),
    ("reflections", 0, dict()), ("reflections", 1, dict(filter_iterations=2)), ("reflections", 1, dict(denoise=0)), ("reflections", 0, dict(spp=3)),
]


@pytest.mark.parametrize("kind,scale,params", SH_LISTS, ids=[f"{k}-s{s}-{'-'.join(f'{a}{b}' for a, b in p.items()) or 'default'}" for k, s, p in SH_LISTS])
def test_stage_names_per_pass(kind, scale, params):
    """a one-render window gives the documented stage list, on every render"""
    W, H = 250, 141
    ctx = _ctx_profiled(W, H)
    p = pyhr.ReflectionsPass(ctx, W, H, scale) if kind == "reflections" else pyhr.Pass(ctx, kind, W, H, scale)
    for k, v in params.items():
        setattr(p.params, k, v)
    P = p.params
    if kind == "shadows":
        want = MH.shadows_stages(P.filter_iterations, P.denoise, scale)
    elif kind == "ao":
        want = MH.ao_stages(P.denoise, scale)
    else:
        want = MH.reflections_stages(P.filter_iterations, P.denoise, scale)
    for i, f in frames(W, H, 3, pan_from=1):
        ctx.gbuffer_render(f.ping_pong, f)
        p.render(f, None) if kind == "reflections" else p.render(f)
        assert _times(p) == want, f"render {i}"
    assert _times(p) == []  # read: the window is empty
    p.destroy()
    ctx.close()


def test_stage_names_other_passes():
    """DDGI, deferred, TAA (the reset blit on every render as the reference has it, on the first only with reset_every_frame = 0),
    tone map, path tracer"""
    W, H = 250, 141
    ctx = _ctx_profiled(W, H)
    dd, de, taa, tm, pt = pyhr.DDGIPass(ctx, W, H, 0), pyhr.DeferredPass(ctx, W, H), pyhr.TAAPass(ctx, W, H), pyhr.TonemapPass(ctx, W, H), pyhr.PathTracerPass(ctx, W, H)
    taa2 = pyhr.TAAPass(ctx, W, H)
    taa2.params.reset_every_frame = 0
    dd.params.probe_distance = 4.0
    for i, f in frames(W, H, 3, pan_from=1):
        ctx.gbuffer_render(f.ping_pong, f)
        dd.render(f, pyhr.rotation_matrix(0.3 * i, (0.0, 1.0, 0.0)))
        de.render(f, None, None, None, dd)
        taa.render(f, de)
        taa2.render(f, de)
        tm.render(taa)
        pt.render(f)
        assert _times(dd) == MH.ddgi_stages()
        assert _times(de) == MH.DEFERRED_STAGES
        assert _times(taa) == MH.taa_stages(True)
        assert _times(taa2) == MH.taa_stages(i == 0), f"render {i}"
        assert _times(tm) == MH.TONEMAP_STAGES
        assert _times(pt) == MH.path_tracer_stages()
    for p in (taa2, pt, tm, taa, de, dd):
        p.destroy()
    ctx.close()


def test_stage_names_sharded():
    """world 2 with hr_shard_config: the gather's "Exchange" mark (on or off); linked ranks: the cooperative trace's "Mask Exchange
    Wait", DDGI's atlas stages, the path tracer's "Gather Wait\""""
    W, H, world = 250, 141, 2
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)

    def make(rank, world):
        c = pyhr.Context(0)
        c.set_bluenoise(*pyhr.blue_noise())
        c.build_scene(sc)
        c.gbuffer_create(W, H)
        c.set_profiling(1)
        if world > 1:
            c.shard_config(rank, world)
        sh, dd, pt = pyhr.Pass(c, "shadows", W, H, 1), pyhr.DDGIPass(c, W, H, 0), pyhr.PathTracerPass(c, W, H)
        dd.params.probe_distance = 4.0
        return c, sh, dd, pt

    # unlinked rank 0 of 2: no peer waits, the gather mark follows the render when the gather is on
    c, sh, dd, pt = make(0, world)
    for gather in (1, 0):
        c.shard_set_gather(gather)
        f = pyhr.make_frame(*CAM_SHADOWS_TEST, W, H)
        c.gbuffer_render(f.ping_pong, f)
        sh.render(f)
        assert _times(sh) == MH.shadows_stages(4, 1, 1, exchange=bool(gather)), f"gather {gather}"
    for p in (pt, dd, sh):
        p.destroy()
    c.close()
    ref, ranks = _linked_ranks(make, world)
    streams = [torch.cuda.Stream() for _ in range(world)]
    for i, f in frames(W, H, 2, pan_from=1):
        for (c, sh, dd, pt), st in zip(ranks, streams):
            c.gbuffer_render(f.ping_pong, f, stream=st.cuda_stream)
        for (c, sh, dd, pt), st in zip(ranks, streams):
            sh.render(f, st.cuda_stream)
        for (c, sh, dd, pt), st in zip(ranks, streams):
            dd.render(f, pyhr.rotation_matrix(0.3 * i, (0.0, 1.0, 0.0)), st.cuda_stream)
        for (c, sh, dd, pt), st in zip(ranks, streams):
            pt.render(f, st.cuda_stream)
        torch.cuda.synchronize()
        for c, sh, dd, pt in ranks:
            assert _times(sh) == MH.shadows_stages(4, 1, 1, linked=True, exchange=True)
            assert _times(dd) == MH.ddgi_stages(linked=True, world=world)
            assert _times(pt) == MH.path_tracer_stages(gather_wait=True)
    for c, sh, dd, pt in [ref] + ranks:
        for p in (pt, dd, sh):
            p.destroy()
    for c, *_ in [ref] + ranks:
        c.close()


def test_stage_times_mixed_windows():
    """windows whose renders record different stage lists report the union of the lists, each name once, in first-seen order; a
    one-render window of each list gives that list"""
    W, H = 250, 141
    ctx = _ctx_profiled(W, H)
    seq = list(frames(W, H, 6, pan_from=1))
    # TAA, reset_every_frame = 0: the window of its first render, then one that starts without the blit and has a reset in it
    de, taa = pyhr.DeferredPass(ctx, W, H), pyhr.TAAPass(ctx, W, H)
    taa.params.reset_every_frame = 0
    lists = []
    for i, f in seq:
        if i == 3:
            taa.reset_history()
        ctx.gbuffer_render(f.ping_pong, f)
        de.render(f, None, None, None, None)
        taa.render(f, de)
        lists.append(MH.taa_stages(i in (0, 3)))
        if i == 1:
            assert _times(taa) == MH.union_names(lists) == ["Reset Blit", "TAA"]
            lists = []
    assert _times(taa) == MH.union_names(lists) == ["TAA", "Reset Blit"]
    # reflections at half resolution whose filter_iterations change inside the window
    rf = pyhr.ReflectionsPass(ctx, W, H, 1)
    lists = []
    for (i, f), it in zip(seq, (1, 4, 0, 2, 1, 3)):
        rf.params.filter_iterations = it
        ctx.gbuffer_render(f.ping_pong, f)
        rf.render(f, None)
        lists.append(MH.reflections_stages(it, 1, 1))
    want = MH.union_names(lists)
    assert want == ["Ray Trace", "Temporal Accumulation", "A-Trous 0", "Upsample", "A-Trous 1", "A-Trous 2", "A-Trous 3"]
    assert _times(rf) == want
    for (i, f), it in zip(seq[:2], (0, 3)):
        rf.params.filter_iterations = it
        rf.render(f, None)
        assert _times(rf) == MH.reflections_stages(it, 1, 1)
    for p in (rf, taa, de):
        p.destroy()
    ctx.close()
    # shadows with the gather switched inside the window (rank 0 of 2, hr_shard_config)
    ctx = _ctx_profiled(W, H)
    ctx.shard_config(0, 2)
    sh = pyhr.Pass(ctx, "shadows", W, H, 1)
    lists = []
    for (i, f), gather in zip(seq, (0, 1, 0, 0, 1, 1)):
        ctx.shard_set_gather(gather)
        ctx.gbuffer_render(f.ping_pong, f)
        sh.render(f)
        lists.append(MH.shadows_stages(4, 1, 1, exchange=bool(gather)))
    assert _times(sh) == MH.union_names(lists) == MH.shadows_stages(4, 1, 1, exchange=True)
    sh.destroy()
    ctx.close()


def test_stage_times_past_1024_undrained_renders():
    """1100 profiled TAA renders without a read keep the last 1024 records: a window that starts without the reset blit and holds
    three resets reports "TAA" then "Reset Blit", once each"""
    W, H = 16, 8
    ctx = _ctx_profiled(W, H)
    de, taa = pyhr.DeferredPass(ctx, W, H), pyhr.TAAPass(ctx, W, H)
    taa.params.reset_every_frame = 0
    f = pyhr.make_frame(*CAM_SHADOWS_TEST, W, H)
    ctx.gbuffer_render(f.ping_pong, f)
    de.render(f, None, None, None, None)
    for i in range(1100):
        if i in (300, 700, 1090):
            taa.reset_history()
        taa.render(f, de)
    assert _times(taa) == ["TAA", "Reset Blit"]
    taa.destroy()
    de.destroy()
    ctx.close()
