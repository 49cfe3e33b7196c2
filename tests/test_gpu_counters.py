"""GPU parity at large sample counts, past the history-length cap and across the frame counter's wraps (cases in counter_cases.py,
the oracle's side checked on the CPU by test_counters_cpu.py).

- Sample counts 3..255 (shadows + AO at two scale pairs, reflections with and without DDGI) over 5 frames with a pan and a cut that
  resets the histories, so frames blending with alpha >= 0.5 occur after frame 0 too; counts, tile flags and history lengths
  exact, images under test_gpu_spp's bars (check_counts) or `close`.  spp 41 / 47 reach an AO tile whose geometry pixels all
  have count == spp on such a frame, spp 3 an open 17x17 window: the two places where count / spp and the window mean must be
  exact quotients.  The blue-noise slot a count selects, and linked ranks at spp 3 and 255 (bit-identical to one GPU).
- Histories past their 32-frame cap: 48 frames of shadows + AO (1 and 2 spp), 40 of DDGI + reflections, every frame under the
  existing bars with the device's history length at min(32, frames of history), and a 300-frame static run at 64x48 whose worst
  errors are printed per 50 frames (-s).
- Frame counters from 250, 2^31 - 3, 2^32 - 3 (wrapping to 0) and, for spp 255 and 4, where num_frames * spp crosses 2^31:
  shadows + AO, DDGI + reflections and the deferred -> TAA -> tone map chain against the oracle; without the oracle, the device's
  mask or count image at frame N equals the one at N mod 256.
"""
import numpy as np
import pytest
import torch

import counter_cases as K
import oracle as O
import pyhr
from test_gpu_multi import frames as multi_frames
from test_gpu_multi_spp import Group, _check_shadows_ao
from test_gpu_parity import check_all, f16
from test_gpu_ragged import Worst, measure_sh_ao, new_context, run_gi_refl, run_post_chain, run_shadows_ao
from test_gpu_spp import check_counts

pytestmark = pytest.mark.gpu


def _spp_hooks(spp, reset_at=None, after=None):
    """before: the oracles take the pass's spp (the device passes get it through sh_params / ao_params) and the cut resets every
    history; after: `after`, if given"""
    def before(i, f, passes, oracles):
        if i == 0:
            for o in oracles:
                o.spp = spp
        if i == reset_at:
            for p in passes:
                p.reset_history()
            for o in oracles:
                o.first = True
    return before, after


def _check_for(spp):
    return check_all if spp == 1 else check_counts


# ---------------------------------------------------------------------------------------------- A. sample counts
@pytest.mark.parametrize("sh_scale,ao_scale", K.SCALES_SH_AO)
@pytest.mark.parametrize("spp,W,H", K.SPP_SH_AO, ids=[f"spp{s}" for s, _, _ in K.SPP_SH_AO])
def test_shadows_ao_sample_counts(spp, W, H, sh_scale, ao_scale):
    reach = {"full_tiles": 0, "open": 0}

    def after(i, f, cur_g, prev_g, passes, oracles):
        osh, oao = oracles
        depth = cur_g.levels[ao_scale][4][:oao.H, :oao.W]
        reach["full_tiles"] += K.full_count_tiles(oao.count, depth, O.h2f(oao.cur_length), spp)
        if i > 0 and i != K.CUT_AT:  # the window mean is only read where history is
            reach["open"] += K.open_windows(osh.count, spp) + K.open_windows(oao.count, spp)

    before, after = _spp_hooks(spp, K.CUT_AT, after)
    run_shadows_ao(f"shadows+ao spp {spp} {W}x{H} scales {sh_scale}/{ao_scale}", W, H, sh_scale, ao_scale, sh_params=dict(spp=spp), ao_params=dict(spp=spp),
                   seq=K.spp_frames(W, H), check=_check_for(spp), before=before, after=after)
    print(f"[spp {spp}] AO tiles of count == spp at alpha >= 0.5: {reach['full_tiles']}, open 17x17 windows: {reach['open']}")
    if spp in (41, 47) and (sh_scale, ao_scale) == (0, 1):
        assert reach["full_tiles"] > 0, "no AO tile with every geometry pixel at count == spp blends with alpha >= 0.5"
    if spp == 3:
        assert reach["open"] > 0, "no all-open 17x17 window on a frame that reads history"


@pytest.mark.parametrize("with_ddgi", [False, True], ids=["plain", "ddgi"])
@pytest.mark.parametrize("spp,W,H", K.SPP_REFL, ids=[f"spp{s}" for s, _, _ in K.SPP_REFL])
def test_reflections_sample_counts(spp, W, H, with_ddgi):
    """ray length exact, every other image under `close`; the cut resets the reflections' history (the DDGI grid keeps its probes)"""
    def before(i, f, passes, oracles):
        if i == K.CUT_AT:
            passes[1].reset_history()
            oracles[1].first = True

    run_gi_refl(f"reflections spp {spp} {W}x{H}{' ddgi' if with_ddgi else ''}", W, H, 0, with_ddgi, params=dict(spp=spp), seq=K.spp_frames(W, H), before=before)


def test_blue_noise_slot_by_sample_count():
    """bn_table (hr_api.cu): a power-of-two count 2^k reads slot k once it is set, any other count the 1-spp table.  Slots 1, 2 and 7
    are set to tables of their own: spp 3 equals the oracle run with the 1-spp table, spp 128 the run with slot 7's"""
    W, H = 128, 96
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    tri, _ = sc.world_triangles()
    osc = O.Scene(tri, brute=False)
    sobol, base = pyhr.blue_noise(1234)
    slots = {k: pyhr.blue_noise(100 + k)[1] for k in (1, 2, 7)}
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(sobol, base)
    for k, sr in slots.items():
        ctx.set_bluenoise_slot(k, sr)
    ctx.build_scene(sc)
    ctx.gbuffer_create(W, H)
    f = pyhr.make_frame(*K.CAM, W, H)
    g = pyhr.write_gbuffer(sc, f, W, H)
    ctx.gbuffer_upload(f.ping_pong, g)
    cur = O.GBufMips(g)
    for spp, want_table, other in ((3, base, slots[2]), (128, slots[7], base)):
        sh = pyhr.Pass(ctx, "shadows", W, H, 0)
        sh.params.spp, sh.params.denoise = spp, 0
        sh.render(f)
        got = sh.download(0)
        sh.destroy()
        want = []
        for sr in (want_table, other):
            o = O.ShadowsOracle(W, H, 0, spp=spp)
            o.params.denoise = 0
            o.render(osc, cur, cur, f, (sobol, sr))
            want.append(o.count.copy())
        assert np.array_equal(got, want[0]), f"spp {spp}: the count image is not the one of its blue-noise table"
        assert not np.array_equal(want[0], want[1])
    ctx.close()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("spp", K.SPP_LINKED)
def test_linked_ranks_sample_counts_bit_identical(spp, world):
    """cooperative trace at counts away from powers of two (cost_shift = 6 + ceil(log2 spp)): count images complete on every rank,
    merged history bands and outputs equal to world 1"""
    W, H = 256, 144
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    g = Group(sc, world, 0, 1, spp)
    try:
        for f in multi_frames(6, pan_from=2, vertical=0.35):
            g.render(f, pyhr.write_gbuffer(sc, f, W, H))
            _check_shadows_ao(g, f, H, H >> 1, 0, 1, f", spp={spp}")
    finally:
        g.close()


# ---------------------------------------------------------------------------------------------- B. histories past the cap
def _history_after(kind_of):
    """after hook (the lengths are compared with the oracle's by the runner's check): the device's longest history is i + 1 frames
    on the static frames before the pan, then 32 on every frame from 31 on, never more"""
    def after(i, f, cur_g, prev_g, passes, oracles):
        for name, ln in kind_of(passes):
            top = float(ln.max())
            if i < 36:
                assert top == min(K.HIST_CAP, i + 1), f"frame {i}: {name} history length reaches {top}"
            if i >= K.HIST_CAP - 1:
                assert top == K.HIST_CAP, f"frame {i}: {name} history length {top}, not {K.HIST_CAP}"
            assert top <= K.HIST_CAP
    return after


def _sh_ao_lengths(passes):
    sh, ao = passes
    return (("shadows", f16(sh.download(4))[..., 2]), ("ao", f16(ao.download(4))))


@pytest.mark.parametrize("spp", [1, 2])
def test_shadows_ao_history_past_cap(spp):
    W, H = 256, 144
    before, _ = _spp_hooks(spp)
    run_shadows_ao(f"shadows+ao 48 frames spp {spp}", W, H, 0, 1, sh_params=dict(spp=spp), ao_params=dict(spp=spp), seq=K.history_frames(W, H),
                   check=_check_for(spp), before=before, after=_history_after(_sh_ao_lengths))


def test_ddgi_reflections_history_past_cap():
    """40 frames at 128x72; DDGI's hysteresis 1.0 from frame 2 keeps the atlas where the first frames put it (the default 0.98
    drifts 2 % a frame), as param_cases does for its long case"""
    W, H = 128, 72

    def ddgi_hook(i, f, rot, dd, odd, fresh):
        if i == 2:
            dd.params.hysteresis = 1.0
        return odd

    def lengths(passes):
        return (("reflections", f16(passes[1].download(4))[..., 2]),)

    run_gi_refl("ddgi+reflections 40 frames", W, H, 0, True, seq=K.history_frames(W, H, 40), ddgi_hook=ddgi_hook, after=_history_after(lengths))


def test_shadows_ao_long_static_run():
    """K.LONG_STATIC static frames at 64x48: alpha = 1/32 feeds the a-trous output back for hundreds of frames and penumbra values
    decay toward fp16 subnormals.  Every frame under check_all; the worst error of each stage per 50 frames is printed"""
    W, H = 64, 48
    windows = {}

    def after(i, f, cur_g, prev_g, passes, oracles):
        w = windows.setdefault(i // 50, Worst(f"frames {50 * (i // 50)}..{50 * (i // 50) + 49}"))
        measure_sh_ao(w, *passes, *oracles)

    run_shadows_ao(f"shadows+ao {K.LONG_STATIC} static frames", W, H, 0, 1, seq=K.frames(W, H, K.LONG_STATIC), after=_both(after, _history_after(_sh_ao_lengths)))
    for k in sorted(windows):
        windows[k].report()


def _both(a, b):
    def hook(*args):
        a(*args)
        b(*args)
    return hook


# ---------------------------------------------------------------------------------------------- C. frame counters
def _starts(spp_filter=None):
    cases = [c for c in K.COUNTER_STARTS if spp_filter is None or spp_filter(c[2])]
    return pytest.mark.parametrize("start,spp", [c[1:] for c in cases], ids=[c[0] for c in cases])


def _counter_size(spp):
    return (128, 72) if spp > 4 else (256, 144)


@_starts()
def test_shadows_ao_frame_counter(start, spp):
    W, H = _counter_size(spp)
    before, _ = _spp_hooks(spp)
    run_shadows_ao(f"shadows+ao from frame {start} spp {spp}", W, H, 0, 1, sh_params=dict(spp=spp), ao_params=dict(spp=spp),
                   seq=K.frames(W, H, 5, start, pan=(3, 4)), check=_check_for(spp), before=before)


@_starts()
def test_ddgi_reflections_frame_counter(start, spp):
    """K18 seeds its RNG with num_frames, K12 draws its GGX sample index from it"""
    W, H = 128, 72
    run_gi_refl(f"ddgi+reflections from frame {start} spp {spp}", W, H, 0, True, params=dict(spp=spp), seq=K.frames(W, H, 5, start, pan=(3, 4)))


@_starts(lambda spp: spp == 1)
def test_post_chain_frame_counter(start, spp):
    """TAA jitters by num_frames % 16 (the Halton table), across the 256, 2^31 and 2^32 wraps"""
    W, H = 256, 144
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    run_post_chain(f"post chain from frame {start}", ctx, W, H, K.frames(W, H, 5, start, pan=(2, 3, 4)))
    ctx.close()


@pytest.mark.parametrize("kind", ["shadows", "ao"])
@pytest.mark.parametrize("spp,n", K.MOD256, ids=[f"spp{s}-{n}" for s, n in K.MOD256])
def test_mask_at_frame_n_equals_frame_n_mod_256(spp, n, kind):
    """no oracle: with a static camera the device's mask (spp 1) or count image at frame N is the one at N mod 256, and not the
    one at the next frame"""
    W, H = _counter_size(spp)
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    p = pyhr.Pass(ctx, kind, W, H, 0)
    p.params.spp, p.params.denoise = spp, 0
    out = []
    for nf in (n, n % 256, (n + 1) % 256):
        f = pyhr.make_frame(*K.CAM, W, H, num_frames=nf)
        ctx.gbuffer_render(f.ping_pong, f)
        p.render(f)
        torch.cuda.synchronize()
        out.append(p.download(0).copy())
    p.destroy()
    ctx.close()
    assert np.array_equal(out[0], out[1]), f"{kind} spp {spp}: frame {n} differs from frame {n % 256}"
    assert not np.array_equal(out[1], out[2])
