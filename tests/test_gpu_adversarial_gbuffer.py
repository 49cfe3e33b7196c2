"""Every G-buffer consumer on the hand-built G-buffers of gbuffer_cases.py against the CPU oracle fed the same arrays: plane distances
and normal dot^2 within ulps of PLANE_DISTANCE / NORMAL_DISTANCE, history coordinates on the frame edges, bilinear weights around
the sumw cut, mesh ids that differ by one fp16 step, sky / geometry patterns, octahedral fold lines, roughness around 0.05 / 0.75,
equal depths, positions on a DDGI probe-cell plane, and histories planted through hr_pass_upload (colours 0 / 1, lengths up to the
32-frame cap).  Each frame's G-buffer enters through hr_gbuffer_upload.

The runners and bars are test_gpu_ragged's and test_gpu_camera's, unchanged: check_all for shadows + AO (masks, tile flags and
history lengths exact), DDGI + reflections with reflection ray lengths, tile flags and history lengths exact, the G-buffer mips
compared bit for bit, every temporal stage also compared in isolation on the device's own history (test_gpu_camera), and TAA bit
for bit.  A last test feeds one case through the three other ways a G-buffer enters: hr_gbuffer_copy_from_device,
hr_gbuffer_bind_device and a descriptor without gb1.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import gbuffer_cases as G
import oracle as O
import pyhr
from test_gpu_camera import Reach, _bounded, _refl_isolated, _sh_ao_isolated
from test_gpu_parity import f16
from test_gpu_ragged import SKY, new_context, run_gi_refl, run_shadows_ao
from widened.test_gpu_taa_tonemap import same_halves, u16

pytestmark = pytest.mark.gpu


def _seq(case):
    return [(i, f) for i, (_, f) in enumerate(case.frames)]


def _upload(case):
    def gbuf(i, f, ctx):
        g = case.frames[i][0]
        ctx.gbuffer_upload(f.ping_pong, g)
        return g
    return gbuf


def _planting(case, before, after, keys):
    """before hook: the case's planted histories into the device passes, the oracle passes and the isolated stages' history, then
    test_gpu_camera's own before hook"""
    def hook(i, f, passes, oracles):
        if keys == ("sh", "ao"):
            G.plant_device(case, i, sh=passes[0], ao=passes[1])
            G.plant_oracle(case, i, f, osh=oracles[0], oao=oracles[1])
        else:
            G.plant_device(case, i, rf=passes[1])
            G.plant_oracle(case, i, f, orf=oracles[1])
        G.plant_hist(case, i, after.hist, keys)
        before(i, f, passes, oracles)
    return hook


@pytest.mark.parametrize("cid", G.CASE_IDS)
def test_shadows_ao_adversarial(cid):
    """shadows at full resolution, AO at half (the mips and the upsample see the case too)"""
    case = G.case(cid)
    reach = Reach(case)
    before, after = _sh_ao_isolated(case, reach)
    run_shadows_ao(f"shadows+ao {cid}", case.W, case.H, 0, 1, seq=_seq(case), before=_planting(case, before, after, ("sh", "ao")), after=after,
                   gbuf=_upload(case), prev_gbuf=case.prev)
    reach.check(("K3", "K9"))


@pytest.mark.parametrize("cid", G.CASE_IDS)
def test_ddgi_reflections_adversarial(cid):
    case = G.case(cid)
    reach = Reach(case)
    before, after = _refl_isolated(case, reach)
    run_gi_refl(f"ddgi+reflections {cid}", case.W, case.H, 0, True, seq=_seq(case), before=_planting(case, before, after, ("rf",)), after=after,
                gbuf=_upload(case), prev_gbuf=case.prev)
    reach.check(("K14",))


def _post_chain(case, put_gbuffer, gb1_null=False):
    """shadows, AO, reflections, the deferred combine and TAA (bit-exact) over the case, each frame's G-buffer put into its slot by
    put_gbuffer(ctx, slot, host G-buffer); returns every frame's pass outputs and G-buffer mips"""
    W, H = case.W, case.H
    ctx = new_context(pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST), W, H)
    sh, ao, rf, de = pyhr.Pass(ctx, "shadows", W, H, 0), pyhr.Pass(ctx, "ao", W, H, 1), pyhr.ReflectionsPass(ctx, W, H, 1), pyhr.DeferredPass(ctx, W, H)
    rf.params.sky_color[0], rf.params.sky_color[1], rf.params.sky_color[2] = SKY
    de.params.env_color[0], de.params.env_color[1], de.params.env_color[2] = SKY
    taa = pyhr.TAAPass(ctx, W, H)
    taa.params.reset_every_frame = 0
    otaa = O.TAAOracle(W, H, reset_every_frame=0)
    outs, prev_j = [], np.zeros(2, np.float32)
    for i, (g, f0) in enumerate(case.frames):
        f = pyhr.hr_frame.from_buffer_copy(f0)
        j = pyhr.taa_jitter(i, W, H)
        pyhr.apply_jitter(f, j, prev_j)
        prev_j = j
        put_gbuffer(ctx, f.ping_pong, g)
        sh.render(f)
        ao.render(f)
        rf.render(f, None)
        de.render(f, sh, ao, rf, None)
        torch.cuda.synchronize()
        gref = pyhr.GBufferHost(W, H)
        gref.gb1, gref.gb2, gref.gb3, gref.depth = (np.zeros_like(g.gb1) if gb1_null else g.gb1), g.gb2, g.gb3, g.depth
        want = f16(O.deferred(gref, f, shadow=sh.download(100), ao=ao.download(100), reflections=rf.download(100), env=SKY))
        _bounded(f16(de.download(100))[..., :3], want[..., :3], f"{case.id} frame {i}: deferred", 1e-3, 2e-2)
        cur = u16(de.download(100))
        taa.render(f, de)
        want_taa = otaa.render(f, cur, g.depth, u16(g.gb2))
        got_taa = u16(taa.download(100))
        assert same_halves(got_taa, want_taa), f"{case.id} frame {i}: TAA: {np.count_nonzero(got_taa != want_taa)} of {got_taa.size} halves differ"
        mips = [ctx.gbuffer_download(f.ping_pong, m, w, W, H) for m in range(3) for w in (0, 2, 3)]
        outs.append([p.download(k) for p in (sh, ao, rf) for k in (0, 1, 4, 6, 100)] + [de.download(100), got_taa] + mips)
    for p in (taa, de, rf, sh, ao):
        p.destroy()
    ctx.close()
    return outs


@pytest.mark.parametrize("cid", ["ties@128x72", "ties@97x53", "depth@97x53", "edges@97x53", "normals@128x72"])
def test_post_chain_adversarial(cid):
    """the deferred combine (test_gpu_camera's bar) and TAA (bit-exact): equal depths in every TAA neighbourhood, sky / geometry
    patterns, history on the frame edges, octahedral fold lines"""
    _post_chain(G.case(cid), lambda ctx, slot, g: ctx.gbuffer_upload(slot, g))


def _dev(g, gb1=True):
    """torch CUDA tensors holding a host G-buffer, and a descriptor of them"""
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (g.gb1, g.gb2.view(np.int16), g.gb3.view(np.int16), g.depth)]
    d = pyhr.hr_gbuffer_desc(g.W, g.H, t[0].data_ptr() if gb1 else None, t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr())
    return t, d


def test_gbuffer_input_paths():
    """one adversarial case through hr_gbuffer_copy_from_device and hr_gbuffer_bind_device (zero-copy) from torch CUDA tensors: every
    pass output and mip is the hr_gbuffer_upload run's, bit for bit; the bound tensors are never written; after a bind,
    hr_gbuffer_upload and hr_gbuffer_render put the slot back on library-owned storage.  A descriptor without gb1 (bound): the deferred combine is the
    oracle's with albedo and metallic 0"""
    case = G.case("depth@97x53")
    ref = _post_chain(case, lambda ctx, slot, g: ctx.gbuffer_upload(slot, g))
    keep = []

    def copy(ctx, slot, g):
        t, d = _dev(g)
        ctx.gbuffer_copy_from_device(slot, d)
        torch.cuda.synchronize()
        keep.append(t)

    def bind(ctx, slot, g):
        t, d = _dev(g)
        ctx.gbuffer_bind_device(slot, d)
        keep.append((t, [x.clone() for x in t]))

    for name, put in (("copy_from_device", copy), ("bind_device", bind)):
        keep.clear()
        got = _post_chain(case, put)
        for i, (a, b) in enumerate(zip(got, ref)):
            bad = [k for k, (x, y) in enumerate(zip(a, b)) if not np.array_equal(x, y)]
            assert not bad, f"{name} frame {i}: outputs {bad} differ from the hr_gbuffer_upload run"
        if name == "bind_device":
            for t, snap in keep:
                assert all(torch.equal(x, y) for x, y in zip(t, snap)), "a bound G-buffer tensor was written"
    # bind, then upload or render: the slot reads the library's storage again, not the (then zeroed) bound tensors
    W, H = case.W, case.H
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ctx = new_context(sc, W, H)
    g0, g1 = case.frames[0][0], case.frames[2][0]
    f = case.frames[0][1]
    for name, refill, want in (("hr_gbuffer_upload", lambda: ctx.gbuffer_upload(0, g1), g1), ("hr_gbuffer_render", lambda: ctx.gbuffer_render(0, f), None)):
        t, d = _dev(g0)
        ctx.gbuffer_bind_device(0, d)
        assert np.array_equal(ctx.gbuffer_download(0, 0, 0, W, H), g0.depth)
        refill()
        torch.cuda.synchronize()
        got = [ctx.gbuffer_download(0, 0, which, W, H) for which in range(4)]
        for x in t:
            x.zero_()
        torch.cuda.synchronize()
        for which in range(4):
            assert np.array_equal(ctx.gbuffer_download(0, 0, which, W, H), got[which]), f"image {which} after bind + {name} follows the bound tensors"
        if want is not None:
            for which, arr in ((0, want.depth), (1, want.gb1), (2, want.gb2), (3, want.gb3)):
                assert np.array_equal(got[which], arr), f"image {which} after bind + {name}"
        else:
            assert (got[0] != 1.0).any(), f"{name} wrote no geometry"
    ctx.close()
    # gb1 = NULL
    keep.clear()
    _post_chain(case, lambda ctx, slot, g: (keep.append(_dev(g, gb1=False)), ctx.gbuffer_bind_device(slot, keep[-1][1])), gb1_null=True)
