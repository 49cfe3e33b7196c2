"""The hand-built G-buffer cases of gbuffer_cases.py are well formed, their ladders straddle their thresholds, and the oracle reaches
every reprojection branch a case targets and tells each case from its tame twin, so test_gpu_adversarial_gbuffer compares the device
at the decisions it is meant to reach.  CPU only; run with -s to print each case's branch counts and ladder sides.
"""
import ctypes as C

import numpy as np
import pytest

import gbuffer_cases as G
import oracle as O
import pyhr

SKY = (0.3, 0.4, 0.6)
_ss = {}


def _scene():
    if "s" not in _ss:
        sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
        _ss["s"] = O.ShadingScene(sc, brute=True)
    return _ss["s"]


def run_oracle(frames, W, H, case=None):
    """shadows (full resolution), AO (half) and reflections (full) over the frames: ({kernel: {branch: max pixels over frames that
    read history}}, the last frame's history lengths and tile flags of the three temporal stages and its reflection ray lengths).
    case: its preceding G-buffer and planted histories are used"""
    ss, bn = _scene(), pyhr.blue_noise()
    osh, oao = O.ShadowsOracle(W, H, 0), O.AOOracle(W, H, 1)
    rp = pyhr.hr_reflections_params()
    pyhr.load_product().hr_reflections_default_params(C.byref(rp))
    rp.sky_color[0], rp.sky_color[1], rp.sky_color[2] = SKY
    orf = O.ReflectionsOracle(W, H, 0, rp)
    n = {}
    prev_g = O.GBufMips(case.prev) if case is not None and case.prev is not None else O.zero_gbuf_mips(W, H)
    for i, (g, f) in enumerate(frames):
        if case is not None:
            G.plant_oracle(case, i, f, osh, oao, orf)
        cur_g = O.GBufMips(g)
        for k, o, run in (("K3", osh, lambda: osh.render(ss.scene, cur_g, prev_g, f, bn)), ("K9", oao, lambda: oao.render(ss.scene, cur_g, prev_g, f, bn)),
                          ("K14", orf, lambda: orf.render(ss, cur_g, prev_g, f, bn))):
            with O.ReprojectCodes(o.W, o.H) as rc:
                run()
            if i:
                d = n.setdefault(k, {})
                for b, v in rc.counts().items():
                    d[b] = max(d.get(b, 0), v)
        prev_g = cur_g
    out = [osh.cur_moments[..., 2], osh.tile_flags, oao.cur_length, oao.tile_flags, orf.rt[..., 3], orf.cur_moments[..., 2], orf.tile_flags]
    return n, [o.copy() for o in out]


_runs = {}


def _run(cid):
    if cid not in _runs:
        c = G.case(cid)
        _runs[cid] = (c, run_oracle(c.frames, c.W, c.H, c))
    return _runs[cid]


@pytest.mark.parametrize("cid", G.CASE_IDS)
def test_case_well_formed(cid):
    c = G.case(cid)
    assert len(c.frames) >= 3
    for g, f in c.frames:
        assert (g.W, g.H) == (c.W, c.H)
        for a in (g.gb2, g.gb3):
            assert a.dtype == np.uint16 and np.isfinite(a.view(np.float16)).all(), f"{cid}: a non-finite fp16 field"
        assert g.depth.dtype == np.float32 and np.isfinite(g.depth).all() and (g.depth >= 0).all() and (g.depth <= 1).all()
        assert (g.depth != 1.0).any(), f"{cid}: no geometry"
        sky = g.depth == 1.0
        assert not g.gb2[sky].any() and not g.gb1[sky].any(), f"{cid}: a sky pixel carries G-buffer data"
    assert all(t.split(":")[0] in ("K3", "K9", "K14") and t.split(":")[1] in O.RP_BITS or t.split(":")[1] == "invalid" for t in c.targets)
    # the frame sequence is static: only the G-buffer's own motion vectors move history
    f0 = c.frames[0][1]
    for _, f in c.frames[1:]:
        assert tuple(f.ubo.view_proj[:]) == tuple(f0.ubo.view_proj[:]) == tuple(f.ubo.prev_view_proj[:])


@pytest.mark.parametrize("cid", [c for c in G.CASE_IDS if G.case(c).ladders])
def test_ladders_straddle_their_thresholds(cid):
    c = G.case(cid)
    for name, r in c.ladders.items():
        above, below = int(np.count_nonzero(r > 0)), int(np.count_nonzero(r < 0))
        print(f"\n[{cid}] {name}: {above} pixels above, {below} below the threshold; nearest {np.abs(r[r != 0]).min():.2e} away (float64)")
        assert above > 0 and below > 0, f"{cid}: the {name} ladder stays on one side"


@pytest.mark.parametrize("cid", [c for c in G.CASE_IDS if c.startswith("edges")])
def test_edge_targets_reached(cid):
    """every history_coord_floor target of the edges case is hit exactly by some border pixel, or (where no fp16 motion reaches it)
    bracketed by the nearest values on both sides"""
    G.case(cid)
    for t, d in G.EDGE_REACH[cid].items():
        print(f"\n[{cid}] {t}: " + ("exact" if (d == 0).any() else f"nearest {d[d < 0].max():.2e} / +{d[d > 0].min():.2e}"))
        assert (d == 0).any() or ((d < 0).any() and (d > 0).any()), f"{cid}: history_coord_floor {t} neither reached nor bracketed"
    exact = sum(bool((d == 0).any()) for d in G.EDGE_REACH[cid].values())
    assert exact >= 4, f"{cid}: only {exact} targets hit exactly"


def test_plane_and_normal_ladders_reach_within_ulps():
    """the plane-distance ladder comes within a few float32 ulps of 5.0 and the normal ladder within a few of 0.1, on both sides"""
    for cid, name, thr in (("plane_distance@128x72", "plane distance", 5.0), ("normal_distance@128x72", "normal dot^2", 0.1)):
        r = G.case(cid).ladders[name]
        ulp = float(np.spacing(np.float32(thr)))
        for side in (r[r > 0], -r[r < 0]):
            assert side.min() < 8 * ulp, f"{cid}: nearest {name} {side.min():.2e} is {side.min() / ulp:.1f} ulps away"


@pytest.mark.parametrize("cid", G.CASE_IDS)
def test_oracle_reaches_targets(cid):
    c, (n, _) = _run(cid)
    print(f"\n[{cid}] reprojection branch pixels: {n}")
    for t in c.targets:
        k, b = t.split(":")
        got = n.get(k, {}).get(b, 0)
        assert got >= G.MIN_PIXELS, f"{cid}: {k} reaches '{b}' in {got} pixels only"


@pytest.mark.parametrize("cid", G.CASE_IDS)
def test_case_differs_from_tame_twin(cid):
    c, (_, out) = _run(cid)
    _, tame = run_oracle(c.tame(), c.W, c.H)
    names = ["K3 history length", "K3 tile flags", "K9 history length", "K9 tile flags", "K12 ray length", "K14 history length", "K14 tile flags"]
    diff = {nm: int(np.count_nonzero(a != b)) for nm, a, b in zip(names, out, tame)}
    print(f"\n[{cid}] pixels / tiles that differ from the tame twin: {diff}")
    assert any(diff.values()), f"{cid}: the oracle's history lengths and tile flags equal the tame twin's"
