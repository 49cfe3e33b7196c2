"""The oracle tells every light case of light_cases.py apart from its twin: run under the case and under the twin, over the same
frames, the case's stages differ by at least 10x the bar the GPU tests apply there (RMSE or max-abs), and a shadows mask in at
least 1 % of its bits.  So a kernel that evaluated the light as the twin (a swapped cone, a cone tested against -data0, 1/d^2
from another distance, the colour channels out of order, the wrong light type) would fail the GPU comparison.  CPU only.

The sequence is test_gpu_ragged.frames' static part: the light changes, the camera does not.
"""
import ctypes as C

import numpy as np
import pytest

import light_cases as LC
import oracle as O
import pyhr

SKY = (0.3, 0.4, 0.6)
N_FRAMES = 3
# stage -> (RMSE bar, max-abs bar) of the GPU comparison: check_all's shadows temporal bars, test_gpu_gi_refl.close's ray-trace bars
# (relative to max(1, |reference|)), the deferred combine's bars (test_deferred)
BARS = {"sh temporal": (1e-3, 2e-3), "rt": (1e-3, 0.02), "deferred": (1e-3, 2e-2)}
MASK_BITS = 0.01
_scenes, _runs = {}, {}


def _scene(name):
    if name not in _scenes:
        kind, tris, _ = LC.SCENES[name]
        sc = pyhr.SynthScene(kind, tris)
        _scenes[name] = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    return _scenes[name]


def oracle_stages(case):
    """every stage of light_cases on every frame: {stage: [image per frame]}"""
    if case.id in _runs:
        return _runs[case.id]
    W, H = LC.SIZE
    ss = _scene(case.scene)
    bn = pyhr.blue_noise()
    osh = O.ShadowsOracle(W, H, 0)
    rp = pyhr.hr_reflections_params()
    pyhr.load_product().hr_reflections_default_params(C.byref(rp))
    rp.sky_color[0], rp.sky_color[1], rp.sky_color[2] = SKY
    orf = O.ReflectionsOracle(W, H, 0, rp)
    out = {k: [] for k in ("mask", "sh temporal", "rt", "deferred")}
    f, prev_g = None, O.zero_gbuf_mips(W, H)
    for i in range(N_FRAMES):
        f = pyhr.make_frame(*LC.SCENES[case.scene][2], W, H, prev=f, num_frames=i, light=LC.light(case, i))
        g = O.gbuffer_render(ss, f, W, H)
        cur_g = O.GBufMips(g)
        osh.render(ss.scene, cur_g, prev_g, f, bn)
        orf.render(ss, cur_g, prev_g, f, bn)
        prev_g = cur_g
        out["mask"].append(osh.mask.copy())
        out["sh temporal"].append(osh.temporal.copy())
        out["rt"].append(orf.rt[..., :3].copy())
        out["deferred"].append(O.deferred(g, f, shadow=osh.final)[..., :3].copy())  # the direct term: no AO, GI, reflections, environment
    _runs[case.id] = out
    return out


def stage_error(stage, a, b):
    """(RMSE, max-abs) as the GPU tests bound them"""
    a, b = O.h2f(a).astype(np.float64), O.h2f(b).astype(np.float64)
    d = np.abs(a - b)
    if stage == "rt":
        d = d / np.maximum(1.0, np.abs(b))
    return float(np.sqrt(np.mean(d ** 2))), float(d.max())


def bits_differ(a, b):
    return float(np.unpackbits((a ^ b).view(np.uint8)).mean())


@pytest.mark.parametrize("case", LC.CASES, ids=LC.ids(LC.CASES))
def test_case_differs_from_its_twin(case):
    twin = LC.BY_ID[case.twin]
    assert twin.scene == case.scene and twin.id != case.id
    got, base = oracle_stages(case), oracle_stages(twin)
    for stage in case.stages:
        if stage == "mask":
            frac = max(bits_differ(g, b) for g, b in zip(got[stage], base[stage]))
            print(f"\n[{case.id} vs {twin.id}] mask: {100 * frac:.2f} % of the bits differ")
            assert frac >= MASK_BITS, f"{case.id}: the mask differs from {twin.id}'s in {100 * frac:.2f} % of its bits only"
            continue
        errs = [stage_error(stage, g, b) for g, b in zip(got[stage], base[stage])]
        rm, mx = max(e[0] for e in errs), max(e[1] for e in errs)
        bar_rm, bar_mx = BARS[stage]
        print(f"\n[{case.id} vs {twin.id}] {stage}: RMSE {rm:.2e} = {rm / bar_rm:.0f} x its bar, max-abs {mx:.2e} = {mx / bar_mx:.0f} x its bar")
        assert rm >= 10 * bar_rm or mx >= 10 * bar_mx, f"{case.id}: the oracle's {stage} differs from {twin.id}'s by RMSE {rm:.2e} / max-abs {mx:.2e} only"


def test_colour_scales_each_channel_of_the_direct_term():
    """colour (1, 1/4, 1/16) against white: Li scales by a power of two per channel, so the direct term's G and B are the white
    light's times 1/4 and 1/16 (exact in fp32; fp16 subnormals round), R unchanged.  A channel swap fails here."""
    got, base = oracle_stages(LC.BY_ID["colored"])["deferred"], oracle_stages(LC.BY_ID["sun_default"])["deferred"]
    for g, b in zip(got, base):
        g, b = O.h2f(g).astype(np.float64), O.h2f(b).astype(np.float64)
        assert b[..., 1].max() > 0.1
        for c, s in enumerate((1.0, 0.25, 0.0625)):
            assert np.abs(g[..., c] - s * b[..., c]).max() <= 2.0 ** -24, f"channel {c}"


def test_degenerate_lights_light_nothing():
    """the overhead sun (NaN tangent), the sun from below and the spot pointing up: under this static camera the mask and the direct
    term are 0 everywhere (the sun from below does trace shadow rays, from the surfaces that face down, and the floor blocks them);
    zero intensity keeps the mask (att excludes intensity) and zeroes the direct term"""
    for cid in ("sun_overhead", "sun_below", "spot_away"):
        r = oracle_stages(LC.BY_ID[cid])
        assert all(not m.any() for m in r["mask"]), cid
        assert all(O.h2f(d).max() == 0.0 for d in r["deferred"]), cid
    z, d = oracle_stages(LC.BY_ID["intensity_zero"]), oracle_stages(LC.BY_ID["sun_default"])
    assert all(np.array_equal(a, b) for a, b in zip(z["mask"], d["mask"]))
    assert all(O.h2f(a).max() == 0.0 for a in z["deferred"])


def test_cases_are_distinct():
    assert len(set(LC.ids(LC.CASES))) == len(LC.CASES)
    for c in LC.CASES:
        assert c.twin in LC.BY_ID and set(c.stages) <= {"mask", *BARS}, c.id
