"""The oracle reacts to every continuous parameter case of param_cases.py: run at the case's value and at the default, over the
same frames, the stage the parameter acts on differs by at least 10x a bar test_gpu_parameters.py applies to it.  So a
kernel that ignored the parameter, or read another one in its place, would fail the GPU comparison.  CPU only.

The sequences restate test_gpu_ragged's runners (camera path, DDGI probe distance and normal bias, rotations) on the oracle alone.
"""
import ctypes as C

import numpy as np
import pytest

import oracle as O
import param_cases as PC
import pyhr

SKY = (0.3, 0.4, 0.6)
_scenes = {}


def _scene(name):
    if name not in _scenes:
        kw = PC.scene_kw(name)
        sc = pyhr.SynthScene(kw["scene"], kw["tris"])
        _scenes[name] = (sc, O.ShadingScene(sc, brute=sc.n_tris <= 4096))
    return _scenes[name]


def _frames(W, H, n, scene, pan_from=3):
    """test_gpu_ragged.frames: static camera, then a lateral pan of 0.05 / frame"""
    kw = PC.scene_kw(scene)
    (px, py, pz), (tx, ty, tz) = kw["cam"]
    light = kw["light"]
    f = None
    for i in range(n):
        dx = 0.0 if i < pan_from else 0.05 * (i - pan_from + 1)
        f = pyhr.make_frame((px + dx, py, pz), (tx + dx, ty, tz), W, H, prev=f, num_frames=i, light=light)
        yield i, f


def _defaults(struct, fn):
    P = struct()
    getattr(pyhr.load_product(), fn)(C.byref(P))
    P.sky_color[0], P.sky_color[1], P.sky_color[2] = SKY
    return P


def oracle_stage(case: PC.Case, changed: bool):
    """the case's stage on every frame, with the case's parameters applied (changed) or left at their defaults"""
    W, H = PC.SIZE
    sc, ss = _scene(case.scene)
    params = case.params if changed else {}
    bn = pyhr.blue_noise()
    out = []
    prev_g = O.zero_gbuf_mips(W, H)
    if case.kind in ("shadows", "ao"):
        osh, oao = O.ShadowsOracle(W, H, 0), O.AOOracle(W, H, 1)
        for k, v in params.items():
            setattr(osh.params if case.kind == "shadows" else oao.params, k, v)
        for i, f in _frames(W, H, case.frames, case.scene):
            cur_g = O.GBufMips(O.gbuffer_render(ss, f, W, H))
            osh.render(ss.scene, cur_g, prev_g, f, bn)
            oao.render(ss.scene, cur_g, prev_g, f, bn)
            prev_g = cur_g
            out.append({"sh temporal": osh.temporal, "sh a-trous": osh.atrous_out, "sh final": osh.final, "ao temporal": oao.temporal,
                        "ao blur": oao.blur[1], "ao final": oao.final}[case.stage].copy())
        return out
    rp = _defaults(pyhr.hr_reflections_params, "hr_reflections_default_params")
    odd = None
    if case.ddgi:
        dp = _defaults(pyhr.hr_ddgi_params, "hr_ddgi_default_params")
        dp.probe_distance = 4.0 if case.scene == "shadows_test" else 12.0
        dp.normal_bias = 1.0
        for k, v in (params.items() if case.kind == "ddgi" else ()):
            setattr(dp, k, v)
        odd = O.DDGIOracle(W, H, 0, dp, *sc.bounds())
    for k, v in (params.items() if case.kind == "reflections" else ()):
        setattr(rp, k, v)
    orf = O.ReflectionsOracle(W, H, 0, rp)
    if case.lut:
        orf.brdf_lut = pyhr.brdf_lut(64)
    for i, f in _frames(W, H, case.frames, case.scene):
        cur_g = O.GBufMips(O.gbuffer_render(ss, f, W, H))
        if odd:
            odd.render(ss, cur_g, f, pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5)))
        orf.render(ss, cur_g, prev_g, f, bn, odd)
        prev_g = cur_g
        if case.stage.startswith("ddgi"):
            img = {"ddgi radiance": odd.radiance, "ddgi irradiance": odd.cur_irr, "ddgi depth": odd.cur_dep, "ddgi sample": odd.sample}[case.stage]
        else:
            img = {"rt": orf.rt[..., :3], "temporal": orf.cur_temporal, "moments": orf.cur_moments, "a-trous": orf.atrous_out, "final": orf.final}[case.stage]
        out.append(np.array(img))
    return out


def stage_error(stage, a, b):
    """(RMSE, max-abs) as the GPU test bounds them: relative to max(1, |reference|) for DDGI and reflections (test_gpu_gi_refl.close)"""
    a, b = O.h2f(a).astype(np.float64), O.h2f(b).astype(np.float64)
    d = np.abs(a - b)
    if stage in PC.RELATIVE:
        d = d / np.maximum(1.0, np.abs(b))
    return float(np.sqrt(np.mean(d ** 2))), float(d.max())


_default_runs = {}


@pytest.mark.parametrize("case", PC.CONTINUOUS, ids=PC.ids(PC.CONTINUOUS))
def test_oracle_is_sensitive_to_the_case(case):
    """the GPU test fails when either of its bars is exceeded, so the stage must move by 10x its RMSE bar or 10x its max-abs bar"""
    key = (case.kind, case.scene, case.frames, case.ddgi, case.lut, case.stage)
    if key not in _default_runs:
        _default_runs[key] = oracle_stage(case, False)
    base, got = _default_runs[key], oracle_stage(case, True)
    errs = [stage_error(case.stage, g, b) for g, b in zip(got, base)]
    rm, mx = max(e[0] for e in errs), max(e[1] for e in errs)
    bar_rm, bar_mx = PC.BARS[case.stage]
    print(f"\n[{case.id}] {case.stage} vs the default: RMSE {rm:.2e} = {rm / bar_rm:.0f} x its bar, max-abs {mx:.2e} = {mx / bar_mx:.0f} x its bar")
    assert rm >= 10 * bar_rm or mx >= 10 * bar_mx, f"{case.id}: the oracle's {case.stage} moves by RMSE {rm:.2e} / max-abs {mx:.2e} only"


def test_cases_change_one_parameter_each():
    """a continuous case changes exactly one parameter, and to a value other than its default"""
    defaults = {"shadows": O.ShadowsOracle(8, 8, 0).params, "ao": O.AOOracle(8, 8, 1).params,
                "reflections": _defaults(pyhr.hr_reflections_params, "hr_reflections_default_params"),
                "ddgi": _defaults(pyhr.hr_ddgi_params, "hr_ddgi_default_params")}
    for c in PC.CONTINUOUS:
        assert len(c.params) == 1 and c.stage in PC.BARS, c.id
        (k, v), = c.params.items()
        assert np.float32(getattr(defaults[c.kind], k)) != np.float32(v), f"{c.id}: the default value"
    assert len(set(PC.ids(PC.CONTINUOUS + PC.LAYOUTS))) == len(PC.CONTINUOUS) + len(PC.LAYOUTS)
