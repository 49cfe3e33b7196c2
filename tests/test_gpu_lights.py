"""Every lit pass under every light case of light_cases.py against the CPU oracle: sun, point and spot lights, a coloured light, the
edges of the light block (the sun at the zenith, the horizon and below, equal and reversed cone angles, zero intensity, fp16
overflow) and a light that changes from frame to frame.

The runners and bars are test_gpu_ragged's, unchanged: shadows + AO under check_all (the mask bit-exact); DDGI + reflections with
the uniforms bytes, probe directions / distances and reflection ray lengths exact and the images under `close`.  The deferred
combine (test_deferred) and the path tracer (widened/) take the cases of their own.  Beyond equality with the oracle:

- sun_overhead: data0 = (-0, 1, -0) makes soft_shadow_dir's tangent normalize(0) = NaN (lighting.glsl:40, DESIGN.md §6), so no
  shadow ray is traced: the mask is 0 and the mode-0 path tracer under a black sky is exactly 0 on every hit, while the hard
  form of K12 and K18 still lights their hits.
- spot_away: the spot points up, att = 0 on every surface: the mask is 0, no shadow ray, no K12 light ray (K12 shades without the
  sky ray), and one sky ray per K18 probe-ray hit, none toward the light.  The sun from below (sun_below) is not dark: att > 0 on
  the surfaces that face down, and on the walls the soft disk tilts Wi onto.  Measured on the H100 at frame 0: 1 616 shadow
  rays and 2 447 K12 light rays, every one blocked (the mask is 0); once the camera pans, a few mask bits are lit.  Device and
  oracle agree bit for bit on that mask as on every other.
- point_overflow: a 1e5 point light saturates fp16.  SameClassThenClose requires every texel to be finite, +inf, -inf or
  NaN on both sides alike and holds the finite ones to the usual bar, up to the first stage where the fp16 cascade parts the
  two (the rule and its measured count are in the class's and the test's docstrings).
"""
import ctypes as C

import numpy as np
import pytest

import light_cases as LC
import oracle as O
import pyhr
from test_gpu_gi_refl import close
from test_gpu_parity import check_all, f16
from test_gpu_ragged import run_gi_refl, run_shadows_ao

pytestmark = pytest.mark.gpu

W, H = LC.SIZE
DARK = {"sun_overhead", "spot_away"}                # the mask is 0 everywhere, no shadow ray is traced
UNLIT = {"spot_away"}                                # att = 0 on every surface: no light ray in K12 or K18
CHANGING = {"moving", "arcade_moving"}               # static camera: only the light changes
MISS = 10000.0                                       # K18's hit distance of a probe ray that hits nothing


def _pan_from(case, n):
    return n if case.id in CHANGING else 3


# ---------------------------------------------------------------------------------------------- shadows + AO
@pytest.mark.parametrize("case", LC.CASES, ids=LC.ids(LC.CASES))
def test_shadows_ao_under_light(case):
    rays = []

    def check(i, sh, ao, osh, oao):
        check_all(i, sh, ao, osh, oao, [])
        rays.append(sh.stats().rays_primary)
        if case.id in DARK:
            assert not osh.mask.any() and not sh.download(0).any(), f"frame {i}: a lit mask bit"
            assert rays[-1] == 0, f"frame {i}: {rays[-1]} shadow rays traced"

    run_shadows_ao(f"shadows+ao {case.id}", W, H, 0, 1, n=5, pan_from=_pan_from(case, 5), check=check, **LC.scene_kw(case))
    if case.id not in DARK:
        assert min(rays) > 0
    print(f"[{case.id}] shadow rays per frame: {rays}")


# ---------------------------------------------------------------------------------------------- DDGI + reflections
def _hit_rays(dirdepth):
    return int(np.count_nonzero(O.h2f(dirdepth)[..., 3] != MISS))


@pytest.mark.parametrize("case", [c for c in LC.CASES if c.id != "point_overflow"], ids=[c.id for c in LC.CASES if c.id != "point_overflow"])
def test_ddgi_reflections_under_light(case):
    def hook(i, dd, odd, rf, orf):
        s_dd, s_rf = dd.stats(), rf.stats()
        if case.id in UNLIT:
            assert s_rf.rays_secondary == 0, f"frame {i}: {s_rf.rays_secondary} K12 light rays"
            assert s_dd.rays_secondary == _hit_rays(odd.dirdepth), f"frame {i}: K18 traced {s_dd.rays_secondary} secondary rays, " \
                                                                     f"{_hit_rays(odd.dirdepth)} probe rays hit"
        if case.id == "sun_overhead":  # the hard form lights the hits the soft form leaves dark: light rays traced, K12 hits not black
            assert s_rf.rays_secondary > 0, f"frame {i}: no K12 light ray"
            assert s_dd.rays_secondary > _hit_rays(odd.dirdepth), f"frame {i}: no K18 light ray"
            for what, rt in (("device", f16(rf.download(0))), ("oracle", O.h2f(orf.rt))):
                hit = rt[..., 3] > 0
                assert hit.mean() > 0.1 and (rt[hit][:, :3] > 0).any(-1).mean() > 0.2, f"frame {i}: {what} K12 hits are black"

    run_gi_refl(f"ddgi+reflections {case.id}", W, H, 0, True, n=4, pan_from=_pan_from(case, 4), frame_hook=hook, **LC.scene_kw(case))


# ---------------------------------------------------------------------------------------------- non-finite values
def classes(a):
    """0 finite, 1 +inf, 2 -inf, 3 NaN"""
    a = np.asarray(a)
    c = np.zeros(a.shape, np.int8)
    c[np.isposinf(a)], c[np.isneginf(a)], c[np.isnan(a)] = 1, 2, 3
    return c


def class_counts(a):
    c = classes(a)
    return {k: int(np.count_nonzero(c == v)) for k, v in (("inf", 1), ("-inf", 2), ("nan", 3))}


class SameClassThenClose:
    """`close` for images that may hold inf and NaN: every texel in the same class (finite, +inf, -inf, NaN) on the device and in
    the oracle, then `close` over the texels finite on both.

    One exception ends the comparison.  sample_irradiance blends atlas texels with bilinear and trilinear weights.  Where an inf
    texel sits at the edge of a footprint, one implementation may give it a weight of exactly 0 (inf * 0 = NaN, which the NaN
    guard turns into 0.5 per channel: `guard`, 0.5^2 x energy preservation x pi / 2 x gi_intensity) or leave it outside the
    footprint (a finite blend), and the other a weight of 1e-7 (inf).  So at the first stage where classes differ, every texel
    whose class differs must be +inf on one side and finite on the other; `flips` records their count and how many of the
    finite ones hold the guard's value, `stopped` is set and no later comparison is made: from there the atlas blends the
    differing texels and the classes part further (DESIGN.md §6).  `log` holds the oracle's non-finite counts (printed with -s).
    Without a guard (None) any difference in class fails."""

    def __init__(self, guard=None):
        self.guard = None if guard is None else np.float32(np.float16(guard))
        self.log, self.flips, self.stopped = [], [], False

    def __call__(self, got, want, name, r=1e-3, m=6e-3):
        assert got.shape == want.shape, name
        if self.stopped:
            return
        cg, cw = classes(got), classes(want)
        self.log.append((name, class_counts(want)))
        bad = cg != cw
        if bad.any():
            assert self.guard is not None, f"{name}: {np.count_nonzero(bad)} texels differ in class; device {class_counts(got)}, oracle {class_counts(want)}"
            fin = np.where(cg[bad] == 0, got[bad], want[bad])                    # the finite side
            inf_vs_finite = ((cg[bad] == 0) | (cw[bad] == 0)) & (np.maximum(cg[bad], cw[bad]) == 1)
            assert inf_vs_finite.all(), f"{name}: {np.count_nonzero(~inf_vs_finite)} texels differ in class other than +inf against finite; " \
                                        f"device {class_counts(got)}, oracle {class_counts(want)}"
            self.flips.append((name, int(np.count_nonzero(bad)), int(np.count_nonzero(fin == self.guard))))
            self.stopped = True
        both = (cg == 0) & (cw == 0)
        close(got[both], want[both], name, r, m)

    def report(self, case):
        print(f"\n[{case}] non-finite texels of the oracle: " + "; ".join(f"{n} {c}" for n, c in self.log if any(c.values())))
        print(f"[{case}] texels +inf on one side, finite on the other (of them the NaN guard's value): {self.flips or 'none'}")


def nan_guard_value(params):
    """sample_irradiance's value for a channel whose blend is NaN, times gi_intensity (the K21 sample): 0.5^2 x energy x pi / 2"""
    return 0.25 * np.float32(params.recursive_energy_preservation) * (0.5 * np.pi) * params.gi_intensity


def test_ddgi_reflections_point_overflow():
    """a 1e5 point light 0.25 above the floor: K18's fp16 radiance saturates, K19 blends the inf into the atlas and the infinite
    bounce reads it back (NaN from an inf probe at weight 0), frame after frame (DESIGN.md §6).  Frame 0: the device reproduces
    every non-finite texel of every stage (6 inf in K18's radiance, 300 in the irradiance atlas, 330 in the K21 sample, none in
    the reflections).  Frame 1: K18's radiance and both atlases still agree texel for texel; in the K21 sample, measured on the
    H100, 633 of 147 456 values are +inf on one side and finite on the other (411 of them the NaN guard's 0.3337, 222 finite
    blends of 0.53-0.55), the rule of SameClassThenClose, and the comparison stops there."""
    case = LC.BY_ID["point_overflow"]
    P = pyhr.hr_ddgi_params()
    pyhr.load_product().hr_ddgi_default_params(C.byref(P))
    cmp = SameClassThenClose(nan_guard_value(P))
    run_gi_refl("ddgi+reflections point_overflow", W, H, 0, True, n=3, cmp=cmp, **LC.scene_kw(case))
    cmp.report(case.id)
    frame0 = [(n, c) for n, c in cmp.log if n.startswith("frame 0 ")]
    assert len(frame0) == 9 and any(any(c.values()) for n, c in frame0), "frame 0: every stage compared, some non-finite"
    assert all(not n.startswith("frame 0 ") and k <= 1000 for n, k, _ in cmp.flips), cmp.flips


# ---------------------------------------------------------------------------------------------- path tracer, overhead sun
def test_path_tracer_overhead_sun_is_black_under_a_black_sky():
    """mode 0 with a black sky: the direct term is the only light, and the NaN tangent zeroes it on every hit"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*pyhr.blue_noise())
    ctx.build_scene(sc)
    pt = pyhr.PathTracerPass(ctx, W, H)
    pt.params.sky_color[0], pt.params.sky_color[1], pt.params.sky_color[2] = 0.0, 0.0, 0.0
    opt = O.PathTracerOracle(W, H, sky=(0.0, 0.0, 0.0))
    f = pyhr.make_frame(*LC.SCENES["shadows_test"][2], W, H, light=LC.light(LC.BY_ID["sun_overhead"]))
    for i in range(2):
        pt.render(f)
        want = f16(opt.render(ss, f))
        assert np.array_equal(pt.download(1), opt.prim)
        hit = opt.prim != 0xFFFFFFFF
        got = f16(pt.download(100))
        assert hit.mean() > 0.2
        assert not want[hit][:, :3].any() and not got[hit][:, :3].any(), f"sample {i}: a lit hit"
    pt.destroy()
    ctx.close()
