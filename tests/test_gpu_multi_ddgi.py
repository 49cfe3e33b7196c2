"""DDGI across linked ranks (DESIGN.md §9): N ranks emulated on one GPU (one hr_ctx and one stream per rank) and linked with
hr_shard_link_local trace and update the probes of their z-slices [cz * r / world, cz * (r + 1) / world) and store those atlas rows
into every peer's atlas.  After every frame each rank's irradiance and depth atlases must equal the single-GPU atlases bit for bit,
and so must its band of the K21 sample and of the half-resolution reflections that read the atlas (linked too).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle as O  # noqa: F401  (path setup)
import pyhr
from param_cases import LAYOUTS, SCENES
from test_gpu_launch_count import check_counted
from test_textures_cpu import textured_scene

pytestmark = pytest.mark.gpu

W, H = 256, 144
SKY = (0.3, 0.4, 0.6)
HR_ERR_INVALID_ARG = -1
DD = dict(irradiance=2, depth=3, sample=100)


def frames(n, cam=((0.0, 14.0, 34.0), (0.0, 3.0, 0.0)), pan_from=2, vertical=0.35):
    """a static start, then a vertical pan (the reflections' reprojection taps cross band borders)"""
    (px, py, pz), (tx, ty, tz) = cam
    f = None
    for i in range(n):
        dx = 0.0 if i < pan_from else 0.05 * (i - pan_from + 1)
        dy = 0.0 if i < pan_from else vertical * (i - pan_from + 1)
        f = pyhr.make_frame((px + dx, py + dy, pz), (tx + dx, ty - dy, tz), W, H, prev=f, num_frames=i)
        yield i, f


def rot(i):
    return pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))


class Rank:
    def __init__(self, scene, params, textures=None, rank=0, world=1, refl=True):
        self.c = c = pyhr.Context(0)
        c.set_bluenoise(*pyhr.blue_noise())
        self.set_scene(scene, textures)
        c.gbuffer_create(W, H)
        if world > 1:
            c.shard_config(rank, world)
        self.dd = pyhr.DDGIPass(c, W, H, 0)
        self.dd.params.normal_bias = 1.0
        self.dd.params.sky_color[0], self.dd.params.sky_color[1], self.dd.params.sky_color[2] = SKY
        for k, v in params.items():
            setattr(self.dd.params, k, v)
        self.rf = None
        if refl:
            self.rf = pyhr.ReflectionsPass(c, W, H, 1)
            self.rf.params.sky_color[0], self.rf.params.sky_color[1], self.rf.params.sky_color[2] = SKY

    def set_scene(self, scene, textures=None):
        s = self.c.build_scene(scene)  # hr_scene_build + hr_scene_set_current
        if textures is not None:
            self.c.set_textures(s, *textures)

    def passes(self):
        return [p for p in (self.dd, self.rf) if p is not None]

    def render(self, i, f, stream=0):
        self.c.gbuffer_render(f.ping_pong, f, stream=stream)
        self.dd.render(f, rot(i), stream)
        if self.rf is not None:
            self.rf.render(f, self.dd, stream)

    def close(self):
        for p in self.passes():
            p.destroy()
        self.c.close()


def linked(scene, params, world, textures=None, refl=True):
    ref = Rank(scene, params, textures, refl=refl)
    ranks = [Rank(scene, params, textures, r, world, refl) for r in range(world)]
    for r in range(world):
        for q in range(world):
            if q != r:
                for p, peer in zip(ranks[r].passes(), ranks[q].passes()):
                    p.link_local(q, peer)
    return ref, ranks


def slices(ref, rank, world):
    u = ref.dd.uniforms()
    cz, cxy = u.probe_counts[2], u.probe_counts[0] * u.probe_counts[1]
    return cz * rank // world, cz * (rank + 1) // world, cxy


def differing_rows(a, b):
    rows = np.nonzero(np.any((a != b).reshape(a.shape[0], -1), axis=1))[0]
    return f"{len(rows)} rows differ, first {rows[:4].tolist()}, last {rows[-4:].tolist()}, of {a.shape[0]}"


def check_frame(ref, ranks, world, what):
    """every rank's atlases whole, its bands of the K21 sample and of the reflections' FINAL, and its primary rays"""
    want = {k: ref.dd.download(w) for k, w in DD.items()}
    want_rf = ref.rf.download(100) if ref.rf is not None else None
    rays = ref.dd.params.rays_per_probe
    total = ref.dd.stats().rays_primary
    primary = 0
    for r, rk in enumerate(ranks):
        at = f"{what}, rank {r}"
        for k in ("irradiance", "depth"):
            got = rk.dd.download(DD[k])
            assert np.array_equal(got, want[k]), f"{at}: {k} atlas differs from the single-GPU atlas ({differing_rows(got, want[k])})"
        b, e = pyhr.shard_rows(H, r, world)
        assert np.array_equal(rk.dd.download(DD["sample"])[b:e], want["sample"][b:e]), f"{at}: K21 sample differs on the band"
        if want_rf is not None:
            hb, he = pyhr.shard_rows(H >> 1, r, world)
            fb, fe = hb << 1, (H if he >= H >> 1 else he << 1)
            assert np.array_equal(rk.rf.download(100)[fb:fe], want_rf[fb:fe]), f"{at}: reflections FINAL differs on the band"
        s0, s1, cxy = slices(ref, r, world)
        got = rk.dd.stats().rays_primary
        assert got == rays * cxy * (s1 - s0), f"{at}: {got} primary rays for slices [{s0}, {s1}) of {cxy} probes"
        primary += got
    assert primary == total, f"{what}: the ranks' primary rays sum to {primary}, the single GPU traced {total}"


def run(scene, params, world, n=6, textures=None, cam=None, between=None, refl=True):
    """n frames on the single-GPU reference and the linked ranks; between(i, ref, ranks) runs before frame i on all of them"""
    ref, ranks = linked(scene, params, world, textures, refl)
    streams = [torch.cuda.Stream() for _ in range(world)]
    for rk in [ref] + ranks:
        rk.dd.stats()
    for i, f in frames(n, **(dict(cam=cam) if cam else {})):
        if between is not None:
            between(i, ref, ranks)
        ref.render(i, f)
        for rk, st in zip(ranks, streams):
            rk.render(i, f, st.cuda_stream)
        torch.cuda.synchronize()
        check_frame(ref, ranks, world, f"world={world} frame {i}")
    for rk in [ref] + ranks:
        rk.close()


@pytest.fixture(scope="module")
def shadows_scene():
    return pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_linked_ddgi_bit_identical(shadows_scene, world):
    """infinite bounce on (the default): from the second frame K18 reads every probe of last frame's atlas"""
    run(shadows_scene, dict(probe_distance=4.0, infinite_bounces=1), world)


@pytest.mark.parametrize("world", [2, 3])
def test_linked_ddgi_probe_distance_change(shadows_scene, world):
    """a probe_distance change re-initialises the grid on every rank in the same render: new atlases, published again"""
    def between(i, ref, ranks):
        if i == 3:
            for rk in [ref] + ranks:
                rk.dd.params.probe_distance = 3.0
    run(shadows_scene, dict(probe_distance=4.0), world, n=7, between=between)


@pytest.mark.parametrize("world", [2, 3])
def test_linked_ddgi_scene_replaced(shadows_scene, world):
    """hr_scene_build + hr_scene_set_current of another scene re-initialises the grid from its bounds"""
    sc2 = pyhr.SynthScene(pyhr.SCENE_ARCADE, 20000)

    def between(i, ref, ranks):
        if i == 3:
            for rk in [ref] + ranks:
                rk.set_scene(sc2)
    run(shadows_scene, dict(probe_distance=8.0), world, n=6, between=between)


def test_linked_ddgi_reinit_memory_bounded(shadows_scene):
    """a grid re-initialised on every frame (probe_distance alternating: ~30 000 probes x 256 rays, over 100 MB of grid per rank) keeps the
    device memory in use bounded: same-process ranks free each replaced grid in stream order"""
    free = []

    def between(i, ref, ranks):
        for rk in [ref] + ranks:
            rk.dd.params.probe_distance = 1.0 if i % 2 == 0 else 1.1
        if i in (3, 9):
            torch.cuda.synchronize()
            free.append(torch.cuda.mem_get_info()[0])
    run(shadows_scene, dict(probe_distance=1.0), 2, n=10, between=between, refl=False)
    assert free[0] - free[1] < 64 << 20, f"device memory in use grew by {(free[0] - free[1]) >> 20} MB over 6 grid re-initialisations"


def test_linked_ddgi_more_ranks_than_slices(shadows_scene):
    """a probe spacing wider than the scene: 2 or 3 z-slices for 5 ranks, so some ranks own no probe; they still publish their ticks"""
    def between(i, ref, ranks):
        if i == 1:
            assert ref.dd.uniforms().probe_counts[2] < 5
    run(shadows_scene, dict(probe_distance=100.0), 5, n=4, between=between)


@pytest.mark.parametrize("case", LAYOUTS, ids=[c.id for c in LAYOUTS])
def test_linked_ddgi_layouts(case):
    """the probe layouts of the parameter tests (1 / 33 / 257 / 1024 rays per probe, oct sides that are not powers of two) at world 3"""
    kind, tris, cam, _ = SCENES["arcade"]
    run(pyhr.SynthScene(kind, tris), dict(case.params), 3, n=4, cam=cam, refl=False)


def test_linked_ddgi_textured():
    """the TEX instantiation of K18 takes the slice range too"""
    sc, asc, textures, bindings = textured_scene()
    run(asc, dict(probe_distance=4.0), 3, n=4, textures=(textures, bindings))


def test_linked_ddgi_launches_counted(shadows_scene):
    """hr_ctx_launch_count equals the kernels torch.profiler records for a linked frame: the publish of the new atlases (first frame),
    K18, K19, K20, the store, the wait and K21 on every rank"""
    ref, ranks = linked(shadows_scene, dict(probe_distance=4.0), 2, refl=False)
    streams = [torch.cuda.Stream() for _ in ranks]
    for i, f in frames(2):
        for rk, st in zip(ranks, streams):
            rk.c.gbuffer_render(f.ping_pong, f, stream=st.cuda_stream)
        torch.cuda.synchronize()

        def go():
            for rk, st in zip(ranks, streams):
                rk.dd.render(f, rot(i), st.cuda_stream)
        check_counted([rk.c for rk in ranks], go, f"linked DDGI pair, frame {i}")
    for rk in [ref] + ranks:
        rk.close()


def test_linked_ddgi_refusals(shadows_scene):
    """a refused parameter block changes nothing on any rank (the next frame stays bit-identical); mismatched links are refused"""
    world = 3
    ref, ranks = linked(shadows_scene, dict(probe_distance=4.0), world)
    streams = [torch.cuda.Stream() for _ in range(world)]
    for i, f in frames(4):
        if i == 2:
            before = [(rk.dd.download(DD["irradiance"]), rk.dd.download(DD["depth"])) for rk in ranks]
            for rk in ranks:
                bad = pyhr.hr_ddgi_params()
                C.memmove(C.byref(bad), C.byref(rk.dd.params), C.sizeof(bad))
                bad.rays_per_probe = 0
                r16 = np.ascontiguousarray(rot(i), np.float32)
                rc = rk.dd.lib.hr_ddgi_render(rk.dd.h, C.byref(f), C.byref(bad), r16.ctypes.data_as(C.c_void_p), None)
                assert rc == HR_ERR_INVALID_ARG
            torch.cuda.synchronize()
            for rk, (irr, dep) in zip(ranks, before):
                assert np.array_equal(rk.dd.download(DD["irradiance"]), irr) and np.array_equal(rk.dd.download(DD["depth"]), dep)
        ref.render(i, f)
        for rk, st in zip(ranks, streams):
            rk.render(i, f, st.cuda_stream)
        torch.cuda.synchronize()
        check_frame(ref, ranks, world, f"frame {i}")
    # a DDGI pass links only with a DDGI pass of the same size
    other = pyhr.DDGIPass(ranks[1].c, W // 2, H // 2, 0)
    for peer in (ranks[1].rf, other):
        with pytest.raises(pyhr.HrError):
            ranks[0].dd.link_local(1, peer)
    other.destroy()
    for rk in [ref] + ranks:
        rk.close()
