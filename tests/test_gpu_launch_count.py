"""hr_ctx_launch_count (bench.py's gpu_launches) counts every kernel a render launches, once.

For one render of each pass kind, the counter's delta must equal the number of kernels torch.profiler records (memcpy and memset
are not kernels).  The render measured is a pass's second, which reads history; the linked ranks are measured on their first
frame too, which waits on no history tick.  Scene builds are left out: cub's radix sort launches kernels of its own that the
library does not count.
"""
import pytest
import torch

import pyhr
from test_gpu_ragged import CAM_SHADOWS_TEST, COVERAGE, kernels_launched, new_context, set_params

pytestmark = pytest.mark.gpu

W, H = 256, 144


def check_counted(ctxs, run, what):
    """the counter's delta over `run` equals the kernels it launched (a render profiled again is a new render: same check)"""
    counted = []

    def counted_run():
        before = [c.launch_count() for c in ctxs]
        run()
        counted[:] = [sum(c.launch_count() - b for c, b in zip(ctxs, before))]
    names = kernels_launched(counted_run)
    assert counted[0] == len(names), f"{what}: the launch counter went up by {counted[0]}, {len(names)} kernels ran: {sorted(names)}"


def make_pass(ctx, kind, w, h, scale, params=None):
    p = pyhr.ReflectionsPass(ctx, w, h, scale) if kind == "reflections" else pyhr.Pass(ctx, kind, w, h, scale)
    set_params([p.params], params)
    return p


def render(p, f, stream=0):
    if p.kind == "reflections":
        p.render(f, None, stream)
    else:
        p.render(f, stream)


def frames(w, h, n=2):
    f = None
    for i in range(n):
        f = pyhr.make_frame(*CAM_SHADOWS_TEST, w, h, prev=f, num_frames=i)
        yield i, f


KINDS = ("shadows", "ao", "reflections")
CASES = ([(f"{k} defaults scale {s}", (k, W, H, s, None)) for k in KINDS for s in (0, 1)]
         + [(f"{k} spp 2", (k, W, H, 1, dict(spp=2))) for k in KINDS]
         + [(f"{k} denoise 0", (k, W, H, 1, dict(denoise=0))) for k in KINDS]
         + [(c[0], c[1]) for c in COVERAGE])  # every fallback kernel of the dispatch


@pytest.mark.parametrize("case,setup", CASES, ids=[c[0] for c in CASES])
def test_render_launches_counted(case, setup):
    kind, w, h, scale, params = setup
    ctx = new_context(pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST), w, h)
    p = make_pass(ctx, kind, w, h, scale, params)
    for i, f in frames(w, h):
        ctx.gbuffer_render(f.ping_pong, f)
        if i == 0:
            render(p, f)
        else:
            check_counted([ctx], lambda: render(p, f), case)
    p.destroy()
    ctx.close()


@pytest.mark.parametrize("kind,scale", [("shadows", 0), ("ao", 1), ("reflections", 1)])
def test_linked_pair_launches_counted(kind, scale):
    """two ranks emulated on one GPU and linked with hr_shard_link_local (test_gpu_multi): cooperative ray trace, pushes, ticks"""
    sc = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST)
    ranks = []
    for r in range(2):
        c = new_context(sc, W, H)
        c.shard_config(r, 2)
        ranks.append((c, make_pass(c, kind, W, H, scale)))
    ranks[0][1].link_local(1, ranks[1][1])
    ranks[1][1].link_local(0, ranks[0][1])
    streams = [torch.cuda.Stream() for _ in ranks]  # linked ranks wait for each other inside a frame: they must run concurrently
    for i, f in frames(W, H):
        for c, _ in ranks:
            c.gbuffer_render(f.ping_pong, f)

        def run():
            for (_, p), st in zip(ranks, streams):
                render(p, f, st.cuda_stream)
        check_counted([c for c, _ in ranks], run, f"{kind} linked pair, frame {i}")
    for _, p in ranks:
        p.destroy()
    for c, _ in ranks:
        c.close()


def test_other_passes_launches_counted():
    """DDGI (with reflections reading its atlas), deferred, TAA, tone map and the path tracer at their defaults; the DDGI probe
    spacing is the one the parity tests use on this scene"""
    ctx = new_context(pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST), W, H)
    dd, rf = pyhr.DDGIPass(ctx, W, H, 1), pyhr.ReflectionsPass(ctx, W, H, 1)
    dd.params.probe_distance = 4.0
    sh, ao = pyhr.Pass(ctx, "shadows", W, H, 0), pyhr.Pass(ctx, "ao", W, H, 1)
    de, taa, tm, pt = pyhr.DeferredPass(ctx, W, H), pyhr.TAAPass(ctx, W, H), pyhr.TonemapPass(ctx, W, H), pyhr.PathTracerPass(ctx, W, H)
    for i, f in frames(W, H):
        ctx.gbuffer_render(f.ping_pong, f)
        rot = pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))
        for name, run in (("ddgi", lambda: dd.render(f, rot)), ("reflections with ddgi", lambda: rf.render(f, dd)), ("shadows", lambda: sh.render(f)),
                          ("ao", lambda: ao.render(f)), ("deferred", lambda: de.render(f, sh, ao, rf, None)), ("taa", lambda: taa.render(f, de)),
                          ("tone map", lambda: tm.render(taa)), ("path tracer", lambda: pt.render(f))):
            if i == 0:
                run()
            else:
                check_counted([ctx], run, name)
    for p in (pt, tm, taa, de, ao, sh, rf, dd):
        p.destroy()
    ctx.close()
