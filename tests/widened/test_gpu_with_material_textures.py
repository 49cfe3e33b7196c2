"""GPU parity with material textures bound (hr_scene_set_textures; fetch_albedo / fetch_roughness / fetch_metallic of
scene_descriptor_set.glsl:164-218, normal maps included) through the C ABI against the oracle: the TEX instantiations of the G-buffer producer (all four images bit
for bit), the reflections and DDGI ray-trace stages (ray lengths / probe distances exact, colours within the shading tolerance) and the
ground-truth path tracer; removing the textures restores the untextured results.  The arithmetic of the texture functions themselves is
checked on the CPU (tests/test_textures_cpu.py: host build of csrc/tex_px.cuh == oracle, bit for bit).  This is one planar-UV scene;
every textured instantiation (K12 without the DDGI terms and at spp > 1 included) at the sampler's edges is compared in
tests/test_gpu_textured_kernels.py, on the cases of tests/texture_cases.py."""
import numpy as np
import pytest

import oracle as O
import pyhr
from test_gpu_gi_refl import close
from test_textures_cpu import textured_scene

pytestmark = pytest.mark.gpu

W, H = 192, 112
SKY = (0.3, 0.4, 0.6)


def f16(a):
    return np.ascontiguousarray(a).view(np.float16).astype(np.float32)


def test_textured_scene_matches_the_oracle():
    sc, asc, textures, bindings = textured_scene()
    ss = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    ss.set_textures(textures, bindings, asc.primitive_uvs(), asc.primitive_tangent_frames())
    bn = pyhr.blue_noise()
    ctx = pyhr.Context(0)
    ctx.set_bluenoise(*bn)
    scene = ctx.build_scene(asc)
    ctx.set_textures(scene, textures, bindings)
    ctx.gbuffer_create(W, H)
    mn, mx = sc.bounds()
    dd, rf, pt = pyhr.DDGIPass(ctx, W, H, 0), pyhr.ReflectionsPass(ctx, W, H, 0), pyhr.PathTracerPass(ctx, W, H)
    dd.params.probe_distance, dd.params.normal_bias = 4.0, 1.0
    for P in (dd.params, rf.params, pt.params):
        P.sky_color[0], P.sky_color[1], P.sky_color[2] = SKY
    odd, orf, opt = O.DDGIOracle(W, H, 0, dd.params, mn, mx), O.ReflectionsOracle(W, H, 0, rf.params), O.PathTracerOracle(W, H, sky=SKY)
    f, prev_g = None, O.zero_gbuf_mips(W, H)
    zero = pyhr.GBufferHost(W, H)
    ctx.gbuffer_upload(0, zero)
    ctx.gbuffer_upload(1, zero)
    for i in range(3):
        f = pyhr.make_frame((0.05 * i, 14.0, 34.0), (0.0, 3.0, 0.0), W, H, prev=f, num_frames=i)
        # G-buffer producer, TEX instantiation: bit for bit like the untextured one (tests/test_gbuffer.py)
        ctx.gbuffer_render(f.ping_pong, f)
        g = O.gbuffer_render(ss, f, W, H)
        for which, want in ((0, g.depth), (1, g.gb1), (2, g.gb2), (3, g.gb3)):
            got = ctx.gbuffer_download(f.ping_pong, 0, which, W, H)
            assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(want).view(np.uint8)), f"frame {i}: G-buffer image {which}"
        cur_g = O.GBufMips(g)
        rot = pyhr.rotation_matrix(0.7 + 1.3 * i, (0.3, 1.0, -0.5))
        dd.render(f, rot)
        odd.render(ss, cur_g, f, rot)
        dird_c = dd.download(1).view(np.uint16)
        assert np.array_equal(dird_c, odd.dirdepth.reshape(dird_c.shape)), f"frame {i}: probe ray direction / hit distance"
        close(f16(dd.download(0)), O.h2f(odd.radiance).reshape(-1, odd.u.rays_per_probe, 4), f"frame {i} ddgi radiance (textured hits)", 2e-3, 0.05)
        rf.render(f, dd)
        orf.render(ss, cur_g, prev_g, f, bn, odd)
        prev_g = cur_g
        rt_c, rt_o = f16(rf.download(0)), O.h2f(orf.rt)
        assert np.array_equal(rt_c[..., 3], rt_o[..., 3]), f"frame {i}: reflection ray length"
        close(rt_c[..., :3], rt_o[..., :3], f"frame {i} reflections ray trace (textured hits)", 1e-3, 0.02)
        pt.render(f)
        want = opt.render(ss, f)
        assert np.array_equal(pt.download(1), opt.prim)
        d = np.abs(f16(pt.download(100))[..., :3] - f16(want)[..., :3])
        assert np.mean(d.max(-1) > 2e-2) <= 2e-3 and float(np.sqrt(np.mean(np.minimum(d, 2e-2) ** 2))) <= 1e-3, f"frame {i}: path tracer"
    # the textures matter (the same frame without them differs) and can be removed again
    gb1_tex = ctx.gbuffer_download(f.ping_pong, 0, 1, W, H).copy()
    ctx.set_textures(scene, [], [])
    ctx.gbuffer_render(f.ping_pong, f)
    plain = O.ShadingScene(sc, brute=sc.n_tris <= 4096)
    g0 = O.gbuffer_render(plain, f, W, H)
    gb1_plain = ctx.gbuffer_download(f.ping_pong, 0, 1, W, H)
    assert np.array_equal(gb1_plain, g0.gb1) and not np.array_equal(gb1_plain, gb1_tex)
    # argument checks
    with pytest.raises(pyhr.HrError, match="one binding per material"):
        ctx.set_textures(scene, textures, bindings[:-1])
    bad = [dict(b) for b in bindings]
    bad[0]["albedo"] = len(textures)
    with pytest.raises(pyhr.HrError, match="index out of range"):
        ctx.set_textures(scene, textures, bad)
    for p in (dd, rf, pt):
        p.destroy()
    ctx.close()
