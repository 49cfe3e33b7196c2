// rt_shade.cu — the two closest-hit ray-trace stages with hit shading.
//   K18 gi/gi_ray_trace.{rgen,rchit,rmiss}                     (256 rays / probe -> radiance + direction/distance images)
//   K12 reflections/reflections_ray_trace.{rgen,rchit,rmiss}   (1 reflection ray / pixel -> RGBA16F colour + ray length)
// Hit shading: fetch_triangle / interpolated_vertex (scene_descriptor_set.glsl:117-160), direct_lighting
// (lighting.glsl:117-196) with its shadow ray, evaluate_uber_brdf (brdf.glsl:130-142), DDGI infinite bounce
// (gi_common.glsl:188-320), in shade_px.cuh.  Environment = constant colour (sky cubemap / IBL assets are not in the repository).
//
// BUILD NOTE: compiled with -fmad=false.  Everything that decides *which surface is hit or whether a shadow ray is
// blocked* (ray directions, hit point, shading normal, shadow-ray origin) follows the deterministic fp32 rules of
// det_math.cuh so that the binary visibility inside the shading is identical to the CPU oracle's; colours are
// tolerance-checked.
#include "shade_px.cuh"

namespace {

// gi_ray_trace.rgen:61-72
__device__ __forceinline__ V3 spherical_fibonacci(float i, float n)
{
    const float PHI = sqrtf(5.0f) * 0.5f + 0.5f;
    const float a   = i * (PHI - 1.0f);
    const float phi = 2.0f * 3.14159265359f * (a - floorf(a));
    const float ct  = 1.0f - (2.0f * i + 1.0f) * (1.0f / n);
    const float st  = sqrtf(det::clampf(1.0f - ct * ct, 0.0f, 1.0f));
    float       sn, cs;
    det::det_sincos(phi, &sn, &cs);
    return det::mk(cs * st, sn * st, ct);
}

struct GiTraceParams { float rot[16]; uint32_t num_frames, infinite_bounces; float gi_intensity; float sky[3]; int probe0, probe1; unsigned long long* ray_ctr; };

// K18: one block per probe, one thread per ray (blockDim = rays_per_probe rounded up to 32, looped if > 256)
template <bool TEX>
__global__ void __launch_bounds__(256) k_ddgi_ray_trace(BvhDev bvh, ShadeDev sd, hr_ddgi_uniforms d, gi::AtlasDev at, hr_light light, GiTraceParams P,
                                                         uint2* __restrict__ radiance, uint2* __restrict__ dirdepth, tex::TexDev T)
{
    const int probe = P.probe0 + blockIdx.x;
    if (probe >= P.probe1) return;
    const int cx = d.probe_counts[0], cxy = d.probe_counts[0] * d.probe_counts[1];
    const V3  origin = det::mk(d.grid_step[0] * (float)(probe % cx) + d.grid_start_position[0], d.grid_step[1] * (float)((probe % cxy) / cx) + d.grid_start_position[1],
                               d.grid_step[2] * (float)(probe / cxy) + d.grid_start_position[2]);
    const float3 sky = make_float3(P.sky[0], P.sky[1], P.sky[2]);
    for (int ray = threadIdx.x; ray < d.rays_per_probe; ray += blockDim.x)
    {
        const V3 sf = spherical_fibonacci((float)ray, (float)d.rays_per_probe);
        Ray      r;
        r.o = origin;
        r.d = det::normalize(det::mk((P.rot[0] * sf.x + P.rot[4] * sf.y) + P.rot[8] * sf.z, (P.rot[1] * sf.x + P.rot[5] * sf.y) + P.rot[9] * sf.z,
                                     (P.rot[2] * sf.x + P.rot[6] * sf.y) + P.rot[10] * sf.z));
        r.tmin = 0.001f;
        r.tmax = 10000.0f;
        gi::RNG  rng = gi::rng_init((uint32_t)ray, (uint32_t)probe, P.num_frames);
        float    t, u, v, hit_distance = 10000.0f;
        uint32_t prim;
        float3   L;
        count_rays(P.ray_ctr, 0, 1u);
        if (trace_closest(bvh, r, t, prim, u, v))
        {
            const float r0 = gi::next_float(rng), r1 = gi::next_float(rng);
            L              = TEX ? shade_hit_tex(bvh, sd, T, light, r, prim, u, v, true, r0, r1, sky, P.infinite_bounces == 1, d, at, P.gi_intensity, P.ray_ctr)
                                 : shade_hit(bvh, sd, light, r, prim, u, v, true, r0, r1, sky, P.infinite_bounces == 1, d, at, P.gi_intensity, P.ray_ctr);
            hit_distance   = 0.001f + t;
        }
        else L = sky;
        const size_t o = (size_t)probe * d.rays_per_probe + ray;
        radiance[o] = pack_h4(L.x, L.y, L.z, 0.0f);
        dirdepth[o] = pack_h4(r.d.x, r.d.y, r.d.z, hit_distance);
    }
}

// K12: warp = 8x4 pixel block (coherent reflection rays), 256 threads = 32x8 pixels
// 2-warp CTAs (16x4 pixels): closest-hit rays + hit shading are heavy-tailed, small CTAs recycle their slots sooner (trace.cu)
// MULTI = false: exactly the reference's one ray per pixel (straight-line code); true: the spp > 1 extension (sample loop)
// MINB: resident 2-warp CTAs per SM the registers are tuned for.  One ray per pixel: 24 (40 registers) without DDGI, 18 (56) with
// it.  Config 3 at 4K on an H100 SXM 80 GB (700 W power limit), the GI = false kernel, K12 per frame: 16 -> 2.68 ms, 18 -> 2.61,
// 20 -> 2.55, 24 -> 2.47: the kernel is latency-bound, resident warps buy more than registers (and than the spills the smaller
// register budgets cost).
// GI = false: sample_gi and approximate_with_ddgi are both off, so the kernel is compiled without the DDGI lookups and the IBL term
// (IBL is only added with sample_gi); their live values would otherwise set the register allocation around the two traversals.
// GI = true: both terms behind their run-time flags.
template <bool MULTI, int MINB, bool TEX, bool GI>
__global__ void __launch_bounds__(64, MINB) k_reflections_ray_trace(GBufLevelDev g, BvhDev bvh, ShadeDev sd, FrameConsts fc, hr_ddgi_uniforms d, gi::AtlasDev at,
                                                                ReflTraceParams P, const uint8_t* __restrict__ sobol, const uint8_t* __restrict__ srk,
                                                                uint2* __restrict__ out, tex::TexDev T)
{
    int x, y;
    P.rows.pixel(x, y);
    if (x >= g.W || y >= g.H || P.rows.past_end(y)) return;
    const size_t idx   = (size_t)y * g.W + x;
    const float  depth = __ldg(g.depth + idx);
    if (depth == 1.0f) { out[idx] = pack_h4(0.0f, 0.0f, 0.0f, -1.0f); return; }
    const float  u = ((float)x + 0.5f) / (float)g.W, v = ((float)y + 0.5f) / (float)g.H;
    const uint2  g2 = __ldg(g.gb2 + idx), g3 = __ldg(g.gb3 + idx);
    const float2 e  = __half22float2(*reinterpret_cast<const __half2*>(&g2.x));
    const float  roughness = __half22float2(*reinterpret_cast<const __half2*>(&g3.x)).x;
    const V3     Pw = det::world_position_from_depth(u, v, depth, fc.view_proj_inverse);
    const V3     N  = det::octohedral_to_direction(e.x, e.y);
    const V3     Wo = det::normalize(det::sub(det::mk(fc.cam_pos[0], fc.cam_pos[1], fc.cam_pos[2]), Pw));
    const float3 sky = make_float3(P.sky[0], P.sky[1], P.sky[2]);
    Ray          r;
    r.o    = det::add(Pw, det::scale(N, P.bias));
    r.tmin = 0.001f;
    r.tmax = 10000.0f;
    float3 color = make_float3(0, 0, 0);
    float  ray_length = -1.0f;
    // spp > 1 (SURVEY.md §8d): the GGX lobe draws spp directions, the clamped radiance is averaged, ray_length = first sample's
    const int  spp = MULTI ? (P.spp > 1 ? P.spp : 1) : 1;
    const bool approx_ddgi = GI && P.approximate_with_ddgi == 1, gi_on = GI && P.sample_gi == 1;
    const bool ggx = !(roughness < 0.05f) && !(roughness > 0.75f && approx_ddgi);
    const int  n_s = MULTI ? (ggx ? spp : 1) : 1;
    float3     acc = make_float3(0, 0, 0);
#pragma unroll 1
    for (int s = 0; s < n_s; s++)
    {
        bool trace = false;
        if (roughness < 0.05f) { r.d = reflect(det::scale(Wo, -1.0f), N); trace = true; }
        else if (roughness > 0.75f && approx_ddgi) color = refl_ddgi_sample(d, at, Pw, N, Wo, P.rough_ddgi_intensity);
        else
        {
            const uint32_t si = fc.num_frames * (uint32_t)spp + (uint32_t)s;
            const float ex = det::sample_blue_noise(x, y, si, 0, sobol, srk) * P.trim;
            const float ey = det::sample_blue_noise(x, y, si, 1, sobol, srk) * P.trim;
            const V3    Wh = importance_sample_ggx(ex, ey, N, roughness);
            r.d   = reflect(det::scale(Wo, -1.0f), Wh);
            trace = true;
        }
        if (trace)
        {
            float    t, hu, hv;
            uint32_t prim;
            count_rays(fc.ray_ctr, 0, 1u);
            if (trace_closest(bvh, r, t, prim, hu, hv))
            {
                color = TEX ? shade_hit_tex(bvh, sd, T, fc.light, r, prim, hu, hv, false, 0.0f, 0.0f, sky, gi_on, d, at, P.gi_intensity, fc.ray_ctr, P.ibl)
                            : shade_hit(bvh, sd, fc.light, r, prim, hu, hv, false, 0.0f, 0.0f, sky, gi_on, d, at, P.gi_intensity, fc.ray_ctr, P.ibl);
                if (s == 0) ray_length = 0.001f + t;
            }
            else color = sky;
        }
        acc = make_float3(acc.x + fminf(color.x, 0.7f), acc.y + fminf(color.y, 0.7f), acc.z + fminf(color.z, 0.7f));
    }
    const float inv_n = 1.0f / (float)n_s;
    out[idx] = pack_h4(acc.x * inv_n, acc.y * inv_n, acc.z * inv_n, ray_length);
}

// ---------------------------------------------------------------------------------------------------------------------------
// Ground-truth progressive path tracer (SURVEY.md §8 f4): ground_truth/ground_truth_path_trace.{rgen,rchit,rmiss}, host
// src/ground_truth_path_tracer.cpp:44-113.  One jittered primary ray per pixel and frame; closest hit -> direct_lighting with SOFT_SHADOWS +
// RAY_THROUGHPUT + SAMPLE_SKY_LIGHT (rchit:13-16): the punctual light sampled on its disk with its shadow ray, one cosine-lobe sky sample
// with its shadow ray; miss -> the sky colour; running average into an RGBA16F image.  As written in the reference the indirect bounce's
// traceRayEXT is commented out (rchit:92-104) and indirect_lighting returns p_IndirectPayload.L = vec3(0): the image converges to direct +
// sky lighting; max_ray_bounces only gates that dead branch.  trace_indirect = 1 (DESIGN.md §7) traces the bounces up to max_ray_bounces
// vertices.  The primary ray, the hit, the two shadow rays and the bounces follow the deterministic chain (det_math.cuh): hit primitives,
// paths and binary visibilities equal the oracle's (oracle/orc_path_trace.cpp, orc_path_trace_indirect.cpp) exactly, colours within tolerance.
struct PathTraceParams {
    float    view_inverse[16], proj_inverse[16];
    hr_light light;
    uint32_t num_frames, max_ray_bounces;
    float    roughness_multiplier;
    float    sky[3];
    int      W, H;
    unsigned long long* ray_ctr;
    RowSet   rows;
};

__device__ __forceinline__ float4 mat_vec4(const float* M, float x, float y, float z, float w)
{ // mat4 * vec4, row r = ((m0r*x + m1r*y) + m2r*z) + m3r*w (oracle/orc_math.h::mul)
    return make_float4(((M[0] * x + M[4] * y) + M[8] * z) + M[12] * w, ((M[1] * x + M[5] * y) + M[9] * z) + M[13] * w,
                       ((M[2] * x + M[6] * y) + M[10] * z) + M[14] * w, ((M[3] * x + M[7] * y) + M[11] * z) + M[15] * w);
}

// direct_lighting, lighting.glsl:117-196 with SOFT_SHADOWS and SAMPLE_SKY_LIGHT at one path vertex (rchit:112-141): draws the light's disk
// sample, then the sky sample (two next_vec2), traces their shadow rays; the throughput (RAY_THROUGHPUT) is applied by the caller
__device__ __forceinline__ float3 path_direct_lighting(const BvhDev& bvh, const PathTraceParams& P, const Surface& s, float roughness, V3 Wo, float3 F0, float3 cd,
                                                       float3 sky, gi::RNG& rng)
{
    using namespace gi;
    const float r1x = next_float(rng), r1y = next_float(rng); // next_vec2: the light's disk sample
    const float r2x = next_float(rng), r2y = next_float(rng); // next_vec2: the sky sample
    float3 Lo = f3(0, 0, 0);
    Ray    sr;
    sr.o    = det::add(s.P, det::scale(s.N, 0.1f));
    sr.tmin = 0.01f;
    {
        const hr_light& light = P.light;
        const float3    Li = make_float3(light.data2[0] * light.data0[3], light.data2[1] * light.data0[3], light.data2[2] * light.data0[3]);
        V3    Wi;
        float t_max, att;
        det::fetch_light_properties_shadow(light, s.P, s.N, r1x, r1y, Wi, t_max, att);
        const V3 Wh = det::normalize(det::add(Wo, Wi));
        if (att > 0.0f)
        {
            sr.d    = Wi;
            sr.tmax = t_max;
            count_rays(P.ray_ctr, 1, 1u);
            att *= trace_any(bvh, sr) ? 0.0f : 1.0f;
        }
        Lo = Lo + (evaluate_uber_brdf(cd, roughness, s.N, F0, Wo, Wh, Wi) * att) * Li;
    }
    {
        const V3 Wi = det::sample_cosine_lobe(s.N, r2x, r2y);
        const V3 Wh = det::normalize(det::add(Wo, Wi));
        sr.d    = Wi;
        sr.tmax = 10000.0f;
        count_rays(P.ray_ctr, 1, 1u);
        const float vis = trace_any(bvh, sr) ? 0.0f : 1.0f;
        Lo = Lo + evaluate_uber_brdf(cd, roughness, s.N, F0, Wo, Wh, Wi) * (sky * vis);
    }
    return Lo;
}

// path-hash end codes (HR_PATH_TRACER_OUT_PATH_HASH)
constexpr uint32_t PT_END_MISS = 0xFFFFFFFFu, PT_END_HORIZON = 0xFFFFFFFEu, PT_END_MAX_BOUNCES = 0xFFFFFFFDu;
__device__ __forceinline__ uint32_t fnv1a(uint32_t h, uint32_t w) { return (h ^ w) * 16777619u; }

// One sampled continuation at a path vertex (trace_indirect = 1, DESIGN.md §7).  Lobe choice, direction and horizon tests are geometry
// (det_math.cuh); the throughput factor is (as-written lobe value) * N.Wi / (lobe probability * sampler pdf), evaluated without a closed-form
// simplification because D_ggx's 1e-4 denominator clamp is active near the highlight.  false: the path ends (below the horizon, or a
// specular sample whose pdf is not positive, e.g. roughness 0 where the as-written D_ggx is 0 everywhere).
__device__ __forceinline__ bool sample_bounce(V3 N, V3 Wo, float3 F0, float3 cd, float roughness, float metallic, float u, float e1, float e2, V3& Wi, float3& weight)
{
    using namespace gi;
    const float p_spec = 0.5f + 0.5f * det::clampf(metallic, 0.0f, 1.0f);
    const bool  spec   = u < p_spec;
    Wi = spec ? reflect(det::scale(Wo, -1.0f), importance_sample_ggx(e1, e2, N, roughness)) : det::sample_cosine_lobe(N, e1, e2);
    if (det::dot(N, Wi) <= 0.0f || det::dot(N, Wo) <= 0.0f) return false;
    const V3     Wh    = det::normalize(det::add(Wo, Wi));
    const float  NdotL = fmaxf(det::dot(N, Wi), 0.0f), NdotV = fmaxf(det::dot(N, Wo), 0.0f), NdotH = fmaxf(det::dot(N, Wh), 0.0f), VdotH = fmaxf(det::dot(Wi, Wh), 0.0f);
    const float  p5    = powf(1.0f - VdotH, 5.0f);
    const float3 F     = F0 + (f3(1, 1, 1) - F0) * p5;
    if (spec)
    {
        const float a2  = (roughness * roughness) * (roughness * roughness), dd = (NdotH * NdotH) * (a2 - 1.0f) + 1.0f;
        const float pdf = p_spec * ((a2 / (3.14159265359f * dd * dd)) * NdotH / (4.0f * VdotH)); // D_true(NH) NH / (4 VH), unclamped GGX
        if (!(pdf > 0.0f)) return false;
        const float sv = D_ggx(NdotH, roughness * roughness) * (G1_schlick_ggx(roughness, NdotL) * G1_schlick_ggx(roughness, NdotV)) / fmaxf(0.0001f, 4.0f * NdotL * NdotV);
        weight = F * (sv * NdotL / pdf);
    }
    else
    {
        const float pdf = (1.0f - p_spec) * (NdotL / 3.14159265359f);
        weight = ((f3(1, 1, 1) - F) * (cd * (1.0f / 3.14159265359f))) * (NdotL / pdf);
    }
    return true;
}

// warp = 8x4 pixel block (coherent primary rays), 2-warp CTAs like K12
// INDIRECT = false: the reference as written (one vertex).  true: trace_indirect = 1, a per-lane bounce loop over up to max_ray_bounces
// vertices (the wavefront split lost for K12 on this card, DESIGN.md §8); out_hash gets the path hash
template <bool TEX, bool INDIRECT>
__global__ void __launch_bounds__(64) k_path_trace(BvhDev bvh, ShadeDev sd, PathTraceParams P, const uint2* __restrict__ prev, uint2* __restrict__ out, uint32_t* __restrict__ out_prim,
                                                   tex::TexDev T, uint32_t* __restrict__ out_hash)
{
    // The RNG is seeded from (x, y, sample): no result depends on the rank.
    int x, y;
    P.rows.pixel(x, y);
    if (x >= P.W || y >= P.H || P.rows.past_end(y)) return;
    const size_t idx = (size_t)y * P.W + x;
    // rgen:56-75
    gi::RNG     rng = gi::rng_init((uint32_t)x, (uint32_t)y, P.num_frames);
    const float j0 = gi::next_float(rng), j1 = gi::next_float(rng);
    const float jx = ((float)x + 0.5f) + j0, jy = ((float)y + 0.5f) + j1;    // pixel_coord + vec2(next_float, next_float)
    const float tx = jx / (float)P.W, ty = jy / (float)P.H;                   // tex_coord
    const float nx = tx * 2.0f - 1.0f, ny = ty * 2.0f - 1.0f;                 // tex_coord_neg_to_pos
    const float4 origin = mat_vec4(P.view_inverse, 0.0f, 0.0f, 0.0f, 1.0f);
    const float4 target = mat_vec4(P.proj_inverse, nx, ny, 1.0f, 1.0f);
    const V3     tn     = det::normalize(det::mk(target.x, target.y, target.z));
    const float4 dir    = mat_vec4(P.view_inverse, tn.x, tn.y, tn.z, 0.0f);
    Ray r;
    r.o = det::mk(origin.x, origin.y, origin.z);
    r.d = det::mk(dir.x, dir.y, dir.z);
    r.tmin = 0.001f;
    r.tmax = 10000.0f;
    const float3 sky = make_float3(P.sky[0], P.sky[1], P.sky[2]);
    float3   L = sky; // rmiss:29-32 at depth 0
    float    t, hu, hv;
    uint32_t prim = 0xFFFFFFFFu;
    count_rays(P.ray_ctr, 0, 1u);
    if (!INDIRECT)
    {
        if (trace_closest(bvh, r, t, prim, hu, hv))
        { // rchit:112-141
            using namespace gi;
            const Surface s  = TEX ? fetch_surface_tex(sd, T, prim, hu, hv) : fetch_surface(sd, prim, hu, hv);
            const float   roughness = s.roughness * P.roughness_multiplier;
            const V3      Wo = det::scale(r.d, -1.0f);
            const float3  F0 = f3(0.04f, 0.04f, 0.04f) * (1.0f - s.metallic) + s.albedo * s.metallic;
            const float3  cd = (s.albedo * (f3(1, 1, 1) - F0)) * (1.0f - s.metallic) + f3(0, 0, 0) * s.metallic;
            // RAY_THROUGHPUT: T = 1 at depth 0
            L = path_direct_lighting(bvh, P, s, roughness, Wo, F0, cd, sky, rng); // + indirect_lighting(...) = vec3(0): the bounce is commented out in the reference (rchit:92-106)
        }
    }
    else
    {
        uint32_t hash = 2166136261u, end = PT_END_MISS;
        if (trace_closest(bvh, r, t, prim, hu, hv))
        {
            using namespace gi;
            float3   Tp = f3(1, 1, 1);
            uint32_t hp = prim;
            L = f3(0, 0, 0);
#pragma unroll 1
            for (uint32_t k = 0;; k++)
            {
                hash = fnv1a(hash, hp);
                const Surface s  = TEX ? fetch_surface_tex(sd, T, hp, hu, hv) : fetch_surface(sd, hp, hu, hv);
                const float   roughness = s.roughness * P.roughness_multiplier;
                const V3      Wo = det::scale(r.d, -1.0f);
                const float3  F0 = f3(0.04f, 0.04f, 0.04f) * (1.0f - s.metallic) + s.albedo * s.metallic;
                const float3  cd = (s.albedo * (f3(1, 1, 1) - F0)) * (1.0f - s.metallic) + f3(0, 0, 0) * s.metallic;
                L = L + Tp * path_direct_lighting(bvh, P, s, roughness, Wo, F0, cd, sky, rng);
                if (k + 1 == P.max_ray_bounces) { end = PT_END_MAX_BOUNCES; break; }
                const float u = next_float(rng), e1 = next_float(rng), e2 = next_float(rng);
                float3      weight;
                V3          Wi;
                if (!sample_bounce(s.N, Wo, F0, cd, roughness, s.metallic, u, e1, e2, Wi, weight)) { end = PT_END_HORIZON; break; }
                Tp     = Tp * weight;
                r.o    = det::add(s.P, det::scale(s.N, 0.1f)); // the shadow-ray origin, lighting.glsl:143
                r.d    = Wi;
                r.tmin = 0.001f;
                r.tmax = 10000.0f;
                count_rays(P.ray_ctr, 1, 1u);
                if (!trace_closest(bvh, r, t, hp, hu, hv)) { end = PT_END_MISS; break; } // rmiss adds the environment at depth 0 only
            }
        }
        out_hash[idx] = fnv1a(hash, end);
    }
    // rgen:94-111: clamp to RADIANCE_CLAMP_COLOR = 1, then the running average the reference writes (weight 1 / num_frames, not 1 / (n + 1))
    const float3 c = make_float3(fminf(L.x, 1.0f), fminf(L.y, 1.0f), fminf(L.z, 1.0f));
    float3 o = c;
    if (P.num_frames != 0)
    {
        const uint2  pw = __ldg(prev + idx);
        const float2 p01 = __half22float2(*reinterpret_cast<const __half2*>(&pw.x)), p2 = __half22float2(*reinterpret_cast<const __half2*>(&pw.y));
        const float  n = (float)P.num_frames;
        o = make_float3(p01.x + (c.x - p01.x) / n, p01.y + (c.y - p01.y) / n, p2.x + (c.z - p2.x) / n);
    }
    out[idx] = pack_h4(o.x, o.y, o.z, 1.0f);
    out_prim[idx] = prim;
}

} // namespace

void launch_ddgi_ray_trace(const hr_scene* sc, const hr_ddgi_uniforms& d, const void* irr_prev, const void* depth_prev, const hr_light& light, const float* rot16,
                           uint32_t num_frames, uint32_t infinite_bounces, float gi_intensity, const float* sky3, int probe0, int probe1, void* radiance,
                           void* dirdepth, unsigned long long* ray_ctr, cudaStream_t st)
{
    if (probe1 <= probe0) return;
    GiTraceParams P;
    memcpy(P.rot, rot16, 64);
    P.num_frames = num_frames; P.infinite_bounces = infinite_bounces; P.gi_intensity = gi_intensity;
    P.sky[0] = sky3[0]; P.sky[1] = sky3[1]; P.sky[2] = sky3[2];
    P.probe0 = probe0; P.probe1 = probe1;
    P.ray_ctr = ray_ctr;
    gi::AtlasDev at { (const uint2*)irr_prev, (const uint32_t*)depth_prev };
    int threads = d.rays_per_probe < 256 ? ((d.rays_per_probe + 31) / 32) * 32 : 256;
    if (sc->tex.n_textures > 0) k_ddgi_ray_trace<true><<<probe1 - probe0, threads, 0, st>>>(hr_bvh_view(sc), shade_view(sc), d, at, light, P, (uint2*)radiance, (uint2*)dirdepth, sc->tex);
    else k_ddgi_ray_trace<false><<<probe1 - probe0, threads, 0, st>>>(hr_bvh_view(sc), shade_view(sc), d, at, light, P, (uint2*)radiance, (uint2*)dirdepth, sc->tex);
}

void launch_reflections_ray_trace(const hr_scene* sc, const GBufLevelDev& g, const FrameConsts& fc, const ReflGi& gi, const hr_reflections_params& prm,
                                  const void* brdf_lut, const uint8_t* sobol, const uint8_t* srk, void* out, RowSet rows, cudaStream_t st)
{
    if (rows.empty(g.H)) return;
    const ReflLaunch L        = refl_launch(gi, prm, brdf_lut, rows); // L.gi: the spp > 1 kernels keep both terms behind their flags
    const bool       textured = sc->tex.n_textures > 0; // material textures: the TEX instantiations
    const dim3       grid     = rows.grid(g.W, g.H);
#define HR_K12_ARGS g, hr_bvh_view(sc), shade_view(sc), fc, L.d, L.at, L.P, sobol, srk, (uint2*)out, sc->tex
    if (textured)
    {
        if (L.P.spp > 1) k_reflections_ray_trace<true, 8, true, true><<<grid, 64, 0, st>>>(HR_K12_ARGS);
        else if (L.gi) k_reflections_ray_trace<false, 18, true, true><<<grid, 64, 0, st>>>(HR_K12_ARGS);
        else k_reflections_ray_trace<false, 24, true, false><<<grid, 64, 0, st>>>(HR_K12_ARGS);
    }
    else if (L.P.spp > 1) k_reflections_ray_trace<true, 8, false, true><<<grid, 64, 0, st>>>(HR_K12_ARGS);
    else if (L.gi) k_reflections_ray_trace<false, 18, false, true><<<grid, 64, 0, st>>>(HR_K12_ARGS);
    else k_reflections_ray_trace<false, 24, false, false><<<grid, 64, 0, st>>>(HR_K12_ARGS);
#undef HR_K12_ARGS
}

void launch_path_trace(const hr_scene* sc, const hr_frame* f, const hr_path_tracer_params& prm, int W, int H, uint32_t num_frames, const void* prev, void* out,
                       uint32_t* out_prim, uint32_t* out_hash, unsigned long long* ray_ctr, RowSet rows, cudaStream_t st)
{
    if (rows.empty(H)) return;
    PathTraceParams P;
    memcpy(P.view_inverse, f->ubo.view_inverse, 64);
    memcpy(P.proj_inverse, f->ubo.proj_inverse, 64);
    P.light = f->ubo.light;
    P.num_frames = num_frames; P.max_ray_bounces = (uint32_t)prm.max_ray_bounces; P.roughness_multiplier = prm.roughness_multiplier;
    P.sky[0] = prm.sky_color[0]; P.sky[1] = prm.sky_color[1]; P.sky[2] = prm.sky_color[2];
    P.W = W; P.H = H;
    P.ray_ctr = ray_ctr;
    P.rows = rows;
    const dim3 grid = rows.grid(W, H);
#define HR_PT_ARGS hr_bvh_view(sc), shade_view(sc), P, (const uint2*)prev, (uint2*)out, out_prim, sc->tex
    const bool textured = sc->tex.n_textures > 0; // material textures change the lobe inputs: both indirect forms have a TEX instantiation
    if (prm.trace_indirect)
    {
        if (textured) k_path_trace<true, true><<<grid, 64, 0, st>>>(HR_PT_ARGS, out_hash);
        else k_path_trace<false, true><<<grid, 64, 0, st>>>(HR_PT_ARGS, out_hash);
    }
    else if (textured) k_path_trace<true, false><<<grid, 64, 0, st>>>(HR_PT_ARGS, nullptr);
    else k_path_trace<false, false><<<grid, 64, 0, st>>>(HR_PT_ARGS, nullptr);
#undef HR_PT_ARGS
}
