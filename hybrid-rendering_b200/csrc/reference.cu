// reference.cu — converged references of the shadows, AO and reflections signals (hr_reference_render, include/hr_api.h).
// One thread per pixel of the full-resolution G-buffer runs a loop over `samples` rays of the pass it references: the ray of
// K1 or K7 (mask_ray, mask_px.cuh, which trace.cu calls too) or K12's sample (refl_ddgi_sample, shade_px.cuh, and refl_trace_shade below),
// with the same G-buffer inputs and parameters.  Only the random numbers differ: (r0, r1) of global sample k come from the xoroshiro64* stream of gi_common.cuh seeded with (x, y, k),
// so any split of the samples over renders traces the same rays.  Mapping and CTA size as K1 / K12 (RowSet, a band): warp = 8x4 pixel
// block, 2-warp CTAs (ray costs are heavy-tailed, trace.cu).
//
// BUILD NOTE: compiled with -fmad=false, like trace.cu and rt_shade.cu: the rays, the hits and the binary visibilities follow
// the deterministic chain (det_math.cuh), so the shadows / AO counts equal the CPU oracle's bit for bit.
#include "glsl_fast.cuh"
#include "mask_px.cuh"
#include "shade_px.cuh"

namespace {

__device__ __forceinline__ void ref_random(int x, int y, uint32_t k, float& r0, float& r1)
{
    gi::RNG rng = gi::rng_init((uint32_t)x, (uint32_t)y, k);
    r0 = gi::next_float(rng);
    r1 = gi::next_float(rng);
}

// MODE 0 = shadows (K1: p0 = bias), 1 = AO (K7: p0 = ray length, p1 = bias).  count[pixel] += unoccluded rays of samples k0 .. k0 + n - 1.
template <int MODE>
__global__ void __launch_bounds__(64) k_reference_mask(GBufLevelDev g, BvhDev bvh, FrameConsts fc, float p0, float p1, uint32_t k0, int n, int row0, int row1,
                                                       uint32_t* __restrict__ count)
{
    int x, y;
    RowSet::band(row0, row1).pixel(x, y);
    uint32_t hits = 0, traced = 0;
    if (x < g.W && y < row1)
    {
        const size_t idx   = (size_t)y * g.W + x;
        const float  depth = __ldg(g.depth + idx);
        if (depth != 1.0f)
        {
            const float  u = ((float)x + 0.5f) / (float)g.W, v = ((float)y + 0.5f) / (float)g.H;
            const V3     P = det::world_position_from_depth(u, v, depth, fc.view_proj_inverse);
            const float2 e = __half22float2(*reinterpret_cast<const __half2*>(g.gb2 + idx));
            const V3     N = det::octohedral_to_direction(e.x, e.y);
#pragma unroll 1
            for (int s = 0; s < n; s++)
            {
                float r0, r1;
                ref_random(x, y, k0 + (uint32_t)s, r0, r1);
                Ray r;
                if (mask_ray<MODE>(fc, P, N, p0, p1, r0, r1, r)) { traced++; hits += trace_any(bvh, r) ? 0u : 1u; }
            }
            count[idx] += hits;
        }
    }
    count_rays(fc.ray_ctr, 0, traced);
}

// The traced branches of K12's sample (mirror, GGX): the closest hit along r shaded without the sky light (with the DDGI and IBL terms
// when gi_on), or the sky colour on a miss; counts the ray.  The statement of k_reflections_ray_trace's loop body (rt_shade.cu), written
// there too: K12 calling this function compiles to different SASS in four of its six instantiations, so K12 keeps its own copy and
// test_gpu_reference.py holds this one to K12's output on mirror pixels, bit for bit.
template <bool TEX>
__device__ __forceinline__ void refl_trace_shade(const BvhDev& bvh, const ShadeDev& sd, const tex::TexDev& T, const FrameConsts& fc, const Ray& r, float3 sky, bool gi_on,
                                                 const hr_ddgi_uniforms& d, const gi::AtlasDev& at, float gi_intensity, IblDev ibl, float3& color)
{
    float    t, hu, hv;
    uint32_t prim;
    count_rays(fc.ray_ctr, 0, 1u);
    if (trace_closest(bvh, r, t, prim, hu, hv))
    {
        color = TEX ? shade_hit_tex(bvh, sd, T, fc.light, r, prim, hu, hv, false, 0.0f, 0.0f, sky, gi_on, d, at, gi_intensity, fc.ray_ctr, ibl)
                    : shade_hit(bvh, sd, fc.light, r, prim, hu, hv, false, 0.0f, 0.0f, sky, gi_on, d, at, gi_intensity, fc.ray_ctr, ibl);
    }
    else color = sky;
}

// K12's sample: the mirror ray (roughness < 0.05), the DDGI lookup (roughness > 0.75 with approximate_with_ddgi) or the GGX lobe
// sample, shaded like K12 and clamped to 0.7 per channel.  acc[6 * pixel] += (sum r, g, b, sum of squares r, g, b) in float64.
// The mirror and DDGI samples do not depend on k: they are evaluated once and added n times.
template <bool TEX, bool GI>
__global__ void __launch_bounds__(64) k_reference_reflections(GBufLevelDev g, BvhDev bvh, ShadeDev sd, FrameConsts fc, hr_ddgi_uniforms d, gi::AtlasDev at,
                                                              ReflTraceParams P, uint32_t k0, int n, double* __restrict__ acc, tex::TexDev T)
{
    int x, y;
    RowSet::band(P.rows.row0, P.rows.row1).pixel(x, y);
    if (x >= g.W || y >= P.rows.row1) return;
    const size_t idx   = (size_t)y * g.W + x;
    const float  depth = __ldg(g.depth + idx);
    if (depth == 1.0f) return;
    const float  u = ((float)x + 0.5f) / (float)g.W, v = ((float)y + 0.5f) / (float)g.H;
    const uint2  g2 = __ldg(g.gb2 + idx), g3 = __ldg(g.gb3 + idx);
    const float2 e  = __half22float2(*reinterpret_cast<const __half2*>(&g2.x));
    const float  roughness = __half22float2(*reinterpret_cast<const __half2*>(&g3.x)).x;
    const V3     Pw = det::world_position_from_depth(u, v, depth, fc.view_proj_inverse);
    const V3     N  = det::octohedral_to_direction(e.x, e.y);
    const V3     Wo = det::normalize(det::sub(det::mk(fc.cam_pos[0], fc.cam_pos[1], fc.cam_pos[2]), Pw));
    const float3 sky = make_float3(P.sky[0], P.sky[1], P.sky[2]);
    const bool   approx_ddgi = GI && P.approximate_with_ddgi == 1, gi_on = GI && P.sample_gi == 1;
    const bool   mirror = roughness < 0.05f, ddgi = !mirror && roughness > 0.75f && approx_ddgi;
    double s[3] = { 0, 0, 0 }, q[3] = { 0, 0, 0 };
#pragma unroll 1
    for (int i = 0; i < ((mirror || ddgi) ? 1 : n); i++)
    {
        float3 color;
        if (ddgi) color = refl_ddgi_sample(d, at, Pw, N, Wo, P.rough_ddgi_intensity);
        else
        {
            Ray r;
            r.o    = det::add(Pw, det::scale(N, P.bias));
            r.tmin = 0.001f;
            r.tmax = 10000.0f;
            if (mirror) r.d = reflect(det::scale(Wo, -1.0f), N);
            else
            {
                float r0, r1;
                ref_random(x, y, k0 + (uint32_t)i, r0, r1);
                r.d = reflect(det::scale(Wo, -1.0f), importance_sample_ggx(r0 * P.trim, r1 * P.trim, N, roughness));
            }
            refl_trace_shade<TEX>(bvh, sd, T, fc, r, sky, gi_on, d, at, P.gi_intensity, P.ibl, color);
        }
        const double c[3] = { fminf(color.x, 0.7f), fminf(color.y, 0.7f), fminf(color.z, 0.7f) };
        for (int ch = 0; ch < 3; ch++) { s[ch] += c[ch]; q[ch] += c[ch] * c[ch]; }
    }
    if (mirror || ddgi)
        for (int ch = 0; ch < 3; ch++) { s[ch] *= (double)n; q[ch] *= (double)n; }
    double* a = acc + 6 * idx;
    for (int ch = 0; ch < 3; ch++) { a[ch] += s[ch]; a[3 + ch] += q[ch]; }
}

// Bernoulli counts: the unbiased variance of the samples is m (1 - m) N / (N - 1)
__device__ __forceinline__ float stderr_of(double sum, double sq, double N)
{
    if (N < 2.0) return 0.0f;
    const double m = sum / N, var = fmax(0.0, (sq - sum * m) / (N - 1.0));
    return (float)sqrt(var / N);
}

// MEAN / STDERR images of rows [row0, row1) from the accumulators.  C = 1: count (sum = sum of squares); C = 4: acc.  Sky pixels
// (depth 1) get sky_value (C = 1) or (0, 0, 0, 1); power != 0: MEAN = pow_pos(mean, power) (the FINAL's transform, gf::pow_pos).
template <int C>
__global__ void __launch_bounds__(256) k_reference_resolve(GBufLevelDev g, const uint32_t* __restrict__ count, const double* __restrict__ acc, double N,
                                                           float sky_value, float power, int row0, int row1, void* __restrict__ mean, void* __restrict__ err)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= g.W || y >= row1) return;
    const size_t idx = (size_t)y * g.W + x;
    const bool   sky = __ldg(g.depth + idx) == 1.0f;
    if constexpr (C == 1)
    {
        const double c = (double)count[idx];
        float        m = sky ? sky_value : (float)(c / N);
        if (!sky && power != 0.0f) m = gf::pow_pos(m, power);
        reinterpret_cast<__half*>(mean)[idx] = __float2half_rn(m);
        reinterpret_cast<__half*>(err)[idx]  = __float2half_rn(sky ? 0.0f : stderr_of(c, c, N));
    }
    else
    {
        const double* a = acc + 6 * idx;
        float         m[3], s[3];
        for (int ch = 0; ch < 3; ch++)
        {
            m[ch] = sky ? 0.0f : (float)(a[ch] / N);
            s[ch] = sky ? 0.0f : stderr_of(a[ch], a[3 + ch], N);
        }
        reinterpret_cast<uint2*>(mean)[idx] = pack_h4(m[0], m[1], m[2], 1.0f);
        reinterpret_cast<uint2*>(err)[idx]  = pack_h4(s[0], s[1], s[2], 0.0f);
    }
}

} // namespace

void launch_reference_mask(int kind, const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, uint32_t k0, int n, RowSet rows,
                           uint32_t* count, cudaStream_t st)
{
    if (rows.empty(g.H)) return;
    const auto k = kind == PASS_AO ? k_reference_mask<1> : k_reference_mask<0>;
    k<<<rows.grid(g.W, g.H), 64, 0, st>>>(g, bvh, fc, p0, p1, k0, n, rows.row0, rows.row1, count);
}

void launch_reference_reflections(const hr_scene* sc, const GBufLevelDev& g, const FrameConsts& fc, const ReflGi& gi, const hr_reflections_params& prm,
                                  const void* brdf_lut, uint32_t k0, int n, RowSet rows, double* acc, cudaStream_t st)
{
    if (rows.empty(g.H)) return;
    const ReflLaunch L    = refl_launch(gi, prm, brdf_lut, rows); // K12's GI = false kernel: no DDGI lookups, no IBL term
    const dim3       grid = rows.grid(g.W, g.H);
#define HR_REF_ARGS g, hr_bvh_view(sc), shade_view(sc), fc, L.d, L.at, L.P, k0, n, acc, sc->tex
    if (sc->tex.n_textures > 0)
    {
        if (L.gi) k_reference_reflections<true, true><<<grid, 64, 0, st>>>(HR_REF_ARGS);
        else k_reference_reflections<true, false><<<grid, 64, 0, st>>>(HR_REF_ARGS);
    }
    else if (L.gi) k_reference_reflections<false, true><<<grid, 64, 0, st>>>(HR_REF_ARGS);
    else k_reference_reflections<false, false><<<grid, 64, 0, st>>>(HR_REF_ARGS);
#undef HR_REF_ARGS
}

void launch_reference_resolve(const GBufLevelDev& g, const uint32_t* count, const double* acc, uint32_t n_samples, float sky_value, float power, int row0, int row1,
                              void* mean, void* err, cudaStream_t st)
{
    if (row1 <= row0) return;
    const dim3 grid((g.W + 31) / 32, (row1 - row0 + 7) / 8, 1);
    if (count) k_reference_resolve<1><<<grid, 256, 0, st>>>(g, count, nullptr, (double)n_samples, sky_value, power, row0, row1, mean, err);
    else k_reference_resolve<4><<<grid, 256, 0, st>>>(g, nullptr, acc, (double)n_samples, 0.0f, 0.0f, row0, row1, mean, err);
}
