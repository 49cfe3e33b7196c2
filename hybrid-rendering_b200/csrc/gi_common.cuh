// gi_common.cuh — device restatement of src/shaders/gi/gi_common.glsl (probe grid addressing + sample_irradiance,
// :10-320) and random.glsl:17-56.  Tolerance-checked maths (colours); usable from both fast-math and -fmad=false files.
#pragma once
#include "../../include/hr_api.h"
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace gi {

struct AtlasDev {
    const uint2*    irr;   // RGBA16F, irradiance_texture_width x irradiance_texture_height
    const uint32_t* depth; // RG16F,   depth_texture_width x depth_texture_height
};

__device__ __forceinline__ float3 f3(float x, float y, float z) { return make_float3(x, y, z); }
__device__ __forceinline__ float3 operator+(float3 a, float3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 operator-(float3 a, float3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 operator*(float3 a, float s) { return f3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float3 operator*(float3 a, float3 b) { return f3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ __forceinline__ float  dot(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float  length(float3 a) { return sqrtf(dot(a, a)); }
__device__ __forceinline__ float3 normalize(float3 a) { const float inv = 1.0f / sqrtf(dot(a, a)); return a * inv; }

// ---- random.glsl:17-56 -----------------------------------------------------------------------------------------------
struct RNG { uint32_t sx, sy; };
__device__ __forceinline__ uint32_t rng_rotl(uint32_t x, uint32_t k) { return (x << k) | (x >> (32 - k)); }
__device__ __forceinline__ uint32_t rng_next(RNG& r)
{
    const uint32_t result = r.sx * 0x9e3779bbu;
    r.sy ^= r.sx;
    r.sx = rng_rotl(r.sx, 26) ^ r.sy ^ (r.sy << 9);
    r.sy = rng_rotl(r.sy, 13);
    return result;
}
__device__ __forceinline__ uint32_t rng_hash(uint32_t seed)
{
    seed = (seed ^ 61u) ^ (seed >> 16);
    seed *= 9u;
    seed = seed ^ (seed >> 4);
    seed *= 0x27d4eb2du;
    seed = seed ^ (seed >> 15);
    return seed;
}
__device__ __forceinline__ RNG rng_init(uint32_t idx, uint32_t idy, uint32_t frame_index)
{
    RNG r;
    r.sx = rng_hash((idx << 16) | idy);
    r.sy = rng_hash(frame_index);
    rng_next(r);
    return r;
}
__device__ __forceinline__ float next_float(RNG& r) { return __uint_as_float(0x3f800000u | (rng_next(r) >> 9)) - 1.0f; }

// ---- gi_common.glsl ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sign_not_zero(float k) { return k >= 0.0f ? 1.0f : -1.0f; }
__device__ __forceinline__ float2 oct_encode(float3 v)
{
    const float inv = 1.0f / (fabsf(v.x) + fabsf(v.y) + fabsf(v.z));
    float2      r   = make_float2(v.x * inv, v.y * inv);
    if (v.z < 0.0f) r = make_float2((1.0f - fabsf(r.y)) * sign_not_zero(r.x), (1.0f - fabsf(r.x)) * sign_not_zero(r.y));
    return r;
}
__device__ __forceinline__ float3 oct_decode(float2 o)
{
    float3 v = f3(o.x, o.y, 1.0f - fabsf(o.x) - fabsf(o.y));
    if (v.z < 0.0f)
    {
        const float nx = (1.0f - fabsf(v.y)) * sign_not_zero(v.x), ny = (1.0f - fabsf(v.x)) * sign_not_zero(v.y);
        v.x = nx;
        v.y = ny;
    }
    return normalize(v);
}
__device__ __forceinline__ float2 texture_coord_from_direction(float3 dir, int probe_index, int tex_w, int tex_h, int side)
{
    const float2 o  = oct_encode(normalize(dir));
    const float  pb = (float)side + 2.0f;
    const int    ppr = (tex_w - 2) / (side + 2);
    const float  tlx = (float)(probe_index % ppr) * pb + 2.0f, tly = (float)(probe_index / ppr) * pb + 2.0f;
    return make_float2(tlx / (float)tex_w + ((o.x + 1.0f) * 0.5f * (float)side) / (float)tex_w, tly / (float)tex_h + ((o.y + 1.0f) * 0.5f * (float)side) / (float)tex_h);
}
// bilinear sampler, CLAMP_TO_EDGE, texel centres at +0.5 (ddgi.cpp:478,499)
__device__ __forceinline__ void bilinear_setup(float u, float v, int W, int H, int& x0, int& x1, int& y0, int& y1, float& fx, float& fy)
{
    const float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
    const float fx0 = floorf(x), fy0 = floorf(y);
    fx = x - fx0;
    fy = y - fy0;
    x0 = min(max((int)fx0, 0), W - 1); x1 = min(max((int)fx0 + 1, 0), W - 1);
    y0 = min(max((int)fy0, 0), H - 1); y1 = min(max((int)fy0 + 1, 0), H - 1);
}
__device__ __forceinline__ float2 h2f2(uint32_t w) { return __half22float2(*reinterpret_cast<const __half2*>(&w)); }
__device__ __forceinline__ float2 sample_depth_atlas(const uint32_t* __restrict__ t, int W, int H, float2 uv)
{
    int   x0, x1, y0, y1;
    float fx, fy;
    bilinear_setup(uv.x, uv.y, W, H, x0, x1, y0, y1, fx, fy);
    const float2 a = h2f2(__ldg(t + (size_t)y0 * W + x0)), b = h2f2(__ldg(t + (size_t)y0 * W + x1));
    const float2 c = h2f2(__ldg(t + (size_t)y1 * W + x0)), d = h2f2(__ldg(t + (size_t)y1 * W + x1));
    return make_float2((a.x * (1.0f - fx) + b.x * fx) * (1.0f - fy) + (c.x * (1.0f - fx) + d.x * fx) * fy,
                       (a.y * (1.0f - fx) + b.y * fx) * (1.0f - fy) + (c.y * (1.0f - fx) + d.y * fx) * fy);
}
__device__ __forceinline__ float3 sample_irr_atlas(const uint2* __restrict__ t, int W, int H, float2 uv)
{
    int   x0, x1, y0, y1;
    float fx, fy;
    bilinear_setup(uv.x, uv.y, W, H, x0, x1, y0, y1, fx, fy);
    const uint2  ta = __ldg(t + (size_t)y0 * W + x0), tb = __ldg(t + (size_t)y0 * W + x1), tc = __ldg(t + (size_t)y1 * W + x0), td = __ldg(t + (size_t)y1 * W + x1);
    const float2 a0 = h2f2(ta.x), a1 = h2f2(ta.y), b0 = h2f2(tb.x), b1 = h2f2(tb.y), c0 = h2f2(tc.x), c1 = h2f2(tc.y), d0 = h2f2(td.x), d1 = h2f2(td.y);
    auto mix2 = [&](float a, float b, float c, float d) { return (a * (1.0f - fx) + b * fx) * (1.0f - fy) + (c * (1.0f - fx) + d * fx) * fy; };
    return f3(mix2(a0.x, b0.x, c0.x, d0.x), mix2(a0.y, b0.y, c0.y, d0.y), mix2(a1.x, b1.x, c1.x, d1.x));
}

// Per-atlas constants of texture_coord_from_direction hoisted out of the 8-probe loop (reciprocals instead of the
// reference's divisions, float reciprocal for the probe's column / row: exact for probe indices below 2^22).
struct AtlasGeom { float inv_w, inv_h, side, pb, inv_ppr; int ppr, W, H; };
__device__ __forceinline__ AtlasGeom atlas_geom(int tex_w, int tex_h, int side)
{
    AtlasGeom a;
    a.W = tex_w; a.H = tex_h;
    a.inv_w = __fdividef(1.0f, (float)tex_w);
    a.inv_h = __fdividef(1.0f, (float)tex_h);
    a.side  = (float)side;
    a.pb    = (float)side + 2.0f;
    a.ppr   = (tex_w - 2) / (side + 2);
    a.inv_ppr = __fdividef(1.0f, (float)a.ppr);
    return a;
}
__device__ __forceinline__ float3 normalize_fast(float3 a) { return a * rsqrtf(dot(a, a)); }
__device__ __forceinline__ float2 oct_encode_fast(float3 v)
{
    const float inv = __fdividef(1.0f, fabsf(v.x) + fabsf(v.y) + fabsf(v.z));
    float2      r   = make_float2(v.x * inv, v.y * inv);
    if (v.z < 0.0f) r = make_float2((1.0f - fabsf(r.y)) * sign_not_zero(r.x), (1.0f - fabsf(r.x)) * sign_not_zero(r.y));
    return r;
}
// dir must be normalised (oct_encode is scale invariant, so the reference's normalize(dir) is a no-op up to rounding)
__device__ __forceinline__ float2 texture_coord_fast(float3 dir, int probe_index, const AtlasGeom& a)
{
    const float2 o   = oct_encode_fast(dir);
    const int    row = (int)(((float)probe_index + 0.5f) * a.inv_ppr), col = probe_index - row * a.ppr;
    const float  tlx = (float)col * a.pb + 2.0f, tly = (float)row * a.pb + 2.0f;
    return make_float2((tlx + (o.x + 1.0f) * 0.5f * a.side) * a.inv_w, (tly + (o.y + 1.0f) * 0.5f * a.side) * a.inv_h);
}

// sqrt(x) as x * rsqrt(x).  The rsqrt argument is clamped to the finite range: at x = +inf (an atlas texel that saturated fp16,
// DESIGN.md §6) the product is then inf, the reference's sqrt(inf), not inf * rsqrt(inf) = inf * 0 = NaN, which
// sample_irradiance's NaN guard would turn into a finite 0.5.  Finite x are unchanged.
__device__ __forceinline__ float sqrt_mul_rsqrt(float x) { return x * rsqrtf(fminf(fmaxf(x, 1e-30f), 3.402823466e38f)); }

// sample_irradiance, gi_common.glsl:188-320 (LINEAR_BLENDING undefined => sqrt-space blend).  A tolerance-checked colour
// stage: reciprocal square roots / approximate reciprocals replace the IEEE sqrt + divide sequences (the IEEE forms made
// K21 instruction-bound), the per-atlas constants are hoisted, and the probe loop is unrolled UNR
// times so the 8 atlas fetches of independent probes are in flight together.
template <int UNR = 1>
__device__ inline float3 sample_irradiance(const hr_ddgi_uniforms& d, const AtlasDev& at, float3 P, float3 N, float3 Wo)
{
    const float3 start = f3(d.grid_start_position[0], d.grid_start_position[1], d.grid_start_position[2]);
    const float3 step  = f3(d.grid_step[0], d.grid_step[1], d.grid_step[2]);
    const float3 istep = f3(__fdividef(1.0f, step.x), __fdividef(1.0f, step.y), __fdividef(1.0f, step.z));
    int base[3];
    base[0] = min(max((int)((P.x - start.x) / step.x), 0), d.probe_counts[0] - 1); // exact divisions: they pick the probe cell
    base[1] = min(max((int)((P.y - start.y) / step.y), 0), d.probe_counts[1] - 1);
    base[2] = min(max((int)((P.z - start.z) / step.z), 0), d.probe_counts[2] - 1);
    const float3 base_pos = f3(step.x * (float)base[0] + start.x, step.y * (float)base[1] + start.y, step.z * (float)base[2] + start.z);
    const float3 alpha    = f3(__saturatef((P.x - base_pos.x) * istep.x), __saturatef((P.y - base_pos.y) * istep.y), __saturatef((P.z - base_pos.z) * istep.z));
    const AtlasGeom gd = atlas_geom(d.depth_texture_width, d.depth_texture_height, d.depth_probe_side_length);
    const AtlasGeom gi_ = atlas_geom(d.irradiance_texture_width, d.irradiance_texture_height, d.irradiance_probe_side_length);
    const float3 bias_v = (N + Wo * 3.0f) * d.normal_bias;
    const float3 Nn     = normalize_fast(N);
    float3 sum_irr = f3(0, 0, 0);
    float  sum_w   = 0.0f;
#pragma unroll UNR
    for (int i = 0; i < 8; ++i)
    {
        const int off0 = i & 1, off1 = (i >> 1) & 1, off2 = (i >> 2) & 1;
        const int g0 = min(base[0] + off0, d.probe_counts[0] - 1), g1 = min(base[1] + off1, d.probe_counts[1] - 1), g2 = min(base[2] + off2, d.probe_counts[2] - 1);
        const int p  = g0 + g1 * d.probe_counts[0] + g2 * d.probe_counts[0] * d.probe_counts[1];
        const float3 probe_pos      = f3(step.x * (float)g0 + start.x, step.y * (float)g1 + start.y, step.z * (float)g2 + start.z);
        const float3 probe_to_point = (P - probe_pos) + bias_v;
        const float  ptp2           = dot(probe_to_point, probe_to_point);
        const float  inv_len        = rsqrtf(ptp2);
        const float3 tri            = f3(off0 ? alpha.x : 1.0f - alpha.x, off1 ? alpha.y : 1.0f - alpha.y, off2 ? alpha.z : 1.0f - alpha.z);
        float weight = 1.0f;
        {
            const float3 tdir = normalize_fast(probe_pos - P);
            const float  t    = fmaxf(0.0001f, (dot(tdir, N) + 1.0f) * 0.5f);
            weight *= t * t + 0.2f;
        }
        if (d.visibility_test == 1)
        {
            // texture_coord_from_direction(-dir) with dir = normalize(-probe_to_point)
            const float2 tc   = texture_coord_fast(probe_to_point * inv_len, p, gd);
            const float  dist = ptp2 * inv_len;
            const float2 t2   = sample_depth_atlas(at.depth, gd.W, gd.H, tc);
            const float  mean = t2.x, variance = fabsf(t2.x * t2.x - t2.y);
            const float  dm   = fmaxf(dist - mean, 0.0f);
            float        cheb = __fdividef(variance, variance + dm * dm);
            cheb              = fmaxf(cheb * cheb * cheb, 0.0f);
            weight *= (dist <= mean) ? 1.0f : cheb;
        }
        weight = fmaxf(0.000001f, weight);
        const float2 tc = texture_coord_fast(Nn, p, gi_);
        const float3 pi = sample_irr_atlas(at.irr, gi_.W, gi_.H, tc);
        if (weight < 0.2f) weight *= weight * weight * (1.0f / (0.2f * 0.2f));
        weight *= tri.x * tri.y * tri.z;
        sum_irr = sum_irr + f3(sqrt_mul_rsqrt(pi.x), sqrt_mul_rsqrt(pi.y), sqrt_mul_rsqrt(pi.z)) * weight;
        sum_w += weight;
    }
    const float inv_w = __fdividef(1.0f, sum_w);
    float3      net   = sum_irr * inv_w;
    if (!(net.x == net.x)) net.x = 0.5f;
    if (!(net.y == net.y)) net.y = 0.5f;
    if (!(net.z == net.z)) net.z = 0.5f;
    net = net * net;
    net = net * d.energy_preservation;
    return net * (0.5f * 3.14159265359f);
}

} // namespace gi
