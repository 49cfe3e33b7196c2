// det_math.cuh — deterministic fp32 device math for the visibility-mask chain (ray generation + ray/triangle).
//
// The reference computes these steps in GLSL (shadows_ray_trace.comp:89-132, ao_ray_trace.comp:90-126,
// lighting.glsl:6-111, brdf.glsl:8-32, common.glsl:150-184, bnd_sampler.glsl:4-24) on a GPU driver; BASELINE.json asks
// for a bit-exact visibility mask, so this chain is specified as a fixed sequence of IEEE-754 binary32 operations:
// + - * / sqrt correctly rounded, no implicit FMA contraction (this translation unit is compiled with -fmad=false),
// fmaf only where written, sin/cos via det_sincos.  Everything here must be used ONLY from files built with -fmad=false.
#pragma once
#include "../../include/hr_api.h"
#include <cuda_runtime.h>
#include <stdint.h>

namespace det {

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 mk(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ V3 add(V3 a, V3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ V3 sub(V3 a, V3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ V3 scale(V3 a, float s) { return mk(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float dot(V3 a, V3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float length(V3 a) { return sqrtf(dot(a, a)); }
__device__ __forceinline__ V3 normalize(V3 a) { float inv = 1.0f / sqrtf(dot(a, a)); return scale(a, inv); }
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }

// k = floor(x*(2/pi)+0.5); r = fma(-k,PIO2_HI,x); r = fma(-k,PIO2_LO,r); fixed minimax polynomials (Cephes sinf/cosf).
__device__ __forceinline__ void det_sincos(float x, float* sn, float* cs)
{
    const float kf = floorf(x * 0.636619772367581343f + 0.5f);
    float       r  = fmaf(-kf, 1.57079625129699707031f, x);
    r              = fmaf(-kf, 7.54978941586159635335e-08f, r);
    const float s  = r * r;
    float       ps = fmaf(s, -1.9515295891e-4f, 8.3321608736e-3f);
    ps             = fmaf(ps, s, -1.6666654611e-1f);
    const float sr = fmaf(r * s, ps, r);
    float       pc = fmaf(s, 2.443315711809948e-5f, -1.388731625493765e-3f);
    pc             = fmaf(pc, s, 4.166664568298827e-2f);
    const float cr = fmaf(s * s, pc, fmaf(s, -0.5f, 1.0f));
    const int   q  = ((int)kf) & 3;
    float       sv = (q & 1) ? cr : sr;
    float       cv = (q & 1) ? sr : cr;
    if (q == 1 || q == 2) cv = -cv;
    if (q >= 2) sv = -sv;
    *sn = sv;
    *cs = cv;
}

// common.glsl:150-156
__device__ __forceinline__ V3 octohedral_to_direction(float ex, float ey)
{
    V3 v = mk(ex, ey, 1.0f - fabsf(ex) - fabsf(ey));
    if (v.z < 0.0f)
    {
        const float nx = (1.0f - fabsf(v.y)) * ((v.x < 0.0f ? 0.0f : 1.0f) * 2.0f - 1.0f);
        const float ny = (1.0f - fabsf(v.x)) * ((v.y < 0.0f ? 0.0f : 1.0f) * 2.0f - 1.0f);
        v.x = nx;
        v.y = ny;
    }
    return normalize(v);
}

// common.glsl:169-184; M column-major, row r = ((m0r*x + m1r*y) + m2r*z) + m3r*w
__device__ __forceinline__ V3 world_position_from_depth(float u, float v, float ndc_depth, const float* M)
{
    const float sx = u * 2.0f - 1.0f, sy = v * 2.0f - 1.0f;
    const float wx = ((M[0] * sx + M[4] * sy) + M[8] * ndc_depth) + M[12];
    const float wy = ((M[1] * sx + M[5] * sy) + M[9] * ndc_depth) + M[13];
    const float wz = ((M[2] * sx + M[6] * sy) + M[10] * ndc_depth) + M[14];
    const float ww = ((M[3] * sx + M[7] * sy) + M[11] * ndc_depth) + M[15];
    return mk(wx / ww, wy / ww, wz / ww);
}

// bnd_sampler.glsl:4-24 on raw bytes
// sample_index: num_frames * spp + s in uint32 arithmetic (DESIGN.md §7), defined for every hr_frame::num_frames
__device__ __forceinline__ float sample_blue_noise(int x, int y, uint32_t sample_index, int dim, const uint8_t* __restrict__ sobol,
                                                   const uint8_t* __restrict__ sr)
{
    x &= 127;
    y &= 127;
    sample_index &= 255u;
    dim &= 3;
    const uint8_t* t     = sr + 4 * (y * 128 + x);
    const int      rsi   = (int)sample_index ^ (int)t[2];
    int            value = (int)sobol[4 * rsi + dim];
    value ^= (int)t[dim & 1];
    return (0.5f + (float)value) / 256.0f;
}

// lighting.glsl:39-47
__device__ __forceinline__ V3 soft_shadow_dir(V3 light_dir, float radius, float r0, float r1)
{
    const V3    tangent   = normalize(cross(light_dir, mk(0.0f, 1.0f, 0.0f)));
    const V3    bitangent = normalize(cross(tangent, light_dir));
    const float pr        = radius * sqrtf(r0);
    const float pa        = r1 * 2.0f * 3.14159265359f;
    float       sn, cs;
    det_sincos(pa, &sn, &cs);
    const float dx = pr * cs, dy = pr * sn;
    return normalize(add(add(light_dir, scale(tangent, dx)), scale(bitangent, dy)));
}

// lighting.glsl:6-111, SOFT_SHADOWS + SHADOW_RAY_ONLY + RAY_TRACING
__device__ __forceinline__ void fetch_light_properties_shadow(const hr_light& L, V3 P, V3 N, float r0, float r1, V3& Wi, float& t_max, float& attenuation)
{
    const int type = (int)L.data3[0];
    const V3  ldir = mk(L.data0[0], L.data0[1], L.data0[2]);
    if (type == 0)
    {
        Wi          = soft_shadow_dir(ldir, L.data1[3], r0, r1);
        t_max       = 10000.0f;
        attenuation = 1.0f;
    }
    else
    {
        const V3    to_light = sub(mk(L.data1[0], L.data1[1], L.data1[2]), P);
        const V3    ld       = normalize(to_light);
        const float dist     = length(to_light);
        Wi                   = soft_shadow_dir(ld, L.data1[3] / dist, r0, r1);
        t_max                = dist;
        if (type == 1) attenuation = 1.0f / (dist * dist);
        else
        {
            float       a = dot(Wi, ldir);
            const float e0 = L.data3[1], e1 = L.data3[2];
            const float t = clampf((a - e0) / (e1 - e0), 0.0f, 1.0f);
            a             = t * t * (3.0f - 2.0f * t);
            attenuation   = a / (dist * dist);
        }
    }
    attenuation *= clampf(dot(N, Wi), 0.0f, 1.0f);
}

// brdf.glsl:8-32
__device__ __forceinline__ V3 sample_cosine_lobe(V3 n, float r0, float r1)
{
    r0 = fmaxf(0.00001f, r0);
    r1 = fmaxf(0.00001f, r1);
    const float phi = 2.0f * 3.14159265359f * r1;
    const float ct  = sqrtf(r0);
    const float st  = sqrtf(1.0f - r0);
    float       sn, cs;
    det_sincos(phi, &sn, &cs);
    const V3 t   = mk(st * cs, st * sn, ct);
    const V3 ref = fabsf(dot(n, mk(0.0f, 1.0f, 0.0f))) > 0.99f ? mk(0.0f, 0.0f, 1.0f) : mk(0.0f, 1.0f, 0.0f);
    const V3 bx  = normalize(cross(ref, n));
    const V3 by  = cross(n, bx);
    return normalize(add(add(scale(bx, t.x), scale(by, t.y)), scale(n, t.z)));
}

} // namespace det
