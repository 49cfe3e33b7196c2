// glsl_fast.cuh — device restatements of the shared GLSL includes used by the floating-point (tolerance-checked)
// denoise kernels.  Unlike det_math.cuh these may be FMA-contracted and use fast intrinsics.
//   common.glsl:143-191, edge_stopping.glsl:10-62, reprojection.glsl:11-67
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gf {

__device__ __forceinline__ float2 h2_to_f2(uint32_t w) { return __half22float2(*reinterpret_cast<const __half2*>(&w)); }
__device__ __forceinline__ uint32_t f2_to_h2(float a, float b)
{
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float4 h4_to_f4(uint2 w)
{
    const float2 a = h2_to_f2(w.x), b = h2_to_f2(w.y);
    return make_float4(a.x, a.y, b.x, b.y);
}

// Pixel-pair arithmetic of the a-trous kernels: one correctly rounded FFMA / FMUL / FADD per lane of the pair, never
// contracted or reassociated, so both pixels get exactly what the scalar kernel computes.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// common.glsl:150-156
__device__ __forceinline__ float3 octohedral_to_direction(float ex, float ey)
{
    float x = ex, y = ey, z = 1.0f - fabsf(ex) - fabsf(ey);
    if (z < 0.0f)
    {
        const float nx = (1.0f - fabsf(y)) * (x < 0.0f ? -1.0f : 1.0f);
        const float ny = (1.0f - fabsf(x)) * (y < 0.0f ? -1.0f : 1.0f);
        x = nx;
        y = ny;
    }
    const float inv = rsqrtf(x * x + y * y + z * z);
    return make_float3(x * inv, y * inv, z * inv);
}

__device__ __forceinline__ float fast_exp2(float x)
{
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_rcp(float x)
{
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// ---- exactly-rounded, never-contracted helpers (__f*_rn intrinsics) ----------------------------------------------------
// History coordinates decide WHICH texel is fetched (truncation / floor): they follow the oracle's operation order so that
// the choice is identical, in particular for the reflections' virtual-point reprojection, which for a static camera lands
// exactly on texel corners (tex_coord = coord / size without +0.5, reprojection.glsl:78-97) where one ulp flips the texel.
__device__ __forceinline__ float rn_mad(float a, float b, float c) { return __fadd_rn(__fmul_rn(a, b), c); }
__device__ __forceinline__ float4 rn_mat_point(const float* __restrict__ M, float x, float y, float z)
{ // M * (x, y, z, 1), row r = ((m0r*x + m1r*y) + m2r*z) + m3r
    float4 r;
    r.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[0], x), __fmul_rn(M[4], y)), __fmul_rn(M[8], z)), M[12]);
    r.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[1], x), __fmul_rn(M[5], y)), __fmul_rn(M[9], z)), M[13]);
    r.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[2], x), __fmul_rn(M[6], y)), __fmul_rn(M[10], z)), M[14]);
    r.w = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[3], x), __fmul_rn(M[7], y)), __fmul_rn(M[11], z)), M[15]);
    return r;
}
// virtual_point_reprojection, reprojection.glsl:78-97, same operation order as oracle/orc_glsl.h
__device__ __forceinline__ float2 rn_virtual_point_reprojection(int x, int y, float fw, float fh, float depth, float ray_length, const float* __restrict__ cam,
                                                                const float* __restrict__ vpi, const float* __restrict__ pvp)
{
    const float  u = __fdiv_rn((float)x, fw), v = __fdiv_rn((float)y, fh);
    const float4 w = rn_mat_point(vpi, __fadd_rn(__fmul_rn(u, 2.0f), -1.0f), __fadd_rn(__fmul_rn(v, 2.0f), -1.0f), depth);
    const float  ox = __fdiv_rn(w.x, w.w), oy = __fdiv_rn(w.y, w.w), oz = __fdiv_rn(w.z, w.w);
    const float  cx = __fadd_rn(ox, -cam[0]), cy = __fadd_rn(oy, -cam[1]), cz = __fadd_rn(oz, -cam[2]);
    const float  d2  = __fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz));
    const float  len = __fsqrt_rn(d2);
    const float  inv = __fdiv_rn(1.0f, len);
    const float  tt  = __fadd_rn(len, ray_length);
    const float  px = __fadd_rn(cam[0], __fmul_rn(__fmul_rn(cx, inv), tt)), py = __fadd_rn(cam[1], __fmul_rn(__fmul_rn(cy, inv), tt)),
                 pz = __fadd_rn(cam[2], __fmul_rn(__fmul_rn(cz, inv), tt));
    const float4 rp = rn_mat_point(pvp, px, py, pz);
    const float  rx = __fdiv_rn(rp.x, rp.w), ry = __fdiv_rn(rp.y, rp.w);
    return make_float2(__fmul_rn(__fadd_rn(__fmul_rn(rx, 0.5f), 0.5f), fw), __fmul_rn(__fadd_rn(__fmul_rn(ry, 0.5f), 0.5f), fh));
}

// common.glsl:169-184
__device__ __forceinline__ float3 world_position_from_depth(float u, float v, float d, const float* __restrict__ M)
{
    const float sx = u * 2.0f - 1.0f, sy = v * 2.0f - 1.0f;
    const float wx = M[0] * sx + M[4] * sy + M[8] * d + M[12];
    const float wy = M[1] * sx + M[5] * sy + M[9] * d + M[13];
    const float wz = M[2] * sx + M[6] * sy + M[10] * d + M[14];
    const float ww = M[3] * sx + M[7] * sy + M[11] * d + M[15];
    const float iw = 1.0f / ww;
    return make_float3(wx * iw, wy * iw, wz * iw);
}

// x^32 for x in [0,1] by repeated squaring (normal_edge_stopping_weight with phi_normal = 32, edge_stopping.glsl:10-13)
__device__ __forceinline__ float pow32(float x)
{
    x *= x; x *= x; x *= x; x *= x; x *= x;
    return x;
}
__device__ __forceinline__ float pow_pos(float x, float p) { return x <= 0.0f ? 0.0f : __expf(p * __logf(x)); }
__device__ __forceinline__ float normal_weight(float ndot, float phi_normal)
{
    const float c = fminf(fmaxf(ndot, 0.0f), 1.0f);
    return phi_normal == 32.0f ? pow32(c) : pow_pos(c, phi_normal);
}

} // namespace gf
