// svgf_misc.cu — the remaining HBM-streaming stages of the shadows / AO / reflections chains and the G-buffer mip chain.
//   K10 ao/ao_denoise_bilateral_blur.comp:75-139   (separable 9-tap bilateral gaussian, run twice)
//   K6  shadows/shadows_upsample.comp:62-109       K11 ao/ao_upsample.comp:63-112       K17 reflections_upsample.comp:62-109
//   mips: GBuffer NEAREST blit chain, src/g_buffer.cpp:236-244 -> vk.cpp:332-407
// The per-pixel kernels (k_ao_blur, k_upsample_scalar, k_upsample_vec4) decode the octahedral normal and linearise the depth of
// EVERY tap (9 resp. 4 per pixel, ~25 instructions each) and are instruction-issue bound.  The staged kernels (k_ao_blur_v2,
// k_upsample_v2, k_upsample_2x) decode every G-buffer texel of the CTA's footprint once into shared memory; the per-pixel
// kernels remain for the shapes the staged ones do not cover.
#include "glsl_fast.cuh"
#include "hr_internal.h"

namespace {

using namespace gf;

// ---- AO bilateral blur ------------------------------------------------------------------------------------------------
struct BlurParams { int W, H, dirx, diry, radius, row0, row1; float zbp_z, zbp_w; }; // k_ao_blur

// One warp per pixel row (32 px): all taps of a row are contiguous spans => coalesced for the horizontal pass,
// row-strided full-line accesses for the vertical pass (neighbouring rows are L1/L2 hits).
__global__ void __launch_bounds__(256) k_ao_blur(GBufLevelDev g, const __half* __restrict__ in, const uint8_t* __restrict__ tile_flags, BlurParams P,
                                                  __half* __restrict__ out)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = P.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= P.W || y >= P.H || y >= P.row1) return;
    const int    TW  = (P.W + 7) >> 3;
    const size_t idx = (size_t)y * P.W + x;
    const __half one = __float2half_rn(1.0f);
    if (!tile_flags[(size_t)(y >> 3) * TW + (x >> 3)]) { out[idx] = one; return; } // image cleared to 1.0, tile not dispatched
    const float depth = __ldg(g.depth + idx);
    if (depth == 1.0f) { out[idx] = one; return; }
    float        total_ao = __half2float(__ldg(in + idx)), total_w = 1.0f;
    const float  cz = 1.0f / (P.zbp_z * depth + P.zbp_w); // linear_eye_depth, common.glsl:188-191
    const float2 ce = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb2 + idx)));
    const float3 cn = octohedral_to_direction(ce.x, ce.y);
    const float  deviation = (float)P.radius / 1.5f;
    const float  gnorm = 1.0f / sqrtf(2.0f * 3.14159265359f * deviation * deviation);
    const float  ginv  = 1.0f / (2.0f * deviation * deviation);
    for (int i = -P.radius; i <= P.radius; i++)
    {
        if (i == 0) continue;
        const int sx = x + P.dirx * i, sy = y + P.diry * i;
        float     sd = 0.0f, sao = 0.0f;
        float2    se = make_float2(0.0f, 0.0f);
        if (sx >= 0 && sy >= 0 && sx < P.W && sy < P.H)
        { // texelFetch out of bounds => zeros (depth 0, ao 0, normal oct(0,0))
            const size_t si = (size_t)sy * P.W + sx;
            sd  = __ldg(g.depth + si);
            sao = __half2float(__ldg(in + si));
            se  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb2 + si)));
        }
        const float  sz = 1.0f / (P.zbp_z * sd + P.zbp_w);
        const float3 sn = octohedral_to_direction(se.x, se.y);
        float        w  = gnorm * __expf(-((float)(i * i)) * ginv);                       // gaussian_weight, common.glsl:160-165
        w *= __expf(-1.0f - __expf(-fabsf(cz - sz))) * pow32(fminf(fmaxf(dot3(cn, sn), 0.0f), 1.0f)); // edge_stopping.glsl:31-62, wL = 1
        total_ao += w * sao;
        total_w += w;
    }
    out[idx] = __float2half_rn(total_ao / fmaxf(total_w, 0.0001f));
}

#define BLUR_MAX_R 8

struct StagedBlurParams { int W, H, radius, row0, row1; float zbp_z, zbp_w; }; // k_ao_blur_v2: the direction is its template argument

// DIRX = 1: horizontal pass (region 32+2R x 8), DIRX = 0: vertical pass (region 32 x 8+2R)
template <int DIRX>
__global__ void __launch_bounds__(256) k_ao_blur_v2(GBufLevelDev g, const __half* __restrict__ in, const uint8_t* __restrict__ tile_flags, StagedBlurParams P,
                                                     __half* __restrict__ out)
{
    constexpr int RWMAX = DIRX ? 32 + 2 * BLUR_MAX_R : 32, RHMAX = DIRX ? 8 : 8 + 2 * BLUR_MAX_R;
    __shared__ float4 s_nz[RWMAX * RHMAX];
    __shared__ float  s_ao[RWMAX * RHMAX];
    __shared__ float  s_gauss[BLUR_MAX_R + 1];
    __shared__ uint32_t s_tf;
    const int W = P.W, H = P.H, R = P.radius;
    const int x0 = blockIdx.x * 32, y0 = P.row0 + blockIdx.y * 8;
    const int RW = DIRX ? 32 + 2 * R : 32, RH = DIRX ? 8 : 8 + 2 * R;
    const int ox = DIRX ? R : 0, oy = DIRX ? 0 : R;
    const int TW = (W + 7) >> 3;
    if (threadIdx.x < 32)
    {
        const int  tx = (x0 >> 3) + threadIdx.x;
        const bool f  = threadIdx.x < 4 && tx < TW && y0 < H && tile_flags[(size_t)(y0 >> 3) * TW + tx] != 0;
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, f);
        if (threadIdx.x == 0) s_tf = b;
        if (threadIdx.x <= BLUR_MAX_R)
        { // gaussian_weight(i, radius / 1.5), common.glsl:160-165
            const float dev = (float)R / 1.5f, i = (float)threadIdx.x;
            s_gauss[threadIdx.x] = (1.0f / sqrtf(2.0f * 3.14159265359f * dev * dev)) * __expf(-(i * i) / (2.0f * dev * dev));
        }
    }
    const int   lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
    const int   x = x0 + lx, y = y0 + ly;
    const bool  inb = x < W && y < H && y < P.row1;
    const float cdepth = inb ? __ldg(g.depth + (size_t)y * W + x) : 1.0f; // requested before the staging loop (overlapping round trips)
    __syncthreads();
    const uint32_t tf = s_tf;
    if (tf != 0)
    {
        for (int i = threadIdx.x; i < RW * RH; i += 256)
        {
            const int rx = i % RW, ry = i / RW, px = x0 - ox + rx, py = y0 - oy + ry;
            float     d = 0.0f, ao = 0.0f; // texelFetch out of bounds => zeros
            float2    e = make_float2(0.0f, 0.0f);
            if (px >= 0 && py >= 0 && px < W && py < H)
            {
                const size_t pi = (size_t)py * W + px;
                d  = __ldg(g.depth + pi);
                ao = __half2float(__ldg(in + pi));
                e  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb2 + pi)));
            }
            const float3 n = octohedral_to_direction(e.x, e.y);
            s_nz[i] = make_float4(n.x, n.y, n.z, 1.0f / (P.zbp_z * d + P.zbp_w)); // linear_eye_depth, common.glsl:188-191
            s_ao[i] = ao;
        }
    }
    __syncthreads();
    if (!inb) return;
    const size_t idx = (size_t)y * W + x;
    const __half one = __float2half_rn(1.0f);
    if (!((tf >> (lx >> 3)) & 1u)) { out[idx] = one; return; } // image cleared to 1.0, tile not dispatched (ray_traced_ao.cpp:1055)
    if (cdepth == 1.0f) { out[idx] = one; return; }
    const int    ci = (ly + oy) * RW + lx + ox;
    const float4 c  = s_nz[ci];
    float        total_ao = s_ao[ci], total_w = 1.0f;
    const int    stride = DIRX ? 1 : RW;
    for (int i = -R; i <= R; i++)
    {
        if (i == 0) continue;
        const float4 s = s_nz[ci + i * stride];
        // edge_stopping.glsl:31-62 with wL = 1: exp(-1 - exp(-|dz|)) * sat(dot)^32
        const float wZ = fast_exp2(-1.44269504f * fabsf(c.w - s.w));
        const float w  = s_gauss[i < 0 ? -i : i] * fast_exp2(fmaf(wZ, -1.44269504f, -1.44269504f)) * pow32(__saturatef(c.x * s.x + c.y * s.y + c.z * s.z));
        total_ao = fmaf(w, s_ao[ci + i * stride], total_ao);
        total_w += w;
    }
    out[idx] = __float2half_rn(total_ao / fmaxf(total_w, 0.0001f));
}

// ---- upsample ---------------------------------------------------------------------------------------------------------
// Each kernel keeps its own parameter layout.
struct UpParams { int W0, H0, Wm, Hm, row0, row1; float sky_value, power; };                    // k_upsample_v2, k_upsample_2x
struct UpScalarParams { int W0, H0, Wm, Hm, in_channels, row0, row1; float sky_value, power; }; // k_upsample_scalar
struct UpVec4Params { int W0, H0, Wm, Hm, row0, row1; };                                        // k_upsample_vec4

// One pixel of the per-pixel kernels, all four taps read from global memory.  C = 1: channel 0 of an image with P.in_channels
// halves per texel -> R16F, sky pixels get P.sky_value, P.power != 0 raises the result to it; C = 4: RGBA16F -> RGBA16F, sky
// pixels get 0.
template <int C, class T, class Params>
__device__ __forceinline__ void upsample_px(const GBufLevelDev& g0, const GBufLevelDev& gm, const T* __restrict__ in, const Params& P, T* __restrict__ out)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = P.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= P.W0 || y >= P.H0 || y >= P.row1) return;
    const size_t idx = (size_t)y * P.W0 + x;
    const float  hz  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g0.gb3 + idx) + 1)).y;
    if (hz == -1.0f)
    {
        if constexpr (C == 1) out[idx] = __float2half_rn(P.sky_value);
        else out[idx] = make_uint2(0u, 0u);
        return;
    }
    const float2 he = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g0.gb2 + idx)));
    const float3 hn = octohedral_to_direction(he.x, he.y);
    const float  tu = ((float)x + 0.5f) / (float)P.W0, tv = ((float)y + 0.5f) / (float)P.H0;
    const float  tsx = 1.0f / (float)P.Wm, tsy = 1.0f / (float)P.Hm;
    const float  kx[4] = { 0.0f, 1.0f, -1.0f, 0.0f }, ky[4] = { 1.0f, 0.0f, 0.0f, -1.0f };
    float        up[C] = {}, tw = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; i++)
    {
        const int    cx = nearest(tu + kx[i] * tsx, P.Wm), cy = nearest(tv + ky[i] * tsy, P.Hm);
        const size_t ci = (size_t)cy * P.Wm + cx;
        const float  cz = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(gm.gb3 + ci) + 1)).y;
        if (cz == -1.0f) continue;
        const float2 ce = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(gm.gb2 + ci)));
        const float3 cn = octohedral_to_direction(ce.x, ce.y);
        const float  w  = __expf(-1.0f - __expf(-fabsf(hz - cz))) * pow32(fminf(fmaxf(dot3(hn, cn), 0.0f), 1.0f));
        if constexpr (C == 1) up[0] += __half2float(__ldg(in + ci * P.in_channels)) * w;
        else
        {
            const float4 v = h4_to_f4(__ldg(in + ci));
            up[0] += v.x * w; up[1] += v.y * w; up[2] += v.z * w; up[3] += v.w * w;
        }
        tw += w;
    }
    if constexpr (C == 1)
    {
        float r = up[0] / fmaxf(tw, 0.00000001f);
        if (P.power != 0.0f) r = pow_pos(r, P.power);
        out[idx] = __float2half_rn(r);
    }
    else
    {
        const float inv = 1.0f / fmaxf(tw, 0.00000001f);
        out[idx] = pack_h4(up[0] * inv, up[1] * inv, up[2] * inv, up[3] * inv);
    }
}

__global__ void __launch_bounds__(256) k_upsample_scalar(GBufLevelDev g0, GBufLevelDev gm, const __half* __restrict__ in, UpScalarParams P, __half* __restrict__ out)
{
    upsample_px<1>(g0, gm, in, P, out);
}

__global__ void __launch_bounds__(256) k_upsample_vec4(GBufLevelDev g0, GBufLevelDev gm, const uint2* __restrict__ in, UpVec4Params P, uint2* __restrict__ out)
{
    upsample_px<4>(g0, gm, in, P, out);
}

#define UP_RW 24
#define UP_RH 12

// C = 1: scalar input (channel 0 of an image with `in_channels` halves per texel) -> R16F; C = 4: RGBA16F -> RGBA16F
template <int C>
__global__ void __launch_bounds__(256) k_upsample_v2(GBufLevelDev g0, GBufLevelDev gm, const void* __restrict__ in, int in_channels, UpParams P, void* __restrict__ out)
{
    __shared__ float4 s_nz[UP_RW * UP_RH];
    __shared__ float4 s_val[C == 4 ? UP_RW * UP_RH : 1];
    __shared__ float  s_v1[C == 1 ? UP_RW * UP_RH : 1];
    const int   x0 = blockIdx.x * 32, y0 = P.row0 + blockIdx.y * 8;
    const float tsx = 1.0f / (float)P.Wm, tsy = 1.0f / (float)P.Hm;
    // coarse footprint of this CTA: nearest() is monotone, so the taps of the corner pixels bound it
    const int x1 = min(x0 + 31, P.W0 - 1), y1 = min(y0 + 7, P.H0 - 1);
    const int cx_min = nearest(((float)x0 + 0.5f) / (float)P.W0 - tsx, P.Wm), cx_max = nearest(((float)x1 + 0.5f) / (float)P.W0 + tsx, P.Wm);
    const int cy_min = nearest(((float)y0 + 0.5f) / (float)P.H0 - tsy, P.Hm), cy_max = nearest(((float)y1 + 0.5f) / (float)P.H0 + tsy, P.Hm);
    const int rw = cx_max - cx_min + 1, rh = cy_max - cy_min + 1; // <= 19 x 7 for scale >= 1 (host checks)
    // the pixel's own G-buffer words are requested before the staging loop so both round trips to HBM overlap
    const int    x = x0 + (threadIdx.x & 31), y = y0 + (threadIdx.x >> 5);
    const bool   inb = x < P.W0 && y < P.H0 && y < P.row1;
    const size_t idx = (size_t)y * P.W0 + x;
    uint32_t     hz_raw = 0u, he_raw = 0u;
    if (inb)
    {
        hz_raw = __ldg(reinterpret_cast<const uint32_t*>(g0.gb3 + idx) + 1);
        he_raw = __ldg(reinterpret_cast<const uint32_t*>(g0.gb2 + idx));
    }
    for (int i = threadIdx.x; i < rw * rh; i += 256)
    {
        const int    rx = i % rw, ry = i / rw;
        const size_t ci = (size_t)(cy_min + ry) * P.Wm + cx_min + rx;
        const float2 e  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(gm.gb2 + ci)));
        const float  z  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(gm.gb3 + ci) + 1)).y;
        const float3 n  = octohedral_to_direction(e.x, e.y);
        s_nz[ry * UP_RW + rx] = make_float4(n.x, n.y, n.z, z);
        if (C == 4) s_val[ry * UP_RW + rx] = h4_to_f4(__ldg(reinterpret_cast<const uint2*>(in) + ci));
        else s_v1[ry * UP_RW + rx] = __half2float(__ldg(reinterpret_cast<const __half*>(in) + ci * in_channels));
    }
    __syncthreads();
    if (!inb) return;
    const float hz = h2_to_f2(hz_raw).y;
    if (hz == -1.0f)
    {
        if (C == 4) reinterpret_cast<uint2*>(out)[idx] = make_uint2(0u, 0u);
        else reinterpret_cast<__half*>(out)[idx] = __float2half_rn(P.sky_value);
        return;
    }
    const float2 he = h2_to_f2(he_raw);
    const float3 hn = octohedral_to_direction(he.x, he.y);
    const float  tu = ((float)x + 0.5f) / (float)P.W0, tv = ((float)y + 0.5f) / (float)P.H0;
    const float  kx[4] = { 0.0f, 1.0f, -1.0f, 0.0f }, ky[4] = { 1.0f, 0.0f, 0.0f, -1.0f };
    float        up[4] = { 0, 0, 0, 0 }, tw = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; i++)
    {
        const int    cx = nearest(tu + kx[i] * tsx, P.Wm), cy = nearest(tv + ky[i] * tsy, P.Hm);
        const int    li = (cy - cy_min) * UP_RW + (cx - cx_min);
        const float4 c  = s_nz[li];
        if (c.w == -1.0f) continue; // coarse texel is sky
        const float wZ = fast_exp2(-1.44269504f * fabsf(hz - c.w));
        const float w  = fast_exp2(fmaf(wZ, -1.44269504f, -1.44269504f)) * pow32(__saturatef(hn.x * c.x + hn.y * c.y + hn.z * c.z));
        if (C == 4)
        {
            const float4 v = s_val[li];
            up[0] = fmaf(v.x, w, up[0]); up[1] = fmaf(v.y, w, up[1]); up[2] = fmaf(v.z, w, up[2]); up[3] = fmaf(v.w, w, up[3]);
        }
        else up[0] = fmaf(s_v1[li], w, up[0]);
        tw += w;
    }
    const float inv = 1.0f / fmaxf(tw, 0.00000001f);
    if (C == 4) reinterpret_cast<uint2*>(out)[idx] = pack_h4(up[0] * inv, up[1] * inv, up[2] * inv, up[3] * inv);
    else
    {
        float r = up[0] * inv;
        if (P.power != 0.0f) r = pow_pos(r, P.power);
        reinterpret_cast<__half*>(out)[idx] = __float2half_rn(r);
    }
}


// ---- exact 2x upsample ------------------------------------------------------------------------------------------------
// W0 == 2*Wm and H0 == 2*Hm (the reference's half-resolution passes on even frame sizes).  textureLod NEAREST of
// uv + (+-1 coarse texel) with uv = (x + 0.5) / W0 lands on coarse texel (x >> 1) +- 1 (fraction .25 / .75, far from the
// rounding edge), clamped to the image: the four pixels of a 2x2 quad share their four taps.  One thread = one quad:
// 16-byte loads of its two G-buffer rows, taps decoded once per CTA into shared memory, no per-pixel address arithmetic.
template <int C>
__global__ void __launch_bounds__(256) k_upsample_2x(GBufLevelDev g0, GBufLevelDev gm, const void* __restrict__ in, int in_channels, UpParams P, void* __restrict__ out)
{
    constexpr int RW = 34, RH = 10;
    __shared__ float4 s_nz[RW * RH];
    __shared__ float4 s_val[C == 4 ? RW * RH : 1];
    __shared__ float  s_v1[C == 1 ? RW * RH : 1];
    const int  lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
    const int  cx0 = blockIdx.x * 32, cy0 = (P.row0 >> 1) + blockIdx.y * 8;
    const int  cx = cx0 + lx, cy = cy0 + ly, x = 2 * cx, y = 2 * cy;
    const bool inb = cx < P.Wm && y < P.row1;
    uint4      a2[2], a3[2];
    if (inb)
    {
#pragma unroll
        for (int r = 0; r < 2; r++)
        {
            const size_t i = (size_t)(y + r) * P.W0 + x; // even => 16-byte aligned
            a2[r] = __ldg(reinterpret_cast<const uint4*>(g0.gb2 + i));
            a3[r] = __ldg(reinterpret_cast<const uint4*>(g0.gb3 + i));
        }
    }
    for (int i = threadIdx.x; i < RW * RH; i += 256)
    {
        const int    rx = i % RW, ry = i / RW;
        const int    gx = min(max(cx0 - 1 + rx, 0), P.Wm - 1), gy = min(max(cy0 - 1 + ry, 0), P.Hm - 1);
        const size_t ci = (size_t)gy * P.Wm + gx;
        const float2 e  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(gm.gb2 + ci)));
        const float  z  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(gm.gb3 + ci) + 1)).y;
        const float3 n  = octohedral_to_direction(e.x, e.y);
        s_nz[i] = make_float4(n.x, n.y, n.z, z);
        if (C == 4) s_val[i] = h4_to_f4(__ldg(reinterpret_cast<const uint2*>(in) + ci));
        else s_v1[i] = __half2float(__ldg(reinterpret_cast<const __half*>(in) + ci * in_channels));
    }
    __syncthreads();
    if (!inb) return;
    // tap order of the reference kernel: (0,+1) (+1,0) (-1,0) (0,-1)
    const int ti[4] = { (ly + 2) * RW + lx + 1, (ly + 1) * RW + lx + 2, (ly + 1) * RW + lx, ly * RW + lx + 1 };
    float4    c[4], v4[4];
    float     v1[4];
#pragma unroll
    for (int t = 0; t < 4; t++)
    {
        c[t] = s_nz[ti[t]];
        if (C == 4) v4[t] = s_val[ti[t]];
        else v1[t] = s_v1[ti[t]];
    }
#pragma unroll
    for (int r = 0; r < 2; r++)
    {
        uint32_t o1[2];
        uint2    o4[2];
#pragma unroll
        for (int q = 0; q < 2; q++)
        {
            const float hz = h2_to_f2(q ? a3[r].w : a3[r].y).y;
            if (hz == -1.0f)
            {
                o1[q] = __half_as_ushort(__float2half_rn(P.sky_value));
                o4[q] = make_uint2(0u, 0u);
                continue;
            }
            const float2 he = h2_to_f2(q ? a2[r].z : a2[r].x);
            const float3 hn = octohedral_to_direction(he.x, he.y);
            float        up[4] = { 0, 0, 0, 0 }, tw = 0.0f;
#pragma unroll
            for (int t = 0; t < 4; t++)
            {
                if (c[t].w == -1.0f) continue; // coarse texel is sky
                const float wZ = fast_exp2(-1.44269504f * fabsf(hz - c[t].w));
                const float w  = fast_exp2(fmaf(wZ, -1.44269504f, -1.44269504f)) * pow32(__saturatef(hn.x * c[t].x + hn.y * c[t].y + hn.z * c[t].z));
                if (C == 4)
                {
                    up[0] = fmaf(v4[t].x, w, up[0]); up[1] = fmaf(v4[t].y, w, up[1]); up[2] = fmaf(v4[t].z, w, up[2]); up[3] = fmaf(v4[t].w, w, up[3]);
                }
                else up[0] = fmaf(v1[t], w, up[0]);
                tw += w;
            }
            const float inv = 1.0f / fmaxf(tw, 0.00000001f);
            if (C == 4) o4[q] = pack_h4(up[0] * inv, up[1] * inv, up[2] * inv, up[3] * inv);
            else
            {
                float rr = up[0] * inv;
                if (P.power != 0.0f) rr = pow_pos(rr, P.power);
                o1[q] = __half_as_ushort(__float2half_rn(rr));
            }
        }
        const size_t oi = (size_t)(y + r) * P.W0 + x;
        if (C == 4) reinterpret_cast<uint4*>(out)[oi >> 1] = make_uint4(o4[0].x, o4[0].y, o4[1].x, o4[1].y);
        else reinterpret_cast<uint32_t*>(out)[oi >> 1] = o1[0] | (o1[1] << 16);
    }
}

bool upsample_is_2x(const GBufLevelDev& g0, const GBufLevelDev& gm, int row0, int row1)
{
    return g0.W == 2 * gm.W && g0.H == 2 * gm.H && (row0 & 1) == 0 && (row1 & 1) == 0;
}

// the staged footprint must fit UP_RW x UP_RH: true when the coarse image is at most 2x smaller... i.e. 32 full-res columns
// map to <= 32*Wm/W0 + 3 coarse columns
bool upsample_fits(const GBufLevelDev& g0, const GBufLevelDev& gm)
{
    const long cw = (32L * gm.W + g0.W - 1) / g0.W + 3, ch = (8L * gm.H + g0.H - 1) / g0.H + 3;
    return cw <= UP_RW && ch <= UP_RH;
}

// C = 1: launch_upsample_scalar; C = 4: launch_upsample_vec4 (in_channels 4, sky 0, no power).  The exact 2x kernel when the
// frame is twice the coarse mip, else the staged kernel when its footprint fits, else the per-pixel kernel.
template <int C>
void launch_upsample(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, int in_channels, float sky_value, float power, void* out, int row0, int row1,
                     cudaStream_t st)
{
    if (row1 <= row0) return;
    UpParams P { g0.W, g0.H, gm.W, gm.H, row0, row1, sky_value, power };
    if (upsample_is_2x(g0, gm, row0, row1))
    {
        dim3 grid2((gm.W + 31) / 32, ((row1 - row0) / 2 + 7) / 8);
        k_upsample_2x<C><<<grid2, 256, 0, st>>>(g0, gm, in, in_channels, P, out);
        return;
    }
    dim3 grid((g0.W + 31) / 32, (row1 - row0 + 7) / 8);
    if (upsample_fits(g0, gm)) k_upsample_v2<C><<<grid, 256, 0, st>>>(g0, gm, in, in_channels, P, out);
    else if constexpr (C == 1)
        k_upsample_scalar<<<grid, 256, 0, st>>>(g0, gm, reinterpret_cast<const __half*>(in), UpScalarParams { g0.W, g0.H, gm.W, gm.H, in_channels, row0, row1, sky_value, power },
                                                 reinterpret_cast<__half*>(out));
    else k_upsample_vec4<<<grid, 256, 0, st>>>(g0, gm, reinterpret_cast<const uint2*>(in), UpVec4Params { g0.W, g0.H, gm.W, gm.H, row0, row1 }, reinterpret_cast<uint2*>(out));
}

// ---- G-buffer mips ----------------------------------------------------------------------------------------------------
// Levels 1 and 2 in one launch: level 2 is a NEAREST blit of level 1, i.e. of level 0 at the composed coordinates
// (min(2*min(2X+1, w1-1)+1, W-1), ...), so it can be read straight from level 0 by the threads (x < w2, y < h2).
__global__ void k_build_mips12(int W, int H, const uint2* __restrict__ gb2, const uint2* __restrict__ gb3, const float* __restrict__ depth,
                               const uint32_t* __restrict__ gb1, uint2* __restrict__ o2a, uint2* __restrict__ o3a, float* __restrict__ oda, uint32_t* __restrict__ o1a,
                               uint2* __restrict__ o2b, uint2* __restrict__ o3b, float* __restrict__ odb, uint32_t* __restrict__ o1b)
{
    const int w1 = max(W / 2, 1), h1 = max(H / 2, 1), w2 = max(w1 / 2, 1), h2 = max(h1 / 2, 1);
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w1 || y >= h1) return;
    {
        const size_t s = (size_t)min(2 * y + 1, H - 1) * W + min(2 * x + 1, W - 1), d = (size_t)y * w1 + x;
        o2a[d] = gb2[s];
        o3a[d] = gb3[s];
        oda[d] = depth[s];
        if (gb1 && o1a) o1a[d] = gb1[s];
    }
    if (x < w2 && y < h2)
    {
        const int    x1 = min(2 * x + 1, w1 - 1), y1 = min(2 * y + 1, h1 - 1);
        const size_t s = (size_t)min(2 * y1 + 1, H - 1) * W + min(2 * x1 + 1, W - 1), d = (size_t)y * w2 + x;
        o2b[d] = gb2[s];
        o3b[d] = gb3[s];
        odb[d] = depth[s];
        if (gb1 && o1b) o1b[d] = gb1[s];
    }
}

} // namespace

void launch_ao_blur(const GBufLevelDev& g, const __half* in, const uint8_t* tile_flags, const float* zbp, int dirx, int diry, int radius, __half* out, int row0,
                    int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    dim3 grid((g.W + 31) / 32, (row1 - row0 + 7) / 8);
    if (radius > BLUR_MAX_R || radius < 1 || !((dirx == 1 && diry == 0) || (dirx == 0 && diry == 1)) || row0 % 8 != 0)
    {
        k_ao_blur<<<grid, 256, 0, st>>>(g, in, tile_flags, BlurParams { g.W, g.H, dirx, diry, radius, row0, row1, zbp[2], zbp[3] }, out);
        return;
    }
    StagedBlurParams P { g.W, g.H, radius, row0, row1, zbp[2], zbp[3] };
    if (dirx) k_ao_blur_v2<1><<<grid, 256, 0, st>>>(g, in, tile_flags, P, out);
    else k_ao_blur_v2<0><<<grid, 256, 0, st>>>(g, in, tile_flags, P, out);
}

void launch_upsample_scalar(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, int in_channels, float sky_value, float power, __half* out, int row0,
                            int row1, cudaStream_t st)
{
    launch_upsample<1>(g0, gm, in, in_channels, sky_value, power, out, row0, row1, st);
}

void launch_upsample_vec4(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, void* out, int row0, int row1, cudaStream_t st)
{
    launch_upsample<4>(g0, gm, in, 4, 0.0f, 0.0f, out, row0, row1, st);
}

static_assert(HR_MAX_MIPS == 3, "hr_launch_build_mips writes mips 1 and 2 with k_build_mips12");

int hr_launch_build_mips(hr_ctx* ctx, GBufSlot& s, int W, int H, cudaStream_t st)
{
    const int w1 = W / 2 > 0 ? W / 2 : 1, h1 = H / 2 > 0 ? H / 2 : 1;
    dim3      b(32, 8), g((w1 + 31) / 32, (h1 + 7) / 8);
    k_build_mips12<<<g, b, 0, st>>>(W, H, (const uint2*)s.gb2[0], (const uint2*)s.gb3[0], s.depth[0], (const uint32_t*)s.gb1[0], (uint2*)s.gb2[1], (uint2*)s.gb3[1],
                                    s.depth[1], (uint32_t*)s.gb1[1], (uint2*)s.gb2[2], (uint2*)s.gb3[2], s.depth[2], (uint32_t*)s.gb1[2]);
    ctx->launches++;
    HR_CHECK_LAUNCH(ctx);
    return HR_OK;
}
