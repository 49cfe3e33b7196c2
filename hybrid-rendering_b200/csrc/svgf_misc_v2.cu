// svgf_misc_v2.cu — shared-memory staged versions of the AO bilateral blur (K10) and the depth/normal-aware upsample
// (K6 / K11 / K17).  The v1 kernels (svgf_misc.cu, svgf_reflections.cu) decode the octahedral normal and linearise the
// depth of EVERY tap (9 resp. 4 per pixel, ~25 instructions each) and were instruction-issue bound.  Here every G-buffer texel of the CTA's footprint is decoded once into shared memory.
//   K10 ao/ao_denoise_bilateral_blur.comp:75-139     K6 shadows_upsample.comp:62-109   K11 ao_upsample.comp:63-112
//   K17 reflections_upsample.comp:62-109
#include "glsl_fast.cuh"
#include "hr_internal.h"

void launch_ao_blur_v1(const GBufLevelDev& g, const __half* in, const uint8_t* tile_flags, const float* zbp, int dirx, int diry, int radius, __half* out,
                       int row0, int row1, cudaStream_t st);
void launch_upsample_scalar_v1(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, int in_channels, float sky_value, float power, __half* out,
                               int row0, int row1, cudaStream_t st);

namespace {

using namespace gf;

#define BLUR_MAX_R 8

struct BlurParams { int W, H, radius, row0, row1; float zbp_z, zbp_w; };

// DIRX = 1: horizontal pass (region 32+2R x 8), DIRX = 0: vertical pass (region 32 x 8+2R)
template <int DIRX>
__global__ void __launch_bounds__(256) k_ao_blur_v2(GBufLevelDev g, const __half* __restrict__ in, const uint8_t* __restrict__ tile_flags, BlurParams P,
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
struct UpParams { int W0, H0, Wm, Hm, row0, row1; float sky_value, power; };

__device__ __forceinline__ int nearest(float uv, int size) { return min(max((int)floorf(uv * (float)size), 0), size - 1); }
__device__ __forceinline__ uint2 pack_h4(float a, float b, float c, float d) { return make_uint2(f2_to_h2(a, b), f2_to_h2(c, d)); }

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

} // namespace

void launch_ao_blur(const GBufLevelDev& g, const __half* in, const uint8_t* tile_flags, const float* zbp, int dirx, int diry, int radius, __half* out, int row0,
                    int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    if (radius > BLUR_MAX_R || radius < 1 || !((dirx == 1 && diry == 0) || (dirx == 0 && diry == 1)) || row0 % 8 != 0)
    {
        launch_ao_blur_v1(g, in, tile_flags, zbp, dirx, diry, radius, out, row0, row1, st);
        return;
    }
    BlurParams P { g.W, g.H, radius, row0, row1, zbp[2], zbp[3] };
    dim3       grid((g.W + 31) / 32, (row1 - row0 + 7) / 8);
    if (dirx) k_ao_blur_v2<1><<<grid, 256, 0, st>>>(g, in, tile_flags, P, out);
    else k_ao_blur_v2<0><<<grid, 256, 0, st>>>(g, in, tile_flags, P, out);
}

void launch_upsample_scalar(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, int in_channels, float sky_value, float power, __half* out, int row0,
                            int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    UpParams P { g0.W, g0.H, gm.W, gm.H, row0, row1, sky_value, power };
    if (upsample_is_2x(g0, gm, row0, row1))
    {
        dim3 grid2((gm.W + 31) / 32, ((row1 - row0) / 2 + 7) / 8);
        k_upsample_2x<1><<<grid2, 256, 0, st>>>(g0, gm, in, in_channels, P, out);
        return;
    }
    if (!upsample_fits(g0, gm)) { launch_upsample_scalar_v1(g0, gm, in, in_channels, sky_value, power, out, row0, row1, st); return; }
    dim3     grid((g0.W + 31) / 32, (row1 - row0 + 7) / 8);
    k_upsample_v2<1><<<grid, 256, 0, st>>>(g0, gm, in, in_channels, P, out);
}

// returns false if the footprint does not fit (caller uses its v1 kernel)
bool launch_upsample_vec4_v2(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, void* out, int row0, int row1, cudaStream_t st)
{
    UpParams P { g0.W, g0.H, gm.W, gm.H, row0, row1, 0.0f, 0.0f };
    if (upsample_is_2x(g0, gm, row0, row1))
    {
        dim3 grid2((gm.W + 31) / 32, ((row1 - row0) / 2 + 7) / 8);
        k_upsample_2x<4><<<grid2, 256, 0, st>>>(g0, gm, in, 4, P, out);
        return true;
    }
    if (!upsample_fits(g0, gm)) return false;
    dim3     grid((g0.W + 31) / 32, (row1 - row0 + 7) / 8);
    k_upsample_v2<4><<<grid, 256, 0, st>>>(g0, gm, in, 4, P, out);
    return true;
}
