// svgf_atrous.cu — edge-aware a-trous wavelet filter for the shadows chain (the roofline kernel).
//   K4  shadows/shadows_denoise_copy_shadow_tiles.comp:32-36   (folded in: tiles not on the denoise list are zero-filled)
//   K5  shadows/shadows_denoise_atrous.comp:94-174 + edge_stopping.glsl:10-62
// Algorithmic traffic per pixel and iteration (SURVEY.md §8d): RG16F in 4 + GB2 8 + GB3 8 read, RG16F 4 written = 24 B.
//
// Three kernel forms, chosen by launch_shadows_atrous:
//   k_atrous_v3 / k_atrous_v3s  pixel pairs (atrous_pairs.cuh), the default.  Six staged planes: nx, ny, nz, z*log2e/sigma,
//                               visibility, variance.  The visibility is the one colour channel and also the luminance the
//                               colour weight compares.
//   k_atrous_tiled              the scalar tiled kernel: odd widths, phi_normal != 32, and the reference of the pixel pairs.
//                               One CTA filters a 64x16 output tile.  The tile plus a halo of `step` texels of
//                                 * the input image (visibility, variance) as float2
//                                 * the decoded G-buffer normal + linear z as float4 (oct decode done ONCE per staged texel)
//                               is staged in shared memory with coalesced 8-byte/4-byte global loads (out-of-image texels are
//                               staged as zeros = texelFetch robust-access semantics); the 3x3 taps at stride `step` then come
//                               from shared memory.  A CTA whose 16 reference tiles are all on the shadow list writes zeros and
//                               exits without loading anything.
//   k_atrous_naive              global memory only: radius != 1 and steps >= 16.
#include "atrous_pairs.cuh"

namespace {

using namespace gf;

constexpr int TILE_W = 64, TILE_H = 16;

struct AtrousParams {
    int   W, H, step, radius;
    float phi_visibility, phi_normal, sigma_depth, power;
    int   row0, row1;
};

// ---- naive kernel (global memory only): the fallback for radius != 1 and steps >= 16, and hr_debug_set(1, 0) ------
__global__ void __launch_bounds__(256) k_atrous_naive(GBufLevelDev g, const uint32_t* __restrict__ in, const uint8_t* __restrict__ tile_flags,
                                                       AtrousParams P, uint32_t* __restrict__ out)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = P.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= P.W || y >= P.H || y >= P.row1) return;
    const int    TW  = (P.W + 7) >> 3;
    const size_t idx = (size_t)y * P.W + x;
    if (!tile_flags[(size_t)(y >> 3) * TW + (x >> 3)]) { out[idx] = 0u; return; }
    const float2 c = h2_to_f2(__ldg(in + idx));
    float        var = 0.0f;
    for (int yy = -1; yy <= 1; yy++)
        for (int xx = -1; xx <= 1; xx++)
        {
            const int   px = x + xx, py = y + yy;
            const float k = (xx == 0 ? 0.5f : 0.25f) * (yy == 0 ? 0.5f : 0.25f); // {1/4,1/8,1/8,1/16}
            if (px >= 0 && py >= 0 && px < P.W && py < P.H) var += h2_to_f2(__ldg(in + (size_t)py * P.W + px)).y * k;
        }
    const float2 e  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb2 + idx)));
    const float  zc = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + idx) + 1)).y;
    if (zc < 0.0f) { out[idx] = f2_to_h2(c.x, c.y); return; }
    const float3 nc      = octohedral_to_direction(e.x, e.y);
    const float  phi_vis = P.phi_visibility * sqrtf(fmaxf(0.0f, 1e-10f + var));
    float        sum_w = 1.0f, s0 = c.x, s1 = c.y;
    for (int yy = -P.radius; yy <= P.radius; yy++)
        for (int xx = -P.radius; xx <= P.radius; xx++)
        {
            const int px = x + xx * P.step, py = y + yy * P.step;
            if ((xx == 0 && yy == 0) || px < 0 || py < 0 || px >= P.W || py >= P.H) continue;
            const float  kw[3] = { 1.0f, 2.0f / 3.0f, 1.0f / 6.0f };
            const float  kern  = kw[abs(xx)] * kw[abs(yy)];
            const size_t pi    = (size_t)py * P.W + px;
            const float2 s     = h2_to_f2(__ldg(in + pi));
            const float2 se    = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb2 + pi)));
            const float  zs    = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + pi) + 1)).y;
            const float3 ns    = octohedral_to_direction(se.x, se.y);
            const float  wZ    = __expf(-fabsf(zc - zs) / P.sigma_depth);
            const float  wL    = fabsf(c.x - s.x) / phi_vis;
            const float  w     = __expf(-wL - wZ) * normal_weight(dot3(nc, ns), P.phi_normal);
            const float  wk    = w * kern;
            sum_w += wk;
            s0 += wk * s.x;
            s1 += wk * wk * s.y;
        }
    float o0 = s0 / sum_w, o1 = s1 / (sum_w * sum_w);
    if (P.power != 0.0f) o0 = pow_pos(o0, P.power);
    out[idx] = f2_to_h2(o0, o1);
}

// ---- tiled kernel -----------------------------------------------------------------------------------------------
// dynamic smem: float4 s_nz[regH*regW] (nx,ny,nz,z) then float2 s_in[regH*regW] (vis,var)
template <int STEP>
__global__ void __launch_bounds__(256) k_atrous_tiled(GBufLevelDev g, const uint32_t* __restrict__ in, const uint8_t* __restrict__ tile_flags,
                                                       AtrousParams P, uint32_t* __restrict__ out)
{
    extern __shared__ float4 smem4[];
    constexpr int RW = TILE_W + 2 * STEP, RH = TILE_H + 2 * STEP;
    float4*       s_nz = smem4;
    float2*       s_in = reinterpret_cast<float2*>(smem4 + RW * RH);
    __shared__ uint32_t s_tf; // 16 tile flags of this CTA (bit = ty*8 + tx)

    const int W = P.W, H = P.H;
    const int x0 = blockIdx.x * TILE_W, y0 = P.row0 + blockIdx.y * TILE_H;
    const int TW = (W + 7) >> 3, TH = (H + 7) >> 3;
    if (threadIdx.x == 0) s_tf = 0;
    __syncthreads();
    if (threadIdx.x < 16)
    {
        const int tx = (x0 >> 3) + (threadIdx.x & 7), ty = (y0 >> 3) + (threadIdx.x >> 3);
        if (tx < TW && ty < TH && tile_flags[(size_t)ty * TW + tx]) atomicOr(&s_tf, 1u << threadIdx.x);
    }
    __syncthreads();
    const uint32_t tf = s_tf;

    if (tf != 0)
    {
        // stage region [x0-STEP, x0+TILE_W+STEP) x [y0-STEP, y0+TILE_H+STEP)
        for (int i = threadIdx.x; i < RW * RH; i += 256)
        {
            const int rx = i % RW, ry = i / RW;
            const int px = x0 - STEP + rx, py = y0 - STEP + ry;
            float4    nz = make_float4(0.0f, 0.0f, 1.0f, 0.0f);
            float2    iv = make_float2(0.0f, 0.0f);
            if (px >= 0 && py >= 0 && px < W && py < H)
            {
                const size_t pi = (size_t)py * W + px;
                const uint2  a  = __ldg(g.gb2 + pi);
                const uint2  b  = __ldg(g.gb3 + pi);
                const float2 e  = h2_to_f2(a.x);
                const float3 n  = octohedral_to_direction(e.x, e.y);
                nz              = make_float4(n.x, n.y, n.z, h2_to_f2(b.y).y);
                iv              = h2_to_f2(__ldg(in + pi));
            }
            s_nz[i] = nz;
            s_in[i] = iv;
        }
    }
    __syncthreads();

    const int   lx = threadIdx.x & 63, lyb = threadIdx.x >> 6; // 64 columns x 4 row lanes
    const float nlog2e_over_sigma = -1.44269504f / P.sigma_depth;
#pragma unroll
    for (int k = 0; k < TILE_H / 4; k++)
    {
        const int ly = lyb + 4 * k;
        const int x = x0 + lx, y = y0 + ly;
        if (x >= W || y >= H || y >= P.row1) continue;
        const size_t idx = (size_t)y * W + x;
        if (!((tf >> ((ly >> 3) * 8 + (lx >> 3))) & 1u)) { out[idx] = 0u; continue; }
        const int    ci = (ly + STEP) * RW + (lx + STEP);
        const float2 c  = s_in[ci];
        const float4 cn = s_nz[ci];
        if (cn.w < 0.0f) { out[idx] = f2_to_h2(c.x, c.y); continue; }
        // compute_variance_center: 3x3 gaussian of the variance channel (out-of-image texels are staged as 0)
        float var = 0.25f * c.y;
        var += 0.125f * (s_in[ci - 1].y + s_in[ci + 1].y + s_in[ci - RW].y + s_in[ci + RW].y);
        var += 0.0625f * (s_in[ci - RW - 1].y + s_in[ci - RW + 1].y + s_in[ci + RW - 1].y + s_in[ci + RW + 1].y);
        const float nlog2e_over_phi = -1.44269504f / (P.phi_visibility * sqrtf(fmaxf(0.0f, 1e-10f + var)));
        float       sum_w = 1.0f, s0 = c.x, s1 = c.y;
#pragma unroll
        for (int yy = -1; yy <= 1; yy++)
#pragma unroll
            for (int xx = -1; xx <= 1; xx++)
            {
                if (xx == 0 && yy == 0) continue;
                const int px = x + xx * STEP, py = y + yy * STEP;
                if (px < 0 || py < 0 || px >= W || py >= H) continue;
                const float  kern = (xx == 0 ? 1.0f : 2.0f / 3.0f) * (yy == 0 ? 1.0f : 2.0f / 3.0f);
                const int    si   = ci + yy * STEP * RW + xx * STEP;
                const float4 sn   = s_nz[si];
                const float2 s    = s_in[si];
                const float  wZ   = fast_exp2(fabsf(cn.w - sn.w) * nlog2e_over_sigma);               // exp(-|dz|/sigma)
                const float  ea   = fmaf(wZ, -1.44269504f, fabsf(c.x - s.x) * nlog2e_over_phi);   // -(wL + wZ) * log2(e)
                const float  nd   = cn.x * sn.x + cn.y * sn.y + cn.z * sn.z;
                const float  w    = fast_exp2(ea) * normal_weight(nd, P.phi_normal);
                const float  wk   = w * kern;
                sum_w += wk;
                s0 = fmaf(wk, s.x, s0);
                s1 = fmaf(wk * wk, s.y, s1);
            }
        const float inv = 1.0f / sum_w;
        float       o0 = s0 * inv, o1 = s1 * inv * inv;
        if (P.power != 0.0f) o0 = pow_pos(o0, P.power);
        out[idx] = f2_to_h2(o0, o1);
    }
}

template <int STEP>
void launch_tiled(const GBufLevelDev& g, const uint32_t* in, const uint8_t* tf, const AtrousParams& P, uint32_t* out, cudaStream_t st)
{
    constexpr int RW = TILE_W + 2 * STEP, RH = TILE_H + 2 * STEP;
    const size_t  smem = (size_t)RW * RH * (sizeof(float4) + sizeof(float2));
    static bool   configured[64] = {};
    if (hr_once_per_device(configured)) cudaFuncSetAttribute(k_atrous_tiled<STEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid((P.W + TILE_W - 1) / TILE_W, (P.row1 - P.row0 + TILE_H - 1) / TILE_H);
    k_atrous_tiled<STEP><<<grid, 256, smem, st>>>(g, in, tf, P, out);
}

// ---- pixel-pair kernels ------------------------------------------------------------------------------------------
struct V3Params {
    int   W, H;
    float c_sigma;   // log2(e) / sigma_depth
    float c_phi0;    // -log2(e) / phi_visibility
    float power;
    int   row0, row1;
};

struct ShadowsPass {
    using In = uint32_t; using Out = uint32_t; using Params = V3Params;
    static constexpr int  NPL = 6, NC = 1;
    static constexpr bool COPY_EMPTY_CTA = false; // a CTA without a flagged tile stages nothing and writes zeros

    // Stage the texel pair (px, px+1) of row py (px even) at region index ri (even): decoded normal, scaled linear depth, visibility,
    // variance; zeros outside the image.
    static __device__ __forceinline__ void stage(const GBufLevelDev& g, const uint32_t* __restrict__ in, float c_sigma, int px, int py, int W, int H, int ri, float* s, int PL)
    {
        float2 nx = make_float2(0.0f, 0.0f), ny = nx, nz = nx, zs = nx, vi = nx, va = nx;
        if (px >= 0 && py >= 0 && px < W && py < H)
        {
            const size_t pi = (size_t)py * W + px;
            const uint4  a  = __ldg(reinterpret_cast<const uint4*>(g.gb2 + pi)); // two RGBA16F texels: .x / .z hold the oct normals
            const uint4  b  = __ldg(reinterpret_cast<const uint4*>(g.gb3 + pi)); // .y / .w hold (mesh id, linear z)
            const uint2  c  = __ldg(reinterpret_cast<const uint2*>(in + pi));    // two RG16F texels (visibility, variance)
            const float2 e0 = h2_to_f2(a.x), e1 = h2_to_f2(a.z);
            const float3 n0 = octohedral_to_direction(e0.x, e0.y), n1 = octohedral_to_direction(e1.x, e1.y);
            const float2 i0 = h2_to_f2(c.x), i1 = h2_to_f2(c.y);
            nx = make_float2(n0.x, n1.x); ny = make_float2(n0.y, n1.y); nz = make_float2(n0.z, n1.z);
            zs = make_float2(h2_to_f2(b.y).y * c_sigma, h2_to_f2(b.w).y * c_sigma);
            vi = make_float2(i0.x, i1.x); va = make_float2(i0.y, i1.y);
        }
        float* p = s + ri;
        *reinterpret_cast<float2*>(p) = nx; p += PL;
        *reinterpret_cast<float2*>(p) = ny; p += PL;
        *reinterpret_cast<float2*>(p) = nz; p += PL;
        *reinterpret_cast<float2*>(p) = zs; p += PL;
        *reinterpret_cast<float2*>(p) = vi; p += PL;
        *reinterpret_cast<float2*>(p) = va;
    }

    static __device__ __forceinline__ float2 side_var(const uint32_t* __restrict__ in, size_t pi)
    {
        const uint2 w = __ldg(reinterpret_cast<const uint2*>(in + pi));
        return make_float2(h2_to_f2(w.x).y, h2_to_f2(w.y).y);
    }

    template <bool ALIGNED_X>
    static __device__ __forceinline__ void filter_store(const GBufLevelDev&, const V3Params& P, const PairTaps& t, uint32_t* __restrict__ out, size_t idx, bool has1, bool flagged)
    {
        if (!flagged)
        {
            out[idx] = 0u;
            if (has1) out[idx + 1] = 0u;
            return;
        }
        const PairSum<1> f  = filter_pair<1, 4, ALIGNED_X>(t, P.c_phi0); // luminance = visibility
        float2           o0 = f.c[0];
        if (P.power != 0.0f) { o0.x = pow_pos(o0.x, P.power); o0.y = pow_pos(o0.y, P.power); }
        // sky pixels (linear z < 0) pass the input through
        const float2   zs = ld_pair(t.s + 3 * t.PL, t.ci, true), vi = ld_pair(t.s + 4 * t.PL, t.ci, true), va = ld_pair(t.s + 5 * t.PL, t.ci, true);
        const uint32_t r0 = zs.x < 0.0f ? f2_to_h2(vi.x, va.x) : f2_to_h2(o0.x, f.v.x);
        const uint32_t r1 = zs.y < 0.0f ? f2_to_h2(vi.y, va.y) : f2_to_h2(o0.y, f.v.y);
        if (has1) *reinterpret_cast<uint2*>(out + idx) = make_uint2(r0, r1); // idx even (W even is required by the launcher)
        else out[idx] = r0;
    }
};

template <int STEP>
__global__ void __launch_bounds__(256) k_atrous_v3(GBufLevelDev g, const uint32_t* __restrict__ in, const uint8_t* __restrict__ tile_flags, V3Params P,
                                                    uint32_t* __restrict__ out)
{
    atrous_dense<ShadowsPass, STEP>(g, in, tile_flags, P, out);
}

template <int STEP>
__global__ void __launch_bounds__(256) k_atrous_v3s(GBufLevelDev g, const uint32_t* __restrict__ in, const uint8_t* __restrict__ tile_flags, V3Params P,
                                                     uint32_t* __restrict__ out)
{
    atrous_interleaved<ShadowsPass, STEP>(g, in, tile_flags, P, out);
}

template <int STEP>
using Dense = DenseTile<STEP, ShadowsPass::NPL>;
template <int STEP>
using Interleaved = InterleavedTile<STEP, ShadowsPass::NPL>;

} // namespace

int g_hr_atrous_impl = 3;

void launch_shadows_atrous(const GBufLevelDev& g, const __half2* in, const uint8_t* tile_flags, int radius, int step, float phi_vis, float phi_n,
                           float sigma_z, float power, __half2* out, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    const uint32_t* i32 = reinterpret_cast<const uint32_t*>(in);
    uint32_t*       o32 = reinterpret_cast<uint32_t*>(out);
    const bool      tiled_step = radius == 1 && (step == 1 || step == 2 || step == 4 || step == 8);
    if (g_hr_atrous_impl == 3 && tiled_step && phi_n == 32.0f && !(g.W & 1) && row0 % 8 == 0)
    { // pixel pairs
        V3Params P { g.W, g.H, 1.44269504f / sigma_z, -1.44269504f / phi_vis, power, row0, row1 };
        switch (step)
        {
            case 1: launch_tiles<Dense<1>>(k_atrous_v3<1>, g, i32, tile_flags, P, o32, st); break;
            case 2: launch_tiles<Dense<2>>(k_atrous_v3<2>, g, i32, tile_flags, P, o32, st); break;
            case 4: launch_tiles<Dense<4>>(k_atrous_v3<4>, g, i32, tile_flags, P, o32, st); break;
            default: launch_tiles<Interleaved<8>>(k_atrous_v3s<8>, g, i32, tile_flags, P, o32, st); break; // DESIGN.md §8
        }
        return;
    }
    AtrousParams P { g.W, g.H, step, radius, phi_vis, phi_n, sigma_z, power, row0, row1 };
    if (g_hr_atrous_impl != 0 && tiled_step)
    {
        switch (step)
        {
            case 1: launch_tiled<1>(g, i32, tile_flags, P, o32, st); break;
            case 2: launch_tiled<2>(g, i32, tile_flags, P, o32, st); break;
            case 4: launch_tiled<4>(g, i32, tile_flags, P, o32, st); break;
            default: launch_tiled<8>(g, i32, tile_flags, P, o32, st); break;
        }
    }
    else
    {
        dim3 grid((g.W + 31) / 32, (row1 - row0 + 7) / 8);
        k_atrous_naive<<<grid, 256, 0, st>>>(g, i32, tile_flags, P, o32);
    }
}
