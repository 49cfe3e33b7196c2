// svgf_atrous.cu — edge-aware a-trous wavelet filter for the shadows chain (the roofline kernel).
//   K4  shadows/shadows_denoise_copy_shadow_tiles.comp:32-36   (folded in: tiles not on the denoise list are zero-filled)
//   K5  shadows/shadows_denoise_atrous.comp:94-174 + edge_stopping.glsl:10-62
// Algorithmic traffic per pixel and iteration (SURVEY.md §8d): RG16F in 4 + GB2 8 + GB3 8 read, RG16F 4 written = 24 B.
//
// Tiled kernel: one CTA filters a 64x16 output tile.  The tile plus a halo of `step` texels of
//   * the input image (visibility, variance) as float2
//   * the decoded G-buffer normal + linear z as float4 (oct decode done ONCE per staged texel, not once per tap)
// is staged in shared memory with coalesced 8-byte/4-byte global loads (out-of-image texels are staged as zeros =
// texelFetch robust-access semantics); the 3x3 taps at stride `step` then come from shared memory.
// A CTA whose 16 reference tiles are all on the shadow list writes zeros and exits without loading anything.
#include "glsl_fast.cuh"
#include "hr_internal.h"

namespace {

using namespace gf;

constexpr int TILE_W = 64, TILE_H = 16, MAX_STEP = 8;
constexpr int REG_W_MAX = TILE_W + 2 * MAX_STEP, REG_H_MAX = TILE_H + 2 * MAX_STEP;

struct AtrousParams {
    int   W, H, step, radius;
    float phi_visibility, phi_normal, sigma_depth, power;
    int   row0, row1;
};

// ---- naive reference kernel (global memory only); kept for A/B validation of the tiled kernel -------------------
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

} // namespace

// 0 = naive, 1 = tiled scalar kernel.  hr_debug_set key 1.  (A sliding-register-window "chain" variant, which traded
// occupancy for shared-memory traffic, has been removed.)
// 3 = pixel-pair kernel (svgf_atrous_v3.cu, default); it falls back to the
// scalar tiled kernel for odd widths / phi_normal != 32.
int g_hr_atrous_impl = 3;
bool launch_shadows_atrous_v3(const GBufLevelDev& g, const uint32_t* in, const uint8_t* tile_flags, int radius, int step, float phi_vis, float phi_n, float sigma_z,
                              float power, uint32_t* out, int row0, int row1, cudaStream_t st); // svgf_atrous_v3.cu (impl 3: pixel pairs)

void launch_shadows_atrous(const GBufLevelDev& g, const __half2* in, const uint8_t* tile_flags, int radius, int step, float phi_vis, float phi_n,
                           float sigma_z, float power, __half2* out, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    AtrousParams P { g.W, g.H, step, radius, phi_vis, phi_n, sigma_z, power, row0, row1 };
    const uint32_t* i32 = reinterpret_cast<const uint32_t*>(in);
    uint32_t*       o32 = reinterpret_cast<uint32_t*>(out);
    const bool tiled_ok = g_hr_atrous_impl != 0 && radius == 1 && (step == 1 || step == 2 || step == 4 || step == 8);
    if (g_hr_atrous_impl == 3 && launch_shadows_atrous_v3(g, i32, tile_flags, radius, step, phi_vis, phi_n, sigma_z, power, o32, row0, row1, st)) return;
    if (tiled_ok)
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
