// svgf_atrous_v3.cu — shadows a-trous (K4+K5, shadows_denoise_atrous.comp:94-174) on pixel pairs.
//
// The scalar tiled kernel (svgf_atrous.cu) is instruction-issue bound: ~23 FP32 instructions per tap.  This kernel lets
// every thread filter TWO horizontally adjacent pixels and keeps each per-pixel quantity of the pair in one 64-bit register
// pair (gf::ffma2 / fmul2 / fadd2: two scalar instructions each on sm_90, which has no packed fp32), so the per-tap address
// arithmetic, shared-memory loads and loop overhead are shared by both pixels.
// Shared memory holds the staged tile as six fp32 planes (nx, ny, nz, z*log2e/sigma, visibility, variance); an aligned
// LDS.64 fetches the same plane value for both pixels of a pair (taps at even column offsets), odd offsets (STEP = 1,
// dx = +-1) use two LDS.32 straight into the register pair.  Out-of-image cells are staged with a zero normal (weight 0,
// = the reference's `inside` test) and zero variance (texelFetch robust-access zeros).
#include "glsl_fast.cuh"
#include "hr_internal.h"

namespace {

using namespace gf;

constexpr int TW3 = 64, TH3 = 16;

struct V3Params {
    int   W, H;
    float c_sigma;   // log2(e) / sigma_depth
    float c_phi0;    // -log2(e) / phi_visibility
    float power;
    int   row0, row1;
};

__device__ __forceinline__ float2 ld_pair(const float* __restrict__ plane, int idx, bool aligned)
{
    if (aligned) return *reinterpret_cast<const float2*>(plane + idx);
    return make_float2(plane[idx], plane[idx + 1]);
}

struct PairCell { float2 nx, ny, nz, zs, vis, var; };

// the six staged planes of a tile region
struct Planes { const float *nx, *ny, *nz, *zs, *vi, *va; };

// Stage the texel pair (px, px+1) of row py (px even) into the six planes at region index ri (even): decoded normal,
// scaled linear depth, visibility, variance; zeros outside the image (zero normal = weight 0, the reference's `inside`).
__device__ __forceinline__ void stage_pair(const GBufLevelDev& g, const uint32_t* __restrict__ in, float c_sigma, int px, int py, int W, int H, int ri, float* s_nx,
                                           float* s_ny, float* s_nz, float* s_zs, float* s_vi, float* s_va)
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
    *reinterpret_cast<float2*>(s_nx + ri) = nx; *reinterpret_cast<float2*>(s_ny + ri) = ny; *reinterpret_cast<float2*>(s_nz + ri) = nz;
    *reinterpret_cast<float2*>(s_zs + ri) = zs; *reinterpret_cast<float2*>(s_vi + ri) = vi; *reinterpret_cast<float2*>(s_va + ri) = va;
}

// Filter the pixel pair whose centre cell is at region index ci and store it at out[idx] (and out[idx + 1] when has1); row /
// column tap strides in cells are (rs, cs).  up / dn: the cells directly above / below the centre at UNIT pixel spacing in a
// variance plane (the dense tile keeps them in its main variance plane, the row-interleaved tile in side buffers).
template <bool ALIGNED_X>
__device__ __forceinline__ void filter_store_pair(const Planes& s, int ci, int rs, int cs, const float* up, const float* dn, const V3Params& P,
                                                  uint32_t* __restrict__ out, size_t idx, bool has1)
{
    const float2 neg1 = make_float2(-1.0f, -1.0f), nl2e = make_float2(-1.44269504f, -1.44269504f);
    const float  LK1 = -0.5849625007f, LK2 = -1.1699250014f; // log2(2/3), log2(4/9): kernel weights folded into the exponent
    PairCell     c;
    c.nx = ld_pair(s.nx, ci, true); c.ny = ld_pair(s.ny, ci, true); c.nz = ld_pair(s.nz, ci, true);
    c.zs = ld_pair(s.zs, ci, true); c.vis = ld_pair(s.vi, ci, true); c.var = ld_pair(s.va, ci, true);
    // compute_variance_center for both pixels: columns ci-1 .. ci+2, rows -1..+1; weights {1/4,1/8,1/16}
    float2 vbar;
    {
        const float  a0 = up[-1], d0 = up[2];
        const float2 m0 = *reinterpret_cast<const float2*>(up);
        const float  a1 = s.va[ci - 1], d1 = s.va[ci + 2];
        const float  a2 = dn[-1], d2 = dn[2];
        const float2 m2 = *reinterpret_cast<const float2*>(dn);
        vbar.x = 0.25f * c.var.x + 0.125f * (a1 + c.var.y + m0.x + m2.x) + 0.0625f * (a0 + m0.y + a2 + m2.y);
        vbar.y = 0.25f * c.var.y + 0.125f * (c.var.x + d1 + m0.y + m2.y) + 0.0625f * (m0.x + d0 + m2.x + d2);
    }
    const float2 cphi = make_float2(P.c_phi0 * rsqrtf(fmaxf(1e-10f + vbar.x, 1e-30f)), P.c_phi0 * rsqrtf(fmaxf(1e-10f + vbar.y, 1e-30f)));
    float2 sumw = make_float2(1.0f, 1.0f), s0 = c.vis, s1 = c.var;
#pragma unroll
    for (int yy = -1; yy <= 1; yy++)
#pragma unroll
        for (int xx = -1; xx <= 1; xx++)
        {
            if (xx == 0 && yy == 0) continue;
            const float lk      = (xx != 0 && yy != 0) ? LK2 : LK1;
            const int   si      = ci + yy * rs + xx * cs;
            const bool  aligned = ALIGNED_X || xx == 0;
            PairCell    t;
            t.nx = ld_pair(s.nx, si, aligned); t.ny = ld_pair(s.ny, si, aligned); t.nz = ld_pair(s.nz, si, aligned);
            t.zs = ld_pair(s.zs, si, aligned); t.vis = ld_pair(s.vi, si, aligned); t.var = ld_pair(s.va, si, aligned);
            const float2 dz = ffma2(t.zs, neg1, c.zs);
            float2       wZ;
            wZ.x = fast_exp2(-fabsf(dz.x));
            wZ.y = fast_exp2(-fabsf(dz.y));
            const float2 dl = ffma2(t.vis, neg1, c.vis);
            float2       ea;
            ea.x = fmaf(fabsf(dl.x), cphi.x, lk);
            ea.y = fmaf(fabsf(dl.y), cphi.y, lk);
            ea   = ffma2(wZ, nl2e, ea);
            float2 e;
            e.x = fast_exp2(ea.x);
            e.y = fast_exp2(ea.y);
            float2 nd = fmul2(c.nz, t.nz);
            nd        = ffma2(c.ny, t.ny, nd);
            nd        = ffma2(c.nx, t.nx, nd);
            nd.x      = fmaxf(nd.x, 0.0f);
            nd.y      = fmaxf(nd.y, 0.0f);
            float2 p = fmul2(nd, nd);
            p        = fmul2(p, p);
            p        = fmul2(p, p);
            p        = fmul2(p, p);
            p        = fmul2(p, p);
            const float2 wk = fmul2(e, p);
            sumw = fadd2(sumw, wk);
            s0   = ffma2(wk, t.vis, s0);
            s1   = ffma2(fmul2(wk, wk), t.var, s1);
        }
    const float2 inv = make_float2(fast_rcp(sumw.x), fast_rcp(sumw.y));
    float2       o0 = fmul2(s0, inv), o1 = fmul2(fmul2(s1, inv), inv);
    if (P.power != 0.0f) { o0.x = pow_pos(o0.x, P.power); o0.y = pow_pos(o0.y, P.power); }
    // sky pixels (linear z < 0) pass the input through
    const uint32_t r0 = c.zs.x < 0.0f ? f2_to_h2(c.vis.x, c.var.x) : f2_to_h2(o0.x, o1.x);
    const uint32_t r1 = c.zs.y < 0.0f ? f2_to_h2(c.vis.y, c.var.y) : f2_to_h2(o0.y, o1.y);
    if (has1) *reinterpret_cast<uint2*>(out + idx) = make_uint2(r0, r1); // idx even (W even is required by the launcher)
    else out[idx] = r0;
}

template <int STEP>
__global__ void __launch_bounds__(256) k_atrous_v3(GBufLevelDev g, const uint32_t* __restrict__ in, const uint8_t* __restrict__ tile_flags, V3Params P,
                                                    uint32_t* __restrict__ out)
{
    extern __shared__ float smem_f[];
    constexpr int PADL = STEP + (STEP & 1);             // even left pad => even region column for even image column
    constexpr int RW   = (TW3 + PADL + STEP + 1) & ~1;  // even row pitch keeps LDS.64 alignment on every row
    constexpr int RH   = TH3 + 2 * STEP;
    constexpr int PL   = RW * RH;
    float* s_nx = smem_f;
    float* s_ny = s_nx + PL;
    float* s_nz = s_ny + PL;
    float* s_zs = s_nz + PL;
    float* s_vi = s_zs + PL;
    float* s_va = s_vi + PL;
    __shared__ uint32_t s_tf;

    const int W = P.W, H = P.H;
    const int x0 = blockIdx.x * TW3, y0 = P.row0 + blockIdx.y * TH3;
    const int TWt = (W + 7) >> 3, THt = (H + 7) >> 3;
    if (threadIdx.x < 32)
    {
        const int  tx = (x0 >> 3) + (threadIdx.x & 7), ty = (y0 >> 3) + (threadIdx.x >> 3);
        const bool f  = threadIdx.x < 16 && tx < TWt && ty < THt && tile_flags[(size_t)ty * TWt + tx] != 0;
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, f);
        if (threadIdx.x == 0) s_tf = b;
    }
    __syncthreads();
    const uint32_t tf = s_tf;

    if (tf != 0)
    {
        // staged two texels at a time: the region starts on an even column and W is even, so a pair is either inside or
        // outside the image and its G-buffer words are one aligned 16-byte load each (half the load / store instructions)
        for (int i = threadIdx.x; i < (RW / 2) * RH; i += 256)
        {
            const int rx = 2 * (i % (RW / 2)), ry = i / (RW / 2);
            const int px = x0 - PADL + rx, py = y0 - STEP + ry;
            stage_pair(g, in, P.c_sigma, px, py, W, H, ry * RW + rx, s_nx, s_ny, s_nz, s_zs, s_vi, s_va);
        }
    }
    __syncthreads();

    const Planes pl { s_nx, s_ny, s_nz, s_zs, s_vi, s_va };
    const int    lx2 = threadIdx.x & 31, lyb = threadIdx.x >> 5; // 32 pixel pairs x 8 rows, 2 rows per thread
    const int    x = x0 + 2 * lx2;
#pragma unroll
    for (int k = 0; k < TH3 / 8; k++)
    {
        const int ly = lyb + 8 * k, y = y0 + ly;
        if (x >= W || y >= H || y >= P.row1) continue;
        const size_t idx  = (size_t)y * W + x;
        const bool   has1 = x + 1 < W;
        if (!((tf >> ((ly >> 3) * 8 + (lx2 >> 2))) & 1u))
        {
            out[idx] = 0u;
            if (has1) out[idx + 1] = 0u;
            continue;
        }
        const int ci = (ly + STEP) * RW + 2 * lx2 + PADL;
        filter_store_pair<(STEP & 1) == 0>(pl, ci, STEP * RW, STEP, s_va + ci - RW, s_va + ci + RW, P, out, idx, has1);
    }
}

// ---- row-interleaved tiles for the wide steps ---------------------------------------------------------------------------
// With the dense 64x16 tile a step-8 iteration stages (64+16) x (16+16) texels for 1024 outputs (2.5x).  The taps of row y
// only touch rows y and y +- STEP, so a CTA that filters the 16 rows {Y0 + phase + STEP*j} (one residue class of the row index) needs just 18 staged rows: (64+16) x 18 = 1.4x.  Rows stay contiguous in x, so
// global accesses are as coalesced as before.  compute_variance_center works at unit pixel spacing whatever the step:
// the variance of the rows y-1 / y+1 (centre columns only) is staged into two extra single-plane buffers.
template <int STEP>
__global__ void __launch_bounds__(256) k_atrous_v3s(GBufLevelDev g, const uint32_t* __restrict__ in, const uint8_t* __restrict__ tile_flags, V3Params P,
                                                     uint32_t* __restrict__ out)
{
    extern __shared__ float smem_f[];
    constexpr int PADL = STEP;                 // STEP is even here
    constexpr int RW   = TW3 + 2 * STEP;       // even
    constexpr int RH   = TH3 + 2;
    constexpr int PL   = RW * RH;
    constexpr int TROWS = (TH3 * STEP) / 8;    // 8-row tile rows spanned by the CTA's 16*STEP image rows
    float* s_nx = smem_f;
    float* s_ny = s_nx + PL;
    float* s_nz = s_ny + PL;
    float* s_zs = s_nz + PL;
    float* s_vi = s_zs + PL;
    float* s_va = s_vi + PL;
    float* s_vadj = s_va + PL;                 // [2][TH3][RW]: variance of rows y-1 (0) and y+1 (1)
    __shared__ uint8_t s_tfl[TROWS][8];
    __shared__ int     s_any;

    const int W = P.W, H = P.H;
    const int x0 = blockIdx.x * TW3;
    const int blk = blockIdx.y / STEP, phase = blockIdx.y - blk * STEP;
    const int Y0 = P.row0 + blk * (TH3 * STEP); // multiple of 8 (row0 is)
    const int TWt = (W + 7) >> 3, THt = (H + 7) >> 3;
    if (threadIdx.x == 0) s_any = 0;
    __syncthreads();
    if (threadIdx.x < TROWS * 8)
    {
        const int  tx = (x0 >> 3) + (threadIdx.x & 7), ty = (Y0 >> 3) + (threadIdx.x >> 3);
        const bool f  = tx < TWt && ty < THt && tile_flags[(size_t)ty * TWt + tx] != 0;
        s_tfl[threadIdx.x >> 3][threadIdx.x & 7] = f ? 1 : 0;
        if (f) s_any = 1;
    }
    __syncthreads();

    if (s_any)
    {
        for (int i = threadIdx.x; i < (RW / 2) * RH; i += 256)
        {
            const int rx = 2 * (i % (RW / 2)), ry = i / (RW / 2);
            const int px = x0 - PADL + rx, py = Y0 + phase + STEP * (ry - 1);
            stage_pair(g, in, P.c_sigma, px, py, W, H, ry * RW + rx, s_nx, s_ny, s_nz, s_zs, s_vi, s_va);
        }
        // variance of the rows above / below each filtered row, texel pairs covering columns x0-2 .. x0+TW3+1
        constexpr int VP = TW3 / 2 + 2;
        for (int i = threadIdx.x; i < 2 * TH3 * VP; i += 256)
        {
            const int a = i / (TH3 * VP), r = i - a * (TH3 * VP), j = r / VP, c = 2 * (r - j * VP);
            const int px = x0 - 2 + c, py = Y0 + phase + STEP * j + (a ? 1 : -1);
            float2    va = make_float2(0.0f, 0.0f);
            if (px >= 0 && py >= 0 && px < W && py < H)
            {
                const uint2 w = __ldg(reinterpret_cast<const uint2*>(in + (size_t)py * W + px));
                va = make_float2(h2_to_f2(w.x).y, h2_to_f2(w.y).y);
            }
            *reinterpret_cast<float2*>(s_vadj + (a * TH3 + j) * RW + PADL - 2 + c) = va;
        }
    }
    __syncthreads();

    const Planes pl { s_nx, s_ny, s_nz, s_zs, s_vi, s_va };
    const int    lx2 = threadIdx.x & 31, lyb = threadIdx.x >> 5; // 32 pixel pairs x 8 rows, 2 rows per thread
    const int    x = x0 + 2 * lx2;
#pragma unroll
    for (int k = 0; k < TH3 / 8; k++)
    {
        const int ly = lyb + 8 * k, y = Y0 + phase + STEP * ly;
        if (x >= W || y >= H || y >= P.row1) continue;
        const size_t idx  = (size_t)y * W + x;
        const bool   has1 = x + 1 < W;
        if (!s_tfl[(phase + STEP * ly) >> 3][lx2 >> 2])
        {
            out[idx] = 0u;
            if (has1) out[idx + 1] = 0u;
            continue;
        }
        const int ci = (ly + 1) * RW + 2 * lx2 + PADL;
        filter_store_pair<true>(pl, ci, RW, STEP, s_vadj + (0 * TH3 + ly) * RW + 2 * lx2 + PADL, s_vadj + (1 * TH3 + ly) * RW + 2 * lx2 + PADL, P, out, idx, has1);
    }
}

template <int STEP>
void launch_v3s(const GBufLevelDev& g, const uint32_t* in, const uint8_t* tf, const V3Params& P, uint32_t* out, cudaStream_t st)
{
    constexpr int RW = TW3 + 2 * STEP, RH = TH3 + 2;
    const size_t  smem = ((size_t)RW * RH * 6 + (size_t)2 * TH3 * RW) * sizeof(float);
    static bool   configured[64] = {};
    if (hr_once_per_device(configured)) cudaFuncSetAttribute(k_atrous_v3s<STEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int rows = P.row1 - P.row0, blocks = (rows + TH3 * STEP - 1) / (TH3 * STEP);
    dim3      grid((P.W + TW3 - 1) / TW3, blocks * STEP);
    k_atrous_v3s<STEP><<<grid, 256, smem, st>>>(g, in, tf, P, out);
}

template <int STEP>
void launch_v3(const GBufLevelDev& g, const uint32_t* in, const uint8_t* tf, const V3Params& P, uint32_t* out, cudaStream_t st)
{
    constexpr int PADL = STEP + (STEP & 1);
    constexpr int RW   = (TW3 + PADL + STEP + 1) & ~1;
    constexpr int RH   = TH3 + 2 * STEP;
    const size_t  smem = (size_t)RW * RH * 6 * sizeof(float);
    static bool   configured[64] = {};
    if (hr_once_per_device(configured)) cudaFuncSetAttribute(k_atrous_v3<STEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid((P.W + TW3 - 1) / TW3, (P.row1 - P.row0 + TH3 - 1) / TH3);
    k_atrous_v3<STEP><<<grid, 256, smem, st>>>(g, in, tf, P, out);
}

} // namespace

// returns false when this variant does not support the configuration (caller falls back to the scalar kernels)
bool launch_shadows_atrous_v3(const GBufLevelDev& g, const uint32_t* in, const uint8_t* tile_flags, int radius, int step, float phi_vis, float phi_n, float sigma_z,
                              float power, uint32_t* out, int row0, int row1, cudaStream_t st)
{
    if (radius != 1 || phi_n != 32.0f || (g.W & 1) || row0 % 8 != 0 || !(step == 1 || step == 2 || step == 4 || step == 8)) return false;
    V3Params P { g.W, g.H, 1.44269504f / sigma_z, -1.44269504f / phi_vis, power, row0, row1 };
    switch (step)
    {
        case 1: launch_v3<1>(g, in, tile_flags, P, out, st); break;
        case 2: launch_v3<2>(g, in, tile_flags, P, out, st); break;
        case 4: launch_v3<4>(g, in, tile_flags, P, out, st); break;
        default: launch_v3s<8>(g, in, tile_flags, P, out, st); break; // row-interleaved tiles (DESIGN.md §8)
    }
    return true;
}
