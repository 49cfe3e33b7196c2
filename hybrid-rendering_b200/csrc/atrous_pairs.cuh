// atrous_pairs.cuh — the pixel-pair a-trous tile kernels of the shadows (svgf_atrous.cu, K4+K5) and reflections
// (svgf_refl_atrous.cu, K15+K16) denoisers.
//
// The scalar a-trous kernels are instruction-issue bound: ~23 FP32 instructions per tap.  Here every thread filters TWO
// horizontally adjacent pixels and keeps each per-pixel quantity of the pair in one 64-bit register pair (gf::ffma2 / fmul2 /
// fadd2: two scalar instructions each on sm_90, which has no packed fp32), so the per-tap address arithmetic, shared-memory
// loads and loop overhead are shared by both pixels.
// A CTA filters a 64x16 pixel tile.  Shared memory holds the staged region as fp32 planes PL floats apart: the decoded normal
// (0-2), linear z * log2(e) / sigma_depth (3), the pass's NC colour planes (4 ..), its variance plane (4 + NC) and, when the
// luminance is not a colour plane, a luminance plane.  An aligned LDS.64 fetches the same plane value for both pixels of a pair
// (taps at even column offsets), odd offsets (STEP = 1, dx = +-1) use two LDS.32 straight into the register pair.
// Out-of-image cells are staged with a zero normal (weight 0, = the reference's `inside` test) and zero colour / variance
// (texelFetch robust-access zeros for compute_variance_center).
//
// The kernel bodies take a pass policy with:
//   In, Out, Params    input / output texel types and the kernel parameters (W, H, c_sigma, c_phi0, row0, row1)
//   NPL, NC            staged planes per cell, colour planes
//   COPY_EMPTY_CTA     true: a CTA without a flagged tile copies in -> out (copy) and returns before staging;
//                      false: it skips staging and filter_store handles its (unflagged) pixels
//   stage(g, in, c_sigma, px, py, W, H, ri, s, PL)  stage the texel pair (px, px+1) of row py (px even) at region index ri (even)
//   side_var(in, pi)                 the variances of the texels pi, pi+1 (row-interleaved side buffers)
//   filter_store<ALIGNED_X>(g, P, taps, out, idx, has1, flagged)   filter and store the pair at out[idx] (and out[idx + 1])
#pragma once
#include "glsl_fast.cuh"
#include "hr_internal.h"

// File-local in each including file, like the kernels.  ptxas starts the dynamic shared memory of every kernel of a file at the
// largest alignment of the file's dynamic shared-memory arrays: 128 bytes in svgf_refl_atrous.cu (the TMA kernel's boxes).
namespace {

constexpr int PAIR_TILE_W = 64, PAIR_TILE_H = 16;

// Dense tile: 64x16 pixels + STEP halo on every side.
template <int STEP, int NPL>
struct DenseTile {
    static constexpr int PADL = STEP + (STEP & 1);                // even left pad => even region column for even image column
    static constexpr int RW   = (PAIR_TILE_W + PADL + STEP + 1) & ~1; // even row pitch keeps LDS.64 alignment on every row
    static constexpr int RH   = PAIR_TILE_H + 2 * STEP;
    static constexpr int PL   = RW * RH;
    static constexpr int SMEM = NPL * PL * (int)sizeof(float);
    static dim3 grid(int W, int rows) { return dim3((W + PAIR_TILE_W - 1) / PAIR_TILE_W, (rows + PAIR_TILE_H - 1) / PAIR_TILE_H); }
};

// Row-interleaved tile for the wide steps.  With the dense tile a step-8 iteration stages (64+16) x (16+16) texels for 1024
// outputs (2.5x).  The taps of row y only touch rows y and y +- STEP, so a CTA that filters the 16 rows {Y0 + phase + STEP*j}
// (one residue class of the row index) needs just 18 staged rows: (64+16) x 18 = 1.4x.  Rows stay contiguous in x, so global
// accesses are as coalesced as before.  compute_variance_center works at unit pixel spacing whatever the step: the variance
// of the rows y-1 / y+1 (centre columns only) is staged into two extra single-plane side buffers.
template <int STEP, int NPL>
struct InterleavedTile {
    static_assert((STEP & 1) == 0, "row-interleaved tiles are for even steps");
    static constexpr int PADL  = STEP;
    static constexpr int RW    = PAIR_TILE_W + 2 * STEP; // even
    static constexpr int RH    = PAIR_TILE_H + 2;
    static constexpr int PL    = RW * RH;
    static constexpr int TROWS = (PAIR_TILE_H * STEP) / 8; // 8-row tile rows spanned by the CTA's 16 * STEP image rows
    static constexpr int SMEM  = (NPL * PL + 2 * PAIR_TILE_H * RW) * (int)sizeof(float);
    static dim3 grid(int W, int rows) { return dim3((W + PAIR_TILE_W - 1) / PAIR_TILE_W, (rows + PAIR_TILE_H * STEP - 1) / (PAIR_TILE_H * STEP) * STEP); }
};

__device__ __forceinline__ float2 ld_pair(const float* __restrict__ plane, int idx, bool aligned)
{
    if (aligned) return *reinterpret_cast<const float2*>(plane + idx);
    return make_float2(plane[idx], plane[idx + 1]);
}

// bit of the 8x8 tile holding pixel pair lx2 of row ly in a dense tile's 16-bit flag mask
__device__ __forceinline__ int dense_flag_bit(int lx2, int ly) { return (ly >> 3) * 8 + (lx2 >> 2); }

// The taps of one pixel pair: centre cell at region index ci of the planes at s, row / column tap strides (rs, cs) in cells.
// up / dn: the cells directly above / below the centre at UNIT pixel spacing in a variance plane (the dense tile keeps them in
// its main variance plane, the row-interleaved tile in side buffers).
struct PairTaps {
    const float* s;
    int          PL, ci, rs, cs;
    const float *up, *dn;
};

template <int NC>
struct PairSum { float2 c[NC], v; }; // filtered colour channels and variance of a pixel pair

// The 3x3 edge-stopping filter of a pixel pair over NC colour planes.  LUM is the plane of the luminance the colour weight
// compares (a colour plane is not loaded twice).
template <int NC, int LUM, bool ALIGNED_X>
__device__ __forceinline__ PairSum<NC> filter_pair(const PairTaps& t, float c_phi0)
{
    using namespace gf;
    static_assert(NC == 1 || NC == 3, "one or three colour planes");
    constexpr int VAR = 4 + NC;
    const float* __restrict__ s = t.s;
    const int    PL = t.PL, ci = t.ci;
    const float2 cnx = ld_pair(s, ci, true), cny = ld_pair(s + PL, ci, true), cnz = ld_pair(s + 2 * PL, ci, true), czs = ld_pair(s + 3 * PL, ci, true);
    float2       acc[NC];
#pragma unroll
    for (int c = 0; c < NC; c++) acc[c] = ld_pair(s + (4 + c) * PL, ci, true);
    const float2 cva = ld_pair(s + VAR * PL, ci, true);
    float2       clu;
    if constexpr (LUM < VAR) clu = acc[LUM - 4];
    else clu = ld_pair(s + LUM * PL, ci, true);
    // compute_variance_center for both pixels: columns ci-1 .. ci+2, rows -1..+1; weights {1/4,1/8,1/16}
    float2 vbar;
    {
        const float  a0 = t.up[-1], d0 = t.up[2];
        const float2 m0 = *reinterpret_cast<const float2*>(t.up);
        const float  a1 = s[VAR * PL + ci - 1], d1 = s[VAR * PL + ci + 2];
        const float  a2 = t.dn[-1], d2 = t.dn[2];
        const float2 m2 = *reinterpret_cast<const float2*>(t.dn);
        vbar.x = 0.25f * cva.x + 0.125f * (a1 + cva.y + m0.x + m2.x) + 0.0625f * (a0 + m0.y + a2 + m2.y);
        vbar.y = 0.25f * cva.y + 0.125f * (cva.x + d1 + m0.y + m2.y) + 0.0625f * (m0.x + d0 + m2.x + d2);
    }
    const float2 cphi = make_float2(c_phi0 * rsqrtf(fmaxf(1e-10f + vbar.x, 1e-30f)), c_phi0 * rsqrtf(fmaxf(1e-10f + vbar.y, 1e-30f)));
    const float2 neg1 = make_float2(-1.0f, -1.0f), nl2e = make_float2(-1.44269504f, -1.44269504f);
    const float  LK1 = -0.5849625007f, LK2 = -1.1699250014f; // log2(2/3), log2(4/9): kernel weights folded into the exponent
    float2       sumw = make_float2(1.0f, 1.0f), av = cva;
#pragma unroll
    for (int yy = -1; yy <= 1; yy++)
#pragma unroll
        for (int xx = -1; xx <= 1; xx++)
        {
            if (xx == 0 && yy == 0) continue;
            const float lk = (xx != 0 && yy != 0) ? LK2 : LK1;
            const int   si = ci + yy * t.rs + xx * t.cs;
            const bool  al = ALIGNED_X || xx == 0;
            const float2 snx = ld_pair(s, si, al), sny = ld_pair(s + PL, si, al), snz = ld_pair(s + 2 * PL, si, al), szs = ld_pair(s + 3 * PL, si, al);
            float2       sc[NC];
#pragma unroll
            for (int c = 0; c < NC; c++) sc[c] = ld_pair(s + (4 + c) * PL, si, al);
            const float2 sv = ld_pair(s + VAR * PL, si, al);
            float2       sl;
            if constexpr (LUM < VAR) sl = sc[LUM - 4];
            else sl = ld_pair(s + LUM * PL, si, al);
            const float2 dz = ffma2(szs, neg1, czs);
            float2       wZ;
            wZ.x = fast_exp2(-fabsf(dz.x));
            wZ.y = fast_exp2(-fabsf(dz.y));
            const float2 dl = ffma2(sl, neg1, clu);
            float2       ea;
            ea.x = fmaf(fabsf(dl.x), cphi.x, lk);
            ea.y = fmaf(fabsf(dl.y), cphi.y, lk);
            ea   = ffma2(wZ, nl2e, ea);
            float2 e;
            e.x = fast_exp2(ea.x);
            e.y = fast_exp2(ea.y);
            float2 nd = fmul2(cnz, snz);
            nd        = ffma2(cny, sny, nd);
            nd        = ffma2(cnx, snx, nd);
            nd.x      = fmaxf(nd.x, 0.0f);
            nd.y      = fmaxf(nd.y, 0.0f);
            float2 p = fmul2(nd, nd); // normal weight: nd^32
            p        = fmul2(p, p);
            p        = fmul2(p, p);
            p        = fmul2(p, p);
            p        = fmul2(p, p);
            const float2 wk = fmul2(e, p);
            sumw = fadd2(sumw, wk);
            // written out, not a loop: a loop over acc[] is unrolled after acc[] becomes registers, and that reorders the arithmetic
            acc[0] = ffma2(wk, sc[0], acc[0]);
            if constexpr (NC == 3) { acc[1] = ffma2(wk, sc[1], acc[1]); acc[2] = ffma2(wk, sc[2], acc[2]); }
            av = ffma2(fmul2(wk, wk), sv, av);
        }
    const float2 inv = make_float2(fast_rcp(sumw.x), fast_rcp(sumw.y));
    PairSum<NC>  r;
    r.c[0] = fmul2(acc[0], inv);
    if constexpr (NC == 3) { r.c[1] = fmul2(acc[1], inv); r.c[2] = fmul2(acc[2], inv); }
    r.v = fmul2(fmul2(av, inv), inv);
    return r;
}

// Dense-tile kernel body: the CTA stages its 64x16 tile + STEP halo and filters it.
template <class Pass, int STEP>
__device__ __forceinline__ void atrous_dense(const GBufLevelDev& g, const typename Pass::In* __restrict__ in, const uint8_t* __restrict__ tile_flags,
                                             const typename Pass::Params& P, typename Pass::Out* __restrict__ out)
{
    using G = DenseTile<STEP, Pass::NPL>;
    extern __shared__ float smem_f[];
    __shared__ uint32_t s_tf;
    const int W = P.W, H = P.H;
    const int x0 = blockIdx.x * PAIR_TILE_W, y0 = P.row0 + blockIdx.y * PAIR_TILE_H;
    const int TWt = (W + 7) >> 3, THt = (H + 7) >> 3;
    if (threadIdx.x < 32)
    {
        const int      tx = (x0 >> 3) + (threadIdx.x & 7), ty = (y0 >> 3) + (threadIdx.x >> 3);
        const bool     f  = threadIdx.x < 16 && tx < TWt && ty < THt && tile_flags[(size_t)ty * TWt + tx] != 0;
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, f);
        if (threadIdx.x == 0) s_tf = b;
    }
    __syncthreads();
    const uint32_t tf = s_tf;
    // A copying pass computes the pair coordinates before its copy branch and reuses them below; the other pass computes them
    // after the staging barrier.  Each keeps the instruction order it was tuned with.
    if constexpr (Pass::COPY_EMPTY_CTA)
    {
        const int lx2 = threadIdx.x & 31, lyb = threadIdx.x >> 5, x = x0 + 2 * lx2;
        if (tf == 0)
        {
#pragma unroll
            for (int k = 0; k < PAIR_TILE_H / 8; k++)
            {
                const int y = y0 + lyb + 8 * k;
                if (x >= W || y >= H || y >= P.row1) continue;
                Pass::copy(in, out, (size_t)y * W + x, x + 1 < W);
            }
            return;
        }
    }
    if (Pass::COPY_EMPTY_CTA || tf != 0)
    {
        // staged two texels at a time: the region starts on an even column and W is even, so a pair is either inside or
        // outside the image and its G-buffer words are one aligned 16-byte load each (half the load / store instructions)
        for (int i = threadIdx.x; i < (G::RW / 2) * G::RH; i += 256)
        {
            const int rx = 2 * (i % (G::RW / 2)), ry = i / (G::RW / 2);
            Pass::stage(g, in, P.c_sigma, x0 - G::PADL + rx, y0 - STEP + ry, W, H, ry * G::RW + rx, smem_f, G::PL);
        }
    }
    __syncthreads();
    const float* s_va = smem_f + (4 + Pass::NC) * G::PL;
    const int    lx2 = threadIdx.x & 31, lyb = threadIdx.x >> 5; // 32 pixel pairs x 8 rows, 2 rows per thread
    const int    x   = x0 + 2 * lx2;
#pragma unroll
    for (int k = 0; k < PAIR_TILE_H / 8; k++)
    {
        const int ly = lyb + 8 * k, y = y0 + ly;
        if (x >= W || y >= H || y >= P.row1) continue;
        const size_t idx  = (size_t)y * W + x;
        const bool   has1 = x + 1 < W;
        const int    ci   = (ly + STEP) * G::RW + 2 * lx2 + G::PADL;
        Pass::template filter_store<(STEP & 1) == 0>(g, P, PairTaps { smem_f, G::PL, ci, STEP * G::RW, STEP, s_va + ci - G::RW, s_va + ci + G::RW }, out, idx, has1,
                                                     (tf >> dense_flag_bit(lx2, ly)) & 1u);
    }
}

// Row-interleaved kernel body: blockIdx.y = 16-row block * STEP + phase; the CTA filters the rows Y0 + phase + STEP * j, j < 16.
template <class Pass, int STEP>
__device__ __forceinline__ void atrous_interleaved(const GBufLevelDev& g, const typename Pass::In* __restrict__ in, const uint8_t* __restrict__ tile_flags,
                                                   const typename Pass::Params& P, typename Pass::Out* __restrict__ out)
{
    using G = InterleavedTile<STEP, Pass::NPL>;
    extern __shared__ float smem_f[];
    float* s_vadj = smem_f + Pass::NPL * G::PL; // [2][PAIR_TILE_H][RW]: variance of rows y-1 (0) and y+1 (1)
    __shared__ uint8_t s_tfl[G::TROWS][8];
    __shared__ int     s_any;
    const int W = P.W, H = P.H;
    const int x0 = blockIdx.x * PAIR_TILE_W;
    const int blk = blockIdx.y / STEP, phase = blockIdx.y - blk * STEP;
    const int Y0 = P.row0 + blk * (PAIR_TILE_H * STEP); // multiple of 8 (row0 is)
    const int TWt = (W + 7) >> 3, THt = (H + 7) >> 3;
    if (threadIdx.x == 0) s_any = 0;
    __syncthreads();
    if (threadIdx.x < G::TROWS * 8)
    {
        const int  tx = (x0 >> 3) + (threadIdx.x & 7), ty = (Y0 >> 3) + (threadIdx.x >> 3);
        const bool f  = tx < TWt && ty < THt && tile_flags[(size_t)ty * TWt + tx] != 0;
        s_tfl[threadIdx.x >> 3][threadIdx.x & 7] = f ? 1 : 0;
        if (f) s_any = 1;
    }
    __syncthreads();
    if constexpr (Pass::COPY_EMPTY_CTA) // as in atrous_dense
    {
        const int lx2 = threadIdx.x & 31, lyb = threadIdx.x >> 5, x = x0 + 2 * lx2;
        if (!s_any)
        {
#pragma unroll
            for (int k = 0; k < PAIR_TILE_H / 8; k++)
            {
                const int y = Y0 + phase + STEP * (lyb + 8 * k);
                if (x >= W || y >= H || y >= P.row1) continue;
                Pass::copy(in, out, (size_t)y * W + x, x + 1 < W);
            }
            return;
        }
    }
    if (Pass::COPY_EMPTY_CTA || s_any)
    {
        for (int i = threadIdx.x; i < (G::RW / 2) * G::RH; i += 256)
        {
            const int rx = 2 * (i % (G::RW / 2)), ry = i / (G::RW / 2);
            Pass::stage(g, in, P.c_sigma, x0 - G::PADL + rx, Y0 + phase + STEP * (ry - 1), W, H, ry * G::RW + rx, smem_f, G::PL);
        }
        // variance of the rows above / below each filtered row, texel pairs covering columns x0-2 .. x0+PAIR_TILE_W+1
        constexpr int VP = PAIR_TILE_W / 2 + 2;
        for (int i = threadIdx.x; i < 2 * PAIR_TILE_H * VP; i += 256)
        {
            const int a = i / (PAIR_TILE_H * VP), r = i - a * (PAIR_TILE_H * VP), j = r / VP, c = 2 * (r - j * VP);
            const int px = x0 - 2 + c, py = Y0 + phase + STEP * j + (a ? 1 : -1);
            float2    va = make_float2(0.0f, 0.0f);
            if (px >= 0 && py >= 0 && px < W && py < H) va = Pass::side_var(in, (size_t)py * W + px);
            *reinterpret_cast<float2*>(s_vadj + (a * PAIR_TILE_H + j) * G::RW + G::PADL - 2 + c) = va;
        }
    }
    __syncthreads();
    const int lx2 = threadIdx.x & 31, lyb = threadIdx.x >> 5;
    const int x   = x0 + 2 * lx2;
#pragma unroll
    for (int k = 0; k < PAIR_TILE_H / 8; k++)
    {
        const int ly = lyb + 8 * k, y = Y0 + phase + STEP * ly;
        if (x >= W || y >= H || y >= P.row1) continue;
        const size_t idx  = (size_t)y * W + x;
        const bool   has1 = x + 1 < W;
        const int    ci   = (ly + 1) * G::RW + 2 * lx2 + G::PADL;
        Pass::template filter_store<true>(g, P,
                                          PairTaps { smem_f, G::PL, ci, G::RW, STEP, s_vadj + ly * G::RW + 2 * lx2 + G::PADL, s_vadj + (PAIR_TILE_H + ly) * G::RW + 2 * lx2 + G::PADL },
                                          out, idx, has1, s_tfl[(phase + STEP * ly) >> 3][lx2 >> 2] != 0);
    }
}

// Launch a pixel-pair kernel with tile geometry G (DenseTile or InterleavedTile) over the rows [P.row0, P.row1).  Each kernel
// has its own (G, Params) pair, so the per-device flag of its shared-memory attribute is its own.
template <class G, class In, class Out, class Params>
void launch_tiles(void (*kernel)(GBufLevelDev, const In*, const uint8_t*, Params, Out*), const GBufLevelDev& g, const In* in, const uint8_t* tf, const Params& P, Out* out,
                  cudaStream_t st)
{
    static bool configured[64] = {};
    if (hr_once_per_device(configured)) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM);
    kernel<<<G::grid(P.W, P.row1 - P.row0), 256, G::SMEM, st>>>(g, in, tf, P, out);
}

} // namespace
