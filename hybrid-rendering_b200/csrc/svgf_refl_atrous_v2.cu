// svgf_refl_atrous_v2.cu — reflections a-trous (K15 + K16, reflections_denoise_atrous.comp:94-181) on pixel pairs.
//
// This is the roofline kernel of BASELINE config 3 (4K full-res reflections: 36 algorithmic B/px/iteration, SURVEY.md §8d).  The
// scalar kernel (svgf_reflections.cu::k_refl_atrous) is instruction-issue bound like its shadows twin was; this one applies the
// same remedy as svgf_atrous_v3.cu: every thread filters TWO horizontally adjacent pixels and keeps each per-pixel quantity of
// the pair in one 64-bit register pair (gf::ffma2 / fmul2 / fadd2), so addressing, shared-memory loads and loop overhead are
// shared by both pixels.  Shared memory holds the staged tile + halo as nine fp32 planes (nx, ny, nz, z * log2e / sigma, r, g, b,
// variance, luminance — the sample luminance is computed once per staged texel instead of once per tap); an aligned LDS.64
// fetches a plane value for both pixels of a pair.  Out-of-image cells are staged with a zero normal (weight 0 = the
// reference's `inside` test) and zero colour / variance (texelFetch robust-access zeros for compute_variance_center).
// Tile classification (K13/K15): tiles whose flag is 0 are copied (reflections_denoise_copy_tiles.comp:35-38).
#include "glsl_fast.cuh"
#include "hr_internal.h"
#include <cuda.h> // CUtensorMap (driver types only; cuTensorMapEncodeTiled is fetched with cudaGetDriverEntryPoint)
#include <vector>

namespace {

using namespace gf;

constexpr int TWR = 64, THR = 16, NPL = 9;

struct R2Params {
    int   W, H;
    float c_sigma; // log2(e) / sigma_depth
    float c_phi0;  // -log2(e) / phi_color
    int   approx;  // approximate_with_ddgi
    int   row0, row1;
};

__device__ __forceinline__ float2 ldp(const float* __restrict__ plane, int idx, bool aligned)
{
    if (aligned) return *reinterpret_cast<const float2*>(plane + idx);
    return make_float2(plane[idx], plane[idx + 1]);
}

__device__ __forceinline__ float lum3(float r, float g, float b) { return fmaxf(r * 0.299f + g * 0.587f + b * 0.114f, 0.0001f); } // common.glsl:143

// Stage the texel pair (px, px+1) of row py (px even) at region index ri (even).
__device__ __forceinline__ void stage_pair9(const GBufLevelDev& g, const uint2* __restrict__ in, float c_sigma, int px, int py, int W, int H, int ri, float* s, int PL)
{
    float2 nx = make_float2(0.0f, 0.0f), ny = nx, nz = nx, zs = nx, cr = nx, cg = nx, cb = nx, va = nx, lu = make_float2(0.0001f, 0.0001f);
    if (px >= 0 && py >= 0 && px < W && py < H)
    {
        const size_t pi = (size_t)py * W + px;
        const uint4  a  = __ldg(reinterpret_cast<const uint4*>(g.gb2 + pi)); // two RGBA16F texels: .x / .z hold the oct normals
        const uint4  b  = __ldg(reinterpret_cast<const uint4*>(g.gb3 + pi)); // .y / .w hold (mesh id, linear z)
        const uint4  c  = __ldg(reinterpret_cast<const uint4*>(in + pi));    // two RGBA16F texels (rgb, variance)
        const float2 e0 = h2_to_f2(a.x), e1 = h2_to_f2(a.z);
        const float3 n0 = octohedral_to_direction(e0.x, e0.y), n1 = octohedral_to_direction(e1.x, e1.y);
        const float2 c0 = h2_to_f2(c.x), c1 = h2_to_f2(c.y), c2 = h2_to_f2(c.z), c3 = h2_to_f2(c.w);
        nx = make_float2(n0.x, n1.x); ny = make_float2(n0.y, n1.y); nz = make_float2(n0.z, n1.z);
        zs = make_float2(h2_to_f2(b.y).y * c_sigma, h2_to_f2(b.w).y * c_sigma);
        cr = make_float2(c0.x, c2.x); cg = make_float2(c0.y, c2.y); cb = make_float2(c1.x, c3.x); va = make_float2(c1.y, c3.y);
        lu = make_float2(lum3(c0.x, c0.y, c1.x), lum3(c2.x, c2.y, c3.x));
    }
    float* p = s + ri;
    *reinterpret_cast<float2*>(p) = nx; p += PL;
    *reinterpret_cast<float2*>(p) = ny; p += PL;
    *reinterpret_cast<float2*>(p) = nz; p += PL;
    *reinterpret_cast<float2*>(p) = zs; p += PL;
    *reinterpret_cast<float2*>(p) = cr; p += PL;
    *reinterpret_cast<float2*>(p) = cg; p += PL;
    *reinterpret_cast<float2*>(p) = cb; p += PL;
    *reinterpret_cast<float2*>(p) = va; p += PL;
    *reinterpret_cast<float2*>(p) = lu;
}

// Filter one pixel pair whose centre cell is at region index ci; row / column tap strides in cells are (rs, cs).
// vrow_up / vrow_dn: region indices of the cells directly above / below the centre at UNIT pixel spacing in the variance plane
// given by vplane_up / vplane_dn (the dense tile keeps them in the main variance plane; the row-interleaved tile in side buffers).
template <bool ALIGNED_X>
__device__ __forceinline__ void filter_pair(const float* __restrict__ s, int PL, int ci, int rs, int cs, const float* __restrict__ v_up, const float* __restrict__ v_dn,
                                            float c_phi0, float2& o_r, float2& o_g, float2& o_b, float2& o_v, float2& c_zs)
{
    const float* s_nx = s;
    const float* s_ny = s + PL;
    const float* s_nz = s + 2 * PL;
    const float* s_zs = s + 3 * PL;
    const float* s_r  = s + 4 * PL;
    const float* s_g  = s + 5 * PL;
    const float* s_b  = s + 6 * PL;
    const float* s_va = s + 7 * PL;
    const float* s_lu = s + 8 * PL;
    const float2 cnx = ldp(s_nx, ci, true), cny = ldp(s_ny, ci, true), cnz = ldp(s_nz, ci, true), czs = ldp(s_zs, ci, true);
    const float2 ccr = ldp(s_r, ci, true), ccg = ldp(s_g, ci, true), ccb = ldp(s_b, ci, true), cva = ldp(s_va, ci, true), clu = ldp(s_lu, ci, true);
    c_zs = czs;
    // compute_variance_center for both pixels (:65-88): columns ci-1 .. ci+2, rows -1..+1 at unit spacing; weights {1/4,1/8,1/16}
    float2 vbar;
    {
        const float  a0 = v_up[-1], d0 = v_up[2];
        const float2 m0 = *reinterpret_cast<const float2*>(v_up);
        const float  a1 = s_va[ci - 1], d1 = s_va[ci + 2];
        const float  a2 = v_dn[-1], d2 = v_dn[2];
        const float2 m2 = *reinterpret_cast<const float2*>(v_dn);
        vbar.x = 0.25f * cva.x + 0.125f * (a1 + cva.y + m0.x + m2.x) + 0.0625f * (a0 + m0.y + a2 + m2.y);
        vbar.y = 0.25f * cva.y + 0.125f * (cva.x + d1 + m0.y + m2.y) + 0.0625f * (m0.x + d0 + m2.x + d2);
    }
    const float2 cphi = make_float2(c_phi0 * rsqrtf(fmaxf(1e-10f + vbar.x, 1e-30f)), c_phi0 * rsqrtf(fmaxf(1e-10f + vbar.y, 1e-30f)));
    const float2 neg1 = make_float2(-1.0f, -1.0f), nl2e = make_float2(-1.44269504f, -1.44269504f);
    const float  LK1 = -0.5849625007f, LK2 = -1.1699250014f; // log2(2/3), log2(4/9): kernel weights folded into the exponent
    float2 sumw = make_float2(1.0f, 1.0f), ar = ccr, ag = ccg, ab = ccb, av = cva;
#pragma unroll
    for (int yy = -1; yy <= 1; yy++)
#pragma unroll
        for (int xx = -1; xx <= 1; xx++)
        {
            if (xx == 0 && yy == 0) continue;
            const float lk = (xx != 0 && yy != 0) ? LK2 : LK1;
            const int   si = ci + yy * rs + xx * cs;
            const bool  al = ALIGNED_X || xx == 0;
            const float2 snx = ldp(s_nx, si, al), sny = ldp(s_ny, si, al), snz = ldp(s_nz, si, al), szs = ldp(s_zs, si, al);
            const float2 sr = ldp(s_r, si, al), sg = ldp(s_g, si, al), sb = ldp(s_b, si, al), sv = ldp(s_va, si, al), sl = ldp(s_lu, si, al);
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
            float2 p = fmul2(nd, nd);
            p        = fmul2(p, p);
            p        = fmul2(p, p);
            p        = fmul2(p, p);
            p        = fmul2(p, p);
            const float2 wk = fmul2(e, p);
            sumw = fadd2(sumw, wk);
            ar   = ffma2(wk, sr, ar);
            ag   = ffma2(wk, sg, ag);
            ab   = ffma2(wk, sb, ab);
            av   = ffma2(fmul2(wk, wk), sv, av);
        }
    const float2 inv = make_float2(fast_rcp(sumw.x), fast_rcp(sumw.y));
    o_r = fmul2(ar, inv);
    o_g = fmul2(ag, inv);
    o_b = fmul2(ab, inv);
    o_v = fmul2(fmul2(av, inv), inv);
}

// per-pixel class of the reference's early-outs (:119-128): 0 = sky -> 0, 1 = mirror / DDGI-rough -> pass-through, 2 = filter
__device__ __forceinline__ int pixel_class(float depth, float roughness, int approx)
{
    if (depth == 1.0f) return 0;
    if (roughness < 0.05f || (approx == 1 && roughness > 0.75f)) return 1;
    return 2;
}

__device__ __forceinline__ void store_pair(uint2* __restrict__ out, size_t idx, bool has1, int k0, int k1, const float* __restrict__ s, int PL, int ci, float2 o_r, float2 o_g,
                                           float2 o_b, float2 o_v)
{
    const float2 ccr = ldp(s + 4 * PL, ci, true), ccg = ldp(s + 5 * PL, ci, true), ccb = ldp(s + 6 * PL, ci, true), cva = ldp(s + 7 * PL, ci, true);
    uint2 r0, r1;
    if (k0 == 0) r0 = make_uint2(0u, 0u);
    else if (k0 == 1) r0 = make_uint2(f2_to_h2(ccr.x, ccg.x), f2_to_h2(ccb.x, cva.x));
    else r0 = make_uint2(f2_to_h2(o_r.x, o_g.x), f2_to_h2(o_b.x, o_v.x));
    if (k1 == 0) r1 = make_uint2(0u, 0u);
    else if (k1 == 1) r1 = make_uint2(f2_to_h2(ccr.y, ccg.y), f2_to_h2(ccb.y, cva.y));
    else r1 = make_uint2(f2_to_h2(o_r.y, o_g.y), f2_to_h2(o_b.y, o_v.y));
    if (has1) *reinterpret_cast<uint4*>(out + idx) = make_uint4(r0.x, r0.y, r1.x, r1.y); // idx even (W even is required by the launcher)
    else out[idx] = r0;
}

// Dense tile: 64x16 pixels + STEP halo.  Registers are tuned for 4 resident CTAs per SM: they hide the staging latency.
template <int STEP>
__global__ void __launch_bounds__(256, 4) k_refl_atrous_v2(GBufLevelDev g, const uint2* __restrict__ in, const uint8_t* __restrict__ tile_flags, R2Params P, uint2* __restrict__ out)
{
    extern __shared__ float smem_f[];
    constexpr int PADL = STEP + (STEP & 1);            // even left pad => even region column for even image column
    constexpr int RW   = (TWR + PADL + STEP + 1) & ~1; // even row pitch keeps LDS.64 alignment on every row
    constexpr int RH   = THR + 2 * STEP;
    constexpr int PL   = RW * RH;
    __shared__ uint32_t s_tf;
    const int W = P.W, H = P.H;
    const int x0 = blockIdx.x * TWR, y0 = P.row0 + blockIdx.y * THR;
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
    const int lx2 = threadIdx.x & 31, lyb = threadIdx.x >> 5; // 32 pixel pairs x 8 rows, 2 rows per thread
    const int x = x0 + 2 * lx2;
    if (tf == 0)
    { // every tile of this CTA is a copy tile: out = in, nothing staged
#pragma unroll
        for (int k = 0; k < THR / 8; k++)
        {
            const int y = y0 + lyb + 8 * k;
            if (x >= W || y >= H || y >= P.row1) continue;
            const size_t idx = (size_t)y * W + x;
            if (x + 1 < W) *reinterpret_cast<uint4*>(out + idx) = __ldg(reinterpret_cast<const uint4*>(in + idx));
            else out[idx] = __ldg(in + idx);
        }
        return;
    }
    for (int i = threadIdx.x; i < (RW / 2) * RH; i += 256)
    {
        const int rx = 2 * (i % (RW / 2)), ry = i / (RW / 2);
        stage_pair9(g, in, P.c_sigma, x0 - PADL + rx, y0 - STEP + ry, W, H, ry * RW + rx, smem_f, PL);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < THR / 8; k++)
    {
        const int ly = lyb + 8 * k, y = y0 + ly;
        if (x >= W || y >= H || y >= P.row1) continue;
        const size_t idx  = (size_t)y * W + x;
        const bool   has1 = x + 1 < W;
        const int    ci   = (ly + STEP) * RW + 2 * lx2 + PADL;
        int          k0 = 1, k1 = 1; // copy tile: pass-through
        if ((tf >> ((ly >> 3) * 8 + (lx2 >> 2))) & 1u)
        {
            const float2 d  = has1 ? __ldg(reinterpret_cast<const float2*>(g.depth + idx)) : make_float2(__ldg(g.depth + idx), 1.0f);
            const float  r0 = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + idx))).x;
            const float  r1 = has1 ? h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + idx + 1))).x : 0.0f;
            k0 = pixel_class(d.x, r0, P.approx);
            k1 = has1 ? pixel_class(d.y, r1, P.approx) : 0;
        }
        float2 o_r = make_float2(0.f, 0.f), o_g = o_r, o_b = o_r, o_v = o_r, czs;
        if (k0 == 2 || k1 == 2)
        {
            const float* s_va = smem_f + 7 * PL;
            filter_pair<(STEP & 1) == 0>(smem_f, PL, ci, STEP * RW, STEP, s_va + ci - RW, s_va + ci + RW, P.c_phi0, o_r, o_g, o_b, o_v, czs);
        }
        store_pair(out, idx, has1, k0, k1, smem_f, PL, ci, o_r, o_g, o_b, o_v);
    }
}

// Row-interleaved tile for the wide steps (see svgf_atrous_v3.cu::k_atrous_v3s): a CTA filters the 16 rows of one residue class
// of the row index modulo STEP, so it stages 18 rows instead of 16 + 2 * STEP; the variance of the rows directly above / below
// each filtered row (unit spacing, compute_variance_center) goes into two single-plane side buffers.
template <int STEP>
__global__ void __launch_bounds__(256) k_refl_atrous_v2s(GBufLevelDev g, const uint2* __restrict__ in, const uint8_t* __restrict__ tile_flags, R2Params P, uint2* __restrict__ out)
{
    extern __shared__ float smem_f[];
    constexpr int PADL  = STEP; // STEP is even here
    constexpr int RW    = TWR + 2 * STEP;
    constexpr int RH    = THR + 2;
    constexpr int PL    = RW * RH;
    constexpr int TROWS = (THR * STEP) / 8; // 8-row tile rows spanned by the CTA's 16 * STEP image rows
    float* s_vadj = smem_f + NPL * PL;      // [2][THR][RW]: variance of rows y-1 (0) and y+1 (1)
    __shared__ uint8_t s_tfl[TROWS][8];
    __shared__ int     s_any;
    const int W = P.W, H = P.H;
    const int x0 = blockIdx.x * TWR;
    const int blk = blockIdx.y / STEP, phase = blockIdx.y - blk * STEP;
    const int Y0 = P.row0 + blk * (THR * STEP); // multiple of 8 (row0 is)
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
    const int lx2 = threadIdx.x & 31, lyb = threadIdx.x >> 5;
    const int x = x0 + 2 * lx2;
    if (!s_any)
    {
#pragma unroll
        for (int k = 0; k < THR / 8; k++)
        {
            const int y = Y0 + phase + STEP * (lyb + 8 * k);
            if (x >= W || y >= H || y >= P.row1) continue;
            const size_t idx = (size_t)y * W + x;
            if (x + 1 < W) *reinterpret_cast<uint4*>(out + idx) = __ldg(reinterpret_cast<const uint4*>(in + idx));
            else out[idx] = __ldg(in + idx);
        }
        return;
    }
    for (int i = threadIdx.x; i < (RW / 2) * RH; i += 256)
    {
        const int rx = 2 * (i % (RW / 2)), ry = i / (RW / 2);
        stage_pair9(g, in, P.c_sigma, x0 - PADL + rx, Y0 + phase + STEP * (ry - 1), W, H, ry * RW + rx, smem_f, PL);
    }
    constexpr int VP = TWR / 2 + 2; // texel pairs covering columns x0-2 .. x0+TWR+1
    for (int i = threadIdx.x; i < 2 * THR * VP; i += 256)
    {
        const int a = i / (THR * VP), r = i - a * (THR * VP), j = r / VP, c = 2 * (r - j * VP);
        const int px = x0 - 2 + c, py = Y0 + phase + STEP * j + (a ? 1 : -1);
        float2    va = make_float2(0.0f, 0.0f);
        if (px >= 0 && py >= 0 && px < W && py < H)
        {
            const uint4 w = __ldg(reinterpret_cast<const uint4*>(in + (size_t)py * W + px));
            va = make_float2(h2_to_f2(w.y).y, h2_to_f2(w.w).y);
        }
        *reinterpret_cast<float2*>(s_vadj + (a * THR + j) * RW + PADL - 2 + c) = va;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < THR / 8; k++)
    {
        const int ly = lyb + 8 * k, y = Y0 + phase + STEP * ly;
        if (x >= W || y >= H || y >= P.row1) continue;
        const size_t idx  = (size_t)y * W + x;
        const bool   has1 = x + 1 < W;
        const int    ci   = (ly + 1) * RW + 2 * lx2 + PADL;
        int          k0 = 1, k1 = 1;
        if (s_tfl[(phase + STEP * ly) >> 3][lx2 >> 2])
        {
            const float2 d  = has1 ? __ldg(reinterpret_cast<const float2*>(g.depth + idx)) : make_float2(__ldg(g.depth + idx), 1.0f);
            const float  r0 = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + idx))).x;
            const float  r1 = has1 ? h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + idx + 1))).x : 0.0f;
            k0 = pixel_class(d.x, r0, P.approx);
            k1 = has1 ? pixel_class(d.y, r1, P.approx) : 0;
        }
        float2 o_r = make_float2(0.f, 0.f), o_g = o_r, o_b = o_r, o_v = o_r, czs;
        if (k0 == 2 || k1 == 2)
            filter_pair<true>(smem_f, PL, ci, RW, STEP, s_vadj + (0 * THR + ly) * RW + 2 * lx2 + PADL, s_vadj + (1 * THR + ly) * RW + 2 * lx2 + PADL, P.c_phi0, o_r, o_g, o_b,
                              o_v, czs);
        store_pair(out, idx, has1, k0, k1, smem_f, PL, ci, o_r, o_g, o_b, o_v);
    }
}

template <int STEP>
void launch_r2(const GBufLevelDev& g, const uint2* in, const uint8_t* tf, const R2Params& P, uint2* out, cudaStream_t st)
{
    constexpr int PADL = STEP + (STEP & 1);
    constexpr int RW   = (TWR + PADL + STEP + 1) & ~1;
    constexpr int RH   = THR + 2 * STEP;
    const size_t  smem = (size_t)RW * RH * NPL * sizeof(float);
    static bool   configured[64] = {};
    if (hr_once_per_device(configured)) cudaFuncSetAttribute(k_refl_atrous_v2<STEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid((P.W + TWR - 1) / TWR, (P.row1 - P.row0 + THR - 1) / THR);
    k_refl_atrous_v2<STEP><<<grid, 256, smem, st>>>(g, in, tf, P, out);
}

template <int STEP>
void launch_r2s(const GBufLevelDev& g, const uint2* in, const uint8_t* tf, const R2Params& P, uint2* out, cudaStream_t st)
{
    constexpr int RW = TWR + 2 * STEP, RH = THR + 2;
    const size_t  smem = ((size_t)RW * RH * NPL + (size_t)2 * THR * RW) * sizeof(float);
    static bool   configured[64] = {};
    if (hr_once_per_device(configured)) cudaFuncSetAttribute(k_refl_atrous_v2s<STEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int rows = P.row1 - P.row0, blocks = (rows + THR * STEP - 1) / (THR * STEP);
    dim3      grid((P.W + TWR - 1) / TWR, blocks * STEP);
    k_refl_atrous_v2s<STEP><<<grid, 256, smem, st>>>(g, in, tf, P, out);
}


// ---------------------------------------------------------------------------------------------------------------------------
// TMA-staged, persistent form of the dense-tile kernel at step 1.
//
// k_refl_atrous_v2 issues far fewer instructions per iteration than the scalar kernel but stalls on long_scoreboard: every CTA
// first waits for its own staging loads from DRAM (the images are larger than L2), and 2-4 resident CTAs per SM are not enough
// to cover that.  Here the loads leave the
// instruction stream: CTAs are persistent, tiles come from an atomic counter, and the three raw images of the NEXT tile (GB2, GB3,
// input colour: tile + halo boxes of 8-byte texels) are fetched by the TMA engine (cp.async.bulk.tensor.2d, one elected
// thread, completion on an mbarrier, out-of-image texels zero-filled by the hardware) while the CTA filters the CURRENT tile.
// Per tile: wait for the mbarrier -> decode raw texel pairs from shared memory into the nine fp32 planes -> barrier -> issue
// the TMA loads of the next active tile into the (now free) raw buffers -> filter from the planes -> barrier.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, uint64_t* bar, int x, int y)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)), "l"(tm),
                 "r"(smem_u32(bar)), "r"(x), "r"(y)
                 : "memory");
}

// the region of k_refl_atrous_v2<1>
struct TmaGeom {
    static constexpr int STEP = 1;
    static constexpr int PADL = STEP + (STEP & 1);
    static constexpr int RW   = (TWR + PADL + STEP + 1) & ~1;
    static constexpr int RH   = THR + 2 * STEP;
    static constexpr int PL   = RW * RH;
    static constexpr int RAWB = (PL * 8 + 127) & ~127; // bytes of one raw image box, padded to the 128-byte TMA destination alignment
    static constexpr int SMEM = 3 * RAWB + NPL * PL * 4 + TWR * THR; // + one class byte per pixel of the tile
};

__global__ void __launch_bounds__(256, 3)
k_refl_atrous_tma(const __grid_constant__ CUtensorMap tm_gb2, const __grid_constant__ CUtensorMap tm_gb3, const __grid_constant__ CUtensorMap tm_in, GBufLevelDev g,
                  const uint2* __restrict__ in, const uint8_t* __restrict__ tile_flags, R2Params P, uint2* __restrict__ out, int tiles_x, int n_tiles,
                  unsigned int* __restrict__ counter)
{
    using G = TmaGeom;
    constexpr int STEP = G::STEP, PADL = G::PADL, RW = G::RW, RH = G::RH, PL = G::PL;
    extern __shared__ __align__(128) unsigned char smem_b[];
    unsigned char* raw0 = smem_b;
    float*         planes = reinterpret_cast<float*>(smem_b + 3 * G::RAWB);
    unsigned char* s_cls  = smem_b + 3 * G::RAWB + NPL * PL * 4; // per pixel of the tile: 0 sky, 1 pass-through, 2 filter (pixel_class)
    __shared__ __align__(8) uint64_t s_mbar;
    __shared__ int      s_tile[2];
    __shared__ uint32_t s_flag[2];
    const int W = P.W, H = P.H;
    const int TWt = (W + 7) >> 3, THt = (H + 7) >> 3;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int lx2 = lane, lyb = warp; // 32 pixel pairs x 8 rows, 2 rows per thread

    // warp 0: take the next tile from the counter and read its 8 x 2 tile flags
    auto fetch_tile = [&](int slot) {
        int t = 0;
        if (lane == 0) t = (int)atomicAdd(counter, 1u);
        t = __shfl_sync(0xFFFFFFFFu, t, 0);
        bool f = false;
        if (t < n_tiles && lane < 16)
        {
            const int x0 = (t % tiles_x) * TWR, y0 = P.row0 + (t / tiles_x) * THR;
            const int tx = (x0 >> 3) + (lane & 7), ty = (y0 >> 3) + (lane >> 3);
            f = tx < TWt && ty < THt && tile_flags[(size_t)ty * TWt + tx] != 0;
        }
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, f);
        if (lane == 0) { s_tile[slot] = t < n_tiles ? t : -1; s_flag[slot] = b; }
    };
    auto issue_tma = [&](int t) { // one thread
        const int x0 = (t % tiles_x) * TWR, y0 = P.row0 + (t / tiles_x) * THR;
        mbar_arrive_expect_tx(&s_mbar, 3u * (uint32_t)(PL * 8));
        tma_load_2d(raw0, &tm_gb2, &s_mbar, x0 - PADL, y0 - STEP);
        tma_load_2d(raw0 + G::RAWB, &tm_gb3, &s_mbar, x0 - PADL, y0 - STEP);
        tma_load_2d(raw0 + 2 * G::RAWB, &tm_in, &s_mbar, x0 - PADL, y0 - STEP);
    };

    if (threadIdx.x == 0) { mbar_init(&s_mbar, 1); fence_mbar_init(); }
    if (warp == 0) fetch_tile(0);
    __syncthreads();
    if (threadIdx.x == 0 && s_tile[0] >= 0 && s_flag[0] != 0u) issue_tma(s_tile[0]);
    uint32_t phase = 0;
    int      slot  = 0;
    for (;;)
    {
        const int      t  = s_tile[slot];
        const uint32_t tf = s_flag[slot];
        if (t < 0) break;
        if (warp == 0) fetch_tile(slot ^ 1); // overlaps the wait below
        const int x0 = (t % tiles_x) * TWR, y0 = P.row0 + (t / tiles_x) * THR;
        if (tf != 0u)
        {
            {
                const long long t_start = clock64();
                while (!mbar_try_wait(&s_mbar, phase))
                    if (clock64() - t_start > 4000000000ll) __trap(); // ~2 s: a lost TMA completion must fail loudly, never hang the GPU
            }
            phase ^= 1u;
            // decode the raw boxes (two texels per step) into the nine planes; cells outside the image get a zero normal (weight 0)
            const uint4* r2 = reinterpret_cast<const uint4*>(raw0);
            const uint4* r3 = reinterpret_cast<const uint4*>(raw0 + G::RAWB);
            const uint4* rc = reinterpret_cast<const uint4*>(raw0 + 2 * G::RAWB);
            for (int i = threadIdx.x; i < (RW / 2) * RH; i += 256)
            {
                const int rx = 2 * (i % (RW / 2)), ry = i / (RW / 2);
                const int px = x0 - PADL + rx, py = y0 - STEP + ry;
                float2 nx = make_float2(0.0f, 0.0f), ny = nx, nz = nx, zs = nx, cr = nx, cg = nx, cb = nx, va = nx, lu = make_float2(0.0001f, 0.0001f);
                float2 rough = make_float2(0.0f, 0.0f);
                if (px >= 0 && py >= 0 && px < W && py < H)
                {
                    const uint4  a = r2[i], b = r3[i], c = rc[i];
                    rough = make_float2(h2_to_f2(b.x).x, h2_to_f2(b.z).x);
                    const float2 e0 = h2_to_f2(a.x), e1 = h2_to_f2(a.z);
                    const float3 n0 = octohedral_to_direction(e0.x, e0.y), n1 = octohedral_to_direction(e1.x, e1.y);
                    const float2 c0 = h2_to_f2(c.x), c1 = h2_to_f2(c.y), c2 = h2_to_f2(c.z), c3 = h2_to_f2(c.w);
                    nx = make_float2(n0.x, n1.x); ny = make_float2(n0.y, n1.y); nz = make_float2(n0.z, n1.z);
                    zs = make_float2(h2_to_f2(b.y).y * P.c_sigma, h2_to_f2(b.w).y * P.c_sigma);
                    cr = make_float2(c0.x, c2.x); cg = make_float2(c0.y, c2.y); cb = make_float2(c1.x, c3.x); va = make_float2(c1.y, c3.y);
                    lu = make_float2(lum3(c0.x, c0.y, c1.x), lum3(c2.x, c2.y, c3.x));
                }
                float* p = planes + ry * RW + rx;
                *reinterpret_cast<float2*>(p) = nx; p += PL;
                *reinterpret_cast<float2*>(p) = ny; p += PL;
                *reinterpret_cast<float2*>(p) = nz; p += PL;
                *reinterpret_cast<float2*>(p) = zs; p += PL;
                *reinterpret_cast<float2*>(p) = cr; p += PL;
                *reinterpret_cast<float2*>(p) = cg; p += PL;
                *reinterpret_cast<float2*>(p) = cb; p += PL;
                *reinterpret_cast<float2*>(p) = va; p += PL;
                *reinterpret_cast<float2*>(p) = lu;
                const int tx = rx - PADL, ty = ry - STEP;
                if (tx >= 0 && tx < TWR && ty >= 0 && ty < THR)
                { // the reference's early-outs (:119-128).  Sky = linear z < 0 (GB3.w = -1): identical to its depth == 1 test whenever the
                  // sky pixels carry the G-buffer clear values (depth 1 and GB3 = (0,0,0,-1) are written together, g_buffer.cpp:72-96)
                    const int c0 = zs.x < 0.0f ? 0 : ((rough.x < 0.05f || (P.approx == 1 && rough.x > 0.75f)) ? 1 : 2);
                    const int c1 = zs.y < 0.0f ? 0 : ((rough.y < 0.05f || (P.approx == 1 && rough.y > 0.75f)) ? 1 : 2);
                    *reinterpret_cast<uchar2*>(s_cls + ty * TWR + tx) = make_uchar2((unsigned char)c0, (unsigned char)c1);
                }
            }
        }
        __syncthreads(); // planes complete, raw boxes free, next tile's index / flags visible
        if (threadIdx.x == 0)
        {
            const int tn = s_tile[slot ^ 1];
            if (tn >= 0 && s_flag[slot ^ 1] != 0u) issue_tma(tn); // flies while this tile is filtered
        }
        const int x = x0 + 2 * lx2;
#pragma unroll
        for (int k = 0; k < THR / 8; k++)
        {
            const int ly = lyb + 8 * k, y = y0 + ly;
            if (x >= W || y >= H || y >= P.row1) continue;
            const size_t idx = (size_t)y * W + x;
            if (tf == 0u)
            { // copy tile (reflections_denoise_copy_tiles.comp:35-38)
                *reinterpret_cast<uint4*>(out + idx) = __ldg(reinterpret_cast<const uint4*>(in + idx));
                continue;
            }
            const int ci = (ly + STEP) * RW + 2 * lx2 + PADL;
            int       k0 = 1, k1 = 1;
            if ((tf >> ((ly >> 3) * 8 + (lx2 >> 2))) & 1u)
            {
                const uchar2 c = *reinterpret_cast<const uchar2*>(s_cls + ly * TWR + 2 * lx2);
                k0 = c.x;
                k1 = c.y;
            }
            float2 o_r = make_float2(0.f, 0.f), o_g = o_r, o_b = o_r, o_v = o_r, czs;
            if (k0 == 2 || k1 == 2)
            {
                const float* s_va = planes + 7 * PL;
                filter_pair<(STEP & 1) == 0>(planes, PL, ci, STEP * RW, STEP, s_va + ci - RW, s_va + ci + RW, P.c_phi0, o_r, o_g, o_b, o_v, czs);
            }
            store_pair(out, idx, true, k0, k1, planes, PL, ci, o_r, o_g, o_b, o_v);
        }
        __syncthreads(); // planes may be overwritten by the next tile's decode
        slot ^= 1;
    }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled tma_encoder()
{
    static PFN_encodeTiled fn     = nullptr;
    static bool            looked = false;
    if (!looked)
    {
        looked = true;
        void*                            p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (PFN_encodeTiled)p;
    }
    return fn;
}

// tensor map of a W x H image of 8-byte texels with a (bw x bh) box; cached per (pointer, size, box)
struct TmCacheEntry { const void* ptr; int W, H, bw, bh; CUtensorMap tm; };
bool tensor_map_2d(const void* ptr, int W, int H, int bw, int bh, CUtensorMap* out)
{
    static std::vector<TmCacheEntry> cache;
    for (const auto& e : cache)
        if (e.ptr == ptr && e.W == W && e.H == H && e.bw == bw && e.bh == bh) { *out = e.tm; return true; }
    PFN_encodeTiled enc = tma_encoder();
    if (!enc) return false;
    TmCacheEntry e { ptr, W, H, bw, bh, {} };
    const cuuint64_t dims[2] = { (cuuint64_t)W, (cuuint64_t)H }, strides[1] = { (cuuint64_t)W * 8 };
    const cuuint32_t box[2] = { (cuuint32_t)bw, (cuuint32_t)bh }, estr[2] = { 1, 1 };
    if (enc(&e.tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return false;
    if (cache.size() > 256) cache.clear();
    cache.push_back(e);
    *out = e.tm;
    return true;
}

// counter: a word owned by the calling pass: passes of different contexts may run concurrently on one device (emulated ranks on
// streams), so the tile counter cannot be a per-device static
bool launch_r2_tma(const GBufLevelDev& g, const uint2* in, const uint8_t* tf, const R2Params& P, uint2* out, unsigned int* counter, cudaStream_t st)
{
    if (!counter) return false;
    using G = TmaGeom;
    if ((((size_t)g.W * 8) & 15) != 0 || ((uintptr_t)g.gb2 & 15) || ((uintptr_t)g.gb3 & 15) || ((uintptr_t)in & 15)) return false;
    CUtensorMap t2, t3, ti;
    if (!tensor_map_2d(g.gb2, g.W, g.H, G::RW, G::RH, &t2) || !tensor_map_2d(g.gb3, g.W, g.H, G::RW, G::RH, &t3) || !tensor_map_2d(in, g.W, g.H, G::RW, G::RH, &ti)) return false;
    static int ctas[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    static bool configured[64] = {};
    if (hr_once_per_device(configured))
    {
        cudaFuncSetAttribute(k_refl_atrous_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM);
        int sms = 132, per_sm = 1;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_refl_atrous_tma, 256, G::SMEM);
        ctas[dev] = sms * (per_sm > 0 ? per_sm : 1);
    }
    const int tiles_x = (P.W + TWR - 1) / TWR, tiles_y = (P.row1 - P.row0 + THR - 1) / THR, n_tiles = tiles_x * tiles_y;
    cudaMemsetAsync(counter, 0, sizeof(unsigned int), st);
    const int grid = ctas[dev] < n_tiles ? ctas[dev] : n_tiles;
    k_refl_atrous_tma<<<grid, 256, G::SMEM, st>>>(t2, t3, ti, g, in, tf, P, out, tiles_x, n_tiles, counter);
    return true;
}

} // namespace

// hr_debug_set key 6: 0 = scalar kernel (svgf_reflections.cu), 2 = pixel pairs with plain staging, row-interleaved tiles for
// steps >= 8, 3 (default) = 2 + the TMA-staged persistent kernel for step 1.  2 is also what step 1 runs when the TMA set-up
// fails, and the bit-exact reference of the TMA kernel.  TMA staging wins at step 1 only (74 KB, 3 CTAs per SM; at step 2 its
// raw boxes + planes allow only 2 CTAs per SM): on an H100 SXM 80 GB, 700 W power limit, step 1 takes 113 us with TMA and
// 118 us with plain staging (DESIGN.md §8).
int g_hr_refl_atrous_impl = 3;

// returns false when this variant does not support the configuration (the caller falls back to the scalar kernel)
bool launch_reflections_atrous_v2(const GBufLevelDev& g, const void* in, const uint8_t* tile_flags, int radius, int step, float phi_color, float phi_normal,
                                  float sigma_depth, int approximate_with_ddgi, void* out, int row0, int row1, unsigned int* counters, cudaStream_t st)
{
    if (g_hr_refl_atrous_impl == 0 || radius != 1 || phi_normal != 32.0f || (g.W & 1) || row0 % 8 != 0 || !(step == 1 || step == 2 || step == 4 || step == 8 || step == 16))
        return false;
    R2Params P { g.W, g.H, 1.44269504f / sigma_depth, -1.44269504f / phi_color, approximate_with_ddgi, row0, row1 };
    const uint2* i2 = (const uint2*)in;
    uint2*       o2 = (uint2*)out;
    switch (step)
    {
        case 1: if (!(g_hr_refl_atrous_impl == 3 && launch_r2_tma(g, i2, tile_flags, P, o2, counters, st))) launch_r2<1>(g, i2, tile_flags, P, o2, st); break;
        case 2: launch_r2<2>(g, i2, tile_flags, P, o2, st); break;
        case 4: launch_r2<4>(g, i2, tile_flags, P, o2, st); break;
        case 8: launch_r2s<8>(g, i2, tile_flags, P, o2, st); break;
        default: launch_r2s<16>(g, i2, tile_flags, P, o2, st); break;
    }
    return true;
}
