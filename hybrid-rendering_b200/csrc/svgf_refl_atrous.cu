// svgf_refl_atrous.cu — reflections a-trous (K15 + K16, reflections_denoise_atrous.comp:94-181).
//
// This is the roofline kernel of BASELINE config 3 (4K full-res reflections: 36 algorithmic B/px/iteration, SURVEY.md §8d).
// The pixel-pair kernels (atrous_pairs.cuh) stage nine planes: nx, ny, nz, z * log2e / sigma, r, g, b, variance, luminance (the
// sample luminance is computed once per staged texel instead of once per tap).  k_refl_atrous is the scalar kernel: the fallback
// for odd widths and phi_normal != 32, and the reference of the pixel pairs.
// Tile classification (K13/K15): tiles whose flag is 0 are copied (reflections_denoise_copy_tiles.comp:35-38).
#include "atrous_pairs.cuh"
#include <cuda.h> // CUtensorMap (driver types only; cuTensorMapEncodeTiled is fetched with cudaGetDriverEntryPoint)
#include <vector>

namespace {

using namespace gf;

struct R2Params {
    int   W, H;
    float c_sigma; // log2(e) / sigma_depth
    float c_phi0;  // -log2(e) / phi_color
    int   approx;  // approximate_with_ddgi
    int   row0, row1;
};

// per-pixel class of the reference's early-outs (:119-128): 0 = sky -> 0, 1 = mirror / DDGI-rough -> pass-through, 2 = filter
__device__ __forceinline__ int pixel_class(float depth, float roughness, int approx)
{
    if (depth == 1.0f) return 0;
    if (roughness < 0.05f || (approx == 1 && roughness > 0.75f)) return 1;
    return 2;
}

__device__ __forceinline__ void store_pair(uint2* __restrict__ out, size_t idx, bool has1, int k0, int k1, const float* __restrict__ s, int PL, int ci, const PairSum<3>& f)
{
    const float2 ccr = ld_pair(s + 4 * PL, ci, true), ccg = ld_pair(s + 5 * PL, ci, true), ccb = ld_pair(s + 6 * PL, ci, true), cva = ld_pair(s + 7 * PL, ci, true);
    uint2 r0, r1;
    if (k0 == 0) r0 = make_uint2(0u, 0u);
    else if (k0 == 1) r0 = make_uint2(f2_to_h2(ccr.x, ccg.x), f2_to_h2(ccb.x, cva.x));
    else r0 = make_uint2(f2_to_h2(f.c[0].x, f.c[1].x), f2_to_h2(f.c[2].x, f.v.x));
    if (k1 == 0) r1 = make_uint2(0u, 0u);
    else if (k1 == 1) r1 = make_uint2(f2_to_h2(ccr.y, ccg.y), f2_to_h2(ccb.y, cva.y));
    else r1 = make_uint2(f2_to_h2(f.c[0].y, f.c[1].y), f2_to_h2(f.c[2].y, f.v.y));
    if (has1) *reinterpret_cast<uint4*>(out + idx) = make_uint4(r0.x, r0.y, r1.x, r1.y); // idx even (W even is required by the launcher)
    else out[idx] = r0;
}

struct ReflectionsPass {
    using In = uint2; using Out = uint2; using Params = R2Params;
    static constexpr int  NPL = 9, NC = 3;
    static constexpr bool COPY_EMPTY_CTA = true; // a CTA whose tiles are all unflagged copies in -> out

    // Stage the texel pair (px, px+1) of row py (px even) at region index ri (even).
    static __device__ __forceinline__ void stage(const GBufLevelDev& g, const uint2* __restrict__ in, float c_sigma, int px, int py, int W, int H, int ri, float* s, int PL)
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
            lu = make_float2(luminance(c0.x, c0.y, c1.x), luminance(c2.x, c2.y, c3.x));
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

    static __device__ __forceinline__ float2 side_var(const uint2* __restrict__ in, size_t pi)
    {
        const uint4 w = __ldg(reinterpret_cast<const uint4*>(in + pi));
        return make_float2(h2_to_f2(w.y).y, h2_to_f2(w.w).y);
    }

    static __device__ __forceinline__ void copy(const uint2* __restrict__ in, uint2* __restrict__ out, size_t idx, bool has1)
    {
        if (has1) *reinterpret_cast<uint4*>(out + idx) = __ldg(reinterpret_cast<const uint4*>(in + idx));
        else out[idx] = __ldg(in + idx);
    }

    template <bool ALIGNED_X>
    static __device__ __forceinline__ void filter_store(const GBufLevelDev& g, const R2Params& P, const PairTaps& t, uint2* __restrict__ out, size_t idx, bool has1, bool flagged)
    {
        int k0 = 1, k1 = 1; // copy tile: pass-through
        if (flagged)
        {
            const float2 d  = has1 ? __ldg(reinterpret_cast<const float2*>(g.depth + idx)) : make_float2(__ldg(g.depth + idx), 1.0f);
            const float  r0 = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + idx))).x;
            const float  r1 = has1 ? h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + idx + 1))).x : 0.0f;
            k0 = pixel_class(d.x, r0, P.approx);
            k1 = has1 ? pixel_class(d.y, r1, P.approx) : 0;
        }
        PairSum<3> f = {};
        if (k0 == 2 || k1 == 2) f = filter_pair<3, 8, ALIGNED_X>(t, P.c_phi0); // plane 8: luminance
        store_pair(out, idx, has1, k0, k1, t.s, t.PL, t.ci, f);
    }
};

// Dense tile.  Registers are tuned for 4 resident CTAs per SM: they hide the staging latency.
template <int STEP>
__global__ void __launch_bounds__(256, 4) k_refl_atrous_v2(GBufLevelDev g, const uint2* __restrict__ in, const uint8_t* __restrict__ tile_flags, R2Params P, uint2* __restrict__ out)
{
    atrous_dense<ReflectionsPass, STEP>(g, in, tile_flags, P, out);
}

template <int STEP>
__global__ void __launch_bounds__(256) k_refl_atrous_v2s(GBufLevelDev g, const uint2* __restrict__ in, const uint8_t* __restrict__ tile_flags, R2Params P, uint2* __restrict__ out)
{
    atrous_interleaved<ReflectionsPass, STEP>(g, in, tile_flags, P, out);
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

// the region of k_refl_atrous_v2<1>; shared memory: three raw image boxes of it, the planes, one class byte per pixel of the tile
struct TmaGeom : DenseTile<1, ReflectionsPass::NPL> {
    static constexpr int RAWB  = (PL * 8 + 127) & ~127; // bytes of one raw image box, padded to the 128-byte TMA destination alignment
    static constexpr int BYTES = 3 * RAWB + SMEM + PAIR_TILE_W * PAIR_TILE_H;
};

__global__ void __launch_bounds__(256, 3)
k_refl_atrous_tma(const __grid_constant__ CUtensorMap tm_gb2, const __grid_constant__ CUtensorMap tm_gb3, const __grid_constant__ CUtensorMap tm_in, GBufLevelDev g,
                  const uint2* __restrict__ in, const uint8_t* __restrict__ tile_flags, R2Params P, uint2* __restrict__ out, int tiles_x, int n_tiles,
                  unsigned int* __restrict__ counter)
{
    using G = TmaGeom;
    constexpr int STEP = 1, PADL = G::PADL, RW = G::RW, RH = G::RH, PL = G::PL;
    extern __shared__ __align__(128) unsigned char smem_b[];
    unsigned char* raw0 = smem_b;
    float*         planes = reinterpret_cast<float*>(smem_b + 3 * G::RAWB);
    unsigned char* s_cls  = smem_b + 3 * G::RAWB + G::SMEM; // per pixel of the tile: 0 sky, 1 pass-through, 2 filter (pixel_class)
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
            const int x0 = (t % tiles_x) * PAIR_TILE_W, y0 = P.row0 + (t / tiles_x) * PAIR_TILE_H;
            const int tx = (x0 >> 3) + (lane & 7), ty = (y0 >> 3) + (lane >> 3);
            f = tx < TWt && ty < THt && tile_flags[(size_t)ty * TWt + tx] != 0;
        }
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, f);
        if (lane == 0) { s_tile[slot] = t < n_tiles ? t : -1; s_flag[slot] = b; }
    };
    auto issue_tma = [&](int t) { // one thread
        const int x0 = (t % tiles_x) * PAIR_TILE_W, y0 = P.row0 + (t / tiles_x) * PAIR_TILE_H;
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
        const int x0 = (t % tiles_x) * PAIR_TILE_W, y0 = P.row0 + (t / tiles_x) * PAIR_TILE_H;
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
                    lu = make_float2(luminance(c0.x, c0.y, c1.x), luminance(c2.x, c2.y, c3.x));
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
                if (tx >= 0 && tx < PAIR_TILE_W && ty >= 0 && ty < PAIR_TILE_H)
                { // the reference's early-outs (:119-128).  Sky = linear z < 0 (GB3.w = -1): identical to its depth == 1 test whenever the
                  // sky pixels carry the G-buffer clear values (depth 1 and GB3 = (0,0,0,-1) are written together, g_buffer.cpp:72-96)
                    const int c0 = zs.x < 0.0f ? 0 : ((rough.x < 0.05f || (P.approx == 1 && rough.x > 0.75f)) ? 1 : 2);
                    const int c1 = zs.y < 0.0f ? 0 : ((rough.y < 0.05f || (P.approx == 1 && rough.y > 0.75f)) ? 1 : 2);
                    *reinterpret_cast<uchar2*>(s_cls + ty * PAIR_TILE_W + tx) = make_uchar2((unsigned char)c0, (unsigned char)c1);
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
        for (int k = 0; k < PAIR_TILE_H / 8; k++)
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
            if ((tf >> dense_flag_bit(lx2, ly)) & 1u)
            {
                const uchar2 c = *reinterpret_cast<const uchar2*>(s_cls + ly * PAIR_TILE_W + 2 * lx2);
                k0 = c.x;
                k1 = c.y;
            }
            PairSum<3> f = {};
            if (k0 == 2 || k1 == 2)
            {
                const float* s_va = planes + 7 * PL;
                f = filter_pair<3, 8, (STEP & 1) == 0>(PairTaps { planes, PL, ci, STEP * RW, STEP, s_va + ci - RW, s_va + ci + RW }, P.c_phi0);
            }
            store_pair(out, idx, true, k0, k1, planes, PL, ci, f);
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
        cudaFuncSetAttribute(k_refl_atrous_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, G::BYTES);
        int sms = 132, per_sm = 1;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_refl_atrous_tma, 256, G::BYTES);
        ctas[dev] = sms * (per_sm > 0 ? per_sm : 1);
    }
    const int tiles_x = (P.W + PAIR_TILE_W - 1) / PAIR_TILE_W, tiles_y = (P.row1 - P.row0 + PAIR_TILE_H - 1) / PAIR_TILE_H, n_tiles = tiles_x * tiles_y;
    cudaMemsetAsync(counter, 0, sizeof(unsigned int), st);
    const int grid = ctas[dev] < n_tiles ? ctas[dev] : n_tiles;
    k_refl_atrous_tma<<<grid, 256, G::BYTES, st>>>(t2, t3, ti, g, in, tf, P, out, tiles_x, n_tiles, counter);
    return true;
}

// ---- scalar kernel ----------------------------------------------------------------------------------------------------
struct ReflAtrousParams { int W, H, step, radius; float phi_color, phi_normal, sigma_depth; int approximate_with_ddgi, row0, row1; };

// K16: tile 32x16 + halo in smem: decoded normal + z (float4) and colour + variance (float4)
template <int STEP>
__global__ void __launch_bounds__(256) k_refl_atrous(GBufLevelDev g, const uint2* __restrict__ in, const uint8_t* __restrict__ tile_flags, ReflAtrousParams P,
                                                      uint2* __restrict__ out)
{
    extern __shared__ float4 smem4[];
    constexpr int TWD = 32, THT = 16, RW = TWD + 2 * STEP, RH = THT + 2 * STEP;
    float4*       s_nz = smem4;
    float4*       s_c  = smem4 + RW * RH;
    __shared__ uint32_t s_tf;
    const int W = P.W, H = P.H;
    const int x0 = blockIdx.x * TWD, y0 = P.row0 + blockIdx.y * THT;
    const int TW = (W + 7) >> 3, TH = (H + 7) >> 3;
    if (threadIdx.x < 32)
    {
        const int  tx = (x0 >> 3) + (threadIdx.x & 3), ty = (y0 >> 3) + (threadIdx.x >> 2);
        const bool f  = threadIdx.x < 8 && tx < TW && ty < TH && tile_flags[(size_t)ty * TW + tx] != 0;
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, f);
        if (threadIdx.x == 0) s_tf = b;
    }
    __syncthreads();
    const uint32_t tf = s_tf;
    for (int i = threadIdx.x; i < RW * RH; i += 256)
    {
        const int rx = i % RW, ry = i / RW, px = x0 - STEP + rx, py = y0 - STEP + ry;
        float4    nz = make_float4(0.0f, 0.0f, 0.0f, 0.0f), c = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (px >= 0 && py >= 0 && px < W && py < H)
        {
            const size_t pi = (size_t)py * W + px;
            const float2 e  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb2 + pi)));
            const float2 zz = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + pi) + 1));
            const float3 n  = octohedral_to_direction(e.x, e.y);
            nz = make_float4(n.x, n.y, n.z, zz.y);
            c  = h4_to_f4(__ldg(in + pi));
        }
        s_nz[i] = nz;
        s_c[i]  = c;
    }
    __syncthreads();
    const int   lx = threadIdx.x & 31, lyb = threadIdx.x >> 5;
    const float c_sigma = -1.44269504f / P.sigma_depth;
#pragma unroll
    for (int k = 0; k < THT / 8; k++)
    {
        const int ly = lyb + 8 * k, x = x0 + lx, y = y0 + ly;
        if (x >= W || y >= H || y >= P.row1) continue;
        const size_t idx = (size_t)y * W + x;
        const int    ci  = (ly + STEP) * RW + lx + STEP;
        const float4 cc  = s_c[ci];
        if (!((tf >> ((ly >> 3) * 4 + (lx >> 3))) & 1u)) { out[idx] = pack_h4(cc.x, cc.y, cc.z, cc.w); continue; } // copy tiles
        const float depth = __ldg(g.depth + idx);
        if (depth == 1.0f) { out[idx] = make_uint2(0u, 0u); continue; }
        const float roughness = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb3 + idx))).x;
        if (roughness < 0.05f || (P.approximate_with_ddgi == 1 && roughness > 0.75f)) { out[idx] = pack_h4(cc.x, cc.y, cc.z, cc.w); continue; }
        const float4 cn = s_nz[ci];
        const float  cl = luminance(cc.x, cc.y, cc.z);
        float var = 0.25f * cc.w + 0.125f * (s_c[ci - 1].w + s_c[ci + 1].w + s_c[ci - RW].w + s_c[ci + RW].w) +
                    0.0625f * (s_c[ci - RW - 1].w + s_c[ci - RW + 1].w + s_c[ci + RW - 1].w + s_c[ci + RW + 1].w);
        const float c_phi = -1.44269504f * rsqrtf(fmaxf(1e-10f + var, 1e-30f)) / P.phi_color;
        float       sum_w = 1.0f, s0 = cc.x, s1 = cc.y, s2 = cc.z, s3 = cc.w;
#pragma unroll
        for (int yy = -1; yy <= 1; yy++)
#pragma unroll
            for (int xx = -1; xx <= 1; xx++)
            {
                if (xx == 0 && yy == 0) continue;
                const float  kern = (xx == 0 ? 1.0f : 2.0f / 3.0f) * (yy == 0 ? 1.0f : 2.0f / 3.0f);
                const int    si   = ci + yy * STEP * RW + xx * STEP;
                const float4 sn = s_nz[si], s = s_c[si];
                const float  sl = luminance(s.x, s.y, s.z);
                const float  wZ = fast_exp2(fabsf(cn.w - sn.w) * c_sigma);
                const float  ea = fmaf(wZ, -1.44269504f, fabsf(cl - sl) * c_phi);
                const float  nd = cn.x * sn.x + cn.y * sn.y + cn.z * sn.z; // out-of-image cells have n = 0 => weight 0 (= `inside` test)
                const float  wk = fast_exp2(ea) * normal_weight(nd, P.phi_normal) * kern;
                sum_w += wk;
                s0 = fmaf(wk, s.x, s0); s1 = fmaf(wk, s.y, s1); s2 = fmaf(wk, s.z, s2);
                s3 = fmaf(wk * wk, s.w, s3);
            }
        const float inv = 1.0f / sum_w;
        out[idx] = pack_h4(s0 * inv, s1 * inv, s2 * inv, s3 * inv * inv);
    }
}

template <int STEP>
void launch_atrous_t(const GBufLevelDev& g, const uint2* in, const uint8_t* tf, const ReflAtrousParams& P, uint2* out, cudaStream_t st)
{
    constexpr int RW = 32 + 2 * STEP, RH = 16 + 2 * STEP;
    const size_t  smem = (size_t)RW * RH * 2 * sizeof(float4);
    static bool   configured[64] = {};
    if (hr_once_per_device(configured)) cudaFuncSetAttribute(k_refl_atrous<STEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid((P.W + 31) / 32, (P.row1 - P.row0 + 15) / 16);
    k_refl_atrous<STEP><<<grid, 256, smem, st>>>(g, in, tf, P, out);
}

template <int STEP>
using Dense = DenseTile<STEP, ReflectionsPass::NPL>;
template <int STEP>
using Interleaved = InterleavedTile<STEP, ReflectionsPass::NPL>;

} // namespace

// Key 6 = 2 is also what step 1 runs when the TMA set-up fails, and the bit-exact reference of the TMA kernel.  TMA staging wins at
// step 1 only (74 KB, 3 CTAs per SM; at step 2 its raw boxes + planes allow only 2 CTAs per SM): on an H100 SXM 80 GB, 700 W power
// limit, step 1 takes 113 us with TMA and 118 us with plain staging (DESIGN.md §8).
int g_hr_refl_atrous_impl = 3;

// -1: radius / step not supported
int launch_reflections_atrous(const GBufLevelDev& g, const void* in, const uint8_t* tile_flags, int radius, int step, float phi_color, float phi_normal,
                              float sigma_depth, int approximate_with_ddgi, void* out, int row0, int row1, unsigned int* counters, cudaStream_t st)
{
    if (row1 <= row0) return 0;
    const bool   steps_ok = radius == 1 && (step == 1 || step == 2 || step == 4 || step == 8 || step == 16);
    const uint2* i2 = (const uint2*)in;
    uint2*       o2 = (uint2*)out;
    if (g_hr_refl_atrous_impl != 0 && steps_ok && phi_normal == 32.0f && !(g.W & 1) && row0 % 8 == 0)
    { // pixel pairs
        R2Params P { g.W, g.H, 1.44269504f / sigma_depth, -1.44269504f / phi_color, approximate_with_ddgi, row0, row1 };
        switch (step)
        {
            case 1:
                if (!(g_hr_refl_atrous_impl == 3 && launch_r2_tma(g, i2, tile_flags, P, o2, counters, st))) launch_tiles<Dense<1>>(k_refl_atrous_v2<1>, g, i2, tile_flags, P, o2, st);
                break;
            case 2: launch_tiles<Dense<2>>(k_refl_atrous_v2<2>, g, i2, tile_flags, P, o2, st); break;
            case 4: launch_tiles<Dense<4>>(k_refl_atrous_v2<4>, g, i2, tile_flags, P, o2, st); break;
            case 8: launch_tiles<Interleaved<8>>(k_refl_atrous_v2s<8>, g, i2, tile_flags, P, o2, st); break;
            default: launch_tiles<Interleaved<16>>(k_refl_atrous_v2s<16>, g, i2, tile_flags, P, o2, st); break;
        }
        return 0;
    }
    if (!steps_ok) return -1;
    ReflAtrousParams P { g.W, g.H, step, radius, phi_color, phi_normal, sigma_depth, approximate_with_ddgi, row0, row1 };
    switch (step)
    {
        case 1: launch_atrous_t<1>(g, i2, tile_flags, P, o2, st); break;
        case 2: launch_atrous_t<2>(g, i2, tile_flags, P, o2, st); break;
        case 4: launch_atrous_t<4>(g, i2, tile_flags, P, o2, st); break;
        case 8: launch_atrous_t<8>(g, i2, tile_flags, P, o2, st); break;
        default: launch_atrous_t<16>(g, i2, tile_flags, P, o2, st); break;
    }
    return 0;
}
