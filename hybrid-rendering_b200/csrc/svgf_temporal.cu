// svgf_temporal.cu — temporal reprojection + accumulation of the shadows, AO and reflections chains.
//   K3  shadows/shadows_denoise_reprojection.comp:196-293  (+ reprojection.glsl:115-328, REPROJECTION_MOMENTS)
//   K9  ao/ao_denoise_reprojection.comp:191-260            (history length in its own R16F image)
//   K14 reflections/reflections_denoise_reprojection.comp:174-289 (+ reprojection.glsl:78-111,115-328 REPROJECTION_REFLECTIONS)
// K2/K8 (reset_args) and the tile *lists* are replaced by a per-8x8-tile flag byte (1 = denoise list): the lists' order
// is non-deterministic in the reference (atomicAdd) and only membership matters.
//
// One CTA = 32x8 pixels (4 reference tiles), one warp per pixel row => every G-buffer / history row access is a
// contiguous 32-pixel span.  K3/K9: the 17x17 box mean of the packed ray mask is computed from 24 64-bit row bitmaps held in
// shared memory: count = sum_rows popcll(row & window) — exact (integers <= 289), like the reference's float sums.
// With spp > 1 the same kernel reads the 8-bit count image instead (k_temporal's COUNT).
#include "glsl_fast.cuh"
#include "hr_internal.h"
#include <type_traits>

namespace {

using namespace gf;

__device__ __forceinline__ bool inside(int x, int y, int W, int H) { return x >= 0 && y >= 0 && x < W && y < H; }

__device__ __forceinline__ HistTap fetch_prev(const GBufLevelDev& p, int x, int y)
{
    HistTap t { 0.0f, 0.0f, 0.0f, 0.0f }; // texelFetch out of bounds => zeros
    if (inside(x, y, p.W, p.H))
    {
        const size_t i  = (size_t)y * p.W + x;
        const float2 e  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(p.gb2 + i)));
        const float2 g3 = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(p.gb3 + i) + 1)); // (mesh id, linear z)
        t = HistTap { e.x, e.y, g3.x, __ldg(p.depth + i) };
    }
    return t;
}

// ---- history fetches through the owner table (HistPeers, hr_internal.h) ----
// Rows owned by this GPU use the read-only path; rows owned by a peer are read over NVLink with L1 bypassed (the mapping
// is rewritten by the peer every frame).  A warp's 32 pixels share their row in the static case, so the branch is uniform.
__device__ __forceinline__ int owner_of(const HistPeers& hp, int row)
{
    int o = 0;
#pragma unroll
    for (int r = 0; r < HR_MAX_RANKS - 1; r++) o += (r < hp.world - 1 && row >= hp.band_end[r]) ? 1 : 0;
    return o;
}
// The rank that owns a history row: `uniform` when one rank owns every row a pixel reads (k_refl_temporal looks it up once per
// pixel), otherwise owner_of per load.
struct HistOwner { int o; bool uniform; };

// element `index` of a history image (hp.img or hp.aux) in row `row`, read as T; a 16-bit T is returned zero-extended to 32 bits
template <bool PEER, class T>
__device__ __forceinline__ std::conditional_t<(sizeof(T) < 4), uint32_t, T> hist_ld(const void* const* tab, const HistPeers& hp, const HistOwner& ho, int row,
                                                                                      size_t index)
{
    if (hp.no_history) return {};
    if (!PEER) return __ldg(reinterpret_cast<const T*>(tab[0]) + index);
    const int o = ho.uniform ? ho.o : owner_of(hp, row);
    const T*  p = reinterpret_cast<const T*>(tab[o]) + index;
    return o == hp.self ? __ldg(p) : __ldcg(p);
}

// Tile classification of a 32x8 CTA: 4 tiles of 8 columns.  Each warp ORs the tiles its row flags into the shared word s_flags
// (zeroed by the kernel before its first barrier), then one flag byte per tile is stored.  A macro, not a function: an inlined
// call renumbers the registers of k_temporal's count forms, and both kernels keep the generated code they were tuned with.
#define STORE_TILE_FLAGS(flag, s_flags, lx, x0, y0, W, H, row1, tile_flags)                                                         \
    do {                                                                                                                            \
        const uint32_t _b = __ballot_sync(0xFFFFFFFFu, (flag));                                                                     \
        if ((lx) == 0 && _b)                                                                                                        \
            atomicOr(&(s_flags), ((_b & 0xFFu) ? 1u : 0u) | ((_b & 0xFF00u) ? 2u : 0u) | ((_b & 0xFF0000u) ? 4u : 0u) |             \
                                     ((_b & 0xFF000000u) ? 8u : 0u));                                                               \
        __syncthreads();                                                                                                            \
        if (threadIdx.x < 4)                                                                                                        \
        {                                                                                                                           \
            const int _tx = ((x0) >> 3) + threadIdx.x, _ty = (y0) >> 3, _TW = ((W) + 7) >> 3;                                       \
            if (_tx < _TW && (y0) < (H) && (y0) < (row1)) (tile_flags)[(size_t)_ty * _TW + _tx] = ((s_flags) >> threadIdx.x) & 1u; \
        }                                                                                                                           \
    } while (0)

// ---- K3 / K9 ----
struct TapRaw { uint32_t e, g3; float depth; };

__device__ __forceinline__ TapRaw fetch_prev_raw(const GBufLevelDev& p, size_t i)
{
    TapRaw r;
    r.e     = __ldg(reinterpret_cast<const uint32_t*>(p.gb2 + i));
    r.g3    = __ldg(reinterpret_cast<const uint32_t*>(p.gb3 + i) + 1); // (mesh id, linear z)
    r.depth = __ldg(p.depth + i);
    return r;
}

__device__ __forceinline__ HistTap decode_tap(const TapRaw& r)
{ // all-zero words decode to the out-of-bounds texel: normal oct(0,0), mesh id 0, depth 0
    const float2 e = h2_to_f2(r.e);
    return HistTap { e.x, e.y, h2_to_f2(r.g3).x, r.depth };
}

// visibility input: the 1-spp ray mask (one word per 8x4 pixel block), or the spp > 1 count image (unoccluded rays per pixel)
template <bool COUNT> struct VisIn { const uint32_t* mask; };
template <> struct VisIn<true> { const uint8_t* count; int spp; };

// MODE 0: shadows (history RG16F .r, moments RGBA16F (m1,m2,N,0)); MODE 1: AO (history R16F, length R16F).
// PEER: linked ranks read a history texel from the rank that owns its row (hist_ld).
// COUNT (spp > 1, SURVEY.md §8d; not in the reference): the 17x17 box mean is the sum of an 8-bit count tile (separable:
// 17-wide row sums, then 17 rows) divided by 289 * spp, the pixel's visibility is count / spp.
template <int MODE, bool PEER, bool COUNT>
__global__ void __launch_bounds__(256, 4) k_temporal(GBufLevelDev cur, GBufLevelDev prev, const VisIn<COUNT> in, const HistPeers hp,
                                                   FrameConsts fc, float alpha_p, float moments_alpha_p,
                                                   void* __restrict__ out_img, void* __restrict__ out_aux, uint8_t* __restrict__ tile_flags, int row0, int row1)
{
    // visibility of region rows y0-8 .. y0+15, columns x0-8 .. x0+39: 24 64-bit row bitmaps, or 24x48 unoccluded-ray counts
    __shared__ std::conditional_t<COUNT, unsigned char[24][48], unsigned long long[24]> s_vis;
    __shared__ std::conditional_t<COUNT, unsigned short[24][34], unsigned char[24][36]> s_h; // [region row][column] 17-wide sums, padded pitch
    __shared__ uint32_t s_flags;
    const int W = cur.W, H = cur.H, MW = (W + 7) >> 3, MH = (H + 3) >> 2;
    const int x0 = blockIdx.x * 32, y0 = row0 + blockIdx.y * 8;
    const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;

    if (threadIdx.x == 0) s_flags = 0;
    if constexpr (COUNT)
    {
        // pixels outside the (8x4-group padded) image read as the 1-bit path's out-of-image mask words: no ray unoccluded for
        // shadows, every ray unoccluded for AO (ao_denoise_reprojection.comp:111-112); padding pixels of partial groups: 0
        const unsigned char oob = MODE == 0 ? 0 : (unsigned char)in.spp;
        for (int i = threadIdx.x; i < 24 * 48; i += 256)
        {
            const int     r = i / 48, c = i - r * 48, px = x0 - 8 + c, py = y0 - 8 + r;
            unsigned char v;
            if (px < 0 || py < 0 || px >= MW * 8 || py >= MH * 4) v = oob;
            else if (px >= W || py >= H) v = 0;
            else v = __ldg(in.count + (size_t)py * W + px);
            s_vis[r][c] = v;
        }
    }
    else if (threadIdx.x < 24)
    {
        const uint32_t     oob_word = MODE == 0 ? 0u : 0xFFFFFFFFu; // ao_denoise_reprojection.comp:111-112
        const int          r  = threadIdx.x;              // region row, pixel y = y0 - 8 + r
        const int          my = (y0 >> 2) - 2 + (r >> 2); // mask row
        unsigned long long bits = 0;
#pragma unroll
        for (int c = 0; c < 6; c++)
        {
            const int      mx = (x0 >> 3) - 1 + c;
            const uint32_t w  = (mx < 0 || my < 0 || mx >= MW || my >= MH) ? oob_word : __ldg(in.mask + (size_t)my * MW + mx);
            bits |= (unsigned long long)((w >> ((r & 3) * 8)) & 0xFFu) << (c * 8);
        }
        s_vis[r] = bits;
    }
    // the pixel's own G-buffer words are requested before the barriers so their HBM round trip overlaps the mask fetch
    const int    x = x0 + lx, y = y0 + ly;
    const bool   inb = x < W && y < H && y < row1;
    const size_t idx = (size_t)y * W + x;
    float        depth = 1.0f;
    uint2        g2raw = make_uint2(0u, 0u);
    uint32_t     g3raw = 0u;
    if (inb)
    {
        depth = __ldg(cur.depth + idx);
        g2raw = __ldg(cur.gb2 + idx);
        g3raw = __ldg(reinterpret_cast<const uint32_t*>(cur.gb3 + idx) + 1);
    }
    __syncthreads();
    // horizontal 17-wide sums (columns lx .. lx+16 of the 48-wide region) for region rows ly, ly+8, ly+16
#pragma unroll
    for (int k = 0; k < 3; k++)
    {
        if constexpr (COUNT)
        {
            int sum = 0;
#pragma unroll
            for (int c = 0; c < 17; c++) sum += s_vis[ly + 8 * k][lx + c];
            s_h[ly + 8 * k][lx] = (unsigned short)sum;
        }
        else s_h[ly + 8 * k][lx] = (unsigned char)__popcll(s_vis[ly + 8 * k] & (0x1FFFFull << lx));
    }
    __syncthreads();

    bool flag = false;
    if (inb)
    {
        float o0 = 0.0f, o1 = 0.0f, m0 = 0.0f, m1 = 0.0f, hlen = 0.0f;
        if (MODE == 1) o0 = 1.0f;
        if (depth != 1.0f)
        {
            float vis;
            // COUNT: count / spp and the box mean below are exact quotients, as the oracle computes them: a multiply by the rounded
            // reciprocal gives 0.99999994 for count == spp at spp 41, 47, 55, ... and an all-open window's mean one ulp off 1 at
            // spp 3, 6, 7, ..., which flips `o0 < 1` / `o0 > 0` tile flags.  Both quotients are exact: 289 * 255 < 2^24.
            if constexpr (COUNT) vis = __fdiv_rn((float)s_vis[ly + 8][lx + 8], (float)in.spp);
            else vis = (float)((s_vis[ly + 8] >> (lx + 8)) & 1ull);
            // ---- reproject(), reprojection.glsl:115-328 ----
            const float  fw = (float)W, fh = (float)H;
            const float  tu = __fdiv_rn((float)x + 0.5f, fw), tv = __fdiv_rn((float)y + 0.5f, fh); // tex_coord, rounded as the validity test needs it
            const float4 g2 = h4_to_f4(g2raw);
            const float  cmesh = h2_to_f2(g3raw).x;
            const float  hfx = rn_mad(g2.z, fw, (float)x), hfy = rn_mad(g2.w, fh, (float)y); // history_coord_floor (:176), exactly rounded
            const int    hcx = (int)__fadd_rn(hfx, 0.5f), hcy = (int)__fadd_rn(hfy, 0.5f);       // history_coord (:175)
            const float  hu = __fadd_rn(tu, g2.z), hv = __fadd_rn(tv, g2.w);       // history_tex_coord (:177)
            const bool   in_frame = inside(hcx, hcy, W, H);                        // out_of_frame_disocclusion_check on history_coord
            const int    bx = (int)hfx, by = (int)hfy;                             // ivec2(history_coord_floor) truncates

            float hcol = 0.0f, hm0 = 0.0f, hm1 = 0.0f, hist_len = 0.0f;
            bool  valid = false;
            if (in_frame)
            {
                const HistOwner per_load { 0, false }; // the owner of every history load is looked up for its row
                // all history-side loads of the common path (<= 4 bilinear taps + history length) are issued back to back,
                // before any of the validity arithmetic, so they share one HBM round trip
                const float fx = hfx - floorf(hfx), fy = hfy - floorf(hfy);
                const float w4[4] = { (1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy };
                {
                    const size_t hi = (size_t)hcy * W + hcx;
                    if (MODE == 0) hist_len = h2_to_f2(hist_ld<PEER, uint32_t>(hp.aux, hp, per_load, hcy, 2 * hi + 1)).x;
                    else hist_len = __half2float(__ushort_as_half(hist_ld<PEER, unsigned short>(hp.aux, hp, per_load, hcy, hi)));
                }
                TapRaw   tr[4];
                uint32_t hraw[4], mraw[4];
#pragma unroll
                for (int s = 0; s < 4; s++)
                {
                    tr[s]   = TapRaw { 0u, 0u, 0.0f };
                    hraw[s] = 0u;
                    mraw[s] = 0u;
                    // A tap with bilinear weight exactly 0 cannot change the result: it adds 0 to every sum, and if only
                    // such taps are valid sumw = 0 < 0.01 sends us to the 3x3 fallback exactly as "no tap valid" does.
                    // Static pixels (motion 0 => fx = fy = 0) therefore need 1 tap instead of 4.
                    const int px = bx + (s & 1), py = by + (s >> 1);
                    if (w4[s] != 0.0f && inside(px, py, W, H))
                    { // texelFetch out of bounds => zeros
                        const size_t pi = (size_t)py * W + px;
                        tr[s] = fetch_prev_raw(prev, pi);
                        if (MODE == 0)
                        {
                            hraw[s] = hist_ld<PEER, uint32_t>(hp.img, hp, per_load, py, pi);
                            mraw[s] = hist_ld<PEER, uint32_t>(hp.aux, hp, per_load, py, 2 * pi);
                        }
                        else hraw[s] = hist_ld<PEER, unsigned short>(hp.img, hp, per_load, py, pi);
                    }
                }
                const float3 cn   = rn_octohedral_to_direction(g2.x, g2.y);
                const float3 cpos = rn_world_position_from_depth(tu, tv, depth, fc.view_proj_inverse);
                float sumw = 0.0f;
                bool  any  = false;
#pragma unroll
                for (int s = 0; s < 4; s++)
                {
                    if (w4[s] == 0.0f) continue;
                    if (rn_tap_valid(decode_tap(tr[s]), cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
                    {
                        any = true;
                        const float2 hh = h2_to_f2(hraw[s]), mm = h2_to_f2(mraw[s]);
                        hcol += w4[s] * hh.x;
                        hm0 += w4[s] * mm.x;
                        hm1 += w4[s] * mm.y;
                        sumw += w4[s];
                    }
                }
                if (any)
                {
                    valid = sumw >= 0.01f;
                    if (valid) { const float inv = fast_rcp(sumw); hcol = __fdiv_rn(hcol, sumw); hm0 *= inv; hm1 *= inv; } // colour: exact quotient (tile classification compares it with 0 / 1)
                    else { hcol = 0.0f; hm0 = 0.0f; hm1 = 0.0f; }
                }
                if (!valid)
                {
                    float cntv = 0.0f;
                    for (int yy = -1; yy <= 1; yy++)
                        for (int xx = -1; xx <= 1; xx++)
                        {
                            const int px = hcx + xx, py = hcy + yy;
                            const HistTap t = fetch_prev(prev, px, py);
                            if (rn_tap_valid(t, cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
                            {
                                if (inside(px, py, W, H))
                                {
                                    const size_t pi = (size_t)py * W + px;
                                    if (MODE == 0)
                                    {
                                        hcol += h2_to_f2(hist_ld<PEER, uint32_t>(hp.img, hp, per_load, py, pi)).x;
                                        const float2 mm = h2_to_f2(hist_ld<PEER, uint32_t>(hp.aux, hp, per_load, py, 2 * pi));
                                        hm0 += mm.x;
                                        hm1 += mm.y;
                                    }
                                    else hcol += __half2float(__ushort_as_half(hist_ld<PEER, unsigned short>(hp.img, hp, per_load, py, pi)));
                                }
                                cntv += 1.0f;
                            }
                        }
                    if (cntv > 0.0f) { valid = true; const float inv = fast_rcp(cntv); hcol = __fdiv_rn(hcol, cntv); hm0 *= inv; hm1 *= inv; }
                }
            }
            if (!valid) { hcol = 0.0f; hm0 = 0.0f; hm1 = 0.0f; hist_len = 0.0f; }
            // ---- accumulate ----
            hlen = fminf(32.0f, valid ? hist_len + 1.0f : 1.0f);
            const float ihlen = __frcp_rn(hlen); // exact: alpha decides whether a saturated pixel lands on 1.0 or one ulp below (tile classification)
            if (valid)
            {
                // neighborhood_mean: rows ly .. ly+16 of the per-row 17-wide sums (separable: 3 row sums per thread instead of 17)
                int cnt = 0;
#pragma unroll
                for (int r = 0; r < 17; r++) cnt += s_h[ly + r][lx];
                float mean;
                if constexpr (COUNT) mean = __fdiv_rn((float)cnt, 289.0f * (float)in.spp); // exact quotient, see vis above
                else
                { // a multiply by the rounded 1/289 is enough for the mask: visibility is 0 or 1, and cnt * (1/289) is exactly 1
                  // for an all-open window (cnt = 289) and exactly 0 for a closed one, so no tile flag can move
                    mean = (float)cnt * (1.0f / 289.0f);
                }
                const float sd   = sqrtf(fmaxf(mean - mean * mean, 0.0f));
                hcol             = fminf(fmaxf(hcol, mean - 0.5f * sd), mean + 0.5f * sd);
            }
            const float alpha = valid ? fmaxf(alpha_p, ihlen) : 1.0f;
            if (MODE == 0)
            {
                const float am = valid ? fmaxf(moments_alpha_p, ihlen) : 1.0f;
                m0 = hm0 * (1.0f - am) + vis * am;
                m1 = hm1 * (1.0f - am) + (vis * vis) * am;
                o1 = fmaxf(0.0f, m1 - m0 * m0);
            }
            o0 = __fadd_rn(__fmul_rn(hcol, __fsub_rn(1.0f, alpha)), __fmul_rn(vis, alpha)); // GLSL mix, never contracted: `o0 < 1` / `o0 > 0` classify the tile
        }
        if (MODE == 0)
        {
            reinterpret_cast<uint32_t*>(out_img)[idx] = f2_to_h2(o0, o1);
            reinterpret_cast<uint2*>(out_aux)[idx]    = make_uint2(f2_to_h2(m0, m1), f2_to_h2(hlen, 0.0f));
            flag = depth != 1.0f && o0 > 0.0f;
        }
        else
        {
            reinterpret_cast<__half*>(out_img)[idx] = __float2half_rn(o0);
            reinterpret_cast<__half*>(out_aux)[idx] = __float2half_rn(hlen);
            flag = o0 < 1.0f;
        }
    }
    STORE_TILE_FLAGS(flag, s_flags, lx, x0, y0, W, H, row1, tile_flags);
}

// ---- K14 ----
struct ReflTemporalParams { float alpha, moments_alpha; int approximate_with_ddgi; int row0, row1; int rot; }; // rot: the last `rot` tile rows are scheduled first

// All history taps of a pixel lie in rows hcy-1 .. hcy+1: the owner is looked up once per pixel (two owner_of calls) and only
// pixels whose taps straddle a band border fall back to a lookup per load.
template <bool PEER>
__device__ __forceinline__ HistOwner owner_cache(const HistPeers& hp, int row_lo, int row_hi)
{
    HistOwner c { 0, true };
    if (PEER) { c.o = owner_of(hp, row_lo); c.uniform = c.o == owner_of(hp, row_hi); }
    return c;
}

// CTA = 32x8 pixels.  17x17 mean / std-dev of the current ray-trace colour (neighborhood_standard_deviation :133-157; the
// reference does 289 fetches per pixel): separable, each direction as a SLIDING window — stage the 48x24 rgb region; 144 threads
// each walk half a staged row of one channel keeping the running 17-tap sums of c and c^2 (17 + 15 * 2 loads instead of
// 16 * 17); 192 threads each walk one column of one of the six horizontal sums (17 + 7 * 2 loads instead of 8 * 17); every
// pixel then reads its six window sums.
// hp.img = last frame's temporal output (or prev_image), hp.aux = last frame's moments, of the rank that owns the row (PEER)
template <bool PEER>
__global__ void __launch_bounds__(256, 5) k_refl_temporal(GBufLevelDev cur, GBufLevelDev prev, const uint2* __restrict__ input, const HistPeers hp, FrameConsts fc,
                                                        ReflTemporalParams P, uint2* __restrict__ out, uint2* __restrict__ mom_out, uint8_t* __restrict__ tile_flags)
{
    __shared__ float    s_c[3][24][49];  // row pitch 49: the 144 row walkers of a phase hit 32 different banks
    __shared__ float    s_h[6][24][33];  // horizontal window sums: [ch] = sum c, [3 + ch] = sum c^2 (pitch 33: the row walkers store one column at a time)
    __shared__ float    s_v[6][8][32];   // 17x17 window sums per pixel of the tile
    __shared__ uint32_t s_flags;
    const int W = cur.W, H = cur.H;
    // PEER: the bottom halo rows read their history across NVLink (slow taps); they are scheduled first so that the bulk of the band
    // covers their latency instead of leaving it as the kernel's tail
    const int by = (int)blockIdx.y < P.rot ? (int)gridDim.y - P.rot + (int)blockIdx.y : (int)blockIdx.y - P.rot;
    const int x0 = blockIdx.x * 32, y0 = P.row0 + by * 8;
    const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_flags = 0;
    for (int i = threadIdx.x; i < 48 * 24; i += 256)
    {
        const int rx = i % 48, ry = i / 48, px = x0 - 8 + rx, py = y0 - 8 + ry;
        float     r = 0.0f, g = 0.0f, b = 0.0f;
        if (inside(px, py, W, H))
        {
            const uint2  w = __ldg(input + (size_t)py * W + px);
            const float2 a = h2_to_f2(w.x), c = h2_to_f2(w.y);
            r = a.x; g = a.y; b = c.x;
        }
        s_c[0][ry][rx] = r; s_c[1][ry][rx] = g; s_c[2][ry][rx] = b;
    }
    __syncthreads();
    if (threadIdx.x < 144)
    { // horizontal: task = (half, channel, row); outputs 16 columns
        const int    row = threadIdx.x % 24, ch = (threadIdx.x / 24) % 3, base = (threadIdx.x / 72) * 16;
        const float* v = &s_c[ch][row][base];
        float        a = 0.0f, b = 0.0f;
#pragma unroll
        for (int t = 0; t < 17; t++) { const float c = v[t]; a += c; b = fmaf(c, c, b); }
        s_h[ch][row][base]     = a;
        s_h[3 + ch][row][base] = b;
#pragma unroll
        for (int i = 1; i < 16; i++)
        {
            const float cin = v[16 + i], cout = v[i - 1];
            a += cin - cout;
            b = fmaf(cin, cin, fmaf(-cout, cout, b));
            s_h[ch][row][base + i]     = a;
            s_h[3 + ch][row][base + i] = b;
        }
    }
    __syncthreads();
    if (threadIdx.x < 192)
    { // vertical: task = (quantity, column); outputs 8 rows
        const int    q = threadIdx.x >> 5, col = threadIdx.x & 31;
        float        a = 0.0f;
#pragma unroll
        for (int r = 0; r < 17; r++) a += s_h[q][r][col];
        s_v[q][0][col] = a;
#pragma unroll
        for (int i = 1; i < 8; i++)
        {
            a += s_h[q][16 + i][col] - s_h[q][i - 1][col];
            s_v[q][i][col] = a;
        }
    }
    __syncthreads();

    const int x = x0 + lx, y = y0 + ly;
    bool      flag = false;
    if (x < W && y < H && y < P.row1)
    {
        const size_t idx   = (size_t)y * W + x;
        const float  depth = __ldg(cur.depth + idx);
        const uint2  g2w = __ldg(cur.gb2 + idx), g3w = __ldg(cur.gb3 + idx);
        const float4 g2 = h4_to_f4(g2w), g3 = h4_to_f4(g3w);
        const float  roughness = g3.x;
        float        o[4] = { 0, 0, 0, 0 }, m[4] = { 0, 0, 0, 0 };
        if (depth != 1.0f)
        {
            const float color[3] = { s_c[0][ly + 8][lx + 8], s_c[1][ly + 8][lx + 8], s_c[2][ly + 8][lx + 8] };
            const float ray_length = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(input + idx) + 1)).y;
            const float fw = (float)W, fh = (float)H;
            const float tu = ((float)x + 0.5f) / fw, tv = ((float)y + 0.5f) / fh;
            const float3 cn = rn_octohedral_to_direction(g2.x, g2.y);
            const float  cmesh = g3.z, curvature = g3.y;
            const float3 cpos = rn_world_position_from_depth(tu, tv, depth, fc.view_proj_inverse);
            // compute_history_coord, reprojection.glsl:101-111
            float hfx = rn_mad(g2.z, fw, (float)x), hfy = rn_mad(g2.w, fh, (float)y);
            if (ray_length > 0.0f && curvature == 0.0f)
            { // virtual_point_reprojection :78-97 — exactly rounded: it lands on texel corners for a static camera
                const float2 vp = rn_virtual_point_reprojection(x, y, fw, fh, depth, ray_length, fc.cam_pos, fc.view_proj_inverse, fc.prev_view_proj);
                hfx = vp.x;
                hfy = vp.y;
            }
            const int   hcx = (int)hfx, hcy = (int)hfy; // ivec2(reprojected_coord) :171
            const float hu = __fadd_rn(tu, g2.z), hv = __fadd_rn(tv, g2.w);
            const bool  in_frame = inside(hcx, hcy, W, H);
            const HistOwner oc = owner_cache<PEER>(hp, max(hcy - 1, 0), min(hcy + 1, H - 1));
            float hc[3] = { 0, 0, 0 }, hm0 = 0.0f, hm1 = 0.0f;
            bool  valid = false;
            if (in_frame)
            {
                const float fx = hfx - floorf(hfx), fy = hfy - floorf(hfy);
                const float w4[4] = { (1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy };
                float sumw = 0.0f;
                bool  any  = false;
#pragma unroll
                for (int s = 0; s < 4; s++)
                {
                    if (w4[s] == 0.0f) continue; // exact: see k_temporal
                    const int px = hcx + (s & 1), py = hcy + (s >> 1);
                    const HistTap t = fetch_prev(prev, px, py);
                    if (rn_tap_valid(t, cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
                    {
                        any = true;
                        if (inside(px, py, W, H))
                        {
                            const size_t pi = (size_t)py * W + px;
                            const float4 hv4 = h4_to_f4(hist_ld<PEER, uint2>(hp.img, hp, oc, py, pi));
                            const float2 mm  = h2_to_f2(hist_ld<PEER, uint32_t>(hp.aux, hp, oc, py, 2 * pi));
                            hc[0] += w4[s] * hv4.x; hc[1] += w4[s] * hv4.y; hc[2] += w4[s] * hv4.z;
                            hm0 += w4[s] * mm.x; hm1 += w4[s] * mm.y;
                        }
                        sumw += w4[s];
                    }
                }
                if (any)
                {
                    valid = sumw >= 0.01f;
                    const float inv = valid ? fast_rcp(sumw) : 0.0f;
                    hc[0] *= inv; hc[1] *= inv; hc[2] *= inv; hm0 *= inv; hm1 *= inv;
                }
                if (!valid)
                {
                    float cnt = 0.0f;
                    for (int yy = -1; yy <= 1; yy++)
                        for (int xx = -1; xx <= 1; xx++)
                        {
                            const int px = hcx + xx, py = hcy + yy;
                            const HistTap t = fetch_prev(prev, px, py);
                            if (rn_tap_valid(t, cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
                            {
                                if (inside(px, py, W, H))
                                {
                                    const size_t pi = (size_t)py * W + px;
                                    const float4 hv4 = h4_to_f4(hist_ld<PEER, uint2>(hp.img, hp, oc, py, pi));
                                    const float2 mm  = h2_to_f2(hist_ld<PEER, uint32_t>(hp.aux, hp, oc, py, 2 * pi));
                                    hc[0] += hv4.x; hc[1] += hv4.y; hc[2] += hv4.z; hm0 += mm.x; hm1 += mm.y;
                                }
                                cnt += 1.0f;
                            }
                        }
                    if (cnt > 0.0f) { valid = true; const float inv = fast_rcp(cnt); hc[0] *= inv; hc[1] *= inv; hc[2] *= inv; hm0 *= inv; hm1 *= inv; }
                }
            }
            float hist_len = 0.0f;
            if (valid) hist_len = h2_to_f2(hist_ld<PEER, uint32_t>(hp.aux, hp, oc, hcy, 2 * ((size_t)hcy * W + hcx) + 1)).x;
            else { hc[0] = hc[1] = hc[2] = 0.0f; hm0 = hm1 = 0.0f; }
            const float hlen = fminf(32.0f, valid ? hist_len + 1.0f : 1.0f);
            if (valid)
            { // clip_aabb(mean - sigma, mean + sigma) :111-129
                float mn[3], mx[3];
#pragma unroll
                for (int ch = 0; ch < 3; ch++)
                {
                    const float m1 = s_v[ch][ly][lx], m2 = s_v[3 + ch][ly][lx];
                    const float mean = m1 * (1.0f / 289.0f), var = m2 * (1.0f / 289.0f) - mean * mean, sd = sqrtf(fmaxf(var, 0.0f));
                    mn[ch] = mean - sd;
                    mx[ch] = mean + sd;
                }
                float cv[3], ctr[3], mabs = 0.0f;
#pragma unroll
                for (int ch = 0; ch < 3; ch++)
                {
                    ctr[ch] = 0.5f * (mx[ch] + mn[ch]);
                    const float ext = 0.5f * (mx[ch] - mn[ch]) + 0.001f;
                    cv[ch] = hc[ch] - ctr[ch];
                    mabs   = fmaxf(mabs, fabsf(cv[ch] * fast_rcp(ext)));
                }
                if (mabs > 1.0f) { const float im = fast_rcp(mabs); hc[0] = ctr[0] + cv[0] * im; hc[1] = ctr[1] + cv[1] * im; hc[2] = ctr[2] + cv[2] * im; }
            }
            const float cdl = sqrtf(fc.camera_delta[0] * fc.camera_delta[0] + fc.camera_delta[1] * fc.camera_delta[1] + fc.camera_delta[2] * fc.camera_delta[2]);
            const float maxacc = cdl > 0.0f ? 8.0f : hlen;
            const float iacc   = fast_rcp(maxacc);
            const float alpha  = valid ? fmaxf(P.alpha, iacc) : 1.0f;
            const float alpham = valid ? fmaxf(P.moments_alpha, iacc) : 1.0f;
            const float lum = luminance(color[0], color[1], color[2]);
            const float mo0 = hm0 * (1.0f - alpham) + lum * alpham, mo1 = hm1 * (1.0f - alpham) + (lum * lum) * alpham;
            o[0] = hc[0] * (1.0f - alpha) + color[0] * alpha;
            o[1] = hc[1] * (1.0f - alpha) + color[1] * alpha;
            o[2] = hc[2] * (1.0f - alpha) + color[2] * alpha;
            o[3] = fmaxf(0.0f, mo1 - mo0 * mo0);
            m[0] = mo0; m[1] = mo1; m[2] = hlen; m[3] = 0.0f;
        }
        mom_out[idx] = pack_h4(m[0], m[1], m[2], m[3]);
        out[idx]     = pack_h4(o[0], o[1], o[2], o[3]);
        flag = depth != 1.0f && roughness >= 0.05f && (P.approximate_with_ddgi != 1 || roughness <= 0.75f);
    }
    STORE_TILE_FLAGS(flag, s_flags, lx, x0, y0, W, H, P.row1, tile_flags);
}

} // namespace

template <bool COUNT>
static void launch_temporal_form(int kind, const GBufLevelDev& cur, const GBufLevelDev& prev, VisIn<COUNT> in, const HistPeers& hist, const FrameConsts& fc, float alpha,
                                 float moments_alpha, void* out_img, void* out_aux, uint8_t* tile_flags, int row0, int row1, cudaStream_t st)
{
    const bool peer = hist.world > 1;
    const auto k    = kind == PASS_AO ? (peer ? k_temporal<1, true, COUNT> : k_temporal<1, false, COUNT>)
                                      : (peer ? k_temporal<0, true, COUNT> : k_temporal<0, false, COUNT>);
    k<<<dim3((cur.W + 31) / 32, (row1 - row0 + 7) / 8), 256, 0, st>>>(cur, prev, in, hist, fc, alpha, moments_alpha, out_img, out_aux, tile_flags, row0, row1);
}

// kind: PASS_SHADOWS (K3) or PASS_AO (K9, moments_alpha unused); visibility from `mask` at spp 1, from `count` at spp > 1
void launch_temporal(int kind, const GBufLevelDev& cur, const GBufLevelDev& prev, const uint32_t* mask, const uint8_t* count, int spp, const HistPeers& hist,
                     const FrameConsts& fc, float alpha, float moments_alpha, void* out_img, void* out_aux, uint8_t* tile_flags, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    if (spp > 1) launch_temporal_form<true>(kind, cur, prev, { count, spp }, hist, fc, alpha, moments_alpha, out_img, out_aux, tile_flags, row0, row1, st);
    else launch_temporal_form<false>(kind, cur, prev, { mask }, hist, fc, alpha, moments_alpha, out_img, out_aux, tile_flags, row0, row1, st);
}

void launch_reflections_temporal(const GBufLevelDev& cur, const GBufLevelDev& prev, const void* input, const HistPeers& hist, const FrameConsts& fc, float alpha,
                                 float moments_alpha, int approximate_with_ddgi, void* out, void* mom_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    dim3               grid((cur.W + 31) / 32, (row1 - row0 + 7) / 8);
    int                rot = 0;
    if (hist.world > 1 && hist.self < hist.world - 1) rot = (row1 - hist.band_end[hist.self] + 7) / 8; // tile rows below this rank's band
    if (rot < 0 || rot >= (int)grid.y) rot = 0;
    ReflTemporalParams P { alpha, moments_alpha, approximate_with_ddgi, row0, row1, rot };
    if (hist.world > 1) k_refl_temporal<true><<<grid, 256, 0, st>>>(cur, prev, (const uint2*)input, hist, fc, P, (uint2*)out, (uint2*)mom_out, tile_flags);
    else k_refl_temporal<false><<<grid, 256, 0, st>>>(cur, prev, (const uint2*)input, hist, fc, P, (uint2*)out, (uint2*)mom_out, tile_flags);
}
