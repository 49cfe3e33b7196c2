// svgf_temporal.cu — temporal reprojection + accumulation for the bit-mask effects.
//   K3  shadows/shadows_denoise_reprojection.comp:196-293  (+ reprojection.glsl:115-328, REPROJECTION_MOMENTS)
//   K9  ao/ao_denoise_reprojection.comp:191-260            (history length in its own R16F image)
// K2/K8 (reset_args) and the tile *lists* are replaced by a per-8x8-tile flag byte (1 = denoise list): the lists' order
// is non-deterministic in the reference (atomicAdd) and only membership matters.
//
// One CTA = 32x8 pixels (4 reference tiles), one warp per pixel row => every G-buffer / history row access is a
// contiguous 32-pixel span.  The 17x17 box mean of the packed ray mask is computed from 24 64-bit row bitmaps held in
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
template <bool PEER>
__device__ __forceinline__ uint32_t hist_ld32(const void* const* tab, const HistPeers& hp, int row, size_t word_index)
{
    if (hp.no_history) return 0u;
    if (!PEER) return __ldg(reinterpret_cast<const uint32_t*>(tab[0]) + word_index);
    const int       o = owner_of(hp, row);
    const uint32_t* p = reinterpret_cast<const uint32_t*>(tab[o]) + word_index;
    return o == hp.self ? __ldg(p) : __ldcg(p);
}
template <bool PEER>
__device__ __forceinline__ uint32_t hist_ld16(const void* const* tab, const HistPeers& hp, int row, size_t half_index)
{
    if (hp.no_history) return 0u;
    if (!PEER) return __ldg(reinterpret_cast<const unsigned short*>(tab[0]) + half_index);
    const int             o = owner_of(hp, row);
    const unsigned short* p = reinterpret_cast<const unsigned short*>(tab[o]) + half_index;
    return o == hp.self ? __ldg(p) : __ldcg(p);
}

// visibility input: the 1-spp ray mask (one word per 8x4 pixel block), or the spp > 1 count image (unoccluded rays per pixel)
template <bool COUNT> struct VisIn { const uint32_t* mask; };
template <> struct VisIn<true> { const uint8_t* count; int spp; };

// MODE 0: shadows (history RG16F .r, moments RGBA16F (m1,m2,N,0)); MODE 1: AO (history R16F, length R16F).
// PEER: linked ranks read a history texel from the rank that owns its row (hist_ld32 / hist_ld16).
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
                // all history-side loads of the common path (<= 4 bilinear taps + history length) are issued back to back,
                // before any of the validity arithmetic, so they share one HBM round trip
                const float fx = hfx - floorf(hfx), fy = hfy - floorf(hfy);
                const float w4[4] = { (1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy };
                {
                    const size_t hi = (size_t)hcy * W + hcx;
                    if (MODE == 0) hist_len = h2_to_f2(hist_ld32<PEER>(hp.aux, hp, hcy, 2 * hi + 1)).x;
                    else hist_len = __half2float(__ushort_as_half((unsigned short)hist_ld16<PEER>(hp.aux, hp, hcy, hi)));
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
                            hraw[s] = hist_ld32<PEER>(hp.img, hp, py, pi);
                            mraw[s] = hist_ld32<PEER>(hp.aux, hp, py, 2 * pi);
                        }
                        else hraw[s] = hist_ld16<PEER>(hp.img, hp, py, pi);
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
                                        hcol += h2_to_f2(hist_ld32<PEER>(hp.img, hp, py, pi)).x;
                                        const float2 mm = h2_to_f2(hist_ld32<PEER>(hp.aux, hp, py, 2 * pi));
                                        hm0 += mm.x;
                                        hm1 += mm.y;
                                    }
                                    else hcol += __half2float(__ushort_as_half((unsigned short)hist_ld16<PEER>(hp.img, hp, py, pi)));
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
    // tile classification: 4 tiles of 8 columns per CTA
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, flag);
    if (lx == 0 && b)
    {
        uint32_t t = ((b & 0xFFu) ? 1u : 0u) | ((b & 0xFF00u) ? 2u : 0u) | ((b & 0xFF0000u) ? 4u : 0u) | ((b & 0xFF000000u) ? 8u : 0u);
        atomicOr(&s_flags, t);
    }
    __syncthreads();
    if (threadIdx.x < 4)
    {
        const int tx = (x0 >> 3) + threadIdx.x, ty = y0 >> 3, TW = (W + 7) >> 3;
        if (tx < TW && y0 < H && y0 < row1) tile_flags[(size_t)ty * TW + tx] = (s_flags >> threadIdx.x) & 1u;
    }
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
