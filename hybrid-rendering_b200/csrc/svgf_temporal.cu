// svgf_temporal.cu — temporal reprojection + accumulation for the bit-mask effects.
//   K3  shadows/shadows_denoise_reprojection.comp:196-293  (+ reprojection.glsl:115-328, REPROJECTION_MOMENTS)
//   K9  ao/ao_denoise_reprojection.comp:191-260            (history length in its own R16F image)
// K2/K8 (reset_args) and the tile *lists* are replaced by a per-8x8-tile flag byte (1 = denoise list): the lists' order
// is non-deterministic in the reference (atomicAdd) and only membership matters.
//
// One CTA = 32x8 pixels (4 reference tiles), one warp per pixel row => every G-buffer / history row access is a
// contiguous 32-pixel span.  The 17x17 box mean of the packed ray mask is computed from 24 64-bit row bitmaps held in
// shared memory: count = sum_rows popcll(row & window) — exact (integers <= 289), like the reference's float sums.
#include "glsl_fast.cuh"
#include "hr_internal.h"

namespace {

using namespace gf;

struct Tap { float3 n; float mesh_id; float depth; };

__device__ __forceinline__ bool inside(int x, int y, int W, int H) { return x >= 0 && y >= 0 && x < W && y < H; }

__device__ __forceinline__ Tap fetch_prev(const GBufLevelDev& p, int x, int y)
{
    Tap t;
    if (inside(x, y, p.W, p.H))
    {
        const size_t i  = (size_t)y * p.W + x;
        const float2 e  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(p.gb2 + i)));
        const float2 g3 = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(p.gb3 + i) + 1)); // (mesh id, linear z)
        t.n       = octohedral_to_direction(e.x, e.y);
        t.mesh_id = g3.x;
        t.depth   = __ldg(p.depth + i);
    }
    else
    { // texelFetch out of bounds => zeros
        t.n       = octohedral_to_direction(0.0f, 0.0f);
        t.mesh_id = 0.0f;
        t.depth   = 0.0f;
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

__device__ __forceinline__ Tap decode_tap(const TapRaw& r)
{ // all-zero words decode to the out-of-bounds texel: normal oct(0,0), mesh id 0, depth 0
    Tap          t;
    const float2 e = h2_to_f2(r.e);
    t.n       = octohedral_to_direction(e.x, e.y);
    t.mesh_id = h2_to_f2(r.g3).x;
    t.depth   = r.depth;
    return t;
}

// world_position_from_depth (common.glsl:175-186) with an approximate reciprocal: only feeds the 5.0-unit plane-distance test
__device__ __forceinline__ float3 world_position_from_depth_fast(float u, float v, float d, const float* __restrict__ M)
{
    const float sx = u * 2.0f - 1.0f, sy = v * 2.0f - 1.0f;
    const float wx = M[0] * sx + M[4] * sy + M[8] * d + M[12];
    const float wy = M[1] * sx + M[5] * sy + M[9] * d + M[13];
    const float wz = M[2] * sx + M[6] * sy + M[10] * d + M[14];
    const float ww = M[3] * sx + M[7] * sy + M[11] * d + M[15];
    const float iw = fast_rcp(ww);
    return make_float3(wx * iw, wy * iw, wz * iw);
}

// is_reprojection_valid, reprojection.glsl:52-67 (frame test hoisted by the caller)
__device__ __forceinline__ bool tap_valid(const Tap& t, float3 cur_pos, float3 cur_n, float cur_mesh, float hu, float hv, const float* vpi)
{
    if (!(cur_mesh == t.mesh_id)) return false;
    const float3 hp = world_position_from_depth_fast(hu, hv, t.depth, vpi);
    const float3 d  = make_float3(cur_pos.x - hp.x, cur_pos.y - hp.y, cur_pos.z - hp.z);
    if (fabsf(dot3(d, cur_n)) > 5.0f) return false; // PLANE_DISTANCE
    const float nd = fabsf(dot3(cur_n, t.n));
    if (!(nd * nd > 0.1f)) return false; // NORMAL_DISTANCE
    return true;
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

// MODE 0: shadows (history RG16F .r, moments RGBA16F (m1,m2,N,0)); MODE 1: AO (history R16F, length R16F)
template <int MODE, bool PEER>
__global__ void __launch_bounds__(256, 4) k_temporal(GBufLevelDev cur, GBufLevelDev prev, const uint32_t* __restrict__ mask, const HistPeers hp,
                                                   FrameConsts fc, float alpha_p, float moments_alpha_p,
                                                   void* __restrict__ out_img, void* __restrict__ out_aux, uint8_t* __restrict__ tile_flags, int row0, int row1)
{
    __shared__ unsigned long long s_rows[24];
    __shared__ unsigned char      s_h[24][36]; // [region row][column], padded pitch
    __shared__ uint32_t           s_flags;
    const int W = cur.W, H = cur.H, MW = (W + 7) >> 3, MH = (H + 3) >> 2;
    const int x0 = blockIdx.x * 32, y0 = row0 + blockIdx.y * 8;
    const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
    const uint32_t oob_word = MODE == 0 ? 0u : 0xFFFFFFFFu; // ao_denoise_reprojection.comp:111-112

    if (threadIdx.x == 0) s_flags = 0;
    if (threadIdx.x < 24)
    {
        const int          r  = threadIdx.x;              // region row, pixel y = y0 - 8 + r
        const int          my = (y0 >> 2) - 2 + (r >> 2); // mask row
        unsigned long long bits = 0;
#pragma unroll
        for (int c = 0; c < 6; c++)
        {
            const int      mx = (x0 >> 3) - 1 + c;
            const uint32_t w  = (mx < 0 || my < 0 || mx >= MW || my >= MH) ? oob_word : __ldg(mask + (size_t)my * MW + mx);
            bits |= (unsigned long long)((w >> ((r & 3) * 8)) & 0xFFu) << (c * 8);
        }
        s_rows[r] = bits;
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
    {   // horizontal 17-wide window counts (columns lx .. lx+16 of the 48-wide region) for region rows ly, ly+8, ly+16
        const unsigned long long win = 0x1FFFFull << lx;
#pragma unroll
        for (int k = 0; k < 3; k++) s_h[ly + 8 * k][lx] = (unsigned char)__popcll(s_rows[ly + 8 * k] & win);
    }
    __syncthreads();

    bool flag = false;
    if (inb)
    {
        float o0 = 0.0f, o1 = 0.0f, m0 = 0.0f, m1 = 0.0f, hlen = 0.0f;
        if (MODE == 1) o0 = 1.0f;
        if (depth != 1.0f)
        {
            const float vis = (float)((s_rows[ly + 8] >> (lx + 8)) & 1ull);
            // ---- reproject(), reprojection.glsl:115-328 ----
            const float  fw = (float)W, fh = (float)H;
            const float  tu = ((float)x + 0.5f) * fast_rcp(fw), tv = ((float)y + 0.5f) * fast_rcp(fh);
            const float4 g2 = h4_to_f4(g2raw);
            const float  cmesh = h2_to_f2(g3raw).x;
            const float  hfx = rn_mad(g2.z, fw, (float)x), hfy = rn_mad(g2.w, fh, (float)y); // history_coord_floor (:176), exactly rounded
            const int    hcx = (int)__fadd_rn(hfx, 0.5f), hcy = (int)__fadd_rn(hfy, 0.5f);       // history_coord (:175)
            const float  hu = tu + g2.z, hv = tv + g2.w;                           // history_tex_coord (:177)
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
                const float3 cn   = octohedral_to_direction(g2.x, g2.y);
                const float3 cpos = world_position_from_depth_fast(tu, tv, depth, fc.view_proj_inverse);
                float sumw = 0.0f;
                bool  any  = false;
#pragma unroll
                for (int s = 0; s < 4; s++)
                {
                    if (w4[s] == 0.0f) continue;
                    if (tap_valid(decode_tap(tr[s]), cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
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
                            const Tap t  = fetch_prev(prev, px, py);
                            if (tap_valid(t, cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
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
                // neighborhood_mean: rows ly .. ly+16 of the per-row 17-wide counts (separable: 3 popcll per thread instead of 17)
                int cnt = 0;
#pragma unroll
                for (int r = 0; r < 17; r++) cnt += s_h[ly + r][lx];
                // a multiply by the rounded 1/289 is enough here (unlike temporal_count): visibility is 0 or 1, and cnt * (1/289)
                // is exactly 1 for an all-open window (cnt = 289) and exactly 0 for a closed one, so no tile flag can move
                const float mean = (float)cnt * (1.0f / 289.0f);
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

// ---- spp > 1: count image instead of the bit mask (SURVEY.md §8d; not in the reference) ---------------------------------
// Same kernel as k_temporal<MODE, false> except for where the visibility comes from: the 17x17 box mean is the sum of an
// 8-bit count tile (separable: 17-wide row sums, then 17 rows) divided by 289 * spp, the pixel's visibility is count / spp.
// Kept as a separate kernel so the 1-spp path stays exactly what the parity runs validated.  PEER: linked ranks read a history texel
// from the rank that owns its row (hist_ld32 / hist_ld16), like k_temporal<MODE, true>.
template <int MODE, bool PEER>
__device__ __forceinline__ void temporal_count(GBufLevelDev cur, GBufLevelDev prev, const uint8_t* __restrict__ count, int spp, const HistPeers hp, FrameConsts fc,
                                               float alpha_p, float moments_alpha_p, void* __restrict__ out_img, void* __restrict__ out_aux,
                                               uint8_t* __restrict__ tile_flags, int row0, int row1)
{
    __shared__ unsigned char  s_cnt[24][48]; // unoccluded rays per pixel, region rows y0-8 .. y0+15, columns x0-8 .. x0+39
    __shared__ unsigned short s_h[24][34];   // per-row 17-wide sums
    __shared__ uint32_t       s_flags;
    const int W = cur.W, H = cur.H, MW = (W + 7) >> 3, MH = (H + 3) >> 2;
    const int x0 = blockIdx.x * 32, y0 = row0 + blockIdx.y * 8;
    const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
    // pixels outside the (8x4-group padded) image read as the 1-bit path's out-of-image mask words: no ray unoccluded for
    // shadows, every ray unoccluded for AO (ao_denoise_reprojection.comp:111-112); padding pixels of partial groups: 0
    const unsigned char oob = MODE == 0 ? 0 : (unsigned char)spp;

    if (threadIdx.x == 0) s_flags = 0;
    for (int i = threadIdx.x; i < 24 * 48; i += 256)
    {
        const int     r = i / 48, c = i - r * 48, px = x0 - 8 + c, py = y0 - 8 + r;
        unsigned char v;
        if (px < 0 || py < 0 || px >= MW * 8 || py >= MH * 4) v = oob;
        else if (px >= W || py >= H) v = 0;
        else v = __ldg(count + (size_t)py * W + px);
        s_cnt[r][c] = v;
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
    {   // horizontal 17-wide sums (columns lx .. lx+16 of the 48-wide region) for region rows ly, ly+8, ly+16
#pragma unroll
        for (int kk = 0; kk < 3; kk++)
        {
            int sum = 0;
#pragma unroll
            for (int c = 0; c < 17; c++) sum += s_cnt[ly + 8 * kk][lx + c];
            s_h[ly + 8 * kk][lx] = (unsigned short)sum;
        }
    }
    __syncthreads();

    bool flag = false;
    if (inb)
    {
        float o0 = 0.0f, o1 = 0.0f, m0 = 0.0f, m1 = 0.0f, hlen = 0.0f;
        if (MODE == 1) o0 = 1.0f;
        if (depth != 1.0f)
        {
            // count / spp and the box mean below are exact quotients, as the oracle computes them: a multiply by the rounded
            // reciprocal gives 0.99999994 for count == spp at spp 41, 47, 55, ... and an all-open window's mean one ulp off 1 at
            // spp 3, 6, 7, ..., which flips `o0 < 1` / `o0 > 0` tile flags.  Both quotients are exact: 289 * 255 < 2^24.
            const float vis = __fdiv_rn((float)s_cnt[ly + 8][lx + 8], (float)spp);
            // ---- reproject(), reprojection.glsl:115-328 ----
            const float  fw = (float)W, fh = (float)H;
            const float  tu = ((float)x + 0.5f) * fast_rcp(fw), tv = ((float)y + 0.5f) * fast_rcp(fh);
            const float4 g2 = h4_to_f4(g2raw);
            const float  cmesh = h2_to_f2(g3raw).x;
            const float  hfx = rn_mad(g2.z, fw, (float)x), hfy = rn_mad(g2.w, fh, (float)y); // history_coord_floor (:176), exactly rounded
            const int    hcx = (int)__fadd_rn(hfx, 0.5f), hcy = (int)__fadd_rn(hfy, 0.5f);       // history_coord (:175)
            const float  hu = tu + g2.z, hv = tv + g2.w;                           // history_tex_coord (:177)
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
                const float3 cn   = octohedral_to_direction(g2.x, g2.y);
                const float3 cpos = world_position_from_depth_fast(tu, tv, depth, fc.view_proj_inverse);
                float sumw = 0.0f;
                bool  any  = false;
#pragma unroll
                for (int s = 0; s < 4; s++)
                {
                    if (w4[s] == 0.0f) continue;
                    if (tap_valid(decode_tap(tr[s]), cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
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
                            const Tap t  = fetch_prev(prev, px, py);
                            if (tap_valid(t, cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
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
                // neighborhood_mean: rows ly .. ly+16 of the per-row 17-wide counts (separable: 3 popcll per thread instead of 17)
                int cnt = 0;
#pragma unroll
                for (int r = 0; r < 17; r++) cnt += s_h[ly + r][lx];
                const float mean = __fdiv_rn((float)cnt, 289.0f * (float)spp);
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

#define TEMPORAL_COUNT_PARAMS                                                                                                           \
    GBufLevelDev cur, GBufLevelDev prev, const uint8_t* __restrict__ count, int spp, const HistPeers hp, FrameConsts fc, float alpha_p, \
        float moments_alpha_p, void* __restrict__ out_img, void* __restrict__ out_aux, uint8_t* __restrict__ tile_flags, int row0, int row1
template <int MODE>
__global__ void __launch_bounds__(256, 4) k_temporal_count(TEMPORAL_COUNT_PARAMS)
{
    temporal_count<MODE, false>(cur, prev, count, spp, hp, fc, alpha_p, moments_alpha_p, out_img, out_aux, tile_flags, row0, row1);
}
template <int MODE>
__global__ void __launch_bounds__(256, 4) k_temporal_count_peer(TEMPORAL_COUNT_PARAMS)
{
    temporal_count<MODE, true>(cur, prev, count, spp, hp, fc, alpha_p, moments_alpha_p, out_img, out_aux, tile_flags, row0, row1);
}
#undef TEMPORAL_COUNT_PARAMS

} // namespace

void launch_shadows_temporal(const GBufLevelDev& cur, const GBufLevelDev& prev, const uint32_t* mask, const HistPeers& hist, const FrameConsts& fc, float alpha,
                             float moments_alpha, __half2* out, uint2* moments_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    dim3 grid((cur.W + 31) / 32, (row1 - row0 + 7) / 8);
    if (hist.world > 1) k_temporal<0, true><<<grid, 256, 0, st>>>(cur, prev, mask, hist, fc, alpha, moments_alpha, out, moments_out, tile_flags, row0, row1);
    else k_temporal<0, false><<<grid, 256, 0, st>>>(cur, prev, mask, hist, fc, alpha, moments_alpha, out, moments_out, tile_flags, row0, row1);
}

void launch_ao_temporal(const GBufLevelDev& cur, const GBufLevelDev& prev, const uint32_t* mask, const HistPeers& hist, const FrameConsts& fc, float alpha,
                        __half* out, __half* len_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    dim3 grid((cur.W + 31) / 32, (row1 - row0 + 7) / 8);
    if (hist.world > 1) k_temporal<1, true><<<grid, 256, 0, st>>>(cur, prev, mask, hist, fc, alpha, 0.0f, out, len_out, tile_flags, row0, row1);
    else k_temporal<1, false><<<grid, 256, 0, st>>>(cur, prev, mask, hist, fc, alpha, 0.0f, out, len_out, tile_flags, row0, row1);
}

void launch_shadows_temporal_count(const GBufLevelDev& cur, const GBufLevelDev& prev, const uint8_t* count, int spp, const HistPeers& hist, const FrameConsts& fc,
                                   float alpha, float moments_alpha, __half2* out, uint2* moments_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    dim3 grid((cur.W + 31) / 32, (row1 - row0 + 7) / 8);
    if (hist.world > 1) k_temporal_count_peer<0><<<grid, 256, 0, st>>>(cur, prev, count, spp, hist, fc, alpha, moments_alpha, out, moments_out, tile_flags, row0, row1);
    else k_temporal_count<0><<<grid, 256, 0, st>>>(cur, prev, count, spp, hist, fc, alpha, moments_alpha, out, moments_out, tile_flags, row0, row1);
}

void launch_ao_temporal_count(const GBufLevelDev& cur, const GBufLevelDev& prev, const uint8_t* count, int spp, const HistPeers& hist, const FrameConsts& fc,
                              float alpha, __half* out, __half* len_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    dim3 grid((cur.W + 31) / 32, (row1 - row0 + 7) / 8);
    if (hist.world > 1) k_temporal_count_peer<1><<<grid, 256, 0, st>>>(cur, prev, count, spp, hist, fc, alpha, 0.0f, out, len_out, tile_flags, row0, row1);
    else k_temporal_count<1><<<grid, 256, 0, st>>>(cur, prev, count, spp, hist, fc, alpha, 0.0f, out, len_out, tile_flags, row0, row1);
}
