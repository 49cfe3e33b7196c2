// svgf_reflections.cu — SVGF stages of the reflections pass (RGBA16F images: rgb + variance).
//   K14 reflections/reflections_denoise_reprojection.comp:174-289 (+ reprojection.glsl:78-111,115-328 REPROJECTION_REFLECTIONS)
//   K15 reflections/reflections_denoise_copy_tiles.comp:35-38 (folded into K16 through the tile-flag byte)
//   K16 reflections/reflections_denoise_atrous.comp:94-181   (algorithmic 36 B/px/iteration, SURVEY.md §8d)
//   K17 reflections/reflections_upsample.comp:62-109
#include "glsl_fast.cuh"
#include "hr_internal.h"

namespace {

using namespace gf;

__device__ __forceinline__ bool inside(int x, int y, int W, int H) { return x >= 0 && y >= 0 && x < W && y < H; }
__device__ __forceinline__ float luminance(float r, float g, float b) { return fmaxf(r * 0.299f + g * 0.587f + b * 0.114f, 0.0001f); }
__device__ __forceinline__ uint2 pack_h4(float a, float b, float c, float d) { return make_uint2(f2_to_h2(a, b), f2_to_h2(c, d)); }

struct Tap { float3 n; float mesh_id; float depth; };
__device__ __forceinline__ Tap fetch_prev(const GBufLevelDev& p, int x, int y)
{
    Tap t;
    if (inside(x, y, p.W, p.H))
    {
        const size_t i  = (size_t)y * p.W + x;
        const float2 e  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(p.gb2 + i)));
        const float2 g3 = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(p.gb3 + i) + 1));
        t.n = octohedral_to_direction(e.x, e.y);
        t.mesh_id = g3.x;
        t.depth   = __ldg(p.depth + i);
    }
    else { t.n = octohedral_to_direction(0.0f, 0.0f); t.mesh_id = 0.0f; t.depth = 0.0f; }
    return t;
}
__device__ __forceinline__ bool tap_valid(const Tap& t, float3 cur_pos, float3 cur_n, float cur_mesh, float hu, float hv, const float* vpi)
{
    if (!(cur_mesh == t.mesh_id)) return false;
    const float3 hp = world_position_from_depth(hu, hv, t.depth, vpi);
    const float3 d  = make_float3(cur_pos.x - hp.x, cur_pos.y - hp.y, cur_pos.z - hp.z);
    if (fabsf(dot3(d, cur_n)) > 5.0f) return false;
    const float nd = fabsf(dot3(cur_n, t.n));
    return nd * nd > 0.1f;
}

struct ReflTemporalParams { float alpha, moments_alpha; int approximate_with_ddgi; int row0, row1; int rot; }; // rot: the last `rot` tile rows are scheduled first

// ---- history fetches through the owner table (HistPeers, hr_internal.h; see svgf_temporal.cu) ----
__device__ __forceinline__ int owner_of(const HistPeers& hp, int row)
{
    int o = 0;
#pragma unroll
    for (int r = 0; r < HR_MAX_RANKS - 1; r++) o += (r < hp.world - 1 && row >= hp.band_end[r]) ? 1 : 0;
    return o;
}
// All history taps of a pixel lie in rows hcy-1 .. hcy+1: the owner is looked up once per pixel (two owner_of calls) and only
// pixels whose taps straddle a band border fall back to a lookup per load.
struct OwnerCache { int o; bool uniform; };
template <bool PEER>
__device__ __forceinline__ OwnerCache owner_cache(const HistPeers& hp, int row_lo, int row_hi)
{
    OwnerCache c { 0, true };
    if (PEER) { c.o = owner_of(hp, row_lo); c.uniform = c.o == owner_of(hp, row_hi); }
    return c;
}
template <bool PEER>
__device__ __forceinline__ uint2 hist_ld64(const void* const* tab, const HistPeers& hp, const OwnerCache& oc, int row, size_t index)
{
    if (hp.no_history) return make_uint2(0u, 0u);
    if (!PEER) return __ldg(reinterpret_cast<const uint2*>(tab[0]) + index);
    const int    o = oc.uniform ? oc.o : owner_of(hp, row);
    const uint2* p = reinterpret_cast<const uint2*>(tab[o]) + index;
    return o == hp.self ? __ldg(p) : __ldcg(p);
}
template <bool PEER>
__device__ __forceinline__ uint32_t hist_ld32(const void* const* tab, const HistPeers& hp, const OwnerCache& oc, int row, size_t word_index)
{
    if (hp.no_history) return 0u;
    if (!PEER) return __ldg(reinterpret_cast<const uint32_t*>(tab[0]) + word_index);
    const int       o = oc.uniform ? oc.o : owner_of(hp, row);
    const uint32_t* p = reinterpret_cast<const uint32_t*>(tab[o]) + word_index;
    return o == hp.self ? __ldg(p) : __ldcg(p);
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
            const float3 cn = octohedral_to_direction(g2.x, g2.y);
            const float  cmesh = g3.z, curvature = g3.y;
            const float3 cpos = world_position_from_depth(tu, tv, depth, fc.view_proj_inverse);
            // compute_history_coord, reprojection.glsl:101-111
            float hfx = rn_mad(g2.z, fw, (float)x), hfy = rn_mad(g2.w, fh, (float)y);
            if (ray_length > 0.0f && curvature == 0.0f)
            { // virtual_point_reprojection :78-97 — exactly rounded: it lands on texel corners for a static camera
                const float2 vp = rn_virtual_point_reprojection(x, y, fw, fh, depth, ray_length, fc.cam_pos, fc.view_proj_inverse, fc.prev_view_proj);
                hfx = vp.x;
                hfy = vp.y;
            }
            const int   hcx = (int)hfx, hcy = (int)hfy; // ivec2(reprojected_coord) :171
            const float hu = tu + g2.z, hv = tv + g2.w;
            const bool  in_frame = inside(hcx, hcy, W, H);
            const OwnerCache oc = owner_cache<PEER>(hp, max(hcy - 1, 0), min(hcy + 1, H - 1));
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
                    if (w4[s] == 0.0f) continue; // exact: see svgf_temporal.cu
                    const int px = hcx + (s & 1), py = hcy + (s >> 1);
                    const Tap t  = fetch_prev(prev, px, py);
                    if (tap_valid(t, cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
                    {
                        any = true;
                        if (inside(px, py, W, H))
                        {
                            const size_t pi = (size_t)py * W + px;
                            const float4 hv4 = h4_to_f4(hist_ld64<PEER>(hp.img, hp, oc, py, pi));
                            const float2 mm  = h2_to_f2(hist_ld32<PEER>(hp.aux, hp, oc, py, 2 * pi));
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
                            const Tap t  = fetch_prev(prev, px, py);
                            if (tap_valid(t, cpos, cn, cmesh, hu, hv, fc.view_proj_inverse))
                            {
                                if (inside(px, py, W, H))
                                {
                                    const size_t pi = (size_t)py * W + px;
                                    const float4 hv4 = h4_to_f4(hist_ld64<PEER>(hp.img, hp, oc, py, pi));
                                    const float2 mm  = h2_to_f2(hist_ld32<PEER>(hp.aux, hp, oc, py, 2 * pi));
                                    hc[0] += hv4.x; hc[1] += hv4.y; hc[2] += hv4.z; hm0 += mm.x; hm1 += mm.y;
                                }
                                cnt += 1.0f;
                            }
                        }
                    if (cnt > 0.0f) { valid = true; const float inv = fast_rcp(cnt); hc[0] *= inv; hc[1] *= inv; hc[2] *= inv; hm0 *= inv; hm1 *= inv; }
                }
            }
            float hist_len = 0.0f;
            if (valid) hist_len = h2_to_f2(hist_ld32<PEER>(hp.aux, hp, oc, hcy, 2 * ((size_t)hcy * W + hcx) + 1)).x;
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
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, flag);
    if (lx == 0 && b) atomicOr(&s_flags, ((b & 0xFFu) ? 1u : 0u) | ((b & 0xFF00u) ? 2u : 0u) | ((b & 0xFF0000u) ? 4u : 0u) | ((b & 0xFF000000u) ? 8u : 0u));
    __syncthreads();
    if (threadIdx.x < 4)
    {
        const int tx = (x0 >> 3) + threadIdx.x, ty = y0 >> 3, TW = (W + 7) >> 3;
        if (tx < TW && y0 < H && y0 < P.row1) tile_flags[(size_t)ty * TW + tx] = (s_flags >> threadIdx.x) & 1u;
    }
}

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

struct UpParams { int W0, H0, Wm, Hm, row0, row1; };
__device__ __forceinline__ int nearest(float uv, int size) { return min(max((int)floorf(uv * (float)size), 0), size - 1); }

__global__ void __launch_bounds__(256) k_upsample_vec4(GBufLevelDev g0, GBufLevelDev gm, const uint2* __restrict__ in, UpParams P, uint2* __restrict__ out)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = P.row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= P.W0 || y >= P.H0 || y >= P.row1) return;
    const size_t idx = (size_t)y * P.W0 + x;
    const float  hz  = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g0.gb3 + idx) + 1)).y;
    if (hz == -1.0f) { out[idx] = make_uint2(0u, 0u); return; }
    const float2 he = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(g0.gb2 + idx)));
    const float3 hn = octohedral_to_direction(he.x, he.y);
    const float  tu = ((float)x + 0.5f) / (float)P.W0, tv = ((float)y + 0.5f) / (float)P.H0;
    const float  tsx = 1.0f / (float)P.Wm, tsy = 1.0f / (float)P.Hm;
    const float  kx[4] = { 0.0f, 1.0f, -1.0f, 0.0f }, ky[4] = { 1.0f, 0.0f, 0.0f, -1.0f };
    float        up[4] = { 0, 0, 0, 0 }, tw = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; i++)
    {
        const int    cx = nearest(tu + kx[i] * tsx, P.Wm), cy = nearest(tv + ky[i] * tsy, P.Hm);
        const size_t ci = (size_t)cy * P.Wm + cx;
        const float  cz = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(gm.gb3 + ci) + 1)).y;
        if (cz == -1.0f) continue;
        const float2 ce = h2_to_f2(__ldg(reinterpret_cast<const uint32_t*>(gm.gb2 + ci)));
        const float3 cn = octohedral_to_direction(ce.x, ce.y);
        const float  w  = __expf(-1.0f - __expf(-fabsf(hz - cz))) * pow32(fminf(fmaxf(dot3(hn, cn), 0.0f), 1.0f));
        const float4 v  = h4_to_f4(__ldg(in + ci));
        up[0] += v.x * w; up[1] += v.y * w; up[2] += v.z * w; up[3] += v.w * w;
        tw += w;
    }
    const float inv = 1.0f / fmaxf(tw, 0.00000001f);
    out[idx] = pack_h4(up[0] * inv, up[1] * inv, up[2] * inv, up[3] * inv);
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

} // namespace

int g_hr_force_peer_temporal = 0; // hr_debug_set(12, 1): run the peer-history variant of K14 on one GPU (overhead A/B of the owner lookups)

void launch_reflections_temporal(const GBufLevelDev& cur, const GBufLevelDev& prev, const void* input, const HistPeers& hist, const FrameConsts& fc, float alpha,
                                 float moments_alpha, int approximate_with_ddgi, void* out, void* mom_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    dim3               grid((cur.W + 31) / 32, (row1 - row0 + 7) / 8);
    int                rot = 0;
    if (hist.world > 1 && hist.self < hist.world - 1) rot = (row1 - hist.band_end[hist.self] + 7) / 8; // tile rows below this rank's band
    if (rot < 0 || rot >= (int)grid.y) rot = 0;
    ReflTemporalParams P { alpha, moments_alpha, approximate_with_ddgi, row0, row1, rot };
    if (hist.world > 1 || g_hr_force_peer_temporal) k_refl_temporal<true><<<grid, 256, 0, st>>>(cur, prev, (const uint2*)input, hist, fc, P, (uint2*)out, (uint2*)mom_out, tile_flags);
    else k_refl_temporal<false><<<grid, 256, 0, st>>>(cur, prev, (const uint2*)input, hist, fc, P, (uint2*)out, (uint2*)mom_out, tile_flags);
}

bool launch_reflections_atrous_v2(const GBufLevelDev& g, const void* in, const uint8_t* tile_flags, int radius, int step, float phi_color, float phi_normal,
                                  float sigma_depth, int approximate_with_ddgi, void* out, int row0, int row1, unsigned int* counters, cudaStream_t st); // svgf_refl_atrous_v2.cu

int launch_reflections_atrous(const GBufLevelDev& g, const void* in, const uint8_t* tile_flags, int radius, int step, float phi_color, float phi_normal,
                              float sigma_depth, int approximate_with_ddgi, void* out, int row0, int row1, unsigned int* counters, cudaStream_t st)
{
    if (row1 <= row0) return 0;
    if (launch_reflections_atrous_v2(g, in, tile_flags, radius, step, phi_color, phi_normal, sigma_depth, approximate_with_ddgi, out, row0, row1, counters, st)) return 0; // packed fp32x2
    if (radius != 1 || !(step == 1 || step == 2 || step == 4 || step == 8 || step == 16)) return -1;
    ReflAtrousParams P { g.W, g.H, step, radius, phi_color, phi_normal, sigma_depth, approximate_with_ddgi, row0, row1 };
    switch (step)
    {
        case 1: launch_atrous_t<1>(g, (const uint2*)in, tile_flags, P, (uint2*)out, st); break;
        case 2: launch_atrous_t<2>(g, (const uint2*)in, tile_flags, P, (uint2*)out, st); break;
        case 4: launch_atrous_t<4>(g, (const uint2*)in, tile_flags, P, (uint2*)out, st); break;
        case 8: launch_atrous_t<8>(g, (const uint2*)in, tile_flags, P, (uint2*)out, st); break;
        default: launch_atrous_t<16>(g, (const uint2*)in, tile_flags, P, (uint2*)out, st); break;
    }
    return 0;
}

bool launch_upsample_vec4_v2(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, void* out, int row0, int row1, cudaStream_t st); // svgf_misc_v2.cu

void launch_upsample_vec4(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, void* out, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    if (launch_upsample_vec4_v2(g0, gm, in, out, row0, row1, st)) return; // shared-memory staged variant
    UpParams P { g0.W, g0.H, gm.W, gm.H, row0, row1 };
    dim3     grid((g0.W + 31) / 32, (row1 - row0 + 7) / 8);
    k_upsample_vec4<<<grid, 256, 0, st>>>(g0, gm, (const uint2*)in, P, (uint2*)out);
}
