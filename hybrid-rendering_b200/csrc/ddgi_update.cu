// ddgi_update.cu — DDGI probe-atlas update and per-pixel probe-grid sampling.
//   K19 gi/gi_probe_update.glsl:136-184 (irradiance 8x8 and depth 16x16 octahedral texels per probe, hysteresis blend)
//   K20 gi/gi_border_update.glsl:151-175 (1-texel gutter of every probe from the g_offsets tables :35-143)
//   K21 gi/gi_sample_probe_grid.comp:75-99 + gi_common.glsl:188-320
// K19 and K20 are fused: one CTA owns one probe, writes its interior texels, then (after a CTA barrier) its gutter —
// the gutter only ever reads the same probe's interior.  All 256 rays of the probe are staged once in shared memory
// (the reference streams them in 64-ray batches).
#include "gi_common.cuh"
#include "hr_internal.h"

namespace {

using namespace gi;

__device__ __forceinline__ uint2 pack_h4(float a, float b, float c, float d)
{
    const __half2 lo = __floats2half2_rn(a, b), hi = __floats2half2_rn(c, d);
    return make_uint2(*reinterpret_cast<const uint32_t*>(&lo), *reinterpret_cast<const uint32_t*>(&hi));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b)
{
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

#define MAX_RAYS 1024

// DEPTH = false: irradiance atlas (RGBA16F, side 8); true: depth atlas (RG16F, side 16).  blockDim = side*side.
template <bool DEPTH>
__global__ void k_probe_update(hr_ddgi_uniforms d, const uint2* __restrict__ radiance, const uint2* __restrict__ dirdepth, const void* __restrict__ prev_atlas,
                               void* __restrict__ out_atlas, int first_frame, int probe0, int probe1)
{
    __shared__ float4 s_dir[MAX_RAYS];
    __shared__ float  s_rad[DEPTH ? 1 : MAX_RAYS * 3];
    const int probe = probe0 + blockIdx.x;
    if (probe >= probe1) return;
    const int side = DEPTH ? d.depth_probe_side_length : d.irradiance_probe_side_length;
    const int TW   = DEPTH ? d.depth_texture_width : d.irradiance_texture_width;
    const int R    = min(d.rays_per_probe, MAX_RAYS);
    for (int r = threadIdx.x; r < R; r += blockDim.x)
    {
        const uint2  w  = __ldg(dirdepth + (size_t)probe * d.rays_per_probe + r);
        const float2 a = h2f2(w.x), b = h2f2(w.y);
        s_dir[r] = make_float4(a.x, a.y, b.x, b.y);
        if (!DEPTH)
        {
            const uint2  q = __ldg(radiance + (size_t)probe * d.rays_per_probe + r);
            const float2 c = h2f2(q.x), e = h2f2(q.y);
            s_rad[3 * r] = c.x * 0.95f; s_rad[3 * r + 1] = c.y * 0.95f; s_rad[3 * r + 2] = e.x * 0.95f; // energy_conservation
        }
    }
    __syncthreads();
    const int ppr = (TW - 2) / (side + 2);
    const int wx = probe % ppr, wy = probe / ppr;
    const int lx = threadIdx.x % side, ly = threadIdx.x / side;
    if (ly < side)
    {
        const int    cx = wx * (side + 2) + 2 + lx, cy = wy * (side + 2) + 2 + ly; // current_coord :138
        const float3 tdir = oct_decode(make_float2(((float)lx + 0.5f) * (2.0f / (float)side) - 1.0f, ((float)ly + 0.5f) * (2.0f / (float)side) - 1.0f));
        float        r0 = 0.0f, r1 = 0.0f, r2 = 0.0f, tw = 0.0f;
        for (int r = 0; r < R; r++)
        {
            const float4 rd = s_dir[r];
            const float  c  = fmaxf(0.0f, tdir.x * rd.x + tdir.y * rd.y + tdir.z * rd.z);
            if (DEPTH)
            {
                float dist = fminf(d.max_distance, rd.w - 0.01f);
                if (dist == -1.0f) dist = d.max_distance;
                const float w = c <= 0.0f ? 0.0f : __expf(d.depth_sharpness * __logf(c));
                if (w >= 0.00000001f) { r0 += dist * w; r1 += (dist * dist) * w; tw += w; }
            }
            else if (c >= 0.00000001f)
            {
                r0 += s_rad[3 * r] * c; r1 += s_rad[3 * r + 1] * c; r2 += s_rad[3 * r + 2] * c;
                tw += c;
            }
        }
        if (tw > 0.00000001f) { const float inv = 1.0f / tw; r0 *= inv; r1 *= inv; r2 *= inv; }
        const size_t ti = (size_t)cy * TW + cx;
        if (DEPTH)
        {
            if (!first_frame)
            {
                const float2 pv = h2f2(__ldg(reinterpret_cast<const uint32_t*>(prev_atlas) + ti));
                r0 = r0 * (1.0f - d.hysteresis) + pv.x * d.hysteresis;
                r1 = r1 * (1.0f - d.hysteresis) + pv.y * d.hysteresis;
            }
            reinterpret_cast<uint32_t*>(out_atlas)[ti] = pack_h2(r0, r1);
        }
        else
        {
            if (!first_frame)
            {
                const uint2  pw = __ldg(reinterpret_cast<const uint2*>(prev_atlas) + ti);
                const float2 pa = h2f2(pw.x), pb = h2f2(pw.y);
                r0 = r0 * (1.0f - d.hysteresis) + pa.x * d.hysteresis;
                r1 = r1 * (1.0f - d.hysteresis) + pa.y * d.hysteresis;
                r2 = r2 * (1.0f - d.hysteresis) + pb.x * d.hysteresis;
            }
            reinterpret_cast<uint2*>(out_atlas)[ti] = pack_h4(r0, r1, r2, 1.0f);
        }
    }
    // ---- K20: gutter of this probe (gi_border_update.glsl).  g_offsets pattern: rows mirror x, columns mirror y, corners
    // take the opposite interior corner.  4*side + 4 texels.
    __syncthreads();
    const int S = side, bx = wx * (S + 2) + 1, by = wy * (S + 2) + 1;
    for (int k = threadIdx.x; k < 4 * S + 4; k += blockDim.x)
    {
        int sx, sy, dx, dy;
        if (k < 4 * S)
        {
            const int e = k / S, i = k % S + 1;
            if (e == 0) { sx = S + 1 - i; sy = 1; dx = i; dy = 0; }
            else if (e == 1) { sx = S + 1 - i; sy = S; dx = i; dy = S + 1; }
            else if (e == 2) { sx = 1; sy = S + 1 - i; dx = 0; dy = i; }
            else { sx = S; sy = S + 1 - i; dx = S + 1; dy = i; }
        }
        else
        {
            const int c = k - 4 * S;
            sx = (c == 0 || c == 2) ? S : 1; sy = (c == 0 || c == 1) ? S : 1;
            dx = (c == 0 || c == 2) ? 0 : S + 1; dy = (c == 0 || c == 1) ? 0 : S + 1;
        }
        const size_t si = (size_t)(by + sy) * TW + bx + sx, di = (size_t)(by + dy) * TW + bx + dx;
        if (DEPTH) reinterpret_cast<uint32_t*>(out_atlas)[di] = reinterpret_cast<uint32_t*>(out_atlas)[si];
        else reinterpret_cast<uint2*>(out_atlas)[di] = reinterpret_cast<uint2*>(out_atlas)[si];
    }
}

// K21
__global__ void __launch_bounds__(256) k_sample_probe_grid(GBufLevelDev g, FrameConsts fc, hr_ddgi_uniforms d, AtlasDev at, float gi_intensity, uint2* __restrict__ out,
                                                            int row0, int row1)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= g.W || y >= g.H || y >= row1) return;
    const size_t idx   = (size_t)y * g.W + x;
    const float  depth = __ldg(g.depth + idx);
    if (depth == 1.0f) { out[idx] = make_uint2(0u, 0u); return; }
    const float  u = ((float)x + 0.5f) / (float)g.W, v = ((float)y + 0.5f) / (float)g.H;
    // world_position_from_depth (common.glsl:169-184) rounded as the reference rounds it: ((m0r*x + m1r*y) + m2r*z) + m3r, no
    // contraction, then an IEEE division by w.  Near the far plane w = m11*depth + m15 cancels (by ~100x at near 0.1 / far 100),
    // so fused products and an approximate reciprocal moved P far enough to change the probe visibility weights.
    const float* M  = fc.view_proj_inverse;
    const float  sx = u * 2.0f - 1.0f, sy = v * 2.0f - 1.0f;
    auto         row = [&](int r) { return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[r], sx), __fmul_rn(M[4 + r], sy)), __fmul_rn(M[8 + r], depth)), M[12 + r]); };
    const float  w  = row(3);
    const float3 P  = f3(__fdiv_rn(row(0), w), __fdiv_rn(row(1), w), __fdiv_rn(row(2), w));
    const float2 e  = h2f2(__ldg(reinterpret_cast<const uint32_t*>(g.gb2 + idx)));
    float3       N  = f3(e.x, e.y, 1.0f - fabsf(e.x) - fabsf(e.y));
    if (N.z < 0.0f)
    {
        const float nx = (1.0f - fabsf(N.y)) * (N.x < 0.0f ? -1.0f : 1.0f), ny = (1.0f - fabsf(N.x)) * (N.y < 0.0f ? -1.0f : 1.0f);
        N.x = nx;
        N.y = ny;
    }
    N = normalize(N);
    const float3 Wo = normalize(f3(fc.cam_pos[0], fc.cam_pos[1], fc.cam_pos[2]) - P);
    const float3 ir = sample_irradiance<8>(d, at, P, N, Wo) * gi_intensity;
    out[idx] = pack_h4(ir.x, ir.y, ir.z, 1.0f);
}

} // namespace

void launch_ddgi_probe_update(const hr_ddgi_uniforms& d, const void* radiance, const void* dirdepth, const void* prev_irr, const void* prev_depth, void* out_irr,
                              void* out_depth, int first_frame, int probe0, int probe1, cudaStream_t st)
{
    if (probe1 <= probe0) return;
    k_probe_update<false><<<probe1 - probe0, d.irradiance_probe_side_length * d.irradiance_probe_side_length, 0, st>>>(
        d, (const uint2*)radiance, (const uint2*)dirdepth, prev_irr, out_irr, first_frame, probe0, probe1);
    k_probe_update<true><<<probe1 - probe0, d.depth_probe_side_length * d.depth_probe_side_length, 0, st>>>(d, (const uint2*)radiance, (const uint2*)dirdepth,
                                                                                                        prev_depth, out_depth, first_frame, probe0, probe1);
}

void launch_ddgi_sample_probe_grid(const GBufLevelDev& g, const FrameConsts& fc, const hr_ddgi_uniforms& d, const void* irr, const void* depth, float gi_intensity,
                                   void* out, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    AtlasDev at { (const uint2*)irr, (const uint32_t*)depth };
    dim3     grid((g.W + 31) / 32, (row1 - row0 + 7) / 8);
    k_sample_probe_grid<<<grid, 256, 0, st>>>(g, fc, d, at, gi_intensity, (uint2*)out, row0, row1);
}
