// trace.cu — software BVH traversal + the two mask-producing ray-trace kernels.
//   K1  shadows/shadows_ray_trace.comp:89-132   (1 soft-shadow ray / pixel -> 1 bit)
//   K7  ao/ao_ray_trace.comp:90-126             (1 cosine-lobe AO ray / pixel -> 1 bit)
// With spp > 1 the same kernels trace spp rays per pixel into an 8-bit count image instead (their COUNT form).
// Ray queries replace rayQueryEXT (ray_query.glsl:6-59): any-hit, t in (t_min, t_max), opaque, no culling.
//
// BUILD NOTE: this file is compiled with -fmad=false: the mask chain (det_math.cuh + ray_triangle below) is specified
// without implicit FMA contraction so that the packed visibility mask is bit-exact against the CPU oracle.  The slab
// test uses explicit fmaf (it only has to be conservative, the boxes are padded at build time).
//
// Mapping: one warp = one 8x4 pixel block = one mask word (bit = lane = (y&3)*8 + (x&7), exactly
// gl_LocalInvocationIndex of the reference's 8x4 workgroup), so the word is a single __ballot_sync.

#include "mask_px.cuh"
#include <type_traits>

namespace {

using det::V3;
using namespace trv;

__device__ __forceinline__ float2 load_oct_normal(const uint2* gb2, size_t idx)
{
    const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(gb2 + idx)); // first two halves = oct normal
    const __half2  h = *reinterpret_cast<const __half2*>(&w);
    return __half22float2(h);
}

// rays a pixel traced: a flag when it traces one ray, a count when it traces spp
template <bool MULTI> using Traced = std::conditional_t<MULTI, uint32_t, bool>;
__device__ __forceinline__ void add_traced(bool& traced) { traced = true; }
__device__ __forceinline__ void add_traced(uint32_t& n_traced) { n_traced++; }
__device__ __forceinline__ uint32_t rays_traced(bool traced) { return traced ? 1u : 0u; }
__device__ __forceinline__ uint32_t rays_traced(uint32_t n_traced) { return n_traced; }

// one pixel of K1 (MODE 0) / K7 (MODE 1): the number of rays that reached the light / left the AO radius unoccluded.
// MULTI = false: one ray with sample index num_frames.  MULTI = true (spp > 1, SURVEY.md §8d, not in the reference): `spp`
// rays with sample indices num_frames * spp + s.
template <int MODE, bool MULTI>
__device__ __forceinline__ uint32_t trace_pixel(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                const uint8_t* __restrict__ sr, int x, int y, int spp, Traced<MULTI>& traced)
{
    uint32_t n = 0;
    traced     = {};
    if (x < g.W && y < g.H)
    {
        const size_t idx   = (size_t)y * g.W + x;
        const float  depth = __ldg(g.depth + idx);
        if (depth != 1.0f)
        {
            const float  u = ((float)x + 0.5f) / (float)g.W, v = ((float)y + 0.5f) / (float)g.H;
            const V3     P  = det::world_position_from_depth(u, v, depth, fc.view_proj_inverse);
            const float2 e  = load_oct_normal(g.gb2, idx);
            const V3     N  = det::octohedral_to_direction(e.x, e.y);
            for (int s = 0; s < (MULTI ? spp : 1); s++)
            {
                const uint32_t si = MULTI ? fc.num_frames * (uint32_t)spp + (uint32_t)s : fc.num_frames;
                const float r0 = det::sample_blue_noise(x, y, si, 0, sobol, sr);
                const float r1 = det::sample_blue_noise(x, y, si, 1, sobol, sr);
                Ray         r;
                if (mask_ray<MODE>(fc, P, N, p0, p1, r0, r1, r)) { add_traced(traced); n += trace_any(bvh, r) ? 0u : 1u; }
            }
        }
    }
    return n;
}

// the band trace's mask rows [mrow0, mrow1) and its output: mask words of one ray per pixel, or counts of spp rays per pixel
template <bool COUNT> struct RtBand { uint32_t* mask; int mrow0, mrow1; static constexpr int spp = 1; };
template <> struct RtBand<true> { uint8_t* count; int spp, mrow0, mrow1; };

// MODE 0 = shadows (K1), 1 = AO (K7).  Block = RT_CTA_WARPS warps; warp w covers mask word (bx*RT_CTA_WARPS + w, by).
// Small CTAs on purpose: ray costs are heavy-tailed and a CTA's slot (registers) is only recycled when its slowest warp
// is done — with 8-warp CTAs the kernel ran its last ~20 % at a fraction of the occupancy.
// COUNT: the count image (one byte per pixel, 0..spp) instead of the mask, same warp <-> 8x4 block mapping.
#define RT_CTA_WARPS 2
template <int MODE, bool COUNT>
__global__ void __launch_bounds__(RT_CTA_WARPS * 32) k_ray_trace(GBufLevelDev g, BvhDev bvh, FrameConsts fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                                 const uint8_t* __restrict__ sr, const RtBand<COUNT> band)
{
    const int MW   = (g.W + 7) >> 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mx = blockIdx.x * RT_CTA_WARPS + warp, my = band.mrow0 + blockIdx.y;
    if (mx >= MW || my >= band.mrow1) return; // whole warp exits together
    const int      x = mx * 8 + (lane & 7), y = my * 4 + (lane >> 3);
    Traced<COUNT>  traced;
    const uint32_t n = trace_pixel<MODE, COUNT>(g, bvh, fc, p0, p1, sobol, sr, x, y, band.spp, traced);
    if constexpr (COUNT)
    {
        if (x < g.W && y < g.H) band.count[(size_t)y * g.W + x] = (uint8_t)n;
    }
    else
    {
        const uint32_t word = __ballot_sync(0xFFFFFFFFu, n != 0);
        if (lane == 0) band.mask[(size_t)my * MW + mx] = word;
    }
    count_rays(fc.ray_ctr, 0, rays_traced(traced));
}

// Multi-GPU variant (shard.cu, "cooperative ray trace"): this rank traces mask rows [bounds[self], bounds[self+1]) — a
// partition of the WHOLE image balanced on last frame's measured cost, read from device memory, so the host never needs
// to know it: the launch grid covers the largest share the partition kernel may hand out (hr_rt_share_cap) and CTAs past
// the end of the share exit at once (measured alternatives, both ~14 % slower on one GPU: a persistent job loop over an
// atomic counter, and walking the share's rows most-expensive-first — the row-major walk keeps neighbouring rows, i.e.
// the same BVH nodes and G-buffer sectors, in flight together).  Mask words go to this rank's own mask image, or with
// COUNT the pixels' counts to its count image `count`; k_rt_push (shard.cu) then copies the share to every peer with wide
// stores.  trace_pixel is the function of k_ray_trace, so the results equal the single-GPU ones bit for bit.  Each warp
// adds its duration to its mask row's cost, the input of the next partition: a COUNT warp's duration grows about linearly
// with spp, so it is added in units of 2^cost_shift cycles, cost_shift = 6 + ceil(log2 spp): the row sums stay in the range
// of the 1-spp trace (scaling every row alike leaves the partition unchanged) and cannot overflow at spp <= 255.
template <int MODE, bool COUNT>
__global__ void __launch_bounds__(RT_CTA_WARPS * 32) k_ray_trace_shared(GBufLevelDev g, BvhDev bvh, FrameConsts fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                                        const uint8_t* __restrict__ sr, uint8_t* __restrict__ count, int spp, int cost_shift, RtShare sh)
{
    const long long t0 = clock64();
    const int MW   = (g.W + 7) >> 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mrow0 = __ldg(sh.bounds + sh.self), mrow1 = __ldg(sh.bounds + sh.self + 1);
    const int mx = blockIdx.x * RT_CTA_WARPS + warp, my = mrow0 + blockIdx.y;
    if (mx >= MW || my >= mrow1) return; // whole warp exits together
    const int      x = mx * 8 + (lane & 7), y = my * 4 + (lane >> 3);
    Traced<COUNT>  traced;
    const uint32_t n = trace_pixel<MODE, COUNT>(g, bvh, fc, p0, p1, sobol, sr, x, y, spp, traced);
    if constexpr (COUNT)
    {
        if (x < g.W && y < g.H) count[(size_t)y * g.W + x] = (uint8_t)n;
        __syncwarp();
        if (lane == 0) atomicAdd(sh.cost_acc + my, (uint32_t)((clock64() - t0) >> cost_shift) + 1u);
    }
    else
    {
        const uint32_t word = __ballot_sync(0xFFFFFFFFu, n != 0);
        if (lane == 0)
        {
            sh.mask_local[(size_t)my * MW + mx] = word;
            atomicAdd(sh.cost_acc + my, (uint32_t)((clock64() - t0) >> 6) + 1u);
        }
    }
    count_rays(fc.ray_ctr, 0, rays_traced(traced));
}

__global__ void k_trace_any(BvhDev bvh, const float* __restrict__ rays, size_t n, uint32_t* __restrict__ out)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = rays + 8 * i;
    Ray          r;
    r.o = det::mk(p[0], p[1], p[2]); r.tmin = p[3];
    r.d = det::mk(p[4], p[5], p[6]); r.tmax = p[7];
    out[i] = trace_any(bvh, r) ? 1u : 0u;
}

__global__ void k_trace_closest(BvhDev bvh, const float* __restrict__ rays, size_t n, float* __restrict__ out_t, uint32_t* __restrict__ out_prim,
                                float* __restrict__ out_uv)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = rays + 8 * i;
    Ray          r;
    r.o = det::mk(p[0], p[1], p[2]); r.tmin = p[3];
    r.d = det::mk(p[4], p[5], p[6]); r.tmax = p[7];
    float    t, u, v;
    uint32_t prim;
    trace_closest(bvh, r, t, prim, u, v);
    out_t[i]    = t;
    out_prim[i] = prim;
    if (out_uv) { out_uv[2 * i] = u; out_uv[2 * i + 1] = v; }
}

} // namespace

static inline dim3 mask_grid(int W, int mrow0, int mrow1) { return dim3(((W + 7) / 8 + RT_CTA_WARPS - 1) / RT_CTA_WARPS, mrow1 - mrow0, 1); }

// kind: PASS_SHADOWS (K1, p0 = bias) or PASS_AO (K7, p0 = ray length, p1 = bias); into `mask` at spp 1, into `count` at spp > 1
void launch_ray_trace(int kind, const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* sobol, const uint8_t* sr,
                      uint32_t* mask, uint8_t* count, int spp, int row0, int row1, cudaStream_t st)
{
    const int mrow0 = row0 / 4, mrow1 = (row1 + 3) / 4;
    if (mrow1 <= mrow0) return;
    const dim3 grid = mask_grid(g.W, mrow0, mrow1);
    if (spp > 1)
    {
        const auto k = kind == PASS_AO ? k_ray_trace<1, true> : k_ray_trace<0, true>;
        k<<<grid, RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, p0, p1, sobol, sr, RtBand<true> { count, spp, mrow0, mrow1 });
    }
    else
    {
        const auto k = kind == PASS_AO ? k_ray_trace<1, false> : k_ray_trace<0, false>;
        k<<<grid, RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, p0, p1, sobol, sr, RtBand<false> { mask, mrow0, mrow1 });
    }
}

// the grid covers the largest share hr_rt_wait_partition may hand to one rank; mask words go to sh.mask_local, counts to `count`
void launch_ray_trace_shared(int kind, const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* sobol,
                             const uint8_t* sr, uint8_t* count, int spp, const RtShare& sh, cudaStream_t st)
{
    int cost_shift = 6;
    while ((1 << (cost_shift - 6)) < spp) cost_shift++;
    const dim3 grid(((g.W + 7) / 8 + RT_CTA_WARPS - 1) / RT_CTA_WARPS, hr_rt_share_cap((g.H + 3) / 4, sh.world), 1);
    const auto k = kind == PASS_AO ? (spp > 1 ? k_ray_trace_shared<1, true> : k_ray_trace_shared<1, false>)
                                   : (spp > 1 ? k_ray_trace_shared<0, true> : k_ray_trace_shared<0, false>);
    k<<<grid, RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, p0, p1, sobol, sr, count, spp, cost_shift, sh);
}

void launch_trace_any(const BvhDev& bvh, const float* rays, size_t n, uint32_t* out, cudaStream_t st)
{
    if (!n) return;
    k_trace_any<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(bvh, rays, n, out);
}

void launch_trace_closest(const BvhDev& bvh, const float* rays, size_t n, float* out_t, uint32_t* out_prim, float* out_uv, cudaStream_t st)
{
    if (!n) return;
    k_trace_closest<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(bvh, rays, n, out_t, out_prim, out_uv);
}
