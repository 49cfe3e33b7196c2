// trace.cu — software BVH traversal + the two mask-producing ray-trace kernels.
//   K1  shadows/shadows_ray_trace.comp:89-132   (1 soft-shadow ray / pixel -> 1 bit)
//   K7  ao/ao_ray_trace.comp:90-126             (1 cosine-lobe AO ray / pixel -> 1 bit)
// Ray queries replace rayQueryEXT (ray_query.glsl:6-59): any-hit, t in (t_min, t_max), opaque, no culling.
//
// BUILD NOTE: this file is compiled with -fmad=false: the mask chain (det_math.cuh + ray_triangle below) is specified
// without implicit FMA contraction so that the packed visibility mask is bit-exact against the CPU oracle.  The slab
// test uses explicit fmaf (it only has to be conservative, the boxes are padded at build time).
//
// Mapping: one warp = one 8x4 pixel block = one mask word (bit = lane = (y&3)*8 + (x&7), exactly
// gl_LocalInvocationIndex of the reference's 8x4 workgroup), so the word is a single __ballot_sync.

#include "traverse.cuh"

namespace {

using det::V3;
using namespace trv;

__device__ __forceinline__ float2 load_oct_normal(const uint2* gb2, size_t idx)
{
    const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(gb2 + idx)); // first two halves = oct normal
    const __half2  h = *reinterpret_cast<const __half2*>(&w);
    return __half22float2(h);
}

// one pixel of K1 (MODE 0) / K7 (MODE 1): 1 = the ray reached the light / left the AO radius unoccluded
template <int MODE>
__device__ __forceinline__ uint32_t trace_pixel(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                const uint8_t* __restrict__ sr, int x, int y, bool& traced)
{
    uint32_t result = 0;
    traced          = false;
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
            const float  r0 = det::sample_blue_noise(x, y, fc.num_frames, 0, sobol, sr);
            const float  r1 = det::sample_blue_noise(x, y, fc.num_frames, 1, sobol, sr);
            Ray          r;
            r.tmin = 0.01f;
            if (MODE == 0)
            {
                r.o = det::add(P, det::scale(N, p0)); // bias
                float att;
                det::fetch_light_properties_shadow(fc.light, P, N, r0, r1, r.d, r.tmax, att);
                if (att > 0.0f) { traced = true; result = trace_any(bvh, r) ? 0u : 1u; }
            }
            else
            {
                r.o    = det::add(P, det::scale(N, p1)); // bias
                r.d    = det::sample_cosine_lobe(N, r0, r1);
                r.tmax = p0; // ray_length
                traced = true;
                result = trace_any(bvh, r) ? 0u : 1u;
            }
        }
    }
    return result;
}

// MODE 0 = shadows (K1), 1 = AO (K7).  Block = RT_CTA_WARPS warps; warp w covers mask word (bx*RT_CTA_WARPS + w, by).
// Small CTAs on purpose: ray costs are heavy-tailed and a CTA's slot (registers) is only recycled when its slowest warp
// is done — with 8-warp CTAs the kernel ran its last ~20 % at a fraction of the occupancy.
#define RT_CTA_WARPS 2
template <int MODE>
__global__ void __launch_bounds__(RT_CTA_WARPS * 32) k_ray_trace_mask(GBufLevelDev g, BvhDev bvh, FrameConsts fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                         const uint8_t* __restrict__ sr, uint32_t* __restrict__ mask, int mrow0, int mrow1)
{
    const int MW   = (g.W + 7) >> 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mx = blockIdx.x * RT_CTA_WARPS + warp, my = mrow0 + blockIdx.y;
    if (mx >= MW || my >= mrow1) return; // whole warp exits together
    const int      x = mx * 8 + (lane & 7), y = my * 4 + (lane >> 3);
    bool           traced;
    const uint32_t result = trace_pixel<MODE>(g, bvh, fc, p0, p1, sobol, sr, x, y, traced);
    const uint32_t word   = __ballot_sync(0xFFFFFFFFu, result != 0);
    if (lane == 0) mask[(size_t)my * MW + mx] = word;
    count_rays(fc.ray_ctr, 0, traced ? 1u : 0u);
}

// spp > 1 (SURVEY.md §8d, not in the reference): `spp` rays per pixel with sample index num_frames * spp + s; returns the number
// of unoccluded rays.  Separate from trace_pixel so the 1-spp kernels stay exactly what the parity runs validated.
template <int MODE>
__device__ __forceinline__ uint32_t trace_pixel_spp(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                    const uint8_t* __restrict__ sr, int x, int y, int spp, uint32_t& n_traced)
{
    uint32_t n = 0;
    n_traced   = 0;
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
            for (int s = 0; s < spp; s++)
            {
                const uint32_t si = fc.num_frames * (uint32_t)spp + (uint32_t)s;
                const float r0 = det::sample_blue_noise(x, y, si, 0, sobol, sr);
                const float r1 = det::sample_blue_noise(x, y, si, 1, sobol, sr);
                Ray         r;
                r.tmin = 0.01f;
                if (MODE == 0)
                {
                    r.o = det::add(P, det::scale(N, p0)); // bias
                    float att;
                    det::fetch_light_properties_shadow(fc.light, P, N, r0, r1, r.d, r.tmax, att);
                    if (att > 0.0f) { n_traced++; n += trace_any(bvh, r) ? 0u : 1u; }
                }
                else
                {
                    r.o    = det::add(P, det::scale(N, p1)); // bias
                    r.d    = det::sample_cosine_lobe(N, r0, r1);
                    r.tmax = p0; // ray_length
                    n_traced++;
                    n += trace_any(bvh, r) ? 0u : 1u;
                }
            }
        }
    }
    return n;
}

// count image: one byte per pixel (0..spp); same warp <-> 8x4 block mapping as the mask kernels
template <int MODE>
__global__ void __launch_bounds__(RT_CTA_WARPS * 32) k_ray_trace_count(GBufLevelDev g, BvhDev bvh, FrameConsts fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                                          const uint8_t* __restrict__ sr, uint8_t* __restrict__ count, int spp, int mrow0, int mrow1)
{
    const int MW   = (g.W + 7) >> 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mx = blockIdx.x * RT_CTA_WARPS + warp, my = mrow0 + blockIdx.y;
    if (mx >= MW || my >= mrow1) return;
    const int      x = mx * 8 + (lane & 7), y = my * 4 + (lane >> 3);
    uint32_t       n_traced;
    const uint32_t n = trace_pixel_spp<MODE>(g, bvh, fc, p0, p1, sobol, sr, x, y, spp, n_traced);
    if (x < g.W && y < g.H) count[(size_t)y * g.W + x] = (uint8_t)n;
    count_rays(fc.ray_ctr, 0, n_traced);
}

// Multi-GPU variant (shard.cu, "cooperative ray trace"): this rank traces mask rows [bounds[self], bounds[self+1]) — a
// partition of the WHOLE image balanced on last frame's measured cost, read from device memory, so the host never needs
// to know it: the launch grid covers the largest share the partition kernel may hand out (hr_rt_share_cap) and CTAs past
// the end of the share exit at once (measured alternatives, both ~14 % slower on one GPU: a persistent job loop over an
// atomic counter, and walking the share's rows most-expensive-first — the row-major walk keeps neighbouring rows, i.e.
// the same BVH nodes and G-buffer sectors, in flight together).  Mask words go to this rank's own mask image; k_rt_push (shard.cu) then copies the share to
// every peer with wide stores.  Each warp adds its duration to its mask row's cost, the input of the next partition.
template <int MODE>
__global__ void __launch_bounds__(RT_CTA_WARPS * 32) k_ray_trace_mask_shared(GBufLevelDev g, BvhDev bvh, FrameConsts fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                                const uint8_t* __restrict__ sr, RtShare sh)
{
    const long long t0 = clock64();
    const int MW   = (g.W + 7) >> 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mrow0 = __ldg(sh.bounds + sh.self), mrow1 = __ldg(sh.bounds + sh.self + 1);
    const int mx = blockIdx.x * RT_CTA_WARPS + warp, my = mrow0 + blockIdx.y;
    if (mx >= MW || my >= mrow1) return; // whole warp exits together
    const int      x = mx * 8 + (lane & 7), y = my * 4 + (lane >> 3);
    bool           traced;
    const uint32_t result = trace_pixel<MODE>(g, bvh, fc, p0, p1, sobol, sr, x, y, traced);
    const uint32_t word   = __ballot_sync(0xFFFFFFFFu, result != 0);
    if (lane == 0)
    {
        sh.mask_local[(size_t)my * MW + mx] = word;
        atomicAdd(sh.cost_acc + my, (uint32_t)((clock64() - t0) >> 6) + 1u);
    }
    count_rays(fc.ray_ctr, 0, traced ? 1u : 0u);
}

// spp > 1 form of the cooperative trace: the share's pixels go to this rank's count image (k_rt_push_count copies them to the
// peers).  trace_pixel_spp is the function of k_ray_trace_count, so the counts equal the single-GPU counts bit for bit.  A warp's
// duration grows about linearly with spp, so it is added to the row cost in units of 2^cost_shift cycles, cost_shift = 6 +
// ceil(log2 spp): the row sums stay in the range of the 1-spp trace (scaling every row alike leaves the partition unchanged)
// and cannot overflow at spp <= 255.
template <int MODE>
__global__ void __launch_bounds__(RT_CTA_WARPS * 32) k_ray_trace_count_shared(GBufLevelDev g, BvhDev bvh, FrameConsts fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                                                 const uint8_t* __restrict__ sr, uint8_t* __restrict__ count, int spp, int cost_shift, RtShare sh)
{
    const long long t0 = clock64();
    const int MW   = (g.W + 7) >> 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mrow0 = __ldg(sh.bounds + sh.self), mrow1 = __ldg(sh.bounds + sh.self + 1);
    const int mx = blockIdx.x * RT_CTA_WARPS + warp, my = mrow0 + blockIdx.y;
    if (mx >= MW || my >= mrow1) return; // whole warp exits together
    const int      x = mx * 8 + (lane & 7), y = my * 4 + (lane >> 3);
    uint32_t       n_traced;
    const uint32_t n = trace_pixel_spp<MODE>(g, bvh, fc, p0, p1, sobol, sr, x, y, spp, n_traced);
    if (x < g.W && y < g.H) count[(size_t)y * g.W + x] = (uint8_t)n;
    __syncwarp();
    if (lane == 0) atomicAdd(sh.cost_acc + my, (uint32_t)((clock64() - t0) >> cost_shift) + 1u);
    count_rays(fc.ray_ctr, 0, n_traced);
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

// kind: PASS_SHADOWS (K1, p0 = bias) or PASS_AO (K7, p0 = ray length, p1 = bias)
void launch_ray_trace_mask(int kind, const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* sobol, const uint8_t* sr,
                           uint32_t* mask, int row0, int row1, cudaStream_t st)
{
    const int mrow0 = row0 / 4, mrow1 = (row1 + 3) / 4;
    if (mrow1 <= mrow0) return;
    const auto k = kind == PASS_AO ? k_ray_trace_mask<1> : k_ray_trace_mask<0>;
    k<<<mask_grid(g.W, mrow0, mrow1), RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, p0, p1, sobol, sr, mask, mrow0, mrow1);
}

// the grid covers the largest share hr_rt_wait_partition may hand to one rank
void launch_ray_trace_mask_shared(int kind, const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* sobol,
                                  const uint8_t* sr, const RtShare& sh, cudaStream_t st)
{
    const dim3 grid(((g.W + 7) / 8 + RT_CTA_WARPS - 1) / RT_CTA_WARPS, hr_rt_share_cap((g.H + 3) / 4, sh.world), 1);
    const auto k = kind == PASS_AO ? k_ray_trace_mask_shared<1> : k_ray_trace_mask_shared<0>;
    k<<<grid, RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, p0, p1, sobol, sr, sh);
}

void launch_ray_trace_count_shared(int kind, const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* sobol,
                                   const uint8_t* sr, uint8_t* count, int spp, const RtShare& sh, cudaStream_t st)
{
    int cost_shift = 6;
    while ((1 << (cost_shift - 6)) < spp) cost_shift++;
    const dim3 grid(((g.W + 7) / 8 + RT_CTA_WARPS - 1) / RT_CTA_WARPS, hr_rt_share_cap((g.H + 3) / 4, sh.world), 1);
    const auto k = kind == PASS_AO ? k_ray_trace_count_shared<1> : k_ray_trace_count_shared<0>;
    k<<<grid, RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, p0, p1, sobol, sr, count, spp, cost_shift, sh);
}

void launch_ray_trace_count(int kind, const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* sobol, const uint8_t* sr,
                            uint8_t* count, int spp, int row0, int row1, cudaStream_t st)
{
    const int mrow0 = row0 / 4, mrow1 = (row1 + 3) / 4;
    if (mrow1 <= mrow0) return;
    const auto k = kind == PASS_AO ? k_ray_trace_count<1> : k_ray_trace_count<0>;
    k<<<mask_grid(g.W, mrow0, mrow1), RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, p0, p1, sobol, sr, count, spp, mrow0, mrow1);
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
