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
            const float  r0 = det::sample_blue_noise(x, y, (int)fc.num_frames, 0, sobol, sr);
            const float  r1 = det::sample_blue_noise(x, y, (int)fc.num_frames, 1, sobol, sr);
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
// ray generation of K1 only (the traversal is done by the caller): returns whether the pixel traces a ray
__device__ __forceinline__ bool shadow_ray_gen(const GBufLevelDev& g, const FrameConsts& fc, float bias, const uint8_t* __restrict__ sobol, const uint8_t* __restrict__ sr,
                                               int x, int y, Ray& r)
{
    r.o = det::mk(0.0f, 0.0f, 0.0f); r.d = det::mk(0.0f, 0.0f, 1.0f); r.tmin = 0.01f; r.tmax = 0.0f;
    if (x >= g.W || y >= g.H) return false;
    const size_t idx   = (size_t)y * g.W + x;
    const float  depth = __ldg(g.depth + idx);
    if (depth == 1.0f) return false;
    const float  u = ((float)x + 0.5f) / (float)g.W, v = ((float)y + 0.5f) / (float)g.H;
    const V3     P  = det::world_position_from_depth(u, v, depth, fc.view_proj_inverse);
    const float2 e  = load_oct_normal(g.gb2, idx);
    const V3     N  = det::octohedral_to_direction(e.x, e.y);
    const float  r0 = det::sample_blue_noise(x, y, (int)fc.num_frames, 0, sobol, sr);
    const float  r1 = det::sample_blue_noise(x, y, (int)fc.num_frames, 1, sobol, sr);
    r.o = det::add(P, det::scale(N, bias));
    float att;
    det::fetch_light_properties_shadow(fc.light, P, N, r0, r1, r.d, r.tmax, att);
    return att > 0.0f;
}

// K1 with packet traversal (hr_debug_set key 9, default on): the soft-shadow rays of an 8x4 block are nearly parallel, so the
// warp walks one path through the tree with a shared stack (traverse.cuh::trace_any_packet); the mask bits are identical.
__global__ void __launch_bounds__(RT_CTA_WARPS * 32) k_ray_trace_mask_packet(GBufLevelDev g, BvhDev bvh, FrameConsts fc, float bias, const uint8_t* __restrict__ sobol,
                                                                               const uint8_t* __restrict__ sr, uint32_t* __restrict__ mask, int mrow0, int mrow1)
{
    __shared__ int s_stack[RT_CTA_WARPS][STACK_SIZE];
    const int MW   = (g.W + 7) >> 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mx = blockIdx.x * RT_CTA_WARPS + warp, my = mrow0 + blockIdx.y;
    if (mx >= MW || my >= mrow1) return; // whole warp exits together
    const int x = mx * 8 + (lane & 7), y = my * 4 + (lane >> 3);
    Ray        r;
    const bool traced   = shadow_ray_gen(g, fc, bias, sobol, sr, x, y, r);
    const bool occluded = trace_any_packet(bvh, r, traced, s_stack[warp]);
    const uint32_t word = __ballot_sync(0xFFFFFFFFu, traced && !occluded);
    if (lane == 0) mask[(size_t)my * MW + mx] = word;
    count_rays(fc.ray_ctr, 0, traced ? 1u : 0u);
}

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
                const int   si = (int)fc.num_frames * spp + s;
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

// ------------------------------------------------------------------------------------------------------------------------
// Persistent-threads variant with warp-wide ray compaction and a shared-memory (LDS) node stack.
//   * grid = a few CTAs per SM; every WARP independently pulls "super-blocks" of 4 horizontally adjacent mask words
//     (32x4 pixels) from a global atomic counter until the frame is done (persistent threads);
//   * ray generation runs for the 128 pixels of a super-block (4 rounds of 32 lanes); only pixels that really need a ray
//     (not sky, attenuation > 0) are appended to a per-warp ray queue in shared memory with ballot/popc prefix sums
//     (warp-wide compaction) — in the reference's 8x4 groups those lanes simply idle;
//   * traversal consumes the queue with all 32 lanes busy; a lane whose ray terminates refills from the queue at the next
//     refill point (every REFILL_STEPS inner iterations), so early any-hit exits do not leave lanes idle;
//   * the per-lane traversal stack lives in shared memory, laid out [entry][thread] (bank-conflict free); entries beyond
//     SM_STACK spill to a small local array.
// Results: bit (pixel) of the 4 mask words is set with a shared-memory atomicOr when the ray is NOT occluded.
#define PT_WARPS 8
#define PT_QUEUE 128
#define SM_STACK 24
#define REFILL_STEPS 12

struct QRay { float ox, oy, oz, tmax, dx, dy, dz; uint32_t pix; };

template <int MODE>
__global__ void __launch_bounds__(PT_WARPS * 32) k_ray_trace_mask_pt(GBufLevelDev g, BvhDev bvh, FrameConsts fc, float p0, float p1, const uint8_t* __restrict__ sobol,
                                                                      const uint8_t* __restrict__ sr, uint32_t* __restrict__ mask, int mrow0, int mrow1,
                                                                      unsigned int* __restrict__ work_counter)
{
    extern __shared__ __align__(16) unsigned char pt_smem[];
    QRay(*s_queue)[PT_QUEUE]         = reinterpret_cast<QRay(*)[PT_QUEUE]>(pt_smem);
    int(*s_stack)[PT_WARPS * 32]     = reinterpret_cast<int(*)[PT_WARPS * 32]>(pt_smem + sizeof(QRay) * PT_WARPS * PT_QUEUE);
    uint32_t(*s_words)[4]            = reinterpret_cast<uint32_t(*)[4]>(pt_smem + sizeof(QRay) * PT_WARPS * PT_QUEUE + sizeof(int) * SM_STACK * PT_WARPS * 32);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
    const int MW = (g.W + 7) >> 3, SBW = (MW + 3) >> 2, n_sb = SBW * (mrow1 - mrow0);
    const uint32_t lt_mask = (1u << lane) - 1u;
    QRay* q = s_queue[warp];

    for (;;)
    {
        int sb = 0;
        if (lane == 0) sb = (int)atomicAdd(work_counter, 1u);
        sb = __shfl_sync(0xFFFFFFFFu, sb, 0);
        if (sb >= n_sb) break;
        const int my = mrow0 + sb / SBW, mx0 = (sb % SBW) * 4;
        if (lane < 4) s_words[warp][lane] = 0u;
        // ---- ray generation + compaction -------------------------------------------------------------------------------
        int count = 0;
#pragma unroll 1
        for (int w = 0; w < 4; w++)
        {
            const int mx = mx0 + w;
            const int x = mx * 8 + (lane & 7), y = my * 4 + (lane >> 3);
            bool need = false;
            QRay r;
            if (mx < MW && x < g.W && y < g.H)
            {
                const size_t idx   = (size_t)y * g.W + x;
                const float  depth = __ldg(g.depth + idx);
                if (depth != 1.0f)
                {
                    const float  u = ((float)x + 0.5f) / (float)g.W, v = ((float)y + 0.5f) / (float)g.H;
                    const V3     P  = det::world_position_from_depth(u, v, depth, fc.view_proj_inverse);
                    const float2 e  = load_oct_normal(g.gb2, idx);
                    const V3     N  = det::octohedral_to_direction(e.x, e.y);
                    const float  r0 = det::sample_blue_noise(x, y, (int)fc.num_frames, 0, sobol, sr);
                    const float  r1 = det::sample_blue_noise(x, y, (int)fc.num_frames, 1, sobol, sr);
                    V3 o, d;
                    float tmax;
                    if (MODE == 0)
                    {
                        o = det::add(P, det::scale(N, p0));
                        float att;
                        det::fetch_light_properties_shadow(fc.light, P, N, r0, r1, d, tmax, att);
                        need = att > 0.0f;
                    }
                    else
                    {
                        o    = det::add(P, det::scale(N, p1));
                        d    = det::sample_cosine_lobe(N, r0, r1);
                        tmax = p0;
                        need = true;
                    }
                    r.ox = o.x; r.oy = o.y; r.oz = o.z; r.tmax = tmax; r.dx = d.x; r.dy = d.y; r.dz = d.z;
                    r.pix = (uint32_t)(w * 32 + lane);
                }
            }
            const uint32_t b = __ballot_sync(0xFFFFFFFFu, need);
            if (need) q[count + __popc(b & lt_mask)] = r;
            count += __popc(b);
        }
        __syncwarp();
        count_rays(fc.ray_ctr, 0, lane == 0 ? (uint32_t)count : 0u);
        // ---- traversal with dynamic refill -----------------------------------------------------------------------------
        int       head  = 0;
        bool      valid = false;
        Ray       ray;
        SlabSetup ss;
        int       node = SENTINEL, sp = 0, ovf[STACK_SIZE - SM_STACK];
        uint32_t  pix  = 0;
        ray.tmin = 0.01f;
        for (;;)
        {
            // refill idle lanes from the queue (warp-uniform control flow)
            const uint32_t idle = __ballot_sync(0xFFFFFFFFu, !valid);
            if (idle)
            {
                if (!valid)
                {
                    const int mine = head + __popc(idle & lt_mask);
                    if (mine < count)
                    {
                        const QRay r = q[mine];
                        ray.o = det::mk(r.ox, r.oy, r.oz); ray.d = det::mk(r.dx, r.dy, r.dz); ray.tmax = r.tmax;
                        pix   = r.pix;
                        ss    = slab_setup(ray);
                        node  = 0;
                        sp    = 0;
                        valid = true;
                    }
                }
                head += __popc(idle);
            }
            if (!__any_sync(0xFFFFFFFFu, valid)) break;
#pragma unroll 1
            for (int it = 0; it < REFILL_STEPS; it++)
            {
                // internal nodes
                while (valid && node >= 0 && node != SENTINEL)
                {
                    bool  h0, h1;
                    float t0, t1;
                    int   c0, c1;
                    node_test(bvh.nodes, node, ss, ray.tmin, ray.tmax, h0, h1, t0, t1, c0, c1);
                    if (!h0 && !h1)
                    {
                        if (sp == 0) node = SENTINEL;
                        else { --sp; node = sp < SM_STACK ? s_stack[sp][tid] : ovf[sp - SM_STACK]; }
                    }
                    else
                    {
                        node = h0 ? c0 : c1;
                        if (h0 && h1)
                        {
                            if (t1 < t0) { const int tmp = c1; c1 = node; node = tmp; }
                            if (sp < SM_STACK) s_stack[sp][tid] = c1;
                            else if (sp < STACK_SIZE) ovf[sp - SM_STACK] = c1;
                            if (sp < STACK_SIZE) sp++;
                        }
                    }
                }
                // leaf
                if (valid && node < 0)
                {
                    const int leaf  = ~node;
                    const int first = leaf >> 3, cnt = (leaf & 7) + 1;
                    bool      hit   = false;
                    for (int k = 0; k < cnt && !hit; k++)
                    {
                        const float4 A = __ldg(bvh.tris + 3ull * (first + k));
                        const float4 B = __ldg(bvh.tris + 3ull * (first + k) + 1);
                        const float4 C = __ldg(bvh.tris + 3ull * (first + k) + 2);
                        float        t, u, v;
                        hit = ray_triangle(A, B, C, ray, t, u, v);
                    }
                    if (hit) valid = false; // occluded: bit stays 0
                    else if (sp == 0) node = SENTINEL;
                    else { --sp; node = sp < SM_STACK ? s_stack[sp][tid] : ovf[sp - SM_STACK]; }
                }
                if (valid && node == SENTINEL)
                { // traversal finished without a hit: unoccluded
                    atomicOr(&s_words[warp][pix >> 5], 1u << (pix & 31u));
                    valid = false;
                }
                if (!__any_sync(0xFFFFFFFFu, valid)) break;
            }
        }
        __syncwarp();
        if (lane < 4 && mx0 + lane < MW) mask[(size_t)my * MW + mx0 + lane] = s_words[warp][lane];
        __syncwarp();
    }
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

// 0 = one warp per 8x4 block (default), 1 = persistent threads + ray compaction + LDS stack (hr_debug_set key 2).
// Config 2 (1080p) on an H100 SXM 80 GB, 700 W power limit: shadows K1 266 us vs 159, AO K7 144 us vs 77 — the 8x4 blocks are almost uniformly
// active (coherent surfaces), so compaction buys little and the queue / refill bookkeeping costs more.
int g_hr_trace_impl = 0;
// hr_debug_set key 9: 1 = packet traversal for the shadow rays of K1 (single-GPU / band-local path), 0 (default) = per-lane traversal.
// Config 2 (1080p) on an H100 SXM 80 GB, 700 W power limit: K1 with packets 352 us vs 159 per-lane — the cone of a soft-shadow ray bundle makes
// the union of the lanes' paths much longer than any single path, and every lane tests every triangle of every visited leaf.
int g_hr_shadow_packet = 0;

static const size_t kPtSmem = sizeof(QRay) * PT_WARPS * PT_QUEUE + sizeof(int) * SM_STACK * PT_WARPS * 32 + sizeof(uint32_t) * PT_WARPS * 4;

template <int MODE>
static void launch_pt(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float p0, float p1, const uint8_t* sobol, const uint8_t* sr, uint32_t* mask,
                      int mrow0, int mrow1, cudaStream_t st)
{
    // per device (a process may drive several GPUs) and per kernel flavour (shadows / AO may overlap on different streams)
    static unsigned int* counter[64] = {};
    static int           ctas[64]    = {};
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!counter[dev])
    {
        cudaMalloc(&counter[dev], sizeof(unsigned int));
        cudaFuncSetAttribute(k_ray_trace_mask_pt<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPtSmem);
        int sms = 132, per_sm = 1;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_ray_trace_mask_pt<MODE>, PT_WARPS * 32, kPtSmem);
        ctas[dev] = sms * (per_sm > 0 ? per_sm : 1);
    }
    cudaMemsetAsync(counter[dev], 0, sizeof(unsigned int), st);
    k_ray_trace_mask_pt<MODE><<<ctas[dev], PT_WARPS * 32, kPtSmem, st>>>(g, bvh, fc, p0, p1, sobol, sr, mask, mrow0, mrow1, counter[dev]);
}

void launch_shadows_ray_trace(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float bias, const uint8_t* sobol, const uint8_t* sr,
                              uint32_t* mask, int row0, int row1, cudaStream_t st)
{
    const int mrow0 = row0 / 4, mrow1 = (row1 + 3) / 4;
    if (mrow1 <= mrow0) return;
    if (g_hr_trace_impl == 1) { launch_pt<0>(g, bvh, fc, bias, 0.0f, sobol, sr, mask, mrow0, mrow1, st); return; }
    if (g_hr_shadow_packet) { k_ray_trace_mask_packet<<<mask_grid(g.W, mrow0, mrow1), RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, bias, sobol, sr, mask, mrow0, mrow1); return; }
    k_ray_trace_mask<0><<<mask_grid(g.W, mrow0, mrow1), RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, bias, 0.0f, sobol, sr, mask, mrow0, mrow1);
}

void launch_ao_ray_trace(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float ray_length, float bias, const uint8_t* sobol,
                         const uint8_t* sr, uint32_t* mask, int row0, int row1, cudaStream_t st)
{
    const int mrow0 = row0 / 4, mrow1 = (row1 + 3) / 4;
    if (mrow1 <= mrow0) return;
    if (g_hr_trace_impl == 1) { launch_pt<1>(g, bvh, fc, ray_length, bias, sobol, sr, mask, mrow0, mrow1, st); return; }
    k_ray_trace_mask<1><<<mask_grid(g.W, mrow0, mrow1), RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, ray_length, bias, sobol, sr, mask, mrow0, mrow1);
}

// the grid covers the largest share hr_rt_wait_partition may hand to one rank
static inline dim3 shared_grid(int W, int H, int world)
{
    const int MH = (H + 3) / 4;
    return dim3(((W + 7) / 8 + RT_CTA_WARPS - 1) / RT_CTA_WARPS, hr_rt_share_cap(MH, world), 1);
}

void launch_shadows_ray_trace_shared(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float bias, const uint8_t* sobol, const uint8_t* sr,
                                     const RtShare& sh, cudaStream_t st)
{
    k_ray_trace_mask_shared<0><<<shared_grid(g.W, g.H, sh.world), RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, bias, 0.0f, sobol, sr, sh);
}

void launch_ao_ray_trace_shared(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float ray_length, float bias, const uint8_t* sobol,
                                const uint8_t* sr, const RtShare& sh, cudaStream_t st)
{
    k_ray_trace_mask_shared<1><<<shared_grid(g.W, g.H, sh.world), RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, ray_length, bias, sobol, sr, sh);
}

void launch_shadows_ray_trace_count(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float bias, const uint8_t* sobol, const uint8_t* sr,
                                    uint8_t* count, int spp, int row0, int row1, cudaStream_t st)
{
    const int mrow0 = row0 / 4, mrow1 = (row1 + 3) / 4;
    if (mrow1 <= mrow0) return;
    k_ray_trace_count<0><<<mask_grid(g.W, mrow0, mrow1), RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, bias, 0.0f, sobol, sr, count, spp, mrow0, mrow1);
}

void launch_ao_ray_trace_count(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float ray_length, float bias, const uint8_t* sobol,
                               const uint8_t* sr, uint8_t* count, int spp, int row0, int row1, cudaStream_t st)
{
    const int mrow0 = row0 / 4, mrow1 = (row1 + 3) / 4;
    if (mrow1 <= mrow0) return;
    k_ray_trace_count<1><<<mask_grid(g.W, mrow0, mrow1), RT_CTA_WARPS * 32, 0, st>>>(g, bvh, fc, ray_length, bias, sobol, sr, count, spp, mrow0, mrow1);
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
