// traverse.cuh — software BVH traversal shared by every ray-tracing kernel (trace.cu, rt_shade.cu).
// Replaces rayQueryEXT / traceRayEXT over the driver TLAS (ray_query.glsl:6-59, reflections_ray_trace.rgen:150,165,
// gi_ray_trace.rgen:96).  MUST be compiled with -fmad=false: ray_triangle is part of the deterministic chain
// (det_math.cuh); the slab test only has to be conservative (boxes are padded at build time, the interval is widened by
// TRV_WIDEN), so that traversal order never changes a hit result.
#pragma once
#include "det_math.cuh"
#include "hr_internal.h"

namespace trv {

using det::V3;


struct Ray { V3 o, d; float tmin, tmax; };

// Moeller-Trumbore, fixed operation order (see oracle/orc_scene.h::ray_triangle for the CPU statement).
__device__ __forceinline__ bool ray_triangle(const float4 A, const float4 B, const float4 C, const Ray& r, float& t, float& u, float& v)
{
    const V3    v0 = det::mk(A.x, A.y, A.z), e1 = det::mk(B.x, B.y, B.z), e2 = det::mk(C.x, C.y, C.z);
    const V3    p   = det::cross(r.d, e2);
    const float dt  = det::dot(e1, p);
    if (dt == 0.0f) return false;
    const float inv = 1.0f / dt;
    const V3    tv  = det::sub(r.o, v0);
    u               = det::dot(tv, p) * inv;
    if (!(u >= 0.0f && u <= 1.0f)) return false;
    const V3 q = det::cross(tv, e1);
    v          = det::dot(r.d, q) * inv;
    if (!(v >= 0.0f && u + v <= 1.0f)) return false;
    t = det::dot(e2, q) * inv;
    return t > r.tmin && t < r.tmax;
}

// Rays traced (SURVEY.md §8d "rays per frame", reported by hr_pass_get_stats): the calling threads — whatever subset of the
// warp is active — add `n` each; one atomic per warp lands in one of HR_RAY_CTR_SLOTS counters picked by the block index
// (fire-and-forget RED, no return value needed).  kind 0 = primary rays, 1 = secondary (shadow / sky-light) rays.
__device__ __forceinline__ void count_rays(unsigned long long* ctr, int kind, uint32_t n)
{
    if (!ctr) return;
    const unsigned am   = __activemask();
    const uint32_t tot  = __reduce_add_sync(am, n); // REDUX: any subset of lanes
    if ((threadIdx.x & 31) == __ffs(am) - 1 && tot)
        atomicAdd(ctr + ((size_t)kind * HR_RAY_CTR_SLOTS + ((blockIdx.x + blockIdx.y * 7u) & (HR_RAY_CTR_SLOTS - 1))) * HR_RAY_CTR_STRIDE, (unsigned long long)tot);
}

// ---- leaf triangles -------------------------------------------------------------------------------------------------
struct Tri { float4 A, B, C; };
__device__ __forceinline__ Tri load_tri(const float4* __restrict__ tris, int idx)
{
    Tri           t;
    const float4* p = tris + 3ull * idx;
    t.A = __ldg(p); t.B = __ldg(p + 1); t.C = __ldg(p + 2);
    return t;
}
// Calls f(tri) for the triangles of leaf reference `node` (< 0) in order; f returns true to stop early.
template <class F>
__device__ __forceinline__ void leaf_tris(const BvhDev& bvh, int node, F&& f)
{
    const int leaf  = ~node;
    const int first = leaf >> 3, cnt = (leaf & 7) + 1;
    for (int k = 0; k < cnt; k++)
        if (f(load_tri(bvh.tris, first + k))) return;
}

#define STACK_SIZE 64
#define SENTINEL 0x7FFFFFFF

struct SlabSetup { float idx, idy, idz, ox, oy, oz; };
__device__ __forceinline__ SlabSetup slab_setup(const Ray& r)
{
    // |d| < 1e-18 is replaced by +-1e-18 for the BOX test only: with an infinite reciprocal (lo - o) * inf is NaN when the
    // origin lies on a face of the slab, and would reject a box the ray runs inside of (not conservative).
    SlabSetup s;
    s.idx = 1.0f / (fabsf(r.d.x) > 1e-18f ? r.d.x : copysignf(1e-18f, r.d.x));
    s.idy = 1.0f / (fabsf(r.d.y) > 1e-18f ? r.d.y : copysignf(1e-18f, r.d.y));
    s.idz = 1.0f / (fabsf(r.d.z) > 1e-18f ? r.d.z : copysignf(1e-18f, r.d.z));
    s.ox  = r.o.x;
    s.oy  = r.o.y;
    s.oz  = r.o.z;
    return s;
}

// Slab distance (b - o) / d, subtracted first: the rounding error is relative to the distance itself.  The fma form
// b * (1/d) - o * (1/d) saves an instruction but rounds o * (1/d), an error proportional to |o|, the ray origin's absolute
// coordinate, which the box padding (relative to the scene's extent) does not cover far from the world origin.
#define TRV_SLAB(B, O, ID) (((B) - (O)) * (ID))
// A box is entered when t_near <= t_far * TRV_WIDEN.  The two slab distances carry at most three roundings each (reciprocal,
// subtraction, product), about 3 ulp relative, and t_far may be the t of a hit from ray_triangle, whose own rounding is a
// few ulp more (for rays from 1e4 scene extents away, 4 ulp was measured to be too little on an H100).  1 + 2^-19 (16 ulp)
// covers both; the cost is boxes longer by 2e-6 of their distance along the ray.
#define TRV_WIDEN 1.0000019073486328125f

// Tests both children of a node; returns entry distances. fminf/fmaxf never see a NaN (finite reciprocals) => conservative.
__device__ __forceinline__ void node_test(const float4* __restrict__ nodes, int node, const SlabSetup& s, float tmin, float tmax, bool& h0, bool& h1,
                                          float& tn0, float& tn1, int& c0, int& c1)
{
    // The 64-byte node is fetched with four 128-bit loads (volatile asm).  ptxas still narrows the last one to the two link
    // words (the upper 8 bytes are padding) and issues it after the box test's branch, where the links are first used: a
    // second L1 round trip per step whose box test passes.  A branch-free step that consumes the links in the test's block
    // issues it with the boxes, but measured slower (DESIGN.md §8).
    const float4* np = nodes + 4ull * node;
    float4        n0, n1, nz;
    int           pad0, pad1;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(n0.x), "=f"(n0.y), "=f"(n0.z), "=f"(n0.w) : "l"(np));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+16];" : "=f"(n1.x), "=f"(n1.y), "=f"(n1.z), "=f"(n1.w) : "l"(np));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+32];" : "=f"(nz.x), "=f"(nz.y), "=f"(nz.z), "=f"(nz.w) : "l"(np));
    asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4+48];" : "=r"(c0), "=r"(c1), "=r"(pad0), "=r"(pad1) : "l"(np));
    float ax = TRV_SLAB(n0.x, s.ox, s.idx), bx = TRV_SLAB(n0.y, s.ox, s.idx);
    float ay = TRV_SLAB(n0.z, s.oy, s.idy), by = TRV_SLAB(n0.w, s.oy, s.idy);
    float az = TRV_SLAB(nz.x, s.oz, s.idz), bz = TRV_SLAB(nz.y, s.oz, s.idz);
    tn0      = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fmaxf(fminf(az, bz), tmin));
    float tf = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fminf(fmaxf(az, bz), tmax));
    h0       = tn0 <= tf * TRV_WIDEN;
    ax = TRV_SLAB(n1.x, s.ox, s.idx); bx = TRV_SLAB(n1.y, s.ox, s.idx);
    ay = TRV_SLAB(n1.z, s.oy, s.idy); by = TRV_SLAB(n1.w, s.oy, s.idy);
    az = TRV_SLAB(nz.z, s.oz, s.idz); bz = TRV_SLAB(nz.w, s.oz, s.idz);
    tn1 = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fmaxf(fminf(az, bz), tmin));
    tf  = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fminf(fmaxf(az, bz), tmax));
    h1  = tn1 <= tf * TRV_WIDEN;
}

// Any-hit traversal (while-while). Returns true as soon as one triangle is hit in (tmin, tmax).
static __device__ bool trace_any(const BvhDev& bvh, const Ray& r)
{
    int       stack[STACK_SIZE];
    int       sp = 0;
    stack[sp++]  = SENTINEL;
    int             node = 0;
    const SlabSetup s    = slab_setup(r);
    while (node != SENTINEL)
    {
        while (node >= 0 && node != SENTINEL)
        {
            bool  h0, h1;
            float t0, t1;
            int   c0, c1;
            node_test(bvh.nodes, node, s, r.tmin, r.tmax, h0, h1, t0, t1, c0, c1);
            if (!h0 && !h1) node = stack[--sp];
            else
            {
                node = h0 ? c0 : c1;
                if (h0 && h1)
                {
                    if (t1 < t0) { int tmp = c1; c1 = node; node = tmp; }
                    if (sp < STACK_SIZE) stack[sp++] = c1;
                }
            }
        }
        if (node < 0)
        {
            bool hit = false;
            leaf_tris(bvh, node, [&](const Tri& tr) { float t, u, v; hit = ray_triangle(tr.A, tr.B, tr.C, r, t, u, v); return hit; });
            if (hit) return true;
            node = stack[--sp];
        }
    }
    return false;
}

// Closest hit; ties broken by the lowest primitive index (order independent).
static __device__ bool trace_closest(const BvhDev& bvh, const Ray& r, float& best_t, uint32_t& best_prim, float& best_u, float& best_v)
{
    int stack[STACK_SIZE];
    int sp      = 0;
    stack[sp++] = SENTINEL;
    int node    = 0;
    best_t      = r.tmax;
    best_prim   = 0xFFFFFFFFu;
    best_u = best_v = 0.0f;
    const SlabSetup s = slab_setup(r);
    while (node != SENTINEL)
    {
        while (node >= 0 && node != SENTINEL)
        {
            bool  h0, h1;
            float t0, t1;
            int   c0, c1;
            node_test(bvh.nodes, node, s, r.tmin, best_t, h0, h1, t0, t1, c0, c1);
            if (!h0 && !h1) node = stack[--sp];
            else
            {
                node = h0 ? c0 : c1;
                if (h0 && h1)
                {
                    if (t1 < t0) { int tmp = c1; c1 = node; node = tmp; }
                    if (sp < STACK_SIZE) stack[sp++] = c1;
                }
            }
        }
        if (node < 0)
        {
            leaf_tris(bvh, node, [&](const Tri& tr) {
                float t, u, v;
                if (ray_triangle(tr.A, tr.B, tr.C, r, t, u, v))
                {
                    const uint32_t prim = __float_as_uint(tr.A.w);
                    if (t < best_t || (t == best_t && prim < best_prim)) { best_t = t; best_prim = prim; best_u = u; best_v = v; }
                }
                return false;
            });
            node = stack[--sp];
        }
    }
    return best_prim != 0xFFFFFFFFu;
}


// Packet traversal for COHERENT rays (primary visibility): the whole warp walks ONE path through the tree — a node is entered if
// any lane's ray hits its box — with a single per-warp stack in shared memory.  Control flow is warp-uniform (no lane-level
// divergence, node loads are one broadcast transaction); every lane still tests boxes and triangles against its own ray and its
// own current best hit, so the result per lane is exactly trace_closest's (closest hit, ties -> lowest primitive; the set of
// triangles a lane tests is a superset of what its own traversal would visit).  All 32 lanes must call it; `active` = lane has a ray.
// warp_stack: STACK_SIZE ints of shared memory owned by this warp.
static __device__ bool trace_closest_packet(const BvhDev& bvh, const Ray& r, bool active, int* __restrict__ warp_stack, float& best_t, uint32_t& best_prim,
                                            float& best_u, float& best_v)
{
    const uint32_t FULL = 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31;
    int sp   = 0;
    int node = 0;
    best_t    = r.tmax;
    best_prim = 0xFFFFFFFFu;
    best_u = best_v = 0.0f;
    const SlabSetup s = slab_setup(r);
    if (!__any_sync(FULL, active)) return false;
    for (;;)
    {
        if (node >= 0)
        {
            bool  h0, h1;
            float t0, t1;
            int   c0, c1;
            node_test(bvh.nodes, node, s, r.tmin, best_t, h0, h1, t0, t1, c0, c1);
            h0 = h0 && active;
            h1 = h1 && active;
            const uint32_t m0 = __ballot_sync(FULL, h0), m1 = __ballot_sync(FULL, h1);
            if (!(m0 | m1))
            {
                if (sp == 0) break;
                node = warp_stack[--sp];
            }
            else if (m0 && m1)
            {
                // visit first the child most lanes would enter first; the other one goes on the stack
                const uint32_t near1 = __ballot_sync(FULL, h1 && (!h0 || t1 < t0));
                const bool     first1 = __popc(near1) > __popc((m0 | m1) & ~near1);
                if (sp < STACK_SIZE) { if (lane == 0) warp_stack[sp] = first1 ? c0 : c1; sp++; }
                __syncwarp();
                node = first1 ? c1 : c0;
            }
            else node = m0 ? c0 : c1;
        }
        else
        {
            leaf_tris(bvh, node, [&](const Tri& tr) {
                float t, u, v;
                if (active && ray_triangle(tr.A, tr.B, tr.C, r, t, u, v))
                {
                    const uint32_t prim = __float_as_uint(tr.A.w);
                    if (t < best_t || (t == best_t && prim < best_prim)) { best_t = t; best_prim = prim; best_u = u; best_v = v; }
                }
                return false;
            });
            if (sp == 0) break;
            node = warp_stack[--sp];
        }
    }
    return best_prim != 0xFFFFFFFFu;
}

} // namespace trv
