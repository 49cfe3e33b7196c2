// traverse.cuh — software BVH traversal shared by every ray-tracing kernel (trace.cu, rt_shade.cu).
// Replaces rayQueryEXT / traceRayEXT over the driver TLAS (ray_query.glsl:6-59, reflections_ray_trace.rgen:150,165,
// gi_ray_trace.rgen:96).  MUST be compiled with -fmad=false: ray_triangle is part of the deterministic chain
// (det_math.cuh); the slab test uses explicit fmaf and only has to be conservative (boxes are padded at build time).
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
// TRV_TRI_MODE (compile time A/B variants; mode 2 vs the default 0 on an H100 SXM 80 GB, 700 W power limit: config 3 K12 2.67 ms vs 2.63,
// config 2 K1 169 us vs 159):
//   0  three __ldg per triangle, issued where the compiler leaves them (it sinks v0 below the dt == 0 branch: two dependent
//      memory round trips per triangle)
//   1  all three 128-bit loads of a triangle issued up front (volatile asm: not sunk, not reordered)
//   2  mode 1 + the next triangle of the leaf is fetched while the current one is tested (one exposed round trip per leaf)
#ifndef TRV_TRI_MODE
#define TRV_TRI_MODE 0
#endif
struct Tri { float4 A, B, C; };
__device__ __forceinline__ Tri load_tri(const float4* __restrict__ tris, int idx)
{
    Tri           t;
    const float4* p = tris + 3ull * idx;
#if TRV_TRI_MODE >= 1
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(t.A.x), "=f"(t.A.y), "=f"(t.A.z), "=f"(t.A.w) : "l"(p));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+16];" : "=f"(t.B.x), "=f"(t.B.y), "=f"(t.B.z), "=f"(t.B.w) : "l"(p));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+32];" : "=f"(t.C.x), "=f"(t.C.y), "=f"(t.C.z), "=f"(t.C.w) : "l"(p));
#else
    t.A = __ldg(p); t.B = __ldg(p + 1); t.C = __ldg(p + 2);
#endif
    return t;
}
// Calls f(tri) for the triangles of leaf reference `node` (< 0) in order; f returns true to stop early.
template <class F>
__device__ __forceinline__ void leaf_tris(const BvhDev& bvh, int node, F&& f)
{
    const int leaf  = ~node;
    const int first = leaf >> 3, cnt = (leaf & 7) + 1;
#if TRV_TRI_MODE >= 2
    Tri cur = load_tri(bvh.tris, first);
    for (int k = 0; k < cnt; k++)
    {
        Tri nxt = cur;
        if (k + 1 < cnt) nxt = load_tri(bvh.tris, first + k + 1);
        if (f(cur)) return;
        cur = nxt;
    }
#else
    for (int k = 0; k < cnt; k++)
        if (f(load_tri(bvh.tris, first + k))) return;
#endif
}

#define STACK_SIZE 64
#define SENTINEL 0x7FFFFFFF

struct SlabSetup { float idx, idy, idz, ox, oy, oz; };
__device__ __forceinline__ SlabSetup slab_setup(const Ray& r)
{
    // |d| < 1e-18 is replaced by +-1e-18 for the BOX test only: with an infinite reciprocal the fma form
    // lo*inf - o*inf turns into NaN/-inf and would reject boxes the ray is inside of (not conservative).
    SlabSetup s;
    s.idx = 1.0f / (fabsf(r.d.x) > 1e-18f ? r.d.x : copysignf(1e-18f, r.d.x));
    s.idy = 1.0f / (fabsf(r.d.y) > 1e-18f ? r.d.y : copysignf(1e-18f, r.d.y));
    s.idz = 1.0f / (fabsf(r.d.z) > 1e-18f ? r.d.z : copysignf(1e-18f, r.d.z));
    s.ox  = r.o.x * s.idx;
    s.oy  = r.o.y * s.idy;
    s.oz  = r.o.z * s.idz;
    return s;
}

// Tests both children of a node; returns entry distances. fminf/fmaxf drop NaNs (0*inf) => conservative.
__device__ __forceinline__ void node_test(const float4* __restrict__ nodes, int node, const SlabSetup& s, float tmin, float tmax, bool& h0, bool& h1,
                                          float& tn0, float& tn1, int& c0, int& c1)
{
    // The 64-byte node is fetched with four 128-bit loads issued back to back (volatile asm): the child indices are loaded
    // up front, so the scheduler cannot sink them below the box tests (a second L1 round trip per traversal step otherwise).
    const float4* np = nodes + 4ull * node;
    float4        n0, n1, nz;
    int           pad0, pad1;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(n0.x), "=f"(n0.y), "=f"(n0.z), "=f"(n0.w) : "l"(np));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+16];" : "=f"(n1.x), "=f"(n1.y), "=f"(n1.z), "=f"(n1.w) : "l"(np));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+32];" : "=f"(nz.x), "=f"(nz.y), "=f"(nz.z), "=f"(nz.w) : "l"(np));
    asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4+48];" : "=r"(c0), "=r"(c1), "=r"(pad0), "=r"(pad1) : "l"(np));
    float ax = fmaf(n0.x, s.idx, -s.ox), bx = fmaf(n0.y, s.idx, -s.ox);
    float ay = fmaf(n0.z, s.idy, -s.oy), by = fmaf(n0.w, s.idy, -s.oy);
    float az = fmaf(nz.x, s.idz, -s.oz), bz = fmaf(nz.y, s.idz, -s.oz);
    tn0      = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fmaxf(fminf(az, bz), tmin));
    float tf = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fminf(fmaxf(az, bz), tmax));
    h0       = tn0 <= tf;
    ax = fmaf(n1.x, s.idx, -s.ox); bx = fmaf(n1.y, s.idx, -s.ox);
    ay = fmaf(n1.z, s.idy, -s.oy); by = fmaf(n1.w, s.idy, -s.oy);
    az = fmaf(nz.z, s.idz, -s.oz); bz = fmaf(nz.w, s.idz, -s.oz);
    tn1 = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fmaxf(fminf(az, bz), tmin));
    tf  = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fminf(fmaxf(az, bz), tmax));
    h1  = tn1 <= tf;
}

// ---- 4-wide nodes (TRV_WIDE, compile time) -----------------------------------------------------------------------------
// Per-lane traversal over bvh.wnodes (bvh_build.cu k_widen): one 112-byte fetch tests four boxes, so a ray makes about half
// the DEPENDENT memory round trips of the binary walk.  Slower than the binary walk on an H100 SXM 80 GB, 700 W power limit: config 3 K12
// 2.88 ms vs 2.63, config 2 K1 168 us vs 159 — the kernels are not bound by that latency chain.
// The hit entries are ordered near-to-far with a 5-exchange network on keys (entry distance bits | entry index; distances
// are >= tmin >= 0, so their bit patterns order like unsigned integers), nearest child next, the others pushed far-to-near.
#ifndef TRV_WIDE
#define TRV_WIDE 0
#endif
// One inner-node step of the wide walk: returns the next node = the nearest hit entry (or a pop when nothing is hit); the other
// hit entries are pushed far-to-near.  Branch-free: (key, ref) pairs go through the exchange network with selects, the three
// possible pushes are unconditional stores whose stack-pointer increments are predicated (the stack has 3 spare slots).
__device__ __forceinline__ int wide_step(const float4* __restrict__ wnodes, int node, const SlabSetup& s, float tmin, float tmax, int* __restrict__ stack, int& sp)
{
    const float4* np = wnodes + 8ull * node;
    float4        lx, hx, ly, hy, lz, hz;
    int           r0, r1, r2, r3;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(lx.x), "=f"(lx.y), "=f"(lx.z), "=f"(lx.w) : "l"(np));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+16];" : "=f"(hx.x), "=f"(hx.y), "=f"(hx.z), "=f"(hx.w) : "l"(np));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+32];" : "=f"(ly.x), "=f"(ly.y), "=f"(ly.z), "=f"(ly.w) : "l"(np));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+48];" : "=f"(hy.x), "=f"(hy.y), "=f"(hy.z), "=f"(hy.w) : "l"(np));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+64];" : "=f"(lz.x), "=f"(lz.y), "=f"(lz.z), "=f"(lz.w) : "l"(np));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+80];" : "=f"(hz.x), "=f"(hz.y), "=f"(hz.z), "=f"(hz.w) : "l"(np));
    asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4+96];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "l"(np));
    uint32_t k0, k1, k2, k3;
#define TRV_BOX(K, LX, HX, LY, HY, LZ, HZ)                                                              \
    {                                                                                                   \
        const float ax = fmaf(LX, s.idx, -s.ox), bx = fmaf(HX, s.idx, -s.ox);                            \
        const float ay = fmaf(LY, s.idy, -s.oy), by = fmaf(HY, s.idy, -s.oy);                            \
        const float az = fmaf(LZ, s.idz, -s.oz), bz = fmaf(HZ, s.idz, -s.oz);                            \
        const float tn = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fmaxf(fminf(az, bz), tmin));        \
        const float tf = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fminf(fmaxf(az, bz), tmax));        \
        K              = tn <= tf ? __float_as_uint(tn) : 0xFFFFFFFFu;                                  \
    }
    TRV_BOX(k0, lx.x, hx.x, ly.x, hy.x, lz.x, hz.x)
    TRV_BOX(k1, lx.y, hx.y, ly.y, hy.y, lz.y, hz.y)
    TRV_BOX(k2, lx.z, hx.z, ly.z, hy.z, lz.z, hz.z)
    TRV_BOX(k3, lx.w, hx.w, ly.w, hy.w, lz.w, hz.w)
#undef TRV_BOX
#define TRV_CX(KA, RA, KB, RB) { const bool sw_ = KB < KA; const uint32_t ka_ = sw_ ? KB : KA, kb_ = sw_ ? KA : KB; const int ra_ = sw_ ? RB : RA, rb_ = sw_ ? RA : RB; KA = ka_; KB = kb_; RA = ra_; RB = rb_; }
    TRV_CX(k0, r0, k1, r1) TRV_CX(k2, r2, k3, r3) TRV_CX(k0, r0, k2, r2) TRV_CX(k1, r1, k3, r3) TRV_CX(k1, r1, k2, r2)
#undef TRV_CX
    const bool room = sp < STACK_SIZE;
    stack[sp] = r3; sp += (room && k3 != 0xFFFFFFFFu) ? 1 : 0;
    stack[sp] = r2; sp += (room && k2 != 0xFFFFFFFFu) ? 1 : 0;
    stack[sp] = r1; sp += (room && k1 != 0xFFFFFFFFu) ? 1 : 0;
    if (k0 == 0xFFFFFFFFu) r0 = stack[--sp];
    return r0;
}

// Any-hit traversal (while-while). Returns true as soon as one triangle is hit in (tmin, tmax).
static __device__ bool trace_any(const BvhDev& bvh, const Ray& r)
{
    int       stack[STACK_SIZE + 4];
    int       sp = 0;
    stack[sp++]  = SENTINEL;
    int             node = 0;
    const SlabSetup s    = slab_setup(r);
    while (node != SENTINEL)
    {
        while (node >= 0 && node != SENTINEL)
        {
#if TRV_WIDE
            node = wide_step(bvh.wnodes, node, s, r.tmin, r.tmax, stack, sp);
#else
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
#endif
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
    int stack[STACK_SIZE + 4];
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
#if TRV_WIDE
            node = wide_step(bvh.wnodes, node, s, r.tmin, best_t, stack, sp);
#else
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
#endif
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

// Any-hit twin of trace_closest_packet for coherent occlusion rays (soft shadows of a small light: the rays of an 8x4 block are
// nearly parallel).  A lane leaves the packet as soon as its ray is occluded; the warp stops when nobody is left or the
// stack is empty.  Per-lane result = trace_any's (a ray is occluded iff some triangle intersects it in (tmin, tmax)).
static __device__ bool trace_any_packet(const BvhDev& bvh, const Ray& r, bool active, int* __restrict__ warp_stack)
{
    const uint32_t FULL = 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31;
    int  sp = 0, node = 0;
    bool alive = active, occluded = false;
    const SlabSetup s = slab_setup(r);
    if (!__any_sync(FULL, alive)) return false;
    for (;;)
    {
        if (node >= 0)
        {
            bool  h0, h1;
            float t0, t1;
            int   c0, c1;
            node_test(bvh.nodes, node, s, r.tmin, r.tmax, h0, h1, t0, t1, c0, c1);
            h0 = h0 && alive;
            h1 = h1 && alive;
            const uint32_t m0 = __ballot_sync(FULL, h0), m1 = __ballot_sync(FULL, h1);
            if (!(m0 | m1))
            {
                if (sp == 0) break;
                node = warp_stack[--sp];
            }
            else if (m0 && m1)
            {
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
                if (alive && ray_triangle(tr.A, tr.B, tr.C, r, t, u, v)) { occluded = true; alive = false; }
                return false;
            });
            if (sp == 0 || !__any_sync(FULL, alive)) break;
            node = warp_stack[--sp];
        }
    }
    return occluded;
}

} // namespace trv
