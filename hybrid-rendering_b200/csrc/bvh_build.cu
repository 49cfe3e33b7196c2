// bvh_build.cu — device LBVH build (replaces the driver BLAS/TLAS build,
// external/dwSampleFramework/extras/ray_traced_scene.cpp:196-248 + src/mesh.cpp:169-231; the reference rebuilds its
// TLAS every frame, src/main.cpp:74).
//
// Pipeline (all on the caller's stream, deterministic):
//   1. k_tri_bounds   per-triangle AABB + scene AABB (ordered-int atomics)
//   2. k_morton       63-bit Morton code of the AABB centre (21 bits / axis)
//   3. cub radix sort (key = Morton, value = primitive index; stable => ties keep primitive order)
//   4. k_hierarchy    Karras 2012 radix tree: children, leaf ranges, parents
//   5. k_fit          bottom-up AABB fit (one atomic flag per internal node)
//   6. k_pack         traversal layout: 64-byte nodes holding both child boxes; sub-trees with <= LEAF_MAX
//                     triangles are collapsed into one leaf (their triangles are contiguous in Morton order)
//
// Topology: hr_debug_set(3, q).  q = 0: Karras radix tree (steps 4-5, fastest build, used by nothing by default).
// q = 1 (default): PLOC — parallel locally-ordered clustering (Meister & Bittner 2018) over the Morton-sorted leaves:
// every round each cluster finds the neighbour within +-PLOC_R array slots that minimises the surface area of the union,
// mutual nearest neighbours are merged, the cluster array is compacted (cub scan) and the loop ends when one cluster is
// left.  The bottom-up agglomeration follows the surface-area heuristic much more closely than Morton-prefix splits
// (fewer node visits per ray).  Hit results do not depend on the topology: any-hit is an existence test and closest-hit
// ties resolve to the lowest primitive index, so the visibility masks stay bit-exact with either builder.
// Internal node ids are handed out downwards from n-2 so that the last merge (the root) is node 0; after the tree is
// complete every leaf walks to the root to find its depth-first position, which makes the triangles of every subtree
// contiguous again (needed for the <= LEAF_MAX leaf collapse) and gives the (first,last) range of every node.
// Before that, g_hr_bvh_treelet_rounds (3) rounds of treelet restructuring (k_treelet) lower the tree's SAH cost; the
// depth-first order and the leaf ranges are computed on the final topology.
//
// Node layout (4 x float4):  n0 = (c0.lo.x, c0.hi.x, c0.lo.y, c0.hi.y)   n1 = (c1.lo.x, c1.hi.x, c1.lo.y, c1.hi.y)
//                            nz = (c0.lo.z, c0.hi.z, c1.lo.z, c1.hi.z)   ch = (int c0, int c1, -, -) as bits
// child >= 0: internal node index;  child < 0: leaf, ~child = (first_tri << 3) | (count - 1).
// Triangle layout (3 x float4, leaf order): (v0.xyz, prim bits) (e1.xyz, 0) (e2.xyz, 0), e = v - v0.
// Boxes are padded by 2^-16 of the scene extent plus 2^-20 of the largest coordinate magnitude (box_pad) so the slab test is
// conservative w.r.t. the fp32 ray/triangle test.
#include "hr_internal.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cfloat>

#ifndef LEAF_MAX
#define LEAF_MAX 2 // fewer triangle tests for a few more node steps than 4; chosen before the port, not re-measured on the H100
#endif

namespace {

__device__ __forceinline__ int   f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7FFFFFFF; }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7FFFFFFF); }

__global__ void k_init_bounds(int* b)
{
    if (threadIdx.x < 3) b[threadIdx.x] = f2ord(FLT_MAX);
    else if (threadIdx.x < 6) b[threadIdx.x] = f2ord(-FLT_MAX);
}

__global__ void k_tri_bounds(const float* __restrict__ verts, uint32_t n, float* __restrict__ aabb, int* __restrict__ bounds)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    float    lo[3] = { FLT_MAX, FLT_MAX, FLT_MAX }, hi[3] = { -FLT_MAX, -FLT_MAX, -FLT_MAX };
    if (i < n)
    {
        const float* p = verts + 9ull * i;
        for (int a = 0; a < 3; a++)
        {
            lo[a] = fminf(fminf(p[a], p[3 + a]), p[6 + a]);
            hi[a] = fmaxf(fmaxf(p[a], p[3 + a]), p[6 + a]);
            aabb[6ull * i + a]     = lo[a];
            aabb[6ull * i + 3 + a] = hi[a];
        }
    }
    for (int a = 0; a < 3; a++)
    {
        for (int o = 16; o; o >>= 1)
        {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xFFFFFFFFu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xFFFFFFFFu, hi[a], o));
        }
        if ((threadIdx.x & 31) == 0)
        {
            atomicMin(bounds + a, f2ord(lo[a]));
            atomicMax(bounds + 3 + a, f2ord(hi[a]));
        }
    }
}

__device__ __forceinline__ uint64_t spread21(uint32_t v)
{
    uint64_t x = v & 0x1FFFFFull;
    x          = (x | x << 32) & 0x1F00000000FFFFull;
    x          = (x | x << 16) & 0x1F0000FF0000FFull;
    x          = (x | x << 8) & 0x100F00F00F00F00Full;
    x          = (x | x << 4) & 0x10C30C30C30C30C3ull;
    x          = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

__global__ void k_morton(const float* __restrict__ aabb, uint32_t n, const int* __restrict__ bounds, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t q[3];
    for (int a = 0; a < 3; a++)
    {
        float lo = ord2f(bounds[a]), hi = ord2f(bounds[3 + a]);
        float c  = 0.5f * (aabb[6ull * i + a] + aabb[6ull * i + 3 + a]);
        float e  = hi - lo;
        float t  = e > 0.0f ? (c - lo) / e : 0.0f;
        t        = fminf(fmaxf(t, 0.0f), 1.0f);
        q[a]     = (uint32_t)fminf(t * 2097152.0f, 2097151.0f);
    }
    keys[i] = (spread21(q[0]) << 2) | (spread21(q[1]) << 1) | spread21(q[2]);
    vals[i] = i;
}

// delta(i,j) = length of the common prefix of key i and key j (ties broken by index), -1 outside [0,n)
__device__ __forceinline__ int delta(const uint64_t* __restrict__ keys, int n, int i, int j)
{
    if (j < 0 || j >= n) return -1;
    uint64_t a = keys[i], b = keys[j];
    if (a == b) return 64 + __clz((uint32_t)i ^ (uint32_t)j);
    return __clzll((long long)(a ^ b));
}

// Karras 2012, "Maximizing parallelism in the construction of BVHs, octrees, and k-d trees", Alg. on p.4.
// Internal nodes 0..n-2; leaves are referred to as n-1+k in the parent array.
__global__ void k_hierarchy(const uint64_t* __restrict__ keys, int n, int2* __restrict__ children, int2* __restrict__ ranges, int* __restrict__ parent)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    int d       = (delta(keys, n, i, i + 1) - delta(keys, n, i, i - 1)) >= 0 ? 1 : -1;
    int dmin    = delta(keys, n, i, i - d);
    int lmax    = 2;
    while (delta(keys, n, i, i + lmax * d) > dmin) lmax <<= 1;
    int l = 0;
    for (int t = lmax >> 1; t >= 1; t >>= 1)
        if (delta(keys, n, i, i + (l + t) * d) > dmin) l += t;
    int j     = i + l * d;
    int dnode = delta(keys, n, i, j);
    int s     = 0;
    for (int t = (l + 1) >> 1;; t = (t + 1) >> 1)
    {
        if (delta(keys, n, i, i + (s + t) * d) > dnode) s += t;
        if (t == 1) break;
    }
    int gamma = i + s * d + min(d, 0);
    int first = min(i, j), last = max(i, j);
    int left  = (first == gamma) ? (n - 1 + gamma) : gamma;          // leaf ids offset by n-1
    int right = (last == gamma + 1) ? (n - 1 + gamma + 1) : gamma + 1;
    children[i] = make_int2(left, right);
    ranges[i]   = make_int2(first, last);
    parent[left]  = i;
    parent[right] = i;
    if (i == 0) parent[0] = -1;
}

__global__ void k_fit(const float* __restrict__ tri_aabb, const uint32_t* __restrict__ sorted_prim, int n, const int2* __restrict__ children,
                      const int* __restrict__ parent, float* __restrict__ node_aabb, int* __restrict__ flags)
{
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    int node = parent[n - 1 + k];
    while (node >= 0)
    {
        if (atomicAdd(flags + node, 1) == 0) return; // first arrival: the sibling subtree is not finished yet
        __threadfence();
        int2  c = children[node];
        float lo[3], hi[3];
        for (int s = 0; s < 2; s++)
        {
            int          ch = s ? c.y : c.x;
            const float* b  = ch >= n - 1 ? tri_aabb + 6ull * sorted_prim[ch - (n - 1)] : node_aabb + 6ull * ch;
            for (int a = 0; a < 3; a++)
            {
                float l = __ldcg(b + a), h = __ldcg(b + 3 + a);
                lo[a] = s ? fminf(lo[a], l) : l;
                hi[a] = s ? fmaxf(hi[a], h) : h;
            }
        }
        for (int a = 0; a < 3; a++)
        {
            __stcg(node_aabb + 6ull * node + a, lo[a]);
            __stcg(node_aabb + 6ull * node + 3 + a, hi[a]);
        }
        __threadfence();
        node = parent[node];
    }
}

// Padding of every box: 2^-16 of the scene extent covers the rounding of the ray/triangle test near edges and vertices.  Far
// from the world origin that pad is smaller than one ulp of the coordinates and rounds away in lo - pad / hi + pad, so it
// is never less than 2^-20 of the largest coordinate magnitude (8 ulp).
__device__ __forceinline__ float box_pad(const int* __restrict__ bounds)
{
    float ext = 0.0f, mag = 0.0f;
    for (int a = 0; a < 3; a++)
    {
        const float lo = ord2f(bounds[a]), hi = ord2f(bounds[3 + a]);
        ext = fmaxf(ext, hi - lo);
        mag = fmaxf(mag, fmaxf(fabsf(lo), fabsf(hi)));
    }
    return ext * (1.0f / 65536.0f) + mag * (1.0f / 1048576.0f) + 1e-7f;
}

// A subtree of <= LEAF_MAX triangles becomes one leaf; as_leaf (null: always) is the treelet optimiser's choice per node.
__device__ __forceinline__ int encode_child(int ch, int n, const int2* __restrict__ ranges, const int* __restrict__ as_leaf)
{
    if (ch >= n - 1) return ~(((ch - (n - 1)) << 3) | 0);
    int2 r = ranges[ch];
    int  cnt = r.y - r.x + 1;
    if (cnt <= LEAF_MAX && (!as_leaf || as_leaf[ch])) return ~((r.x << 3) | (cnt - 1));
    return ch;
}

__global__ void k_pack_nodes(int n, const int2* __restrict__ children, const int2* __restrict__ ranges, const int* __restrict__ as_leaf,
                             const float* __restrict__ tri_aabb, const uint32_t* __restrict__ sorted_prim, const float* __restrict__ node_aabb,
                             const int* __restrict__ bounds, float4* __restrict__ out)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    const float pad = box_pad(bounds);
    int2  c = children[i];
    float b[2][6];
    for (int s = 0; s < 2; s++)
    {
        int          ch  = s ? c.y : c.x;
        const float* src = ch >= n - 1 ? tri_aabb + 6ull * sorted_prim[ch - (n - 1)] : node_aabb + 6ull * ch;
        for (int a = 0; a < 3; a++)
        {
            b[s][a]     = src[a] - pad;
            b[s][3 + a] = src[3 + a] + pad;
        }
    }
    out[4ull * i + 0] = make_float4(b[0][0], b[0][3], b[0][1], b[0][4]);
    out[4ull * i + 1] = make_float4(b[1][0], b[1][3], b[1][1], b[1][4]);
    out[4ull * i + 2] = make_float4(b[0][2], b[0][5], b[1][2], b[1][5]);
    out[4ull * i + 3] = make_float4(__int_as_float(encode_child(c.x, n, ranges, as_leaf)), __int_as_float(encode_child(c.y, n, ranges, as_leaf)), 0.0f, 0.0f);
}

// n <= LEAF_MAX (or n == 1): a single node whose child 0 is the leaf [0,n) with the scene box, child 1 is empty.
__global__ void k_pack_tiny(int n, const int* __restrict__ bounds, float4* __restrict__ out)
{
    float lo[3], hi[3];
    for (int a = 0; a < 3; a++)
    {
        lo[a] = ord2f(bounds[a]);
        hi[a] = ord2f(bounds[3 + a]);
    }
    const float pad = box_pad(bounds);
    out[0] = make_float4(lo[0] - pad, hi[0] + pad, lo[1] - pad, hi[1] + pad);
    // child 1 is unused: a degenerate box far outside any scene (an inverted box would read as infinite in a min/max slab
    // test) that still refers to a valid leaf, so even a visit is harmless.
    out[1] = make_float4(1e30f, 1e30f, 1e30f, 1e30f);
    out[2] = make_float4(lo[2] - pad, hi[2] + pad, 1e30f, 1e30f);
    out[3] = make_float4(__int_as_float(~((0 << 3) | (n - 1))), __int_as_float(~((0 << 3) | 0)), 0.0f, 0.0f);
}

// Height of the binary tree: every leaf counts the edges to the root (both builders keep parent[], leaves at n-1+k, root -1).
// The traversal stacks are sized for HR_BVH_MAX_DEPTH; hr_scene_build / hr_scene_rebuild refuse a deeper tree.
__global__ void k_depth(int n, const int* __restrict__ parent, int* __restrict__ depth)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    int d = 0;
    for (int cur = n - 1 + k; d < (1 << 20) && parent[cur] >= 0; cur = parent[cur]) d++;
    d = __reduce_max_sync(__activemask(), d);
    if ((threadIdx.x & 31) == __ffs(__activemask()) - 1) atomicMax(depth, d);
}

__global__ void k_pack_tris(const float* __restrict__ verts, const uint32_t* __restrict__ sorted_prim, uint32_t n, float4* __restrict__ out)
{
    uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    uint32_t     prim = sorted_prim[k];
    const float* p    = verts + 9ull * prim;
    out[3ull * k + 0] = make_float4(p[0], p[1], p[2], __uint_as_float(prim));
    out[3ull * k + 1] = make_float4(p[3] - p[0], p[4] - p[1], p[5] - p[2], 0.0f);
    out[3ull * k + 2] = make_float4(p[6] - p[0], p[7] - p[1], p[8] - p[2], 0.0f);
}


// ---- PLOC -------------------------------------------------------------------------------------------------------------
#define PLOC_R 24
#define PLOC_T 256

struct Cluster { float4 lo, hi; }; // lo.w = node id bits (leaf k = n-1+k), hi.w = triangle count bits

__global__ void k_ploc_init(int n, const float* __restrict__ tri_aabb, const uint32_t* __restrict__ sorted_prim, Cluster* __restrict__ out, int* __restrict__ parent)
{
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const float* b = tri_aabb + 6ull * sorted_prim[k];
    Cluster      c;
    c.lo   = make_float4(b[0], b[1], b[2], __int_as_float(n - 1 + k));
    c.hi   = make_float4(b[3], b[4], b[5], __int_as_float(1));
    out[k] = c;
    if (k == 0) parent[0] = -1;
}

// nearest neighbour (smallest union surface area, ties -> lowest index) within +-PLOC_R slots
__global__ void __launch_bounds__(PLOC_T) k_ploc_nn(const Cluster* __restrict__ c, int m, int* __restrict__ nn)
{
    __shared__ float s[6][PLOC_T + 2 * PLOC_R];
    const int base = blockIdx.x * PLOC_T - PLOC_R;
    for (int t = threadIdx.x; t < PLOC_T + 2 * PLOC_R; t += PLOC_T)
    {
        const int j = base + t;
        if (j >= 0 && j < m)
        {
            const float4 lo = c[j].lo, hi = c[j].hi;
            s[0][t] = lo.x; s[1][t] = lo.y; s[2][t] = lo.z;
            s[3][t] = hi.x; s[4][t] = hi.y; s[5][t] = hi.z;
        }
    }
    __syncthreads();
    const int i = blockIdx.x * PLOC_T + threadIdx.x;
    if (i >= m) return;
    const int   ti = threadIdx.x + PLOC_R;
    const float lx = s[0][ti], ly = s[1][ti], lz = s[2][ti], hx = s[3][ti], hy = s[4][ti], hz = s[5][ti];
    float       best = FLT_MAX;
    int         bj = -1;
    const int   j0 = max(i - PLOC_R, 0), j1 = min(i + PLOC_R, m - 1);
    for (int j = j0; j <= j1; j++)
    {
        if (j == i) continue;
        const int   t  = j - base;
        const float dx = fmaxf(hx, s[3][t]) - fminf(lx, s[0][t]);
        const float dy = fmaxf(hy, s[4][t]) - fminf(ly, s[1][t]);
        const float dz = fmaxf(hz, s[5][t]) - fminf(lz, s[2][t]);
        const float a  = dx * dy + dy * dz + dz * dx;
        if (a < best) { best = a; bj = j; }
    }
    nn[i] = bj;
}

// flags packed as (merges << 32 | survivors) so one scan yields both the new node index and the compacted slot
__global__ void k_ploc_flags(int m, const int* __restrict__ nn, unsigned long long* __restrict__ flags)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int  j      = nn[i];
    const bool mutual = j >= 0 && nn[j] == i;
    const unsigned long long merge = (mutual && i < j) ? 1ull : 0ull, survive = (mutual && i > j) ? 0ull : 1ull;
    flags[i] = (merge << 32) | survive;
}

__global__ void k_ploc_apply(int m, int n, const Cluster* __restrict__ cin, const int* __restrict__ nn, const unsigned long long* __restrict__ flags,
                             const unsigned long long* __restrict__ scan, int node_base, Cluster* __restrict__ cout, int2* __restrict__ children,
                             int* __restrict__ parent, float* __restrict__ node_aabb, int* __restrict__ sizes, int* __restrict__ counts)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const unsigned long long f = flags[i], sc = scan[i];
    if (i == m - 1)
    {
        counts[0] = (int)((sc + f) & 0xFFFFFFFFull); // survivors
        counts[1] = (int)((sc + f) >> 32);           // merges
    }
    if (!(f & 1ull)) return; // absorbed by its partner
    Cluster a = cin[i];
    if (f >> 32)
    {
        const Cluster b    = cin[nn[i]];
        const int     node = node_base - 1 - (int)(sc >> 32);
        const int     ia = __float_as_int(a.lo.w), ib = __float_as_int(b.lo.w);
        const int     sz = __float_as_int(a.hi.w) + __float_as_int(b.hi.w);
        children[node] = make_int2(ia, ib);
        parent[ia]     = node;
        parent[ib]     = node;
        sizes[node]    = sz;
        a.lo = make_float4(fminf(a.lo.x, b.lo.x), fminf(a.lo.y, b.lo.y), fminf(a.lo.z, b.lo.z), __int_as_float(node));
        a.hi = make_float4(fmaxf(a.hi.x, b.hi.x), fmaxf(a.hi.y, b.hi.y), fmaxf(a.hi.z, b.hi.z), __int_as_float(sz));
        float* o = node_aabb + 6ull * node;
        o[0] = a.lo.x; o[1] = a.lo.y; o[2] = a.lo.z; o[3] = a.hi.x; o[4] = a.hi.y; o[5] = a.hi.z;
    }
    cout[(int)(sc & 0xFFFFFFFFull)] = a;
}

// depth-first offset of every node / leaf: sum of the left siblings' triangle counts along the path to the root
__global__ void k_ploc_offsets(int n, const int2* __restrict__ children, const int* __restrict__ parent, const int* __restrict__ sizes,
                               const uint32_t* __restrict__ sorted_prim, int2* __restrict__ ranges, int* __restrict__ leaf_pos, uint32_t* __restrict__ new_prim)
{
    int id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= 2 * n - 1) return;
    int off = 0, cur = id, p;
    while ((p = parent[cur]) >= 0)
    {
        const int2 c = children[p];
        if (c.y == cur) off += c.x >= n - 1 ? 1 : sizes[c.x];
        cur = p;
    }
    if (id < n - 1) ranges[id] = make_int2(off, off + sizes[id] - 1);
    else
    {
        leaf_pos[id - (n - 1)] = off;
        new_prim[off]          = sorted_prim[id - (n - 1)];
    }
}

__global__ void k_ploc_remap(int n, int2* __restrict__ children, const int* __restrict__ leaf_pos)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    int2 c = children[i];
    if (c.x >= n - 1) c.x = n - 1 + leaf_pos[c.x - (n - 1)];
    if (c.y >= n - 1) c.y = n - 1 + leaf_pos[c.y - (n - 1)];
    children[i] = c;
}

// ---- treelet restructuring (Karras & Aila 2013, "Fast Parallel Construction of High-Quality BVHs") ----------------------
// PLOC clusters within +-PLOC_R slots of the Morton order, which leaves poor splits in the upper levels of long planar scenes.
// Every round walks the binary tree bottom-up (the k_fit flag pattern: the second arrival at a node owns it, and its whole
// subtree is final).  At each node one warp grows a treelet of up to TREELET_LEAVES leaves by repeatedly opening the treelet
// leaf of largest area, finds the topology of least SAH cost over those leaves by dynamic programming over their subsets, and
// rewires the treelet's internal nodes (same ids, new children, refitted boxes) when that is cheaper.
//
// Cost model of the traversal (per ray, in issued instructions): a node step tests both child boxes (~75), a triangle test
// ~80.  SAH(node) = SAH_CI * A(node) + SAH(children), a leaf of c triangles costs SAH_CT * c * A(leaf); a subtree of
// <= LEAF_MAX triangles is packed as one leaf when that is cheaper (as_leaf), which k_pack_nodes follows.
// A treelet whose new height would take a triangle deeper than max_depth keeps its input topology: depth[] holds every
// internal node's depth at the start of the round, and a node's ancestors are restructured only after it.
#define TREELET_LEAVES 7
#define TREELET_WARPS  4
#define SAH_CI 75.0f
#define SAH_CT 80.0f

struct Treelet
{
    int           leaf[TREELET_LEAVES], size[TREELET_LEAVES], height[TREELET_LEAVES], inner[TREELET_LEAVES - 1];
    float         box[TREELET_LEAVES][6], cost[TREELET_LEAVES];
    float         area[1 << TREELET_LEAVES], sah[1 << TREELET_LEAVES];
    unsigned char part[1 << TREELET_LEAVES], as_leaf[1 << TREELET_LEAVES];
};

__device__ __forceinline__ float half_area(const float* b)
{
    const float dx = b[3] - b[0], dy = b[4] - b[1], dz = b[5] - b[2];
    return dx * dy + dy * dz + dz * dx;
}

// box, triangle count, SAH cost and height of a node or triangle (ids >= n-1); written earlier in this kernel, hence L2 loads
__device__ __forceinline__ void treelet_leaf(Treelet& t, int slot, int id, int n, const float* __restrict__ tri_aabb, const uint32_t* __restrict__ prim,
                                             const float* node_aabb, const int* sizes, const float* cost, const int* height)
{
    const bool   tri = id >= n - 1;
    const float* b   = tri ? tri_aabb + 6ull * prim[id - (n - 1)] : node_aabb + 6ull * id;
    for (int a = 0; a < 6; a++) t.box[slot][a] = __ldcg(b + a);
    t.leaf[slot]   = id;
    t.size[slot]   = tri ? 1 : __ldcg(sizes + id);
    t.cost[slot]   = tri ? SAH_CT * half_area(t.box[slot]) : __ldcg(cost + id);
    t.height[slot] = tri ? 0 : __ldcg(height + id);
}

__device__ void treelet_node(Treelet& t, int root, int n, const float* __restrict__ tri_aabb, const uint32_t* __restrict__ prim, int2* children,
                             int* parent, float* node_aabb, int* sizes, float* cost, int* height, int* as_leaf, const int* __restrict__ depth, int max_depth)
{
    const unsigned FULL = 0xFFFFFFFFu;
    const int      lane = threadIdx.x & 31;
    int            L    = 0;
    if (lane == 0)
    {
        const int2 c = __ldcg(children + root);
        treelet_leaf(t, 0, c.x, n, tri_aabb, prim, node_aabb, sizes, cost, height);
        treelet_leaf(t, 1, c.y, n, tri_aabb, prim, node_aabb, sizes, cost, height);
        t.inner[0] = root;
        for (L = 2; L < TREELET_LEAVES; L++)
        {
            int   open = -1;
            float best = -1.0f;
            for (int i = 0; i < L; i++)
                if (t.leaf[i] < n - 1 && half_area(t.box[i]) > best) { best = half_area(t.box[i]); open = i; }
            if (open < 0) break;
            const int2 oc = __ldcg(children + t.leaf[open]);
            t.inner[L - 1] = t.leaf[open];
            treelet_leaf(t, open, oc.x, n, tri_aabb, prim, node_aabb, sizes, cost, height);
            treelet_leaf(t, L, oc.y, n, tri_aabb, prim, node_aabb, sizes, cost, height);
        }
    }
    L = __shfl_sync(FULL, L, 0);
    __syncwarp();
    const unsigned full = (1u << L) - 1;
    // areas of all subsets; singletons cost what their subtree costs, larger subsets start from the one-leaf option
    for (unsigned m = 1 + lane; m <= full; m += 32)
    {
        float b[6] = { FLT_MAX, FLT_MAX, FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX };
        int   sz   = 0;
        for (int i = 0; i < L; i++)
            if (m >> i & 1)
            {
                for (int a = 0; a < 3; a++) { b[a] = fminf(b[a], t.box[i][a]); b[3 + a] = fmaxf(b[3 + a], t.box[i][3 + a]); }
                sz += t.size[i];
            }
        t.area[m] = half_area(b);
        t.sah[m]  = __popc(m) == 1 ? t.cost[__ffs(m) - 1] : sz <= LEAF_MAX ? SAH_CT * (float)sz * t.area[m] : FLT_MAX;
    }
    __syncwarp();
    // subsets by size: the best split of m into p (holding m's lowest leaf) and m ^ p
    for (int k = 2; k <= L; k++)
    {
        for (unsigned m = 1 + lane; m <= full; m += 32)
        {
            if (__popc(m) != k) continue;
            const unsigned low = m & (0u - m), rest = m ^ low;
            float          best = FLT_MAX;
            unsigned       bp   = low;
            unsigned       q    = rest;
            do
            {
                q = (q - 1) & rest;
                const unsigned p = low | q;
                const float    c = t.sah[p] + t.sah[m ^ p];
                if (c < best) { best = c; bp = p; }
            } while (q);
            const float inner = SAH_CI * t.area[m] + best, leafc = t.sah[m];
            t.part[m]    = (unsigned char)bp;
            t.as_leaf[m] = leafc <= inner;
            t.sah[m]     = fminf(leafc, inner);
        }
        __syncwarp();
    }
    if (lane == 0)
    {
        // the input topology's cost, from the root's children
        const int2  c     = __ldcg(children + root);
        float       cc[2];
        int         hh[2];
        for (int s = 0; s < 2; s++)
        {
            const int ch = s ? c.y : c.x;
            if (ch >= n - 1)
            {
                const float* b = tri_aabb + 6ull * prim[ch - (n - 1)];
                float        bb[6];
                for (int a = 0; a < 6; a++) bb[a] = b[a];
                cc[s] = SAH_CT * half_area(bb);
                hh[s] = 0;
            }
            else { cc[s] = __ldcg(cost + ch); hh[s] = __ldcg(height + ch); }
        }
        const int   sz    = __ldcg(sizes + root);
        const float inner = SAH_CI * t.area[full] + cc[0] + cc[1], leafc = sz <= LEAF_MAX ? SAH_CT * (float)sz * t.area[full] : FLT_MAX;
        float       old_c = fminf(inner, leafc);
        int         old_h = 1 + max(hh[0], hh[1]);
        bool        keep  = true;
        if (L > 2 && t.sah[full] < old_c * (1.0f - 1e-5f))
        {
            // new internal nodes in pre-order (root first); ref >= 0: internal node ord, < 0: treelet leaf ~ref
            unsigned om[TREELET_LEAVES - 1];
            int      ref[TREELET_LEAVES - 1][2], nh[TREELET_LEAVES - 1];
            int      cnt = 1;
            om[0]        = full;
            for (int i = 0; i < cnt; i++)
                for (int s = 0; s < 2; s++)
                {
                    const unsigned side = s ? om[i] ^ t.part[om[i]] : t.part[om[i]];
                    if (__popc(side) == 1) ref[i][s] = ~(__ffs(side) - 1);
                    else { ref[i][s] = cnt; om[cnt++] = side; }
                }
            for (int i = cnt - 1; i >= 0; i--)
            {
                const int h0 = ref[i][0] >= 0 ? nh[ref[i][0]] : t.height[~ref[i][0]];
                const int h1 = ref[i][1] >= 0 ? nh[ref[i][1]] : t.height[~ref[i][1]];
                nh[i]        = 1 + max(h0, h1);
            }
            if (nh[0] <= max_depth - __ldcg(depth + root))
            {
                keep = false;
                for (int i = 0; i < cnt; i++)
                {
                    const int id = t.inner[i];
                    int       ids[2];
                    for (int s = 0; s < 2; s++) ids[s] = ref[i][s] >= 0 ? t.inner[ref[i][s]] : t.leaf[~ref[i][s]];
                    float b[6] = { FLT_MAX, FLT_MAX, FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX };
                    int   nsz  = 0;
                    for (int j = 0; j < L; j++)
                        if (om[i] >> j & 1)
                        {
                            for (int a = 0; a < 3; a++) { b[a] = fminf(b[a], t.box[j][a]); b[3 + a] = fmaxf(b[3 + a], t.box[j][3 + a]); }
                            nsz += t.size[j];
                        }
                    __stcg(children + id, make_int2(ids[0], ids[1]));
                    __stcg(parent + ids[0], id);
                    __stcg(parent + ids[1], id);
                    for (int a = 0; a < 6; a++) __stcg(node_aabb + 6ull * id + a, b[a]);
                    __stcg(sizes + id, nsz);
                    __stcg(cost + id, t.sah[om[i]]);
                    __stcg(height + id, nh[i]);
                    __stcg(as_leaf + id, (int)t.as_leaf[om[i]]);
                }
            }
        }
        if (keep)
        {
            __stcg(cost + root, old_c);
            __stcg(height + root, old_h);
            __stcg(as_leaf + root, (int)(leafc <= inner));
        }
        __threadfence();
    }
    __syncwarp();
}

// One restructuring round: one thread per triangle walks up; the warp restructures the treelets its lanes own, one at a time.
__global__ void __launch_bounds__(32 * TREELET_WARPS)
    k_treelet(int n, const float* __restrict__ tri_aabb, const uint32_t* __restrict__ prim, int2* children, int* parent, float* node_aabb, int* sizes,
              float* cost, int* height, int* as_leaf, const int* __restrict__ depth, int* flags, int max_depth)
{
    __shared__ Treelet sh[TREELET_WARPS];
    Treelet&           t    = sh[threadIdx.x >> 5];
    const int          k    = blockIdx.x * blockDim.x + threadIdx.x;
    int                node = k < n ? __ldcg(parent + n - 1 + k) : -1;
    bool               active = node >= 0;
    while (__any_sync(0xFFFFFFFFu, active))
    {
        bool ready = false;
        if (active)
        {
            ready  = atomicAdd(flags + node, 1) != 0; // first arrival: the sibling subtree is not finished yet
            active = ready;
            __threadfence();
        }
        __syncwarp();
        for (unsigned todo = __ballot_sync(0xFFFFFFFFu, ready); todo; todo &= todo - 1)
        {
            const int root = __shfl_sync(0xFFFFFFFFu, node, __ffs(todo) - 1);
            treelet_node(t, root, n, tri_aabb, prim, children, parent, node_aabb, sizes, cost, height, as_leaf, depth, max_depth);
        }
        if (ready)
        {
            node   = __ldcg(parent + node);
            active = node >= 0;
        }
    }
}

// depth of every internal node (edges from the root)
__global__ void k_node_depth(int n, const int* __restrict__ parent, int* __restrict__ depth)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    int d = 0;
    for (int cur = i; d < (1 << 20) && parent[cur] >= 0; cur = parent[cur]) d++;
    depth[i] = d;
}

} // namespace

int g_hr_bvh_quality = 1;
int g_hr_bvh_treelet_rounds = 3;

extern "C" HR_API int hr_internal_bvh_treelet_rounds(int rounds)
{
    const int prev = g_hr_bvh_treelet_rounds;
    if (rounds >= 0) g_hr_bvh_treelet_rounds = rounds;
    return prev;
}

namespace {

// Builds children / ranges / node_aabb (and the depth-first primitive order in sc->d_vals) with PLOC, then restructures its
// treelets for g_hr_bvh_treelet_rounds rounds; *as_leaf is the per-node leaf choice for k_pack_nodes (null without rounds).
// Returns HR_OK, a negative hr_status on a CUDA error, or 1 if the round cap is hit (caller falls back to the radix tree).
int ploc_build(hr_scene* sc, cudaStream_t st, const int** as_leaf)
{
    hr_ctx*   ctx = sc->ctx;
    const int n   = (int)sc->n_tris;
    const int T   = 256;
    // scratch: 2 cluster arrays, nn, flags, scan, counts, cub temp
    size_t scan_tmp = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (unsigned long long*)nullptr, (unsigned long long*)nullptr, n, st);
    const size_t o_c0 = 0, o_c1 = o_c0 + sizeof(Cluster) * n, o_nn = o_c1 + sizeof(Cluster) * n, o_fl = o_nn + ((sizeof(int) * n + 15) & ~size_t(15)),
                 o_sc = o_fl + 8ull * n, o_cnt = o_sc + 8ull * n, o_tmp = o_cnt + 16, o_tl = (o_tmp + scan_tmp + 15) & ~size_t(15),
                 total = o_tl + 5ull * sizeof(int) * n;
    if (total > sc->ploc_bytes)
    {
        if (sc->d_ploc) cudaFree(sc->d_ploc);
        sc->d_ploc = nullptr;
        HR_CUDA(ctx, cudaMalloc(&sc->d_ploc, total));
        sc->ploc_bytes = total;
    }
    char*    base = (char*)sc->d_ploc;
    Cluster* c[2] = { (Cluster*)(base + o_c0), (Cluster*)(base + o_c1) };
    int*     nn   = (int*)(base + o_nn);
    unsigned long long *flags = (unsigned long long*)(base + o_fl), *scan = (unsigned long long*)(base + o_sc);
    int*     counts = (int*)(base + o_cnt);
    int*     sizes  = sc->d_flags; // n-1 ints, unused by this builder otherwise

    k_ploc_init<<<(n + T - 1) / T, T, 0, st>>>(n, sc->d_tri_aabb, sc->d_vals_sorted, c[0], sc->d_parent);
    ctx->launches++;
    int m = n, node_base = n - 1, cur = 0, rounds = 0;
    while (m > 1)
    {
        if (++rounds > 1024) return 1;
        const int g = (m + T - 1) / T;
        k_ploc_nn<<<(m + PLOC_T - 1) / PLOC_T, PLOC_T, 0, st>>>(c[cur], m, nn);
        k_ploc_flags<<<g, T, 0, st>>>(m, nn, flags);
        HR_CUDA(ctx, cub::DeviceScan::ExclusiveSum(base + o_tmp, scan_tmp, flags, scan, m, st));
        k_ploc_apply<<<g, T, 0, st>>>(m, n, c[cur], nn, flags, scan, node_base, c[cur ^ 1], sc->d_children, sc->d_parent, sc->d_node_aabb, sizes, counts);
        ctx->launches += 4;
        int h[2];
        HR_CUDA(ctx, cudaMemcpyAsync(h, counts, sizeof(h), cudaMemcpyDeviceToHost, st));
        HR_CUDA(ctx, cudaStreamSynchronize(st));
        if (h[1] <= 0 || h[0] != m - h[1]) return 1;
        m = h[0];
        node_base -= h[1];
        cur ^= 1;
    }
    if (node_base != 0) return 1;
    *as_leaf = nullptr;
    if (g_hr_bvh_treelet_rounds > 0)
    {
        // treelet scratch: SAH cost, height, leaf choice, depth and walk flags of every internal node
        float* cost   = (float*)(base + o_tl);
        int*   height = (int*)(base + o_tl) + n;
        int*   leaf   = height + n;
        int*   depth  = leaf + n;
        int*   tflags = depth + n;
        for (int r = 0; r < g_hr_bvh_treelet_rounds; r++)
        {
            HR_CUDA(ctx, cudaMemsetAsync(tflags, 0, sizeof(int) * (n - 1), st));
            k_node_depth<<<(n - 1 + T - 1) / T, T, 0, st>>>(n, sc->d_parent, depth);
            k_treelet<<<(n + 32 * TREELET_WARPS - 1) / (32 * TREELET_WARPS), 32 * TREELET_WARPS, 0, st>>>(
                n, sc->d_tri_aabb, sc->d_vals_sorted, sc->d_children, sc->d_parent, sc->d_node_aabb, sizes, cost, height, leaf, depth, tflags, HR_BVH_MAX_DEPTH);
            ctx->launches += 2;
        }
        *as_leaf = leaf;
    }
    int* leaf_pos = reinterpret_cast<int*>(sc->d_keys); // the unsorted keys / values are dead after the radix sort
    k_ploc_offsets<<<(2 * n - 1 + T - 1) / T, T, 0, st>>>(n, sc->d_children, sc->d_parent, sizes, sc->d_vals_sorted, sc->d_ranges, leaf_pos, sc->d_vals);
    k_ploc_remap<<<(n - 1 + T - 1) / T, T, 0, st>>>(n, sc->d_children, leaf_pos);
    ctx->launches += 2;
    HR_CHECK_LAUNCH(ctx);
    return HR_OK;
}

} // namespace

int hr_bvh_build(hr_scene* sc, cudaStream_t st)
{
    hr_ctx*        ctx = sc->ctx;
    const uint32_t n   = sc->n_tris;
    const int      T   = 256;
    const int      gb  = (int)((n + T - 1) / T);
    k_init_bounds<<<1, 32, 0, st>>>(sc->d_bounds_i);
    k_tri_bounds<<<gb, T, 0, st>>>(sc->d_tri_verts, n, sc->d_tri_aabb, sc->d_bounds_i);
    k_morton<<<gb, T, 0, st>>>(sc->d_tri_aabb, n, sc->d_bounds_i, sc->d_keys, sc->d_vals);
    HR_CHECK_LAUNCH(ctx);
    ctx->launches += 3;
    size_t need = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, need, sc->d_keys, sc->d_keys_sorted, sc->d_vals, sc->d_vals_sorted, (int)n, 0, 63, st);
    if (need > sc->sort_tmp_bytes)
    {
        if (sc->d_sort_tmp) cudaFree(sc->d_sort_tmp);
        HR_CUDA(ctx, cudaMalloc(&sc->d_sort_tmp, need));
        sc->sort_tmp_bytes = need;
    }
    HR_CUDA(ctx, cub::DeviceRadixSort::SortPairs(sc->d_sort_tmp, sc->sort_tmp_bytes, sc->d_keys, sc->d_keys_sorted, sc->d_vals, sc->d_vals_sorted,
                                                 (int)n, 0, 63, st));
    const uint32_t* prim_order = sc->d_vals_sorted;
    if (n > LEAF_MAX)
    {
        const int gi = (int)((n - 1 + T - 1) / T);
        bool      ploc = false;
        const int* as_leaf = nullptr;
        if (g_hr_bvh_quality >= 1)
        {
            const int rc = ploc_build(sc, st, &as_leaf);
            if (rc < 0) return rc; // CUDA error, already recorded (rc > 0: round cap hit, fall back to the radix tree)
            ploc = rc == HR_OK;
        }
        if (ploc) prim_order = sc->d_vals;
        else
        {
            as_leaf = nullptr;
            HR_CUDA(ctx, cudaMemsetAsync(sc->d_flags, 0, sizeof(int) * (n - 1), st));
            k_hierarchy<<<gi, T, 0, st>>>(sc->d_keys_sorted, (int)n, sc->d_children, sc->d_ranges, sc->d_parent);
            k_fit<<<gb, T, 0, st>>>(sc->d_tri_aabb, sc->d_vals_sorted, (int)n, sc->d_children, sc->d_parent, sc->d_node_aabb, sc->d_flags);
            ctx->launches += 2;
        }
        k_pack_nodes<<<gi, T, 0, st>>>((int)n, sc->d_children, sc->d_ranges, as_leaf, sc->d_tri_aabb, prim_order, sc->d_node_aabb, sc->d_bounds_i, sc->d_nodes);
        HR_CUDA(ctx, cudaMemsetAsync(sc->d_depth, 0, sizeof(int), st));
        k_depth<<<gb, T, 0, st>>>((int)n, sc->d_parent, sc->d_depth);
        sc->n_nodes = n - 1;
        ctx->launches += 2;
    }
    else
    {
        k_pack_tiny<<<1, 1, 0, st>>>((int)n, sc->d_bounds_i, sc->d_nodes);
        HR_CUDA(ctx, cudaMemsetAsync(sc->d_depth, 0, sizeof(int), st));
        sc->n_nodes = 1;
        ctx->launches += 1;
    }
    k_pack_tris<<<gb, T, 0, st>>>(sc->d_tri_verts, prim_order, n, sc->d_tris);
    ctx->launches += 1;
    HR_CHECK_LAUNCH(ctx);
    return HR_OK;
}

BvhDev hr_bvh_view(const hr_scene* sc)
{
    BvhDev v;
    v.nodes         = sc->d_nodes;
    v.tris          = sc->d_tris;
    v.root_is_valid = sc->n_tris > 0;
    return v;
}
