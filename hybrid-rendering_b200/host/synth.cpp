// synth.cpp — CPU-side synthetic scene / camera / G-buffer / blue-noise producers (see synth.h).
// Host-only C++; replaces the reference's raster G-buffer stage and asset loading for headless runs.
#include "synth.h"
#include "hr_math.h"
#include <algorithm>
#include <cfloat>
#include <cstdlib>
#include <immintrin.h>
#include <numeric>
#include <vector>

using namespace hrm;

struct hrs_scene {
    std::vector<hr_vertex>   vertices;
    std::vector<uint32_t>    indices;
    std::vector<hr_instance> instances;
    std::vector<hr_material> materials;
    // derived: world-space soup + BVH for primary visibility
    struct Tri { V3 v0, e1, e2; V3 n0, n1, n2; uint32_t inst; V3 v1, v2; }; // v1, v2: the original vertices (v0 + e1 != v1 in fp32)
    struct Node { float lo[3], hi[3]; int left, right, first, count; };
    std::vector<Tri>  tris;     // primitive order (instances in order, triangles in index order)
    std::vector<Tri>  bvh_tris; // BVH leaf order
    std::vector<Node> nodes;
    V3                bmin { 0, 0, 0 }, bmax { 0, 0, 0 };
    void finalize();
    int  build_rec(int first, int last, std::vector<V3>& cen, std::vector<V3>& tmin, std::vector<V3>& tmax, std::vector<uint32_t>& order);
    bool closest(V3 o, V3 d, float tmax, float& t, float& u, float& v, uint32_t& prim) const;
};

namespace {

uint32_t add_material(hrs_scene& s, float r, float g, float b, float roughness, float metallic)
{
    hr_material m {};
    m.albedo[0] = r; m.albedo[1] = g; m.albedo[2] = b; m.albedo[3] = 1.0f;
    m.roughness = roughness;
    m.metallic  = metallic;
    s.materials.push_back(m);
    return (uint32_t)s.materials.size() - 1;
}

struct MeshBuilder {
    hrs_scene& s;
    uint32_t   base_vertex, first_index;
    explicit MeshBuilder(hrs_scene& sc) : s(sc), base_vertex((uint32_t)sc.vertices.size()), first_index((uint32_t)sc.indices.size()) {}
    uint32_t vert(V3 p, V3 n, float u = 0, float v = 0)
    {
        hr_vertex vx {};
        vx.position[0] = p.x; vx.position[1] = p.y; vx.position[2] = p.z; vx.position[3] = 1.0f;
        vx.tex_coord[0] = u; vx.tex_coord[1] = v;
        vx.normal[0] = n.x; vx.normal[1] = n.y; vx.normal[2] = n.z;
        V3 t = normalize(cross(std::fabs(n.y) > 0.99f ? V3 { 1, 0, 0 } : V3 { 0, 1, 0 }, n));
        V3 b = cross(n, t);
        vx.tangent[0] = t.x; vx.tangent[1] = t.y; vx.tangent[2] = t.z;
        vx.bitangent[0] = b.x; vx.bitangent[1] = b.y; vx.bitangent[2] = b.z;
        s.vertices.push_back(vx);
        return (uint32_t)s.vertices.size() - 1 - base_vertex;
    }
    void tri(uint32_t a, uint32_t b, uint32_t c) { s.indices.push_back(a); s.indices.push_back(b); s.indices.push_back(c); }
    void finish(uint32_t material)
    {
        hr_instance in {};
        M4 id = identity();
        memcpy(in.model, id.m, 64);
        in.first_index  = first_index;
        in.index_count  = (uint32_t)s.indices.size() - first_index;
        in.base_vertex  = base_vertex;
        in.material_idx = material;
        s.instances.push_back(in);
    }
};

// Rectangular grid origin + i*du + j*dv, (nu x nv) cells, constant normal.
void add_grid(hrs_scene& s, V3 origin, V3 du, V3 dv, int nu, int nv, V3 n, uint32_t mat)
{
    MeshBuilder mb(s);
    for (int j = 0; j <= nv; j++)
        for (int i = 0; i <= nu; i++) mb.vert(origin + du * ((float)i / nu) + dv * ((float)j / nv), n, (float)i / nu, (float)j / nv);
    for (int j = 0; j < nv; j++)
        for (int i = 0; i < nu; i++)
        {
            uint32_t a = j * (nu + 1) + i, b = a + 1, c = a + nu + 1, d = c + 1;
            mb.tri(a, b, d);
            mb.tri(a, d, c);
        }
    mb.finish(mat);
}

void add_box(hrs_scene& s, V3 lo, V3 hi, uint32_t mat, int tess = 1)
{
    V3 d = hi - lo;
    // six faces as separate grids but ONE instance: build manually
    MeshBuilder mb(s);
    auto face = [&](V3 o, V3 du, V3 dv, V3 n) {
        uint32_t base = (uint32_t)s.vertices.size() - mb.base_vertex;
        for (int j = 0; j <= tess; j++)
            for (int i = 0; i <= tess; i++) mb.vert(o + du * ((float)i / tess) + dv * ((float)j / tess), n);
        for (int j = 0; j < tess; j++)
            for (int i = 0; i < tess; i++)
            {
                uint32_t a = base + j * (tess + 1) + i, b = a + 1, c = a + tess + 1, e = c + 1;
                mb.tri(a, b, e);
                mb.tri(a, e, c);
            }
    };
    face(lo, { d.x, 0, 0 }, { 0, 0, d.z }, { 0, -1, 0 });
    face({ lo.x, hi.y, lo.z }, { d.x, 0, 0 }, { 0, 0, d.z }, { 0, 1, 0 });
    face(lo, { d.x, 0, 0 }, { 0, d.y, 0 }, { 0, 0, -1 });
    face({ lo.x, lo.y, hi.z }, { d.x, 0, 0 }, { 0, d.y, 0 }, { 0, 0, 1 });
    face(lo, { 0, 0, d.z }, { 0, d.y, 0 }, { -1, 0, 0 });
    face({ hi.x, lo.y, lo.z }, { 0, 0, d.z }, { 0, d.y, 0 }, { 1, 0, 0 });
    mb.finish(mat);
}

// Vertical cylinder (smooth normals) with caps.
void add_cylinder(hrs_scene& s, V3 base, float radius, float height, int segs, int rings, uint32_t mat)
{
    MeshBuilder mb(s);
    const float PI2 = 6.28318530718f;
    for (int r = 0; r <= rings; r++)
        for (int i = 0; i <= segs; i++)
        {
            float a = PI2 * (float)i / segs;
            V3    n = { std::cos(a), 0, std::sin(a) };
            mb.vert(base + n * radius + V3 { 0, height * (float)r / rings, 0 }, n, (float)i / segs, (float)r / rings);
        }
    for (int r = 0; r < rings; r++)
        for (int i = 0; i < segs; i++)
        {
            uint32_t a = r * (segs + 1) + i, b = a + 1, c = a + segs + 1, d = c + 1;
            mb.tri(a, b, d);
            mb.tri(a, d, c);
        }
    // top cap fan
    uint32_t ctr = mb.vert(base + V3 { 0, height, 0 }, { 0, 1, 0 });
    uint32_t rim = (uint32_t)s.vertices.size() - mb.base_vertex;
    for (int i = 0; i <= segs; i++)
    {
        float a = PI2 * (float)i / segs;
        mb.vert(base + V3 { std::cos(a) * radius, height, std::sin(a) * radius }, { 0, 1, 0 });
    }
    for (int i = 0; i < segs; i++) mb.tri(ctr, rim + i, rim + i + 1);
    mb.finish(mat);
}

// Half torus arch in the plane spanned by `axis` (horizontal unit vector) and +Y, centred at c.
void add_arch(hrs_scene& s, V3 c, V3 axis, float major_r, float minor_r, int segs_major, int segs_minor, uint32_t mat)
{
    MeshBuilder mb(s);
    const float PI = 3.14159265359f;
    V3          side = cross(axis, V3 { 0, 1, 0 });
    for (int i = 0; i <= segs_major; i++)
    {
        float a  = PI * (float)i / segs_major;
        V3    rc = axis * std::cos(a) + V3 { 0, 1, 0 } * std::sin(a); // radial direction of the ring centre
        for (int j = 0; j <= segs_minor; j++)
        {
            float b = 2 * PI * (float)j / segs_minor;
            V3    n = rc * std::cos(b) + side * std::sin(b);
            mb.vert(c + rc * major_r + n * minor_r, n, (float)i / segs_major, (float)j / segs_minor);
        }
    }
    for (int i = 0; i < segs_major; i++)
        for (int j = 0; j < segs_minor; j++)
        {
            uint32_t a = i * (segs_minor + 1) + j, b = a + 1, cc = a + segs_minor + 1, d = cc + 1;
            mb.tri(a, b, d);
            mb.tri(a, d, cc);
        }
    mb.finish(mat);
}

struct Rng {
    uint64_t s;
    explicit Rng(uint64_t seed) : s(seed * 0x9E3779B97F4A7C15ull + 0x1234567ull) {}
    uint32_t next()
    {
        s += 0x9E3779B97F4A7C15ull;
        uint64_t z = s;
        z          = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z          = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return (uint32_t)((z ^ (z >> 31)) >> 16);
    }
    float uniform() { return (float)(next() & 0xFFFFFF) / 16777216.0f; }
};

void build_single_triangle(hrs_scene& s)
{
    uint32_t    m = add_material(s, 0.8f, 0.8f, 0.8f, 0.5f, 0.0f);
    MeshBuilder mb(s);
    mb.vert({ -4, 3, -4 }, { 0, 1, 0 });
    mb.vert({ 4, 3, -4 }, { 0, 1, 0 });
    mb.vert({ 0, 3, 4 }, { 0, 1, 0 });
    mb.tri(0, 1, 2);
    mb.finish(m);
}

void build_ground_plane(hrs_scene& s)
{
    uint32_t m = add_material(s, 0.7f, 0.7f, 0.7f, 0.5f, 0.0f);
    add_grid(s, { -200, 0, -200 }, { 400, 0, 0 }, { 0, 0, 400 }, 1, 1, { 0, 1, 0 }, m);
}

void build_shadows_test(hrs_scene& s, uint32_t seed)
{
    Rng      rng(seed);
    uint32_t mfloor = add_material(s, 0.6f, 0.6f, 0.6f, 0.5f, 0.0f);
    add_grid(s, { -30, 0, -30 }, { 60, 0, 0 }, { 0, 0, 60 }, 8, 8, { 0, 1, 0 }, mfloor);
    const float rough[4] = { 0.02f, 0.2f, 0.5f, 0.9f };
    for (int i = 0; i < 6; i++)
    {
        uint32_t m = add_material(s, 0.3f + 0.1f * i, 0.5f, 0.8f - 0.1f * i, rough[i & 3], (i & 1) ? 1.0f : 0.0f);
        float    x = -20.0f + 8.0f * i, z = -6.0f + 12.0f * rng.uniform();
        float    h = 2.0f + 6.0f * rng.uniform();
        add_box(s, { x - 1.5f, 0, z - 1.5f }, { x + 1.5f, h, z + 1.5f }, m, 2);
    }
    for (int i = 0; i < 5; i++)
    {
        uint32_t m = add_material(s, 0.8f, 0.4f + 0.1f * i, 0.3f, rough[(i + 1) & 3], 0.0f);
        add_cylinder(s, { -16.0f + 8.0f * i, 0, 8.0f + 4.0f * rng.uniform() }, 1.0f, 7.0f, 24, 4, m);
    }
    uint32_t mslab = add_material(s, 0.5f, 0.5f, 0.5f, 0.3f, 0.0f);
    add_box(s, { -12, 7, 4 }, { 12, 7.6f, 14 }, mslab, 2); // overhanging slab for AO / contact shadows
    uint32_t march = add_material(s, 0.7f, 0.7f, 0.5f, 0.2f, 0.0f);
    add_arch(s, { 0, 0, -12 }, { 1, 0, 0 }, 6.0f, 0.7f, 24, 10, march);
}

// Two-storey arcade along +Z: floor, two rows of columns per storey, arches between columns, galleries, ceiling, end walls.
void build_arcade(hrs_scene& s, int target_tris, uint32_t seed)
{
    Rng         rng(seed);
    const float rough[4] = { 0.02f, 0.2f, 0.5f, 0.9f };
    auto mat = [&](int i) { return add_material(s, 0.45f + 0.4f * rng.uniform(), 0.45f + 0.4f * rng.uniform(), 0.4f + 0.4f * rng.uniform(), rough[i & 3], (i % 5 == 0) ? 1.0f : 0.0f); };
    const int   ncol = 14;     // columns per row
    const float L = 112.0f, spacing = L / ncol, halfw = 12.0f, storey = 14.0f;
    auto count = [&](float k, bool emit) -> long {
        long n = 0;
        int  fl = std::max(2, (int)(96 * k)), segs = std::max(8, (int)(48 * k)), rings = std::max(2, (int)(12 * k));
        int  am = std::max(6, (int)(28 * k)), an = std::max(6, (int)(14 * k)), wt = std::max(2, (int)(40 * k));
        int  mi = 0;
        // floor + ceiling + two gallery slabs
        n += 2L * fl * fl;
        if (emit) add_grid(s, { -30, 0, -8 }, { 60, 0, 0 }, { 0, 0, L + 16 }, fl, fl, { 0, 1, 0 }, mat(mi));
        mi++;
        for (int side = -1; side <= 1; side += 2)
        {
            // roof over the side aisles only: the nave (|x| < halfw) is open to the sky so the sun reaches the floor
            n += 2L * (fl / 4) * fl;
            float xr = side < 0 ? -30.0f : halfw;
            if (emit) add_grid(s, { xr, 2 * storey, -8 }, { 30 - halfw, 0, 0 }, { 0, 0, L + 16 }, fl / 4, fl, { 0, -1, 0 }, mat(mi));
            mi++;
            n += 2L * (fl / 4) * fl;
            float x0 = side < 0 ? -30.0f : halfw;
            if (emit) add_grid(s, { x0, storey, -8 }, { 30 - halfw, 0, 0 }, { 0, 0, L + 16 }, fl / 4, fl, { 0, 1, 0 }, mat(mi));
            mi++;
            // outer wall
            n += 2L * wt * wt;
            if (emit) add_grid(s, { side * 30.0f, 0, -8 }, { 0, 0, L + 16 }, { 0, 2 * storey, 0 }, wt, wt, { (float)-side, 0, 0 }, mat(mi));
            mi++;
        }
        n += 2L * wt * wt; // back wall
        if (emit) add_grid(s, { -30, 0, L + 8 }, { 60, 0, 0 }, { 0, 2 * storey, 0 }, wt, wt, { 0, 0, -1 }, mat(mi));
        mi++;
        for (int st = 0; st < 2; st++)
            for (int side = -1; side <= 1; side += 2)
                for (int c = 0; c <= ncol; c++)
                {
                    float z = c * spacing, x = side * halfw, y = st * storey;
                    n += 2L * segs * rings + segs;
                    if (emit) add_cylinder(s, { x, y, z }, 1.1f - 0.15f * st, storey - spacing * 0.5f + 1.0f, segs, rings, mat(mi));
                    mi++;
                    if (c < ncol)
                    {
                        n += 2L * am * an;
                        if (emit) add_arch(s, { x, y + storey - spacing * 0.5f, z + spacing * 0.5f }, { 0, 0, 1 }, spacing * 0.5f, 0.6f, am, an, mat(mi));
                        mi++;
                    }
                }
        // a few free-standing boxes on the floor (statues / crates)
        for (int b = 0; b < 10; b++)
        {
            n += 12L * 4;
            if (emit)
            {
                float z = 6.0f + b * 10.5f, x = (b & 1) ? 4.5f : -4.5f, h = 1.5f + 0.35f * b;
                add_box(s, { x - 1.2f, 0, z - 1.2f }, { x + 1.2f, h, z + 1.2f }, mat(mi), 2);
            }
            mi++;
        }
        return n;
    };
    // find tessellation factor k hitting the target
    float lo = 0.02f, hi = 8.0f;
    for (int it = 0; it < 40; it++)
    {
        float mid = 0.5f * (lo + hi);
        if (count(mid, false) < target_tris) lo = mid; else hi = mid;
    }
    Rng saved = rng;
    (void)saved;
    count(hi, true);
}

inline uint16_t f2h(float f) { return (uint16_t)_cvtss_sh(f, _MM_FROUND_TO_NEAREST_INT | _MM_FROUND_NO_EXC); }

// g_buffer.frag:47-51
inline void direction_to_octohedral(V3 n, float out[2])
{
    float inv = 1.0f / (std::fabs(n.x) + std::fabs(n.y) + std::fabs(n.z));
    float px = n.x * inv, py = n.y * inv;
    if (n.z > 0.0f) { out[0] = px; out[1] = py; }
    else
    {
        out[0] = (1.0f - std::fabs(py)) * (px >= 0.0f ? 1.0f : -1.0f);
        out[1] = (1.0f - std::fabs(px)) * (py >= 0.0f ? 1.0f : -1.0f);
    }
}

} // namespace

// ------------------------------------------------------------------------------------------------
void hrs_scene::finalize()
{
    tris.clear();
    for (uint32_t ii = 0; ii < instances.size(); ii++)
    {
        const hr_instance& in = instances[ii];
        M4                 model;
        memcpy(model.m, in.model, 64);
        for (uint32_t k = 0; k + 2 < in.index_count; k += 3)
        {
            V3 p[3], n[3];
            for (int j = 0; j < 3; j++)
            {
                const hr_vertex& v = vertices[in.base_vertex + indices[in.first_index + k + j]];
                float            pin[4] = { v.position[0], v.position[1], v.position[2], 1.0f }, po[4];
                mul_point(model, pin, po);
                p[j] = { po[0], po[1], po[2] };
                float nin[4] = { v.normal[0], v.normal[1], v.normal[2], 0.0f }, no[4];
                mul_point(model, nin, no);
                n[j] = normalize(V3 { no[0], no[1], no[2] });
            }
            tris.push_back({ p[0], p[1] - p[0], p[2] - p[0], n[0], n[1], n[2], ii, p[1], p[2] });
        }
    }
    size_t n = tris.size();
    std::vector<V3> cen(n), tmin(n), tmax(n);
    bmin = { FLT_MAX, FLT_MAX, FLT_MAX };
    bmax = { -FLT_MAX, -FLT_MAX, -FLT_MAX };
    for (size_t i = 0; i < n; i++)
    {
        V3 a = tris[i].v0, b = tris[i].v1, c = tris[i].v2;
        tmin[i] = { std::min({ a.x, b.x, c.x }), std::min({ a.y, b.y, c.y }), std::min({ a.z, b.z, c.z }) };
        tmax[i] = { std::max({ a.x, b.x, c.x }), std::max({ a.y, b.y, c.y }), std::max({ a.z, b.z, c.z }) };
        cen[i]  = (tmin[i] + tmax[i]) * 0.5f;
        bmin = { std::min(bmin.x, tmin[i].x), std::min(bmin.y, tmin[i].y), std::min(bmin.z, tmin[i].z) };
        bmax = { std::max(bmax.x, tmax[i].x), std::max(bmax.y, tmax[i].y), std::max(bmax.z, tmax[i].z) };
    }
    std::vector<uint32_t> order(n);
    std::iota(order.begin(), order.end(), 0u);
    nodes.clear();
    if (n) build_rec(0, (int)n, cen, tmin, tmax, order);
    bvh_tris.resize(n);
    for (size_t i = 0; i < n; i++) bvh_tris[i] = tris[order[i]];
}

int hrs_scene::build_rec(int first, int last, std::vector<V3>& cen, std::vector<V3>& tmin, std::vector<V3>& tmax, std::vector<uint32_t>& order)
{
    int idx = (int)nodes.size();
    nodes.push_back({});
    V3 lo = { FLT_MAX, FLT_MAX, FLT_MAX }, hi = { -FLT_MAX, -FLT_MAX, -FLT_MAX }, clo = lo, chi = hi;
    for (int i = first; i < last; i++)
    {
        uint32_t t = order[i];
        lo  = { std::min(lo.x, tmin[t].x), std::min(lo.y, tmin[t].y), std::min(lo.z, tmin[t].z) };
        hi  = { std::max(hi.x, tmax[t].x), std::max(hi.y, tmax[t].y), std::max(hi.z, tmax[t].z) };
        clo = { std::min(clo.x, cen[t].x), std::min(clo.y, cen[t].y), std::min(clo.z, cen[t].z) };
        chi = { std::max(chi.x, cen[t].x), std::max(chi.y, cen[t].y), std::max(chi.z, cen[t].z) };
    }
    const float pad = 1e-4f;
    Node nd;
    nd.lo[0] = lo.x - pad; nd.lo[1] = lo.y - pad; nd.lo[2] = lo.z - pad;
    nd.hi[0] = hi.x + pad; nd.hi[1] = hi.y + pad; nd.hi[2] = hi.z + pad;
    nd.left = nd.right = -1;
    nd.first = first;
    nd.count = 0;
    int n = last - first;
    if (n <= 4) { nd.count = n; nodes[idx] = nd; return idx; }
    float ex = chi.x - clo.x, ey = chi.y - clo.y, ez = chi.z - clo.z;
    int   ax = (ex >= ey && ex >= ez) ? 0 : (ey >= ez ? 1 : 2);
    int   mid = (first + last) / 2;
    auto  key = [&](uint32_t t) { return ax == 0 ? cen[t].x : (ax == 1 ? cen[t].y : cen[t].z); };
    std::nth_element(order.begin() + first, order.begin() + mid, order.begin() + last, [&](uint32_t a, uint32_t b) { return key(a) < key(b); });
    nodes[idx] = nd;
    int l = build_rec(first, mid, cen, tmin, tmax, order);
    int r = build_rec(mid, last, cen, tmin, tmax, order);
    nodes[idx].left  = l;
    nodes[idx].right = r;
    return idx;
}

bool hrs_scene::closest(V3 o, V3 d, float tmax, float& bt, float& bu, float& bv, uint32_t& prim) const
{
    bt   = tmax;
    prim = 0xFFFFFFFFu;
    if (nodes.empty()) return false;
    const float inv[3] = { 1.0f / d.x, 1.0f / d.y, 1.0f / d.z }, oo[3] = { o.x, o.y, o.z };
    int         stack[128], sp = 0;
    stack[sp++] = 0;
    while (sp)
    {
        const Node& n  = nodes[stack[--sp]];
        float       t0 = 0.0f, t1 = bt;
        for (int a = 0; a < 3; a++)
        {
            float ta = (n.lo[a] - oo[a]) * inv[a], tb = (n.hi[a] - oo[a]) * inv[a];
            t0 = std::max(t0, std::min(ta, tb) == std::min(ta, tb) ? std::min(ta, tb) : t0);
            t1 = std::min(t1, std::max(ta, tb) == std::max(ta, tb) ? std::max(ta, tb) : t1);
        }
        if (t0 > t1 * 1.000001f) continue;
        if (n.count)
        {
            for (int i = 0; i < n.count; i++)
            {
                const Tri& tr  = bvh_tris[n.first + i];
                V3         p   = cross(d, tr.e2);
                float      det = dot(tr.e1, p);
                if (det == 0.0f) continue;
                float idet = 1.0f / det;
                V3    tv   = o - tr.v0;
                float u    = dot(tv, p) * idet;
                if (!(u >= 0.0f && u <= 1.0f)) continue;
                V3    q = cross(tv, tr.e1);
                float v = dot(d, q) * idet;
                if (!(v >= 0.0f && u + v <= 1.0f)) continue;
                float t = dot(tr.e2, q) * idet;
                if (t > 0.0f && t < bt) { bt = t; bu = u; bv = v; prim = (uint32_t)(n.first + i); }
            }
        }
        else { stack[sp++] = n.left; stack[sp++] = n.right; }
    }
    return prim != 0xFFFFFFFFu;
}

// ================================================================================================
extern "C" {

hrs_scene* hrs_scene_create(int kind, int target_tris, uint32_t seed)
{
    hrs_scene* s = new hrs_scene();
    switch (kind)
    {
        case HRS_SCENE_SINGLE_TRIANGLE: build_single_triangle(*s); break;
        case HRS_SCENE_GROUND_PLANE: build_ground_plane(*s); break;
        case HRS_SCENE_SHADOWS_TEST: build_shadows_test(*s, seed); break;
        case HRS_SCENE_ARCADE: build_arcade(*s, target_tris > 0 ? target_tris : 262144, seed); break;
        default: delete s; return nullptr;
    }
    s->finalize();
    return s;
}
void hrs_scene_destroy(hrs_scene* s) { delete s; }
void hrs_scene_counts(const hrs_scene* s, uint64_t* nv, uint64_t* ni, uint64_t* nin, uint64_t* nm)
{
    if (nv) *nv = s->vertices.size();
    if (ni) *ni = s->indices.size();
    if (nin) *nin = s->instances.size();
    if (nm) *nm = s->materials.size();
}
const hr_vertex*   hrs_scene_vertices(const hrs_scene* s) { return s->vertices.data(); }
const uint32_t*    hrs_scene_indices(const hrs_scene* s) { return s->indices.data(); }
const hr_instance* hrs_scene_instances(const hrs_scene* s) { return s->instances.data(); }
const hr_material* hrs_scene_materials(const hrs_scene* s) { return s->materials.data(); }
void hrs_scene_bounds(const hrs_scene* s, float mn[3], float mx[3])
{
    mn[0] = s->bmin.x; mn[1] = s->bmin.y; mn[2] = s->bmin.z;
    mx[0] = s->bmax.x; mx[1] = s->bmax.y; mx[2] = s->bmax.z;
}
void hrs_scene_world_triangles(const hrs_scene* s, float* out9, uint32_t* prim_instance)
{
    for (size_t i = 0; i < s->tris.size(); i++)
    {
        const hrs_scene::Tri& t = s->tris[i];
        V3 a = t.v0, b = t.v1, c = t.v2;
        if (out9)
        {
            float* o = out9 + 9 * i;
            o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = b.x; o[4] = b.y; o[5] = b.z; o[6] = c.x; o[7] = c.y; o[8] = c.z;
        }
        if (prim_instance) prim_instance[i] = t.inst;
    }
}

void hrs_scene_world_normals(const hrs_scene* s, float* out9, uint32_t* prim_material)
{
    for (size_t i = 0; i < s->tris.size(); i++)
    {
        const hrs_scene::Tri& t = s->tris[i];
        if (out9)
        {
            float* o = out9 + 9 * i;
            o[0] = t.n0.x; o[1] = t.n0.y; o[2] = t.n0.z; o[3] = t.n1.x; o[4] = t.n1.y; o[5] = t.n1.z; o[6] = t.n2.x; o[7] = t.n2.y; o[8] = t.n2.z;
        }
        if (prim_material) prim_material[i] = s->instances[t.inst].material_idx;
    }
}

void hrs_default_light(hrs_light_desc* l)
{
    memset(l, 0, sizeof(*l));
    l->type      = HR_LIGHT_DIRECTIONAL;
    l->rot_y_deg = 50.0f;
    l->rot_x_deg = 50.0f;
    l->radius    = 0.1f;
    l->intensity = 1.0f;
    l->color[0] = l->color[1] = l->color[2] = 1.0f;
    l->cone_inner_deg = 40.0f;
    l->cone_outer_deg = 50.0f;
}

void hrs_make_frame(hr_frame* out, const float cam_pos[3], const float cam_target[3], int width, int height, const hrs_light_desc* light,
                    const hr_frame* prev, uint32_t num_frames)
{
    const float up[3] = { 0.0f, 1.0f, 0.0f };
    hrs_make_frame_ex(out, cam_pos, cam_target, up, 60.0f, 1.0f, 1000.0f, width, height, light, prev, num_frames); // src/common.h:19-20
}

void hrs_make_frame_ex(hr_frame* out, const float cam_pos[3], const float cam_target[3], const float cam_up[3], float fovy_deg, float kNear,
                       float kFar, int width, int height, const hrs_light_desc* light, const hr_frame* prev, uint32_t num_frames)
{
    memset(out, 0, sizeof(*out));
    const float rad   = 3.14159265358979f / 180.0f;
    V3 pos = { cam_pos[0], cam_pos[1], cam_pos[2] }, tgt = { cam_target[0], cam_target[1], cam_target[2] };
    M4 proj = perspective(fovy_deg * rad, (float)width / (float)height, kNear, kFar);
    M4 view = look_at(pos, tgt, { cam_up[0], cam_up[1], cam_up[2] });
    M4 vp   = mul(proj, view);
    M4 vpi = inverse(vp), vi = inverse(view), pi = inverse(proj);
    memcpy(out->ubo.view_inverse, vi.m, 64);
    memcpy(out->ubo.proj_inverse, pi.m, 64);
    memcpy(out->ubo.view_proj_inverse, vpi.m, 64);
    memcpy(out->ubo.view_proj, vp.m, 64);
    if (prev) memcpy(out->ubo.prev_view_proj, prev->ubo.view_proj, 64);
    else { M4 id = identity(); memcpy(out->ubo.prev_view_proj, id.m, 64); } // Camera ctor: m_prev_view_projection = mat4(1), camera.cpp:25
    out->ubo.cam_pos[0] = pos.x; out->ubo.cam_pos[1] = pos.y; out->ubo.cam_pos[2] = pos.z; out->ubo.cam_pos[3] = 1.0f;
    // light (main.cpp:948-966)
    hrs_light_desc dl;
    if (!light) { hrs_default_light(&dl); light = &dl; }
    M4 lt = mul(rotate_axis(light->rot_y_deg * rad, { 0, 1, 0 }), rotate_axis(light->rot_x_deg * rad, { 1, 0, 0 }));
    float din[4] = { 0, -1, 0, 0 }, dout[4];
    mul_point(lt, din, dout);
    V3 ldir = normalize(V3 { dout[0], dout[1], dout[2] });
    hr_light& L = out->ubo.light;
    L.data0[0] = -ldir.x; L.data0[1] = -ldir.y; L.data0[2] = -ldir.z; L.data0[3] = light->intensity;
    L.data1[0] = light->position[0]; L.data1[1] = light->position[1]; L.data1[2] = light->position[2]; L.data1[3] = light->radius;
    L.data2[0] = light->color[0]; L.data2[1] = light->color[1]; L.data2[2] = light->color[2];
    L.data3[0] = (float)light->type;
    L.data3[1] = std::cos(light->cone_outer_deg * rad);
    L.data3[2] = std::cos(light->cone_inner_deg * rad);
    out->num_frames  = num_frames;
    out->first_frame = prev ? 0 : 1;
    out->ping_pong   = prev ? !prev->ping_pong : 0; // main.cpp:128
    float zx = -1.0f + kNear / kFar;
    out->z_buffer_params[0] = zx; out->z_buffer_params[1] = 1.0f; out->z_buffer_params[2] = zx / kNear; out->z_buffer_params[3] = 1.0f / kNear; // main.cpp:253-254
    if (prev)
    {
        out->camera_delta[0] = pos.x - prev->ubo.cam_pos[0];
        out->camera_delta[1] = pos.y - prev->ubo.cam_pos[1];
        out->camera_delta[2] = pos.z - prev->ubo.cam_pos[2];
    }
    out->frame_time = 1.0f / 60.0f;
}

void hrs_write_gbuffer(const hrs_scene* vis, const hr_frame* frame, int W, int H, uint8_t* gb1, uint16_t* gb2, uint16_t* gb3, float* depth)
{
    M4 vpi, vp, pvp;
    memcpy(vpi.m, frame->ubo.view_proj_inverse, 64);
    memcpy(vp.m, frame->ubo.view_proj, 64);
    memcpy(pvp.m, frame->ubo.prev_view_proj, 64);
    std::vector<V3>       nrm((size_t)W * H);
    std::vector<uint32_t> mid((size_t)W * H, 0xFFFFFFFFu);
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++)
        {
            size_t pi = (size_t)y * W + x;
            float  nx = ((float)x + 0.5f) / (float)W * 2.0f - 1.0f, ny = ((float)y + 0.5f) / (float)H * 2.0f - 1.0f;
            float  a[4] = { nx, ny, 0.0f, 1.0f }, b[4] = { nx, ny, 1.0f, 1.0f }, wa[4], wb[4];
            mul_point(vpi, a, wa);
            mul_point(vpi, b, wb);
            V3 o = { wa[0] / wa[3], wa[1] / wa[3], wa[2] / wa[3] }, e = { wb[0] / wb[3], wb[1] / wb[3], wb[2] / wb[3] };
            V3 dv = e - o;
            float len = length(dv);
            V3    d   = dv * (1.0f / len);
            float    t, u, v;
            uint32_t prim;
            bool     hit = vis->closest(o, d, len, t, u, v, prim);
            float    dz  = 1.0f;
            if (hit)
            {
                const hrs_scene::Tri& tr = vis->bvh_tris[prim];
                V3    P = o + d * t;
                float pin[4] = { P.x, P.y, P.z, 1.0f }, c[4], pc[4];
                mul_point(vp, pin, c);
                mul_point(pvp, pin, pc);
                dz = c[2] / c[3];
                if (!(dz >= 0.0f && dz < 1.0f)) hit = false;
                else
                {
                    V3 n = normalize(tr.n0 * (1.0f - u - v) + tr.n1 * u + tr.n2 * v);
                    float oct[2];
                    direction_to_octohedral(n, oct);
                    float cu = c[0] / c[3] * 0.5f + 0.5f, cv = c[1] / c[3] * 0.5f + 0.5f;
                    float pu = pc[0] / pc[3] * 0.5f + 0.5f, pv = pc[1] / pc[3] * 0.5f + 0.5f;
                    const hr_material& m = vis->materials[vis->instances[tr.inst].material_idx];
                    uint16_t* g2 = gb2 + 4 * pi;
                    uint16_t* g3 = gb3 + 4 * pi;
                    g2[0] = f2h(oct[0]); g2[1] = f2h(oct[1]); g2[2] = f2h(pu - cu); g2[3] = f2h(pv - cv);
                    g3[0] = f2h(m.roughness); g3[1] = 0; g3[2] = f2h((float)tr.inst); g3[3] = f2h(c[2]); // linear_z = gl_FragCoord.z / gl_FragCoord.w = z_clip
                    depth[pi] = dz;
                    if (gb1)
                    {
                        uint8_t* g1 = gb1 + 4 * pi;
                        for (int k = 0; k < 3; k++) g1[k] = (uint8_t)std::min(255.0f, std::max(0.0f, m.albedo[k] * 255.0f + 0.5f));
                        g1[3] = (uint8_t)std::min(255.0f, std::max(0.0f, m.metallic * 255.0f + 0.5f));
                    }
                    nrm[pi] = n;
                    mid[pi] = tr.inst;
                }
            }
            if (!hit)
            { // clears: g_buffer.cpp:72-96 (GB3.w = -1, depth = 1)
                uint16_t* g2 = gb2 + 4 * pi;
                uint16_t* g3 = gb3 + 4 * pi;
                g2[0] = g2[1] = g2[2] = g2[3] = 0;
                g3[0] = g3[1] = g3[2] = 0;
                g3[3] = f2h(-1.0f);
                depth[pi] = 1.0f;
                if (gb1) memset(gb1 + 4 * pi, 0, 4);
            }
        }
    // curvature = sqrt(max(|dFdx N|^2, |dFdy N|^2)) per 2x2 quad (g_buffer.frag:71-80); 0 across mesh boundaries.
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++)
        {
            size_t pi = (size_t)y * W + x;
            if (mid[pi] == 0xFFFFFFFFu) continue;
            int    x0 = x & ~1, y0 = y & ~1, x1 = std::min(x0 + 1, W - 1), y1 = std::min(y0 + 1, H - 1);
            size_t ax = (size_t)y * W + x0, bx = (size_t)y * W + x1, ay = (size_t)y0 * W + x, by = (size_t)y1 * W + x;
            float  cx = 0, cy = 0;
            if (mid[ax] == mid[pi] && mid[bx] == mid[pi]) { V3 dd = nrm[bx] - nrm[ax]; cx = dot(dd, dd); }
            if (mid[ay] == mid[pi] && mid[by] == mid[pi]) { V3 dd = nrm[by] - nrm[ay]; cy = dot(dd, dd); }
            float curv = std::sqrt(std::max(cx, cy));
            if (curv < 1e-4f) curv = 0.0f; // flat surfaces give exactly 0 in the rasteriser (constant interpolant)
            gb3[4 * pi + 1] = f2h(curv);
        }
}

void hrs_blue_noise(uint32_t seed, uint8_t* sobol, uint8_t* sr)
{
    // Sobol' dims 0..3, Joe-Kuo direction numbers (s,a,m): d1 = van der Corput; d2: (1,0,[1]); d3: (2,1,[1,3]); d4: (3,1,[1,3,1])
    uint32_t V[4][32];
    for (int i = 0; i < 32; i++) V[0][i] = 1u << (31 - i);
    const int      S[3]    = { 1, 2, 3 };
    const uint32_t A[3]    = { 0, 1, 1 };
    const uint32_t Mi[3][3] = { { 1, 0, 0 }, { 1, 3, 0 }, { 1, 3, 1 } };
    for (int d = 0; d < 3; d++)
    {
        int s = S[d];
        for (int i = 0; i < s; i++) V[d + 1][i] = Mi[d][i] << (31 - i);
        for (int i = s; i < 32; i++)
        {
            uint32_t v = V[d + 1][i - s] ^ (V[d + 1][i - s] >> s);
            for (int k = 1; k < s; k++) v ^= (((A[d] >> (s - 1 - k)) & 1u) * V[d + 1][i - k]);
            V[d + 1][i] = v;
        }
    }
    for (int idx = 0; idx < 256; idx++)
        for (int d = 0; d < 4; d++)
        {
            uint32_t x = 0;
            for (int b = 0; b < 8; b++)
                if (idx & (1 << b)) x ^= V[d][b];
            sobol[4 * idx + d] = (uint8_t)(x >> 24);
        }
    Rng rng(seed);
    for (int i = 0; i < 128 * 128 * 4; i++) sr[i] = (uint8_t)(rng.next() & 0xFF);
}

// Stand-in for textures/brdf_lut.bin (release-zip asset): the usual split-sum environment-BRDF integral (Karis 2013) over a
// Hammersley / GGX-importance-sampled hemisphere; texel (i, j): N.V = (i + .5) / 512, roughness = (j + .5) / 512; RG16F.
void hrs_brdf_lut(int samples, uint16_t* out_512x512x2)
{
    const int N = 512;
    if (samples < 16) samples = 16;
#pragma omp parallel for schedule(dynamic, 4)
    for (int j = 0; j < N; j++)
        for (int i = 0; i < N; i++)
        {
            const float ndv = ((float)i + 0.5f) / N, rough = ((float)j + 0.5f) / N;
            const float vx = std::sqrt(1.0f - ndv * ndv), vz = ndv;
            const float a = rough * rough, k = a / 2.0f;
            float A = 0.0f, B = 0.0f;
            for (int s = 0; s < samples; s++)
            {
                uint32_t bits = (uint32_t)s;
                bits = (bits << 16) | (bits >> 16);
                bits = ((bits & 0x55555555u) << 1) | ((bits & 0xAAAAAAAAu) >> 1);
                bits = ((bits & 0x33333333u) << 2) | ((bits & 0xCCCCCCCCu) >> 2);
                bits = ((bits & 0x0F0F0F0Fu) << 4) | ((bits & 0xF0F0F0F0u) >> 4);
                bits = ((bits & 0x00FF00FFu) << 8) | ((bits & 0xFF00FF00u) >> 8);
                const float e1 = (float)s / (float)samples, e2 = (float)bits * 2.3283064365386963e-10f;
                const float phi = 6.28318530718f * e1, ct = std::sqrt((1.0f - e2) / (1.0f + (a * a - 1.0f) * e2)), st = std::sqrt(1.0f - ct * ct);
                const float hx = std::cos(phi) * st, hy = std::sin(phi) * st, hz = ct;
                const float vdh = vx * hx + vz * hz;
                const float lz  = 2.0f * vdh * hz - vz;
                (void)hy;
                const float ndl = std::max(lz, 0.0f), ndh = std::max(hz, 0.0f), vh = std::max(vdh, 0.0f);
                if (ndl > 0.0f)
                {
                    const float g = (ndv / (ndv * (1.0f - k) + k)) * (ndl / (ndl * (1.0f - k) + k));
                    const float gv = g * vh / std::max(ndh * ndv, 1e-6f), fc = std::pow(1.0f - vh, 5.0f);
                    A += (1.0f - fc) * gv;
                    B += fc * gv;
                }
            }
            out_512x512x2[2 * ((size_t)j * N + i)]     = f2h(A / samples);
            out_512x512x2[2 * ((size_t)j * N + i) + 1] = f2h(B / samples);
        }
}

} // extern "C"
