// gbuffer.cu — G-buffer producer on the device (SURVEY.md §8 f1): replaces the reference's raster G-buffer pass
//   src/g_buffer.cpp:100-263 (attachments :254-263, clears :72-96), src/shaders/g_buffer.vert,
//   src/shaders/g_buffer.frag:47-51 (direction_to_octohedral), :55-67 (compute_motion_vector), :71-80 (compute_curvature), :87-111
// with a primary-visibility ray cast over the scene's BVH, so that a headless frame needs no host -> device G-buffer upload
// (199 MB per 4K frame over PCIe otherwise).  One warp = one 8x4 pixel block (the 2x2 derivative quads of compute_curvature
// live inside a warp: lane ^ 1 is the x partner, lane ^ 8 the y partner).
//
// BUILD NOTE: compiled with -fmad=false.  Every output is a fixed sequence of binary32 operations shared with the CPU
// statement oracle/orc_gbuffer.cpp (see its header for the sequence); the two agree bit for bit on all four images.
#include "traverse.cuh"

namespace {

using det::V3;
using namespace trv;

struct GbufScene {
    const float4*      vnormals;  // 3 per primitive, world-space unit vertex normals
    const uint32_t*    prim_inst; // mesh id per primitive (g_buffer.cpp:140-176: increments per drawn sub-mesh)
    const uint32_t*    prim_mat;
    const hr_material* materials;
};

struct GbufParams {
    float vpi[16], vp[16], pvp[16];
    int    W, H;
    RowSet rows;
};

__device__ __forceinline__ float4 mul_m4(const float* M, V3 p)
{ // mat4 * vec4(p, 1), row r = ((m0r*x + m1r*y) + m2r*z) + m3r*1
    return make_float4(((M[0] * p.x + M[4] * p.y) + M[8] * p.z) + M[12] * 1.0f, ((M[1] * p.x + M[5] * p.y) + M[9] * p.z) + M[13] * 1.0f,
                       ((M[2] * p.x + M[6] * p.y) + M[10] * p.z) + M[14] * 1.0f, ((M[3] * p.x + M[7] * p.y) + M[11] * p.z) + M[15] * 1.0f);
}

__device__ __forceinline__ uint32_t pack_h2(float a, float b)
{
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

__device__ __forceinline__ uint32_t unorm8(float v)
{
    const float s = v * 255.0f + 0.5f;
    return (uint32_t)(s < 0.0f ? 0.0f : (s > 255.0f ? 255.0f : s));
}

// TEX: material textures bound (hr_scene_set_textures): albedo / metallic / roughness of GB1 / GB3 come from fetch_albedo / fetch_metallic /
// fetch_roughness at the hit (g_buffer.frag:90-105), sampled at mip 0 (a ray cast has no screen-space derivatives; the raster pass filters
// trilinearly).  The untextured instantiation compiles exactly as before.
template <bool TEX>
__global__ void __launch_bounds__(64) k_gbuffer_render(BvhDev bvh, GbufScene sc, GbufParams P, uint32_t* __restrict__ gb1, uint2* __restrict__ gb2, uint2* __restrict__ gb3,
                                                        float* __restrict__ depth, unsigned long long* ray_ctr, tex::TexDev T)
{
    __shared__ int s_stack[2][STACK_SIZE]; // one packet-traversal stack per warp
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int       x, y;
    P.rows.pixel(x, y);
    const int  y_end = P.rows.end(P.H);
    const bool in_img = x < P.W && y < P.H && y < y_end;
    V3       N   = det::mk(0.0f, 0.0f, 0.0f);
    uint32_t mid = 0xFFFFFFFFu;
    uint32_t g2x = 0u, g2y = 0u, g3x = 0u, g3w_mid = 0u, g1 = 0u;
    float    dz  = 1.0f, linz = -1.0f, fmid = 0.0f;
    // primary rays of an 8x4 block are coherent: packet traversal (traverse.cuh), warp-uniform control flow.  Lanes outside the
    // image carry a dummy ray and stay inactive.
    Ray r;
    V3  o = det::mk(0.0f, 0.0f, 0.0f);
    r.o = o; r.d = det::mk(0.0f, 0.0f, 1.0f); r.tmin = 0.0f; r.tmax = 0.0f;
    if (in_img)
    {
        const float u = ((float)x + 0.5f) / (float)P.W, v = ((float)y + 0.5f) / (float)P.H;
        o = det::world_position_from_depth(u, v, 0.0f, P.vpi);
        const V3    e   = det::world_position_from_depth(u, v, 1.0f, P.vpi);
        const V3    dv  = det::sub(e, o);
        const float len = det::length(dv);
        r.o    = o;
        r.d    = det::scale(dv, 1.0f / len);
        r.tmax = len;
        count_rays(ray_ctr, 0, 1u);
    }
    float    t, hu, hv;
    uint32_t prim;
    const bool hit = trace_closest_packet(bvh, r, in_img, s_stack[warp], t, prim, hu, hv);
    if (in_img)
    {
        if (hit)
        {
            const V3     Pw = det::add(o, det::scale(r.d, t));
            const float4 c = mul_m4(P.vp, Pw), pc = mul_m4(P.pvp, Pw);
            const float  d = c.z / c.w;
            if (d >= 0.0f && d < 1.0f)
            {
                const float4 n0 = __ldg(sc.vnormals + 3ull * prim), n1 = __ldg(sc.vnormals + 3ull * prim + 1), n2 = __ldg(sc.vnormals + 3ull * prim + 2);
                const float  b0 = 1.0f - hu - hv;
                N = det::normalize(det::add(det::add(det::scale(det::mk(n0.x, n0.y, n0.z), b0), det::scale(det::mk(n1.x, n1.y, n1.z), hu)), det::scale(det::mk(n2.x, n2.y, n2.z), hv)));
                V3 Ne = N; // the encoded normal: fetch_normal (g_buffer.frag:100); compute_curvature keeps using the interpolated normal (:73-74)
                if (TEX) tex::normal_at_hit(T, __ldg(sc.prim_mat + prim), prim, b0, hu, hv, false, Ne.x, Ne.y, Ne.z);
                const float inv = 1.0f / ((fabsf(Ne.x) + fabsf(Ne.y)) + fabsf(Ne.z)); // direction_to_octohedral, g_buffer.frag:47-51
                const float px = Ne.x * inv, py = Ne.y * inv;
                float       ox = px, oy = py;
                if (!(Ne.z > 0.0f))
                {
                    ox = (1.0f - fabsf(py)) * (px >= 0.0f ? 1.0f : -1.0f);
                    oy = (1.0f - fabsf(px)) * (py >= 0.0f ? 1.0f : -1.0f);
                }
                const float cu = (c.x / c.w) * 0.5f + 0.5f, cv = (c.y / c.w) * 0.5f + 0.5f; // compute_motion_vector :55-67
                const float pu = (pc.x / pc.w) * 0.5f + 0.5f, pv = (pc.y / pc.w) * 0.5f + 0.5f;
                const hr_material* m = sc.materials + __ldg(sc.prim_mat + prim);
                mid  = __ldg(sc.prim_inst + prim);
                fmid = (float)mid;
                g2x  = pack_h2(ox, oy);
                g2y  = pack_h2(pu - cu, pv - cv);
                linz = c.z; // gl_FragCoord.z / gl_FragCoord.w = z_clip, g_buffer.frag:107
                dz   = d;
                if (TEX)
                {
                    float ar = m->albedo[0], ag = m->albedo[1], ab = m->albedo[2], rough = m->roughness, metal = m->metallic;
                    tex::material_at_hit(T, __ldg(sc.prim_mat + prim), prim, b0, hu, hv, ar, ag, ab, rough, metal);
                    g3x = pack_h2(rough, 0.0f);
                    g1  = unorm8(ar) | (unorm8(ag) << 8) | (unorm8(ab) << 16) | (unorm8(metal) << 24);
                }
                else
                {
                    g3x = pack_h2(m->roughness, 0.0f);
                    g1  = unorm8(m->albedo[0]) | (unorm8(m->albedo[1]) << 8) | (unorm8(m->albedo[2]) << 16) | (unorm8(m->metallic) << 24);
                }
            }
        }
    }
    // compute_curvature (:71-80): fine differences inside the 2x2 quad, 0 across mesh boundaries.  The quad partners are
    // lanes (lane & ~1, lane | 1) in x and (lane & ~8, lane | 8) in y; a partner outside the image is the pixel itself.
    const uint32_t full = 0xFFFFFFFFu;
    const int      lx0 = lane & ~1, lx1 = lane | 1, ly0 = lane & ~8, ly1 = lane | 8;
    const bool     x1_in = (x | 1) < P.W, y1_in = (y | 1) < P.H && (y | 1) < y_end; // row1 is a multiple of 4 or H
    V3 ax, bx, ay, by;
    ax.x = __shfl_sync(full, N.x, lx0); ax.y = __shfl_sync(full, N.y, lx0); ax.z = __shfl_sync(full, N.z, lx0);
    bx.x = __shfl_sync(full, N.x, lx1); bx.y = __shfl_sync(full, N.y, lx1); bx.z = __shfl_sync(full, N.z, lx1);
    ay.x = __shfl_sync(full, N.x, ly0); ay.y = __shfl_sync(full, N.y, ly0); ay.z = __shfl_sync(full, N.z, ly0);
    by.x = __shfl_sync(full, N.x, ly1); by.y = __shfl_sync(full, N.y, ly1); by.z = __shfl_sync(full, N.z, ly1);
    const uint32_t max_ = __shfl_sync(full, mid, lx0), mbx = __shfl_sync(full, mid, lx1), may = __shfl_sync(full, mid, ly0), mby = __shfl_sync(full, mid, ly1);
    if (!in_img) return;
    const size_t pi = (size_t)y * P.W + x;
    if (mid != 0xFFFFFFFFu)
    {
        float cx = 0.0f, cy = 0.0f;
        if (x1_in && max_ == mid && mbx == mid) { const V3 dd = det::sub(bx, ax); cx = det::dot(dd, dd); }
        if (y1_in && may == mid && mby == mid) { const V3 dd = det::sub(by, ay); cy = det::dot(dd, dd); }
        float curv = sqrtf(fmaxf(cx, cy));
        if (curv < 1e-4f) curv = 0.0f;
        const __half hc = __float2half_rn(curv);
        g3x = (g3x & 0xFFFFu) | ((uint32_t)__half_as_ushort(hc) << 16);
        g3w_mid = pack_h2(fmid, linz);
    }
    else g3w_mid = pack_h2(0.0f, -1.0f); // clears, g_buffer.cpp:72-96: GB3 = (0, 0, 0, -1), depth = 1
    gb2[pi]   = make_uint2(g2x, g2y);
    gb3[pi]   = make_uint2(g3x, g3w_mid);
    depth[pi] = dz;
    if (gb1) gb1[pi] = g1;
}

} // namespace

void launch_gbuffer_render(const hr_scene* sc, const hr_frame* f, int W, int H, RowSet rows, void* gb1, void* gb2, void* gb3, float* depth, unsigned long long* ray_ctr,
                           cudaStream_t st)
{
    if (rows.empty(H)) return;
    GbufScene gs { sc->d_vnormals, sc->d_prim_inst, sc->d_prim_mat, sc->d_materials };
    GbufParams P;
    memcpy(P.vpi, f->ubo.view_proj_inverse, 64);
    memcpy(P.vp, f->ubo.view_proj, 64);
    memcpy(P.pvp, f->ubo.prev_view_proj, 64);
    P.W = W; P.H = H; P.rows = rows;
    const dim3 grid = rows.grid(W, H);
    if (sc->tex.n_textures > 0) k_gbuffer_render<true><<<grid, 64, 0, st>>>(hr_bvh_view(sc), gs, P, (uint32_t*)gb1, (uint2*)gb2, (uint2*)gb3, depth, ray_ctr, sc->tex);
    else k_gbuffer_render<false><<<grid, 64, 0, st>>>(hr_bvh_view(sc), gs, P, (uint32_t*)gb1, (uint2*)gb2, (uint2*)gb3, depth, ray_ctr, sc->tex);
}
