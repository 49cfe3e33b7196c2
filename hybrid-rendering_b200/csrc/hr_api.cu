// hr_api.cu — implementation of the C ABI declared in include/hr_api.h.
// Host sequencing mirrors the reference's pass classes:
//   RayTracedShadows::render  src/ray_traced_shadows.cpp:100-116 (+ stages :938-1255)
//   RayTracedAO::render       src/ray_traced_ao.cpp:98-112      (+ stages :829-1137)
#include "hr_internal.h"
#include <utility>
#include <cstdarg>
#include <cstring>
#include <atomic>
#include <mutex>

static std::string g_last_error;
static std::mutex  g_err_mutex;

void hr_set_error(hr_ctx* ctx, const char* fmt, ...)
{
    char    buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    std::lock_guard<std::mutex> lk(g_err_mutex);
    g_last_error = buf;
    if (ctx) ctx->last_error = buf;
}

static int round_up8(int v) { return (v + 7) & ~7; }

// scrambling / ranking table a pass rendered with `spp` samples reads (hr_bluenoise_set_slot)
static const uint8_t* bn_table(const hr_ctx* ctx, int spp)
{
    if (spp > 1 && (spp & (spp - 1)) == 0)
    {
        int slot = 0;
        while ((1 << slot) < spp) slot++;
        if (slot <= 8 && ctx->d_scr_rank_slot[slot]) return ctx->d_scr_rank_slot[slot];
    }
    return ctx->d_scr_rank;
}

static FrameConsts make_consts(const hr_frame* f, const hr_pass* p)
{
    FrameConsts c;
    c.ray_ctr = p ? p->ray_ctr : nullptr;
    memcpy(c.view_proj_inverse, f->ubo.view_proj_inverse, 64);
    memcpy(c.prev_view_proj, f->ubo.prev_view_proj, 64);
    memcpy(c.cam_pos, f->ubo.cam_pos, 16);
    c.light = f->ubo.light;
    memcpy(c.z_buffer_params, f->z_buffer_params, 16);
    memcpy(c.camera_delta, f->camera_delta, 12);
    c.num_frames = f->num_frames;
    return c;
}

// extent of mip `mip` of an image `v` texels wide (or high): halved per level, never below 1
static int mip_extent(int v, int mip)
{
    for (int m = 0; m < mip; m++) v = v / 2 > 0 ? v / 2 : 1;
    return v;
}

static GBufLevelDev level_view(const hr_ctx* ctx, int slot, int mip)
{
    GBufLevelDev l;
    l.W     = mip_extent(ctx->gb_w, mip);
    l.H     = mip_extent(ctx->gb_h, mip);
    l.gb1   = (const uint32_t*)ctx->slot[slot].gb1[mip];
    l.gb2   = (const uint2*)ctx->slot[slot].gb2[mip];
    l.gb3   = (const uint2*)ctx->slot[slot].gb3[mip];
    l.depth = ctx->slot[slot].depth[mip];
    return l;
}

// ---- stage timing (DW_SCOPED_SAMPLE equivalent) ---------------------------------------------------------------
static cudaEvent_t timer_event(hr_pass* p)
{
    cudaEvent_t e;
    if (!p->timer.pool.empty()) { e = p->timer.pool.back(); p->timer.pool.pop_back(); }
    else cudaEventCreate(&e);
    return e;
}
static void timer_begin(hr_pass* p, cudaStream_t st)
{
    if (!p->ctx->profiling) return;
    if (p->timer.recs.size() >= 1024)
    { // nobody is reading: recycle the oldest record
        for (auto e : p->timer.recs.front().ev) p->timer.pool.push_back(e);
        p->timer.recs.erase(p->timer.recs.begin());
    }
    p->timer.recs.emplace_back();
    cudaEvent_t e = timer_event(p);
    cudaEventRecord(e, st);
    p->timer.recs.back().ev.push_back(e);
}
static void timer_mark(hr_pass* p, const char* name, cudaStream_t st)
{
    if (!p->ctx->profiling || p->timer.recs.empty()) return;
    cudaEvent_t e = timer_event(p);
    cudaEventRecord(e, st);
    p->timer.recs.back().names.push_back(name);
    p->timer.recs.back().ev.push_back(e);
}

extern "C" {

int hr_version(void) { return HR_VERSION; }

int hr_init(int device, hr_ctx** out)
{
    if (!out) return HR_ERR_INVALID_ARG;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0)
    {
        hr_set_error(nullptr, "hr_init: no CUDA device available (this library has no CPU fallback)");
        return HR_ERR_CUDA;
    }
    if (device < 0 || device >= n) { hr_set_error(nullptr, "hr_init: device %d out of range (%d devices)", device, n); return HR_ERR_INVALID_ARG; }
    hr_ctx* ctx = new hr_ctx();
    ctx->device = device;
    HR_CUDA(ctx, cudaSetDevice(device));
    cudaDeviceProp prop;
    HR_CUDA(ctx, cudaGetDeviceProperties(&prop, device));
    ctx->sm_count = prop.multiProcessorCount;
    HR_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->build_stream, cudaStreamNonBlocking));
    *out = ctx;
    return HR_OK;
}

int hr_shutdown(hr_ctx* ctx)
{
    if (!ctx) return HR_ERR_INVALID_ARG;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (int s = 0; s < 2; s++)
    {
        for (int m = 1; m < HR_MAX_MIPS; m++)
        {
            cudaFree(ctx->slot[s].gb1[m]); cudaFree(ctx->slot[s].gb2[m]); cudaFree(ctx->slot[s].gb3[m]); cudaFree(ctx->slot[s].depth[m]);
        }
        for (int k = 0; k < 4; k++) cudaFree(ctx->owned_mip0[s][k]);
    }
    for (int k = 0; k < 4; k++) cudaFree(ctx->staging_mip0[k]);
    if (ctx->upload_stream) cudaStreamDestroy(ctx->upload_stream);
    if (ctx->ev_staged) cudaEventDestroy(ctx->ev_staged);
    if (ctx->ev_storage_free) cudaEventDestroy(ctx->ev_storage_free);
    cudaFree(ctx->d_sobol);
    cudaFree(ctx->d_scr_rank);
    cudaFree(ctx->d_brdf_lut);
    for (int k = 1; k < 9; k++) cudaFree(ctx->d_scr_rank_slot[k]);
    if (ctx->build_stream) cudaStreamDestroy(ctx->build_stream);
    if (ctx->nccl_comm) hr_shard_shutdown(ctx);
    if (ctx->comm_stream) cudaStreamDestroy(ctx->comm_stream);
    delete ctx;
    return HR_OK;
}

const char* hr_last_error(hr_ctx* ctx)
{
    std::lock_guard<std::mutex> lk(g_err_mutex);
    return ctx ? ctx->last_error.c_str() : g_last_error.c_str();
}

int hr_debug_set(int key, int value)
{
    if (key == 1 && (value == 0 || value == 1 || value == 3)) { g_hr_atrous_impl = value; return HR_OK; }
    if (key == 3 && (value == 0 || value == 1)) { g_hr_bvh_quality = value; return HR_OK; }
    if (key == 6 && (value == 0 || value == 2 || value == 3)) { g_hr_refl_atrous_impl = value; return HR_OK; }
    return HR_ERR_INVALID_ARG;
}

int      hr_ctx_set_profiling(hr_ctx* ctx, int enabled) { if (!ctx) return HR_ERR_INVALID_ARG; ctx->profiling = enabled != 0; return HR_OK; }
uint64_t hr_ctx_launch_count(hr_ctx* ctx) { return ctx ? ctx->launches : 0; }

int hr_bluenoise_set(hr_ctx* ctx, const uint8_t* sobol, const uint8_t* sr)
{
    HR_REQUIRE(ctx, ctx && sobol && sr, HR_ERR_INVALID_ARG, "hr_bluenoise_set: null argument");
    if (!ctx->d_sobol) HR_CUDA(ctx, cudaMalloc(&ctx->d_sobol, 256 * 4));
    if (!ctx->d_scr_rank) HR_CUDA(ctx, cudaMalloc(&ctx->d_scr_rank, 128 * 128 * 4));
    HR_CUDA(ctx, cudaMemcpy(ctx->d_sobol, sobol, 256 * 4, cudaMemcpyHostToDevice));
    HR_CUDA(ctx, cudaMemcpy(ctx->d_scr_rank, sr, 128 * 128 * 4, cudaMemcpyHostToDevice));
    ctx->bn_set = true;
    ctx->d_scr_rank_slot[0] = ctx->d_scr_rank;
    return HR_OK;
}

int hr_bluenoise_set_slot(hr_ctx* ctx, int slot, const uint8_t* sr)
{
    HR_REQUIRE(ctx, ctx && sr && slot >= 0 && slot <= 8, HR_ERR_INVALID_ARG, "hr_bluenoise_set_slot: slot must be 0..8 (1, 2, 4, ..., 256 spp)");
    if (slot == 0)
    {
        if (!ctx->d_scr_rank) HR_CUDA(ctx, cudaMalloc(&ctx->d_scr_rank, 128 * 128 * 4));
        ctx->d_scr_rank_slot[0] = ctx->d_scr_rank;
    }
    else if (!ctx->d_scr_rank_slot[slot]) HR_CUDA(ctx, cudaMalloc(&ctx->d_scr_rank_slot[slot], 128 * 128 * 4));
    HR_CUDA(ctx, cudaMemcpy(ctx->d_scr_rank_slot[slot], sr, 128 * 128 * 4, cudaMemcpyHostToDevice));
    return HR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Scene
// ---------------------------------------------------------------------------------------------------------------
static int scene_check_depth(hr_scene* sc);
static std::atomic<uint64_t> g_scene_serial { 0 }; // hr_scene::serial of the last hr_scene_build, in any context

int hr_scene_build(hr_ctx* ctx, const hr_vertex* vertices, size_t n_vertices, const uint32_t* indices, size_t n_indices, const hr_instance* instances,
                   size_t n_instances, const hr_material* materials, size_t n_materials, hr_scene** out)
{
    HR_REQUIRE(ctx, ctx && vertices && indices && instances && out, HR_ERR_INVALID_ARG, "hr_scene_build: null argument");
    // flatten instances to a world-space triangle soup in primitive order (instances in order, triangles in index order);
    // same arithmetic as transform_vertex (scene_descriptor_set.glsl:147-156): mat4 * vec4 position, normalize(mat3 * normal).
    std::vector<float>    soup;
    std::vector<float>    vnorm;
    std::vector<float>    vuv; // texture coordinates per primitive corner (host copy; on the device only when textures are bound)
    std::vector<float>    vtb; // world-space unit tangents (3 corners) then bitangents (3 corners) per primitive, transform_vertex :155-156
    std::vector<uint32_t> prim_inst, prim_mat;
    for (size_t ii = 0; ii < n_instances; ii++)
    {
        const hr_instance& in = instances[ii];
        const float*       M  = in.model;
        if ((size_t)in.first_index + in.index_count > n_indices) { hr_set_error(ctx, "hr_scene_build: instance %zu index range out of bounds", ii); return HR_ERR_INVALID_ARG; }
        // every shading kernel reads d_materials[prim_mat] (and, with textures, TexDev::mat[prim_mat]) unchecked; a scene without materials
        // (shadows and AO only) is legal and refused by the shading renders instead
        if (n_materials > 0 && in.material_idx >= n_materials)
        {
            hr_set_error(ctx, "hr_scene_build: instance %zu material_idx %u out of range (%zu materials)", ii, in.material_idx, n_materials);
            return HR_ERR_INVALID_ARG;
        }
        for (uint32_t k = 0; k + 2 < in.index_count; k += 3)
        {
            float tb[18];
            for (int j = 0; j < 3; j++)
            {
                const size_t vi = (size_t)in.base_vertex + indices[in.first_index + k + j];
                if (vi >= n_vertices) { hr_set_error(ctx, "hr_scene_build: vertex index out of bounds"); return HR_ERR_INVALID_ARG; }
                const hr_vertex& v = vertices[vi];
                const float      x = v.position[0], y = v.position[1], z = v.position[2];
                soup.push_back(((M[0] * x + M[4] * y) + M[8] * z) + M[12]);
                soup.push_back(((M[1] * x + M[5] * y) + M[9] * z) + M[13]);
                soup.push_back(((M[2] * x + M[6] * y) + M[10] * z) + M[14]);
                const float nx = v.normal[0], ny = v.normal[1], nz = v.normal[2];
                float       wx = (M[0] * nx + M[4] * ny) + M[8] * nz, wy = (M[1] * nx + M[5] * ny) + M[9] * nz, wz = (M[2] * nx + M[6] * ny) + M[10] * nz;
                const float l = sqrtf((wx * wx + wy * wy) + wz * wz);
                const float il = l > 0.0f ? 1.0f / l : 0.0f;
                vnorm.push_back(wx * il); vnorm.push_back(wy * il); vnorm.push_back(wz * il); vnorm.push_back(0.0f);
                vuv.push_back(v.tex_coord[0]); vuv.push_back(v.tex_coord[1]);
                for (int w = 0; w < 2; w++)
                { // normalize(mat3(model) * tangent / bitangent), like the normal above
                    const float* a = w ? v.bitangent : v.tangent;
                    float tx = (M[0] * a[0] + M[4] * a[1]) + M[8] * a[2], ty = (M[1] * a[0] + M[5] * a[1]) + M[9] * a[2], tz = (M[2] * a[0] + M[6] * a[1]) + M[10] * a[2];
                    const float tl = sqrtf((tx * tx + ty * ty) + tz * tz), til = tl > 0.0f ? 1.0f / tl : 0.0f;
                    tb[9 * w + 3 * j] = tx * til; tb[9 * w + 3 * j + 1] = ty * til; tb[9 * w + 3 * j + 2] = tz * til;
                }
            }
            vtb.insert(vtb.end(), tb, tb + 18);
            prim_inst.push_back((uint32_t)ii);
            prim_mat.push_back(in.material_idx);
        }
    }
    const size_t n = prim_inst.size();
    HR_REQUIRE(ctx, n > 0, HR_ERR_INVALID_ARG, "hr_scene_build: scene has no triangles");
    HR_REQUIRE(ctx, n < (1u << 28), HR_ERR_UNSUPPORTED, "hr_scene_build: more than 2^28 triangles");
    HR_CUDA(ctx, cudaSetDevice(ctx->device));
    hr_scene* sc = new hr_scene();
    sc->ctx      = ctx;
    sc->serial   = ++g_scene_serial;
    sc->n_tris   = (uint32_t)n;
    sc->h_vuv    = std::move(vuv);
    sc->h_vtb    = std::move(vtb);
    const size_t ni = n > 1 ? n - 1 : 1;
#define ALLOC(ptr, bytes) HR_CUDA(ctx, cudaMalloc((void**)&(ptr), (bytes)))
    ALLOC(sc->d_tri_verts, n * 9 * sizeof(float));
    ALLOC(sc->d_prim_inst, n * sizeof(uint32_t));
    ALLOC(sc->d_prim_mat, n * sizeof(uint32_t));
    ALLOC(sc->d_vnormals, n * 3 * sizeof(float4));
    ALLOC(sc->d_keys, n * sizeof(uint64_t));
    ALLOC(sc->d_keys_sorted, n * sizeof(uint64_t));
    ALLOC(sc->d_vals, n * sizeof(uint32_t));
    ALLOC(sc->d_vals_sorted, n * sizeof(uint32_t));
    ALLOC(sc->d_tri_aabb, n * 6 * sizeof(float));
    ALLOC(sc->d_bounds_i, 6 * sizeof(int));
    ALLOC(sc->d_children, ni * sizeof(int2));
    ALLOC(sc->d_ranges, ni * sizeof(int2));
    ALLOC(sc->d_parent, (2 * n) * sizeof(int));
    ALLOC(sc->d_node_aabb, ni * 6 * sizeof(float));
    ALLOC(sc->d_flags, ni * sizeof(int));
    ALLOC(sc->d_nodes, ni * 4 * sizeof(float4));
    ALLOC(sc->d_depth, sizeof(int));
    ALLOC(sc->d_tris, n * 3 * sizeof(float4));
    if (n_materials && materials)
    {
        ALLOC(sc->d_materials, n_materials * sizeof(hr_material));
        HR_CUDA(ctx, cudaMemcpy(sc->d_materials, materials, n_materials * sizeof(hr_material), cudaMemcpyHostToDevice));
        sc->n_materials = (uint32_t)n_materials;
    }
#undef ALLOC
    HR_CUDA(ctx, cudaMemcpy(sc->d_tri_verts, soup.data(), n * 9 * sizeof(float), cudaMemcpyHostToDevice));
    HR_CUDA(ctx, cudaMemcpy(sc->d_prim_inst, prim_inst.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice));
    HR_CUDA(ctx, cudaMemcpy(sc->d_prim_mat, prim_mat.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice));
    HR_CUDA(ctx, cudaMemcpy(sc->d_vnormals, vnorm.data(), n * 3 * sizeof(float4), cudaMemcpyHostToDevice));
    int rc = hr_scene_rebuild(sc, ctx->build_stream);
    if (rc != HR_OK) { hr_scene_destroy(sc); return rc; }
    HR_CUDA(ctx, cudaStreamSynchronize(ctx->build_stream));
    rc = scene_check_depth(sc);
    if (rc != HR_OK) { hr_scene_destroy(sc); return rc; }
    // bounds for info
    int bi[6];
    HR_CUDA(ctx, cudaMemcpy(bi, sc->d_bounds_i, sizeof(bi), cudaMemcpyDeviceToHost));
    for (int a = 0; a < 6; a++)
    {
        int   i = bi[a] >= 0 ? bi[a] : bi[a] ^ 0x7FFFFFFF;
        float f;
        memcpy(&f, &i, 4);
        (a < 3 ? sc->info.bounds_min[a] : sc->info.bounds_max[a - 3]) = f;
    }
    *out = sc;
    if (!ctx->scene) ctx->scene = sc;
    return HR_OK;
}

// The binary walks push at most one pending sibling per level, so their stacks (STACK_SIZE = HR_BVH_MAX_DEPTH + 1 entries, one of
// them the sentinel) cannot overflow on a tree of height <= HR_BVH_MAX_DEPTH.  A deeper tree is refused here instead of being
// traversed with dropped pushes.  Blocking read of one int: called where the host waits anyway.
static int scene_check_depth(hr_scene* sc)
{
    hr_ctx* ctx = sc->ctx;
    int     d   = 0;
    HR_CUDA(ctx, cudaMemcpy(&d, sc->d_depth, sizeof(int), cudaMemcpyDeviceToHost));
    sc->info.depth = (uint32_t)d;
    HR_REQUIRE(ctx, d <= HR_BVH_MAX_DEPTH, HR_ERR_UNSUPPORTED, "scene: the BVH is deeper than the traversal stack (HR_BVH_MAX_DEPTH)");
    return HR_OK;
}

int hr_scene_rebuild(hr_scene* sc, void* stream)
{
    if (!sc) return HR_ERR_INVALID_ARG;
    hr_ctx*      ctx = sc->ctx;
    cudaStream_t st  = (cudaStream_t)stream;
    cudaEvent_t  e0 = nullptr, e1 = nullptr;
    if (ctx->profiling) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, st); }
    int rc = hr_bvh_build(sc, st);
    if (rc != HR_OK) return rc;
    if (ctx->profiling)
    {
        cudaEventRecord(e1, st);
        cudaEventSynchronize(e1);
        cudaEventElapsedTime(&sc->info.build_ms, e0, e1);
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        rc = scene_check_depth(sc); // the host has just waited for the build anyway
        if (rc != HR_OK) return rc;
    }
    sc->info.n_triangles = sc->n_tris;
    sc->info.n_nodes     = sc->n_nodes;
    return HR_OK;
}

int hr_scene_destroy(hr_scene* sc)
{
    if (!sc) return HR_ERR_INVALID_ARG;
    if (sc->ctx && sc->ctx->scene == sc) sc->ctx->scene = nullptr;
    void* ptrs[] = { sc->d_tri_verts, sc->d_prim_inst, sc->d_prim_mat, sc->d_vnormals, sc->d_keys, sc->d_keys_sorted, sc->d_vals, sc->d_vals_sorted,
                     sc->d_tri_aabb, sc->d_bounds_i, sc->d_children, sc->d_ranges, sc->d_parent, sc->d_node_aabb, sc->d_flags, sc->d_nodes, sc->d_depth, sc->d_tris,
                     sc->d_materials, sc->d_sort_tmp, sc->d_ploc, sc->d_vuv, sc->d_vtb, sc->d_texels, sc->d_tex_desc, sc->d_mat_tex, sc->d_srgb_lut };
    for (void* p : ptrs) cudaFree(p);
    delete sc;
    return HR_OK;
}

// Material textures: Material::load uploads one VkImage per texture and RayTracedScene binds them as s_Textures[] (ray_traced_scene.cpp:345-420);
// here every texture is expanded to RGBA8 and concatenated into one buffer (tex_px.cuh).
int hr_scene_set_textures(hr_scene* sc, const hr_texture* textures, size_t n_textures, const hr_material_textures* bindings, size_t n_materials)
{
    if (!sc) return HR_ERR_INVALID_ARG;
    hr_ctx* ctx = sc->ctx;
    HR_CUDA(ctx, cudaSetDevice(ctx->device));
    auto drop = [&]() {
        void* ptrs[] = { sc->d_texels, sc->d_tex_desc, sc->d_mat_tex };
        for (void* p : ptrs) cudaFree(p);
        sc->d_texels = nullptr; sc->d_tex_desc = nullptr; sc->d_mat_tex = nullptr;
        sc->tex = tex::TexDev {};
    };
    if (n_textures == 0) { cudaDeviceSynchronize(); drop(); return HR_OK; }
    HR_REQUIRE(ctx, textures && bindings, HR_ERR_INVALID_ARG, "hr_scene_set_textures: null argument");
    HR_REQUIRE(ctx, n_materials == sc->n_materials && n_materials > 0, HR_ERR_INVALID_ARG, "hr_scene_set_textures: one binding per material of the scene is required");
    HR_REQUIRE(ctx, n_textures < (1u << 20), HR_ERR_UNSUPPORTED, "hr_scene_set_textures: too many textures");
    std::vector<tex::TexDesc> desc(n_textures);
    size_t total = 0;
    for (size_t i = 0; i < n_textures; i++)
    {
        const hr_texture& t = textures[i];
        HR_REQUIRE(ctx, t.data && t.width > 0 && t.height > 0 && t.width <= 16384 && t.height <= 16384 && (t.channels == 1 || t.channels == 2 || t.channels == 4),
                   HR_ERR_INVALID_ARG, "hr_scene_set_textures: a texture has no data, a bad size (1..16384) or a channel count other than 1, 2, 4");
        desc[i].offset = (uint32_t)total; desc[i].width = t.width; desc[i].height = t.height; desc[i].srgb = t.srgb ? 1 : 0;
        total += (size_t)t.width * t.height;
        HR_REQUIRE(ctx, total < (1ull << 32), HR_ERR_UNSUPPORTED, "hr_scene_set_textures: more than 2^32 texels in total");
    }
    std::vector<tex::MatTex> mt(n_materials);
    for (size_t m = 0; m < n_materials; m++)
    {
        const hr_material_textures& b = bindings[m];
        const int32_t idx[5] = { b.albedo, b.normal, b.roughness, b.metallic, b.emissive };
        for (int32_t i : idx) HR_REQUIRE(ctx, i >= -1 && i < (int32_t)n_textures, HR_ERR_INVALID_ARG, "hr_scene_set_textures: texture index out of range");
        HR_REQUIRE(ctx, (b.roughness < 0 || (b.roughness_channel >= 0 && b.roughness_channel <= 3)) && (b.metallic < 0 || (b.metallic_channel >= 0 && b.metallic_channel <= 3)),
                   HR_ERR_INVALID_ARG, "hr_scene_set_textures: roughness / metallic channel must be 0..3");
        mt[m] = tex::MatTex { b.albedo, b.normal, b.roughness, b.roughness_channel, b.metallic, b.metallic_channel, b.emissive, 0 };
    }
    std::vector<uint32_t> texels(total);
    for (size_t i = 0; i < n_textures; i++)
    { // missing components read (0, 0, 1) like a sampler on an R8 / RG8 image
        const hr_texture& t = textures[i];
        uint32_t* dst = texels.data() + desc[i].offset;
        const size_t px = (size_t)t.width * t.height;
        for (size_t k = 0; k < px; k++)
        {
            const uint8_t* q = t.data + k * t.channels;
            dst[k] = t.channels == 4 ? ((uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24))
                   : t.channels == 2 ? ((uint32_t)q[0] | ((uint32_t)q[1] << 8) | 0xFF000000u) : ((uint32_t)q[0] | 0xFF000000u);
        }
    }
    float lut[256];
    for (int i = 0; i < 256; i++)
    { // sRGB EOTF in double, rounded once (the oracle builds the same table)
        const double c = i / 255.0;
        lut[i] = (float)(c <= 0.04045 ? c / 12.92 : pow((c + 0.055) / 1.055, 2.4));
    }
    HR_REQUIRE(ctx, sc->h_vuv.size() == 6ull * sc->n_tris, HR_ERR_NOT_READY, "hr_scene_set_textures: the scene holds no texture coordinates");
    cudaDeviceSynchronize();
    drop();
    if (!sc->d_vuv)
    {
        HR_CUDA(ctx, cudaMalloc((void**)&sc->d_vuv, sc->h_vuv.size() * sizeof(float)));
        HR_CUDA(ctx, cudaMemcpy(sc->d_vuv, sc->h_vuv.data(), sc->h_vuv.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    if (!sc->d_srgb_lut)
    {
        HR_CUDA(ctx, cudaMalloc((void**)&sc->d_srgb_lut, sizeof(lut)));
        HR_CUDA(ctx, cudaMemcpy(sc->d_srgb_lut, lut, sizeof(lut), cudaMemcpyHostToDevice));
    }
    HR_CUDA(ctx, cudaMalloc((void**)&sc->d_texels, total * sizeof(uint32_t)));
    HR_CUDA(ctx, cudaMalloc((void**)&sc->d_tex_desc, n_textures * sizeof(tex::TexDesc)));
    HR_CUDA(ctx, cudaMalloc((void**)&sc->d_mat_tex, n_materials * sizeof(tex::MatTex)));
    HR_CUDA(ctx, cudaMemcpy(sc->d_texels, texels.data(), total * sizeof(uint32_t), cudaMemcpyHostToDevice));
    HR_CUDA(ctx, cudaMemcpy(sc->d_tex_desc, desc.data(), n_textures * sizeof(tex::TexDesc), cudaMemcpyHostToDevice));
    HR_CUDA(ctx, cudaMemcpy(sc->d_mat_tex, mt.data(), n_materials * sizeof(tex::MatTex), cudaMemcpyHostToDevice));
    bool any_normal_map = false;
    for (const auto& m : mt) any_normal_map = any_normal_map || m.normal >= 0;
    if (any_normal_map && !sc->d_vtb)
    {
        HR_REQUIRE(ctx, sc->h_vtb.size() == 18ull * sc->n_tris, HR_ERR_NOT_READY, "hr_scene_set_textures: the scene holds no tangent frames");
        HR_CUDA(ctx, cudaMalloc((void**)&sc->d_vtb, sc->h_vtb.size() * sizeof(float)));
        HR_CUDA(ctx, cudaMemcpy(sc->d_vtb, sc->h_vtb.data(), sc->h_vtb.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    sc->tex = tex::TexDev { sc->d_texels, sc->d_tex_desc, sc->d_mat_tex, sc->d_vuv, sc->d_srgb_lut, (int32_t)n_textures, any_normal_map ? sc->d_vtb : nullptr };
    return HR_OK;
}

int hr_scene_set_current(hr_ctx* ctx, hr_scene* scene) { if (!ctx) return HR_ERR_INVALID_ARG; ctx->scene = scene; return HR_OK; }
int hr_scene_get_info(hr_scene* sc, hr_scene_info* out) { if (!sc || !out) return HR_ERR_INVALID_ARG; *out = sc->info; return HR_OK; }

int hr_scene_download_bvh(hr_scene* sc, void* nodes, size_t nodes_bytes, void* tris, size_t tris_bytes)
{
    if (!sc) return HR_ERR_INVALID_ARG;
    hr_ctx* ctx = sc->ctx;
    HR_REQUIRE(ctx, !nodes || nodes_bytes == sc->n_nodes * 4 * sizeof(float4), HR_ERR_INVALID_ARG, "hr_scene_download_bvh: nodes_bytes must be n_nodes * 64");
    HR_REQUIRE(ctx, !tris || tris_bytes == sc->n_tris * 3 * sizeof(float4), HR_ERR_INVALID_ARG, "hr_scene_download_bvh: tris_bytes must be n_triangles * 48");
    HR_CUDA(ctx, cudaSetDevice(ctx->device));
    HR_CUDA(ctx, cudaDeviceSynchronize());
    if (nodes) HR_CUDA(ctx, cudaMemcpy(nodes, sc->d_nodes, nodes_bytes, cudaMemcpyDeviceToHost));
    if (tris) HR_CUDA(ctx, cudaMemcpy(tris, sc->d_tris, tris_bytes, cudaMemcpyDeviceToHost));
    return HR_OK;
}

int hr_trace_any(hr_ctx* ctx, const float* d_rays, size_t n, uint32_t* d_out, void* stream)
{
    HR_REQUIRE(ctx, ctx && ctx->scene, HR_ERR_NOT_READY, "hr_trace_any: no current scene");
    launch_trace_any(hr_bvh_view(ctx->scene), d_rays, n, d_out, (cudaStream_t)stream);
    ctx->launches++;
    HR_CHECK_LAUNCH(ctx);
    return HR_OK;
}
int hr_trace_closest(hr_ctx* ctx, const float* d_rays, size_t n, float* d_t, uint32_t* d_prim, float* d_uv, void* stream)
{
    HR_REQUIRE(ctx, ctx && ctx->scene, HR_ERR_NOT_READY, "hr_trace_closest: no current scene");
    launch_trace_closest(hr_bvh_view(ctx->scene), d_rays, n, d_t, d_prim, d_uv, (cudaStream_t)stream);
    ctx->launches++;
    HR_CHECK_LAUNCH(ctx);
    return HR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// G-buffer
// ---------------------------------------------------------------------------------------------------------------
int hr_gbuffer_create(hr_ctx* ctx, int width, int height)
{
    HR_REQUIRE(ctx, ctx && width > 0 && height > 0, HR_ERR_INVALID_ARG, "hr_gbuffer_create: bad size");
    HR_REQUIRE(ctx, ctx->gb_w == 0, HR_ERR_INVALID_ARG, "hr_gbuffer_create: already created");
    HR_CUDA(ctx, cudaSetDevice(ctx->device));
    ctx->gb_w = width;
    ctx->gb_h = height;
    for (int s = 0; s < 2; s++)
    {
        for (int m = 0; m < HR_MAX_MIPS; m++)
        {
            const size_t px = (size_t)mip_extent(width, m) * mip_extent(height, m);
            HR_CUDA(ctx, cudaMalloc(&ctx->slot[s].gb1[m], px * 4));
            HR_CUDA(ctx, cudaMalloc(&ctx->slot[s].gb2[m], px * 8));
            HR_CUDA(ctx, cudaMalloc(&ctx->slot[s].gb3[m], px * 8));
            HR_CUDA(ctx, cudaMalloc((void**)&ctx->slot[s].depth[m], px * 4));
            HR_CUDA(ctx, cudaMemset(ctx->slot[s].gb1[m], 0, px * 4));
            HR_CUDA(ctx, cudaMemset(ctx->slot[s].gb2[m], 0, px * 8));
            HR_CUDA(ctx, cudaMemset(ctx->slot[s].gb3[m], 0, px * 8));
            HR_CUDA(ctx, cudaMemset(ctx->slot[s].depth[m], 0, px * 4));
        }
        ctx->owned_mip0[s][0] = ctx->slot[s].gb1[0];
        ctx->owned_mip0[s][1] = ctx->slot[s].gb2[0];
        ctx->owned_mip0[s][2] = ctx->slot[s].gb3[0];
        ctx->owned_mip0[s][3] = ctx->slot[s].depth[0];
        ctx->slot[s].valid    = true; // zero-initialised history is a valid (empty) frame
    }
    return HR_OK;
}

// Point slot `slot` at its library-owned mip-0 storage (the slot may have been bound zero-copy before).
static GBufSlot& use_owned_mip0(hr_ctx* ctx, int slot)
{
    GBufSlot& s = ctx->slot[slot];
    s.gb1[0]   = ctx->owned_mip0[slot][0];
    s.gb2[0]   = ctx->owned_mip0[slot][1];
    s.gb3[0]   = ctx->owned_mip0[slot][2];
    s.depth[0] = (float*)ctx->owned_mip0[slot][3];
    return s;
}

static int gbuffer_copy_in(hr_ctx* ctx, int slot, const hr_gbuffer_desc* src, cudaMemcpyKind kind, cudaStream_t st)
{
    HR_REQUIRE(ctx, ctx && src && (slot == 0 || slot == 1), HR_ERR_INVALID_ARG, "hr_gbuffer_upload: bad argument");
    HR_REQUIRE(ctx, ctx->gb_w > 0, HR_ERR_NOT_READY, "hr_gbuffer_upload: call hr_gbuffer_create first");
    HR_REQUIRE(ctx, src->width == ctx->gb_w && src->height == ctx->gb_h, HR_ERR_INVALID_ARG, "hr_gbuffer_upload: size mismatch");
    HR_REQUIRE(ctx, src->gb2 && src->gb3 && src->depth, HR_ERR_INVALID_ARG, "hr_gbuffer_upload: gb2/gb3/depth are required");
    GBufSlot&    s  = use_owned_mip0(ctx, slot);
    const size_t px = (size_t)ctx->gb_w * ctx->gb_h;
    if (src->gb1) HR_CUDA(ctx, cudaMemcpyAsync(s.gb1[0], src->gb1, px * 4, kind, st));
    HR_CUDA(ctx, cudaMemcpyAsync(s.gb2[0], src->gb2, px * 8, kind, st));
    HR_CUDA(ctx, cudaMemcpyAsync(s.gb3[0], src->gb3, px * 8, kind, st));
    HR_CUDA(ctx, cudaMemcpyAsync(s.depth[0], src->depth, px * 4, kind, st));
    return hr_launch_build_mips(ctx, s, ctx->gb_w, ctx->gb_h, st);
}

int hr_gbuffer_upload(hr_ctx* ctx, int slot, const hr_gbuffer_desc* host, void* stream) { return gbuffer_copy_in(ctx, slot, host, cudaMemcpyHostToDevice, (cudaStream_t)stream); }
int hr_gbuffer_copy_from_device(hr_ctx* ctx, int slot, const hr_gbuffer_desc* dev, void* stream) { return gbuffer_copy_in(ctx, slot, dev, cudaMemcpyDeviceToDevice, (cudaStream_t)stream); }

// Streaming host frames.  PCIe moves ~24 B/pixel per frame (199 MB at 4K, ~3.6 ms on a Gen5 x16 link) — longer than the
// frame's kernels — so the upload of frame N+1 has to overlap the render of frame N.  The G-buffer is double buffered by
// design (current / previous, src/g_buffer.cpp:236-244), and slot (N+1)%2 is still being read as "previous" while frame N
// renders, so the copy goes to a third surface on the library's upload stream; commit swaps that surface with the slot's
// storage.  The storage handed back by the swap was last read by renders already enqueued on `stream`: an event recorded
// there gates the next staged upload.
// The staging surface, the upload stream and its events are created on the first staged frame; the upload stream then waits
// until the storage that the last commit handed back is no longer read.
static int staging_begin(hr_ctx* ctx)
{
    HR_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->upload_stream)
    {
        const size_t px = (size_t)ctx->gb_w * ctx->gb_h;
        HR_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->upload_stream, cudaStreamNonBlocking));
        HR_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_staged, cudaEventDisableTiming));
        HR_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_storage_free, cudaEventDisableTiming));
        const size_t bytes[4] = { px * 4, px * 8, px * 8, px * 4 };
        for (int k = 0; k < 4; k++)
        {
            HR_CUDA(ctx, cudaMalloc(&ctx->staging_mip0[k], bytes[k]));
            HR_CUDA(ctx, cudaMemset(ctx->staging_mip0[k], 0, bytes[k]));
        }
    }
    if (ctx->storage_free_recorded) HR_CUDA(ctx, cudaStreamWaitEvent(ctx->upload_stream, ctx->ev_storage_free, 0));
    return HR_OK;
}

int hr_gbuffer_stage_upload(hr_ctx* ctx, const hr_gbuffer_desc* host)
{
    HR_REQUIRE(ctx, ctx && host, HR_ERR_INVALID_ARG, "hr_gbuffer_stage_upload: bad argument");
    HR_REQUIRE(ctx, ctx->gb_w > 0, HR_ERR_NOT_READY, "hr_gbuffer_stage_upload: call hr_gbuffer_create first");
    HR_REQUIRE(ctx, host->width == ctx->gb_w && host->height == ctx->gb_h, HR_ERR_INVALID_ARG, "hr_gbuffer_stage_upload: size mismatch");
    HR_REQUIRE(ctx, host->gb2 && host->gb3 && host->depth, HR_ERR_INVALID_ARG, "hr_gbuffer_stage_upload: gb2/gb3/depth are required");
    HR_REQUIRE(ctx, !ctx->staged_pending, HR_ERR_INVALID_ARG, "hr_gbuffer_stage_upload: a staged frame is already waiting for hr_gbuffer_commit_staged");
    int rc = staging_begin(ctx);
    if (rc != HR_OK) return rc;
    const size_t px = (size_t)ctx->gb_w * ctx->gb_h;
    if (host->gb1) HR_CUDA(ctx, cudaMemcpyAsync(ctx->staging_mip0[0], host->gb1, px * 4, cudaMemcpyHostToDevice, ctx->upload_stream));
    HR_CUDA(ctx, cudaMemcpyAsync(ctx->staging_mip0[1], host->gb2, px * 8, cudaMemcpyHostToDevice, ctx->upload_stream));
    HR_CUDA(ctx, cudaMemcpyAsync(ctx->staging_mip0[2], host->gb3, px * 8, cudaMemcpyHostToDevice, ctx->upload_stream));
    HR_CUDA(ctx, cudaMemcpyAsync(ctx->staging_mip0[3], host->depth, px * 4, cudaMemcpyHostToDevice, ctx->upload_stream));
    HR_CUDA(ctx, cudaEventRecord(ctx->ev_staged, ctx->upload_stream));
    ctx->staged_pending = true;
    return HR_OK;
}

// Pipelined device G-buffer: render the NEXT frame's G-buffer into the staging surface on the library's side stream while the
// caller's stream still runs this frame's passes (which read both G-buffer slots); hr_gbuffer_commit_staged swaps it in.
int hr_gbuffer_stage_render(hr_ctx* ctx, const hr_frame* frame)
{
    HR_REQUIRE(ctx, ctx && frame, HR_ERR_INVALID_ARG, "hr_gbuffer_stage_render: bad argument");
    HR_REQUIRE(ctx, ctx->gb_w > 0, HR_ERR_NOT_READY, "hr_gbuffer_stage_render: call hr_gbuffer_create first");
    HR_REQUIRE(ctx, ctx->scene && ctx->scene->d_materials, HR_ERR_NOT_READY, "hr_gbuffer_stage_render: no current scene with materials (hr_scene_build)");
    HR_REQUIRE(ctx, !ctx->staged_pending, HR_ERR_INVALID_ARG, "hr_gbuffer_stage_render: a staged frame is already waiting for hr_gbuffer_commit_staged");
    int rc = staging_begin(ctx);
    if (rc != HR_OK) return rc;
    launch_gbuffer_render(ctx->scene, frame, ctx->gb_w, ctx->gb_h, 0, ctx->gb_h, 0, 1, ctx->staging_mip0[0], ctx->staging_mip0[1], ctx->staging_mip0[2],
                          (float*)ctx->staging_mip0[3], ctx->gbuf_ray_ctr, ctx->upload_stream);
    ctx->launches++;
    HR_CHECK_LAUNCH(ctx);
    HR_CUDA(ctx, cudaEventRecord(ctx->ev_staged, ctx->upload_stream));
    ctx->staged_pending = true;
    return HR_OK;
}

int hr_gbuffer_commit_staged(hr_ctx* ctx, int slot, void* stream)
{
    HR_REQUIRE(ctx, ctx && (slot == 0 || slot == 1), HR_ERR_INVALID_ARG, "hr_gbuffer_commit_staged: bad argument");
    HR_REQUIRE(ctx, ctx->staged_pending, HR_ERR_NOT_READY, "hr_gbuffer_commit_staged: no staged frame (call hr_gbuffer_stage_upload first)");
    cudaStream_t st = (cudaStream_t)stream;
    // everything enqueued on `stream` so far may still read the storage we are about to recycle as the staging surface
    HR_CUDA(ctx, cudaEventRecord(ctx->ev_storage_free, st));
    ctx->storage_free_recorded = true;
    HR_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_staged, 0));
    for (int k = 0; k < 4; k++) std::swap(ctx->owned_mip0[slot][k], ctx->staging_mip0[k]);
    GBufSlot& s = use_owned_mip0(ctx, slot);
    ctx->staged_pending = false;
    return hr_launch_build_mips(ctx, s, ctx->gb_w, ctx->gb_h, st);
}

int hr_gbuffer_bind_device(hr_ctx* ctx, int slot, const hr_gbuffer_desc* dev, void* stream)
{
    HR_REQUIRE(ctx, ctx && dev && (slot == 0 || slot == 1), HR_ERR_INVALID_ARG, "hr_gbuffer_bind_device: bad argument");
    HR_REQUIRE(ctx, ctx->gb_w > 0, HR_ERR_NOT_READY, "hr_gbuffer_bind_device: call hr_gbuffer_create first");
    HR_REQUIRE(ctx, dev->width == ctx->gb_w && dev->height == ctx->gb_h, HR_ERR_INVALID_ARG, "hr_gbuffer_bind_device: size mismatch");
    HR_REQUIRE(ctx, dev->gb2 && dev->gb3 && dev->depth, HR_ERR_INVALID_ARG, "hr_gbuffer_bind_device: gb2/gb3/depth are required");
    GBufSlot& s = ctx->slot[slot];
    s.gb1[0]    = const_cast<void*>(dev->gb1);
    s.gb2[0]    = const_cast<void*>(dev->gb2);
    s.gb3[0]    = const_cast<void*>(dev->gb3);
    s.depth[0]  = (float*)const_cast<void*>(dev->depth);
    return hr_launch_build_mips(ctx, s, ctx->gb_w, ctx->gb_h, (cudaStream_t)stream);
}

int hr_gbuffer_render(hr_ctx* ctx, int slot, const hr_frame* frame, int row0, int row1, void* stream)
{
    HR_REQUIRE(ctx, ctx && frame && (slot == 0 || slot == 1), HR_ERR_INVALID_ARG, "hr_gbuffer_render: bad argument");
    HR_REQUIRE(ctx, ctx->gb_w > 0, HR_ERR_NOT_READY, "hr_gbuffer_render: call hr_gbuffer_create first");
    HR_REQUIRE(ctx, ctx->scene && ctx->scene->d_materials, HR_ERR_NOT_READY, "hr_gbuffer_render: no current scene with materials (hr_scene_build)");
    if (row1 <= 0) { row0 = 0; row1 = ctx->gb_h; }
    HR_REQUIRE(ctx, row0 >= 0 && row1 > row0 && row1 <= ctx->gb_h && row0 % 8 == 0 && (row1 % 8 == 0 || row1 == ctx->gb_h), HR_ERR_INVALID_ARG,
               "hr_gbuffer_render: rows must be multiples of 8 (or end at the image height)");
    GBufSlot& s = use_owned_mip0(ctx, slot);
    launch_gbuffer_render(ctx->scene, frame, ctx->gb_w, ctx->gb_h, row0, row1, 0, 1, s.gb1[0], s.gb2[0], s.gb3[0], s.depth[0], ctx->gbuf_ray_ctr, (cudaStream_t)stream);
    ctx->launches++;
    HR_CHECK_LAUNCH(ctx);
    return hr_launch_build_mips(ctx, s, ctx->gb_w, ctx->gb_h, (cudaStream_t)stream);
}

// The rows a sharded rank's FULL-RESOLUTION passes consume: its band +- halo_rows (denoise stages) and the 8-row chunks it traces
// in the interleaved cooperative ray trace (shard.cu).  Single GPU: the whole image.
int hr_gbuffer_render_sharded(hr_ctx* ctx, int slot, const hr_frame* frame, int halo_rows, void* stream)
{
    HR_REQUIRE(ctx, ctx && frame && (slot == 0 || slot == 1) && halo_rows >= 0, HR_ERR_INVALID_ARG, "hr_gbuffer_render_sharded: bad argument");
    if (ctx->world <= 1) return hr_gbuffer_render(ctx, slot, frame, 0, 0, stream);
    HR_REQUIRE(ctx, ctx->gb_w > 0, HR_ERR_NOT_READY, "hr_gbuffer_render_sharded: call hr_gbuffer_create first");
    HR_REQUIRE(ctx, ctx->scene && ctx->scene->d_materials, HR_ERR_NOT_READY, "hr_gbuffer_render_sharded: no current scene with materials (hr_scene_build)");
    GBufSlot& s = use_owned_mip0(ctx, slot);
    int b0, b1, r0, r1;
    hr_band(ctx, ctx->gb_h, &b0, &b1);
    hr_extend(b0, b1, round_up8(halo_rows), ctx->gb_h, &r0, &r1);
    launch_gbuffer_render(ctx->scene, frame, ctx->gb_w, ctx->gb_h, r0, r1, 0, 1, s.gb1[0], s.gb2[0], s.gb3[0], s.depth[0], ctx->gbuf_ray_ctr, (cudaStream_t)stream);
    launch_gbuffer_render(ctx->scene, frame, ctx->gb_w, ctx->gb_h, 0, 0, ctx->rank, ctx->world, s.gb1[0], s.gb2[0], s.gb3[0], s.depth[0], ctx->gbuf_ray_ctr, (cudaStream_t)stream);
    ctx->launches += 2;
    HR_CHECK_LAUNCH(ctx);
    return hr_launch_build_mips(ctx, s, ctx->gb_w, ctx->gb_h, (cudaStream_t)stream);
}

int hr_gbuffer_download(hr_ctx* ctx, int slot, int mip, int which, void* dst, size_t bytes)
{
    HR_REQUIRE(ctx, ctx && dst && (slot == 0 || slot == 1) && mip >= 0 && mip < HR_MAX_MIPS && which >= 0 && which <= 3, HR_ERR_INVALID_ARG,
               "hr_gbuffer_download: bad argument");
    GBufLevelDev l  = level_view(ctx, slot, mip);
    const size_t px = (size_t)l.W * l.H;
    const void*  src = which == 0 ? (const void*)l.depth : which == 1 ? (const void*)l.gb1 : which == 2 ? (const void*)l.gb2 : (const void*)l.gb3;
    const size_t need = px * (which == 0 || which == 1 ? 4 : 8);
    HR_REQUIRE(ctx, bytes == need, HR_ERR_INVALID_ARG, "hr_gbuffer_download: byte count mismatch");
    HR_CUDA(ctx, cudaDeviceSynchronize());
    HR_CUDA(ctx, cudaMemcpy(dst, src, need, cudaMemcpyDeviceToHost));
    return HR_OK;
}

} // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Pass helpers
// ---------------------------------------------------------------------------------------------------------------
static int texel_size(int fmt)
{
    switch (fmt)
    {
        case HR_FMT_R32_UINT: return 4;
        case HR_FMT_R16F: return 2;
        case HR_FMT_RG16F: return 4;
        case HR_FMT_RGBA16F: return 8;
        case HR_FMT_R8_UINT: return 1;
        case HR_FMT_RGBA8: return 4;
    }
    return 0;
}

template <typename T>
static int pass_alloc(hr_pass* p, T*& ptr, size_t count, int fill_byte = 0)
{
    HR_CUDA(p->ctx, cudaMalloc((void**)&ptr, count * sizeof(T)));
    HR_CUDA(p->ctx, cudaMemset(ptr, fill_byte, count * sizeof(T)));
    p->allocs.push_back(ptr);
    return HR_OK;
}

// The images of a pass being created: after the first failed allocation the later ones are skipped and `rc` keeps the error.
struct PassAllocs {
    hr_pass* p;
    int      rc = HR_OK;
    template <typename T>
    void operator()(T*& ptr, size_t count, int fill_byte = 0) { if (rc == HR_OK) rc = pass_alloc(p, ptr, count, fill_byte); }
};

// multi-GPU ray-trace sharing (shard.cu): second ray-mask image (frame parity), cost tables, device-side row partition.  The two
// spp > 1 count images of the cooperative trace are allocated when the pass is linked (rt_alloc_counts, shard.cu).
static void pass_alloc_rt_share(PassAllocs& A)
{
    hr_pass*     p  = A.p;
    const size_t mw = (p->W + 7) / 8, mh = (p->H + 3) / 4;
    p->mask_pp[0] = p->mask;
    A(p->mask_pp[1], mw * mh);
    A(p->rt_cost_all, 2 * mh);
    A(p->rt_cost_acc, mh);
    A(p->rt_bounds, (size_t)HR_CTL_WORDS);
}

static void set_view(hr_pass* p, int which, void* ptr, int w, int h, int fmt) { p->out_view[which] = { ptr, w, h, fmt }; }

// A pass of `kind` at (width, height) / 2^scale; `alloc` allocates its images through the PassAllocs it is given.  If an
// allocation fails the pass is destroyed and *out is null.
template <typename Alloc>
static int pass_create(hr_ctx* ctx, int width, int height, int scale, int kind, hr_pass** out, Alloc alloc)
{
    HR_REQUIRE(ctx, ctx && out && width > 0 && height > 0 && scale >= 0 && scale < HR_MAX_MIPS, HR_ERR_INVALID_ARG, "pass create: bad argument");
    HR_CUDA(ctx, cudaSetDevice(ctx->device));
    hr_pass* p = new hr_pass();
    p->ctx     = ctx;
    p->kind    = kind;
    p->W0      = width;
    p->H0      = height;
    p->scale   = scale;
    p->W       = mip_extent(width, scale); // = swapchain / 2^scale, ray_traced_shadows.cpp:78-83
    p->H       = mip_extent(height, scale);
    const size_t ctr_bytes = sizeof(unsigned long long) * 2 * HR_RAY_CTR_SLOTS * HR_RAY_CTR_STRIDE;
    if (cudaMalloc((void**)&p->ray_ctr, ctr_bytes) != cudaSuccess) { delete p; hr_set_error(ctx, "pass create: out of memory"); return HR_ERR_OUT_OF_MEMORY; }
    cudaMemset(p->ray_ctr, 0, ctr_bytes);
    p->allocs.push_back(p->ray_ctr);
    PassAllocs A { p };
    alloc(A);
    if (A.rc != HR_OK) { hr_pass_destroy(p); *out = nullptr; return A.rc; }
    *out = p;
    return HR_OK;
}

// Recompute halos of a sharded rank, derived from the parameters (rows beyond the owned band, multiples of 8 so tile and mask
// alignment are kept).  An a-trous iteration at step 2^i with the given radius reads rows y +- radius * 2^i, so n iterations
// erode sum(radius << i) rows (+1: the upsample stage reads one coarse row beyond the band); the temporal stage's 17x17
// statistics read the ray-trace output 8 rows beyond its own rows.
static int atrous_halo_rows(int radius, int iterations)
{
    long h = 0;
    for (int i = 0; i < iterations; i++) h += (long)radius << i;
    return round_up8((int)(h > (1 << 20) ? (1 << 20) : h) + 1);
}

// The whole plan: rows beyond its band that a sharded rank's temporal / a-trous / horizontal-blur stages compute (`denoise`), that its
// band-local ray trace covers for them (`ray_trace`), and that the AO vertical blur computes (`vblur`: band + 8, the upsample reads one
// coarse row beyond the band; it reads +- blur_radius rows of the horizontal blur, which is pointwise in y over the temporal output).
struct HaloPlan { int denoise, ray_trace, vblur; };
static_assert(PASS_SHADOWS == HR_PASS_KIND_SHADOWS && PASS_AO == HR_PASS_KIND_AO && PASS_REFLECTIONS == HR_PASS_KIND_REFLECTIONS, "pass kinds");
static HaloPlan halo_plan(int kind, int radius, int filter_iterations, int blur_radius)
{
    HaloPlan h;
    h.vblur     = kind == PASS_AO ? 8 : 0;
    h.denoise   = kind == PASS_AO ? h.vblur + round_up8(blur_radius) : atrous_halo_rows(radius, filter_iterations);
    h.ray_trace = h.denoise + 8; // 17x17 statistics of the temporal stage
    return h;
}

// The plan above as a pure query (no context, no GPU): which rows beyond its band a sharded rank computes.  Tests restate the plan on
// the CPU oracle with these numbers (tests/test_sharding_cpu.py); the render functions take their halos from halo_plan too.
int hr_shard_halo_rows(int pass_kind, int radius, int filter_iterations, int blur_radius, int* denoise_halo, int* ray_trace_halo)
{
    if (!denoise_halo || !ray_trace_halo || radius < 0 || filter_iterations < 0 || blur_radius < 0) return HR_ERR_INVALID_ARG;
    if (pass_kind != HR_PASS_KIND_SHADOWS && pass_kind != HR_PASS_KIND_AO && pass_kind != HR_PASS_KIND_REFLECTIONS) return HR_ERR_INVALID_ARG;
    const HaloPlan h = halo_plan(pass_kind, radius, filter_iterations, blur_radius);
    *denoise_halo    = h.denoise;
    *ray_trace_halo  = h.ray_trace;
    return HR_OK;
}

// ---- the frame protocol of the shadows, AO and reflections renders ------------------------------------------------
// One render: the rows its stages compute, its frame tick and its final output.  frame_begin / frame_end are the parts the three
// renders share; the clears, the history waits and the gathers between them are per pass.
struct PassFrame {
    cudaStream_t st;
    int          pp, epoch;
    bool         no_history;        // first frame after creation / hr_pass_reset_history: the reprojection reads no history
    bool         signalled = false; // this frame's history tick is published (frame_signal)
    int          b0, b1;            // owned band (hr_band)
    int          rt0, rt1, rt_halo; // band-local ray trace: band +- rt_halo
    int          row0, row1;        // temporal / a-trous / horizontal blur
    int          v0, v1;            // AO vertical blur
    int          up0, up1;          // full-resolution rows of the upsample
    hr_pass::Img final;             // output 100
};

static int frame_begin(hr_pass* p, const hr_frame* f, bool denoise, const HaloPlan& plan, cudaStream_t st, PassFrame* fr)
{
    hr_ctx*        ctx = p->ctx;
    const HaloPlan h   = ctx->world > 1 && denoise ? plan : HaloPlan { 0, 0, 0 };
    fr->st = st;
    fr->pp = f->ping_pong;
    hr_band(ctx, p->H, &fr->b0, &fr->b1);
    hr_extend(fr->b0, fr->b1, h.ray_trace, p->H, &fr->rt0, &fr->rt1);
    hr_extend(fr->b0, fr->b1, h.denoise, p->H, &fr->row0, &fr->row1);
    hr_extend(fr->b0, fr->b1, h.vblur, p->H, &fr->v0, &fr->v1);
    fr->rt_halo     = h.ray_trace;
    fr->up0         = fr->b0 << p->scale;
    fr->up1         = fr->b1 >= p->H ? p->H0 : (fr->b1 << p->scale);
    p->last_rows[0] = denoise ? fr->row0 : 0; // the tile statistics cover the rows the denoise stages ran on: none without them
    p->last_rows[1] = denoise ? fr->row1 : 0;
    timer_begin(p, st);
    int rc = hr_peer_link_ipc(p, st); // first sharded render: map the peers' history / ray-trace images (collective, shard.cu)
    if (rc != HR_OK) return rc;
    fr->epoch = ++p->epoch;
    p->n_renders++;
    fr->no_history = p->first;
    return HR_OK;
}

// Publish this frame's history tick: every history image the next frame's reprojection reads from this rank is complete.
static int frame_signal(hr_pass* p, PassFrame& fr)
{
    fr.signalled = true;
    return hr_peer_signal(p, TICK_HIST, fr.epoch, fr.st);
}

static int frame_end(hr_pass* p, PassFrame& fr)
{
    if (!fr.signalled)
    {
        const int rc = frame_signal(p, fr);
        if (rc != HR_OK) return rc;
    }
    p->out_view[100] = fr.final;
    HR_CHECK_LAUNCH(p->ctx);
    return HR_OK;
}

static const char* const atrous_stage_names[8] = { "A-Trous 0", "A-Trous 1", "A-Trous 2", "A-Trous 3", "A-Trous 4", "A-Trous 5", "A-Trous 6", "A-Trous 7" };

// ---- stages shared by shadows and AO -------------------------------------------------------------------------------
static_assert((int)HR_SHADOWS_OUT_RAY_TRACE == (int)HR_AO_OUT_RAY_TRACE && (int)HR_SHADOWS_OUT_UPSAMPLE == (int)HR_AO_OUT_UPSAMPLE, "shared output slots");

// ray_trace (ray_traced_shadows.cpp:972-1011, ray_traced_ao.cpp:864-903): K1 (p0 = bias) or K7 (p0 = ray length, p1 = bias) into
// the mask image, or with spp > 1 into the count image, then the wait for last frame's history if the temporal stage reads it.
// Linked to peers: this rank traces its cost-balanced share of the WHOLE image and stores the mask words (spp > 1: the counts) into
// every rank's image of this frame's parity (no halo re-trace); otherwise its band +- the ray-trace halo into its own image.
static int trace_mask(hr_pass* p, PassFrame& fr, const GBufLevelDev& cur, const FrameConsts& fc, float p0, float p1, int spp, bool denoise, uint32_t** mask_out,
                      uint8_t** count_out, bool* shared_out)
{
    hr_ctx*      ctx    = p->ctx;
    const int    parity = fr.epoch & 1;
    const BvhDev bvh    = hr_bvh_view(ctx->scene);
    RtShare      rts;
    const bool   shared = hr_rt_share(p, parity, &rts);
    uint32_t*    mask   = shared ? p->mask_pp[parity] : p->mask;
    uint8_t*     count  = shared ? p->count_pp[parity] : p->count;
    int          rc;
    if (shared)
    {
        launch_ray_trace_shared(p->kind, cur, bvh, fc, p0, p1, ctx->d_sobol, bn_table(ctx, spp), count, spp, rts, fr.st);
        ctx->launches++;
        if ((rc = hr_rt_share_finish(p, parity, fr.epoch, spp > 1, fr.st)) != HR_OK) return rc;
        timer_mark(p, "Ray Trace", fr.st);
        // every rank's share of this frame's mask (and cost table) has arrived and, when the temporal stage reads it, last frame's
        // history is complete: this wait also covers the history tick, so the temporal stage does not wait on it again
        if ((rc = hr_rt_wait_partition(p, parity, fr.epoch, (denoise && !fr.no_history) ? fr.epoch - 1 : 0, fr.st)) != HR_OK) return rc;
        timer_mark(p, "Mask Exchange Wait", fr.st);
    }
    else
    {
        // SURVEY.md §8d: with spp > 1, spp rays per pixel into an 8-bit count image (allocated on first use)
        if (spp > 1 && !p->count && (rc = pass_alloc(p, p->count, (size_t)p->W * p->H)) != HR_OK) return rc;
        count = p->count;
        launch_ray_trace(p->kind, cur, bvh, fc, p0, p1, ctx->d_sobol, bn_table(ctx, spp), mask, count, spp, fr.rt0, fr.rt1, fr.st);
        ctx->launches++;
        timer_mark(p, "Ray Trace", fr.st);
        // the history = last frame's images of whichever rank owns the reprojected row (peer history, shard.cu): wait until every
        // peer has finished writing them (tick epoch - 1), overlapped with the ray trace above
        if (denoise && !fr.no_history && (rc = hr_peer_wait(p, TICK_HIST, fr.epoch - 1, fr.st)) != HR_OK) return rc;
    }
    if (spp > 1) fr.final = { count, p->W, p->H, HR_FMT_R8_UINT };
    else fr.final = { mask, (p->W + 7) / 8, (p->H + 3) / 4, HR_FMT_R32_UINT };
    p->out_view[HR_SHADOWS_OUT_RAY_TRACE] = fr.final;
    *mask_out   = mask;
    *count_out  = count;
    *shared_out = shared;
    return HR_OK;
}

// upsample (ray_traced_shadows.cpp:1219-1255, ray_traced_ao.cpp:918-957): the pass's last image to full resolution, the final output
static void upsample_scalar(hr_pass* p, PassFrame& fr, const GBufLevelDev& cur, const void* in, int in_channels, float sky_value, float power)
{
    hr_ctx* ctx = p->ctx;
    launch_upsample_scalar(level_view(ctx, fr.pp, 0), cur, in, in_channels, sky_value, power, p->upsample_out, fr.up0, fr.up1, fr.st);
    ctx->launches++;
    timer_mark(p, "Upsample", fr.st);
    fr.final = { p->upsample_out, p->W0, p->H0, HR_FMT_R16F };
    p->out_view[HR_SHADOWS_OUT_UPSAMPLE] = fr.final;
}

static int check_render_ready(hr_pass* p, const hr_frame* f, const void* params, bool needs_scene)
{
    hr_ctx* ctx = p ? p->ctx : nullptr;
    HR_REQUIRE(ctx, p && f && params, HR_ERR_INVALID_ARG, "render: null argument");
    HR_REQUIRE(ctx, ctx->gb_w == p->W0 && ctx->gb_h == p->H0, HR_ERR_NOT_READY, "render: G-buffer not created or size differs from the pass");
    HR_REQUIRE(ctx, !needs_scene || ctx->scene, HR_ERR_NOT_READY, "render: no scene set (hr_scene_build / hr_scene_set_current)");
    HR_REQUIRE(ctx, ctx->bn_set, HR_ERR_NOT_READY, "render: blue-noise tables not set (hr_bluenoise_set)");
    HR_REQUIRE(ctx, f->ping_pong == 0 || f->ping_pong == 1, HR_ERR_INVALID_ARG, "render: ping_pong must be 0 or 1");
    return HR_OK;
}

extern "C" {

// ---------------------------------------------------------------------------------------------------------------
// Shadows
// ---------------------------------------------------------------------------------------------------------------
void hr_shadows_default_params(hr_shadows_params* p)
{
    p->bias = 0.5f; p->alpha = 0.01f; p->moments_alpha = 0.2f; p->phi_visibility = 10.0f; p->phi_normal = 32.0f; p->sigma_depth = 1.0f;
    p->power = 1.2f; p->radius = 1; p->filter_iterations = 4; p->feedback_iteration = 1; p->denoise = 1; p->spp = 1;
}

int hr_shadows_create(hr_ctx* ctx, int width, int height, int scale, hr_pass** out)
{
    return pass_create(ctx, width, height, scale, PASS_SHADOWS, out, [](PassAllocs& A) {
        hr_pass*     p  = A.p;
        const size_t px = (size_t)p->W * p->H, mw = (p->W + 7) / 8, mh = (p->H + 3) / 4, tw = (p->W + 7) / 8, th = (p->H + 7) / 8;
        A(p->mask, mw * mh);
        A(p->temporal_out, px);
        A(p->moments[0], px);
        A(p->moments[1], px);
        A(p->prev_image[0], px);
        A(p->prev_image[1], px);
        A(p->atrous[0], px);
        A(p->atrous[1], px);
        A(p->tile_flags, tw * th);
        if (p->scale != HR_SCALE_FULL) A(p->upsample_out, (size_t)p->W0 * p->H0);
        pass_alloc_rt_share(A);
        void* hist[SHARED_N_SHADOWS_AO] = { p->prev_image[0], p->prev_image[1], p->moments[0], p->moments[1], p->mask_pp[0], p->mask_pp[1], p->rt_cost_all,
                                            p->count_pp[0], p->count_pp[1] };
        hr_peer_register(p, hist, SHARED_N_SHADOWS_AO);
        for (int i = 0; i < 2; i++)
        {
            p->hist_view[HR_SHADOWS_OUT_PREV_IMAGE][i] = { p->prev_image[i], p->W, p->H, HR_FMT_RG16F };
            p->hist_view[HR_SHADOWS_OUT_MOMENTS][i]    = { p->moments[i], p->W, p->H, HR_FMT_RGBA16F };
        }
    });
}

int hr_shadows_render(hr_pass* p, const hr_frame* f, const hr_shadows_params* prm, void* stream)
{
    int rc = check_render_ready(p, f, prm, true);
    if (rc != HR_OK) return rc;
    hr_ctx* ctx = p->ctx;
    HR_REQUIRE(ctx, p->kind == PASS_SHADOWS, HR_ERR_INVALID_ARG, "hr_shadows_render: not a shadows pass");
    HR_REQUIRE(ctx, prm->filter_iterations >= 0 && prm->filter_iterations <= 8 && prm->radius >= 1 && prm->radius <= 2, HR_ERR_INVALID_ARG,
               "hr_shadows_render: filter_iterations must be 0..8 and radius 1..2");
    cudaStream_t       st  = (cudaStream_t)stream;
    const int          pp  = f->ping_pong;
    const FrameConsts  fc  = make_consts(f, p);
    const GBufLevelDev cur = level_view(ctx, pp, p->scale), prev = level_view(ctx, !pp, p->scale);
    const size_t       px = (size_t)p->W * p->H;
    const int spp = prm->spp > 1 ? prm->spp : 1;
    HR_REQUIRE(ctx, spp <= 255, HR_ERR_UNSUPPORTED, "hr_shadows_render: spp must be <= 255");
    PassFrame fr;
    if ((rc = frame_begin(p, f, prm->denoise, halo_plan(PASS_SHADOWS, prm->radius, prm->filter_iterations, 0), st, &fr)) != HR_OK) return rc;
    hr_wait_exchange(p, st); // last frame's gather of the final output (side stream) reads images this frame rewrites
    // clear_images (ray_traced_shadows.cpp:938-968): first frame => history image and moments[!pp] = 0.  The reprojection
    // kernel is told not to read any history on that frame (same values as reading the cleared images, and no peer can be
    // caught reading a surface while it is being cleared); hr_pass_reset_history must be called on all ranks together.
    if (p->first)
    {
        HR_CUDA(ctx, cudaMemsetAsync(p->prev_image[!pp], 0, px * sizeof(__half2), st));
        HR_CUDA(ctx, cudaMemsetAsync(p->moments[!pp], 0, px * sizeof(uint2), st));
        p->first = false; // nothing below reads it (unlike reflections)
    }
    uint32_t* mask;
    uint8_t*  count;
    bool      shared_rt;
    if ((rc = trace_mask(p, fr, cur, fc, prm->bias, 0.0f, spp, prm->denoise != 0, &mask, &count, &shared_rt)) != HR_OK) return rc;
    if (prm->denoise)
    {
        // temporal_accumulation (:1041-1090); reset_args (:1015-1037) is subsumed by the per-tile flag image.
        // History = prev_image[!pp] / moments[!pp] of whichever rank owns the reprojected row (peer history, shard.cu).
        HistPeers hist;
        hr_peer_hist(p, SHARED_HIST + !pp, SHARED_HIST_AUX + !pp, p->H, fr.no_history, &hist);
        launch_temporal(PASS_SHADOWS, cur, prev, mask, count, spp, hist, fc, prm->alpha, prm->moments_alpha, p->temporal_out, p->moments[pp], p->tile_flags,
                        fr.row0, fr.row1, st);
        ctx->launches++;
        timer_mark(p, "Temporal Accumulation", st);
        // a_trous_filter (:1094-1215).  The reference ping-pongs image[0]/image[1] and copies the output of
        // feedback_iteration into prev_image; here that iteration writes this frame's history image directly and the next
        // one reads it.  prev_image is double buffered by frame parity (peers may still read last frame's).
        __half2* const hist_out = p->prev_image[pp];
        const __half2* in      = p->temporal_out;
        __half2*       last    = p->temporal_out;
        int            toggle  = 1; // reference: first write_idx = 1
        bool           fed_back = false;
        for (int i = 0; i < prm->filter_iterations; i++)
        {
            __half2* dst = (i == prm->feedback_iteration) ? hist_out : p->atrous[toggle];
            if (i == prm->filter_iterations - 1 && dst == hist_out)
            { // final output must not alias the history image: filter into atrous[], then copy (reference semantics)
                dst = p->atrous[toggle];
            }
            const float power = (i == prm->filter_iterations - 1) ? prm->power : 0.0f;
            launch_shadows_atrous(cur, in, p->tile_flags, prm->radius, 1 << i, prm->phi_visibility, prm->phi_normal, prm->sigma_depth, power, dst, fr.row0, fr.row1, st);
            ctx->launches++;
            if (i == prm->feedback_iteration)
            {
                if (dst != hist_out) HR_CUDA(ctx, cudaMemcpyAsync(hist_out, dst, px * sizeof(__half2), cudaMemcpyDeviceToDevice, st));
                fed_back = true;
                // shadows signal here, not after the temporal stage: prev_image[pp] is only complete after the feedback iteration
                if ((rc = frame_signal(p, fr)) != HR_OK) return rc;
            }
            in     = dst;
            last   = dst;
            toggle = !toggle;
            timer_mark(p, atrous_stage_names[i], st);
        }
        if (!fed_back)
        { // no feedback: the history image keeps its previous contents, like the reference's single prev_image
            HR_CUDA(ctx, cudaMemcpyAsync(hist_out, p->prev_image[!pp], px * sizeof(__half2), cudaMemcpyDeviceToDevice, st));
        }
        set_view(p, HR_SHADOWS_OUT_TEMPORAL_ACCUMULATION, p->temporal_out, p->W, p->H, HR_FMT_RG16F);
        set_view(p, HR_SHADOWS_OUT_ATROUS, last, p->W, p->H, HR_FMT_RG16F);
        set_view(p, HR_SHADOWS_OUT_MOMENTS, p->moments[pp], p->W, p->H, HR_FMT_RGBA16F);
        set_view(p, HR_SHADOWS_OUT_PREV_IMAGE, hist_out, p->W, p->H, HR_FMT_RG16F);
        set_view(p, HR_SHADOWS_OUT_TILE_FLAGS, p->tile_flags, (p->W + 7) / 8, (p->H + 7) / 8, HR_FMT_R8_UINT);
        fr.final = { last, p->W, p->H, HR_FMT_RG16F };
        if (p->scale != HR_SCALE_FULL) upsample_scalar(p, fr, cur, last, 2, 0.0f, 0.0f);
    }
    if ((rc = frame_end(p, fr)) != HR_OK) return rc;
    if (ctx->world > 1 && ctx->gather_final && !(shared_rt && !prm->denoise))
    { // every rank ends up with the complete final output (the history stays distributed: peer history, shard.cu)
        ExchangeItem it[2];
        int          n = 0;
        if (prm->denoise)
        {
            if (fr.final.fmt == HR_FMT_RG16F) it[n++] = { fr.final.p, (size_t)p->W * 4, p->H, 0, 1, p->H };
            if (fr.final.fmt == HR_FMT_R16F) it[n++] = { fr.final.p, (size_t)p->W0 * 2, p->H, p->scale, 1, p->H0 };
        }
        else it[n++] = { mask, (size_t)((p->W + 7) / 8) * 4, p->H, 0, 4, (p->H + 3) / 4 };
        rc = hr_shard_exchange(p, it, n, st);
        if (rc != HR_OK) return rc;
        timer_mark(p, "Exchange", st);
    }
    return HR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Ambient occlusion
// ---------------------------------------------------------------------------------------------------------------
void hr_ao_default_params(hr_ao_params* p)
{
    p->ray_length = 7.0f; p->bias = 0.3f; p->alpha = 0.01f; p->power = 1.2f; p->blur_radius = 4; p->denoise = 1; p->spp = 1;
}

int hr_ao_create(hr_ctx* ctx, int width, int height, int scale, hr_pass** out)
{
    return pass_create(ctx, width, height, scale, PASS_AO, out, [](PassAllocs& A) {
        hr_pass*     p  = A.p;
        const size_t px = (size_t)p->W * p->H, mw = (p->W + 7) / 8, mh = (p->H + 3) / 4, tw = (p->W + 7) / 8, th = (p->H + 7) / 8;
        A(p->mask, mw * mh);
        for (int i = 0; i < 2; i++)
        {
            A(p->ao_color[i], px);
            A(p->ao_len[i], px);
            A(p->ao_blur[i], px);
        }
        A(p->tile_flags, tw * th);
        if (p->scale != HR_SCALE_FULL) A(p->upsample_out, (size_t)p->W0 * p->H0);
        pass_alloc_rt_share(A);
        void* hist[SHARED_N_SHADOWS_AO] = { p->ao_color[0], p->ao_color[1], p->ao_len[0], p->ao_len[1], p->mask_pp[0], p->mask_pp[1], p->rt_cost_all,
                                            p->count_pp[0], p->count_pp[1] };
        hr_peer_register(p, hist, SHARED_N_SHADOWS_AO);
        for (int i = 0; i < 2; i++)
        {
            p->hist_view[HR_AO_OUT_TEMPORAL_ACCUMULATION][i] = { p->ao_color[i], p->W, p->H, HR_FMT_R16F };
            p->hist_view[HR_AO_OUT_HISTORY_LENGTH][i]        = { p->ao_len[i], p->W, p->H, HR_FMT_R16F };
        }
    });
}

int hr_ao_render(hr_pass* p, const hr_frame* f, const hr_ao_params* prm, void* stream)
{
    int rc = check_render_ready(p, f, prm, true);
    if (rc != HR_OK) return rc;
    hr_ctx* ctx = p->ctx;
    HR_REQUIRE(ctx, p->kind == PASS_AO, HR_ERR_INVALID_ARG, "hr_ao_render: not an AO pass");
    HR_REQUIRE(ctx, prm->blur_radius >= 1 && prm->blur_radius <= 16, HR_ERR_INVALID_ARG, "hr_ao_render: blur_radius must be 1..16");
    cudaStream_t       st  = (cudaStream_t)stream;
    const int          pp  = f->ping_pong;
    const FrameConsts  fc  = make_consts(f, p);
    const GBufLevelDev cur = level_view(ctx, pp, p->scale), prev = level_view(ctx, !pp, p->scale);
    const size_t       px = (size_t)p->W * p->H;
    const int spp = prm->spp > 1 ? prm->spp : 1;
    HR_REQUIRE(ctx, spp <= 255, HR_ERR_UNSUPPORTED, "hr_ao_render: spp must be <= 255");
    PassFrame fr;
    if ((rc = frame_begin(p, f, prm->denoise, halo_plan(PASS_AO, 0, 0, prm->blur_radius), st, &fr)) != HR_OK) return rc;
    hr_wait_exchange(p, st);
    if (p->first)
    { // clear_images, ray_traced_ao.cpp:829-860 (see hr_shadows_render for the first-frame / peer rules)
        HR_CUDA(ctx, cudaMemsetAsync(p->ao_len[!pp], 0, px * sizeof(__half), st));
        HR_CUDA(ctx, cudaMemsetAsync(p->ao_color[!pp], 0, px * sizeof(__half), st));
        p->first = false;
    }
    uint32_t* mask;
    uint8_t*  count;
    bool      shared_rt;
    if ((rc = trace_mask(p, fr, cur, fc, prm->ray_length, prm->bias, spp, prm->denoise != 0, &mask, &count, &shared_rt)) != HR_OK) return rc;
    if (prm->denoise)
    {
        // history = ao_color[!pp] / ao_len[!pp] of the rank that owns the reprojected row (peer history, shard.cu)
        HistPeers hist;
        hr_peer_hist(p, SHARED_HIST + !pp, SHARED_HIST_AUX + !pp, p->H, fr.no_history, &hist);
        launch_temporal(PASS_AO, cur, prev, mask, count, spp, hist, fc, prm->alpha, 0.0f, p->ao_color[pp], p->ao_len[pp], p->tile_flags, fr.row0, fr.row1, st);
        ctx->launches++;
        if ((rc = frame_signal(p, fr)) != HR_OK) return rc; // this frame's history (ao_color[pp], ao_len[pp]) is complete
        timer_mark(p, "Temporal Accumulation", st);
        // bilateral_blur (:1032-1137): pass labelled "Vertical" uses direction (1,0), then (0,1)
        launch_ao_blur(cur, p->ao_color[pp], p->tile_flags, f->z_buffer_params, 1, 0, prm->blur_radius, p->ao_blur[0], fr.row0, fr.row1, st);
        launch_ao_blur(cur, p->ao_blur[0], p->tile_flags, f->z_buffer_params, 0, 1, prm->blur_radius, p->ao_blur[1], fr.v0, fr.v1, st);
        ctx->launches += 2;
        timer_mark(p, "Bilateral Blur", st);
        set_view(p, HR_AO_OUT_TEMPORAL_ACCUMULATION, p->ao_color[pp], p->W, p->H, HR_FMT_R16F);
        set_view(p, HR_AO_OUT_HISTORY_LENGTH, p->ao_len[pp], p->W, p->H, HR_FMT_R16F);
        set_view(p, HR_AO_OUT_BILATERAL_BLUR, p->ao_blur[1], p->W, p->H, HR_FMT_R16F);
        set_view(p, HR_AO_OUT_TILE_FLAGS, p->tile_flags, (p->W + 7) / 8, (p->H + 7) / 8, HR_FMT_R8_UINT);
        fr.final = { p->ao_blur[1], p->W, p->H, HR_FMT_R16F };
        if (p->scale != HR_SCALE_FULL) upsample_scalar(p, fr, cur, p->ao_blur[1], 1, 1.0f, prm->power);
    }
    if ((rc = frame_end(p, fr)) != HR_OK) return rc;
    if (ctx->world > 1 && ctx->gather_final && !(shared_rt && !prm->denoise))
    {
        ExchangeItem it[4];
        int          n = 0;
        if (prm->denoise)
        {
            if (p->scale == HR_SCALE_FULL) it[n++] = { p->ao_blur[1], (size_t)p->W * 2, p->H, 0, 1, p->H };
            else it[n++] = { p->upsample_out, (size_t)p->W0 * 2, p->H, p->scale, 1, p->H0 };
        }
        else it[n++] = { mask, (size_t)((p->W + 7) / 8) * 4, p->H, 0, 4, (p->H + 3) / 4 };
        rc = hr_shard_exchange(p, it, n, st);
        if (rc != HR_OK) return rc;
        timer_mark(p, "Exchange", st);
    }
    return HR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Common pass functions
// ---------------------------------------------------------------------------------------------------------------
int hr_pass_output(hr_pass* p, int which, hr_image* out)
{
    hr_ctx* ctx = p ? p->ctx : nullptr;
    HR_REQUIRE(ctx, p && out && which >= 0 && which < 128, HR_ERR_INVALID_ARG, "hr_pass_output: bad argument");
    const hr_pass::Img& v = p->out_view[which];
    HR_REQUIRE(ctx, v.p != nullptr, HR_ERR_NOT_READY, "hr_pass_output: output not produced by the last render");
    // a borrowed pointer may be consumed on any stream: finish a pending band exchange first (sharded runs only)
    if (p->xchg_pending && p->ev_done) { cudaEventSynchronize(p->ev_done); p->xchg_pending = false; }
    out->data = v.p; out->width = v.w; out->height = v.h; out->format = v.fmt;
    return HR_OK;
}

} // extern "C"

// Rows [row0,row1) of output `which` (all of them when all_rows) into dst, enqueued on `st` after the pass's pending exchange;
// `who` names the entry point in error messages.
static int download_rows(hr_pass* p, int which, bool all_rows, int row0, int row1, void* dst, size_t bytes, cudaMemcpyKind kind, cudaStream_t st, const char* who)
{
    hr_image img;
    int      rc = hr_pass_output(p, which, &img);
    if (rc != HR_OK) return rc;
    hr_ctx* ctx = p->ctx;
    if (all_rows) { row0 = 0; row1 = img.height; }
    if (!(row0 >= 0 && row1 >= row0 && row1 <= img.height)) { hr_set_error(ctx, "%s: bad row range", who); return HR_ERR_INVALID_ARG; }
    const size_t row_bytes = (size_t)img.width * texel_size(img.format), need = row_bytes * (size_t)(row1 - row0);
    if (!(dst && bytes == need)) { hr_set_error(ctx, "%s: byte count mismatch", who); return HR_ERR_INVALID_ARG; }
    hr_wait_exchange(p, st);
    if (need) HR_CUDA(ctx, cudaMemcpyAsync(dst, static_cast<const char*>(img.data) + row_bytes * row0, need, kind, st));
    return HR_OK;
}

extern "C" {

// hr_pass_download without the host synchronisation: the caller orders it with its own stream / event waits.
int hr_pass_download_async(hr_pass* p, int which, void* dst, size_t bytes, void* stream)
{
    return download_rows(p, which, true, 0, 0, dst, bytes, cudaMemcpyDefault, (cudaStream_t)stream, "hr_pass_download_async");
}

// Rows [row0,row1) of an image (a rank's own band of a distributed output), asynchronous like hr_pass_download_async.
int hr_pass_download_rows_async(hr_pass* p, int which, int row0, int row1, void* dst, size_t bytes, void* stream)
{
    return download_rows(p, which, false, row0, row1, dst, bytes, cudaMemcpyDefault, (cudaStream_t)stream, "hr_pass_download_rows_async");
}

int hr_pass_download(hr_pass* p, int which, void* dst, size_t bytes, void* stream)
{
    const int rc = download_rows(p, which, true, 0, 0, dst, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream, "hr_pass_download");
    if (rc != HR_OK) return rc;
    HR_CUDA(p->ctx, cudaStreamSynchronize((cudaStream_t)stream));
    return HR_OK;
}

// Restore half of checkpoint / resume (the reference keeps its temporal history only in GPU images and has no such
// facility, SURVEY.md §5): overwrite one of the pass's images, e.g. the history surfaces saved with hr_pass_download.
int hr_pass_upload(hr_pass* p, int which, const void* src, size_t bytes, void* stream)
{
    if (p && p->epoch == 0 && which >= 0 && which < 8 && p->hist_view[which][0].p)
    { // cold start (a fresh process restoring a checkpoint before its first render): the next render reads the history of
      // parity !ping_pong, which is not known yet — restore both parities and skip that render's first-frame clear
        hr_ctx*             ctx  = p->ctx;
        const hr_pass::Img& v    = p->hist_view[which][0];
        const size_t        need = (size_t)v.w * v.h * texel_size(v.fmt);
        HR_REQUIRE(ctx, src && bytes == need, HR_ERR_INVALID_ARG, "hr_pass_upload: byte count mismatch");
        for (int i = 0; i < 2; i++) HR_CUDA(ctx, cudaMemcpyAsync(p->hist_view[which][i].p, src, need, cudaMemcpyHostToDevice, (cudaStream_t)stream));
        HR_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
        p->first = false;
        return HR_OK;
    }
    hr_image img;
    int      rc = hr_pass_output(p, which, &img);
    if (rc != HR_OK) return rc;
    hr_ctx*      ctx  = p->ctx;
    const size_t need = (size_t)img.width * img.height * texel_size(img.format);
    HR_REQUIRE(ctx, src && bytes == need, HR_ERR_INVALID_ARG, "hr_pass_upload: byte count mismatch");
    hr_wait_exchange(p, (cudaStream_t)stream);
    HR_CUDA(ctx, cudaMemcpyAsync(img.data, src, need, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    HR_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    return HR_OK;
}

int hr_pass_reset_history(hr_pass* p) { if (!p) return HR_ERR_INVALID_ARG; p->first = true; return HR_OK; }

int hr_pass_get_stats(hr_pass* p, hr_pass_stats* out, void* stream)
{
    hr_ctx* ctx = p ? p->ctx : nullptr;
    HR_REQUIRE(ctx, p && out, HR_ERR_INVALID_ARG, "hr_pass_get_stats: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    memset(out, 0, sizeof(*out));
    unsigned long long* d = nullptr;
    HR_CUDA(ctx, cudaMalloc((void**)&d, 4 * sizeof(unsigned long long)));
    HR_CUDA(ctx, cudaMemsetAsync(d, 0, 4 * sizeof(unsigned long long), st));
    launch_drain_ray_counters(p->ray_ctr, d, st);
    const int r0 = p->last_rows[0], r1 = p->last_rows[1], TW = (p->W + 7) / 8;
    const int t0 = r0 / 8, t1 = (r1 + 7) / 8;
    if (p->tile_flags && r1 > r0) launch_tile_stats(p->tile_flags, TW, t0, t1, d + 2, st);
    unsigned long long h[4] = {};
    cudaError_t e = cudaMemcpyAsync(h, d, sizeof(h), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    HR_CUDA(ctx, e);
    out->rays_primary   = h[0];
    out->rays_secondary = h[1];
    out->renders        = p->n_renders;
    p->n_renders        = 0;
    if (p->tile_flags && r1 > r0)
    {
        out->tiles_total   = (uint64_t)(t1 - t0) * TW;
        out->tiles_denoise = h[2];
        out->pixels_total  = (uint64_t)(r1 - r0) * p->W;
    }
    return HR_OK;
}

int hr_pass_output_checksum(hr_pass* p, int which, int row0, int row1, uint64_t* out, void* stream)
{
    hr_image img;
    int      rc = hr_pass_output(p, which, &img);
    if (rc != HR_OK) return rc;
    hr_ctx* ctx = p->ctx;
    HR_REQUIRE(ctx, out != nullptr, HR_ERR_INVALID_ARG, "hr_pass_output_checksum: null argument");
    if (row1 <= 0) { row0 = 0; row1 = img.height; }
    HR_REQUIRE(ctx, row0 >= 0 && row1 >= row0 && row1 <= img.height, HR_ERR_INVALID_ARG, "hr_pass_output_checksum: bad row range");
    cudaStream_t st = (cudaStream_t)stream;
    hr_wait_exchange(p, st);
    unsigned long long* d = nullptr;
    HR_CUDA(ctx, cudaMalloc((void**)&d, sizeof(unsigned long long)));
    HR_CUDA(ctx, cudaMemsetAsync(d, 0, sizeof(unsigned long long), st));
    launch_checksum(img.data, texel_size(img.format), (size_t)img.width * row0, (size_t)img.width * row1, d, st);
    unsigned long long h = 0;
    cudaError_t e = cudaMemcpyAsync(&h, d, sizeof(h), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    HR_CUDA(ctx, e);
    *out = h;
    return HR_OK;
}

int hr_pass_destroy(hr_pass* p)
{
    if (!p) return HR_ERR_INVALID_ARG;
    cudaSetDevice(p->ctx->device);
    cudaDeviceSynchronize();
    hr_peer_unlink(p);
    for (void* a : p->allocs) cudaFree(a);
    for (void* a : p->ddgi_grid_allocs) cudaFree(a);
    for (void* a : p->ddgi_retired) cudaFree(a);
    if (p->ddgi_pool) cudaMemPoolDestroy(p->ddgi_pool);
    if (p->ev_ready) cudaEventDestroy(p->ev_ready);
    if (p->ev_done) cudaEventDestroy(p->ev_done);
    for (auto& r : p->timer.recs) for (auto e : r.ev) cudaEventDestroy(e);
    for (auto e : p->timer.pool) cudaEventDestroy(e);
    delete p;
    return HR_OK;
}

int hr_pass_stage_times(hr_pass* p, const char** names, float* ms, int cap, int* n)
{
    if (!p || !n) return HR_ERR_INVALID_ARG;
    *n = 0;
    StageTimer& T = p->timer;
    if (T.recs.empty()) return HR_OK;
    // by name: the stage list changes between renders (a first TAA render's reset blit, filter_iterations, the gather, the upsample),
    // so each name's entry is the mean over the renders that recorded it, in first-seen order
    std::vector<double> sum;
    std::vector<int>    cnt;
    T.last_names.clear();
    for (auto& r : T.recs)
    {
        cudaEventSynchronize(r.ev.back());
        for (size_t i = 0; i + 1 < r.ev.size(); i++)
        {
            float t = 0.0f;
            cudaEventElapsedTime(&t, r.ev[i], r.ev[i + 1]);
            size_t j = 0;
            while (j < T.last_names.size() && T.last_names[j] != r.names[i]) j++;
            if (j == T.last_names.size()) { sum.push_back(0.0); cnt.push_back(0); T.last_names.push_back(r.names[i]); }
            sum[j] += t;
            cnt[j]++;
        }
        for (auto e : r.ev) T.pool.push_back(e);
    }
    T.recs.clear();
    for (size_t i = 0; i < sum.size() && (int)i < cap; i++)
    {
        if (names) names[i] = T.last_names[i].c_str();
        if (ms) ms[i] = (float)(sum[i] / cnt[i]);
        (*n)++;
    }
    return HR_OK;
}

int hr_shard_rows(int height, int rank, int world, int* row_begin, int* row_end)
{
    if (height <= 0 || world <= 0 || rank < 0 || rank >= world || !row_begin || !row_end) return HR_ERR_INVALID_ARG;
    const int tiles = (height + 7) / 8;
    const int base = tiles / world, rem = tiles % world;
    const int t0 = rank * base + (rank < rem ? rank : rem), t1 = t0 + base + (rank < rem ? 1 : 0);
    *row_begin = t0 * 8 < height ? t0 * 8 : height;
    *row_end   = t1 * 8 < height ? t1 * 8 : height;
    return HR_OK;
}

// Band assignment without a communicator: the caller performs the exchange itself (tests emulate N ranks on one GPU).
int hr_shard_config(hr_ctx* ctx, int rank, int world)
{
    HR_REQUIRE(ctx, ctx && world >= 1 && rank >= 0 && rank < world, HR_ERR_INVALID_ARG, "hr_shard_config: bad rank/world");
    HR_REQUIRE(ctx, world <= HR_MAX_RANKS, HR_ERR_UNSUPPORTED, "hr_shard_config: at most 8 ranks (the GPUs of one box)");
    ctx->rank  = rank;
    ctx->world = world;
    return HR_OK;
}

} // extern "C"

#include "hr_api_gi.inc"
#include "hr_api_post.inc"
#include "hr_api_reference.inc"
