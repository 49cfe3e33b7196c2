// hybrid_rendering.h — C++ host classes that keep the reference's pass interfaces on top of the C ABI (hr_api.h).
//
//   reference                                      here
//   CommonResources (src/common.h:181-243)         hr::CommonResources  (hr_ctx + per-frame hr_frame + blue noise + scene)
//   GBuffer         (src/g_buffer.h)               hr::GBuffer          (two device slots; output()/history() by ping_pong)
//   RayTracedShadows(src/ray_traced_shadows.h)     hr::RayTracedShadows (ctor(common, gbuffer, scale); render(stream); output())
//   RayTracedAO     (src/ray_traced_ao.h)          hr::RayTracedAO
//   DDGI / RayTracedReflections / DeferredShading  hr::DDGI, hr::RayTracedReflections, hr::DeferredShading
//   TemporalAA / ToneMap / GroundTruthPathTracer   hr::TemporalAA, hr::ToneMap, hr::GroundTruthPathTracer
// Same method names and argument meaning; `dw::vk::CommandBuffer::Ptr` becomes a CUDA stream, descriptor sets become
// hr_image views; construction errors throw std::runtime_error like the reference (common.cpp:350-353), render() does
// not fail observably in the reference — here a failed launch throws as well.
#pragma once
#include "../../include/hr_api.h"
#include "assets.h"
#include "hr_math.h"
#include "synth.h"
#include <stdexcept>
#include <string>

namespace hr {

enum RayTraceScale { RAY_TRACE_SCALE_FULL_RES = HR_SCALE_FULL, RAY_TRACE_SCALE_HALF_RES = HR_SCALE_HALF, RAY_TRACE_SCALE_QUARTER_RES = HR_SCALE_QUARTER }; // common.h:39-44

inline void check(hr_ctx* ctx, int rc, const char* what)
{
    if (rc != HR_OK) throw std::runtime_error(std::string(what) + ": " + hr_last_error(ctx));
}

struct CommonResources {
    hr_ctx*   ctx   = nullptr;
    hr_scene* scene = nullptr;
    // the fields the passes read every frame (common.h:186-191)
    bool      first_frame = true;
    bool      ping_pong   = false;
    int32_t   num_frames  = 0;
    hr_frame  frame {};
    uint32_t  width, height;

    CommonResources(int device, uint32_t w, uint32_t h) : width(w), height(h)
    {
        if (hr_init(device, &ctx) != HR_OK) throw std::runtime_error(std::string("hr_init: ") + hr_last_error(nullptr));
    }
    ~CommonResources()
    {
        if (scene) hr_scene_destroy(scene);
        if (ctx) hr_shutdown(ctx);
    }
    CommonResources(const CommonResources&)            = delete;
    CommonResources& operator=(const CommonResources&) = delete;

    void set_blue_noise(const uint8_t* sobol, const uint8_t* scr_rank) { check(ctx, hr_bluenoise_set(ctx, sobol, scr_rank), "hr_bluenoise_set"); }
    void load_scene(const hrs_scene* s)
    { // CommonResources::load_mesh + RayTracedScene creation (common.cpp:340-534)
        uint64_t nv, ni, nin, nm;
        hrs_scene_counts(s, &nv, &ni, &nin, &nm);
        check(ctx, hr_scene_build(ctx, hrs_scene_vertices(s), nv, hrs_scene_indices(s), ni, hrs_scene_instances(s), nin, hrs_scene_materials(s), nm, &scene),
              "hr_scene_build");
        check(ctx, hr_scene_set_current(ctx, scene), "hr_scene_set_current");
    }
    // the same with meshes read from disk: dw::Mesh::load + RayTracedScene::create (common.cpp:340-534) = hra_mesh_load + hra_scene_* (assets.h)
    void load_scene(const hra_scene* s)
    {
        uint64_t nv, ni, nin, nm;
        hra_scene_counts(s, &nv, &ni, &nin, &nm);
        if (scene) { hr_scene_destroy(scene); scene = nullptr; }
        check(ctx, hr_scene_build(ctx, hra_scene_vertices(s), nv, hra_scene_indices(s), ni, hra_scene_instances(s), nin, hra_scene_materials(s), nm, &scene),
              "hr_scene_build");
        check(ctx, hr_scene_set_current(ctx, scene), "hr_scene_set_current");
        uint64_t nt = 0, nb = 0; // Material::load: the images the materials reference (PNG), bound like s_Textures[] (hr_scene_set_textures)
        hra_scene_texture_counts(s, &nt, &nb);
        if (nt > 0) check(ctx, hr_scene_set_textures(scene, hra_scene_textures(s), nt, hra_scene_material_textures(s), nb), "hr_scene_set_textures");
    }
    // BlueNoise::BlueNoise (blue_noise.cpp:21-33): the Sobol' table and every scrambling / ranking table found in `dir`
    void load_blue_noise(const char* dir)
    {
        std::string sobol(256 * 4, '\0'), sr(9ull * 128 * 128 * 4, '\0');
        uint32_t    slots = 0;
        if (hra_bluenoise_load(dir, (uint8_t*)&sobol[0], (uint8_t*)&sr[0], &slots) != HRA_OK) throw std::runtime_error(std::string("hra_bluenoise_load: ") + hra_last_error());
        set_blue_noise((const uint8_t*)sobol.data(), (const uint8_t*)sr.data());
        for (int s = 1; s < 9; s++)
            if (slots & (1u << s)) check(ctx, hr_bluenoise_set_slot(ctx, s, (const uint8_t*)sr.data() + (size_t)s * 128 * 128 * 4), "hr_bluenoise_set_slot");
    }
    hr_scene* current_scene() { return scene; }
    // HybridRendering::update_uniforms (main.cpp:937-972) for a look-at camera
    void update_uniforms(const float cam_pos[3], const float cam_target[3], const hrs_light_desc* light)
    {
        hr_frame prev = frame;
        hrs_make_frame(&frame, cam_pos, cam_target, (int)width, (int)height, light, first_frame ? nullptr : &prev, (uint32_t)num_frames);
        frame.ping_pong   = ping_pong ? 1 : 0;
        frame.first_frame = first_frame ? 1 : 0;
    }
    // end of HybridRendering::update (main.cpp:123-128)
    void end_frame()
    {
        num_frames++;
        first_frame = false;
        ping_pong   = !ping_pong;
    }
};

struct GBuffer {
    CommonResources* common;
    GBuffer(CommonResources* c) : common(c) { check(c->ctx, hr_gbuffer_create(c->ctx, (int)c->width, (int)c->height), "hr_gbuffer_create"); }
    // GBuffer::render (g_buffer.cpp:39-189) replaced by: upload the CPU-written G-buffer of this frame into slot[ping_pong]
    void render(const hr_gbuffer_desc* host_mip0, void* stream) { check(common->ctx, hr_gbuffer_upload(common->ctx, common->ping_pong ? 1 : 0, host_mip0, stream), "hr_gbuffer_upload"); }
    // streaming host frames (INTEGRATION.md §4): stage_next() starts the PCIe copy of the NEXT frame on the library's upload
    // stream, render_staged() swaps the staged surface into this frame's slot on `stream` (no copy) and builds the mips
    void stage_next(const hr_gbuffer_desc* host_mip0) { check(common->ctx, hr_gbuffer_stage_upload(common->ctx, host_mip0), "hr_gbuffer_stage_upload"); }
    void render_staged(void* stream) { check(common->ctx, hr_gbuffer_commit_staged(common->ctx, common->ping_pong ? 1 : 0, stream), "hr_gbuffer_commit_staged"); }
    // GBuffer::render (g_buffer.cpp:100-263) on the device: primary-visibility ray cast of the current scene for this frame's camera
    void render(void* stream) { check(common->ctx, hr_gbuffer_render(common->ctx, common->ping_pong ? 1 : 0, &common->frame, 0, 0, stream), "hr_gbuffer_render"); }
    void bind_device(const hr_gbuffer_desc* dev_mip0, void* stream) { check(common->ctx, hr_gbuffer_bind_device(common->ctx, common->ping_pong ? 1 : 0, dev_mip0, stream), "hr_gbuffer_bind_device"); }
};

class RayTracedShadows {
public:
    enum OutputType { OUTPUT_RAY_TRACE = 0, OUTPUT_TEMPORAL_ACCUMULATION = 1, OUTPUT_ATROUS = 2, OUTPUT_UPSAMPLE = 3 }; // ray_traced_shadows.h:10-16
    RayTracedShadows(CommonResources* common, GBuffer* g_buffer, RayTraceScale scale = RAY_TRACE_SCALE_FULL_RES) : m_common(common), m_scale(scale)
    {
        (void)g_buffer;
        hr_shadows_default_params(&params);
        check(common->ctx, hr_shadows_create(common->ctx, (int)common->width, (int)common->height, scale, &m_pass), "hr_shadows_create");
        m_width  = common->width >> scale;
        m_height = common->height >> scale;
    }
    ~RayTracedShadows() { if (m_pass) hr_pass_destroy(m_pass); }
    void       render(void* stream) { check(m_common->ctx, hr_shadows_render(m_pass, &m_common->frame, &params, stream), "hr_shadows_render"); }
    hr_image   output_ds() const { return output(m_current_output_final ? 100 : (int)m_current_output); }
    hr_image   output(int which) const { hr_image img {}; check(m_common->ctx, hr_pass_output(m_pass, which, &img), "hr_pass_output"); return img; }
    uint32_t   width() const { return m_width; }
    uint32_t   height() const { return m_height; }
    RayTraceScale scale() const { return m_scale; }
    OutputType current_output() const { return m_current_output; }
    void       set_current_output(OutputType t) { m_current_output = t; m_current_output_final = false; }
    hr_pass*   handle() { return m_pass; }
    hr_shadows_params params; // the ImGui-bound members of the reference (ray_traced_shadows.cpp:120-131)
private:
    CommonResources* m_common;
    hr_pass*         m_pass = nullptr;
    RayTraceScale    m_scale;
    uint32_t         m_width = 0, m_height = 0;
    OutputType       m_current_output = OUTPUT_ATROUS;
    bool             m_current_output_final = true;
};

class RayTracedAO {
public:
    enum OutputType { OUTPUT_RAY_TRACE = 0, OUTPUT_TEMPORAL_ACCUMULATION = 1, OUTPUT_BILATERAL_BLUR = 2, OUTPUT_UPSAMPLE = 3 }; // ray_traced_ao.h:10-16
    RayTracedAO(CommonResources* common, GBuffer* g_buffer, RayTraceScale scale = RAY_TRACE_SCALE_HALF_RES) : m_common(common), m_scale(scale)
    {
        (void)g_buffer;
        hr_ao_default_params(&params);
        check(common->ctx, hr_ao_create(common->ctx, (int)common->width, (int)common->height, scale, &m_pass), "hr_ao_create");
        m_width  = common->width >> scale;
        m_height = common->height >> scale;
    }
    ~RayTracedAO() { if (m_pass) hr_pass_destroy(m_pass); }
    void       render(void* stream) { check(m_common->ctx, hr_ao_render(m_pass, &m_common->frame, &params, stream), "hr_ao_render"); }
    hr_image   output_ds() const { return output(100); }
    hr_image   output(int which) const { hr_image img {}; check(m_common->ctx, hr_pass_output(m_pass, which, &img), "hr_pass_output"); return img; }
    uint32_t   width() const { return m_width; }
    uint32_t   height() const { return m_height; }
    RayTraceScale scale() const { return m_scale; }
    hr_pass*   handle() { return m_pass; }
    hr_ao_params params;
private:
    CommonResources* m_common;
    hr_pass*         m_pass = nullptr;
    RayTraceScale    m_scale;
    uint32_t         m_width = 0, m_height = 0;
};

// DDGI (src/ddgi.h): ctor(backend, common, g_buffer, scale); render(cmd_buf); current_read_ds(); probe_counts(); restart_accumulation()
class DDGI {
public:
    DDGI(CommonResources* common, GBuffer* g_buffer, RayTraceScale scale = RAY_TRACE_SCALE_FULL_RES) : m_common(common), m_scale(scale)
    {
        (void)g_buffer;
        hr_ddgi_default_params(&params);
        check(common->ctx, hr_ddgi_create(common->ctx, (int)common->width, (int)common->height, scale, &m_pass), "hr_ddgi_create");
    }
    ~DDGI() { if (m_pass) hr_pass_destroy(m_pass); }
    // random_orientation replaces the std::mt19937(std::random_device()) draw of ddgi.cpp:73,788 (the caller seeds it)
    void     render(const float* random_orientation16, void* stream) { check(m_common->ctx, hr_ddgi_render(m_pass, &m_common->frame, &params, random_orientation16, stream), "hr_ddgi_render"); }
    hr_image output_ds() const { hr_image img {}; check(m_common->ctx, hr_pass_output(m_pass, HR_DDGI_OUT_FINAL, &img), "hr_pass_output"); return img; }
    hr_image current_read_ds(int which /* HR_DDGI_OUT_IRRADIANCE or _DEPTH */) const { hr_image img {}; check(m_common->ctx, hr_pass_output(m_pass, which, &img), "hr_pass_output"); return img; }
    void     probe_counts(int out[3]) const { hr_ddgi_uniforms u; check(m_common->ctx, hr_ddgi_get_uniforms(m_pass, &u), "hr_ddgi_get_uniforms"); out[0] = u.probe_counts[0]; out[1] = u.probe_counts[1]; out[2] = u.probe_counts[2]; }
    void     restart_accumulation() { hr_pass_reset_history(m_pass); } // ddgi.h:33
    void     set_probe_distance(float v) { params.probe_distance = v; }
    void     set_normal_bias(float v) { params.normal_bias = v; }
    RayTraceScale scale() const { return m_scale; }
    hr_pass* handle() { return m_pass; }
    hr_ddgi_params params;
private:
    CommonResources* m_common;
    hr_pass*         m_pass = nullptr;
    RayTraceScale    m_scale;
};

// DeferredShading (src/deferred_shading.h): render(cmd_buf, shadows, ao, reflections, ddgi) -> output image
class DeferredShading {
public:
    DeferredShading(CommonResources* common, GBuffer* g_buffer) : m_common(common)
    {
        (void)g_buffer;
        params.env_color[0] = params.env_color[1] = params.env_color[2] = 0.0f;
        check(common->ctx, hr_deferred_create(common->ctx, (int)common->width, (int)common->height, &m_pass), "hr_deferred_create");
    }
    ~DeferredShading() { if (m_pass) hr_pass_destroy(m_pass); }
    void     render(void* stream, hr_pass* shadows, hr_pass* ao, hr_pass* reflections, hr_pass* ddgi)
    {
        check(m_common->ctx, hr_deferred_render(m_pass, &m_common->frame, &params, shadows, ao, reflections, ddgi, stream), "hr_deferred_render");
    }
    hr_image output_ds() const { hr_image img {}; check(m_common->ctx, hr_pass_output(m_pass, 100, &img), "hr_pass_output"); return img; }
    hr_pass* handle() { return m_pass; }
    hr_deferred_params params;
private:
    CommonResources* m_common;
    hr_pass*         m_pass = nullptr;
};

// RayTracedReflections (src/ray_traced_reflections.h): render(cmd_buf, DDGI*)
class RayTracedReflections {
public:
    enum OutputType { OUTPUT_RAY_TRACE = 0, OUTPUT_TEMPORAL_ACCUMULATION = 1, OUTPUT_ATROUS = 2, OUTPUT_UPSAMPLE = 3 };
    RayTracedReflections(CommonResources* common, GBuffer* g_buffer, RayTraceScale scale = RAY_TRACE_SCALE_HALF_RES) : m_common(common), m_scale(scale)
    {
        (void)g_buffer;
        hr_reflections_default_params(&params);
        check(common->ctx, hr_reflections_create(common->ctx, (int)common->width, (int)common->height, scale, &m_pass), "hr_reflections_create");
        m_width  = common->width >> scale;
        m_height = common->height >> scale;
    }
    ~RayTracedReflections() { if (m_pass) hr_pass_destroy(m_pass); }
    void     render(void* stream, DDGI* ddgi) { check(m_common->ctx, hr_reflections_render(m_pass, &m_common->frame, &params, ddgi ? ddgi->handle() : nullptr, stream), "hr_reflections_render"); }
    hr_image output_ds() const { hr_image img {}; check(m_common->ctx, hr_pass_output(m_pass, HR_REFLECTIONS_OUT_FINAL, &img), "hr_pass_output"); return img; }
    uint32_t width() const { return m_width; }
    uint32_t height() const { return m_height; }
    RayTraceScale scale() const { return m_scale; }
    hr_pass* handle() { return m_pass; }
    hr_reflections_params params;
private:
    CommonResources* m_common;
    hr_pass*         m_pass = nullptr;
    RayTraceScale    m_scale;
    uint32_t         m_width = 0, m_height = 0;
};

// TemporalAA (src/temporal_aa.h:13-63): update() advances the Halton jitter, render() resolves the visualised pass's output.
// update_uniforms (main.cpp:937-957) multiplies the projection by translate(current_jitter): apply_jitter() does that to an hr_frame
// built without jitter (projection' = J * projection, so view_proj' = J * view_proj and the inverses gain J^-1 on the right).
class TemporalAA {
public:
    TemporalAA(CommonResources* common, GBuffer* g_buffer) : m_common(common)
    {
        (void)g_buffer;
        hr_taa_default_params(&params);
        check(common->ctx, hr_taa_create(common->ctx, (int)common->width, (int)common->height, &m_pass), "hr_taa_create");
    }
    ~TemporalAA() { if (m_pass) hr_pass_destroy(m_pass); }
    void update()
    { // temporal_aa.cpp:66-81
        if (m_enabled)
        {
            m_prev_jitter[0] = m_current_jitter[0]; m_prev_jitter[1] = m_current_jitter[1];
            hr_taa_jitter((uint32_t)m_common->num_frames, (int)m_common->width, (int)m_common->height, m_current_jitter);
        }
        else m_prev_jitter[0] = m_prev_jitter[1] = m_current_jitter[0] = m_current_jitter[1] = 0.0f;
    }
    // what update_uniforms does with the jitter (main.cpp:941-957); call after CommonResources::update_uniforms
    void apply_jitter()
    {
        hr_frame& f = m_common->frame;
        f.ubo.current_prev_jitter[0] = m_current_jitter[0]; f.ubo.current_prev_jitter[1] = m_current_jitter[1];
        f.ubo.current_prev_jitter[2] = m_prev_jitter[0];    f.ubo.current_prev_jitter[3] = m_prev_jitter[1];
        if (!m_enabled) return;
        const hrm::M4 J = hrm::translate({ m_current_jitter[0], m_current_jitter[1], 0.0f }), Ji = hrm::translate({ -m_current_jitter[0], -m_current_jitter[1], 0.0f });
        auto left  = [&](float* m) { hrm::M4 a; std::memcpy(a.m, m, 64); a = hrm::mul(J, a); std::memcpy(m, a.m, 64); };
        auto right = [&](float* m) { hrm::M4 a; std::memcpy(a.m, m, 64); a = hrm::mul(a, Ji); std::memcpy(m, a.m, 64); };
        left(f.ubo.view_proj);
        right(f.ubo.view_proj_inverse);
        right(f.ubo.proj_inverse);
        if (!m_common->first_frame) left(f.ubo.prev_view_proj); // main.cpp:955
    }
    void     render(void* stream, hr_pass* input) { if (m_enabled) check(m_common->ctx, hr_taa_render(m_pass, &m_common->frame, &params, input, stream), "hr_taa_render"); }
    hr_image output_ds() const { hr_image img {}; check(m_common->ctx, hr_pass_output(m_pass, 100, &img), "hr_pass_output"); return img; }
    bool     enabled() const { return m_enabled; }
    void     set_enabled(bool e) { if (e && !m_enabled) hr_pass_reset_history(m_pass); m_enabled = e; } // gui(): enabling sets m_reset (temporal_aa.cpp:181-185)
    const float* current_jitter() const { return m_current_jitter; }
    const float* prev_jitter() const { return m_prev_jitter; }
    hr_pass* handle() { return m_pass; }
    hr_taa_params params;
private:
    CommonResources* m_common;
    hr_pass*         m_pass = nullptr;
    bool             m_enabled = true;
    float            m_current_jitter[2] = { 0.0f, 0.0f }, m_prev_jitter[2] = { 0.0f, 0.0f };
};

// ToneMap (src/tone_map.h): render(cmd_buf, temporal_aa, deferred, ...) picks the TAA output when TAA is enabled, else the visualised pass
class ToneMap {
public:
    ToneMap(CommonResources* common) : m_common(common)
    {
        hr_tonemap_default_params(&params);
        check(common->ctx, hr_tonemap_create(common->ctx, (int)common->width, (int)common->height, &m_pass), "hr_tonemap_create");
    }
    ~ToneMap() { if (m_pass) hr_pass_destroy(m_pass); }
    void     render(void* stream, TemporalAA* temporal_aa, hr_pass* visualised)
    { // tone_map.cpp:106-125
        hr_pass* in = temporal_aa && temporal_aa->enabled() ? temporal_aa->handle() : visualised;
        check(m_common->ctx, hr_tonemap_render(m_pass, &params, in, stream), "hr_tonemap_render");
    }
    hr_image output() const { hr_image img {}; check(m_common->ctx, hr_pass_output(m_pass, 100, &img), "hr_pass_output"); return img; }
    hr_tonemap_params params;
private:
    CommonResources* m_common;
    hr_pass*         m_pass = nullptr;
};

// GroundTruthPathTracer (src/ground_truth_path_tracer.h:9-50): render(cmd_buf); restart_accumulation(); output_ds()
class GroundTruthPathTracer {
public:
    GroundTruthPathTracer(CommonResources* common) : m_common(common)
    {
        hr_path_tracer_default_params(&params);
        check(common->ctx, hr_path_tracer_create(common->ctx, (int)common->width, (int)common->height, &m_pass), "hr_path_tracer_create");
    }
    ~GroundTruthPathTracer() { if (m_pass) hr_pass_destroy(m_pass); }
    void     render(void* stream) { check(m_common->ctx, hr_path_tracer_render(m_pass, &m_common->frame, &params, stream), "hr_path_tracer_render"); }
    void     restart_accumulation() { hr_pass_reset_history(m_pass); } // ground_truth_path_tracer.h:17
    hr_image output_ds() const { hr_image img {}; check(m_common->ctx, hr_pass_output(m_pass, HR_PATH_TRACER_OUT_FINAL, &img), "hr_pass_output"); return img; }
    hr_pass* handle() { return m_pass; }
    // params.trace_indirect = 1 traces the indirect bounces up to params.max_ray_bounces path vertices; 0 (the default) renders the
    // reference as written, direct light plus one sky sample (hr_path_tracer_params)
    hr_path_tracer_params params;
private:
    CommonResources* m_common;
    hr_pass*         m_pass = nullptr;
};

} // namespace hr
