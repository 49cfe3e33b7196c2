// oracle/orc_glsl.h — TEST INFRASTRUCTURE ONLY (CPU oracle). Never linked into the product library.
//
// One C++ function per GLSL function of the reference's shared shader includes, same names,
// each citing the file:line under /root/reference/src/shaders it restates.
// Status: parity unpinned — the reference ships no tests/golden vectors and cannot be built or
// run here (Vulkan RT + GLSL, SURVEY.md §8c); this restatement follows the shader source.
#pragma once
#include "../include/hr_api.h"
#include "orc_constants.h"
#include "orc_math.h"
#include <algorithm>
#include <atomic>
#include <vector>

namespace orc {

// ------------------------------------------------------------------------------------------------
// Image access: texelFetch with integer coords; out-of-bounds => all-zero (robust image access the
// reference silently relies on, SURVEY.md Appendix A).
// ------------------------------------------------------------------------------------------------
struct GBufLevel {
    int             W = 0, H = 0;
    const uint16_t* gb2   = nullptr; // RGBA16F: oct normal.xy | motion.xy          (g_buffer.frag:95-99)
    const uint16_t* gb3   = nullptr; // RGBA16F: roughness|curvature|mesh id|linear z (g_buffer.frag:101-108)
    const float*    depth = nullptr; // D32
    bool inside(ivec2 p) const { return p.x >= 0 && p.y >= 0 && p.x < W && p.y < H; }
    vec4 fetch2(ivec2 p) const
    {
        if (!inside(p)) return { 0, 0, 0, 0 };
        const uint16_t* t = gb2 + 4 * ((size_t)p.y * W + p.x);
        return { h2f(t[0]), h2f(t[1]), h2f(t[2]), h2f(t[3]) };
    }
    vec4 fetch3(ivec2 p) const
    {
        if (!inside(p)) return { 0, 0, 0, 0 };
        const uint16_t* t = gb3 + 4 * ((size_t)p.y * W + p.x);
        return { h2f(t[0]), h2f(t[1]), h2f(t[2]), h2f(t[3]) };
    }
    float fetchd(ivec2 p) const { return inside(p) ? depth[(size_t)p.y * W + p.x] : 0.0f; }
};

struct ImgH { // fp16 image with C channels
    int             W = 0, H = 0, C = 1;
    const uint16_t* d = nullptr;
    bool  inside(ivec2 p) const { return p.x >= 0 && p.y >= 0 && p.x < W && p.y < H; }
    float fetch(ivec2 p, int c) const { return inside(p) ? h2f(d[C * ((size_t)p.y * W + p.x) + c]) : 0.0f; }
};

inline mat4 load_mat4(const float* m) { mat4 r; memcpy(r.m, m, 64); return r; }

// ------------------------------------------------------------------------------------------------
// common.glsl
// ------------------------------------------------------------------------------------------------
static constexpr float M_PI_F = orc_const::M_PI_REF; // common.glsl:16

// common.glsl:143-146
inline float luminance(vec3 rgb) { return fmaxf(dot(rgb, vec3{ 0.299f, 0.587f, 0.114f }), 0.0001f); }

// common.glsl:150-156
inline vec3 octohedral_to_direction(vec2 e)
{
    vec3 v = { e.x, e.y, 1.0f - fabsf(e.x) - fabsf(e.y) };
    if (v.z < 0.0f)
    {
        float nx = (1.0f - fabsf(v.y)) * (stepf(0.0f, v.x) * 2.0f - 1.0f);
        float ny = (1.0f - fabsf(v.x)) * (stepf(0.0f, v.y) * 2.0f - 1.0f);
        v.x = nx;
        v.y = ny;
    }
    return normalize(v);
}

// common.glsl:160-165
inline float gaussian_weight(float offset, float deviation)
{
    float weight = 1.0f / sqrtf(2.0f * M_PI_F * deviation * deviation);
    weight *= expf(-(offset * offset) / (2.0f * deviation * deviation));
    return weight;
}

// common.glsl:169-184
inline vec3 world_position_from_depth(vec2 tex_coords, float ndc_depth, const mat4& view_proj_inverse)
{
    vec2 screen_pos = { tex_coords.x * 2.0f - 1.0f, tex_coords.y * 2.0f - 1.0f };
    vec4 ndc_pos    = { screen_pos.x, screen_pos.y, ndc_depth, 1.0f };
    vec4 world_pos  = mul(view_proj_inverse, ndc_pos);
    return { world_pos.x / world_pos.w, world_pos.y / world_pos.w, world_pos.z / world_pos.w };
}

// common.glsl:188-191
inline float linear_eye_depth(float z, const float* z_buffer_params) { return 1.0f / (z_buffer_params[2] * z + z_buffer_params[3]); }

// common.glsl:87-139 light accessors
inline vec3  light_direction(const hr_light& l) { return { l.data0[0], l.data0[1], l.data0[2] }; }
inline vec3  light_color(const hr_light& l) { return { l.data2[0], l.data2[1], l.data2[2] }; }
inline float light_intensity(const hr_light& l) { return l.data0[3]; }
inline float light_radius(const hr_light& l) { return l.data1[3]; }
inline vec3  light_position(const hr_light& l) { return { l.data1[0], l.data1[1], l.data1[2] }; }
inline int   light_type(const hr_light& l) { return (int)l.data3[0]; }
inline float light_cos_theta_outer(const hr_light& l) { return l.data3[1]; }
inline float light_cos_theta_inner(const hr_light& l) { return l.data3[2]; }

// ------------------------------------------------------------------------------------------------
// bnd_sampler.glsl:4-24 — tables treated as raw bytes (UNORM*256 clamp is the identity, SURVEY A.1)
// ------------------------------------------------------------------------------------------------
struct BlueNoise {
    const uint8_t* sobol;     // 256 x RGBA8
    const uint8_t* scr_rank;  // 128 x 128 x RGBA8
};
// sample_index is unsigned (DESIGN.md §7): callers pass num_frames * spp + s in uint32 arithmetic, so every hr_frame::num_frames
// maps to (num_frames * spp + s) mod 256.  The shader's `% 256` on a signed int would be negative for indices >= 2^31.
inline float sample_blue_noise(ivec2 coord, uint32_t sample_index, int sample_dimension, const BlueNoise& bn)
{
    coord.x          = coord.x % 128;
    coord.y          = coord.y % 128;
    sample_index     = sample_index & 255u;
    sample_dimension = sample_dimension % 4;
    const uint8_t* sr = bn.scr_rank + 4 * (coord.y * 128 + coord.x);
    int ranked_sample_index = (int)sample_index ^ (int)sr[2];
    int value               = (int)bn.sobol[4 * ranked_sample_index + sample_dimension];
    value                   = value ^ (int)sr[sample_dimension % 2];
    return (0.5f + (float)value) / 256.0f;
}

// ------------------------------------------------------------------------------------------------
// lighting.glsl:6-111 fetch_light_properties, variant SOFT_SHADOWS + SHADOW_RAY_ONLY + RAY_TRACING
// (shadows_ray_trace.comp:8-15).  Mask chain => deterministic arithmetic (orc_math.h).
// ------------------------------------------------------------------------------------------------
inline vec3 soft_shadow_dir(vec3 light_dir, float radius, vec2 rng)
{
    vec3  light_tangent   = normalize(cross(light_dir, vec3{ 0.0f, 1.0f, 0.0f })); // :40
    vec3  light_bitangent = normalize(cross(light_tangent, light_dir));             // :41
    float point_radius    = radius * sqrtf(rng.x);                                  // :44
    float point_angle     = rng.y * 2.0f * M_PI_F;                                  // :45
    float sn, cs;
    det_sincos(point_angle, &sn, &cs);
    vec2 disk_point = { point_radius * cs, point_radius * sn };                     // :46
    return normalize((light_dir + light_tangent * disk_point.x) + light_bitangent * disk_point.y); // :47
}

inline float smoothstepf(float e0, float e1, float x)
{
    float t = clampf((x - e0) / (e1 - e0), 0.0f, 1.0f);
    return t * t * (3.0f - 2.0f * t);
}

inline void fetch_light_properties_shadow(const hr_light& light, vec3 P, vec3 N, vec2 rng, vec3& Wi, float& t_max, float& attenuation)
{
    const int type = light_type(light);
    if (type == HR_LIGHT_DIRECTIONAL)
    {
        Wi          = soft_shadow_dir(light_direction(light), light_radius(light), rng);
        t_max       = 10000.0f; // :52
        attenuation = 1.0f;
    }
    else if (type == HR_LIGHT_POINT)
    {
        vec3  to_light       = light_position(light) - P;
        vec3  light_dir      = normalize(to_light);
        float light_distance = length(to_light);
        Wi                   = soft_shadow_dir(light_dir, light_radius(light) / light_distance, rng); // :67-71
        t_max                = light_distance;
        attenuation          = 1.0f / (light_distance * light_distance);
    }
    else
    {
        vec3  to_light       = light_position(light) - P;
        vec3  light_dir      = normalize(to_light);
        float light_distance = length(to_light);
        Wi                   = soft_shadow_dir(light_dir, light_radius(light) / light_distance, rng);
        t_max                = light_distance;
        float angle_attenuation = dot(Wi, light_direction(light));                                                        // :102
        angle_attenuation       = smoothstepf(light_cos_theta_outer(light), light_cos_theta_inner(light), angle_attenuation); // :103
        attenuation             = angle_attenuation / (light_distance * light_distance);
    }
    attenuation *= clampf(dot(N, Wi), 0.0f, 1.0f); // :110
}

// ------------------------------------------------------------------------------------------------
// brdf.glsl:8-32
// ------------------------------------------------------------------------------------------------
struct mat3 { vec3 x, y, z; }; // columns
inline mat3 make_rotation_matrix(vec3 z)
{
    const vec3 ref = fabsf(dot(z, vec3{ 0, 1, 0 })) > 0.99f ? vec3{ 0, 0, 1 } : vec3{ 0, 1, 0 };
    const vec3 x   = normalize(cross(ref, z));
    const vec3 y   = cross(z, x);
    return { x, y, z };
}
inline vec3 mul(const mat3& M, vec3 t) { return (M.x * t.x + M.y * t.y) + M.z * t.z; }

inline vec3 sample_cosine_lobe(vec3 n, vec2 r)
{
    vec2        rs        = { fmaxf(0.00001f, r.x), fmaxf(0.00001f, r.y) };
    const float phi       = 2.0f * M_PI_F * rs.y;
    const float cos_theta = sqrtf(rs.x);
    const float sin_theta = sqrtf(1.0f - rs.x);
    float       sn, cs;
    det_sincos(phi, &sn, &cs);
    vec3 t = { sin_theta * cs, sin_theta * sn, cos_theta };
    return normalize(mul(make_rotation_matrix(n), t));
}

// ------------------------------------------------------------------------------------------------
// edge_stopping.glsl:10-62
// ------------------------------------------------------------------------------------------------
inline float normal_edge_stopping_weight(vec3 cn, vec3 sn, float power) { return powf(clampf(dot(cn, sn), 0.0f, 1.0f), power); }
inline float depth_edge_stopping_weight(float cd, float sd, float phi) { return expf(-fabsf(cd - sd) / phi); }
inline float luma_edge_stopping_weight(float cl, float sl, float phi) { return fabsf(cl - sl) / phi; }
// use_luma = USE_EDGE_STOPPING_LUMA_WEIGHT defined; normal weight is defined at every call site on this path.
inline float compute_edge_stopping_weight(float center_depth, float sample_depth, float phi_z, vec3 center_normal, vec3 sample_normal,
                                          float phi_normal, bool use_luma, float center_luma, float sample_luma, float phi_luma)
{
    const float wZ      = depth_edge_stopping_weight(center_depth, sample_depth, phi_z);
    const float wNormal = normal_edge_stopping_weight(center_normal, sample_normal, phi_normal);
    const float wL      = use_luma ? luma_edge_stopping_weight(center_luma, sample_luma, phi_luma) : 1.0f; // :53-59
    return expf(0.0f - fmaxf(wL, 0.0f) - fmaxf(wZ, 0.0f)) * wNormal;                                       // :59
}

// ------------------------------------------------------------------------------------------------
// reprojection.glsl
// ------------------------------------------------------------------------------------------------
static constexpr float NORMAL_DISTANCE = orc_const::NORMAL_DISTANCE; // :6
static constexpr float PLANE_DISTANCE  = orc_const::PLANE_DISTANCE; // :7

inline bool plane_distance_disocclusion_check(vec3 current_pos, vec3 history_pos, vec3 current_normal) // :11-17
{
    return fabsf(dot(current_pos - history_pos, current_normal)) > PLANE_DISTANCE;
}
inline bool out_of_frame_disocclusion_check(ivec2 c, ivec2 dim) { return c.x < 0 || c.y < 0 || c.x > dim.x - 1 || c.y > dim.y - 1; } // :21-28
inline bool mesh_id_disocclusion_check(float a, float b) { return !(a == b); }                                                       // :32-38
inline bool normals_disocclusion_check(vec3 cn, vec3 hn)                                                                              // :42-48
{
    float d = fabsf(dot(cn, hn));
    return !(d * d > NORMAL_DISTANCE); // pow(x, 2)
}
inline bool is_reprojection_valid(ivec2 coord, vec3 current_pos, vec3 history_pos, vec3 current_normal, vec3 history_normal,
                                  float current_mesh_id, float history_mesh_id, ivec2 image_dim) // :52-67
{
    if (out_of_frame_disocclusion_check(coord, image_dim)) return false;
    if (mesh_id_disocclusion_check(current_mesh_id, history_mesh_id)) return false;
    if (plane_distance_disocclusion_check(current_pos, history_pos, current_normal)) return false;
    if (normals_disocclusion_check(current_normal, history_normal)) return false;
    return true;
}

// :78-97
inline vec2 virtual_point_reprojection(ivec2 current_coord, ivec2 size, float depth, float ray_length, vec3 cam_pos,
                                       const mat4& view_proj_inverse, const mat4& prev_view_proj)
{
    const vec2 tex_coord  = { (float)current_coord.x / (float)size.x, (float)current_coord.y / (float)size.y };
    vec3       ray_origin = world_position_from_depth(tex_coord, depth, view_proj_inverse);
    vec3       camera_ray = ray_origin - cam_pos;
    float      camera_ray_length = length(camera_ray);
    camera_ray                   = normalize(camera_ray);
    vec3 parallax_hit_point      = cam_pos + camera_ray * (camera_ray_length + ray_length);
    vec4 rp                      = mul(prev_view_proj, vec4{ parallax_hit_point.x, parallax_hit_point.y, parallax_hit_point.z, 1.0f });
    rp.x /= rp.w;
    rp.y /= rp.w;
    return { (rp.x * 0.5f + 0.5f) * (float)size.x, (rp.y * 0.5f + 0.5f) * (float)size.y };
}

// :101-111
inline vec2 compute_history_coord(ivec2 current_coord, ivec2 size, float depth, vec2 motion, float curvature, float ray_length,
                                  vec3 cam_pos, const mat4& view_proj_inverse, const mat4& prev_view_proj)
{
    vec2 history_coord = { (float)current_coord.x + motion.x * (float)size.x, (float)current_coord.y + motion.y * (float)size.y }; // :71-74
    if (ray_length > 0.0f && curvature == 0.0f)
        history_coord = virtual_point_reprojection(current_coord, size, depth, ray_length, cam_pos, view_proj_inverse, prev_view_proj);
    return history_coord;
}

// reproject(), reprojection.glsl:115-328.  NC = number of history colour channels (1 or 3).
// moments: REPROJECTION_MOMENTS (history length in .b of the moments image); else separate length image.
struct ReprojectIn {
    ivec2     frag_coord;
    float     depth;
    const GBufLevel* cur;
    const GBufLevel* prev;
    ImgH      history_output;  // NC channels used from it
    ImgH      history_moments; // RGBA16F (moments variant) or R16F history length
    bool      moments;
    bool      reflections;
    vec3      cam_pos;
    mat4      view_proj_inverse;
    mat4      prev_view_proj;
    float     ray_length;
};
struct ReprojectOut {
    float history_color[3] = { 0, 0, 0 };
    float history_moments[2] = { 0, 0 };
    float history_length = 0;
};

// Optional per-pixel record of the branches reproject() takes (tests only, orc_set_reproject_codes): one byte per pass pixel, the
// ORC_RP_* bits OR-ed in.  Recording reads nothing the outputs depend on and writes nothing else.
enum {
    ORC_RP_REACHED  = 1,   // reproject() ran for the pixel (it has geometry)
    ORC_RP_OUT      = 2,   // history_coord out of frame
    ORC_RP_TRUNC    = 4,   // a history_coord_floor component in (-1, 0): ivec2() truncates it to 0 where floor gives -1
    ORC_RP_ALL      = 8,   // bilinear, all four taps valid
    ORC_RP_SOME     = 16,  // bilinear, one to three taps valid, sumw >= 0.01
    ORC_RP_SUMW     = 32,  // some tap valid but sumw < 0.01: sent to the 3x3 fallback
    ORC_RP_FALLBACK = 64,  // the 3x3 fallback found a valid texel
    ORC_RP_VIRTUAL  = 128  // reflections: virtual-point reprojection (else the motion vector); invalid = REACHED without ALL/SOME/FALLBACK
};
inline uint8_t*& reproject_codes() { static uint8_t* codes = nullptr; return codes; }

// Rays the trace stages cast (tests only, orc_take_ray_counts): [0] primary, [1] secondary, the kinds of hr_pass_stats — K1 a ray
// per sample whose light attenuation is > 0, K7 a ray per sample on geometry, K12 a reflection ray per traced sample (primary) and
// direct_lighting's shadow / sky rays at its hits (secondary), K18 a ray per probe ray (primary) and its hits' direct_lighting rays.
inline std::atomic<uint64_t>* ray_counts() { static std::atomic<uint64_t> c[2]; return c; }
inline void count_rays(int kind, uint64_t n) { if (n) ray_counts()[kind].fetch_add(n, std::memory_order_relaxed); }

template <int NC>
inline bool reproject(const ReprojectIn& in, ReprojectOut& out)
{
    const ivec2 frag_coord = in.frag_coord;
    const vec2  image_dim  = { (float)in.history_output.W, (float)in.history_output.H }; // :147
    const ivec2 idim       = { in.history_output.W, in.history_output.H };
    const vec2  pixel_center = { (float)frag_coord.x + 0.5f, (float)frag_coord.y + 0.5f };
    const vec2  tex_coord    = { pixel_center.x / image_dim.x, pixel_center.y / image_dim.y };

    const vec4 center_g_buffer_2 = in.cur->fetch2(frag_coord);
    const vec4 center_g_buffer_3 = in.cur->fetch3(frag_coord);

    const vec2  current_motion  = { center_g_buffer_2.z, center_g_buffer_2.w };
    const vec3  current_normal  = octohedral_to_direction({ center_g_buffer_2.x, center_g_buffer_2.y });
    const float current_mesh_id = center_g_buffer_3.z;
    const vec3  current_pos     = world_position_from_depth(tex_coord, in.depth, in.view_proj_inverse);

    ivec2 history_coord;
    vec2  history_coord_floor;
    const vec2 history_tex_coord = { tex_coord.x + current_motion.x, tex_coord.y + current_motion.y };
    if (in.reflections)
    {
        const float curvature         = center_g_buffer_3.y;
        const vec2  reprojected_coord = compute_history_coord(frag_coord, idim, in.depth, current_motion, curvature, in.ray_length,
                                                              in.cam_pos, in.view_proj_inverse, in.prev_view_proj); // :162-170
        history_coord       = { f2i(reprojected_coord.x), f2i(reprojected_coord.y) };                                // :171
        history_coord_floor = reprojected_coord;                                                                    // :172
    }
    else
    {
        history_coord       = { f2i((float)frag_coord.x + current_motion.x * image_dim.x + 0.5f),
                                f2i((float)frag_coord.y + current_motion.y * image_dim.y + 0.5f) };     // :175
        history_coord_floor = { (float)frag_coord.x + current_motion.x * image_dim.x,
                                (float)frag_coord.y + current_motion.y * image_dim.y };                  // :176
    }

    float hc[3] = { 0, 0, 0 };
    float hm[2] = { 0, 0 };
    uint8_t code = ORC_RP_REACHED;
    if (out_of_frame_disocclusion_check(history_coord, idim)) code |= ORC_RP_OUT;
    if ((history_coord_floor.x > -1.0f && history_coord_floor.x < 0.0f) || (history_coord_floor.y > -1.0f && history_coord_floor.y < 0.0f)) code |= ORC_RP_TRUNC;
    if (in.reflections && in.ray_length > 0.0f && center_g_buffer_3.y == 0.0f) code |= ORC_RP_VIRTUAL;

    bool        v[4];
    const ivec2 offset[4] = { { 0, 0 }, { 1, 0 }, { 0, 1 }, { 1, 1 } };
    const ivec2 base      = { f2i(history_coord_floor.x), f2i(history_coord_floor.y) }; // ivec2() truncates toward zero

    bool valid = false;
    for (int s = 0; s < 4; s++)
    {
        ivec2 loc               = { base.x + offset[s].x, base.y + offset[s].y };
        vec4  sample_g_buffer_2 = in.prev->fetch2(loc);
        vec4  sample_g_buffer_3 = in.prev->fetch3(loc);
        float sample_depth      = in.prev->fetchd(loc);
        vec3  history_normal    = octohedral_to_direction({ sample_g_buffer_2.x, sample_g_buffer_2.y });
        float history_mesh_id   = sample_g_buffer_3.z;
        vec3  history_pos       = world_position_from_depth(history_tex_coord, sample_depth, in.view_proj_inverse); // :204
        v[s] = is_reprojection_valid(history_coord, current_pos, history_pos, current_normal, history_normal, current_mesh_id, history_mesh_id, idim);
        valid = valid || v[s];
    }

    if (valid)
    {
        float sumw = 0;
        float x    = fractf(history_coord_floor.x);
        float y    = fractf(history_coord_floor.y);
        float w[4] = { (1 - x) * (1 - y), x * (1 - y), (1 - x) * y, x * y };
        for (int c = 0; c < 3; c++) hc[c] = 0;
        hm[0] = hm[1] = 0;
        for (int s = 0; s < 4; s++)
        {
            ivec2 loc = { base.x + offset[s].x, base.y + offset[s].y };
            if (v[s])
            {
                for (int c = 0; c < NC; c++) hc[c] += w[s] * in.history_output.fetch(loc, c);
                if (in.moments)
                {
                    hm[0] += w[s] * in.history_moments.fetch(loc, 0);
                    hm[1] += w[s] * in.history_moments.fetch(loc, 1);
                }
                sumw += w[s];
            }
        }
        valid = (sumw >= 0.01f); // :252
        code |= !valid ? ORC_RP_SUMW : (v[0] && v[1] && v[2] && v[3]) ? ORC_RP_ALL : ORC_RP_SOME;
        for (int c = 0; c < NC; c++) hc[c] = valid ? hc[c] / sumw : 0.0f;
        if (in.moments)
        {
            hm[0] = valid ? hm[0] / sumw : 0.0f;
            hm[1] = valid ? hm[1] / sumw : 0.0f;
        }
    }
    if (!valid) // :262-304
    {
        float cnt = 0.0f;
        for (int yy = -1; yy <= 1; yy++)
            for (int xx = -1; xx <= 1; xx++)
            {
                ivec2 p                 = { history_coord.x + xx, history_coord.y + yy };
                vec4  sample_g_buffer_2 = in.prev->fetch2(p);
                vec4  sample_g_buffer_3 = in.prev->fetch3(p);
                float sample_depth      = in.prev->fetchd(p);
                vec3  history_normal    = octohedral_to_direction({ sample_g_buffer_2.x, sample_g_buffer_2.y });
                float history_mesh_id   = sample_g_buffer_3.z;
                vec3  history_pos       = world_position_from_depth(history_tex_coord, sample_depth, in.view_proj_inverse);
                if (is_reprojection_valid(history_coord, current_pos, history_pos, current_normal, history_normal, current_mesh_id, history_mesh_id, idim))
                {
                    for (int c = 0; c < NC; c++) hc[c] += in.history_output.fetch(p, c);
                    if (in.moments)
                    {
                        hm[0] += in.history_moments.fetch(p, 0);
                        hm[1] += in.history_moments.fetch(p, 1);
                    }
                    cnt += 1.0f;
                }
            }
        if (cnt > 0)
        {
            valid = true;
            code |= ORC_RP_FALLBACK;
            for (int c = 0; c < NC; c++) hc[c] /= cnt;
            if (in.moments)
            {
                hm[0] /= cnt;
                hm[1] /= cnt;
            }
        }
    }

    if (valid)
    {
        out.history_length = in.moments ? in.history_moments.fetch(history_coord, 2) : in.history_moments.fetch(history_coord, 0); // :309-312
    }
    else
    {
        for (int c = 0; c < 3; c++) hc[c] = 0;
        hm[0] = hm[1] = 0;
        out.history_length = 0.0f;
    }
    for (int c = 0; c < 3; c++) out.history_color[c] = hc[c];
    out.history_moments[0] = hm[0];
    out.history_moments[1] = hm[1];
    if (uint8_t* codes = reproject_codes()) codes[(size_t)frag_coord.y * idim.x + frag_coord.x] = code;
    return valid;
}

} // namespace orc
