// oracle/orc_shading.h — TEST INFRASTRUCTURE ONLY (CPU oracle). Never linked into the product library.
//
// Hit shading shared by the reflections and DDGI ray-trace shaders, and the DDGI probe-grid sampling:
//   scene_descriptor_set.glsl:102-229 (fetch_triangle / interpolated_vertex / transform_vertex / material fetches)
//   brdf.glsl:36-142, lighting.glsl:117-196 (direct_lighting variants), gi/gi_common.glsl:10-320, random.glsl:17-56
// Geometry-deciding arithmetic (hit point, shading normal, shadow-ray origin / direction, probe-ray directions) follows
// the deterministic fp32 rules of orc_math.h because it feeds binary visibility decisions; BRDF / irradiance maths is
// ordinary fp32 (tolerance-checked).  Parity unpinned (no reference tests or golden vectors exist).
#pragma once
#include "orc_glsl.h"
#include "orc_scene.h"

namespace orc {

// ---- random.glsl:17-56 (xoroshiro64*, Wang hash) ------------------------------------------------------------------
struct RNG { uint32_t sx, sy; };
inline uint32_t rng_rotl(uint32_t x, uint32_t k) { return (x << k) | (x >> (32 - k)); }
inline uint32_t rng_next(RNG& r)
{
    uint32_t result = r.sx * orc_const::RNG_STAR_MULTIPLIER;
    r.sy ^= r.sx;
    r.sx = rng_rotl(r.sx, orc_const::RNG_ROTL_A) ^ r.sy ^ (r.sy << orc_const::RNG_SHIFT_B);
    r.sy = rng_rotl(r.sy, orc_const::RNG_ROTL_C);
    return result;
}
inline uint32_t rng_hash(uint32_t seed)
{
    seed = (seed ^ orc_const::RNG_HASH_XOR0) ^ (seed >> orc_const::RNG_HASH_SHR0);
    seed *= orc_const::RNG_HASH_MUL0;
    seed = seed ^ (seed >> orc_const::RNG_HASH_SHR1);
    seed *= orc_const::RNG_HASH_MUL1;
    seed = seed ^ (seed >> orc_const::RNG_HASH_SHR2);
    return seed;
}
inline RNG rng_init(uint32_t idx, uint32_t idy, uint32_t frame_index)
{
    RNG r;
    r.sx = rng_hash((idx << orc_const::RNG_SEED_SHIFT) | idy);
    r.sy = rng_hash(frame_index);
    rng_next(r);
    return r;
}
inline float next_float(RNG& r)
{
    uint32_t u = orc_const::RNG_FLOAT_ONE | (rng_next(r) >> orc_const::RNG_FLOAT_SHIFT);
    float    f;
    memcpy(&f, &u, 4);
    return f - 1.0f;
}

// ---- material textures: the bindless s_Textures[] array + Material::texture_indices0 / 1 (scene_descriptor_set.glsl:84-93) -------------------
// texture(s_Textures[i], uv) outside a fragment shader = textureLod(.., 0): base level, VK_FILTER_LINEAR, REPEAT (dw::Material::m_common_sampler,
// material.cpp:210-228).  Albedo images are VK_FORMAT_*_SRGB (material.cpp:114): texels are decoded to linear before filtering.
struct Texture2D {
    int W = 0, H = 0, C = 4; // C = 1, 2 or 4 (stb_image's channel count; RGB files arrive as RGBA, vk.cpp:163-168)
    bool srgb = false;
    std::vector<uint8_t> px;
    static float srgb_to_linear(uint8_t b)
    {
        const double c = b / 255.0;
        return (float)(c <= 0.04045 ? c / 12.92 : pow((c + 0.055) / 1.055, 2.4));
    }
    vec4 texel(int x, int y) const
    { // REPEAT
        x %= W; if (x < 0) x += W;
        y %= H; if (y < 0) y += H;
        const uint8_t* t = px.data() + (size_t)C * ((size_t)y * W + x);
        auto dec = [&](uint8_t b) { return srgb ? srgb_to_linear(b) : (float)b / 255.0f; };
        vec4 r = { dec(t[0]), 0.0f, 0.0f, 1.0f };
        if (C >= 2) r.y = dec(t[1]);
        if (C == 4) { r.z = dec(t[2]); r.w = (float)t[3] / 255.0f; }
        return r;
    }
    vec4 sample(vec2 uv) const
    {
        float x = uv.x * (float)W - 0.5f, y = uv.y * (float)H - 0.5f;
        float i0 = floorf(x), j0 = floorf(y);
        float a = x - i0, b = y - j0;
        int   i = f2i(i0), j = f2i(j0);
        // the neighbour of a saturated index (|u * W| >= 2^31) wraps to INT_MIN, as a GPU's 32-bit add does; written unsigned (no signed overflow)
        int   i1 = (int)((uint32_t)i + 1u), j1 = (int)((uint32_t)j + 1u);
        vec4  t00 = texel(i, j), t10 = texel(i1, j), t01 = texel(i, j1), t11 = texel(i1, j1);
        auto  lerp2 = [&](float p, float q, float r, float s) { return (p * (1.0f - a) + q * a) * (1.0f - b) + (r * (1.0f - a) + s * a) * b; };
        return { lerp2(t00.x, t10.x, t01.x, t11.x), lerp2(t00.y, t10.y, t01.y, t11.y), lerp2(t00.z, t10.z, t01.z, t11.z), lerp2(t00.w, t10.w, t01.w, t11.w) };
    }
};
struct MaterialTextures { int32_t albedo = -1, normal = -1, roughness = -1, roughness_channel = 0, metallic = -1, metallic_channel = 0, emissive = -1; }; // = hr_material_textures

// ---- shading inputs (what RayTracedScene binds: vertices, materials) ------------------------------------------------
struct ShadingScene {
    const Scene*       scene      = nullptr;
    std::vector<float> verts;    // n*9 world-space positions, primitive order
    std::vector<float> vnormals; // n*9 world-space unit vertex normals
    std::vector<uint32_t>    prim_mat;
    std::vector<hr_material> materials;
    // optional: textures + per-material bindings + per-primitive texture coordinates (6 floats each)
    std::vector<Texture2D>        textures;
    std::vector<MaterialTextures> bindings;
    std::vector<float>            vuv;
    std::vector<float>            vtb; // 18 per primitive: world-space unit tangents of the three corners, then bitangents (only with normal maps)
};

// fetch_albedo / fetch_roughness / fetch_metallic (scene_descriptor_set.glsl:180-218) at barycentrics (b0, b1, b2) of primitive prim;
// the constants come in through the arguments (fetch_roughness's MIN_ROUGHNESS clamp applies to both paths)
inline void fetch_material(const ShadingScene& ss, uint32_t prim, float b0, float b1, float b2, vec3& albedo, float& roughness, float& metallic)
{
    if (ss.textures.empty()) return;
    const MaterialTextures& mt = ss.bindings[ss.prim_mat[prim]];
    if (mt.albedo < 0 && mt.roughness < 0 && mt.metallic < 0) return;
    const float* q = ss.vuv.data() + 6ull * prim;
    const vec2 texcoord = { (q[0] * b0 + q[2] * b1) + q[4] * b2, (q[1] * b0 + q[3] * b1) + q[5] * b2 }; // interpolated_vertex :141
    auto comp = [](vec4 v, int c) { return c == 0 ? v.x : (c == 1 ? v.y : (c == 2 ? v.z : v.w)); };
    if (mt.albedo >= 0) { const vec4 c = ss.textures[mt.albedo].sample(texcoord); albedo = { c.x, c.y, c.z }; }
    if (mt.roughness >= 0) roughness = fmaxf(comp(ss.textures[mt.roughness].sample(texcoord), mt.roughness_channel), orc_const::MIN_ROUGHNESS);
    if (mt.metallic >= 0) metallic = comp(ss.textures[mt.metallic].sample(texcoord), mt.metallic_channel);
}

// fetch_normal / get_normal_from_map (scene_descriptor_set.glsl:164-195).  `tangent`, `bitangent`, `normal` as the caller passes them: the hit
// shaders pass vertex.tangent TWICE (reflections_ray_trace.rchit:134, gi_ray_trace.rchit:112, ground_truth_path_trace.rchit:131), the G-buffer
// pass the real frame (g_buffer.frag:100).  Deterministic arithmetic (orc_math.h): the result decides shadow rays.
inline vec3 get_normal_from_map(const Texture2D& normal_map, vec3 tangent, vec3 bitangent, vec3 normal, vec2 tex_coord)
{
    const vec3 T = normalize(tangent), B = normalize(bitangent), N = normalize(normal); // mat3 TBN
    const vec4 t = normal_map.sample(tex_coord);
    vec3 n = normalize(vec3{ t.x * 2.0f - 1.0f, t.y * 2.0f - 1.0f, t.z * 2.0f - 1.0f });
    n = normalize((T * n.x + B * n.y) + N * n.z); // TBN * n
    return n;
}
inline vec3 fetch_normal(const ShadingScene& ss, uint32_t prim, float b0, float b1, float b2, bool hit_shader, vec3 normal)
{
    if (ss.textures.empty() || ss.vtb.empty()) return normal;
    const MaterialTextures& mt = ss.bindings[ss.prim_mat[prim]];
    if (mt.normal < 0) return normal;
    const float* q = ss.vuv.data() + 6ull * prim;
    const vec2 texcoord = { (q[0] * b0 + q[2] * b1) + q[4] * b2, (q[1] * b0 + q[3] * b1) + q[5] * b2 };
    const float* t = ss.vtb.data() + 18ull * prim;
    // interpolated_vertex :143-144 (the per-vertex frames are already in world space, like the normals)
    const vec3 tangent   = normalize((vec3{ t[0], t[1], t[2] } * b0 + vec3{ t[3], t[4], t[5] } * b1) + vec3{ t[6], t[7], t[8] } * b2);
    const vec3 bitangent = normalize((vec3{ t[9], t[10], t[11] } * b0 + vec3{ t[12], t[13], t[14] } * b1) + vec3{ t[15], t[16], t[17] } * b2);
    return get_normal_from_map(ss.textures[mt.normal], tangent, hit_shader ? tangent : bitangent, normal, texcoord);
}

struct Surface { vec3 P, N, albedo; float roughness, metallic; };

// fetch_triangle + interpolated_vertex + material fetches (scene_descriptor_set.glsl:117-229), vertices pre-transformed to
// world space at scene build (hr_scene_build).  barycentrics = (1-u-v, u, v) (reflections_ray_trace.rchit:124).
inline Surface fetch_surface(const ShadingScene& ss, const Hit& h)
{
    const float* p = ss.verts.data() + 9ull * h.prim;
    const float* n = ss.vnormals.data() + 9ull * h.prim;
    const float  b0 = 1.0f - h.u - h.v, b1 = h.u, b2 = h.v;
    Surface      s;
    s.P = (vec3{ p[0], p[1], p[2] } * b0 + vec3{ p[3], p[4], p[5] } * b1) + vec3{ p[6], p[7], p[8] } * b2;
    s.N = normalize((vec3{ n[0], n[1], n[2] } * b0 + vec3{ n[3], n[4], n[5] } * b1) + vec3{ n[6], n[7], n[8] } * b2);
    const hr_material& m = ss.materials[ss.prim_mat[h.prim]];
    s.albedo    = { m.albedo[0], m.albedo[1], m.albedo[2] };
    s.roughness = fmaxf(m.roughness, orc_const::MIN_ROUGHNESS); // MIN_ROUGHNESS, scene_descriptor_set.glsl:202
    s.metallic  = m.metallic;
    fetch_material(ss, h.prim, b0, b1, b2, s.albedo, s.roughness, s.metallic);
    s.N = fetch_normal(ss, h.prim, b0, b1, b2, true, s.N); // rchit:134: N = fetch_normal(material, vertex.tangent.xyz, vertex.tangent.xyz, vertex.normal.xyz, uv)
    return s;
}

// ---- brdf.glsl:36-142 ------------------------------------------------------------------------------------------------
static constexpr float EPSILON_F = orc_const::EPSILON;
inline float D_ggx(float ndoth, float alpha)
{
    float a2 = alpha * alpha, denom = (ndoth * ndoth) * (a2 - 1.0f) + 1.0f;
    return a2 / fmaxf(EPSILON_F, M_PI_F * denom * denom);
}
inline float G1_schlick_ggx(float roughness, float ndotv)
{
    float k = ((roughness + 1.0f) * (roughness + 1.0f)) / 8.0f;
    return ndotv / fmaxf(EPSILON_F, ndotv * (1.0f - k) + k);
}
inline vec3 F_schlick(vec3 f0, float vdoth)
{
    float p = powf(1.0f - vdoth, 5.0f);
    return f0 + (vec3{ 1, 1, 1 } - f0) * p;
}
inline vec3 evaluate_uber_brdf(vec3 diffuse_color, float roughness, vec3 N, vec3 F0, vec3 Wo, vec3 Wh, vec3 Wi)
{
    float NdotL = fmaxf(dot(N, Wi), 0.0f), NdotV = fmaxf(dot(N, Wo), 0.0f), NdotH = fmaxf(dot(N, Wh), 0.0f), VdotH = fmaxf(dot(Wi, Wh), 0.0f);
    vec3  F     = F_schlick(F0, VdotH);
    float alpha = roughness * roughness;
    float spec  = D_ggx(NdotH, alpha) * (G1_schlick_ggx(roughness, NdotL) * G1_schlick_ggx(roughness, NdotV)) / fmaxf(EPSILON_F, 4.0f * NdotL * NdotV);
    vec3  specular = F * spec;
    vec3  diffuse  = diffuse_color * (1.0f / M_PI_F);
    return (vec3{ 1, 1, 1 } - F) * diffuse + specular;
}

// fetch_light_properties without SOFT_SHADOWS, with RAY_TRACING (lighting.glsl:6-111): Wi = exact light direction
inline void fetch_light_properties_hard(const hr_light& light, vec3 P, vec3 N, vec3& Li, vec3& Wi, float& t_max, float& attenuation)
{
    const int type = light_type(light);
    Li = light_color(light) * light_intensity(light);
    if (type == HR_LIGHT_DIRECTIONAL) { Wi = light_direction(light); t_max = 10000.0f; attenuation = 1.0f; }
    else
    {
        vec3  to_light = light_position(light) - P;
        float dist     = length(to_light);
        Wi             = normalize(to_light);
        t_max          = dist;
        if (type == HR_LIGHT_POINT) attenuation = 1.0f / (dist * dist);
        else
        {
            float a = smoothstepf(light_cos_theta_outer(light), light_cos_theta_inner(light), dot(Wi, light_direction(light)));
            attenuation = a / (dist * dist);
        }
    }
    attenuation *= clampf(dot(N, Wi), 0.0f, 1.0f);
}

// direct_lighting (lighting.glsl:117-196).  sky_light: SAMPLE_SKY_LIGHT variant (gi_ray_trace.rchit:9-16), rng2 = its sample.
inline vec3 direct_lighting(const Scene& scene, const hr_light& light, vec3 Wo, vec3 N, vec3 P, vec3 F0, vec3 diffuse_color, float roughness,
                            bool sky_light, vec2 rng2, vec3 sky_color)
{
    vec3 Lo         = { 0, 0, 0 };
    vec3 ray_origin = P + N * 0.1f; // :143
    {
        vec3  Li, Wi;
        float t_max, attenuation;
        fetch_light_properties_hard(light, P, N, Li, Wi, t_max, attenuation);
        vec3 Wh = normalize(Wo + Wi);
        if (attenuation > 0.0f) { count_rays(1, 1); attenuation *= scene.query_visibility(ray_origin, Wi, t_max); } // query_distance :172
        vec3 brdf = evaluate_uber_brdf(diffuse_color, roughness, N, F0, Wo, Wh, Wi);
        Lo = Lo + (brdf * attenuation) * Li;
    }
    if (sky_light)
    {
        vec3 Wi = sample_cosine_lobe(N, rng2);
        vec3 Li = sky_color; // texture(sky_cubemap, Wi): constant-colour environment
        vec3 Wh = normalize(Wo + Wi);
        count_rays(1, 1);
        Li      = Li * scene.query_visibility(ray_origin, Wi, 10000.0f);
        vec3 brdf = evaluate_uber_brdf(diffuse_color, roughness, N, F0, Wo, Wh, Wi);
        Lo = Lo + brdf * Li;
    }
    return Lo;
}

// ---- gi/gi_common.glsl ------------------------------------------------------------------------------------------------
struct DDGIUniforms { // gi_common.glsl:10-28, scalar layout = hr_ddgi_uniforms
    float   grid_start_position[3];
    float   grid_step[3];
    int32_t probe_counts[3];
    float   max_distance, depth_sharpness, hysteresis, normal_bias, energy_preservation;
    int32_t irradiance_probe_side_length, irradiance_texture_width, irradiance_texture_height;
    int32_t depth_probe_side_length, depth_texture_width, depth_texture_height;
    int32_t rays_per_probe, visibility_test;
};

inline float sign_not_zero(float k) { return k >= 0.0f ? 1.0f : -1.0f; }
inline vec2  oct_encode(vec3 v) // :110-117
{
    float l1 = fabsf(v.x) + fabsf(v.y) + fabsf(v.z);
    vec2  r  = { v.x * (1.0f / l1), v.y * (1.0f / l1) };
    if (v.z < 0.0f) r = { (1.0f - fabsf(r.y)) * sign_not_zero(r.x), (1.0f - fabsf(r.x)) * sign_not_zero(r.y) };
    return r;
}
inline vec3 oct_decode(vec2 o) // :121-127
{
    vec3 v = { o.x, o.y, 1.0f - fabsf(o.x) - fabsf(o.y) };
    if (v.z < 0.0f)
    {
        float nx = (1.0f - fabsf(v.y)) * sign_not_zero(v.x), ny = (1.0f - fabsf(v.x)) * sign_not_zero(v.y);
        v.x = nx;
        v.y = ny;
    }
    return normalize(v);
}
inline vec3 probe_location(const DDGIUniforms& d, int index) // :53-80
{
    int ix = index % d.probe_counts[0];
    int iy = (index % (d.probe_counts[0] * d.probe_counts[1])) / d.probe_counts[0];
    int iz = index / (d.probe_counts[0] * d.probe_counts[1]);
    return { d.grid_step[0] * (float)ix + d.grid_start_position[0], d.grid_step[1] * (float)iy + d.grid_start_position[1],
             d.grid_step[2] * (float)iz + d.grid_start_position[2] };
}
// :153-160
inline vec2 normalized_oct_coord(ivec2 frag_coord, int side)
{
    int pb = side + 2;
    int ox = (frag_coord.x - 2) % pb, oy = (frag_coord.y - 2) % pb;
    return { ((float)ox + 0.5f) * (2.0f / (float)side) - 1.0f, ((float)oy + 0.5f) * (2.0f / (float)side) - 1.0f };
}
// :164-184
inline vec2 texture_coord_from_direction(vec3 dir, int probe_index, int tex_w, int tex_h, int side)
{
    vec2  o  = oct_encode(normalize(dir));
    vec2  o01 = { (o.x + 1.0f) * 0.5f, (o.y + 1.0f) * 0.5f };
    float pb = (float)side + 2.0f;
    vec2  oc = { (o01.x * (float)side) / (float)tex_w, (o01.y * (float)side) / (float)tex_h };
    int   ppr = (tex_w - 2) / (int)pb;
    vec2  tl  = { (float)(probe_index % ppr) * pb + 2.0f, (float)(probe_index / ppr) * pb + 2.0f };
    return { tl.x / (float)tex_w + oc.x, tl.y / (float)tex_h + oc.y };
}
// textureLod with the BILINEAR sampler + CLAMP_TO_EDGE (ddgi.cpp:478,499), unnormalised texel centres at +0.5
inline void bilinear(const ImgH& img, vec2 uv, int nch, float* out)
{
    float x = uv.x * (float)img.W - 0.5f, y = uv.y * (float)img.H - 0.5f;
    float fx0 = floorf(x), fy0 = floorf(y);
    float fx = x - fx0, fy = y - fy0;
    int   x0 = std::min(std::max((int)fx0, 0), img.W - 1), x1 = std::min(std::max((int)fx0 + 1, 0), img.W - 1);
    int   y0 = std::min(std::max((int)fy0, 0), img.H - 1), y1 = std::min(std::max((int)fy0 + 1, 0), img.H - 1);
    for (int c = 0; c < nch; c++)
    {
        float a = img.fetch({ x0, y0 }, c), b = img.fetch({ x1, y0 }, c), cc = img.fetch({ x0, y1 }, c), d = img.fetch({ x1, y1 }, c);
        out[c] = (a * (1.0f - fx) + b * fx) * (1.0f - fy) + (cc * (1.0f - fx) + d * fx) * fy;
    }
}

// sample_irradiance, gi_common.glsl:188-320 (LINEAR_BLENDING undefined => sqrt-space blend)
inline vec3 sample_irradiance(const DDGIUniforms& d, vec3 P, vec3 N, vec3 Wo, const ImgH& irr_tex, const ImgH& depth_tex)
{
    const vec3 start = { d.grid_start_position[0], d.grid_start_position[1], d.grid_start_position[2] };
    const vec3 step  = { d.grid_step[0], d.grid_step[1], d.grid_step[2] };
    int base[3];
    {
        vec3 q = { (P.x - start.x) / step.x, (P.y - start.y) / step.y, (P.z - start.z) / step.z };
        base[0] = std::min(std::max(f2i(q.x), 0), d.probe_counts[0] - 1);
        base[1] = std::min(std::max(f2i(q.y), 0), d.probe_counts[1] - 1);
        base[2] = std::min(std::max(f2i(q.z), 0), d.probe_counts[2] - 1);
    }
    vec3 base_pos = { step.x * (float)base[0] + start.x, step.y * (float)base[1] + start.y, step.z * (float)base[2] + start.z };
    vec3 alpha    = { clampf((P.x - base_pos.x) / step.x, 0, 1), clampf((P.y - base_pos.y) / step.y, 0, 1), clampf((P.z - base_pos.z) / step.z, 0, 1) };
    vec3  sum_irr = { 0, 0, 0 };
    float sum_w   = 0.0f;
    for (int i = 0; i < 8; ++i)
    {
        int off[3] = { i & 1, (i >> 1) & 1, (i >> 2) & 1 };
        int gc[3];
        for (int a = 0; a < 3; a++) gc[a] = std::min(std::max(base[a] + off[a], 0), d.probe_counts[a] - 1);
        int  p         = gc[0] + gc[1] * d.probe_counts[0] + gc[2] * d.probe_counts[0] * d.probe_counts[1];
        vec3 probe_pos = { step.x * (float)gc[0] + start.x, step.y * (float)gc[1] + start.y, step.z * (float)gc[2] + start.z };
        vec3 probe_to_point = (P - probe_pos) + (N + Wo * 3.0f) * d.normal_bias;
        vec3 dir            = normalize(-probe_to_point);
        vec3 tri            = { off[0] ? alpha.x : 1.0f - alpha.x, off[1] ? alpha.y : 1.0f - alpha.y, off[2] ? alpha.z : 1.0f - alpha.z };
        float weight = 1.0f;
        {
            vec3  tdir = normalize(probe_pos - P);
            float t    = fmaxf(0.0001f, (dot(tdir, N) + 1.0f) * 0.5f);
            weight *= t * t + 0.2f;
        }
        if (d.visibility_test == 1)
        {
            vec2  tc   = texture_coord_from_direction(-dir, p, d.depth_texture_width, d.depth_texture_height, d.depth_probe_side_length);
            float dist = length(probe_to_point);
            float t2[2];
            bilinear(depth_tex, tc, 2, t2);
            float mean = t2[0], variance = fabsf(t2[0] * t2[0] - t2[1]);
            float dm   = fmaxf(dist - mean, 0.0f);
            float cheb = variance / (variance + dm * dm);
            cheb       = fmaxf(cheb * cheb * cheb, 0.0f);
            weight *= (dist <= mean) ? 1.0f : cheb;
        }
        weight = fmaxf(0.000001f, weight);
        vec2  tc = texture_coord_from_direction(normalize(N), p, d.irradiance_texture_width, d.irradiance_texture_height, d.irradiance_probe_side_length);
        float c3[3];
        bilinear(irr_tex, tc, 3, c3);
        if (weight < 0.2f) weight *= weight * weight * (1.0f / (0.2f * 0.2f));
        weight *= tri.x * tri.y * tri.z;
        sum_irr = sum_irr + vec3{ sqrtf(c3[0]), sqrtf(c3[1]), sqrtf(c3[2]) } * weight;
        sum_w += weight;
    }
    vec3 net = { sum_irr.x / sum_w, sum_irr.y / sum_w, sum_irr.z / sum_w };
    if (!(net.x == net.x)) net.x = 0.5f;
    if (!(net.y == net.y)) net.y = 0.5f;
    if (!(net.z == net.z)) net.z = 0.5f;
    net = net * net;
    net = net * d.energy_preservation;
    return net * (0.5f * M_PI_F);
}

// IBL specular of reflections_ray_trace.rchit:97-104 (IBL_INDIRECT_SPECULAR) / deferred.frag:167-170:
//   prefiltered_color * (F * brdf.x + brdf.y) * intensity, brdf = texture(s_BRDF, (max(N.Wo, 0), roughness)) with the bilinear
//   CLAMP_TO_EDGE sampler (vk.cpp:3453-3471, common.cpp:814-816) on the 512 x 512 RG16F LUT (brdf_preintegrate_lut.cpp:8-31).
// The prefiltered environment cubemap is a constant colour here (asset absent), so every mip returns it.
struct BrdfLut { const uint16_t* rg = nullptr; int N = 512; };
inline vec3 ibl_specular(const BrdfLut& lut, vec3 prefiltered, vec3 F, float n_dot_v, float roughness, float intensity)
{
    if (!lut.rg) return { 0, 0, 0 };
    ImgH  img { lut.N, lut.N, 2, lut.rg };
    float b[2];
    bilinear(img, { n_dot_v, roughness }, 2, b);
    return (prefiltered * (F * b[0] + vec3{ b[1], b[1], b[1] })) * intensity;
}
inline vec3 fresnel_schlick_roughness(float cos_theta, vec3 F0, float roughness) // reflections_ray_trace.rchit:80-83, deferred.frag:146-149
{
    float p5 = powf(fmaxf(1.0f - cos_theta, 0.0f), 5.0f), omr = 1.0f - roughness;
    return F0 + (vec3{ fmaxf(omr, F0.x), fmaxf(omr, F0.y), fmaxf(omr, F0.z) } - F0) * p5;
}

// fresnel_schlick_roughness + indirect diffuse term shared by both rchit shaders
// (reflections_ray_trace.rchit:80-111; gi_ray_trace.rchit:74-93)
inline vec3 indirect_diffuse(const DDGIUniforms& d, const ImgH& irr, const ImgH& dep, vec3 Wo, vec3 N, vec3 P, vec3 F0, vec3 diffuse_color, float roughness,
                             float metallic, float gi_intensity)
{
    float ct = fmaxf(dot(N, Wo), 0.0f);
    float p5 = powf(fmaxf(1.0f - ct, 0.0f), 5.0f);
    float omr = 1.0f - roughness;
    vec3  F  = F0 + (vec3{ fmaxf(omr, F0.x), fmaxf(omr, F0.y), fmaxf(omr, F0.z) } - F0) * p5;
    vec3  kD = (vec3{ 1, 1, 1 } - F) * (1.0f - metallic);
    vec3  irrv = sample_irradiance(d, P, N, Wo, irr, dep);
    return (kD * diffuse_color) * irrv * gi_intensity;
}

} // namespace orc
