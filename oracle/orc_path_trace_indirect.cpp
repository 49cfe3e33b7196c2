// oracle/orc_path_trace_indirect.cpp — TEST INFRASTRUCTURE ONLY (CPU oracle). Never linked into the product library.
//
// CPU statement of the ground-truth path tracer with trace_indirect = 1 (hr_path_tracer_params, DESIGN.md §7): the bounce the reference
// comments out (src/shaders/ground_truth/ground_truth_path_trace.rchit:92-104) traced up to max_ray_bounces path vertices.  Vertex 0 and
// everything before it are orc_path_trace.cpp's mode 0 (same ray generation, same direct_lighting with RAY_THROUGHPUT, same draws), so
// max_ray_bounces = 1 renders what orc_path_trace renders, bit for bit; the accumulation (rgen:94-111) is the same too.
// The lobe choice, the sampled directions, the horizon tests and the bounce rays are geometry (orc_math.h rules), so the whole path --
// reported as a hash of its primitives -- equals the device's bit for bit; the throughput is colour (ordinary fp32, tolerance-checked).
#include "orc_shading.h"
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

namespace {

inline vec2 next_vec2(RNG& rng) { vec2 r; r.x = next_float(rng); r.y = next_float(rng); return r; } // random.glsl:64-67, left to right

// direct_lighting, lighting.glsl:117-196: SOFT_SHADOWS (rng1), RAY_THROUGHPUT (T), SAMPLE_SKY_LIGHT (rng2, sky)
vec3 direct_lighting_path(const Scene& scene, const hr_light& light, vec3 Wo, vec3 N, vec3 P, vec3 F0, vec3 diffuse_color, float roughness, vec3 T, vec2 rng1, vec2 rng2,
                          vec3 sky, uint64_t& n_rays)
{
    vec3 Lo         = { 0, 0, 0 };
    vec3 ray_origin = P + N * 0.1f; // :143
    { // punctual light
        vec3  Li = light_color(light) * light_intensity(light); // fetch_light_properties :35
        vec3  Wi;
        float t_max, attenuation;
        fetch_light_properties_shadow(light, P, N, rng1, Wi, t_max, attenuation); // the SOFT_SHADOWS branches (:37-105) + :110
        vec3 Wh = normalize(Wo + Wi);                                              // :108
        if (attenuation > 0.0f) { attenuation *= scene.query_visibility(ray_origin, Wi, t_max); n_rays++; } // query_distance :172
        vec3 brdf = evaluate_uber_brdf(diffuse_color, roughness, N, F0, Wo, Wh, Wi);
        Lo = Lo + ((T * brdf) * attenuation) * Li; // :176
    }
    { // sky light :180-192
        vec3 Wi = sample_cosine_lobe(N, rng2);
        vec3 Li = sky;
        vec3 Wh = normalize(Wo + Wi);
        Li      = Li * scene.query_visibility(ray_origin, Wi, 10000.0f);
        n_rays++;
        vec3 brdf = evaluate_uber_brdf(diffuse_color, roughness, N, F0, Wo, Wh, Wi);
        Lo = Lo + (T * brdf) * Li;
    }
    return Lo;
}

// reflections_ray_trace.rgen:78-105 (K12's sampler, as oracle/orc_gi_refl.cpp states it): the GGX half vector for (e1, e2) around N
inline vec3 importance_sample_ggx(vec2 E, vec3 N, float roughness)
{
    float a = roughness * roughness, m2 = a * a;
    float phi      = 2.0f * M_PI_F * E.x;
    float cosTheta = sqrtf((1.0f - E.y) / (1.0f + (m2 - 1.0f) * E.y));
    float sinTheta = sqrtf(1.0f - cosTheta * cosTheta);
    float sn, cs;
    det_sincos(phi, &sn, &cs);
    vec3 H  = { cs * sinTheta, sn * sinTheta, cosTheta };
    vec3 up = fabsf(N.z) < 0.999f ? vec3{ 0, 0, 1 } : vec3{ 1, 0, 0 };
    vec3 tangent   = normalize(cross(up, N));
    vec3 bitangent = cross(N, tangent);
    return normalize((tangent * H.x + bitangent * H.y) + N * H.z);
}
inline vec3 reflect(vec3 I, vec3 N) { return I - N * (2.0f * dot(N, I)); }

// path-hash end codes (HR_PATH_TRACER_OUT_PATH_HASH)
constexpr uint32_t END_MISS = 0xFFFFFFFFu, END_HORIZON = 0xFFFFFFFEu, END_MAX_BOUNCES = 0xFFFFFFFDu;
inline uint32_t fnv1a(uint32_t h, uint32_t w) { return (h ^ w) * 16777619u; }

// One sampled continuation of the path at a vertex (DESIGN.md §7): lobe choice by p_spec = 0.5 + 0.5 * clamp(metallic, 0, 1), the K12 GGX sampler
// or the cosine lobe, then the throughput factor (as-written lobe value) * N.Wi / (lobe probability * sampler pdf).  Returns false when the
// path ends below the horizon (or on a specular sample whose pdf is not positive).
inline bool sample_bounce(vec3 N, vec3 Wo, vec3 F0, vec3 diffuse_color, float roughness, float metallic, float u, vec2 e, vec3& Wi, vec3& weight)
{
    const float p_spec = 0.5f + 0.5f * clampf(metallic, 0.0f, 1.0f);
    const bool  spec   = u < p_spec;
    Wi = spec ? reflect(-Wo, importance_sample_ggx(e, N, roughness)) : sample_cosine_lobe(N, e);
    if (dot(N, Wi) <= 0.0f || dot(N, Wo) <= 0.0f) return false;
    const vec3  Wh    = normalize(Wo + Wi);
    const float NdotL = fmaxf(dot(N, Wi), 0.0f), NdotV = fmaxf(dot(N, Wo), 0.0f), NdotH = fmaxf(dot(N, Wh), 0.0f), VdotH = fmaxf(dot(Wi, Wh), 0.0f);
    const vec3  F     = F_schlick(F0, VdotH);
    if (spec)
    {
        const float a2  = (roughness * roughness) * (roughness * roughness), dd = (NdotH * NdotH) * (a2 - 1.0f) + 1.0f;
        const float pdf = p_spec * ((a2 / (M_PI_F * dd * dd)) * NdotH / (4.0f * VdotH)); // D_true(NH) NH / (4 VH), unclamped GGX
        if (!(pdf > 0.0f)) return false;
        const float s = D_ggx(NdotH, roughness * roughness) * (G1_schlick_ggx(roughness, NdotL) * G1_schlick_ggx(roughness, NdotV)) / fmaxf(EPSILON_F, 4.0f * NdotL * NdotV);
        weight = F * (s * NdotL / pdf);
    }
    else
    {
        const float pdf = (1.0f - p_spec) * (NdotL / M_PI_F);
        weight = ((vec3{ 1, 1, 1 } - F) * (diffuse_color * (1.0f / M_PI_F))) * (NdotL / pdf);
    }
    return true;
}

} // namespace

// One render of GroundTruthPathTracer with trace_indirect = 1 (one sample per pixel).  prev: the image written by the previous render (ignored
// when num_frames == 0); out: RGBA16F; out_prim (may be NULL): primitive hit by the primary ray, 0xFFFFFFFF = miss; out_hash (may be NULL):
// FNV-1a of the primitives of the path's segments, then its end code (HR_PATH_TRACER_OUT_PATH_HASH); out_secondary_rays (may be NULL): shadow
// + bounce rays traced, added to *out_secondary_rays.
extern "C" void orc_path_trace_indirect(void* shading_scene, const hr_frame* f, int W, int H, uint32_t num_frames, uint32_t max_ray_bounces,
                                        float roughness_multiplier, const float* sky3, const uint16_t* prev, uint16_t* out, uint32_t* out_prim,
                                        uint32_t* out_hash, uint64_t* out_secondary_rays)
{
    const ShadingScene& ss  = *(const ShadingScene*)shading_scene;
    const mat4 view_inverse = load_mat4(f->ubo.view_inverse), proj_inverse = load_mat4(f->ubo.proj_inverse);
    const vec3 sky = { sky3[0], sky3[1], sky3[2] };
    const float RADIANCE_CLAMP_COLOR = 1.0f; // common.glsl:19
    uint64_t n_secondary = 0;
#pragma omp parallel for schedule(dynamic, 2) reduction(+ : n_secondary)
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++)
        {
            // rgen:56-75
            vec3 L = { 0, 0, 0 }, T = { 1, 1, 1 };
            uint32_t depth = 0;
            RNG  rng = rng_init((uint32_t)x, (uint32_t)y, num_frames);
            const vec2 pixel_coord = { (float)x + 0.5f, (float)y + 0.5f };
            const vec2 jitter = next_vec2(rng); // vec2(next_float, next_float): arguments evaluate left to right
            const vec2 jittered_coord = pixel_coord + jitter;
            const vec2 tex_coord = { jittered_coord.x / (float)W, jittered_coord.y / (float)H };
            const vec2 ndc = { tex_coord.x * 2.0f - 1.0f, tex_coord.y * 2.0f - 1.0f };
            const vec4 origin = mul(view_inverse, vec4{ 0.0f, 0.0f, 0.0f, 1.0f });
            const vec4 target = mul(proj_inverse, vec4{ ndc.x, ndc.y, 1.0f, 1.0f });
            const vec3 tn = normalize(vec3{ target.x, target.y, target.z });
            const vec4 direction = mul(view_inverse, vec4{ tn.x, tn.y, tn.z, 0.0f });
            const vec3 o = { origin.x, origin.y, origin.z }, d = { direction.x, direction.y, direction.z };
            Hit h;
            uint32_t prim = 0xFFFFFFFFu, hash = 2166136261u, end = END_MISS;
            if (ss.scene->closest(o, d, 0.001f, 10000.0f, h))
            { // rchit main :112-141
                prim = h.prim;
                vec3 ray_d = d;
                for (;; depth++)
                {
                    hash = fnv1a(hash, h.prim);
                    Surface s = fetch_surface(ss, h);
                    const float roughness = s.roughness * roughness_multiplier; // fetch_roughness (max(., MIN_ROUGHNESS)) * u_PushConstants.roughness_multiplier
                    const vec3 N = s.N, Wo = -ray_d;
                    const vec3 F0 = mix3(vec3{ 0.04f, 0.04f, 0.04f }, s.albedo, s.metallic);
                    const vec3 c_diffuse = mix3(s.albedo * (vec3{ 1, 1, 1 } - F0), vec3{ 0, 0, 0 }, s.metallic);
                    const vec2 rng1 = next_vec2(rng), rng2 = next_vec2(rng);
                    L = L + direct_lighting_path(*ss.scene, f->ubo.light, Wo, N, s.P, F0, c_diffuse, roughness, T, rng1, rng2, sky, n_secondary);
                    if (depth + 1 == max_ray_bounces) { end = END_MAX_BOUNCES; break; }
                    const float u = next_float(rng);
                    const vec2  e = next_vec2(rng);
                    vec3 Wi, weight;
                    if (!sample_bounce(N, Wo, F0, c_diffuse, roughness, s.metallic, u, e, Wi, weight)) { end = END_HORIZON; break; }
                    T = T * weight;
                    n_secondary++;
                    ray_d = Wi;
                    if (!ss.scene->closest(s.P + N * 0.1f, Wi, 0.001f, 10000.0f, h)) { end = END_MISS; break; } // rmiss adds the environment at depth 0 only
                }
            }
            else L = sky; // rmiss: depth == 0 -> L = environment sample
            if (out_hash) out_hash[(size_t)y * W + x] = fnv1a(hash, end);
            // rgen:94-111
            const vec3 clamped = { fminf(L.x, RADIANCE_CLAMP_COLOR), fminf(L.y, RADIANCE_CLAMP_COLOR), fminf(L.z, RADIANCE_CLAMP_COLOR) };
            vec3 final_color = clamped;
            if (num_frames != 0)
            {
                const uint16_t* p = prev + 4 * ((size_t)y * W + x);
                const vec3 prev_color = { h2f(p[0]), h2f(p[1]), h2f(p[2]) };
                const float n = (float)num_frames;
                final_color = { prev_color.x + (clamped.x - prev_color.x) / n, prev_color.y + (clamped.y - prev_color.y) / n, prev_color.z + (clamped.z - prev_color.z) / n };
            }
            uint16_t* q = out + 4 * ((size_t)y * W + x);
            q[0] = f2h(final_color.x); q[1] = f2h(final_color.y); q[2] = f2h(final_color.z); q[3] = f2h(1.0f);
            if (out_prim) out_prim[(size_t)y * W + x] = prim;
        }
    if (out_secondary_rays) *out_secondary_rays += n_secondary;
}
