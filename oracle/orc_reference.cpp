// oracle/orc_reference.cpp — TEST INFRASTRUCTURE ONLY (CPU oracle). Never linked into the product library.
//
// CPU restatement of the converged references (hybrid-rendering_b200/csrc/reference.cu, include/hr_api.h "Converged references"):
// samples k0 .. k0 + n - 1 of K1's soft-shadow ray, K7's cosine-lobe ray or K12's sample per pixel of rows [row0, row1), with
// (r0, r1) = the first two next_float of rng_init(x, y, k) (random.glsl) instead of the blue noise.  The ray functions are the
// oracle's own (orc_glsl.h, orc_scene.h, orc_shading.h); the accumulators are added to, like the device's.
#include "orc_shading.h"
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

namespace {

inline vec2 ref_random(int x, int y, uint32_t k)
{
    RNG         r  = rng_init((uint32_t)x, (uint32_t)y, k);
    const float r0 = next_float(r);
    return { r0, next_float(r) };
}

inline vec3 reflect(vec3 I, vec3 N) { return I - N * (2.0f * dot(N, I)); }

// importance_sample_ggx, reflections_ray_trace.rgen:78-105 (as orc_gi_refl.cpp states it for K12)
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

} // namespace

extern "C" {

struct orc_gbuf { int32_t W, H; const uint16_t* gb2; const uint16_t* gb3; const float* depth; };

// count[pixel] += unoccluded rays; ao = 0: K1 (p0 = bias), 1: K7 (p0 = ray length, p1 = bias)
void orc_reference_mask(void* scene, const orc_gbuf* gb, const hr_frame* f, int ao, float p0, float p1, uint32_t k0, int n, int row0, int row1, uint32_t* count)
{
    const Scene&    sc = *(const Scene*)scene;
    const GBufLevel g { gb->W, gb->H, gb->gb2, gb->gb3, gb->depth };
    const mat4      vpi = load_mat4(f->ubo.view_proj_inverse);
#pragma omp parallel for schedule(dynamic, 1)
    for (int y = row0; y < row1; y++)
        for (int x = 0; x < g.W; x++)
        {
            const ivec2 c = { x, y };
            const float depth = g.fetchd(c);
            if (depth == 1.0f) continue;
            const vec2 tc  = { ((float)x + 0.5f) / (float)g.W, ((float)y + 0.5f) / (float)g.H };
            const vec3 P   = world_position_from_depth(tc, depth, vpi);
            const vec4 gb2 = g.fetch2(c);
            const vec3 N   = octohedral_to_direction({ gb2.x, gb2.y });
            uint32_t   hits = 0, rays = 0;
            for (int s = 0; s < n; s++)
            {
                const vec2 rnd = ref_random(x, y, k0 + (uint32_t)s);
                if (ao) { rays++; hits += (uint32_t)sc.query_visibility(P + N * p1, sample_cosine_lobe(N, rnd), p0); }
                else
                {
                    vec3  Wi;
                    float t_max, attenuation;
                    fetch_light_properties_shadow(f->ubo.light, P, N, rnd, Wi, t_max, attenuation);
                    if (attenuation > 0.0f) { rays++; hits += (uint32_t)sc.query_visibility(P + N * p0, Wi, t_max); }
                }
            }
            count[(size_t)y * g.W + x] += hits;
            count_rays(0, rays);
        }
}

// acc[6 * pixel] += (sum r, g, b, sum of squares r, g, b) of K12's clamped sample; d / irr / dep / brdf_lut may be NULL
void orc_reference_reflections(void* ssp, const orc_gbuf* gb, const hr_frame* f, float bias, float trim, int sample_gi, int approximate_with_ddgi, float gi_intensity,
                               float rough_ddgi_intensity, const float* sky3, const DDGIUniforms* d, const uint16_t* irr_p, const uint16_t* dep_p,
                               const uint16_t* brdf_lut, float ibl_intensity, uint32_t k0, int n, int row0, int row1, double* acc)
{
    const ShadingScene& ss = *(const ShadingScene*)ssp;
    const GBufLevel     g { gb->W, gb->H, gb->gb2, gb->gb3, gb->depth };
    const mat4          vpi = load_mat4(f->ubo.view_proj_inverse);
    const vec3          cam = { f->ubo.cam_pos[0], f->ubo.cam_pos[1], f->ubo.cam_pos[2] };
    const vec3          sky = { sky3[0], sky3[1], sky3[2] };
    const ImgH          irr = d ? ImgH { d->irradiance_texture_width, d->irradiance_texture_height, 4, irr_p } : ImgH {};
    const ImgH          dep = d ? ImgH { d->depth_texture_width, d->depth_texture_height, 2, dep_p } : ImgH {};
    BrdfLut             lut;
    lut.rg = brdf_lut;
#pragma omp parallel for schedule(dynamic, 1)
    for (int y = row0; y < row1; y++)
        for (int x = 0; x < g.W; x++)
        {
            const ivec2 c = { x, y };
            const float depth = g.fetchd(c);
            if (depth == 1.0f) continue;
            const vec2  tc = { ((float)x + 0.5f) / (float)g.W, ((float)y + 0.5f) / (float)g.H };
            const float roughness = g.fetch3(c).x;
            const vec3  P  = world_position_from_depth(tc, depth, vpi);
            const vec4  g2 = g.fetch2(c);
            const vec3  N  = octohedral_to_direction({ g2.x, g2.y });
            const vec3  Wo = normalize(cam - P);
            const bool  mirror = roughness < orc_const::MIRROR_REFLECTIONS_ROUGHNESS_THRESHOLD;
            const bool  ddgi   = !mirror && roughness > orc_const::DDGI_REFLECTIONS_ROUGHNESS_THRESHOLD && approximate_with_ddgi == 1;
            double      s[3] = { 0, 0, 0 }, q[3] = { 0, 0, 0 };
            for (int i = 0; i < ((mirror || ddgi) ? 1 : n); i++)
            {
                vec3 color;
                if (ddgi) color = sample_irradiance(*d, P, reflect(-Wo, N), Wo, irr, dep) * rough_ddgi_intensity;
                else
                {
                    const vec3 dir = mirror ? reflect(-Wo, N) : reflect(-Wo, importance_sample_ggx(ref_random(x, y, k0 + (uint32_t)i) * trim, N, roughness));
                    Hit        h;
                    count_rays(0, 1);
                    if (ss.scene->closest(P + N * bias, dir, 0.001f, 10000.0f, h))
                    {
                        Surface s_ = fetch_surface(ss, h);
                        vec3    wo = -dir;
                        vec3    F0 = mix3(vec3{ 0.04f, 0.04f, 0.04f }, s_.albedo, s_.metallic);
                        vec3    cd = mix3(s_.albedo * (vec3{ 1, 1, 1 } - F0), vec3{ 0, 0, 0 }, s_.metallic);
                        vec3    Lo = direct_lighting(*ss.scene, f->ubo.light, wo, s_.N, s_.P, F0, cd, s_.roughness, false, { 0, 0 }, sky);
                        if (sample_gi == 1)
                        {
                            Lo = Lo + indirect_diffuse(*d, irr, dep, wo, s_.N, s_.P, F0, cd, s_.roughness, s_.metallic, gi_intensity);
                            const float ndv = fmaxf(dot(s_.N, wo), 0.0f);
                            Lo = Lo + ibl_specular(lut, sky, fresnel_schlick_roughness(ndv, F0, s_.roughness), ndv, s_.roughness, ibl_intensity);
                        }
                        color = Lo;
                    }
                    else color = sky;
                }
                const double v[3] = { fminf(color.x, 0.7f), fminf(color.y, 0.7f), fminf(color.z, 0.7f) };
                for (int ch = 0; ch < 3; ch++) { s[ch] += v[ch]; q[ch] += v[ch] * v[ch]; }
            }
            double* a = acc + 6 * ((size_t)y * g.W + x);
            const double m = (mirror || ddgi) ? (double)n : 1.0;
            for (int ch = 0; ch < 3; ch++) { a[ch] += s[ch] * m; a[3 + ch] += q[ch] * m; }
        }
}

} // extern "C"
