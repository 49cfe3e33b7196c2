// oracle/orc_gi_refl.cpp — TEST INFRASTRUCTURE ONLY (CPU oracle). Never linked into the product library.
//
// CPU restatement of the DDGI pass (K18-K21) and the reflections pass (K12, K14-K17), SURVEY.md §2.2:
//   gi/gi_ray_trace.{rgen,rchit,rmiss}, gi/gi_probe_update.glsl, gi/gi_border_update.glsl, gi/gi_sample_probe_grid.comp,
//   reflections/reflections_ray_trace.{rgen,rchit,rmiss}, reflections_denoise_reprojection.comp,
//   reflections_denoise_atrous.comp (+copy_tiles), reflections_upsample.comp.
// Environment = constant colour (sky cubemaps / IBL prefilter / BRDF LUT are release-zip assets: the IBL specular
// term of reflections_ray_trace.rchit:97-104 is therefore 0).  Parity unpinned (SURVEY.md §8c).
#include "orc_shading.h"
#include <array>
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

namespace {

inline void store4(uint16_t* img, int W, int x, int y, float a, float b, float c, float d)
{
    uint16_t* t = img + 4 * ((size_t)y * W + x);
    t[0] = f2h(a); t[1] = f2h(b); t[2] = f2h(c); t[3] = f2h(d);
}

// mat3(M) * v with M column-major mat4
inline vec3 mul_mat3(const float* M, vec3 v)
{
    return { (M[0] * v.x + M[4] * v.y) + M[8] * v.z, (M[1] * v.x + M[5] * v.y) + M[9] * v.z, (M[2] * v.x + M[6] * v.y) + M[10] * v.z };
}

// gi_ray_trace.rgen:61-72
inline vec3 spherical_fibonacci(float i, float n)
{
    const float PHI = sqrtf(5.0f) * 0.5f + 0.5f;
    const float a   = i * (PHI - 1.0f);
    float phi       = 2.0f * M_PI_F * (a - floorf(a));
    float cos_theta = 1.0f - (2.0f * i + 1.0f) * (1.0f / n);
    float sin_theta = sqrtf(clampf(1.0f - cos_theta * cos_theta, 0.0f, 1.0f));
    float sn, cs;
    det_sincos(phi, &sn, &cs);
    return { cs * sin_theta, sn * sin_theta, cos_theta };
}

inline vec3 reflect(vec3 I, vec3 N) { return I - N * (2.0f * dot(N, I)); }

// K18  gi_ray_trace.rgen:78-100 + rchit:95-128 + rmiss:24-27
void ddgi_ray_trace(const ShadingScene& ss, const DDGIUniforms& d, const hr_frame& f, const float* rot, uint32_t infinite_bounces, float gi_intensity,
                    vec3 sky, const ImgH& irr_prev, const ImgH& dep_prev, uint16_t* radiance, uint16_t* dirdepth)
{
    const int P = d.probe_counts[0] * d.probe_counts[1] * d.probe_counts[2], R = d.rays_per_probe;
#pragma omp parallel for schedule(dynamic, 4)
    for (int probe = 0; probe < P; probe++)
        for (int ray = 0; ray < R; ray++)
        {
            vec3  origin = probe_location(d, probe);
            vec3  dir    = normalize(mul_mat3(rot, spherical_fibonacci((float)ray, (float)R)));
            RNG   rng    = rng_init((uint32_t)ray, (uint32_t)probe, f.num_frames);
            vec3  L      = { 0, 0, 0 };
            float hit_distance = 10000.0f;
            Hit   h;
            count_rays(0, 1);
            if (ss.scene->closest(origin, dir, 0.001f, 10000.0f, h))
            {
                Surface s   = fetch_surface(ss, h);
                vec3    Wo  = -dir;
                vec3    F0  = mix3(vec3{ 0.04f, 0.04f, 0.04f }, s.albedo, s.metallic);
                vec3    cd  = mix3(s.albedo * (vec3{ 1, 1, 1 } - F0), vec3{ 0, 0, 0 }, s.metallic);
                vec2    r2  = { 0, 0 };
                r2.x        = next_float(rng);
                r2.y        = next_float(rng);
                L           = direct_lighting(*ss.scene, f.ubo.light, Wo, s.N, s.P, F0, cd, s.roughness, true, r2, sky);
                if (infinite_bounces == 1) L = L + indirect_diffuse(d, irr_prev, dep_prev, Wo, s.N, s.P, F0, cd, s.roughness, s.metallic, gi_intensity);
                hit_distance = 0.001f + h.t;
            }
            else L = sky;
            store4(radiance, R, ray, probe, L.x, L.y, L.z, 0.0f);
            store4(dirdepth, R, ray, probe, dir.x, dir.y, dir.z, hit_distance);
        }
}

// K19  gi_probe_update.glsl:136-184 (depth: DEPTH_PROBE_UPDATE)
void ddgi_probe_update(const DDGIUniforms& d, const uint16_t* radiance, const uint16_t* dirdepth, const ImgH& prev, int first_frame, bool depth, uint16_t* out)
{
    const int side = depth ? d.depth_probe_side_length : d.irradiance_probe_side_length;
    const int TWd  = depth ? d.depth_texture_width : d.irradiance_texture_width;
    const int C    = depth ? 2 : 4;
    const int px = d.probe_counts[0] * d.probe_counts[1], pz = d.probe_counts[2], R = d.rays_per_probe;
    const ImgH rad = { R, px * pz, 4, radiance }, dd = { R, px * pz, 4, dirdepth };
#pragma omp parallel for schedule(dynamic, 1)
    for (int wy = 0; wy < pz; wy++)
        for (int wx = 0; wx < px; wx++)
            for (int ly = 0; ly < side; ly++)
                for (int lx = 0; lx < side; lx++)
                {
                    const ivec2 cc = { wx * side + lx + 2 * wx + 2, wy * side + ly + 2 * wy + 2 }; // :138
                    const int   pb = side + 2, pps = (TWd - 2) / pb;
                    const int   rel_probe = f2i((float)cc.x / (float)pb) + pps * f2i((float)cc.y / (float)pb); // probe_id :131-137
                    float       res[3] = { 0, 0, 0 }, total_w = 0.0f;
                    const vec3  texel_dir = oct_decode(normalized_oct_coord(cc, side));
                    for (int r = 0; r < R; r++)
                    {
                        vec3  rdir = { dd.fetch({ r, rel_probe }, 0), dd.fetch({ r, rel_probe }, 1), dd.fetch({ r, rel_probe }, 2) };
                        float w;
                        if (depth)
                        {
                            float dist = fminf(d.max_distance, dd.fetch({ r, rel_probe }, 3) - 0.01f);
                            if (dist == -1.0f) dist = d.max_distance;
                            w = powf(fmaxf(0.0f, dot(texel_dir, rdir)), d.depth_sharpness);
                            if (w >= 0.00000001f) { res[0] += dist * w; res[1] += (dist * dist) * w; total_w += w; }
                        }
                        else
                        {
                            w = fmaxf(0.0f, dot(texel_dir, rdir));
                            if (w >= 0.00000001f)
                            {
                                for (int c = 0; c < 3; c++) res[c] += (rad.fetch({ r, rel_probe }, c) * 0.95f) * w;
                                total_w += w;
                            }
                        }
                    }
                    if (total_w > 0.00000001f) for (int c = 0; c < 3; c++) res[c] /= total_w;
                    if (first_frame == 0)
                        for (int c = 0; c < 3; c++) { float pv = c < C ? prev.fetch(cc, c) : 0.0f; res[c] = mixf(res[c], pv, d.hysteresis); }
                    uint16_t* t = out + C * ((size_t)cc.y * TWd + cc.x);
                    t[0] = f2h(res[0]); t[1] = f2h(res[1]);
                    if (!depth) { t[2] = f2h(res[2]); t[3] = f2h(1.0f); }
                }
}

// K20  gi_border_update.glsl:151-175.  The g_offsets tables (:35-143) follow one pattern — top / bottom rows mirror x, left /
// right columns mirror y, corners copy the opposite interior corner — generated here in the reference's order and checked
// entry by entry against the reference's two literal tables (tests/test_ref_constants.py, tests/golden/ref_constants.json).
// Entry = (src.x, src.y, dst.x, dst.y) relative to the probe's gutter origin.
static std::vector<std::array<int, 4>> border_offsets(int S)
{
    std::vector<std::array<int, 4>> t;
    for (int i = 1; i <= S; i++) t.push_back({ S + 1 - i, 1, i, 0 });
    for (int i = 1; i <= S; i++) t.push_back({ S + 1 - i, S, i, S + 1 });
    for (int i = 1; i <= S; i++) t.push_back({ 1, S + 1 - i, 0, i });
    for (int i = 1; i <= S; i++) t.push_back({ S, S + 1 - i, S + 1, i });
    t.push_back({ S, S, 0, 0 });
    t.push_back({ 1, S, S + 1, 0 });
    t.push_back({ S, 1, 0, S + 1 });
    t.push_back({ 1, 1, S + 1, S + 1 });
    return t;
}

void ddgi_border_update(const DDGIUniforms& d, bool depth, uint16_t* atlas)
{
    const int S = depth ? d.depth_probe_side_length : d.irradiance_probe_side_length;
    const int TWd = depth ? d.depth_texture_width : d.irradiance_texture_width;
    const int C = depth ? 2 : 4;
    const int px = d.probe_counts[0] * d.probe_counts[1], pz = d.probe_counts[2];
    const auto offs = border_offsets(S);
    for (int wy = 0; wy < pz; wy++)
        for (int wx = 0; wx < px; wx++)
        {
            const int bx = wx * (S + 2) + 1, by = wy * (S + 2) + 1; // :169
            for (const auto& o : offs) // copy_texel :151-161
                memcpy(atlas + C * ((size_t)(by + o[3]) * TWd + bx + o[2]), atlas + C * ((size_t)(by + o[1]) * TWd + bx + o[0]), C * 2);
        }
}

// K21  gi_sample_probe_grid.comp:75-99
void ddgi_sample_probe_grid(const GBufLevel& g, const hr_frame& f, const DDGIUniforms& d, const ImgH& irr, const ImgH& dep, float gi_intensity, uint16_t* out)
{
    const mat4 vpi = load_mat4(f.ubo.view_proj_inverse);
    const vec3 cam = { f.ubo.cam_pos[0], f.ubo.cam_pos[1], f.ubo.cam_pos[2] };
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < g.H; y++)
        for (int x = 0; x < g.W; x++)
        {
            float depth = g.fetchd({ x, y });
            if (depth == 1.0f) { store4(out, g.W, x, y, 0, 0, 0, 0); continue; }
            vec2 tc = { ((float)x + 0.5f) / (float)g.W, ((float)y + 0.5f) / (float)g.H };
            vec3 P  = world_position_from_depth(tc, depth, vpi);
            vec4 g2 = g.fetch2({ x, y });
            vec3 N  = octohedral_to_direction({ g2.x, g2.y });
            vec3 Wo = normalize(cam - P);
            vec3 ir = sample_irradiance(d, P, N, Wo, irr, dep) * gi_intensity;
            store4(out, g.W, x, y, ir.x, ir.y, ir.z, 1.0f);
        }
}

// importance_sample_ggx, reflections_ray_trace.rgen:78-105 (xyz only; the pdf is unused)
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

struct ReflParams { float bias, trim; int sample_gi, approximate_with_ddgi; float gi_intensity, rough_ddgi_intensity; float sky[3]; int spp = 1;
                    BrdfLut lut; float ibl_intensity = 0.0f; };

// K12  reflections_ray_trace.rgen:119-171 + rchit:117-150 + rmiss:26-30
void reflections_ray_trace(const ShadingScene& ss, const GBufLevel& g, const hr_frame& f, const ReflParams& rp, const BlueNoise& bn, const DDGIUniforms* d,
                           const ImgH& irr, const ImgH& dep, uint16_t* out)
{
    const mat4 vpi = load_mat4(f.ubo.view_proj_inverse);
    const vec3 cam = { f.ubo.cam_pos[0], f.ubo.cam_pos[1], f.ubo.cam_pos[2] };
    const vec3 sky = { rp.sky[0], rp.sky[1], rp.sky[2] };
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < g.H; y++)
        for (int x = 0; x < g.W; x++)
        {
            ivec2 c     = { x, y };
            float depth = g.fetchd(c);
            if (depth == 1.0f) { store4(out, g.W, x, y, 0, 0, 0, -1.0f); continue; }
            vec2  tc = { ((float)x + 0.5f) / (float)g.W, ((float)y + 0.5f) / (float)g.H };
            float roughness = g.fetch3(c).x;
            vec3  P  = world_position_from_depth(tc, depth, vpi);
            vec4  g2 = g.fetch2(c);
            vec3  N  = octohedral_to_direction({ g2.x, g2.y });
            vec3  Wo = normalize(cam - P);
            vec3  ray_origin = P + N * rp.bias;
            vec3  color = { 0, 0, 0 };
            float ray_length = -1.0f;
            bool  trace = false;
            vec3  dir   = { 0, 0, 1 };
            // spp > 1 (SURVEY.md §8d, not in the reference): the GGX lobe draws `spp` directions with sample index num_frames * spp + s
            // and averages the clamped radiance; ray_length is the first sample's (it only steers the virtual-point reprojection)
            const int  spp  = rp.spp > 1 ? rp.spp : 1;
            const bool ggx  = !(roughness < orc_const::MIRROR_REFLECTIONS_ROUGHNESS_THRESHOLD) &&
                              !(roughness > orc_const::DDGI_REFLECTIONS_ROUGHNESS_THRESHOLD && rp.approximate_with_ddgi == 1);
            const int  n_s  = ggx ? spp : 1;
            vec3       acc  = { 0, 0, 0 };
            for (int smp = 0; smp < n_s; smp++)
            {
            trace = false;
            if (roughness < orc_const::MIRROR_REFLECTIONS_ROUGHNESS_THRESHOLD) { dir = reflect(-Wo, N); trace = true; }
            else if (roughness > orc_const::DDGI_REFLECTIONS_ROUGHNESS_THRESHOLD && rp.approximate_with_ddgi == 1)
            {
                vec3 R = reflect(-Wo, N);
                color  = sample_irradiance(*d, P, R, Wo, irr, dep) * rp.rough_ddgi_intensity;
            }
            else
            {
                const uint32_t si = f.num_frames * (uint32_t)spp + (uint32_t)smp;
                vec2 Xi = { sample_blue_noise(c, si, 0, bn) * rp.trim, sample_blue_noise(c, si, 1, bn) * rp.trim };
                vec3 Wh = importance_sample_ggx(Xi, N, roughness);
                dir     = reflect(-Wo, Wh);
                trace   = true;
            }
            if (trace)
            {
                Hit h;
                count_rays(0, 1);
                if (ss.scene->closest(ray_origin, dir, 0.001f, 10000.0f, h))
                {
                    Surface s  = fetch_surface(ss, h);
                    vec3    wo = -dir;
                    vec3    F0 = mix3(vec3{ 0.04f, 0.04f, 0.04f }, s.albedo, s.metallic);
                    vec3    cd = mix3(s.albedo * (vec3{ 1, 1, 1 } - F0), vec3{ 0, 0, 0 }, s.metallic);
                    vec3    Lo = direct_lighting(*ss.scene, f.ubo.light, wo, s.N, s.P, F0, cd, s.roughness, false, { 0, 0 }, sky);
                    if (rp.sample_gi == 1)
                    { // indirect_lighting, rchit:87-111: kD * diffuse + specular
                        Lo = Lo + indirect_diffuse(*d, irr, dep, wo, s.N, s.P, F0, cd, s.roughness, s.metallic, rp.gi_intensity);
                        const float ndv = fmaxf(dot(s.N, wo), 0.0f);
                        Lo = Lo + ibl_specular(rp.lut, sky, fresnel_schlick_roughness(ndv, F0, s.roughness), ndv, s.roughness, rp.ibl_intensity);
                    }
                    color = Lo;
                    if (smp == 0) ray_length = 0.001f + h.t;
                }
                else { color = sky; if (smp == 0) ray_length = -1.0f; }
            }
            acc = acc + vec3{ fminf(color.x, 0.7f), fminf(color.y, 0.7f), fminf(color.z, 0.7f) };
            }
            color = acc * (1.0f / (float)n_s);
            store4(out, g.W, x, y, color.x, color.y, color.z, ray_length);
        }
}

// clip_aabb, reflections_denoise_reprojection.comp:111-129
inline void clip_aabb(const float* mn, const float* mx, float* h)
{
    float center[3], ext[3], cv[3], mabs = 0.0f;
    for (int c = 0; c < 3; c++)
    {
        center[c] = 0.5f * (mx[c] + mn[c]);
        ext[c]    = 0.5f * (mx[c] - mn[c]) + 0.001f;
        cv[c]     = h[c] - center[c];
        mabs      = fmaxf(mabs, fabsf(cv[c] / ext[c]));
    }
    if (mabs > 1.0f) for (int c = 0; c < 3; c++) h[c] = center[c] + cv[c] / mabs;
}

// K14  reflections_denoise_reprojection.comp:174-289.  tile_flags: 1 = denoise list, 0 = copy list.
void reflections_temporal(const GBufLevel& cur, const GBufLevel& prev, const uint16_t* input, const uint16_t* hist, const uint16_t* hist_moments,
                          const hr_frame& f, float alpha_p, float moments_alpha_p, int approximate_with_ddgi, uint16_t* out, uint16_t* moments_out, uint8_t* tile_flags)
{
    const int  W = cur.W, H = cur.H, TW = (W + 7) / 8, TH = (H + 7) / 8;
    const ImgH in = { W, H, 4, input };
    const mat4 vpi = load_mat4(f.ubo.view_proj_inverse), pvp = load_mat4(f.ubo.prev_view_proj);
    const vec3 cam = { f.ubo.cam_pos[0], f.ubo.cam_pos[1], f.ubo.cam_pos[2] };
    const float cam_delta_len = sqrtf(f.camera_delta[0] * f.camera_delta[0] + f.camera_delta[1] * f.camera_delta[1] + f.camera_delta[2] * f.camera_delta[2]);
#pragma omp parallel for schedule(dynamic, 1)
    for (int ty = 0; ty < TH; ty++)
        for (int tx = 0; tx < TW; tx++)
        {
            bool should = false;
            for (int ly = 0; ly < 8; ly++)
                for (int lx = 0; lx < 8; lx++)
                {
                    ivec2 c = { tx * 8 + lx, ty * 8 + ly };
                    if (!cur.inside(c)) continue;
                    const float depth = cur.fetchd(c), roughness = cur.fetch3(c).x;
                    float orad[4] = { 0, 0, 0, 0 }, omom[4] = { 0, 0, 0, 0 };
                    if (depth != 1.0f)
                    {
                        float color[3] = { in.fetch(c, 0), in.fetch(c, 1), in.fetch(c, 2) };
                        const float ray_length = in.fetch(c, 3);
                        ReprojectIn ri;
                        ri.frag_coord = c; ri.depth = depth; ri.cur = &cur; ri.prev = &prev;
                        ri.history_output  = { W, H, 4, hist };
                        ri.history_moments = { W, H, 4, hist_moments };
                        ri.moments = true; ri.reflections = true; ri.cam_pos = cam; ri.view_proj_inverse = vpi; ri.prev_view_proj = pvp; ri.ray_length = ray_length;
                        ReprojectOut ro;
                        bool  success = reproject<3>(ri, ro);
                        float hlen    = fminf(32.0f, success ? ro.history_length + 1.0f : 1.0f);
                        float hc[3]   = { ro.history_color[0], ro.history_color[1], ro.history_color[2] };
                        if (success)
                        { // neighborhood_standard_deviation :133-157
                            float m1[3] = { 0, 0, 0 }, m2[3] = { 0, 0, 0 };
                            for (int dx = -8; dx <= 8; dx++)
                                for (int dy = -8; dy <= 8; dy++)
                                    for (int k = 0; k < 3; k++) { float v = in.fetch({ c.x + dx, c.y + dy }, k); m1[k] += v; m2[k] += v * v; }
                            float mn[3], mx[3];
                            for (int k = 0; k < 3; k++)
                            {
                                float mean = m1[k] / 289.0f, var = (m2[k] / 289.0f) - mean * mean, sd = sqrtf(fmaxf(var, 0.0f));
                                mn[k] = mean - sd;
                                mx[k] = mean + sd;
                            }
                            clip_aabb(mn, mx, hc);
                        }
                        const float maxacc = cam_delta_len > 0.0f ? 8.0f : hlen; // compute_max_accumulated_frame :162-168
                        const float alpha  = success ? fmaxf(alpha_p, 1.0f / maxacc) : 1.0f;
                        const float alpham = success ? fmaxf(moments_alpha_p, 1.0f / maxacc) : 1.0f;
                        float lum = luminance({ color[0], color[1], color[2] });
                        float mo0 = mixf(ro.history_moments[0], lum, alpham), mo1 = mixf(ro.history_moments[1], lum * lum, alpham);
                        float variance = fmaxf(0.0f, mo1 - mo0 * mo0);
                        for (int k = 0; k < 3; k++) orad[k] = mixf(hc[k], color[k], alpha);
                        orad[3] = variance;
                        omom[0] = mo0; omom[1] = mo1; omom[2] = hlen; omom[3] = 0.0f;
                    }
                    store4(moments_out, W, c.x, c.y, omom[0], omom[1], omom[2], omom[3]);
                    store4(out, W, c.x, c.y, orad[0], orad[1], orad[2], orad[3]);
                    if (depth != 1.0f && roughness >= orc_const::MIRROR_REFLECTIONS_ROUGHNESS_THRESHOLD)
                    {
                        if (approximate_with_ddgi == 1) { if (roughness <= orc_const::DDGI_REFLECTIONS_ROUGHNESS_THRESHOLD) should = true; }
                        else should = true;
                    }
                }
            tile_flags[(size_t)ty * TW + tx] = should ? 1 : 0;
        }
}

// K15 + K16  reflections_denoise_copy_tiles.comp:35-38, reflections_denoise_atrous.comp:94-181
void reflections_atrous(const GBufLevel& g, const uint16_t* in_img, const uint8_t* tile_flags, int radius, int step_size, float phi_color, float phi_normal,
                        float sigma_depth, int approximate_with_ddgi, uint16_t* out)
{
    const int   W = g.W, H = g.H, TW = (W + 7) / 8;
    const ImgH  in = { W, H, 4, in_img };
    const float* kernel_weights = orc_const::ATROUS_KERNEL_WEIGHTS;
    const auto& vk = orc_const::ATROUS_VARIANCE_KERNEL;
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++)
        {
            ivec2 ipos = { x, y };
            float cc[4] = { in.fetch(ipos, 0), in.fetch(ipos, 1), in.fetch(ipos, 2), in.fetch(ipos, 3) };
            if (!tile_flags[(size_t)(y / 8) * TW + x / 8]) { store4(out, W, x, y, cc[0], cc[1], cc[2], cc[3]); continue; } // copy tiles
            const float center_luma = luminance({ cc[0], cc[1], cc[2] });
            float var = 0.0f;
            for (int yy = -1; yy <= 1; yy++)
                for (int xx = -1; xx <= 1; xx++) var += in.fetch({ x + xx, y + yy }, 3) * vk[abs(xx)][abs(yy)];
            vec4  c2 = g.fetch2(ipos), c3 = g.fetch3(ipos);
            vec3  current_normal = octohedral_to_direction({ c2.x, c2.y });
            float center_depth = c3.w, depth = g.fetchd(ipos), roughness = c3.x;
            if (depth == 1.0f) { store4(out, W, x, y, 0, 0, 0, 0); continue; }
            if (roughness < orc_const::MIRROR_REFLECTIONS_ROUGHNESS_THRESHOLD || (approximate_with_ddgi == 1 && roughness > orc_const::DDGI_REFLECTIONS_ROUGHNESS_THRESHOLD)) { store4(out, W, x, y, cc[0], cc[1], cc[2], cc[3]); continue; }
            const float phi_c = phi_color * sqrtf(fmaxf(0.0f, orc_const::ATROUS_EPS_VARIANCE + var));
            float sum_w = 1.0f, sc[4] = { cc[0], cc[1], cc[2], cc[3] };
            for (int yy = -radius; yy <= radius; yy++)
                for (int xx = -radius; xx <= radius; xx++)
                {
                    const ivec2 p = { x + xx * step_size, y + yy * step_size };
                    const bool  inside = p.x >= 0 && p.y >= 0 && p.x < W && p.y < H;
                    const float kernel = kernel_weights[abs(xx)] * kernel_weights[abs(yy)];
                    if (inside && (xx != 0 || yy != 0))
                    {
                        float s[4] = { in.fetch(p, 0), in.fetch(p, 1), in.fetch(p, 2), in.fetch(p, 3) };
                        const float sl = luminance({ s[0], s[1], s[2] });
                        vec4  s2 = g.fetch2(p), s3 = g.fetch3(p);
                        vec3  sn = octohedral_to_direction({ s2.x, s2.y });
                        const float w  = compute_edge_stopping_weight(center_depth, s3.w, sigma_depth, current_normal, sn, phi_normal, true, center_luma, sl, phi_c);
                        const float wc = w * kernel;
                        sum_w += wc;
                        for (int k = 0; k < 3; k++) sc[k] += wc * s[k];
                        sc[3] += (wc * wc) * s[3];
                    }
                }
            store4(out, W, x, y, sc[0] / sum_w, sc[1] / sum_w, sc[2] / sum_w, sc[3] / (sum_w * sum_w));
        }
}

inline ivec2 nearest_texel(vec2 uv, int W, int H)
{
    int x = (int)floorf(uv.x * (float)W), y = (int)floorf(uv.y * (float)H);
    return { std::min(std::max(x, 0), W - 1), std::min(std::max(y, 0), H - 1) };
}

// K17  reflections_upsample.comp:62-109
void upsample_vec4(const GBufLevel& g0, const GBufLevel& gm, const uint16_t* in_img, uint16_t* out)
{
    const int  W0 = g0.W, H0 = g0.H;
    const ImgH in = { gm.W, gm.H, 4, in_img };
    const vec2 ts = { 1.0f / (float)gm.W, 1.0f / (float)gm.H };
    const vec2 gk[4] = { { 0.0f, 1.0f }, { 1.0f, 0.0f }, { -1.0f, 0.0f }, { 0.0f, -1.0f } };
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < H0; y++)
        for (int x = 0; x < W0; x++)
        {
            ivec2 c  = { x, y };
            vec2  tc = { ((float)x + 0.5f) / (float)W0, ((float)y + 0.5f) / (float)H0 };
            float hz = g0.fetch3(c).w;
            if (hz == -1.0f) { store4(out, W0, x, y, 0, 0, 0, 0); continue; }
            vec4  h2 = g0.fetch2(c);
            vec3  hn = octohedral_to_direction({ h2.x, h2.y });
            float up[4] = { 0, 0, 0, 0 }, tw = 0.0f;
            for (int i = 0; i < 4; i++)
            {
                ivec2 ct = nearest_texel({ tc.x + gk[i].x * ts.x, tc.y + gk[i].y * ts.y }, gm.W, gm.H);
                float cz = gm.fetch3(ct).w;
                if (cz == -1.0f) continue;
                vec4  c2 = gm.fetch2(ct);
                vec3  cn = octohedral_to_direction({ c2.x, c2.y });
                float w  = compute_edge_stopping_weight(hz, cz, 1.0f, hn, cn, 32.0f, false, 0, 0, 0);
                for (int k = 0; k < 4; k++) up[k] += in.fetch(ct, k) * w;
                tw += w;
            }
            float inv = fmaxf(tw, 0.00000001f);
            store4(out, W0, x, y, up[0] / inv, up[1] / inv, up[2] / inv, up[3] / inv);
        }
}

} // namespace

// ================================================================================================
extern "C" {

struct orc_gbuf { int32_t W, H; const uint16_t* gb2; const uint16_t* gb3; const float* depth; };
static GBufLevel lvl(const orc_gbuf* g) { GBufLevel l; l.W = g->W; l.H = g->H; l.gb2 = g->gb2; l.gb3 = g->gb3; l.depth = g->depth; return l; }

void* orc_shading_create(void* scene, const float* verts9, const float* vnormals9, const uint32_t* prim_mat, size_t n_tris, const hr_material* mats, size_t n_mats)
{
    ShadingScene* s = new ShadingScene();
    s->scene = (const Scene*)scene;
    s->verts.assign(verts9, verts9 + 9 * n_tris);
    s->vnormals.assign(vnormals9, vnormals9 + 9 * n_tris);
    s->prim_mat.assign(prim_mat, prim_mat + n_tris);
    s->materials.assign(mats, mats + n_mats);
    return s;
}
void orc_shading_destroy(void* s) { delete (ShadingScene*)s; }
// hr_scene_set_textures on the oracle's scene: n_textures images (w, h, channels, srgb, data), one MaterialTextures per material,
// 6 texture coordinates per primitive; n_textures = 0 removes them
struct orc_texture { int32_t width, height, channels, srgb; const uint8_t* data; };
void orc_shading_set_textures(void* s, const orc_texture* textures, size_t n_textures, const MaterialTextures* bindings, size_t n_materials, const float* vuv6,
                              const float* vtb18)
{
    ShadingScene& ss = *(ShadingScene*)s;
    ss.textures.clear(); ss.bindings.clear(); ss.vuv.clear(); ss.vtb.clear();
    if (!n_textures) return;
    for (size_t i = 0; i < n_textures; i++)
    {
        Texture2D t;
        t.W = textures[i].width; t.H = textures[i].height; t.C = textures[i].channels; t.srgb = textures[i].srgb != 0;
        t.px.assign(textures[i].data, textures[i].data + (size_t)t.W * t.H * t.C);
        ss.textures.push_back(std::move(t));
    }
    ss.bindings.assign(bindings, bindings + n_materials);
    ss.vuv.assign(vuv6, vuv6 + 6 * ss.prim_mat.size());
    if (vtb18) ss.vtb.assign(vtb18, vtb18 + 18 * ss.prim_mat.size());
}
// fetch_surface's shading normal for n hits (unit tests): out = 3 floats each; hit_shader = the rchit call (tangent passed as bitangent)
void orc_fetch_normal(void* s, const uint32_t* prim, const float* bary_uv, size_t n, int hit_shader, float* out3)
{
    const ShadingScene& ss = *(const ShadingScene*)s;
    for (size_t i = 0; i < n; i++)
    {
        const float  u = bary_uv[2 * i], v = bary_uv[2 * i + 1], b0 = 1.0f - u - v;
        const float* nn = ss.vnormals.data() + 9ull * prim[i];
        const vec3   N = normalize((vec3{ nn[0], nn[1], nn[2] } * b0 + vec3{ nn[3], nn[4], nn[5] } * u) + vec3{ nn[6], nn[7], nn[8] } * v);
        const vec3   r = fetch_normal(ss, prim[i], b0, u, v, hit_shader != 0, N);
        out3[3 * i] = r.x; out3[3 * i + 1] = r.y; out3[3 * i + 2] = r.z;
    }
}
// fetch_surface's material part for n hits (primitive, barycentric u, v): out = albedo rgb, roughness, metallic (5 floats each)
void orc_fetch_material(void* s, const uint32_t* prim, const float* bary_uv, size_t n, float* out5)
{
    const ShadingScene& ss = *(const ShadingScene*)s;
    for (size_t i = 0; i < n; i++)
    {
        const Hit h { 0.0f, prim[i], bary_uv[2 * i], bary_uv[2 * i + 1] };
        const Surface sf = fetch_surface(ss, h);
        out5[5 * i] = sf.albedo.x; out5[5 * i + 1] = sf.albedo.y; out5[5 * i + 2] = sf.albedo.z; out5[5 * i + 3] = sf.roughness; out5[5 * i + 4] = sf.metallic;
    }
}
// texture(s_Textures[..], uv) of one image, for unit tests: out = 4 floats per uv
void orc_texture_sample(const orc_texture* t, const float* uv, size_t n, float* out4)
{
    Texture2D tx;
    tx.W = t->width; tx.H = t->height; tx.C = t->channels; tx.srgb = t->srgb != 0;
    tx.px.assign(t->data, t->data + (size_t)tx.W * tx.H * tx.C);
    for (size_t i = 0; i < n; i++)
    {
        const vec4 c = tx.sample({ uv[2 * i], uv[2 * i + 1] });
        out4[4 * i] = c.x; out4[4 * i + 1] = c.y; out4[4 * i + 2] = c.z; out4[4 * i + 3] = c.w;
    }
}

static ImgH atlas_irr(const DDGIUniforms* d, const uint16_t* p) { return { d->irradiance_texture_width, d->irradiance_texture_height, 4, p }; }
static ImgH atlas_dep(const DDGIUniforms* d, const uint16_t* p) { return { d->depth_texture_width, d->depth_texture_height, 2, p }; }

void orc_ddgi_ray_trace(void* ss, const DDGIUniforms* d, const hr_frame* f, const float* rot16, uint32_t infinite_bounces, float gi_intensity, const float* sky3,
                        const uint16_t* irr_prev, const uint16_t* dep_prev, uint16_t* radiance, uint16_t* dirdepth)
{ ddgi_ray_trace(*(ShadingScene*)ss, *d, *f, rot16, infinite_bounces, gi_intensity, { sky3[0], sky3[1], sky3[2] }, atlas_irr(d, irr_prev), atlas_dep(d, dep_prev), radiance, dirdepth); }

void orc_ddgi_probe_update(const DDGIUniforms* d, const uint16_t* radiance, const uint16_t* dirdepth, const uint16_t* prev, int first_frame, int depth, uint16_t* out)
{ ddgi_probe_update(*d, radiance, dirdepth, depth ? atlas_dep(d, prev) : atlas_irr(d, prev), first_frame, depth != 0, out); }

void orc_ddgi_border_update(const DDGIUniforms* d, int depth, uint16_t* atlas) { ddgi_border_update(*d, depth != 0, atlas); }
// the generated g_offsets table for probe side S: 4*S + 4 entries of (src.x, src.y, dst.x, dst.y); returns the entry count
int orc_border_offsets(int S, int32_t* out4)
{
    const auto t = border_offsets(S);
    if (out4) for (size_t i = 0; i < t.size(); i++) for (int k = 0; k < 4; k++) out4[4 * i + k] = t[i][k];
    return (int)t.size();
}
// named constant of orc_constants.h by name (tests compare them with the values parsed from the reference's sources)
int orc_get_constant(const char* name, double* out, int cap)
{
    namespace oc = orc_const;
    struct E { const char* n; int cnt; double v[6]; };
    const E table[] = {
        { "M_PI", 1, { oc::M_PI_REF } }, { "EPSILON", 1, { oc::EPSILON } },
        { "MIRROR_REFLECTIONS_ROUGHNESS_THRESHOLD", 1, { oc::MIRROR_REFLECTIONS_ROUGHNESS_THRESHOLD } },
        { "DDGI_REFLECTIONS_ROUGHNESS_THRESHOLD", 1, { oc::DDGI_REFLECTIONS_ROUGHNESS_THRESHOLD } },
        { "NORMAL_DISTANCE", 1, { oc::NORMAL_DISTANCE } }, { "PLANE_DISTANCE", 1, { oc::PLANE_DISTANCE } }, { "MIN_ROUGHNESS", 1, { oc::MIN_ROUGHNESS } },
        { "atrous_eps_variance", 1, { oc::ATROUS_EPS_VARIANCE } },
        { "atrous_kernel_weights", 3, { oc::ATROUS_KERNEL_WEIGHTS[0], oc::ATROUS_KERNEL_WEIGHTS[1], oc::ATROUS_KERNEL_WEIGHTS[2] } },
        { "atrous_variance_kernel", 4, { oc::ATROUS_VARIANCE_KERNEL[0][0], oc::ATROUS_VARIANCE_KERNEL[0][1], oc::ATROUS_VARIANCE_KERNEL[1][0], oc::ATROUS_VARIANCE_KERNEL[1][1] } },
        { "rng.star_multiplier", 1, { (double)oc::RNG_STAR_MULTIPLIER } }, { "rng.rotl_a", 1, { (double)oc::RNG_ROTL_A } }, { "rng.shift_b", 1, { (double)oc::RNG_SHIFT_B } },
        { "rng.rotl_c", 1, { (double)oc::RNG_ROTL_C } },
        { "rng.hash", 6, { (double)oc::RNG_HASH_XOR0, (double)oc::RNG_HASH_SHR0, (double)oc::RNG_HASH_MUL0, (double)oc::RNG_HASH_SHR1, (double)oc::RNG_HASH_MUL1, (double)oc::RNG_HASH_SHR2 } },
        { "rng.seed_shift", 1, { (double)oc::RNG_SEED_SHIFT } }, { "rng.float_bits", 2, { (double)oc::RNG_FLOAT_ONE, (double)oc::RNG_FLOAT_SHIFT } },
    };
    for (const E& e : table)
        if (!strcmp(e.n, name))
        {
            for (int i = 0; i < e.cnt && i < cap; i++) out[i] = e.v[i];
            return e.cnt;
        }
    return 0;
}

void orc_ddgi_sample_probe_grid(const orc_gbuf* g, const hr_frame* f, const DDGIUniforms* d, const uint16_t* irr, const uint16_t* dep, float gi_intensity, uint16_t* out)
{ ddgi_sample_probe_grid(lvl(g), *f, *d, atlas_irr(d, irr), atlas_dep(d, dep), gi_intensity, out); }

void orc_reflections_ray_trace(void* ss, const orc_gbuf* g, const hr_frame* f, float bias, float trim, int sample_gi, int approximate_with_ddgi, float gi_intensity,
                               float rough_ddgi_intensity, const float* sky3, const uint8_t* sobol, const uint8_t* sr, const DDGIUniforms* d, const uint16_t* irr,
                               const uint16_t* dep, uint16_t* out)
{
    ReflParams rp { bias, trim, sample_gi, approximate_with_ddgi, gi_intensity, rough_ddgi_intensity, { sky3[0], sky3[1], sky3[2] } };
    BlueNoise  bn { sobol, sr };
    ImgH       ii = d ? atlas_irr(d, irr) : ImgH {}, dd = d ? atlas_dep(d, dep) : ImgH {};
    reflections_ray_trace(*(ShadingScene*)ss, lvl(g), *f, rp, bn, d, ii, dd, out);
}

// extended form: spp > 1 and / or the IBL specular term (brdf_lut = 512 x 512 RG16F or NULL)
void orc_reflections_ray_trace_spp(void* ss, const orc_gbuf* g, const hr_frame* f, float bias, float trim, int sample_gi, int approximate_with_ddgi, float gi_intensity,
                                   float rough_ddgi_intensity, const float* sky3, int spp, const uint8_t* sobol, const uint8_t* sr, const DDGIUniforms* d,
                                   const uint16_t* irr, const uint16_t* dep, uint16_t* out, const uint16_t* brdf_lut, float ibl_intensity)
{
    ReflParams rp { bias, trim, sample_gi, approximate_with_ddgi, gi_intensity, rough_ddgi_intensity, { sky3[0], sky3[1], sky3[2] } };
    rp.spp = spp;
    rp.lut.rg = brdf_lut;
    rp.ibl_intensity = ibl_intensity;
    BlueNoise bn { sobol, sr };
    ImgH      ii = d ? atlas_irr(d, irr) : ImgH {}, dd = d ? atlas_dep(d, dep) : ImgH {};
    reflections_ray_trace(*(ShadingScene*)ss, lvl(g), *f, rp, bn, d, ii, dd, out);
}

void orc_reflections_temporal(const orc_gbuf* cur, const orc_gbuf* prev, const uint16_t* input, const uint16_t* hist, const uint16_t* hist_moments, const hr_frame* f,
                              float alpha, float moments_alpha, int approximate_with_ddgi, uint16_t* out, uint16_t* moments_out, uint8_t* tile_flags)
{ reflections_temporal(lvl(cur), lvl(prev), input, hist, hist_moments, *f, alpha, moments_alpha, approximate_with_ddgi, out, moments_out, tile_flags); }

void orc_reflections_atrous(const orc_gbuf* g, const uint16_t* in_img, const uint8_t* tile_flags, int radius, int step_size, float phi_color, float phi_normal,
                            float sigma_depth, int approximate_with_ddgi, uint16_t* out)
{ reflections_atrous(lvl(g), in_img, tile_flags, radius, step_size, phi_color, phi_normal, sigma_depth, approximate_with_ddgi, out); }

void orc_upsample_vec4(const orc_gbuf* g0, const orc_gbuf* gm, const uint16_t* in_img, uint16_t* out) { upsample_vec4(lvl(g0), lvl(gm), in_img, out); }

uint32_t orc_rng_sequence(uint32_t x, uint32_t y, uint32_t frame, float* out, int n)
{
    RNG r = rng_init(x, y, frame);
    for (int i = 0; i < n; i++) out[i] = next_float(r);
    return r.sx;
}

} // extern "C"
