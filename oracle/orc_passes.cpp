// oracle/orc_passes.cpp — TEST INFRASTRUCTURE ONLY (CPU oracle). Never linked into the product library.
//
// CPU restatement of the reference's shadows and AO pass chains (kernels K1-K11 of SURVEY.md §2.2):
// one function per GLSL entry shader, host sequencing per src/ray_traced_shadows.cpp / src/ray_traced_ao.cpp.
// Parity unpinned: the reference has no tests or golden vectors for this path (SURVEY.md §8c).
// Images are stored in the reference's VkFormats (fp16 channels, round-to-nearest-even on store).
#include "orc_glsl.h"
#include "orc_scene.h"
#include <cstdio>
#include <cstdlib>
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

namespace {

inline void store_h(uint16_t* img, int W, int C, ivec2 p, int c, float v) { img[C * ((size_t)p.y * W + p.x) + c] = f2h(v); }

// ------------------------------------------------------------------------------------------------
// K1  shadows/shadows_ray_trace.comp:89-132
// mask image: ceil(W/8) x ceil(H/4) uint32, bit (y%4)*8 + (x%8)  (= gl_LocalInvocationIndex of the 8x4 group).
// Threads outside the image contribute bit 0 (documented deviation for W%8 / H%4 != 0, DESIGN.md).
// ------------------------------------------------------------------------------------------------
void shadows_ray_trace(const Scene& scene, const GBufLevel& g, const hr_frame& f, float bias, const BlueNoise& bn, uint32_t* mask)
{
    const int   MW  = (g.W + 7) / 8, MH = (g.H + 3) / 4;
    const mat4  vpi = load_mat4(f.ubo.view_proj_inverse);
    memset(mask, 0, sizeof(uint32_t) * (size_t)MW * MH);
#pragma omp parallel for schedule(dynamic, 4)
    for (int my = 0; my < MH; my++)
        for (int mx = 0; mx < MW; mx++)
        {
            uint32_t word = 0, rays = 0;
            for (int li = 0; li < 32; li++)
            {
                ivec2 c = { mx * 8 + (li & 7), my * 4 + (li >> 3) };
                if (!g.inside(c)) continue;
                const vec2 tex_coord = { ((float)c.x + 0.5f) / (float)g.W, ((float)c.y + 0.5f) / (float)g.H };
                float      depth     = g.fetchd(c);
                uint32_t   result    = 0;
                if (depth != 1.0f)
                {
                    vec3 world_pos  = world_position_from_depth(tex_coord, depth, vpi);
                    vec4 gb2        = g.fetch2(c);
                    vec3 normal     = octohedral_to_direction({ gb2.x, gb2.y });
                    vec3 ray_origin = world_pos + normal * bias;
                    vec2 rnd        = { sample_blue_noise(c, f.num_frames, 0, bn), sample_blue_noise(c, f.num_frames, 1, bn) };
                    vec3  Wi;
                    float t_max, attenuation;
                    fetch_light_properties_shadow(f.ubo.light, world_pos, normal, rnd, Wi, t_max, attenuation);
                    if (attenuation > 0.0f) { rays++; result = (uint32_t)scene.query_visibility(ray_origin, Wi, t_max); } // query_distance
                }
                word |= result << li;
            }
            mask[(size_t)my * MW + mx] = word;
            count_rays(0, rays);
        }
}

// K7  ao/ao_ray_trace.comp:90-126
void ao_ray_trace(const Scene& scene, const GBufLevel& g, const hr_frame& f, float ray_length, float bias, const BlueNoise& bn, uint32_t* mask)
{
    const int  MW  = (g.W + 7) / 8, MH = (g.H + 3) / 4;
    const mat4 vpi = load_mat4(f.ubo.view_proj_inverse);
#pragma omp parallel for schedule(dynamic, 4)
    for (int my = 0; my < MH; my++)
        for (int mx = 0; mx < MW; mx++)
        {
            uint32_t word = 0, rays = 0;
            for (int li = 0; li < 32; li++)
            {
                ivec2 c = { mx * 8 + (li & 7), my * 4 + (li >> 3) };
                if (!g.inside(c)) continue;
                const vec2 tex_coord = { ((float)c.x + 0.5f) / (float)g.W, ((float)c.y + 0.5f) / (float)g.H };
                float      depth     = g.fetchd(c);
                uint32_t   result    = 0;
                if (depth != 1.0f)
                {
                    rays++;
                    vec3 world_pos  = world_position_from_depth(tex_coord, depth, vpi);
                    vec4 gb2        = g.fetch2(c);
                    vec3 normal     = octohedral_to_direction({ gb2.x, gb2.y });
                    vec3 ray_origin = world_pos + normal * bias;
                    vec2 rnd        = { sample_blue_noise(c, f.num_frames, 0, bn), sample_blue_noise(c, f.num_frames, 1, bn) };
                    vec3 dir        = sample_cosine_lobe(normal, rnd);
                    result          = (uint32_t)scene.query_visibility(ray_origin, dir, ray_length);
                }
                word |= result << li;
            }
            mask[(size_t)my * MW + mx] = word;
            count_rays(0, rays);
        }
}

// ------------------------------------------------------------------------------------------------
// spp > 1 (NOT in the reference; defined by SURVEY.md §8d for configs 4-5): `spp` rays per pixel with sample index
// num_frames * spp + s; the 1-bit mask cannot hold the result, the kernels emit an 8-bit image of the number of
// unoccluded rays per pixel; the temporal stage uses visibility = count / spp, everything downstream is unchanged.
// ------------------------------------------------------------------------------------------------
void ray_trace_count(const Scene& scene, const GBufLevel& g, const hr_frame& f, bool ao, float p0, float bias, int spp, const BlueNoise& bn, uint8_t* count)
{
    const mat4 vpi = load_mat4(f.ubo.view_proj_inverse);
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < g.H; y++)
        for (int x = 0; x < g.W; x++)
        {
            const ivec2 c = { x, y };
            const vec2  tex_coord = { ((float)c.x + 0.5f) / (float)g.W, ((float)c.y + 0.5f) / (float)g.H };
            const float depth = g.fetchd(c);
            uint32_t    n = 0, rays = 0;
            if (depth != 1.0f)
            {
                const vec3 world_pos  = world_position_from_depth(tex_coord, depth, vpi);
                const vec4 gb2        = g.fetch2(c);
                const vec3 normal     = octohedral_to_direction({ gb2.x, gb2.y });
                const vec3 ray_origin = world_pos + normal * bias;
                for (int s = 0; s < spp; s++)
                {
                    const uint32_t idx = f.num_frames * (uint32_t)spp + (uint32_t)s;
                    const vec2 rnd = { sample_blue_noise(c, idx, 0, bn), sample_blue_noise(c, idx, 1, bn) };
                    if (ao) { rays++; n += (uint32_t)scene.query_visibility(ray_origin, sample_cosine_lobe(normal, rnd), p0); }
                    else
                    {
                        vec3  Wi;
                        float t_max, attenuation;
                        fetch_light_properties_shadow(f.ubo.light, world_pos, normal, rnd, Wi, t_max, attenuation);
                        if (attenuation > 0.0f) { rays++; n += (uint32_t)scene.query_visibility(ray_origin, Wi, t_max); }
                    }
                }
            }
            count[(size_t)y * g.W + x] = (uint8_t)n;
            count_rays(0, rays);
        }
}

// unpack_*_hit_value + neighborhood_mean (shadows_denoise_reprojection.comp:114-190, ao twin :101-185):
// exact 17x17 box sum of mask bits; mask words outside the mask image read as `oob_word`.
inline uint32_t mask_bit(const uint32_t* mask, int MW, int MH, ivec2 p, uint32_t oob_word)
{
    // p may be negative: floor division into mask words like the shader's cache addressing.
    int      mx = (p.x >= 0) ? p.x / 8 : -((-p.x + 7) / 8);
    int      my = (p.y >= 0) ? p.y / 4 : -((-p.y + 3) / 4);
    int      bx = p.x - mx * 8, by = p.y - my * 4;
    uint32_t w  = (mx < 0 || my < 0 || mx >= MW || my >= MH) ? oob_word : mask[(size_t)my * MW + mx];
    return (w >> (by * 8 + bx)) & 1u;
}
inline float neighborhood_mean(const uint32_t* mask, int MW, int MH, ivec2 c, uint32_t oob_word)
{
    float mean = 0.0f;
    for (int y = -8; y <= 8; y++)
    {
        float row = 0.0f;
        for (int x = -8; x <= 8; x++) row += (float)mask_bit(mask, MW, MH, { c.x + x, c.y + y }, oob_word);
        mean += row;
    }
    return mean / 289.0f;
}

// Visibility source of the temporal stages: the packed 1-bit ray mask (spp = 1, the reference's format) or, for spp > 1,
// the 8-bit count image (see ray_trace_count).  Pixels outside the image read as `oob_word`'s bit (shadows 0, AO all rays
// unoccluded: ao_denoise_reprojection.comp:111-112).
struct VisSrc {
    const uint32_t* mask;
    const uint8_t*  count;
    int             W, H, spp;
    uint32_t        oob_word;
    float hits(ivec2 p) const
    {
        if (!count) return (float)mask_bit(mask, (W + 7) / 8, (H + 3) / 4, p, oob_word);
        // the mask image covers whole 8x4 groups: pixels of a partially covered group that lie outside the image count 0
        const int MW = (W + 7) / 8, MH = (H + 3) / 4;
        if (p.x < 0 || p.y < 0 || p.x >= MW * 8 || p.y >= MH * 4) return oob_word ? (float)spp : 0.0f;
        if (p.x >= W || p.y >= H) return 0.0f;
        return (float)count[(size_t)p.y * W + p.x];
    }
    float visibility(ivec2 p) const { return spp == 1 ? hits(p) : hits(p) / (float)spp; }
    float mean(ivec2 c) const
    {
        float m = 0.0f;
        for (int y = -8; y <= 8; y++)
        {
            float row = 0.0f;
            for (int x = -8; x <= 8; x++) row += hits({ c.x + x, c.y + y });
            m += row;
        }
        return m / (289.0f * (float)spp);
    }
};

// ------------------------------------------------------------------------------------------------
// K3  shadows/shadows_denoise_reprojection.comp:196-293
// tile_flags: 1 = tile appended to DenoiseTileData, 0 = to ShadowTileData (:274-292).
// ------------------------------------------------------------------------------------------------
void shadows_temporal(const GBufLevel& cur, const GBufLevel& prev, const VisSrc& vs, const uint16_t* prev_image, const uint16_t* prev_moments,
                      const hr_frame& f, float alpha_p, float moments_alpha_p, uint16_t* out, uint16_t* moments_out, uint8_t* tile_flags)
{
    const int  W = cur.W, H = cur.H, TW = (W + 7) / 8, TH = (H + 7) / 8;
    const mat4 vpi = load_mat4(f.ubo.view_proj_inverse);
    memset(tile_flags, 0, (size_t)TW * TH);
#pragma omp parallel for schedule(dynamic, 1)
    for (int ty = 0; ty < TH; ty++)
        for (int tx = 0; tx < TW; tx++)
        {
            bool should_denoise = false;
            for (int ly = 0; ly < 8; ly++)
                for (int lx = 0; lx < 8; lx++)
                {
                    ivec2 c = { tx * 8 + lx, ty * 8 + ly };
                    if (!cur.inside(c)) continue;
                    float mean  = vs.mean(c);
                    float depth = cur.fetchd(c);
                    float visibility = 0.0f, ov = 0.0f, ovar = 0.0f, om0 = 0.0f, om1 = 0.0f, history_length = 0.0f;
                    if (depth != 1.0f)
                    {
                        visibility = vs.visibility(c);
                        ReprojectIn in;
                        in.frag_coord        = c;
                        in.depth             = depth;
                        in.cur               = &cur;
                        in.prev              = &prev;
                        in.history_output    = { W, H, 2, prev_image };
                        in.history_moments   = { W, H, 4, prev_moments };
                        in.moments           = true;
                        in.reflections       = false;
                        in.view_proj_inverse = vpi;
                        ReprojectOut ro;
                        bool  success            = reproject<1>(in, ro);
                        float history_visibility = ro.history_color[0];
                        history_length           = fminf(32.0f, success ? ro.history_length + 1.0f : 1.0f);
                        if (success)
                        {
                            float spatial_variance = fmaxf(mean - mean * mean, 0.0f);
                            float std_deviation    = sqrtf(spatial_variance);
                            float nmin = mean - 0.5f * std_deviation, nmax = mean + 0.5f * std_deviation;
                            history_visibility = clampf(history_visibility, nmin, nmax);
                        }
                        const float alpha         = success ? fmaxf(alpha_p, 1.0f / history_length) : 1.0f;
                        const float alpha_moments = success ? fmaxf(moments_alpha_p, 1.0f / history_length) : 1.0f;
                        om0  = visibility;
                        om1  = om0 * om0;
                        om0  = mixf(ro.history_moments[0], om0, alpha_moments);
                        om1  = mixf(ro.history_moments[1], om1, alpha_moments);
                        ovar = fmaxf(0.0f, om1 - om0 * om0);
                        ov   = mixf(history_visibility, visibility, alpha);
                    }
                    store_h(moments_out, W, 4, c, 0, om0);
                    store_h(moments_out, W, 4, c, 1, om1);
                    store_h(moments_out, W, 4, c, 2, history_length);
                    store_h(moments_out, W, 4, c, 3, 0.0f);
                    store_h(out, W, 2, c, 0, ov);
                    store_h(out, W, 2, c, 1, ovar);
                    if (depth != 1.0f && ov > 0.0f) should_denoise = true;
                }
            tile_flags[(size_t)ty * TW + tx] = should_denoise ? 1 : 0;
        }
}

// ------------------------------------------------------------------------------------------------
// K4 + K5  shadows_denoise_copy_shadow_tiles.comp:32-36, shadows_denoise_atrous.comp:94-174
// ------------------------------------------------------------------------------------------------
void shadows_atrous(const GBufLevel& g, const uint16_t* in_img, const uint8_t* tile_flags, int radius, int step_size, float phi_visibility,
                    float phi_normal, float sigma_depth, float power, uint16_t* out)
{
    const int   W = g.W, H = g.H, TW = (W + 7) / 8;
    const ImgH  in = { W, H, 2, in_img };
    const float* kernel_weights = orc_const::ATROUS_KERNEL_WEIGHTS;
    const auto& vk = orc_const::ATROUS_VARIANCE_KERNEL;
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++)
        {
            ivec2 ipos = { x, y };
            if (!tile_flags[(size_t)(y / 8) * TW + x / 8])
            { // copy_shadow_tiles: whole tile = 0
                store_h(out, W, 2, ipos, 0, 0.0f);
                store_h(out, W, 2, ipos, 1, 0.0f);
                continue;
            }
            const float cv0 = in.fetch(ipos, 0), cv1 = in.fetch(ipos, 1);
            float       var = 0.0f; // compute_variance_center :65-88
            for (int yy = -1; yy <= 1; yy++)
                for (int xx = -1; xx <= 1; xx++) var += in.fetch({ x + xx, y + yy }, 1) * vk[abs(xx)][abs(yy)];
            vec4  c2 = g.fetch2(ipos), c3 = g.fetch3(ipos);
            vec3  current_normal = octohedral_to_direction({ c2.x, c2.y });
            float center_depth   = c3.w;
            if (center_depth < 0.0f)
            {
                store_h(out, W, 2, ipos, 0, cv0);
                store_h(out, W, 2, ipos, 1, cv1);
                continue;
            }
            const float phi_vis = phi_visibility * sqrtf(fmaxf(0.0f, orc_const::ATROUS_EPS_VARIANCE + var));
            float       sum_w = 1.0f, s0 = cv0, s1 = cv1;
            for (int yy = -radius; yy <= radius; yy++)
                for (int xx = -radius; xx <= radius; xx++)
                {
                    const ivec2 p      = { x + xx * step_size, y + yy * step_size };
                    const bool  inside = p.x >= 0 && p.y >= 0 && p.x < W && p.y < H;
                    const float kernel = kernel_weights[abs(xx)] * kernel_weights[abs(yy)];
                    if (inside && (xx != 0 || yy != 0))
                    {
                        const float sv0 = in.fetch(p, 0), sv1 = in.fetch(p, 1);
                        vec4  s2 = g.fetch2(p), s3 = g.fetch3(p);
                        vec3  sample_normal = octohedral_to_direction({ s2.x, s2.y });
                        float w = compute_edge_stopping_weight(center_depth, s3.w, sigma_depth, current_normal, sample_normal, phi_normal, true, cv0, sv0, phi_vis);
                        const float wv = w * kernel;
                        sum_w += wv;
                        s0 += wv * sv0;
                        s1 += (wv * wv) * sv1;
                    }
                }
            float o0 = s0 / sum_w, o1 = s1 / (sum_w * sum_w);
            if (power != 0.0f) o0 = powf(o0, power);
            store_h(out, W, 2, ipos, 0, o0);
            store_h(out, W, 2, ipos, 1, o1);
        }
}

// textureLod(img, uv, mip) with NEAREST + CLAMP_TO_EDGE (vk.cpp:3453-3484): texel = clamp(floor(uv*size), 0, size-1)
inline ivec2 nearest_texel(vec2 uv, int W, int H)
{
    int x = (int)floorf(uv.x * (float)W), y = (int)floorf(uv.y * (float)H);
    return { std::min(std::max(x, 0), W - 1), std::min(std::max(y, 0), H - 1) };
}

// ------------------------------------------------------------------------------------------------
// K6 / K11  shadows_upsample.comp:62-109, ao_upsample.comp:63-112
// in_img: coarse image with C channels, channel 0 used.  sky_value: 0 (shadows) / 1 (ao).  power: 0 = none.
// ------------------------------------------------------------------------------------------------
void upsample_scalar(const GBufLevel& g0, const GBufLevel& gm, const uint16_t* in_img, int in_channels, float sky_value, float power, uint16_t* out)
{
    const int   W0 = g0.W, H0 = g0.H;
    const ImgH  in = { gm.W, gm.H, in_channels, in_img };
    const vec2  texel_size = { 1.0f / (float)gm.W, 1.0f / (float)gm.H };
    const vec2  g_kernel[4] = { { 0.0f, 1.0f }, { 1.0f, 0.0f }, { -1.0f, 0.0f }, { 0.0f, -1.0f } };
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < H0; y++)
        for (int x = 0; x < W0; x++)
        {
            ivec2 c = { x, y };
            const vec2 tex_coord = { ((float)x + 0.5f) / (float)W0, ((float)y + 0.5f) / (float)H0 };
            float hi_res_depth = g0.fetch3(c).w;
            if (hi_res_depth == -1.0f) { out[(size_t)y * W0 + x] = f2h(sky_value); continue; }
            vec4  h2 = g0.fetch2(c);
            vec3  hi_res_normal = octohedral_to_direction({ h2.x, h2.y });
            float upsampled = 0.0f, total_w = 0.0f;
            for (int i = 0; i < 4; i++)
            {
                vec2  ctc = { tex_coord.x + g_kernel[i].x * texel_size.x, tex_coord.y + g_kernel[i].y * texel_size.y };
                ivec2 ct  = nearest_texel(ctc, gm.W, gm.H);
                float coarse_depth = gm.fetch3(ct).w;
                if (coarse_depth == -1.0f) continue;
                vec4 c2 = gm.fetch2(ct);
                vec3 coarse_normal = octohedral_to_direction({ c2.x, c2.y });
                float w = compute_edge_stopping_weight(hi_res_depth, coarse_depth, 1.0f, hi_res_normal, coarse_normal, 32.0f, false, 0, 0, 0);
                upsampled += in.fetch(ct, 0) * w;
                total_w += w;
            }
            upsampled = upsampled / fmaxf(total_w, 0.00000001f);
            if (power != 0.0f) upsampled = powf(upsampled, power);
            out[(size_t)y * W0 + x] = f2h(upsampled);
        }
}

// ------------------------------------------------------------------------------------------------
// K9  ao/ao_denoise_reprojection.comp:191-260
// ------------------------------------------------------------------------------------------------
void ao_temporal(const GBufLevel& cur, const GBufLevel& prev, const VisSrc& vs, const uint16_t* prev_ao, const uint16_t* prev_len,
                 const hr_frame& f, float alpha_p, uint16_t* out, uint16_t* len_out, uint8_t* tile_flags)
{
    const int  W = cur.W, H = cur.H, TW = (W + 7) / 8, TH = (H + 7) / 8;
    const mat4 vpi = load_mat4(f.ubo.view_proj_inverse);
#pragma omp parallel for schedule(dynamic, 1)
    for (int ty = 0; ty < TH; ty++)
        for (int tx = 0; tx < TW; tx++)
        {
            bool should_denoise = false;
            for (int ly = 0; ly < 8; ly++)
                for (int lx = 0; lx < 8; lx++)
                {
                    ivec2 c = { tx * 8 + lx, ty * 8 + ly };
                    if (!cur.inside(c)) continue;
                    float mean   = vs.mean(c); // out-of-image words read as all-visible, :111-112
                    float depth  = cur.fetchd(c);
                    float out_ao = 1.0f, history_length = 0.0f;
                    if (depth != 1.0f)
                    {
                        float ao = vs.visibility(c);
                        ReprojectIn in;
                        in.frag_coord        = c;
                        in.depth             = depth;
                        in.cur               = &cur;
                        in.prev              = &prev;
                        in.history_output    = { W, H, 1, prev_ao };
                        in.history_moments   = { W, H, 1, prev_len };
                        in.moments           = false;
                        in.reflections       = false;
                        in.view_proj_inverse = vpi;
                        ReprojectOut ro;
                        bool  success    = reproject<1>(in, ro);
                        float history_ao = ro.history_color[0];
                        history_length   = fminf(32.0f, success ? ro.history_length + 1.0f : 1.0f);
                        if (success)
                        {
                            float spatial_variance = fmaxf(mean - mean * mean, 0.0f);
                            float std_deviation    = sqrtf(spatial_variance);
                            history_ao             = clampf(history_ao, mean - 0.5f * std_deviation, mean + 0.5f * std_deviation);
                        }
                        const float alpha = success ? fmaxf(alpha_p, 1.0f / history_length) : 1.0f;
                        out_ao            = mixf(history_ao, ao, alpha);
                    }
                    out[(size_t)c.y * W + c.x]     = f2h(out_ao);
                    len_out[(size_t)c.y * W + c.x] = f2h(history_length);
                    if (out_ao < 1.0f) should_denoise = true;
                }
            tile_flags[(size_t)ty * TW + tx] = should_denoise ? 1 : 0;
        }
}

// ------------------------------------------------------------------------------------------------
// K10 ao/ao_denoise_bilateral_blur.comp:75-139.  Untouched tiles keep the cleared value 1.0 (ray_traced_ao.cpp:1055,1104).
// ------------------------------------------------------------------------------------------------
void ao_bilateral_blur(const GBufLevel& g, const uint16_t* in_img, const uint8_t* tile_flags, const float* zbp, int dirx, int diry, int radius, uint16_t* out)
{
    const int   W = g.W, H = g.H, TW = (W + 7) / 8;
    const ImgH  in = { W, H, 1, in_img };
    const float deviation = (float)radius / 1.5f; // GAUSS_BLUR_DEVIATION
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++)
        {
            ivec2 c = { x, y };
            if (!tile_flags[(size_t)(y / 8) * TW + x / 8]) { out[(size_t)y * W + x] = f2h(1.0f); continue; }
            float depth = g.fetchd(c);
            if (depth == 1.0f) { out[(size_t)y * W + x] = f2h(1.0f); continue; }
            float total_ao = in.fetch(c, 0), total_weight = 1.0f;
            float center_depth = linear_eye_depth(depth, zbp);
            vec4  c2 = g.fetch2(c);
            vec3  center_normal = octohedral_to_direction({ c2.x, c2.y });
            for (int i = -radius; i <= radius; i++)
            {
                if (i == 0) continue;
                ivec2 sc = { x + dirx * i, y + diry * i };
                float sample_depth = linear_eye_depth(g.fetchd(sc), zbp);
                float sample_ao    = in.fetch(sc, 0);
                vec4  s2 = g.fetch2(sc);
                vec3  sample_normal = octohedral_to_direction({ s2.x, s2.y });
                float weight = gaussian_weight((float)i, deviation);
                weight *= compute_edge_stopping_weight(center_depth, sample_depth, 1.0f, center_normal, sample_normal, 32.0f, false, 0, 0, 0);
                total_ao += weight * sample_ao;
                total_weight += weight;
            }
            out[(size_t)y * W + x] = f2h(total_ao / fmaxf(total_weight, 0.0001f));
        }
}

// NEAREST blit mip chain (g_buffer.cpp:236-244 -> vk.cpp:332-407): dst(x,y) = src(min(2x+1,W-1), min(2y+1,H-1)).
void build_mip(int W, int H, const uint16_t* gb2, const uint16_t* gb3, const float* depth, uint16_t* ogb2, uint16_t* ogb3, float* odepth)
{
    int w = std::max(W / 2, 1), h = std::max(H / 2, 1);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
        {
            int sx = std::min(2 * x + 1, W - 1), sy = std::min(2 * y + 1, H - 1);
            memcpy(ogb2 + 4 * ((size_t)y * w + x), gb2 + 4 * ((size_t)sy * W + sx), 8);
            memcpy(ogb3 + 4 * ((size_t)y * w + x), gb3 + 4 * ((size_t)sy * W + sx), 8);
            odepth[(size_t)y * w + x] = depth[(size_t)sy * W + sx];
        }
}

} // namespace

// ================================================================================================
// C interface for the tests (ctypes).  Plain host pointers.
// ================================================================================================
extern "C" {

// record reproject()'s branches (ORC_RP_* bits, orc_glsl.h) into `codes` (one byte per pixel of the next temporal stage's pass), or stop (NULL)
void orc_set_reproject_codes(uint8_t* codes) { reproject_codes() = codes; }

// the rays counted since the previous call (ray_counts, orc_glsl.h): out[0] primary, out[1] secondary; the counts restart at 0
void orc_take_ray_counts(uint64_t* out)
{
    for (int k = 0; k < 2; k++) out[k] = ray_counts()[k].exchange(0);
}

struct orc_gbuf { int32_t W, H; const uint16_t* gb2; const uint16_t* gb3; const float* depth; };
static GBufLevel lvl(const orc_gbuf* g) { GBufLevel l; l.W = g->W; l.H = g->H; l.gb2 = g->gb2; l.gb3 = g->gb3; l.depth = g->depth; return l; }

void* orc_scene_create(const float* tri_verts9, size_t n_tris, int brute_force)
{
    Scene* s = new Scene();
    s->bvh.build(tri_verts9, n_tris);
    s->brute = brute_force != 0;
    return s;
}
void orc_scene_set_brute(void* s, int brute) { ((Scene*)s)->brute = brute != 0; }
void orc_scene_destroy(void* s) { delete (Scene*)s; }

// rays: n x 8 floats {o.xyz, tmin, d.xyz, tmax}
void orc_trace_any(void* sp, const float* rays, size_t n, uint32_t* out_hit)
{
    const Scene& s = *(Scene*)sp;
#pragma omp parallel for schedule(dynamic, 64)
    for (long i = 0; i < (long)n; i++)
    {
        const float* r = rays + 8 * i;
        vec3 o = { r[0], r[1], r[2] }, d = { r[4], r[5], r[6] };
        out_hit[i] = s.brute ? s.bvh.any_hit_brute(o, d, r[3], r[7]) : s.bvh.any_hit(o, d, r[3], r[7]);
    }
}
void orc_trace_closest(void* sp, const float* rays, size_t n, float* out_t, uint32_t* out_prim, float* out_uv)
{
    const Scene& s = *(Scene*)sp;
#pragma omp parallel for schedule(dynamic, 64)
    for (long i = 0; i < (long)n; i++)
    {
        const float* r = rays + 8 * i;
        vec3 o = { r[0], r[1], r[2] }, d = { r[4], r[5], r[6] };
        Hit  h;
        s.closest(o, d, r[3], r[7], h);
        out_t[i] = h.t; out_prim[i] = h.prim; out_uv[2 * i] = h.u; out_uv[2 * i + 1] = h.v;
    }
}

void orc_det_sincos(const float* x, size_t n, float* s, float* c) { for (size_t i = 0; i < n; i++) det_sincos(x[i], s + i, c + i); }
void orc_oct_decode(const float* e, size_t n, float* out) { for (size_t i = 0; i < n; i++) { vec3 v = octohedral_to_direction({ e[2*i], e[2*i+1] }); out[3*i]=v.x; out[3*i+1]=v.y; out[3*i+2]=v.z; } }
float orc_sample_blue_noise(int x, int y, int idx, int dim, const uint8_t* sobol, const uint8_t* sr) { BlueNoise bn{ sobol, sr }; return sample_blue_noise({ x, y }, (uint32_t)idx, dim, bn); }

void orc_build_mip(int W, int H, const uint16_t* gb2, const uint16_t* gb3, const float* depth, uint16_t* ogb2, uint16_t* ogb3, float* odepth)
{ build_mip(W, H, gb2, gb3, depth, ogb2, ogb3, odepth); }

void orc_shadows_ray_trace(void* scene, const orc_gbuf* g, const hr_frame* f, float bias, const uint8_t* sobol, const uint8_t* sr, uint32_t* mask)
{ BlueNoise bn{ sobol, sr }; shadows_ray_trace(*(Scene*)scene, lvl(g), *f, bias, bn, mask); }

void orc_ao_ray_trace(void* scene, const orc_gbuf* g, const hr_frame* f, float ray_length, float bias, const uint8_t* sobol, const uint8_t* sr, uint32_t* mask)
{ BlueNoise bn{ sobol, sr }; ao_ray_trace(*(Scene*)scene, lvl(g), *f, ray_length, bias, bn, mask); }

void orc_shadows_temporal(const orc_gbuf* cur, const orc_gbuf* prev, const uint32_t* mask, const uint16_t* prev_image, const uint16_t* prev_moments,
                          const hr_frame* f, float alpha, float moments_alpha, uint16_t* out, uint16_t* moments_out, uint8_t* tile_flags)
{ VisSrc vs{ mask, nullptr, cur->W, cur->H, 1, 0u }; shadows_temporal(lvl(cur), lvl(prev), vs, prev_image, prev_moments, *f, alpha, moments_alpha, out, moments_out, tile_flags); }

void orc_shadows_atrous(const orc_gbuf* g, const uint16_t* in_img, const uint8_t* tile_flags, int radius, int step_size, float phi_visibility,
                        float phi_normal, float sigma_depth, float power, uint16_t* out)
{ shadows_atrous(lvl(g), in_img, tile_flags, radius, step_size, phi_visibility, phi_normal, sigma_depth, power, out); }

void orc_upsample_scalar(const orc_gbuf* g0, const orc_gbuf* gm, const uint16_t* in_img, int in_channels, float sky_value, float power, uint16_t* out)
{ upsample_scalar(lvl(g0), lvl(gm), in_img, in_channels, sky_value, power, out); }

void orc_ao_temporal(const orc_gbuf* cur, const orc_gbuf* prev, const uint32_t* mask, const uint16_t* prev_ao, const uint16_t* prev_len,
                     const hr_frame* f, float alpha, uint16_t* out, uint16_t* len_out, uint8_t* tile_flags)
{ VisSrc vs{ mask, nullptr, cur->W, cur->H, 1, 0xFFFFFFFFu }; ao_temporal(lvl(cur), lvl(prev), vs, prev_ao, prev_len, *f, alpha, out, len_out, tile_flags); }

void orc_ao_bilateral_blur(const orc_gbuf* g, const uint16_t* in_img, const uint8_t* tile_flags, const float* zbp, int dirx, int diry, int radius, uint16_t* out)
{ ao_bilateral_blur(lvl(g), in_img, tile_flags, zbp, dirx, diry, radius, out); }

// ---- spp > 1 (count images) ----
void orc_shadows_ray_trace_spp(void* scene, const orc_gbuf* g, const hr_frame* f, float bias, int spp, const uint8_t* sobol, const uint8_t* sr, uint8_t* count)
{ BlueNoise bn{ sobol, sr }; ray_trace_count(*(Scene*)scene, lvl(g), *f, false, 0.0f, bias, spp, bn, count); }

void orc_ao_ray_trace_spp(void* scene, const orc_gbuf* g, const hr_frame* f, float ray_length, float bias, int spp, const uint8_t* sobol, const uint8_t* sr,
                          uint8_t* count)
{ BlueNoise bn{ sobol, sr }; ray_trace_count(*(Scene*)scene, lvl(g), *f, true, ray_length, bias, spp, bn, count); }

void orc_shadows_temporal_spp(const orc_gbuf* cur, const orc_gbuf* prev, const uint8_t* count, int spp, const uint16_t* prev_image, const uint16_t* prev_moments,
                              const hr_frame* f, float alpha, float moments_alpha, uint16_t* out, uint16_t* moments_out, uint8_t* tile_flags)
{ VisSrc vs{ nullptr, count, cur->W, cur->H, spp, 0u }; shadows_temporal(lvl(cur), lvl(prev), vs, prev_image, prev_moments, *f, alpha, moments_alpha, out, moments_out, tile_flags); }

void orc_ao_temporal_spp(const orc_gbuf* cur, const orc_gbuf* prev, const uint8_t* count, int spp, const uint16_t* prev_ao, const uint16_t* prev_len,
                         const hr_frame* f, float alpha, uint16_t* out, uint16_t* len_out, uint8_t* tile_flags)
{ VisSrc vs{ nullptr, count, cur->W, cur->H, spp, 0xFFFFFFFFu }; ao_temporal(lvl(cur), lvl(prev), vs, prev_ao, prev_len, *f, alpha, out, len_out, tile_flags); }

// bench.py sets the thread count explicitly (launchers such as torchrun export OMP_NUM_THREADS=1)
void orc_set_num_threads(int n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#endif
}

int orc_num_threads(void)
{
    int n = 1;
#ifdef _OPENMP
#pragma omp parallel
    {
#pragma omp master
        n = omp_get_num_threads();
    }
#endif
    return n;
}

} // extern "C"
