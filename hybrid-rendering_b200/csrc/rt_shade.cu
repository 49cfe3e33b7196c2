// rt_shade.cu — the two closest-hit ray-trace stages with hit shading.
//   K18 gi/gi_ray_trace.{rgen,rchit,rmiss}                     (256 rays / probe -> radiance + direction/distance images)
//   K12 reflections/reflections_ray_trace.{rgen,rchit,rmiss}   (1 reflection ray / pixel -> RGBA16F colour + ray length)
// Hit shading: fetch_triangle / interpolated_vertex (scene_descriptor_set.glsl:117-160), direct_lighting
// (lighting.glsl:117-196) with its shadow ray, evaluate_uber_brdf (brdf.glsl:130-142), DDGI infinite bounce
// (gi_common.glsl:188-320).  Environment = constant colour (sky cubemap / IBL assets are not in the repository).
//
// BUILD NOTE: compiled with -fmad=false.  Everything that decides *which surface is hit or whether a shadow ray is
// blocked* (ray directions, hit point, shading normal, shadow-ray origin) follows the deterministic fp32 rules of
// det_math.cuh so that the binary visibility inside the shading is identical to the CPU oracle's; colours are
// tolerance-checked.
#include "gi_common.cuh"
#include "traverse.cuh"

namespace {

using det::V3;
using namespace trv;

struct ShadeDev {
    const float*       verts;    // n*9 world-space positions, primitive order
    const float4*      vnormals; // n*3 world-space unit vertex normals
    const uint32_t*    prim_mat;
    const hr_material* materials;
};

struct Surface { V3 P, N; float3 albedo; float roughness, metallic; };

__device__ __forceinline__ float3 to_f3(V3 v) { return make_float3(v.x, v.y, v.z); }

__device__ __forceinline__ Surface fetch_surface(const ShadeDev& sd, uint32_t prim, float u, float v)
{
    const float* p  = sd.verts + 9ull * prim;
    const float4 n0 = __ldg(sd.vnormals + 3ull * prim), n1 = __ldg(sd.vnormals + 3ull * prim + 1), n2 = __ldg(sd.vnormals + 3ull * prim + 2);
    const float  b0 = 1.0f - u - v, b1 = u, b2 = v;
    Surface      s;
    s.P = det::add(det::add(det::scale(det::mk(__ldg(p), __ldg(p + 1), __ldg(p + 2)), b0), det::scale(det::mk(__ldg(p + 3), __ldg(p + 4), __ldg(p + 5)), b1)),
                   det::scale(det::mk(__ldg(p + 6), __ldg(p + 7), __ldg(p + 8)), b2));
    s.N = det::normalize(det::add(det::add(det::scale(det::mk(n0.x, n0.y, n0.z), b0), det::scale(det::mk(n1.x, n1.y, n1.z), b1)), det::scale(det::mk(n2.x, n2.y, n2.z), b2)));
    const hr_material* m = sd.materials + __ldg(sd.prim_mat + prim);
    s.albedo    = make_float3(m->albedo[0], m->albedo[1], m->albedo[2]);
    s.roughness = fmaxf(m->roughness, 0.1f); // MIN_ROUGHNESS
    s.metallic  = m->metallic;
    return s;
}

// ---- brdf.glsl:36-142 (colour maths) ----------------------------------------------------------------------------------
__device__ __forceinline__ float D_ggx(float ndoth, float alpha)
{
    const float a2 = alpha * alpha, denom = (ndoth * ndoth) * (a2 - 1.0f) + 1.0f;
    return a2 / fmaxf(0.0001f, 3.14159265359f * denom * denom);
}
__device__ __forceinline__ float G1_schlick_ggx(float roughness, float ndotv)
{
    const float k = ((roughness + 1.0f) * (roughness + 1.0f)) / 8.0f;
    return ndotv / fmaxf(0.0001f, ndotv * (1.0f - k) + k);
}
__device__ __forceinline__ float3 evaluate_uber_brdf(float3 diffuse_color, float roughness, V3 N, float3 F0, V3 Wo, V3 Wh, V3 Wi)
{
    using namespace gi;
    const float NdotL = fmaxf(det::dot(N, Wi), 0.0f), NdotV = fmaxf(det::dot(N, Wo), 0.0f), NdotH = fmaxf(det::dot(N, Wh), 0.0f), VdotH = fmaxf(det::dot(Wi, Wh), 0.0f);
    const float p5 = powf(1.0f - VdotH, 5.0f);
    const float3 F = F0 + (f3(1, 1, 1) - F0) * p5;
    const float spec = D_ggx(NdotH, roughness * roughness) * (G1_schlick_ggx(roughness, NdotL) * G1_schlick_ggx(roughness, NdotV)) / fmaxf(0.0001f, 4.0f * NdotL * NdotV);
    return (f3(1, 1, 1) - F) * (diffuse_color * (1.0f / 3.14159265359f)) + F * spec;
}

// fetch_light_properties without SOFT_SHADOWS (lighting.glsl:6-111)
__device__ __forceinline__ void fetch_light_properties_hard(const hr_light& L, V3 P, V3 N, float3& Li, V3& Wi, float& t_max, float& attenuation)
{
    const int type = (int)L.data3[0];
    const V3  ldir = det::mk(L.data0[0], L.data0[1], L.data0[2]);
    Li = make_float3(L.data2[0] * L.data0[3], L.data2[1] * L.data0[3], L.data2[2] * L.data0[3]);
    if (type == 0) { Wi = ldir; t_max = 10000.0f; attenuation = 1.0f; }
    else
    {
        const V3    to_light = det::sub(det::mk(L.data1[0], L.data1[1], L.data1[2]), P);
        const float dist     = det::length(to_light);
        Wi    = det::normalize(to_light);
        t_max = dist;
        if (type == 1) attenuation = 1.0f / (dist * dist);
        else
        {
            const float e0 = L.data3[1], e1 = L.data3[2];
            const float t = det::clampf((det::dot(Wi, ldir) - e0) / (e1 - e0), 0.0f, 1.0f);
            attenuation   = (t * t * (3.0f - 2.0f * t)) / (dist * dist);
        }
    }
    attenuation *= det::clampf(det::dot(N, Wi), 0.0f, 1.0f);
}

// direct_lighting, lighting.glsl:117-196
__device__ float3 direct_lighting(const BvhDev& bvh, const hr_light& light, V3 Wo, V3 N, V3 P, float3 F0, float3 diffuse_color, float roughness, bool sky_light,
                                  float r0, float r1, float3 sky, unsigned long long* ray_ctr)
{
    using namespace gi;
    float3 Lo = f3(0, 0, 0);
    Ray    sr;
    sr.o    = det::add(P, det::scale(N, 0.1f));
    sr.tmin = 0.01f;
    {
        float3 Li;
        V3     Wi;
        float  t_max, att;
        fetch_light_properties_hard(light, P, N, Li, Wi, t_max, att);
        const V3 Wh = det::normalize(det::add(Wo, Wi));
        if (att > 0.0f)
        {
            sr.d    = Wi;
            sr.tmax = t_max;
            count_rays(ray_ctr, 1, 1u);
            att *= trace_any(bvh, sr) ? 0.0f : 1.0f;
        }
        const float3 brdf = evaluate_uber_brdf(diffuse_color, roughness, N, F0, Wo, Wh, Wi);
        Lo = Lo + (brdf * att) * Li;
    }
    if (sky_light)
    {
        const V3 Wi = det::sample_cosine_lobe(N, r0, r1);
        const V3 Wh = det::normalize(det::add(Wo, Wi));
        sr.d    = Wi;
        sr.tmax = 10000.0f;
        count_rays(ray_ctr, 1, 1u);
        const float  vis  = trace_any(bvh, sr) ? 0.0f : 1.0f;
        const float3 brdf = evaluate_uber_brdf(diffuse_color, roughness, N, F0, Wo, Wh, Wi);
        Lo = Lo + brdf * (sky * vis);
    }
    return Lo;
}

__device__ float3 indirect_diffuse(const hr_ddgi_uniforms& d, const gi::AtlasDev& at, V3 Wo, V3 N, V3 P, float3 F0, float3 diffuse_color, float roughness,
                                   float metallic, float gi_intensity)
{
    using namespace gi;
    const float  ct = fmaxf(det::dot(N, Wo), 0.0f);
    const float  p5 = powf(fmaxf(1.0f - ct, 0.0f), 5.0f), omr = 1.0f - roughness;
    const float3 F  = F0 + (f3(fmaxf(omr, F0.x), fmaxf(omr, F0.y), fmaxf(omr, F0.z)) - F0) * p5;
    const float3 kD = (f3(1, 1, 1) - F) * (1.0f - metallic);
    const float3 irr = sample_irradiance(d, at, to_f3(P), to_f3(N), to_f3(Wo));
    return (kD * diffuse_color) * irr * gi_intensity;
}

// IBL specular, reflections_ray_trace.rchit:97-104: prefiltered * (F * brdf.x + brdf.y) * intensity; brdf = bilinear CLAMP_TO_EDGE fetch of
// the 512 x 512 RG16F LUT at (max(N.Wo, 0), roughness); the prefiltered environment is the constant sky colour
struct IblDev { const uint32_t* lut; float intensity; };
__device__ __forceinline__ float2 brdf_lut_fetch(const uint32_t* __restrict__ lut, float u, float v)
{
    const float x = u * 512.0f - 0.5f, y = v * 512.0f - 0.5f;
    const float fx0 = floorf(x), fy0 = floorf(y), fx = x - fx0, fy = y - fy0;
    const int   x0 = min(max((int)fx0, 0), 511), x1 = min(max((int)fx0 + 1, 0), 511), y0 = min(max((int)fy0, 0), 511), y1 = min(max((int)fy0 + 1, 0), 511);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(lut + y0 * 512 + x0)), b = __half22float2(*reinterpret_cast<const __half2*>(lut + y0 * 512 + x1));
    const float2 c = __half22float2(*reinterpret_cast<const __half2*>(lut + y1 * 512 + x0)), e = __half22float2(*reinterpret_cast<const __half2*>(lut + y1 * 512 + x1));
    return make_float2((a.x * (1.0f - fx) + b.x * fx) * (1.0f - fy) + (c.x * (1.0f - fx) + e.x * fx) * fy,
                       (a.y * (1.0f - fx) + b.y * fx) * (1.0f - fy) + (c.y * (1.0f - fx) + e.y * fx) * fy);
}

__device__ __forceinline__ float3 shade_hit(const BvhDev& bvh, const ShadeDev& sd, const hr_light& light, const Ray& r, uint32_t prim, float u, float v, bool sky_light,
                                            float r0, float r1, float3 sky, bool gi_on, const hr_ddgi_uniforms& d, const gi::AtlasDev& at, float gi_intensity,
                                            unsigned long long* ray_ctr, IblDev ibl = IblDev { nullptr, 0.0f })
{
    using namespace gi;
    const Surface s  = fetch_surface(sd, prim, u, v);
    const V3      Wo = det::scale(r.d, -1.0f);
    const float3  F0 = f3(0.04f, 0.04f, 0.04f) * (1.0f - s.metallic) + s.albedo * s.metallic;             // mix(0.04, albedo, metallic)
    const float3  cd = (s.albedo * (f3(1, 1, 1) - F0)) * (1.0f - s.metallic) + f3(0, 0, 0) * s.metallic; // mix(albedo*(1-F0), 0, metallic)
    float3        Lo = direct_lighting(bvh, light, Wo, s.N, s.P, F0, cd, s.roughness, sky_light, r0, r1, sky, ray_ctr);
    if (gi_on)
    {
        Lo = Lo + indirect_diffuse(d, at, Wo, s.N, s.P, F0, cd, s.roughness, s.metallic, gi_intensity);
        if (ibl.lut)
        {
            const float  ct = fmaxf(det::dot(s.N, Wo), 0.0f), p5 = powf(fmaxf(1.0f - ct, 0.0f), 5.0f), omr = 1.0f - s.roughness;
            const float3 F  = F0 + (f3(fmaxf(omr, F0.x), fmaxf(omr, F0.y), fmaxf(omr, F0.z)) - F0) * p5;
            const float2 b  = brdf_lut_fetch(ibl.lut, ct, s.roughness);
            Lo = Lo + (sky * (F * b.x + f3(b.y, b.y, b.y))) * ibl.intensity;
        }
    }
    return Lo;
}

// Material textures (hr_scene_set_textures, tex_px.cuh): fetch_albedo / fetch_roughness / fetch_metallic at the hit point.  The TEX
// instantiations of the kernels below call these; the untextured instantiations compile exactly as before (tools/sass_function_hashes.py).
__device__ __forceinline__ Surface fetch_surface_tex(const ShadeDev& sd, const tex::TexDev& T, uint32_t prim, float u, float v)
{
    Surface s = fetch_surface(sd, prim, u, v);
    const uint32_t mat = __ldg(sd.prim_mat + prim);
    tex::material_at_hit(T, mat, prim, 1.0f - u - v, u, v, s.albedo.x, s.albedo.y, s.albedo.z, s.roughness, s.metallic);
    tex::normal_at_hit(T, mat, prim, 1.0f - u - v, u, v, true, s.N.x, s.N.y, s.N.z); // the hit shaders pass the tangent as bitangent (rchit:134)
    return s;
}
__device__ __forceinline__ float3 shade_hit_tex(const BvhDev& bvh, const ShadeDev& sd, const tex::TexDev& T, const hr_light& light, const Ray& r, uint32_t prim, float u, float v,
                                                bool sky_light, float r0, float r1, float3 sky, bool gi_on, const hr_ddgi_uniforms& d, const gi::AtlasDev& at, float gi_intensity,
                                                unsigned long long* ray_ctr, IblDev ibl = IblDev { nullptr, 0.0f })
{ // shade_hit with the textured surface
    using namespace gi;
    const Surface s  = fetch_surface_tex(sd, T, prim, u, v);
    const V3      Wo = det::scale(r.d, -1.0f);
    const float3  F0 = f3(0.04f, 0.04f, 0.04f) * (1.0f - s.metallic) + s.albedo * s.metallic;
    const float3  cd = (s.albedo * (f3(1, 1, 1) - F0)) * (1.0f - s.metallic) + f3(0, 0, 0) * s.metallic;
    float3        Lo = direct_lighting(bvh, light, Wo, s.N, s.P, F0, cd, s.roughness, sky_light, r0, r1, sky, ray_ctr);
    if (gi_on)
    {
        Lo = Lo + indirect_diffuse(d, at, Wo, s.N, s.P, F0, cd, s.roughness, s.metallic, gi_intensity);
        if (ibl.lut)
        {
            const float  ct = fmaxf(det::dot(s.N, Wo), 0.0f), p5 = powf(fmaxf(1.0f - ct, 0.0f), 5.0f), omr = 1.0f - s.roughness;
            const float3 F  = F0 + (f3(fmaxf(omr, F0.x), fmaxf(omr, F0.y), fmaxf(omr, F0.z)) - F0) * p5;
            const float2 b  = brdf_lut_fetch(ibl.lut, ct, s.roughness);
            Lo = Lo + (sky * (F * b.x + f3(b.y, b.y, b.y))) * ibl.intensity;
        }
    }
    return Lo;
}

__device__ __forceinline__ uint2 pack_h4(float a, float b, float c, float d)
{
    const __half2 lo = __floats2half2_rn(a, b), hi = __floats2half2_rn(c, d);
    return make_uint2(*reinterpret_cast<const uint32_t*>(&lo), *reinterpret_cast<const uint32_t*>(&hi));
}

// gi_ray_trace.rgen:61-72
__device__ __forceinline__ V3 spherical_fibonacci(float i, float n)
{
    const float PHI = sqrtf(5.0f) * 0.5f + 0.5f;
    const float a   = i * (PHI - 1.0f);
    const float phi = 2.0f * 3.14159265359f * (a - floorf(a));
    const float ct  = 1.0f - (2.0f * i + 1.0f) * (1.0f / n);
    const float st  = sqrtf(det::clampf(1.0f - ct * ct, 0.0f, 1.0f));
    float       sn, cs;
    det::det_sincos(phi, &sn, &cs);
    return det::mk(cs * st, sn * st, ct);
}

struct GiTraceParams { float rot[16]; uint32_t num_frames, infinite_bounces; float gi_intensity; float sky[3]; int probe0, probe1; unsigned long long* ray_ctr; };

// K18: one block per probe, one thread per ray (blockDim = rays_per_probe rounded up to 32, looped if > 256)
template <bool TEX>
__global__ void __launch_bounds__(256) k_ddgi_ray_trace(BvhDev bvh, ShadeDev sd, hr_ddgi_uniforms d, gi::AtlasDev at, hr_light light, GiTraceParams P,
                                                         uint2* __restrict__ radiance, uint2* __restrict__ dirdepth, tex::TexDev T)
{
    const int probe = P.probe0 + blockIdx.x;
    if (probe >= P.probe1) return;
    const int cx = d.probe_counts[0], cxy = d.probe_counts[0] * d.probe_counts[1];
    const V3  origin = det::mk(d.grid_step[0] * (float)(probe % cx) + d.grid_start_position[0], d.grid_step[1] * (float)((probe % cxy) / cx) + d.grid_start_position[1],
                               d.grid_step[2] * (float)(probe / cxy) + d.grid_start_position[2]);
    const float3 sky = make_float3(P.sky[0], P.sky[1], P.sky[2]);
    for (int ray = threadIdx.x; ray < d.rays_per_probe; ray += blockDim.x)
    {
        const V3 sf = spherical_fibonacci((float)ray, (float)d.rays_per_probe);
        Ray      r;
        r.o = origin;
        r.d = det::normalize(det::mk((P.rot[0] * sf.x + P.rot[4] * sf.y) + P.rot[8] * sf.z, (P.rot[1] * sf.x + P.rot[5] * sf.y) + P.rot[9] * sf.z,
                                     (P.rot[2] * sf.x + P.rot[6] * sf.y) + P.rot[10] * sf.z));
        r.tmin = 0.001f;
        r.tmax = 10000.0f;
        gi::RNG  rng = gi::rng_init((uint32_t)ray, (uint32_t)probe, P.num_frames);
        float    t, u, v, hit_distance = 10000.0f;
        uint32_t prim;
        float3   L;
        count_rays(P.ray_ctr, 0, 1u);
        if (trace_closest(bvh, r, t, prim, u, v))
        {
            const float r0 = gi::next_float(rng), r1 = gi::next_float(rng);
            L              = TEX ? shade_hit_tex(bvh, sd, T, light, r, prim, u, v, true, r0, r1, sky, P.infinite_bounces == 1, d, at, P.gi_intensity, P.ray_ctr)
                                 : shade_hit(bvh, sd, light, r, prim, u, v, true, r0, r1, sky, P.infinite_bounces == 1, d, at, P.gi_intensity, P.ray_ctr);
            hit_distance   = 0.001f + t;
        }
        else L = sky;
        const size_t o = (size_t)probe * d.rays_per_probe + ray;
        radiance[o] = pack_h4(L.x, L.y, L.z, 0.0f);
        dirdepth[o] = pack_h4(r.d.x, r.d.y, r.d.z, hit_distance);
    }
}

__device__ __forceinline__ V3 reflect(V3 I, V3 N) { return det::sub(I, det::scale(N, 2.0f * det::dot(N, I))); }

// importance_sample_ggx, reflections_ray_trace.rgen:78-105
__device__ __forceinline__ V3 importance_sample_ggx(float ex, float ey, V3 N, float roughness)
{
    const float a = roughness * roughness, m2 = a * a;
    const float phi = 2.0f * 3.14159265359f * ex;
    const float ct  = sqrtf((1.0f - ey) / (1.0f + (m2 - 1.0f) * ey));
    const float st  = sqrtf(1.0f - ct * ct);
    float       sn, cs;
    det::det_sincos(phi, &sn, &cs);
    const V3 H  = det::mk(cs * st, sn * st, ct);
    const V3 up = fabsf(N.z) < 0.999f ? det::mk(0, 0, 1) : det::mk(1, 0, 0);
    const V3 tangent   = det::normalize(det::cross(up, N));
    const V3 bitangent = det::cross(N, tangent);
    return det::normalize(det::add(det::add(det::scale(tangent, H.x), det::scale(bitangent, H.y)), det::scale(N, H.z)));
}

struct ReflTraceParams { float bias, trim; int sample_gi, approximate_with_ddgi; float gi_intensity, rough_ddgi_intensity; float sky[3]; int row0, row1;
                         int chunk_first, chunk_stride; int spp; IblDev ibl; }; // chunk_stride > 1: the 8-row chunks c = chunk_first + i * chunk_stride of the whole image

// K12: warp = 8x4 pixel block (coherent reflection rays), 256 threads = 32x8 pixels
// 2-warp CTAs (16x4 pixels): closest-hit rays + hit shading are heavy-tailed, small CTAs recycle their slots sooner (trace.cu)
// MULTI = false: exactly the reference's one ray per pixel (straight-line code); true: the spp > 1 extension (sample loop)
template <bool MULTI, int MINB, bool TEX>
__global__ void __launch_bounds__(64, MINB) k_reflections_ray_trace(GBufLevelDev g, BvhDev bvh, ShadeDev sd, FrameConsts fc, hr_ddgi_uniforms d, gi::AtlasDev at,
                                                                ReflTraceParams P, const uint8_t* __restrict__ sobol, const uint8_t* __restrict__ srk,
                                                                uint2* __restrict__ out, tex::TexDev T)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // rows: [row0, row1) or, when the ranks trace cooperatively, the 8-row chunks c = chunk_first + i * chunk_stride of the whole image
    const int x = blockIdx.x * 16 + warp * 8 + (lane & 7);
    const int y = (P.chunk_stride > 1 ? 8 * (P.chunk_first + ((int)blockIdx.y >> 1) * P.chunk_stride) + 4 * ((int)blockIdx.y & 1) : P.row0 + (int)blockIdx.y * 4) + (lane >> 3);
    if (x >= g.W || y >= g.H || (P.chunk_stride <= 1 && y >= P.row1)) return;
    const size_t idx   = (size_t)y * g.W + x;
    const float  depth = __ldg(g.depth + idx);
    if (depth == 1.0f) { out[idx] = pack_h4(0.0f, 0.0f, 0.0f, -1.0f); return; }
    const float  u = ((float)x + 0.5f) / (float)g.W, v = ((float)y + 0.5f) / (float)g.H;
    const uint2  g2 = __ldg(g.gb2 + idx), g3 = __ldg(g.gb3 + idx);
    const float2 e  = __half22float2(*reinterpret_cast<const __half2*>(&g2.x));
    const float  roughness = __half22float2(*reinterpret_cast<const __half2*>(&g3.x)).x;
    const V3     Pw = det::world_position_from_depth(u, v, depth, fc.view_proj_inverse);
    const V3     N  = det::octohedral_to_direction(e.x, e.y);
    const V3     Wo = det::normalize(det::sub(det::mk(fc.cam_pos[0], fc.cam_pos[1], fc.cam_pos[2]), Pw));
    const float3 sky = make_float3(P.sky[0], P.sky[1], P.sky[2]);
    Ray          r;
    r.o    = det::add(Pw, det::scale(N, P.bias));
    r.tmin = 0.001f;
    r.tmax = 10000.0f;
    float3 color = make_float3(0, 0, 0);
    float  ray_length = -1.0f;
    // spp > 1 (SURVEY.md §8d): the GGX lobe draws spp directions, the clamped radiance is averaged, ray_length = first sample's
    const int  spp = MULTI ? (P.spp > 1 ? P.spp : 1) : 1;
    const bool ggx = !(roughness < 0.05f) && !(roughness > 0.75f && P.approximate_with_ddgi == 1);
    const int  n_s = MULTI ? (ggx ? spp : 1) : 1;
    float3     acc = make_float3(0, 0, 0);
#pragma unroll 1
    for (int s = 0; s < n_s; s++)
    {
        bool trace = false;
        if (roughness < 0.05f) { r.d = reflect(det::scale(Wo, -1.0f), N); trace = true; }
        else if (roughness > 0.75f && P.approximate_with_ddgi == 1)
        {
            const V3 R = reflect(det::scale(Wo, -1.0f), N);
            using namespace gi;
            color = sample_irradiance(d, at, to_f3(Pw), to_f3(R), to_f3(Wo)) * P.rough_ddgi_intensity;
        }
        else
        {
            const int   si = (int)fc.num_frames * spp + s;
            const float ex = det::sample_blue_noise(x, y, si, 0, sobol, srk) * P.trim;
            const float ey = det::sample_blue_noise(x, y, si, 1, sobol, srk) * P.trim;
            const V3    Wh = importance_sample_ggx(ex, ey, N, roughness);
            r.d   = reflect(det::scale(Wo, -1.0f), Wh);
            trace = true;
        }
        if (trace)
        {
            float    t, hu, hv;
            uint32_t prim;
            count_rays(fc.ray_ctr, 0, 1u);
            if (trace_closest(bvh, r, t, prim, hu, hv))
            {
                color = TEX ? shade_hit_tex(bvh, sd, T, fc.light, r, prim, hu, hv, false, 0.0f, 0.0f, sky, P.sample_gi == 1, d, at, P.gi_intensity, fc.ray_ctr, P.ibl)
                            : shade_hit(bvh, sd, fc.light, r, prim, hu, hv, false, 0.0f, 0.0f, sky, P.sample_gi == 1, d, at, P.gi_intensity, fc.ray_ctr, P.ibl);
                if (s == 0) ray_length = 0.001f + t;
            }
            else color = sky;
        }
        acc = make_float3(acc.x + fminf(color.x, 0.7f), acc.y + fminf(color.y, 0.7f), acc.z + fminf(color.z, 0.7f));
    }
    const float inv_n = 1.0f / (float)n_s;
    out[idx] = pack_h4(acc.x * inv_n, acc.y * inv_n, acc.z * inv_n, ray_length);
}

// ---------------------------------------------------------------------------------------------------------------------------
// K12, wavefront form (hr_debug_set(7, 1)).  The fused kernel above has about half of its 32 lanes active on average —
// glossy reflection rays of one 8x4 block take different paths through the BVH, and lanes that missed idle while their
// neighbours shade and trace shadow rays.  Split in two:
//   pass A  k_refl_trace: persistent warps pull 32x4-pixel jobs from an atomic counter, generate the reflection rays (sky and
//           DDGI-rough pixels are finished right there), compact the rays that need tracing into a per-warp shared-memory
//           queue, and traverse with all lanes busy: a lane whose ray terminates refills from the queue (closest hit, ties ->
//           lowest primitive, so the result does not depend on the traversal order).  Node stack in shared memory.  Output:
//           one 16-byte hit record per pixel (t, primitive, u, v).
//   pass B  k_refl_shade: a CTA compacts the pixels of its 32x8 tile that hit something, so every lane shades a hit
//           (surface fetch, direct light + its shadow ray, DDGI diffuse); misses get the sky colour.
// Ray generation is a shared device function (pass B recomputes the ray direction instead of reading 16 more bytes).
#define RA_WARPS 8
#define RA_QUEUE 128
#define RA_SM_STACK 24
#define RA_REFILL_STEPS 8
#define HIT_NO_RAY 0xFFFFFFFEu
#define HIT_MISS 0xFFFFFFFFu

enum { RG_SKY = 0, RG_DDGI = 1, RG_TRACE = 2 };

// reflections_ray_trace.rgen:119-171 up to the traceRayEXT call: lobe selection and the reflection ray
__device__ __forceinline__ int refl_ray_gen(const GBufLevelDev& g, const FrameConsts& fc, const ReflTraceParams& P, const uint8_t* __restrict__ sobol,
                                            const uint8_t* __restrict__ srk, int x, int y, Ray& r, V3& Pw, V3& Wo, V3& N)
{
    const size_t idx   = (size_t)y * g.W + x;
    const float  depth = __ldg(g.depth + idx);
    if (depth == 1.0f) return RG_SKY;
    const float  u = ((float)x + 0.5f) / (float)g.W, v = ((float)y + 0.5f) / (float)g.H;
    const uint2  g2 = __ldg(g.gb2 + idx), g3 = __ldg(g.gb3 + idx);
    const float2 e  = __half22float2(*reinterpret_cast<const __half2*>(&g2.x));
    const float  roughness = __half22float2(*reinterpret_cast<const __half2*>(&g3.x)).x;
    Pw = det::world_position_from_depth(u, v, depth, fc.view_proj_inverse);
    N  = det::octohedral_to_direction(e.x, e.y);
    Wo = det::normalize(det::sub(det::mk(fc.cam_pos[0], fc.cam_pos[1], fc.cam_pos[2]), Pw));
    r.o    = det::add(Pw, det::scale(N, P.bias));
    r.tmin = 0.001f;
    r.tmax = 10000.0f;
    if (roughness < 0.05f) { r.d = reflect(det::scale(Wo, -1.0f), N); return RG_TRACE; }
    if (roughness > 0.75f && P.approximate_with_ddgi == 1) return RG_DDGI;
    const float ex = det::sample_blue_noise(x, y, (int)fc.num_frames, 0, sobol, srk) * P.trim;
    const float ey = det::sample_blue_noise(x, y, (int)fc.num_frames, 1, sobol, srk) * P.trim;
    const V3    Wh = importance_sample_ggx(ex, ey, N, roughness);
    r.d = reflect(det::scale(Wo, -1.0f), Wh);
    return RG_TRACE;
}

struct QRayC { float ox, oy, oz; uint32_t pix; float dx, dy, dz, pad; };

__global__ void __launch_bounds__(RA_WARPS * 32, 3) k_refl_trace(GBufLevelDev g, BvhDev bvh, FrameConsts fc, hr_ddgi_uniforms d, gi::AtlasDev at, ReflTraceParams P,
                                                              const uint8_t* __restrict__ sobol, const uint8_t* __restrict__ srk, uint2* __restrict__ out,
                                                              float4* __restrict__ hits, unsigned int* __restrict__ work_counter)
{
    extern __shared__ __align__(16) unsigned char ra_smem[];
    QRayC(*s_queue)[RA_QUEUE]     = reinterpret_cast<QRayC(*)[RA_QUEUE]>(ra_smem);
    int(*s_stack)[RA_WARPS * 32]  = reinterpret_cast<int(*)[RA_WARPS * 32]>(ra_smem + sizeof(QRayC) * RA_WARPS * RA_QUEUE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
    const int MW = (g.W + 7) >> 3, SBW = (MW + 3) >> 2;
    const int mrow0 = P.row0 >> 2, mrow1 = (P.row1 + 3) >> 2;
    const int n_chunks_mine = P.chunk_stride > 1 ? (((g.H + 7) >> 3) - P.chunk_first + P.chunk_stride - 1) / P.chunk_stride : 0;
    const int n_sb = P.chunk_stride > 1 ? SBW * 2 * n_chunks_mine : SBW * (mrow1 - mrow0);
    const uint32_t lt_mask = (1u << lane) - 1u;
    QRayC* q = s_queue[warp];

    for (;;)
    {
        int sb = 0;
        if (lane == 0) sb = (int)atomicAdd(work_counter, 1u);
        sb = __shfl_sync(0xFFFFFFFFu, sb, 0);
        if (sb >= n_sb) break;
        const int jr = sb / SBW, mx0 = (sb % SBW) * 4; // job row: a mask row (4 pixel rows) of the row range, or of this rank's chunk list
        const int my = P.chunk_stride > 1 ? 2 * (P.chunk_first + (jr >> 1) * P.chunk_stride) + (jr & 1) : mrow0 + jr;
        // ---- ray generation + compaction ----------------------------------------------------------------------------------
        int count = 0;
#pragma unroll 1
        for (int w = 0; w < 4; w++)
        {
            const int x = (mx0 + w) * 8 + (lane & 7), y = my * 4 + (lane >> 3);
            bool  need = false;
            QRayC qr;
            if (x < g.W && y < g.H && (P.chunk_stride > 1 || (y >= P.row0 && y < P.row1)))
            {
                const size_t idx = (size_t)y * g.W + x;
                Ray r;
                V3  Pw, Wo, N;
                const int kind = refl_ray_gen(g, fc, P, sobol, srk, x, y, r, Pw, Wo, N);
                if (kind == RG_TRACE)
                {
                    need  = true;
                    qr.ox = r.o.x; qr.oy = r.o.y; qr.oz = r.o.z; qr.dx = r.d.x; qr.dy = r.d.y; qr.dz = r.d.z;
                    qr.pix = (uint32_t)(w * 32 + lane);
                    qr.pad = 0.0f;
                }
                else
                {
                    float3 color = make_float3(0.0f, 0.0f, 0.0f);
                    if (kind == RG_DDGI)
                    {
                        using namespace gi;
                        const V3 R = reflect(det::scale(Wo, -1.0f), N);
                        color      = sample_irradiance(d, at, to_f3(Pw), to_f3(R), to_f3(Wo)) * P.rough_ddgi_intensity;
                    }
                    out[idx]  = pack_h4(fminf(color.x, 0.7f), fminf(color.y, 0.7f), fminf(color.z, 0.7f), -1.0f);
                    hits[idx] = make_float4(0.0f, __uint_as_float(HIT_NO_RAY), 0.0f, 0.0f);
                }
            }
            const uint32_t b = __ballot_sync(0xFFFFFFFFu, need);
            if (need) q[count + __popc(b & lt_mask)] = qr;
            count += __popc(b);
        }
        __syncwarp();
        count_rays(fc.ray_ctr, 0, lane == 0 ? (uint32_t)count : 0u);
        // ---- closest-hit traversal with dynamic refill ---------------------------------------------------------------------
        int       head  = 0;
        bool      valid = false;
        Ray       ray;
        SlabSetup ss;
        int       node = SENTINEL, sp = 0, ovf[STACK_SIZE - RA_SM_STACK];
        uint32_t  pix = 0, best_prim = HIT_MISS;
        float     best_t = 0.0f, best_u = 0.0f, best_v = 0.0f;
        ray.tmin = 0.001f;
        ray.tmax = 10000.0f;
        for (;;)
        {
            const uint32_t idle = __ballot_sync(0xFFFFFFFFu, !valid);
            if (idle)
            {
                if (!valid)
                {
                    const int mine = head + __popc(idle & lt_mask);
                    if (mine < count)
                    {
                        const QRayC r = q[mine];
                        ray.o = det::mk(r.ox, r.oy, r.oz); ray.d = det::mk(r.dx, r.dy, r.dz);
                        pix   = r.pix;
                        ss    = slab_setup(ray);
                        node  = 0;
                        sp    = 0;
                        best_t = ray.tmax; best_prim = HIT_MISS; best_u = best_v = 0.0f;
                        valid = true;
                    }
                }
                head += __popc(idle);
            }
            if (!__any_sync(0xFFFFFFFFu, valid)) break;
#pragma unroll 1
            for (int it = 0; it < RA_REFILL_STEPS; it++)
            {
                while (valid && node >= 0 && node != SENTINEL)
                {
                    bool  h0, h1;
                    float t0, t1;
                    int   c0, c1;
                    node_test(bvh.nodes, node, ss, ray.tmin, best_t, h0, h1, t0, t1, c0, c1);
                    if (!h0 && !h1)
                    {
                        if (sp == 0) node = SENTINEL;
                        else { --sp; node = sp < RA_SM_STACK ? s_stack[sp][tid] : ovf[sp - RA_SM_STACK]; }
                    }
                    else
                    {
                        node = h0 ? c0 : c1;
                        if (h0 && h1)
                        {
                            if (t1 < t0) { const int tmp = c1; c1 = node; node = tmp; }
                            if (sp < RA_SM_STACK) s_stack[sp][tid] = c1;
                            else if (sp < STACK_SIZE) ovf[sp - RA_SM_STACK] = c1;
                            if (sp < STACK_SIZE) sp++;
                        }
                    }
                }
                if (valid && node < 0)
                {
                    const int leaf  = ~node;
                    const int first = leaf >> 3, cnt = (leaf & 7) + 1;
                    for (int k = 0; k < cnt; k++)
                    {
                        const float4 A = __ldg(bvh.tris + 3ull * (first + k));
                        const float4 B = __ldg(bvh.tris + 3ull * (first + k) + 1);
                        const float4 C = __ldg(bvh.tris + 3ull * (first + k) + 2);
                        float        t, u, v;
                        if (ray_triangle(A, B, C, ray, t, u, v))
                        {
                            const uint32_t prim = __float_as_uint(A.w);
                            if (t < best_t || (t == best_t && prim < best_prim)) { best_t = t; best_prim = prim; best_u = u; best_v = v; }
                        }
                    }
                    if (sp == 0) node = SENTINEL;
                    else { --sp; node = sp < RA_SM_STACK ? s_stack[sp][tid] : ovf[sp - RA_SM_STACK]; }
                }
                if (valid && node == SENTINEL)
                { // traversal finished: publish the hit record of this lane's pixel
                    const int x = (mx0 + (int)(pix >> 5)) * 8 + (int)(pix & 7u), y = my * 4 + (int)((pix & 31u) >> 3);
                    hits[(size_t)y * g.W + x] = make_float4(best_t, __uint_as_float(best_prim), best_u, best_v);
                    valid = false;
                }
                if (__any_sync(0xFFFFFFFFu, !valid)) break; // somebody can refill (or everybody is done)
            }
        }
        __syncwarp();
    }
}

// pass B: 32x8-pixel tile per CTA, hit pixels compacted so that every lane shades
__global__ void __launch_bounds__(256) k_refl_shade(GBufLevelDev g, BvhDev bvh, ShadeDev sd, FrameConsts fc, hr_ddgi_uniforms d, gi::AtlasDev at, ReflTraceParams P,
                                                     const uint8_t* __restrict__ sobol, const uint8_t* __restrict__ srk, const float4* __restrict__ hits,
                                                     uint2* __restrict__ out)
{
    __shared__ uint16_t s_list[256];
    __shared__ int      s_warp_base[9];
    const int    lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int    x0 = blockIdx.x * 32, y0 = P.chunk_stride > 1 ? 8 * (P.chunk_first + (int)blockIdx.y * P.chunk_stride) : P.row0 + blockIdx.y * 8;
    const int    y_end = P.chunk_stride > 1 ? g.H : P.row1;
    const float3 sky = make_float3(P.sky[0], P.sky[1], P.sky[2]);
    {
        const int x = x0 + lane, y = y0 + warp;
        bool      is_hit = false;
        if (x < g.W && y < g.H && y < y_end)
        {
            const size_t   idx  = (size_t)y * g.W + x;
            const uint32_t prim = __float_as_uint(__ldg(reinterpret_cast<const float*>(hits + idx) + 1));
            if (prim == HIT_MISS) out[idx] = pack_h4(fminf(sky.x, 0.7f), fminf(sky.y, 0.7f), fminf(sky.z, 0.7f), -1.0f); // rmiss: colour = sky, ray_length stays -1
            else if (prim != HIT_NO_RAY) is_hit = true;
        }
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, is_hit);
        if (lane == 0) s_warp_base[warp + 1] = __popc(b);
        __syncthreads();
        if (threadIdx.x == 0)
        {
            s_warp_base[0] = 0;
            for (int w = 1; w <= 8; w++) s_warp_base[w] += s_warp_base[w - 1];
        }
        __syncthreads();
        if (is_hit) s_list[s_warp_base[warp] + __popc(b & ((1u << lane) - 1u))] = (uint16_t)threadIdx.x;
        __syncthreads();
    }
    const int n_hits = s_warp_base[8];
    if ((int)threadIdx.x >= n_hits) return;
    const int    t   = s_list[threadIdx.x];
    const int    x = x0 + (t & 31), y = y0 + (t >> 5);
    const size_t idx = (size_t)y * g.W + x;
    const float4 h   = __ldg(hits + idx);
    Ray r;
    V3  Pw, Wo, N;
    refl_ray_gen(g, fc, P, sobol, srk, x, y, r, Pw, Wo, N);
    const float3 color = shade_hit(bvh, sd, fc.light, r, __float_as_uint(h.y), h.z, h.w, false, 0.0f, 0.0f, sky, P.sample_gi == 1, d, at, P.gi_intensity, fc.ray_ctr, P.ibl);
    out[idx] = pack_h4(fminf(color.x, 0.7f), fminf(color.y, 0.7f), fminf(color.z, 0.7f), 0.001f + h.x);
}

// ---------------------------------------------------------------------------------------------------------------------------
// Ground-truth progressive path tracer (SURVEY.md §8 f4): ground_truth/ground_truth_path_trace.{rgen,rchit,rmiss}, host
// src/ground_truth_path_tracer.cpp:44-113.  One jittered primary ray per pixel and frame; closest hit -> direct_lighting with SOFT_SHADOWS +
// RAY_THROUGHPUT + SAMPLE_SKY_LIGHT (rchit:13-16): the punctual light sampled on its disk with its shadow ray, one cosine-lobe sky sample
// with its shadow ray; miss -> the sky colour; running average into an RGBA16F image.  As written in the reference the indirect bounce's
// traceRayEXT is commented out (rchit:92-104) and indirect_lighting returns p_IndirectPayload.L = vec3(0): the image converges to direct +
// sky lighting; max_ray_bounces only gates that dead branch.  The primary ray, the hit and the two shadow rays follow the deterministic chain
// (det_math.cuh): hit primitive and binary visibilities equal the oracle's (oracle/orc_path_trace.cpp) exactly, colours within tolerance.
struct PathTraceParams {
    float    view_inverse[16], proj_inverse[16];
    hr_light light;
    uint32_t num_frames, max_ray_bounces;
    float    roughness_multiplier;
    float    sky[3];
    int      W, H;
    unsigned long long* ray_ctr;
};

__device__ __forceinline__ float4 mat_vec4(const float* M, float x, float y, float z, float w)
{ // mat4 * vec4, row r = ((m0r*x + m1r*y) + m2r*z) + m3r*w (oracle/orc_math.h::mul)
    return make_float4(((M[0] * x + M[4] * y) + M[8] * z) + M[12] * w, ((M[1] * x + M[5] * y) + M[9] * z) + M[13] * w,
                       ((M[2] * x + M[6] * y) + M[10] * z) + M[14] * w, ((M[3] * x + M[7] * y) + M[11] * z) + M[15] * w);
}

// warp = 8x4 pixel block (coherent primary rays), 2-warp CTAs like K12
template <bool TEX>
__global__ void __launch_bounds__(64) k_path_trace(BvhDev bvh, ShadeDev sd, PathTraceParams P, const uint2* __restrict__ prev, uint2* __restrict__ out, uint32_t* __restrict__ out_prim,
                                                   tex::TexDev T)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int x = blockIdx.x * 16 + warp * 8 + (lane & 7), y = blockIdx.y * 4 + (lane >> 3);
    if (x >= P.W || y >= P.H) return;
    const size_t idx = (size_t)y * P.W + x;
    // rgen:56-75
    gi::RNG     rng = gi::rng_init((uint32_t)x, (uint32_t)y, P.num_frames);
    const float j0 = gi::next_float(rng), j1 = gi::next_float(rng);
    const float jx = ((float)x + 0.5f) + j0, jy = ((float)y + 0.5f) + j1;    // pixel_coord + vec2(next_float, next_float)
    const float tx = jx / (float)P.W, ty = jy / (float)P.H;                   // tex_coord
    const float nx = tx * 2.0f - 1.0f, ny = ty * 2.0f - 1.0f;                 // tex_coord_neg_to_pos
    const float4 origin = mat_vec4(P.view_inverse, 0.0f, 0.0f, 0.0f, 1.0f);
    const float4 target = mat_vec4(P.proj_inverse, nx, ny, 1.0f, 1.0f);
    const V3     tn     = det::normalize(det::mk(target.x, target.y, target.z));
    const float4 dir    = mat_vec4(P.view_inverse, tn.x, tn.y, tn.z, 0.0f);
    Ray r;
    r.o = det::mk(origin.x, origin.y, origin.z);
    r.d = det::mk(dir.x, dir.y, dir.z);
    r.tmin = 0.001f;
    r.tmax = 10000.0f;
    const float3 sky = make_float3(P.sky[0], P.sky[1], P.sky[2]);
    float3   L = sky; // rmiss:29-32 at depth 0
    float    t, hu, hv;
    uint32_t prim = 0xFFFFFFFFu;
    count_rays(P.ray_ctr, 0, 1u);
    if (trace_closest(bvh, r, t, prim, hu, hv))
    { // rchit:112-141
        using namespace gi;
        const Surface s  = TEX ? fetch_surface_tex(sd, T, prim, hu, hv) : fetch_surface(sd, prim, hu, hv);
        const float   roughness = s.roughness * P.roughness_multiplier;
        const V3      Wo = det::scale(r.d, -1.0f);
        const float3  F0 = f3(0.04f, 0.04f, 0.04f) * (1.0f - s.metallic) + s.albedo * s.metallic;
        const float3  cd = (s.albedo * (f3(1, 1, 1) - F0)) * (1.0f - s.metallic) + f3(0, 0, 0) * s.metallic;
        const float   r1x = next_float(rng), r1y = next_float(rng); // next_vec2: the light's disk sample
        const float   r2x = next_float(rng), r2y = next_float(rng); // next_vec2: the sky sample
        // direct_lighting, lighting.glsl:117-196 with SOFT_SHADOWS, RAY_THROUGHPUT (T = 1 at depth 0), SAMPLE_SKY_LIGHT
        float3 Lo = f3(0, 0, 0);
        Ray    sr;
        sr.o    = det::add(s.P, det::scale(s.N, 0.1f));
        sr.tmin = 0.01f;
        {
            const hr_light& light = P.light;
            const float3    Li = make_float3(light.data2[0] * light.data0[3], light.data2[1] * light.data0[3], light.data2[2] * light.data0[3]);
            V3    Wi;
            float t_max, att;
            det::fetch_light_properties_shadow(light, s.P, s.N, r1x, r1y, Wi, t_max, att);
            const V3 Wh = det::normalize(det::add(Wo, Wi));
            if (att > 0.0f)
            {
                sr.d    = Wi;
                sr.tmax = t_max;
                count_rays(P.ray_ctr, 1, 1u);
                att *= trace_any(bvh, sr) ? 0.0f : 1.0f;
            }
            Lo = Lo + (evaluate_uber_brdf(cd, roughness, s.N, F0, Wo, Wh, Wi) * att) * Li;
        }
        {
            const V3 Wi = det::sample_cosine_lobe(s.N, r2x, r2y);
            const V3 Wh = det::normalize(det::add(Wo, Wi));
            sr.d    = Wi;
            sr.tmax = 10000.0f;
            count_rays(P.ray_ctr, 1, 1u);
            const float vis = trace_any(bvh, sr) ? 0.0f : 1.0f;
            Lo = Lo + evaluate_uber_brdf(cd, roughness, s.N, F0, Wo, Wh, Wi) * (sky * vis);
        }
        L = Lo; // + indirect_lighting(...) = vec3(0): the bounce is commented out in the reference (rchit:92-106)
    }
    // rgen:94-111: clamp to RADIANCE_CLAMP_COLOR = 1, then the running average the reference writes (weight 1 / num_frames, not 1 / (n + 1))
    const float3 c = make_float3(fminf(L.x, 1.0f), fminf(L.y, 1.0f), fminf(L.z, 1.0f));
    float3 o = c;
    if (P.num_frames != 0)
    {
        const uint2  pw = __ldg(prev + idx);
        const float2 p01 = __half22float2(*reinterpret_cast<const __half2*>(&pw.x)), p2 = __half22float2(*reinterpret_cast<const __half2*>(&pw.y));
        const float  n = (float)P.num_frames;
        o = make_float3(p01.x + (c.x - p01.x) / n, p01.y + (c.y - p01.y) / n, p2.x + (c.z - p2.x) / n);
    }
    out[idx] = pack_h4(o.x, o.y, o.z, 1.0f);
    out_prim[idx] = prim;
}

ShadeDev shade_view(const hr_scene* sc)
{
    ShadeDev s;
    s.verts     = sc->d_tri_verts;
    s.vnormals  = sc->d_vnormals;
    s.prim_mat  = sc->d_prim_mat;
    s.materials = sc->d_materials;
    return s;
}

} // namespace

void launch_ddgi_ray_trace(const hr_scene* sc, const hr_ddgi_uniforms& d, const void* irr_prev, const void* depth_prev, const hr_light& light, const float* rot16,
                           uint32_t num_frames, uint32_t infinite_bounces, float gi_intensity, const float* sky3, int probe0, int probe1, void* radiance,
                           void* dirdepth, unsigned long long* ray_ctr, cudaStream_t st)
{
    if (probe1 <= probe0) return;
    GiTraceParams P;
    memcpy(P.rot, rot16, 64);
    P.num_frames = num_frames; P.infinite_bounces = infinite_bounces; P.gi_intensity = gi_intensity;
    P.sky[0] = sky3[0]; P.sky[1] = sky3[1]; P.sky[2] = sky3[2];
    P.probe0 = probe0; P.probe1 = probe1;
    P.ray_ctr = ray_ctr;
    gi::AtlasDev at { (const uint2*)irr_prev, (const uint32_t*)depth_prev };
    int threads = d.rays_per_probe < 256 ? ((d.rays_per_probe + 31) / 32) * 32 : 256;
    if (sc->tex.n_textures > 0) k_ddgi_ray_trace<true><<<probe1 - probe0, threads, 0, st>>>(hr_bvh_view(sc), shade_view(sc), d, at, light, P, (uint2*)radiance, (uint2*)dirdepth, sc->tex);
    else k_ddgi_ray_trace<false><<<probe1 - probe0, threads, 0, st>>>(hr_bvh_view(sc), shade_view(sc), d, at, light, P, (uint2*)radiance, (uint2*)dirdepth, sc->tex);
}

// 0 (default) = fused kernel (one warp per 8x4 block: ray generation, closest hit, hit shading incl. its shadow ray);
// 1 = wavefront (k_refl_trace + k_refl_shade): 3.74 ms vs 2.63 per 4K frame (config 3, H100 SXM 80 GB, 700 W power limit) — the refill keeps lanes supplied with rays, but
// lane-level divergence inside the while-while traversal (about half of the 32 lanes active in both forms) is what costs, and
// the 56 KB queue / stack footprint per CTA takes L1 away from the BVH.
// hr_debug_set key 7.
int g_hr_refl_trace_impl = 0;
// hr_debug_set key 10: resident 2-warp CTAs per SM the fused kernel's registers are tuned for (18 = 56 registers = default; 20 = 48;
// 16 = 64; 14 = 72; 12 = 80).  Config 3 at 4K on an H100 SXM 80 GB (400 W power limit), K12 per frame: 12 -> 3.15 ms, 14 -> 3.00,
// 16 -> 2.94, 18 -> 2.91, 20 -> 2.91: the kernel is latency-bound, resident warps buy more than registers (and than the spills
// the smaller register budgets cost).
int g_hr_refl_trace_minb = 18;

void launch_reflections_ray_trace(const hr_scene* sc, const GBufLevelDev& g, const FrameConsts& fc, const hr_ddgi_uniforms* d, const void* irr, const void* depth,
                                  float bias, float trim, int sample_gi, int approximate_with_ddgi, float gi_intensity, float rough_ddgi_intensity, const float* sky3,
                                  const uint8_t* sobol, const uint8_t* srk, void* out, void* hits, int row0, int row1, int chunk_first, int chunk_stride,
                                  int spp, const void* brdf_lut, float ibl_intensity, cudaStream_t st)
{
    const int n_chunks_mine = chunk_stride > 1 ? (((g.H + 7) / 8) - chunk_first + chunk_stride - 1) / chunk_stride : 0;
    if (chunk_stride > 1 ? n_chunks_mine <= 0 : row1 <= row0) return;
    ReflTraceParams P { bias, trim, sample_gi, approximate_with_ddgi, gi_intensity, rough_ddgi_intensity, { sky3[0], sky3[1], sky3[2] }, row0, row1, chunk_first, chunk_stride, spp,
                        IblDev { (const uint32_t*)brdf_lut, ibl_intensity } };
    hr_ddgi_uniforms du;
    memset(&du, 0, sizeof(du));
    if (d) du = *d;
    gi::AtlasDev at { (const uint2*)irr, (const uint32_t*)depth };
    const bool textured = sc->tex.n_textures > 0; // material textures: the TEX instantiations of the fused kernel (the wavefront variant has none)
    if (g_hr_refl_trace_impl == 1 && hits && row0 % 4 == 0 && spp <= 1 && !textured) // spp > 1 runs on the fused kernel
    {
        static unsigned int* counter[64] = {};
        static int           ctas[64]    = {};
        const size_t smem = sizeof(QRayC) * RA_WARPS * RA_QUEUE + sizeof(int) * RA_SM_STACK * RA_WARPS * 32;
        int dev = 0;
        cudaGetDevice(&dev);
        dev &= 63;
        if (!counter[dev])
        {
            cudaMalloc(&counter[dev], 64 * sizeof(unsigned int)); // one counter per stream slot would be needed for concurrent reflections passes; one pass per device here
            cudaFuncSetAttribute(k_refl_trace, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            int sms = 132, per_sm = 1;
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_refl_trace, RA_WARPS * 32, smem);
            ctas[dev] = sms * (per_sm > 0 ? per_sm : 1);
        }
        cudaMemsetAsync(counter[dev], 0, sizeof(unsigned int), st);
        k_refl_trace<<<ctas[dev], RA_WARPS * 32, smem, st>>>(g, hr_bvh_view(sc), fc, du, at, P, sobol, srk, (uint2*)out, (float4*)hits, counter[dev]);
        dim3 gridb((g.W + 31) / 32, chunk_stride > 1 ? n_chunks_mine : (row1 - row0 + 7) / 8);
        k_refl_shade<<<gridb, 256, 0, st>>>(g, hr_bvh_view(sc), shade_view(sc), fc, du, at, P, sobol, srk, (const float4*)hits, (uint2*)out);
        return;
    }
    dim3 grid((g.W + 15) / 16, chunk_stride > 1 ? 2 * n_chunks_mine : (row1 - row0 + 3) / 4);
    const tex::TexDev& T = sc->tex;
#define HR_K12_ARGS g, hr_bvh_view(sc), shade_view(sc), fc, du, at, P, sobol, srk, (uint2*)out, T
    if (textured)
    {
        if (spp > 1) k_reflections_ray_trace<true, 8, true><<<grid, 64, 0, st>>>(HR_K12_ARGS);
        else k_reflections_ray_trace<false, 18, true><<<grid, 64, 0, st>>>(HR_K12_ARGS);
    }
    else if (spp > 1) k_reflections_ray_trace<true, 8, false><<<grid, 64, 0, st>>>(HR_K12_ARGS);
    else if (g_hr_refl_trace_minb == 14) k_reflections_ray_trace<false, 14, false><<<grid, 64, 0, st>>>(HR_K12_ARGS);
    else if (g_hr_refl_trace_minb == 12) k_reflections_ray_trace<false, 12, false><<<grid, 64, 0, st>>>(HR_K12_ARGS);
    else if (g_hr_refl_trace_minb == 16) k_reflections_ray_trace<false, 16, false><<<grid, 64, 0, st>>>(HR_K12_ARGS);
    else if (g_hr_refl_trace_minb == 20) k_reflections_ray_trace<false, 20, false><<<grid, 64, 0, st>>>(HR_K12_ARGS);
    else k_reflections_ray_trace<false, 18, false><<<grid, 64, 0, st>>>(HR_K12_ARGS);
#undef HR_K12_ARGS
}

void launch_path_trace(const hr_scene* sc, const hr_frame* f, int W, int H, uint32_t num_frames, uint32_t max_ray_bounces, float roughness_multiplier, const float* sky3,
                       const void* prev, void* out, uint32_t* out_prim, unsigned long long* ray_ctr, cudaStream_t st)
{
    PathTraceParams P;
    memcpy(P.view_inverse, f->ubo.view_inverse, 64);
    memcpy(P.proj_inverse, f->ubo.proj_inverse, 64);
    P.light = f->ubo.light;
    P.num_frames = num_frames; P.max_ray_bounces = max_ray_bounces; P.roughness_multiplier = roughness_multiplier;
    P.sky[0] = sky3[0]; P.sky[1] = sky3[1]; P.sky[2] = sky3[2];
    P.W = W; P.H = H;
    P.ray_ctr = ray_ctr;
    dim3 grid((W + 15) / 16, (H + 3) / 4);
    if (sc->tex.n_textures > 0) k_path_trace<true><<<grid, 64, 0, st>>>(hr_bvh_view(sc), shade_view(sc), P, (const uint2*)prev, (uint2*)out, out_prim, sc->tex);
    else k_path_trace<false><<<grid, 64, 0, st>>>(hr_bvh_view(sc), shade_view(sc), P, (const uint2*)prev, (uint2*)out, out_prim, sc->tex);
}
