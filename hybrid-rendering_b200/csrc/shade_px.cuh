// shade_px.cuh — hit shading of the closest-hit ray traces (rt_shade.cu: K12, K18, the path tracer) and of the reflections
// reference (reference.cu): fetch_triangle / interpolated_vertex (scene_descriptor_set.glsl:117-160), direct_lighting
// (lighting.glsl:117-196) with its shadow ray, evaluate_uber_brdf (brdf.glsl:130-142), DDGI infinite bounce (gi_common.glsl:188-320),
// the GGX lobe sample (reflections_ray_trace.rgen:78-105).  Compile with -fmad=false (rt_shade.cu, BUILD NOTE).
// Everything here is in an anonymous namespace: each .cu file that includes it compiles its own copy (direct_lighting and
// indirect_diffuse are not inlined, so each file has its own out-of-line instance).
#pragma once
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
        // evaluated before the shadow ray: only brdf, att and Li stay live across its traversal, not the surface and the directions
        const float3 brdf = evaluate_uber_brdf(diffuse_color, roughness, N, F0, Wo, Wh, Wi);
        if (att > 0.0f)
        {
            sr.d    = Wi;
            sr.tmax = t_max;
            count_rays(ray_ctr, 1, 1u);
            att *= trace_any(bvh, sr) ? 0.0f : 1.0f;
        }
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
// instantiations of the shading kernels (rt_shade.cu, reference.cu) call these; their untextured instantiations do not.
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

// The DDGI branch of K12's sample (roughness > 0.75 with approximate_with_ddgi), shared by k_reflections_ray_trace and the reflections
// reference (reference.cu): the probe irradiance in the mirror direction.
__device__ __forceinline__ float3 refl_ddgi_sample(const hr_ddgi_uniforms& d, const gi::AtlasDev& at, V3 Pw, V3 N, V3 Wo, float rough_ddgi_intensity)
{
    using namespace gi;
    const V3 R = reflect(det::scale(Wo, -1.0f), N);
    return sample_irradiance(d, at, to_f3(Pw), to_f3(R), to_f3(Wo)) * rough_ddgi_intensity;
}

// K12's launch parameters, which the reflections reference (reference.cu) takes too so that both trace the same sample: the sample
// parameters of a reflections render (hr_reflections_params with the DDGI terms refl_gi decided), the rows and spp, the DDGI uniforms
// (zero without a DDGI grid) and atlases, and whether the kernels need the DDGI and IBL terms (GI).  The field order is K12's.
struct ReflTraceParams { float bias, trim; int sample_gi, approximate_with_ddgi; float gi_intensity, rough_ddgi_intensity; float sky[3]; RowSet rows;
                         int spp; IblDev ibl; };
struct ReflLaunch { ReflTraceParams P; hr_ddgi_uniforms d; gi::AtlasDev at; bool gi; };
inline ReflLaunch refl_launch(const ReflGi& gi, const hr_reflections_params& prm, const void* brdf_lut, RowSet rows)
{
    ReflLaunch L {}; // no DDGI grid: zero uniforms
    L.P = { prm.bias, prm.trim, gi.sample_gi, gi.approx, prm.gi_intensity, prm.rough_ddgi_intensity, { prm.sky_color[0], prm.sky_color[1], prm.sky_color[2] },
            rows, prm.spp > 1 ? prm.spp : 1, IblDev { (const uint32_t*)brdf_lut, prm.ibl_indirect_specular_intensity } };
    if (gi.d) L.d = *gi.d;
    L.at = { (const uint2*)gi.irr, (const uint32_t*)gi.dep };
    L.gi = gi.sample_gi == 1 || gi.approx == 1;
    return L;
}

inline ShadeDev shade_view(const hr_scene* sc)
{
    ShadeDev s;
    s.verts     = sc->d_tri_verts;
    s.vnormals  = sc->d_vnormals;
    s.prim_mat  = sc->d_prim_mat;
    s.materials = sc->d_materials;
    return s;
}

} // namespace
