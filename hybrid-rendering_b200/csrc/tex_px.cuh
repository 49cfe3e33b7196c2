// tex_px.cuh — material textures at a hit point: fetch_albedo / fetch_roughness / fetch_metallic of the reference
// (src/shaders/scene_descriptor_set.glsl:180-218) with the bindless texture array replaced by one packed RGBA8 buffer.
//   texture(s_Textures[i], uv) in a ray-tracing / compute stage = textureLod(.., 0): base level, bilinear, REPEAT addressing
//   (dw::Material::m_common_sampler, external/dwSampleFramework/src/material.cpp:210-228); albedo images are sRGB (material.cpp:114:
//   load_image(.., true)), so their texels are decoded to linear BEFORE filtering, like the sampler hardware does; UNORM8 -> float = c / 255.
//   texcoord = v0.uv * b.x + v1.uv * b.y + v2.uv * b.z (interpolated_vertex, scene_descriptor_set.glsl:141).
// __host__ __device__ like post_px.cuh: the TEX instantiations of the hit-shading kernels (rt_shade.cu, gbuffer.cu, both built with
// -fmad=false) call these functions, tests/hostemu builds them for the CPU and the oracle (oracle/orc_shading.h) restates them
// independently.  Texel SELECTION (floor of u * W - 0.5, wrap) is bit-specified; the filtered colour is tolerance-checked downstream.
#pragma once
#include <math.h>
#include <stdint.h>
#ifdef __CUDACC__
#define HR_TEX_HD __host__ __device__ __forceinline__
#else
#define HR_TEX_HD inline
#endif

namespace tex {

struct MatTex { // one per material: texture index or -1 (Material::texture_indices0 / 1, scene_descriptor_set.glsl:84-93) = hr_material_textures + padding
    int32_t albedo, normal, roughness, roughness_channel, metallic, metallic_channel, emissive, _pad;
};
struct TexDesc { uint32_t offset; int32_t width, height, srgb; }; // texels [offset, offset + width * height) of TexDev::texels
struct TexDev {                // device view of a scene's textures (hr_scene_set_textures); n_textures == 0: none
    const uint32_t* texels;    // every texture as RGBA8 (r in the low byte); 1- and 2-channel images were expanded to (r, 0, 0, 255) / (r, g, 0, 255)
    const TexDesc*  desc;
    const MatTex*   mat;       // n_materials entries
    const float*    vuv;       // 6 floats per primitive (primitive order): uv of the three vertices
    const float*    srgb_lut;  // 256 floats: sRGB byte -> linear
    int32_t         n_textures;
    const float*    vtb;       // 18 floats per primitive: world-space unit tangents of the three corners, then their bitangents; null when no
                               // material binds a normal map
};

struct RGBA { float r, g, b, a; };

HR_TEX_HD int tex_f2i(float f)
{ // cvt.rzi.s32.f32: toward zero, saturating, NaN -> 0
#ifdef __CUDA_ARCH__
    return __float2int_rz(f);
#else
    if (!(f == f)) return 0;
    if (f >= 2147483648.0f) return 2147483647;
    if (f <= -2147483648.0f) return (int)0x80000000;
    return (int)f;
#endif
}
HR_TEX_HD int next_texel(int i)
{ // i + 1; a saturated x0 = INT_MAX wraps to INT_MIN like the device's 32-bit add (signed overflow is undefined in host C++)
#ifdef __CUDA_ARCH__
    return i + 1;
#else
    return (int)((uint32_t)i + 1u);
#endif
}
HR_TEX_HD int wrap_repeat(int i, int n) { const int m = i % n; return m < 0 ? m + n : m; } // VK_SAMPLER_ADDRESS_MODE_REPEAT

HR_TEX_HD RGBA fetch(const TexDev& T, const TexDesc& d, int x, int y)
{
    const uint32_t t = T.texels[d.offset + (uint32_t)wrap_repeat(y, d.height) * (uint32_t)d.width + (uint32_t)wrap_repeat(x, d.width)];
    RGBA c;
    if (d.srgb) { c.r = T.srgb_lut[t & 255u]; c.g = T.srgb_lut[(t >> 8) & 255u]; c.b = T.srgb_lut[(t >> 16) & 255u]; }
    else { c.r = (float)(t & 255u) / 255.0f; c.g = (float)((t >> 8) & 255u) / 255.0f; c.b = (float)((t >> 16) & 255u) / 255.0f; }
    c.a = (float)(t >> 24) / 255.0f; // alpha is never sRGB-encoded
    return c;
}

// textureLod(s_Textures[ti], (u, v), 0)
HR_TEX_HD RGBA sample(const TexDev& T, int ti, float u, float v)
{
    const TexDesc d = T.desc[ti];
    const float x = u * (float)d.width - 0.5f, y = v * (float)d.height - 0.5f;
    const float fx0 = floorf(x), fy0 = floorf(y);
    const float fx = x - fx0, fy = y - fy0;
    const int   x0 = tex_f2i(fx0), y0 = tex_f2i(fy0);
    const int   x1 = next_texel(x0), y1 = next_texel(y0);
    const RGBA  a = fetch(T, d, x0, y0), b = fetch(T, d, x1, y0), c = fetch(T, d, x0, y1), e = fetch(T, d, x1, y1);
    const float wx0 = 1.0f - fx, wy0 = 1.0f - fy;
    RGBA r;
    r.r = (a.r * wx0 + b.r * fx) * wy0 + (c.r * wx0 + e.r * fx) * fy;
    r.g = (a.g * wx0 + b.g * fx) * wy0 + (c.g * wx0 + e.g * fx) * fy;
    r.b = (a.b * wx0 + b.b * fx) * wy0 + (c.b * wx0 + e.b * fx) * fy;
    r.a = (a.a * wx0 + b.a * fx) * wy0 + (c.a * wx0 + e.a * fx) * fy;
    return r;
}
HR_TEX_HD float channel(const RGBA& c, int ch) { return ch == 0 ? c.r : (ch == 1 ? c.g : (ch == 2 ? c.b : c.a)); }

// Overrides the material constants (albedo rgb, roughness already clamped to MIN_ROUGHNESS, metallic) of material `mat` with its textures
// at the hit point of primitive `prim` with barycentrics (b0, b1, b2) = (1 - u - v, u, v).
HR_TEX_HD void material_at_hit(const TexDev& T, uint32_t mat, uint32_t prim, float b0, float b1, float b2, float& ar, float& ag, float& ab, float& roughness, float& metallic)
{
    const MatTex m = T.mat[mat];
    if (m.albedo < 0 && m.roughness < 0 && m.metallic < 0) return;
    const float* q = T.vuv + 6ull * prim;
    const float  u = (q[0] * b0 + q[2] * b1) + q[4] * b2, v = (q[1] * b0 + q[3] * b1) + q[5] * b2;
    if (m.albedo >= 0) { const RGBA c = sample(T, m.albedo, u, v); ar = c.r; ag = c.g; ab = c.b; }                               // fetch_albedo :180-186
    if (m.roughness >= 0) roughness = fmaxf(channel(sample(T, m.roughness, u, v), m.roughness_channel), 0.1f);                    // fetch_roughness :200-208 (MIN_ROUGHNESS)
    if (m.metallic >= 0) metallic = channel(sample(T, m.metallic, u, v), m.metallic_channel);                                     // fetch_metallic :212-218
}

// fetch_normal + get_normal_from_map (scene_descriptor_set.glsl:164-195): the interpolated unit normal (nx, ny, nz) is replaced by
// normalize(TBN * normalize(texel.rgb * 2 - 1)), TBN = (normalize(T), normalize(B), normalize(N)).  The hit shaders pass the TANGENT as bitangent
// (reflections_ray_trace.rchit:134, gi_ray_trace.rchit:112, ground_truth_path_trace.rchit:131: fetch_normal(material, vertex.tangent.xyz,
// vertex.tangent.xyz, ...)) — tangent_as_bitangent = true reproduces that; the G-buffer pass passes the real bitangent (g_buffer.frag:100).
// The result feeds shadow-ray origins and N.L tests: written in the deterministic chain's operation order (dot = (xx + yy) + zz,
// normalize = v * (1 / sqrt(dot)), mat3 * vec3 = (c0 * x + c1 * y) + c2 * z); this header is only compiled without FMA contraction.
HR_TEX_HD void normalize3(float& x, float& y, float& z)
{
    const float inv = 1.0f / sqrtf((x * x + y * y) + z * z);
    x = x * inv; y = y * inv; z = z * inv;
}
HR_TEX_HD void normal_at_hit(const TexDev& T, uint32_t mat, uint32_t prim, float b0, float b1, float b2, bool tangent_as_bitangent, float& nx, float& ny, float& nz)
{
    const MatTex m = T.mat[mat];
    if (m.normal < 0 || !T.vtb) return;
    const float* q = T.vuv + 6ull * prim;
    const float  u = (q[0] * b0 + q[2] * b1) + q[4] * b2, v = (q[1] * b0 + q[3] * b1) + q[5] * b2;
    const RGBA   c = sample(T, m.normal, u, v);
    float tx_ = c.r * 2.0f - 1.0f, ty_ = c.g * 2.0f - 1.0f, tz_ = c.b * 2.0f - 1.0f; // texel.rgb * 2.0 - 1.0
    normalize3(tx_, ty_, tz_);
    const float* t = T.vtb + 18ull * prim; // interpolated_vertex :143-144: normalize(t0 * b.x + t1 * b.y + t2 * b.z)
    float Tx = (t[0] * b0 + t[3] * b1) + t[6] * b2, Ty = (t[1] * b0 + t[4] * b1) + t[7] * b2, Tz = (t[2] * b0 + t[5] * b1) + t[8] * b2;
    normalize3(Tx, Ty, Tz);
    float Bx = Tx, By = Ty, Bz = Tz;
    if (!tangent_as_bitangent)
    {
        Bx = (t[9] * b0 + t[12] * b1) + t[15] * b2; By = (t[10] * b0 + t[13] * b1) + t[16] * b2; Bz = (t[11] * b0 + t[14] * b1) + t[17] * b2;
        normalize3(Bx, By, Bz);
    }
    // mat3 TBN = mat3(normalize(tangent), normalize(bitangent), normalize(normal)): the arguments arrive normalised (interpolated_vertex /
    // g_buffer.frag:100) and are normalised AGAIN here, as the shader does — a second normalisation can move the last bit
    normalize3(Tx, Ty, Tz);
    normalize3(Bx, By, Bz);
    float Nx = nx, Ny = ny, Nz = nz;
    normalize3(Nx, Ny, Nz);
    float rx = (Tx * tx_ + Bx * ty_) + Nx * tz_, ry = (Ty * tx_ + By * ty_) + Ny * tz_, rz = (Tz * tx_ + Bz * ty_) + Nz * tz_;
    normalize3(rx, ry, rz);
    nx = rx; ny = ry; nz = rz;
}

} // namespace tex
