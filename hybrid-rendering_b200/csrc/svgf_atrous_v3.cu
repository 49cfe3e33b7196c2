// svgf_atrous_v3.cu — shadows a-trous (K4+K5, shadows_denoise_atrous.comp:94-174) on pixel pairs (atrous_pairs.cuh).
//
// Six staged planes: nx, ny, nz, z*log2e/sigma, visibility, variance.  The visibility is the one colour channel and also the
// luminance the colour weight compares.
#include "atrous_pairs.cuh"

namespace {

using namespace gf;

struct V3Params {
    int   W, H;
    float c_sigma;   // log2(e) / sigma_depth
    float c_phi0;    // -log2(e) / phi_visibility
    float power;
    int   row0, row1;
};

struct ShadowsPass {
    using In = uint32_t; using Out = uint32_t; using Params = V3Params;
    static constexpr int  NPL = 6, NC = 1;
    static constexpr bool COPY_EMPTY_CTA = false; // a CTA without a flagged tile stages nothing and writes zeros

    // Stage the texel pair (px, px+1) of row py (px even) at region index ri (even): decoded normal, scaled linear depth, visibility,
    // variance; zeros outside the image.
    static __device__ __forceinline__ void stage(const GBufLevelDev& g, const uint32_t* __restrict__ in, float c_sigma, int px, int py, int W, int H, int ri, float* s, int PL)
    {
        float2 nx = make_float2(0.0f, 0.0f), ny = nx, nz = nx, zs = nx, vi = nx, va = nx;
        if (px >= 0 && py >= 0 && px < W && py < H)
        {
            const size_t pi = (size_t)py * W + px;
            const uint4  a  = __ldg(reinterpret_cast<const uint4*>(g.gb2 + pi)); // two RGBA16F texels: .x / .z hold the oct normals
            const uint4  b  = __ldg(reinterpret_cast<const uint4*>(g.gb3 + pi)); // .y / .w hold (mesh id, linear z)
            const uint2  c  = __ldg(reinterpret_cast<const uint2*>(in + pi));    // two RG16F texels (visibility, variance)
            const float2 e0 = h2_to_f2(a.x), e1 = h2_to_f2(a.z);
            const float3 n0 = octohedral_to_direction(e0.x, e0.y), n1 = octohedral_to_direction(e1.x, e1.y);
            const float2 i0 = h2_to_f2(c.x), i1 = h2_to_f2(c.y);
            nx = make_float2(n0.x, n1.x); ny = make_float2(n0.y, n1.y); nz = make_float2(n0.z, n1.z);
            zs = make_float2(h2_to_f2(b.y).y * c_sigma, h2_to_f2(b.w).y * c_sigma);
            vi = make_float2(i0.x, i1.x); va = make_float2(i0.y, i1.y);
        }
        float* p = s + ri;
        *reinterpret_cast<float2*>(p) = nx; p += PL;
        *reinterpret_cast<float2*>(p) = ny; p += PL;
        *reinterpret_cast<float2*>(p) = nz; p += PL;
        *reinterpret_cast<float2*>(p) = zs; p += PL;
        *reinterpret_cast<float2*>(p) = vi; p += PL;
        *reinterpret_cast<float2*>(p) = va;
    }

    static __device__ __forceinline__ float2 side_var(const uint32_t* __restrict__ in, size_t pi)
    {
        const uint2 w = __ldg(reinterpret_cast<const uint2*>(in + pi));
        return make_float2(h2_to_f2(w.x).y, h2_to_f2(w.y).y);
    }

    template <bool ALIGNED_X>
    static __device__ __forceinline__ void filter_store(const GBufLevelDev&, const V3Params& P, const PairTaps& t, uint32_t* __restrict__ out, size_t idx, bool has1, bool flagged)
    {
        if (!flagged)
        {
            out[idx] = 0u;
            if (has1) out[idx + 1] = 0u;
            return;
        }
        const PairSum<1> f  = filter_pair<1, 4, ALIGNED_X>(t, P.c_phi0); // luminance = visibility
        float2           o0 = f.c[0];
        if (P.power != 0.0f) { o0.x = pow_pos(o0.x, P.power); o0.y = pow_pos(o0.y, P.power); }
        // sky pixels (linear z < 0) pass the input through
        const float2   zs = ld_pair(t.s + 3 * t.PL, t.ci, true), vi = ld_pair(t.s + 4 * t.PL, t.ci, true), va = ld_pair(t.s + 5 * t.PL, t.ci, true);
        const uint32_t r0 = zs.x < 0.0f ? f2_to_h2(vi.x, va.x) : f2_to_h2(o0.x, f.v.x);
        const uint32_t r1 = zs.y < 0.0f ? f2_to_h2(vi.y, va.y) : f2_to_h2(o0.y, f.v.y);
        if (has1) *reinterpret_cast<uint2*>(out + idx) = make_uint2(r0, r1); // idx even (W even is required by the launcher)
        else out[idx] = r0;
    }
};

template <int STEP>
__global__ void __launch_bounds__(256) k_atrous_v3(GBufLevelDev g, const uint32_t* __restrict__ in, const uint8_t* __restrict__ tile_flags, V3Params P,
                                                    uint32_t* __restrict__ out)
{
    atrous_dense<ShadowsPass, STEP>(g, in, tile_flags, P, out);
}

template <int STEP>
__global__ void __launch_bounds__(256) k_atrous_v3s(GBufLevelDev g, const uint32_t* __restrict__ in, const uint8_t* __restrict__ tile_flags, V3Params P,
                                                     uint32_t* __restrict__ out)
{
    atrous_interleaved<ShadowsPass, STEP>(g, in, tile_flags, P, out);
}

template <int STEP>
using Dense = DenseTile<STEP, ShadowsPass::NPL>;
template <int STEP>
using Interleaved = InterleavedTile<STEP, ShadowsPass::NPL>;

} // namespace

// returns false when this variant does not support the configuration (caller falls back to the scalar kernels)
bool launch_shadows_atrous_v3(const GBufLevelDev& g, const uint32_t* in, const uint8_t* tile_flags, int radius, int step, float phi_vis, float phi_n, float sigma_z,
                              float power, uint32_t* out, int row0, int row1, cudaStream_t st)
{
    if (radius != 1 || phi_n != 32.0f || (g.W & 1) || row0 % 8 != 0 || !(step == 1 || step == 2 || step == 4 || step == 8)) return false;
    V3Params P { g.W, g.H, 1.44269504f / sigma_z, -1.44269504f / phi_vis, power, row0, row1 };
    switch (step)
    {
        case 1: launch_tiles<Dense<1>>(k_atrous_v3<1>, g, in, tile_flags, P, out, st); break;
        case 2: launch_tiles<Dense<2>>(k_atrous_v3<2>, g, in, tile_flags, P, out, st); break;
        case 4: launch_tiles<Dense<4>>(k_atrous_v3<4>, g, in, tile_flags, P, out, st); break;
        default: launch_tiles<Interleaved<8>>(k_atrous_v3s<8>, g, in, tile_flags, P, out, st); break; // DESIGN.md §8
    }
    return true;
}
