// compare.cu — image comparison on the device (hr_image_compare): error sums and SSIM of a test image against a reference image.
// Not on the frame path.  The per-pixel arithmetic is bit-specified (hr_api.h, DESIGN.md §5; tests/image_compare.py restates it in
// numpy): IEEE + - * / in the written order, no FMA contraction (compiled with -fmad=false), no exp / rsqrt / approximate division.
//
// k_compare: one CTA per 32 x 16 tile of the row range.  It stages the luminance of both images for the tile and a 5-pixel halo
// (taps clamped to the image) in shared memory, reading each image once (64-bit loads for RGBA16F); the error terms of the tile's
// own pixels come from those loads.  Then the horizontal pass of the window's five quantities (Y_t, Y_r, Y_t^2, Y_r^2, Y_t Y_r) over
// the staged rows, the vertical pass per pixel, and SSIM.  Every term is converted to a 128-bit fixed-point integer and the CTA
// writes one record of integer sums; k_compare_total adds the records (grid-stride shares per CTA, then the last CTA to finish adds
// the shares).  Integer sums: the result is the same for any
// launch shape, tile order or row split.
#include "hr_internal.h"
#include <cmath>

namespace {

typedef unsigned __int128 u128;
typedef __int128          i128;

constexpr int CMP_TW = 32, CMP_TH = 16, CMP_R = 5, CMP_NT = 256;
constexpr int CMP_RW = CMP_TW + 2 * CMP_R, CMP_RH = CMP_TH + 2 * CMP_R; // staged region: 42 x 26

struct Window { float w[2 * CMP_R + 1]; };
struct CmpParams { float eps, c1, c2; };

// the 11-tap Gaussian of sigma 1.5: each weight in double, normalised by the sum (taken in tap order), then rounded to float
Window gaussian_window()
{
    double g[2 * CMP_R + 1], s = 0.0;
    for (int k = -CMP_R; k <= CMP_R; k++) { g[k + CMP_R] = std::exp(-(double)(k * k) / (2.0 * 1.5 * 1.5)); s += g[k + CMP_R]; }
    Window w;
    for (int k = 0; k < 2 * CMP_R + 1; k++) w.w[k] = (float)(g[k] / s);
    return w;
}

struct Acc {
    unsigned long long px, nft, nfr;
    u128               sq, ab, rel;
    i128               ss;
    unsigned           mx;
};

__device__ __forceinline__ void acc_add(Acc& a, const Acc& b)
{
    a.px += b.px; a.nft += b.nft; a.nfr += b.nfr;
    a.sq += b.sq; a.ab += b.ab; a.rel += b.rel; a.ss += b.ss;
    a.mx = a.mx > b.mx ? a.mx : b.mx;
}

__device__ __forceinline__ u128 shfl_xor128(u128 v, int o)
{
    const unsigned long long lo = __shfl_xor_sync(0xFFFFFFFFu, (unsigned long long)v, o);
    const unsigned long long hi = __shfl_xor_sync(0xFFFFFFFFu, (unsigned long long)(v >> 64), o);
    return ((u128)hi << 64) | lo;
}

// butterfly over the warp: the two 64-bit halves are shuffled, the 128-bit add carries from the low half into the high half
__device__ __forceinline__ void warp_reduce(Acc& a)
{
    for (int o = 16; o > 0; o >>= 1)
    {
        Acc b;
        b.px  = __shfl_xor_sync(0xFFFFFFFFu, a.px, o);
        b.nft = __shfl_xor_sync(0xFFFFFFFFu, a.nft, o);
        b.nfr = __shfl_xor_sync(0xFFFFFFFFu, a.nfr, o);
        b.sq  = shfl_xor128(a.sq, o);
        b.ab  = shfl_xor128(a.ab, o);
        b.rel = shfl_xor128(a.rel, o);
        b.ss  = (i128)shfl_xor128((u128)a.ss, o);
        b.mx  = a.mx;
        acc_add(a, b);
    }
    a.mx = __reduce_max_sync(0xFFFFFFFFu, a.mx);
}

__device__ __forceinline__ void store_sums(hr_compare_sums* o, const Acc& a)
{
    o->pixels = a.px; o->nonfinite_test = a.nft; o->nonfinite_ref = a.nfr;
    o->sq_err[0]  = (unsigned long long)a.sq;        o->sq_err[1]  = (unsigned long long)(a.sq >> 64);
    o->abs_err[0] = (unsigned long long)a.ab;        o->abs_err[1] = (unsigned long long)(a.ab >> 64);
    o->rel_err[0] = (unsigned long long)a.rel;       o->rel_err[1] = (unsigned long long)(a.rel >> 64);
    o->ssim[0]    = (unsigned long long)(u128)a.ss;  o->ssim[1]    = (unsigned long long)((u128)a.ss >> 64);
    o->max_abs_err = a.mx;
    o->_pad        = 0;
}

// the whole CTA's sum into `o` (thread 0 writes); `part` holds one Acc per warp
template <int NT>
__device__ __forceinline__ void block_reduce_store(Acc a, Acc* part, hr_compare_sums* o)
{
    warp_reduce(a);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) part[warp] = a;
    __syncthreads();
    if (warp == 0)
    {
        Acc b = {};
        if (lane < NT / 32) b = part[lane];
        warp_reduce(b);
        if (lane == 0) store_sums(o, b);
    }
}

// round-to-nearest-even(x * 2^32) as a 128-bit integer, x clamped to [-2^63, 2^63], NaN -> 0.  x * 2^32 is exact in float and
// rintf leaves an integer-valued float, whose mantissa is shifted into place.
__device__ __forceinline__ i128 fixed32(float x)
{
    if (x != x) return 0;
    x = fminf(fmaxf(x, -0x1p63f), 0x1p63f);
    const float    y = rintf(x * 0x1p32f);
    const unsigned b = __float_as_uint(y);
    const int      e = (int)((b >> 23) & 0xFFu);
    if (e == 0) return 0; // +-0: an integer-valued float is never subnormal
    const unsigned long long m  = (b & 0x7FFFFFu) | 0x800000u;
    const int                sh = e - 150;
    const u128               v  = sh >= 0 ? (u128)m << sh : (u128)(m >> -sh);
    return (b >> 31) ? -(i128)v : (i128)v;
}

// the pixel's channels as float: RGBA16F / RGBA8 -> rgb, RG16F -> r, g, R16F -> r (RGBA8 as UNORM b / 255)
template <int FMT> struct Px;
template <> struct Px<HR_FMT_RGBA16F> {
    static constexpr int C = 3;
    static __device__ __forceinline__ void load(const void* p, size_t i, float* c)
    {
        const uint2 v = __ldg(static_cast<const uint2*>(p) + i);
        c[0] = __half2float(__ushort_as_half((unsigned short)(v.x & 0xFFFFu)));
        c[1] = __half2float(__ushort_as_half((unsigned short)(v.x >> 16)));
        c[2] = __half2float(__ushort_as_half((unsigned short)(v.y & 0xFFFFu)));
    }
};
template <> struct Px<HR_FMT_RGBA8> {
    static constexpr int C = 3;
    static __device__ __forceinline__ void load(const void* p, size_t i, float* c)
    {
        const unsigned v = __ldg(static_cast<const unsigned*>(p) + i);
        c[0] = (float)(v & 0xFFu) / 255.0f;
        c[1] = (float)((v >> 8) & 0xFFu) / 255.0f;
        c[2] = (float)((v >> 16) & 0xFFu) / 255.0f;
    }
};
template <> struct Px<HR_FMT_RG16F> {
    static constexpr int C = 2;
    static __device__ __forceinline__ void load(const void* p, size_t i, float* c)
    {
        const unsigned v = __ldg(static_cast<const unsigned*>(p) + i);
        c[0] = __half2float(__ushort_as_half((unsigned short)(v & 0xFFFFu)));
        c[1] = __half2float(__ushort_as_half((unsigned short)(v >> 16)));
    }
};
template <> struct Px<HR_FMT_R16F> {
    static constexpr int C = 1;
    static __device__ __forceinline__ void load(const void* p, size_t i, float* c)
    {
        c[0] = __half2float(__ldg(static_cast<const __half*>(p) + i));
    }
};

template <int C>
__device__ __forceinline__ bool all_finite(const float* c)
{
    bool f = true;
#pragma unroll
    for (int k = 0; k < C; k++) f = f && isfinite(c[k]);
    return f;
}

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }

// the reference's luminance weights (common.glsl:143) without its 1e-4 floor, on clamped channels
template <int C>
__device__ __forceinline__ float luminance(const float* c)
{
    if (C == 1) return clamp01(c[0]);
    const float c2 = C == 3 ? clamp01(c[2]) : 0.0f;
    return (0.299f * clamp01(c[0]) + 0.587f * clamp01(c[1])) + 0.114f * c2;
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

template <int FMT>
__global__ void __launch_bounds__(CMP_NT) k_compare(const void* __restrict__ test, const void* __restrict__ ref, int W, int H, int row0, int row1,
                                                    Window win, CmpParams prm, uint2* __restrict__ emap, hr_compare_sums* __restrict__ rec)
{
    constexpr int C = Px<FMT>::C;
    __shared__ float         yl[2][CMP_RH][CMP_RW];     // luminance of test, ref (0 at a left-out pixel)
    __shared__ float         hq[5][CMP_RH][CMP_TW];     // horizontal pass: Y_t, Y_r, Y_t^2, Y_r^2, Y_t Y_r
    __shared__ float         term[3][CMP_TH][CMP_TW];   // ae, se, rel of the tile's pixels (error map)
    __shared__ unsigned char state[CMP_TH][CMP_TW];     // 0 outside the range, 1 left out (non-finite), 2 summed
    __shared__ Acc           part[CMP_NT / 32];
    const int x0 = blockIdx.x * CMP_TW, y0 = row0 + blockIdx.y * CMP_TH;
    Acc       a  = {};

    for (int i = threadIdx.x; i < CMP_RW * CMP_RH; i += CMP_NT)
    {
        const int    ry = i / CMP_RW, rx = i - ry * CMP_RW;
        const int    gx = clampi(x0 - CMP_R + rx, 0, W - 1), gy = clampi(y0 - CMP_R + ry, 0, H - 1);
        const size_t idx = (size_t)gy * W + gx;
        float        t[C], r[C];
        Px<FMT>::load(test, idx, t);
        Px<FMT>::load(ref, idx, r);
        const bool ft = all_finite<C>(t), fr = all_finite<C>(r), ok = ft && fr;
        yl[0][ry][rx] = ok ? luminance<C>(t) : 0.0f;
        yl[1][ry][rx] = ok ? luminance<C>(r) : 0.0f;
        const int px = rx - CMP_R, py = ry - CMP_R;
        if (px < 0 || px >= CMP_TW || py < 0 || py >= CMP_TH) continue;
        // a tile pixel inside the image and the range is its own tap (gx, gy unclamped)
        const bool in = x0 + px < W && y0 + py < row1;
        state[py][px] = in ? (ok ? 2 : 1) : 0;
        if (!in) continue;
        a.nft += ft ? 0 : 1;
        a.nfr += fr ? 0 : 1;
        if (!ok) continue;
        float se = 0.0f, ae = 0.0f, rl = 0.0f, mx = 0.0f;
#pragma unroll
        for (int k = 0; k < C; k++)
        {
            const float d = t[k] - r[k], d2 = d * d, ad = fabsf(d);
            se = se + d2;
            ae = ae + ad;
            rl = rl + d2 / (r[k] * r[k] + prm.eps);
            mx = fmaxf(mx, ad);
        }
        se = se / (float)C;
        ae = ae / (float)C;
        rl = rl / (float)C;
        a.px++;
        a.sq += (u128)fixed32(se);
        a.ab += (u128)fixed32(ae);
        a.rel += (u128)fixed32(rl);
        a.mx = a.mx > __float_as_uint(mx) ? a.mx : __float_as_uint(mx);
        term[0][py][px] = ae;
        term[1][py][px] = se;
        term[2][py][px] = rl;
    }
    __syncthreads();

    // rows first: the window along x over every staged row (region column px + k is the tap x + k - 5)
    for (int i = threadIdx.x; i < CMP_RH * CMP_TW; i += CMP_NT)
    {
        const int ry = i / CMP_TW, px = i - ry * CMP_TW;
        float     s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f, s4 = 0.0f;
#pragma unroll
        for (int k = 0; k < 2 * CMP_R + 1; k++)
        {
            const float u = yl[0][ry][px + k], v = yl[1][ry][px + k], w = win.w[k];
            s0 = s0 + w * u;
            s1 = s1 + w * v;
            s2 = s2 + w * (u * u);
            s3 = s3 + w * (v * v);
            s4 = s4 + w * (u * v);
        }
        hq[0][ry][px] = s0; hq[1][ry][px] = s1; hq[2][ry][px] = s2; hq[3][ry][px] = s3; hq[4][ry][px] = s4;
    }
    __syncthreads();

    // then columns, SSIM, the error map
    for (int i = threadIdx.x; i < CMP_TH * CMP_TW; i += CMP_NT)
    {
        const int py = i / CMP_TW, px = i - py * CMP_TW, s = state[py][px];
        if (s == 0) continue;
        const size_t o = (size_t)(y0 + py) * W + (x0 + px);
        if (s == 1)
        {
            if (emap) emap[o] = make_uint2(0x7E007E00u, 0x7E007E00u);
            continue;
        }
        float m[5] = { 0.0f, 0.0f, 0.0f, 0.0f, 0.0f };
#pragma unroll
        for (int k = 0; k < 2 * CMP_R + 1; k++)
        {
            const float w = win.w[k];
#pragma unroll
            for (int j = 0; j < 5; j++) m[j] = m[j] + w * hq[j][py + k][px];
        }
        const float mt = m[0], mr = m[1];
        const float vt = m[2] - mt * mt, vr = m[3] - mr * mr, cv = m[4] - mt * mr;
        const float ss = (((2.0f * mt) * mr + prm.c1) * (2.0f * cv + prm.c2)) / (((mt * mt + mr * mr) + prm.c1) * ((vt + vr) + prm.c2));
        a.ss += fixed32(ss);
        if (emap)
        {
            const unsigned h0 = __half_as_ushort(__float2half_rn(term[0][py][px])), h1 = __half_as_ushort(__float2half_rn(term[1][py][px]));
            const unsigned h2 = __half_as_ushort(__float2half_rn(term[2][py][px])), h3 = __half_as_ushort(__float2half_rn(ss));
            emap[o] = make_uint2(h0 | (h1 << 16), h2 | (h3 << 16));
        }
    }
    block_reduce_store<CMP_NT>(a, part, rec + (size_t)blockIdx.y * gridDim.x + blockIdx.x);
}

// a record as Acc; `cg`: through L2 only (the partial sums other CTAs of the same launch wrote)
template <bool cg>
__device__ __forceinline__ Acc load_record(const hr_compare_sums* r)
{
    const unsigned long long* q = reinterpret_cast<const unsigned long long*>(r); // 12 words: counts, 4 x (lo, hi), max_abs_err | _pad
    unsigned long long        w[12];
#pragma unroll
    for (int k = 0; k < 12; k++) w[k] = cg ? __ldcg(q + k) : __ldg(q + k);
    Acc b;
    b.px  = w[0]; b.nft = w[1]; b.nfr = w[2];
    b.sq  = ((u128)w[4] << 64) | w[3];
    b.ab  = ((u128)w[6] << 64) | w[5];
    b.rel = ((u128)w[8] << 64) | w[7];
    b.ss  = (i128)(((u128)w[10] << 64) | w[9]);
    b.mx  = (unsigned)w[11];
    return b;
}

// The total of the n per-tile records: each CTA sums a grid-stride share into partial[blockIdx.x]; the CTA that takes the last ticket
// adds the partials into out.  Integer sums: the result does not depend on which CTA finishes last.
constexpr int CMP_TOTAL_NT = 256;
__global__ void __launch_bounds__(CMP_TOTAL_NT) k_compare_total(const hr_compare_sums* __restrict__ rec, int n, hr_compare_sums* partial,
                                                               unsigned* ticket, hr_compare_sums* __restrict__ out)
{
    __shared__ Acc  part[CMP_TOTAL_NT / 32];
    __shared__ bool last;
    Acc             a = {};
    for (int i = blockIdx.x * CMP_TOTAL_NT + threadIdx.x; i < n; i += gridDim.x * CMP_TOTAL_NT) acc_add(a, load_record<false>(rec + i));
    block_reduce_store<CMP_TOTAL_NT>(a, part, partial + blockIdx.x); // thread 0 stores
    if (threadIdx.x == 0)
    {
        __threadfence();
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    Acc b = {};
    for (int i = threadIdx.x; i < (int)gridDim.x; i += CMP_TOTAL_NT) acc_add(b, load_record<true>(partial + i));
    block_reduce_store<CMP_TOTAL_NT>(b, part, out);
}

template <int FMT>
void launch_fmt(const hr_image& t, const hr_image& r, int row0, int row1, const Window& w, const CmpParams& p, uint2* emap, hr_compare_sums* rec, dim3 grid,
                cudaStream_t st)
{
    k_compare<FMT><<<grid, CMP_NT, 0, st>>>(t.data, r.data, t.width, t.height, row0, row1, w, p, emap, rec);
}

bool is_finite_nonneg(float v) { return v >= 0.0f && std::isfinite(v); }

int texel_bytes(int fmt) { return fmt == HR_FMT_RGBA16F ? 8 : fmt == HR_FMT_R16F ? 2 : 4; } // the formats hr_image_compare accepts

// the byte ranges of two dense images intersect
bool overlaps(const hr_image& a, const hr_image& b)
{
    const uintptr_t a0 = (uintptr_t)a.data, a1 = a0 + (size_t)a.width * a.height * texel_bytes(a.format);
    const uintptr_t b0 = (uintptr_t)b.data, b1 = b0 + (size_t)b.width * b.height * texel_bytes(b.format);
    return a0 < b1 && b0 < a1;
}

} // namespace

extern "C" {

void hr_compare_default_params(hr_compare_params* p)
{
    if (!p) return;
    p->relmse_eps = 0.01f;
    p->ssim_c1    = 1e-4f;
    p->ssim_c2    = 9e-4f;
}

void hr_compare_sums_add(hr_compare_sums* acc, const hr_compare_sums* s)
{
    if (!acc || !s) return;
    auto add128 = [](uint64_t* a, const uint64_t* b) {
        const u128 v = (((u128)a[1] << 64) | a[0]) + (((u128)b[1] << 64) | b[0]);
        a[0] = (uint64_t)v;
        a[1] = (uint64_t)(v >> 64);
    };
    acc->pixels += s->pixels;
    acc->nonfinite_test += s->nonfinite_test;
    acc->nonfinite_ref += s->nonfinite_ref;
    add128(acc->sq_err, s->sq_err);
    add128(acc->abs_err, s->abs_err);
    add128(acc->rel_err, s->rel_err);
    add128(acc->ssim, s->ssim);
    acc->max_abs_err = acc->max_abs_err > s->max_abs_err ? acc->max_abs_err : s->max_abs_err;
}

void hr_compare_finish(const hr_compare_sums* s, hr_compare_result* out)
{
    if (!s || !out) return;
    const double n = (double)s->pixels;
    auto mean_u = [n](const uint64_t* v) { return (double)(((u128)v[1] << 64) | v[0]) * 0x1p-32 / n; };
    auto mean_s = [n](const uint64_t* v) { return (double)(i128)(((u128)v[1] << 64) | v[0]) * 0x1p-32 / n; };
    float mx;
    memcpy(&mx, &s->max_abs_err, 4);
    out->mse      = mean_u(s->sq_err);
    out->rmse     = std::sqrt(out->mse);
    out->psnr     = out->mse == 0.0 ? INFINITY : 10.0 * std::log10(1.0 / out->mse);
    out->relmse   = mean_u(s->rel_err);
    out->mean_abs = mean_u(s->abs_err);
    out->max_abs  = (double)mx;
    out->ssim     = mean_s(s->ssim);
    out->pixels   = s->pixels;
    out->nonfinite_test = s->nonfinite_test;
    out->nonfinite_ref  = s->nonfinite_ref;
}

int hr_image_compare(hr_ctx* ctx, const hr_image* test, const hr_image* ref, const hr_compare_params* params, int row0, int row1, hr_compare_sums* out,
                     hr_image* error_map, void* stream)
{
    HR_REQUIRE(ctx, ctx && test && ref && params && out && test->data && ref->data, HR_ERR_INVALID_ARG, "hr_image_compare: null argument");
    HR_REQUIRE(ctx, test->width > 0 && test->height > 0 && test->width == ref->width && test->height == ref->height && test->format == ref->format,
               HR_ERR_INVALID_ARG, "hr_image_compare: the images differ in size or format");
    const int fmt = test->format, W = test->width, H = test->height;
    HR_REQUIRE(ctx, fmt != HR_FMT_R32_UINT && fmt != HR_FMT_R8_UINT, HR_ERR_UNSUPPORTED, "hr_image_compare: integer images (masks, counts) are not compared");
    HR_REQUIRE(ctx, fmt == HR_FMT_RGBA16F || fmt == HR_FMT_RGBA8 || fmt == HR_FMT_RG16F || fmt == HR_FMT_R16F, HR_ERR_INVALID_ARG, "hr_image_compare: unknown format");
    HR_REQUIRE(ctx, is_finite_nonneg(params->relmse_eps) && is_finite_nonneg(params->ssim_c1) && is_finite_nonneg(params->ssim_c2), HR_ERR_INVALID_ARG,
               "hr_image_compare: parameters must be finite and >= 0");
    if (row1 <= 0) { row0 = 0; row1 = H; }
    HR_REQUIRE(ctx, row0 >= 0 && row1 >= row0 && row1 <= H, HR_ERR_INVALID_ARG, "hr_image_compare: bad row range");
    HR_REQUIRE(ctx, !error_map || (error_map->data && error_map->width == W && error_map->height == H && error_map->format == HR_FMT_RGBA16F),
               HR_ERR_INVALID_ARG, "hr_image_compare: the error map must be an RGBA16F image of the images' size");
    // the kernel reads the inputs' halo rows through the read-only path while other CTAs write the error map
    HR_REQUIRE(ctx, !error_map || (!overlaps(*error_map, *test) && !overlaps(*error_map, *ref)), HR_ERR_INVALID_ARG,
               "hr_image_compare: the error map overlaps an input image");
    cudaStream_t    st = (cudaStream_t)stream;
    hr_compare_sums h  = {};
    if (row1 > row0)
    {
        static const Window win = gaussian_window();
        const CmpParams     p   = { params->relmse_eps, params->ssim_c1, params->ssim_c2 };
        const dim3          grid((W + CMP_TW - 1) / CMP_TW, (row1 - row0 + CMP_TH - 1) / CMP_TH);
        const int           n = (int)(grid.x * grid.y);
        const int           nb = (n + 2 * CMP_TOTAL_NT - 1) / (2 * CMP_TOTAL_NT) < 256 ? (n + 2 * CMP_TOTAL_NT - 1) / (2 * CMP_TOTAL_NT) : 256;
        hr_compare_sums*    d = nullptr; // [n records][nb partials][total][ticket]
        HR_CUDA(ctx, cudaMallocAsync((void**)&d, sizeof(hr_compare_sums) * (n + nb + 2), st));
        unsigned* ticket = reinterpret_cast<unsigned*>(d + n + nb + 1);
        if (cudaMemsetAsync(ticket, 0, sizeof(unsigned), st) != cudaSuccess)
        {
            cudaFreeAsync(d, st);
            HR_CUDA(ctx, cudaGetLastError());
            return HR_ERR_CUDA;
        }
        uint2* emap = error_map ? static_cast<uint2*>(error_map->data) : nullptr;
        switch (fmt)
        {
            case HR_FMT_RGBA16F: launch_fmt<HR_FMT_RGBA16F>(*test, *ref, row0, row1, win, p, emap, d, grid, st); break;
            case HR_FMT_RGBA8: launch_fmt<HR_FMT_RGBA8>(*test, *ref, row0, row1, win, p, emap, d, grid, st); break;
            case HR_FMT_RG16F: launch_fmt<HR_FMT_RG16F>(*test, *ref, row0, row1, win, p, emap, d, grid, st); break;
            default: launch_fmt<HR_FMT_R16F>(*test, *ref, row0, row1, win, p, emap, d, grid, st); break;
        }
        k_compare_total<<<nb, CMP_TOTAL_NT, 0, st>>>(d, n, d + n, ticket, d + n + nb);
        ctx->launches += 2;
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(&h, d + n + nb, sizeof(h), cudaMemcpyDeviceToHost, st);
        cudaFreeAsync(d, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        HR_CUDA(ctx, e);
    }
    else HR_CUDA(ctx, cudaStreamSynchronize(st));
    *out = h;
    return HR_OK;
}

} // extern "C"
