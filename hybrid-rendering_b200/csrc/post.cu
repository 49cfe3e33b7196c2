// post.cu — kernels of the post-processing passes (SURVEY.md §8 f4): temporal anti-aliasing (src/shaders/taa.comp, host
// src/temporal_aa.cpp:83-172), the history reset blit (temporal_aa.cpp:112-121) and the tone map (src/shaders/tone_map.frag).
// One thread per pixel, 32 x 8 pixel CTAs; the arithmetic lives in post_px.cuh (shared with the CPU-side host emulation test).
//
// BUILD NOTE: compiled with -fmad=false — the TAA resolve is specified without FMA contraction (post_px.cuh header).
//
// Algorithmic bytes per pixel (SURVEY.md §8d convention: every distinct input texel once + every output texel once):
//   TAA       8 (current colour) + 8 (history) + 4 (depth) + 8 (GB2 velocity) + 8 (output) = 36
//   tone map  8 (input) + 4 (RGBA8 output) = 12
// Both are HBM-bound by construction (the 11 bilinear taps of the resolve hit a 4 x 4 texel window that stays in L1).
#include "hr_internal.h"
#include "post_px.cuh"

namespace {

using namespace post;

// rows [row0, row1): a sharded rank resolves its band (the inputs it reads are complete on every rank, hr_taa_render)
__global__ void __launch_bounds__(256) k_taa(TaaArgs A, int row0, int row1, uint2* __restrict__ out)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= A.W || y >= row1) return;
    const F4 c = taa_pixel(A, x, y);
    out[(size_t)y * A.W + x] = make_uint2((uint32_t)float_to_half_bits(c.x) | ((uint32_t)float_to_half_bits(c.y) << 16),
                                          (uint32_t)float_to_half_bits(c.z) | ((uint32_t)float_to_half_bits(c.w) << 16));
}

// vkCmdBlitImage(src -> RGBA16F dst, NEAREST, same extent): per-texel format conversion with Vulkan's component fill
__global__ void __launch_bounds__(256) k_blit_rgba16f(ImgView src, uint2* __restrict__ out)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= src.W || y >= src.H) return;
    const F4 c = fetch_texel(src, x, y);
    out[(size_t)y * src.W + x] = make_uint2((uint32_t)float_to_half_bits(c.x) | ((uint32_t)float_to_half_bits(c.y) << 16),
                                            (uint32_t)float_to_half_bits(c.z) | ((uint32_t)float_to_half_bits(c.w) << 16));
}

__global__ void __launch_bounds__(256) k_tonemap(ImgView src, float exposure, int single_channel, int row0, int row1, uint32_t* __restrict__ out)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = row0 + blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= src.W || y >= row1) return;
    out[(size_t)y * src.W + x] = tonemap_pixel(fetch_texel(src, x, y), exposure, single_channel);
}

ImgView view(const void* p, int W, int H, int channels)
{
    ImgView v;
    v.p = (const uint16_t*)p; v.W = W; v.H = H; v.channels = channels;
    return v;
}

} // namespace

void launch_taa(const GBufLevelDev& g, const void* current, int current_channels, const void* history, const float* jitter_xy, float feedback_min, float feedback_max,
                int sharpen, void* out, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    TaaArgs A;
    A.cur   = view(current, g.W, g.H, current_channels);
    A.prev  = view(history, g.W, g.H, 4);
    A.depth = g.depth;
    A.gb2   = (const uint16_t*)g.gb2;
    A.W = g.W; A.H = g.H;
    A.texel_x = 1.0f / (float)g.W; A.texel_y = 1.0f / (float)g.H; // push_constants.texel_size, temporal_aa.cpp:123
    A.jitter_x = jitter_xy[0]; A.jitter_y = jitter_xy[1];
    A.feedback_min = feedback_min; A.feedback_max = feedback_max;
    A.sharpen = sharpen;
    dim3 grid((g.W + 31) / 32, (row1 - row0 + 7) / 8);
    k_taa<<<grid, 256, 0, st>>>(A, row0, row1, (uint2*)out);
}

void launch_blit_rgba16f(const void* src, int channels, int W, int H, void* out, cudaStream_t st)
{
    dim3 grid((W + 31) / 32, (H + 7) / 8);
    k_blit_rgba16f<<<grid, 256, 0, st>>>(view(src, W, H, channels), (uint2*)out);
}

void launch_tonemap(const void* src, int channels, int W, int H, float exposure, int single_channel, void* out_rgba8, int row0, int row1, cudaStream_t st)
{
    if (row1 <= row0) return;
    dim3 grid((W + 31) / 32, (row1 - row0 + 7) / 8);
    k_tonemap<<<grid, 256, 0, st>>>(view(src, W, H, channels), exposure, single_channel, row0, row1, (uint32_t*)out_rgba8);
}
