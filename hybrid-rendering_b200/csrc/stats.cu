// stats.cu — measurement helpers behind hr_pass_get_stats / hr_pass_output_checksum (not on the frame path).
//   * tile statistics: how many 8x8 tiles of the rows a render covered were on the denoise list (tile flag = 1) — bench.py
//     computes the a-trous roofline on the bytes the launch really processed (SURVEY.md §8d; the reference's K2/K4 tile lists
//     `ray_traced_shadows.cpp:224` are this flag image here);
//   * ray counters: drained from the per-pass counter slots the trace kernels add to (traverse.cuh::count_rays);
//   * image checksum: order-independent 64-bit sum over the texels of an output of a mix of (texel index, texel value), the formula
//     hr_api.h states — lets a sharded run prove on the device that its gathered frame, or the sum of its ranks' own rows, equals the
//     single-GPU frame.
#include "hr_internal.h"

namespace {

__global__ void k_tile_stats(const uint8_t* __restrict__ flags, int TW, int t0, int t1, unsigned long long* __restrict__ out)
{
    unsigned long long n = 0;
    const size_t first = (size_t)t0 * TW, count = (size_t)(t1 - t0) * TW;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) n += flags[first + i] ? 1u : 0u;
    n = __reduce_add_sync(0xFFFFFFFFu, (unsigned)n);
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(out, n);
}

__global__ void k_drain_ray_counters(unsigned long long* __restrict__ ctr, unsigned long long* __restrict__ out)
{
    const int kind = threadIdx.x >> 5, slot = threadIdx.x & 31; // 64 threads: 2 kinds x 32 slots
    unsigned long long* p = ctr + ((size_t)kind * HR_RAY_CTR_SLOTS + slot) * HR_RAY_CTR_STRIDE;
    unsigned long long  v = *p;
    *p                    = 0ull;
    // 64-bit warp sum through two 32-bit halves
    const unsigned lo = __reduce_add_sync(0xFFFFFFFFu, (unsigned)(v & 0xFFFFu)), m1 = __reduce_add_sync(0xFFFFFFFFu, (unsigned)((v >> 16) & 0xFFFFu)),
                   m2 = __reduce_add_sync(0xFFFFFFFFu, (unsigned)((v >> 32) & 0xFFFFu)), hi = __reduce_add_sync(0xFFFFFFFFu, (unsigned)(v >> 48));
    if (slot == 0) out[kind] = (unsigned long long)lo + ((unsigned long long)m1 << 16) + ((unsigned long long)m2 << 32) + ((unsigned long long)hi << 48);
}

__device__ __forceinline__ unsigned long long mix64(unsigned long long z)
{ // splitmix64 finaliser
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// the texel's TS bytes as a little-endian unsigned integer (images are allocated with at least TS-byte alignment)
template <int TS>
__device__ __forceinline__ unsigned long long load_texel(const uint8_t* base, size_t i)
{
    if (TS == 1) return base[i];
    if (TS == 2) return reinterpret_cast<const uint16_t*>(base)[i];
    if (TS == 4) return reinterpret_cast<const uint32_t*>(base)[i];
    return reinterpret_cast<const unsigned long long*>(base)[i];
}

// texels [t0, t1) of an image of TS-byte texels; texel i (row-major index from the start of the IMAGE, not of the row range) adds
// mix64(mix64(i + 0x9E3779B97F4A7C15) ^ value), so the sums of any split of the rows add up to the whole image's (mod 2^64).
template <int TS>
__global__ void k_checksum(const uint8_t* __restrict__ base, size_t t0, size_t t1, unsigned long long* __restrict__ out)
{
    unsigned long long acc = 0;
    for (size_t i = t0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < t1; i += (size_t)gridDim.x * blockDim.x)
        acc += mix64(mix64(i + 0x9E3779B97F4A7C15ull) ^ load_texel<TS>(base, i));
    // block reduction
    __shared__ unsigned long long s[32];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xFFFFFFFFu, acc, o);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32)
    {
        unsigned long long v = threadIdx.x < (blockDim.x >> 5) ? s[threadIdx.x] : 0ull;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
        if (threadIdx.x == 0) atomicAdd(out, v);
    }
}

} // namespace

// out[0] = tiles with flag != 0 in tile rows [t0, t1)
void launch_tile_stats(const uint8_t* flags, int TW, int t0, int t1, unsigned long long* d_out, cudaStream_t st)
{
    if (t1 <= t0) return;
    k_tile_stats<<<64, 256, 0, st>>>(flags, TW, t0, t1, d_out);
}

// out[0] = primary, out[1] = secondary rays since the last drain (counters reset)
void launch_drain_ray_counters(unsigned long long* ctr, unsigned long long* d_out, cudaStream_t st) { k_drain_ray_counters<<<1, 64, 0, st>>>(ctr, d_out); }

void launch_checksum(const void* base, int texel_bytes, size_t texel0, size_t texel1, unsigned long long* d_out, cudaStream_t st)
{
    if (texel1 <= texel0) return;
    const uint8_t* b = static_cast<const uint8_t*>(base);
    switch (texel_bytes)
    {
        case 1: k_checksum<1><<<296, 256, 0, st>>>(b, texel0, texel1, d_out); break;
        case 2: k_checksum<2><<<296, 256, 0, st>>>(b, texel0, texel1, d_out); break;
        case 4: k_checksum<4><<<296, 256, 0, st>>>(b, texel0, texel1, d_out); break;
        default: k_checksum<8><<<296, 256, 0, st>>>(b, texel0, texel1, d_out); break;
    }
}
