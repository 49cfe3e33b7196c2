// shard.cu — screen-space row-band sharding across the GPUs of one box (SURVEY.md §8e; no reference counterpart: the
// reference is a single-GPU sample).
//
// One process per GPU.  A pass image of height H is split into `world` contiguous bands of whole 8-row tiles
// (hr_shard_rows).  Every rank keeps a full replica of the G-buffer, the BVH and the blue-noise tables, computes all
// stages on its band plus a recompute halo (rays and stencils are pure functions of replicated inputs, so the halo is
// exact).  Two things cross GPUs:
//   * PEER HISTORY (shadows / AO): next frame's reprojection may read ANY row of the history images under camera motion.
//     Instead of all-gathering ~16 B/pixel of history every frame, each rank keeps only its band and maps every peer's
//     history images into its address space (CUDA IPC over NVLink / NVSwitch); the temporal kernel fetches a history
//     texel from the GPU that owns its row (HistPeers) — the exchange is fused into the kernel and moves exactly the
//     texels the reprojection touches (a few boundary rows for a static camera).  Ordering is a per-pass frame tick:
//     after its last history write of frame N a rank stores N into every peer's tick array (st.release.sys); before
//     the reprojection of frame N+1 a one-warp kernel spins (ld.acquire.sys, 10 s time-out) until every peer's tick
//     is >= N.  History images are double buffered by frame parity, so that wait also covers the write-after-read hazard.
//   * the pass's FINAL OUTPUT (optional, hr_shard_set_gather; on by default): one NCCL group of point-to-point transfers (an
//     all-gather with unequal counts: 2160 rows = 270 tiles do not divide evenly by 8) on a side stream, so every rank
//     ends up with the complete denoised frame.
//   * DDGI ATLASES: linked ranks split the probe stages by z-slices and store their slices' atlas rows into every peer's atlas
//     (k_ddgi_push), ordered by one frame tick; the atlases move on a grid re-initialisation, so the peers' addresses are read from
//     a device-side table at run time.
// The 1/2/4/8-GPU results are bit-identical to the single-GPU result (tests/test_gpu_multi.py).
//
// NCCL is dlopen'ed on first use so the single-GPU library has no NCCL dependency; inside a PyTorch process the
// already-loaded torch-bundled libnccl.so.2 is picked up.
#include "hr_internal.h"
#include <dlfcn.h>
#include <nccl.h>
#include <vector>

namespace {

struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*)                                                                 = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int)                                          = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t)                                                                    = nullptr;
    ncclResult_t (*GroupStart)()                                                                               = nullptr;
    ncclResult_t (*GroupEnd)()                                                                                 = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t)            = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t)                   = nullptr; // NCCL 2.7+
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t)                         = nullptr; // NCCL 2.7+
    const char* (*GetErrorString)(ncclResult_t)                                                                = nullptr;
    bool ok = false;
};

NcclApi& nccl()
{
    static NcclApi api;
    if (api.handle) return api;
    const char* names[] = { "libnccl.so.2", "libnccl.so" };
    for (const char* n : names)
    {
        api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (api.handle) break;
    }
    if (!api.handle) return api;
#define LOAD(field, sym) api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.handle, sym))
    LOAD(GetUniqueId, "ncclGetUniqueId");
    LOAD(CommInitRank, "ncclCommInitRank");
    LOAD(CommDestroy, "ncclCommDestroy");
    LOAD(GroupStart, "ncclGroupStart");
    LOAD(GroupEnd, "ncclGroupEnd");
    LOAD(AllGather, "ncclAllGather");
    LOAD(Send, "ncclSend");
    LOAD(Recv, "ncclRecv");
    LOAD(GetErrorString, "ncclGetErrorString");
#undef LOAD
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.GroupStart && api.GroupEnd && api.AllGather && api.Send && api.Recv &&
             api.GetErrorString;
    return api;
}

} // namespace

#define HR_NCCL(ctx, expr)                                                                                      \
    do {                                                                                                        \
        ncclResult_t _r = (expr);                                                                               \
        if (_r != ncclSuccess) {                                                                                \
            hr_set_error((ctx), "%s failed: %s (%s:%d)", #expr, nccl().GetErrorString(_r), __FILE__, __LINE__); \
            return HR_ERR_NCCL;                                                                                 \
        }                                                                                                       \
    } while (0)

void hr_band(const hr_ctx* ctx, int H, int* b0, int* b1)
{
    if (ctx->world <= 1) { *b0 = 0; *b1 = H; return; }
    hr_shard_rows(H, ctx->rank, ctx->world, b0, b1);
}

void hr_wait_exchange(hr_pass* p, cudaStream_t st)
{
    if (p && p->xchg_pending && p->ev_done) cudaStreamWaitEvent(st, p->ev_done, 0);
}

int hr_shard_exchange(hr_pass* p, const ExchangeItem* items, int n, cudaStream_t caller)
{
    hr_ctx* ctx = p->ctx;
    if (ctx->world <= 1 || !ctx->nccl_comm) return HR_OK;
    NcclApi& N = nccl();
    if (!ctx->comm_stream) HR_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->comm_stream, cudaStreamNonBlocking));
    if (!p->ev_ready)
    {
        HR_CUDA(ctx, cudaEventCreateWithFlags(&p->ev_ready, cudaEventDisableTiming));
        HR_CUDA(ctx, cudaEventCreateWithFlags(&p->ev_done, cudaEventDisableTiming));
    }
    HR_CUDA(ctx, cudaEventRecord(p->ev_ready, caller));
    HR_CUDA(ctx, cudaStreamWaitEvent(ctx->comm_stream, p->ev_ready, 0));
    cudaStream_t st = ctx->comm_stream;
    HR_NCCL(ctx, N.GroupStart());
    for (int i = 0; i < n; i++)
        for (int r = 0; r < ctx->world; r++)
        {
            int rb, re;
            hr_shard_rows(items[i].H, r, ctx->world, &rb, &re);
            const bool last_band = re >= items[i].H;
            if (items[i].shift) { rb <<= items[i].shift; re <<= items[i].shift; }
            if (items[i].div > 1) { rb /= items[i].div; re = (re + items[i].div - 1) / items[i].div; }
            if (last_band || re > items[i].rows) re = items[i].rows;
            if (re <= rb) continue;
            char*        p     = static_cast<char*>(items[i].base) + (size_t)rb * items[i].row_bytes;
            const size_t bytes = (size_t)(re - rb) * items[i].row_bytes;
            // point to point: every rank sends its band to each peer and receives theirs (7 independent NVSwitch transfers per
            // rank instead of 8 serial broadcast rings)
            if (r != ctx->rank) HR_NCCL(ctx, N.Recv(p, bytes, ncclUint8, r, (ncclComm_t)ctx->nccl_comm, st));
            else
                for (int q = 0; q < ctx->world; q++)
                    if (q != ctx->rank) HR_NCCL(ctx, N.Send(p, bytes, ncclUint8, q, (ncclComm_t)ctx->nccl_comm, st));
        }
    HR_NCCL(ctx, N.GroupEnd());
    HR_CUDA(ctx, cudaEventRecord(p->ev_done, st));
    p->xchg_pending = true;
    return HR_OK;
}


// ---- peer history -----------------------------------------------------------------------------------------------------
static int rt_init_bounds(hr_pass* p);

namespace {

// One pointer per rank: a shared image or tick array of every rank as this process sees it.
template <class T> struct PeerPtrs { T* p[HR_MAX_RANKS]; };

// The peers' tick arrays (a pass's tick publications write slot [self] of each).
PeerPtrs<int> peer_tick_ptrs(const hr_pass* p)
{
    PeerPtrs<int> t {};
    for (int r = 0; r < p->ctx->world; r++) t.p[r] = p->peer_ticks[r];
    return t;
}

// Shared image k (SharedImage) of every rank.
template <class T> PeerPtrs<T> peer_image_ptrs(const hr_pass* p, int k)
{
    PeerPtrs<T> m {};
    for (int r = 0; r < p->ctx->world; r++) m.p[r] = static_cast<T*>(p->hist_peer[r][k]);
    return m;
}

__device__ __forceinline__ void st_release_sys(int* a, int v) { asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(a), "r"(v) : "memory"); }

// Lane r (a peer) spins until its tick `*t` reached `tick`.  After 10 s it gives up and sets *err = 1 + r: a peer died or the ranks
// render different frame counts, and the GPU must not hang.  Returns false on a time-out.
__device__ __forceinline__ bool wait_tick(const int* t, int r, int tick, int* err, unsigned sleep_ns)
{
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;)
    {
        int v;
        asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(t) : "memory");
        if (v >= tick) return true;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > 10000000000ull) { *err = 1 + r; return false; }
        __nanosleep(sleep_ns);
    }
}

// The end of a push kernel: every block makes its stores visible system-wide and counts itself done; the last block resets the
// counter and publishes `tick` in slot `slot` of every peer's tick array.
__device__ __forceinline__ void publish_when_grid_done(int* __restrict__ ctl, const PeerPtrs<int>& ticks, int world, int self, int slot, int tick)
{
    __threadfence_system();
    __syncthreads();
    __shared__ int s_last;
    if (threadIdx.x == 0) s_last = atomicAdd(ctl + HR_CTL_BLOCKS_DONE, 1) == (int)gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    if (threadIdx.x == 0) ctl[HR_CTL_BLOCKS_DONE] = 0;
    const int r = threadIdx.x;
    if (r < world && r != self && ticks.p[r])
    {
        __threadfence_system(); // all blocks' stores (ordered before their atomicAdd) are visible before the tick
        st_release_sys(ticks.p[r] + slot * HR_MAX_RANKS + self, tick);
    }
}

__global__ void k_peer_signal(PeerPtrs<int> peers, int world, int self, int slot, int tick)
{
    const int r = threadIdx.x;
    if (r >= world || r == self || !peers.p[r]) return;
    __threadfence_system(); // the writes of the kernels before us in stream order become visible system-wide first
    st_release_sys(peers.p[r] + slot * HR_MAX_RANKS + self, tick);
}

// Bytes [first, last) of `src` to the same offsets of every peer's image dst[r] (r != self; null: skipped).  The images are 256-byte
// aligned, so a 16-byte body [a0, a1) is framed by a byte-wise head and tail of at most 15 bytes each, copied by threads 0-31 of the grid.
__device__ __forceinline__ void push_bytes(const uint8_t* __restrict__ src, uint8_t* const (&dst)[HR_MAX_RANKS], int world, int self, size_t first, size_t last, size_t tid, size_t nthr)
{
    const size_t a0 = min((first + 15) & ~(size_t)15, last), a1 = max(last & ~(size_t)15, a0);
    for (size_t i = a0 / 16 + tid; i < a1 / 16; i += nthr)
    {
        const uint4 v = reinterpret_cast<const uint4*>(src)[i];
        for (int r = 0; r < world; r++)
            if (r != self && dst[r]) reinterpret_cast<uint4*>(dst[r])[i] = v;
    }
    if (tid < 32)
    {
        const size_t i = tid < 16 ? first + tid : a1 + (tid - 16);
        if (i < (tid < 16 ? a0 : last))
        {
            const uint8_t v = src[i];
            for (int r = 0; r < world; r++)
                if (r != self && dst[r]) dst[r][i] = v;
        }
    }
}

// ---- cooperative ray trace: push of the traced share + cost-balanced partition ----
// After the shadows / AO ray trace: copy this rank's share, mask rows [ctl[self], ctl[self + 1]), of the mask or count image to every
// peer, drain the cost accumulation into every rank's cost table, and publish the ray-trace tick.  A mask row is `rows` image rows of
// `row_bytes` bytes (mask image: 1 row of 4 * MW bytes; count image: 4 rows of W bytes), clamped to the image height H.
__global__ void __launch_bounds__(256) k_rt_push(PeerPtrs<uint8_t> imgs, PeerPtrs<uint32_t> costs, int* __restrict__ ctl, uint32_t* __restrict__ acc,
                                                 PeerPtrs<int> ticks, int world, int self, int parity, int MH, size_t row_bytes, int rows, int H, int tick)
{
    const int    b0 = ctl[self], b1 = ctl[self + 1];
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)gridDim.x * blockDim.x;
    push_bytes(imgs.p[self], imgs.p, world, self, (size_t)rows * b0 * row_bytes, (size_t)min(rows * b1, H) * row_bytes, tid, nthr);
    if (blockIdx.x == 0)
        for (int row = b0 + threadIdx.x; row < b1; row += blockDim.x)
        {
            const uint32_t v = acc[row];
            acc[row]         = 0u;
            for (int r = 0; r < world; r++) costs.p[r][(size_t)parity * MH + row] = v;
        }
    publish_when_grid_done(ctl, ticks, world, self, TICK_RT, tick);
}

// One warp.  Lanes wait until every peer's ray-trace tick reached `rt_tick` and its history tick `hist_tick`, then the warp computes
// next frame's partition: bounds[k] = first mask row whose cost prefix reaches k/world of the total.
// Every rank computes the same table from the same (complete) cost table.  Any height: each lane sums one 1/32 chunk of the
// rows; a bound lies in the chunk of the first lane whose inclusive chunk prefix reaches its target, which the warp then scans
// 32 rows at a time.
__global__ void k_rt_wait_partition(const int* __restrict__ ticks, int rt_tick, int hist_tick, int* err, const uint32_t* __restrict__ cost, int MH, int world, int self,
                                    int cap, int* __restrict__ bounds)
{
    const int lane = threadIdx.x;
    if (lane < world && lane != self && wait_tick(ticks + TICK_RT * HR_MAX_RANKS + lane, lane, rt_tick, err, 100))
        wait_tick(ticks + TICK_HIST * HR_MAX_RANKS + lane, lane, hist_tick, err, 100); // ticks only grow: the same as one joint wait
    __syncwarp();
    const int          chunk = (MH + 31) / 32;
    unsigned long long local = 0;
    for (int i = lane * chunk; i < min((lane + 1) * chunk, MH); i++) local += __ldcg(cost + i);
    unsigned long long incl = local;
    for (int o = 1; o < 32; o <<= 1)
    {
        const unsigned long long v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= o) incl += v;
    }
    const unsigned long long total = __shfl_sync(0xFFFFFFFFu, incl, 31);
    int                      prev  = 0;
    if (lane == 0) bounds[0] = 0;
    for (int k = 1; k < world; k++)
    {
        int b;
        if (total == 0) b = (int)(((long long)MH * k) / world); // no cost information: uniform split
        else
        {
            // first row index b with prefix[b] >= target (prefix[b] = sum of cost[0, b)), at least prev
            const unsigned long long target = (total * (unsigned long long)k) / (unsigned long long)world;
            int                      first  = 0;
            if (target > 0)
            {
                const int          L   = __ffs(__ballot_sync(0xFFFFFFFFu, incl >= target)) - 1; // lanes past the rows hold incl == total
                unsigned long long run = __shfl_sync(0xFFFFFFFFu, incl - local, L);
                const int          r1  = min((L + 1) * chunk, MH);
                for (int r0 = L * chunk;; r0 += 32) // ends inside the chunk: its inclusive prefix reaches the target
                {
                    const int          i = r0 + lane;
                    unsigned long long v = i < r1 ? __ldcg(cost + i) : 0ull;
                    for (int o = 1; o < 32; o <<= 1)
                    {
                        const unsigned long long u = __shfl_up_sync(0xFFFFFFFFu, v, o);
                        if (lane >= o) v += u;
                    }
                    const unsigned m = __ballot_sync(0xFFFFFFFFu, i < r1 && run + v >= target);
                    if (m) { first = r0 + __ffs(m); break; } // prefix[i + 1] reaches the target first
                    run += __shfl_sync(0xFFFFFFFFu, v, 31);
                }
            }
            b = max(first, prev);
        }
        b = max(b, prev + 1);               // at least one row per rank
        b = min(b, prev + cap);             // the fixed launch grid covers at most `cap` rows
        b = min(b, MH - (world - k));       // leave a row for each remaining rank
        b = max(b, MH - (world - k) * cap); // the remaining ranks must be able to cover the rest
        if (lane == 0) bounds[k] = b;
        prev = b;
    }
    if (lane == 0) bounds[world] = MH;
}

__global__ void k_peer_wait(const int* __restrict__ ticks, int world, int self, int tick, int* err)
{
    const int r = threadIdx.x;
    if (r < world && r != self) wait_tick(ticks + r, r, tick, err, 200);
}

// Interleaved cooperative ray trace (reflections, path tracer): block b copies the b-th chunk of this rank (RowSet::interleave, 8 image
// rows of RGBA16F texels) to every rank that reads those rows; the last block to finish publishes the ray-trace tick.  A rank that owns
// no chunk still runs PUSH_SPLIT blocks so that its tick is published.
#define PUSH_SPLIT 4
struct NeedRows { int r0[HR_MAX_RANKS], r1[HR_MAX_RANKS]; };
__global__ void __launch_bounds__(256) k_rt_push_chunks(PeerPtrs<uint2> imgs, NeedRows need, PeerPtrs<int> ticks, int* __restrict__ ctl, int world, int self, int W, int H,
                                                        int tick)
{
    // PUSH_SPLIT blocks share one chunk (a chunk is 8 rows x W texels = 245 KB at 4K: one block would walk it in 60 dependent round trips)
    const int c = RowSet::interleave(self, world).chunk((int)blockIdx.x / PUSH_SPLIT), part = (int)blockIdx.x % PUSH_SPLIT, r0 = c * 8, r1 = min(r0 + 8, H);
    if (r0 < H)
        for (int q = 0; q < world; q++)
        {
            if (q == self) continue;
            const int a = max(r0, need.r0[q]), b = min(r1, need.r1[q]);
            if (b <= a) continue;
            const size_t first = (size_t)a * W, n = (size_t)(b - a) * W; // W is even: 16-byte pairs
            const uint4* s4 = reinterpret_cast<const uint4*>(imgs.p[self] + first);
            uint4*       d4 = reinterpret_cast<uint4*>(imgs.p[q] + first);
            for (size_t i = (size_t)part * blockDim.x + threadIdx.x; i < n / 2; i += (size_t)PUSH_SPLIT * blockDim.x) d4[i] = s4[i];
        }
    publish_when_grid_done(ctl, ticks, world, self, TICK_RT, tick);
}

// The two count images of the cooperative spp > 1 trace (SHARED_COUNT, by frame parity): allocated when a shadows / AO pass is
// linked, so only linked passes pay their 2 B per pass pixel (16.6 MB at 3840x2160, 66 MB at 7680x4320).  They exist before the
// first render, so switching spp on linked ranks needs no further collective.
int rt_alloc_counts(hr_pass* p)
{
    if ((p->kind != PASS_SHADOWS && p->kind != PASS_AO) || p->count_pp[0]) return HR_OK;
    for (int k = 0; k < 2; k++)
    {
        HR_CUDA(p->ctx, cudaMalloc((void**)&p->count_pp[k], (size_t)p->W * p->H));
        p->allocs.push_back(p->count_pp[k]);
        HR_CUDA(p->ctx, cudaMemset(p->count_pp[k], 0, (size_t)p->W * p->H));
        p->hist_local[SHARED_COUNT + k] = p->count_pp[k];
    }
    return HR_OK;
}

int peer_alloc_ticks(hr_pass* p)
{
    hr_ctx* ctx = p->ctx;
    if (p->sync_ticks) return HR_OK;
    HR_CUDA(ctx, cudaMalloc((void**)&p->sync_ticks, sizeof(int) * 2 * HR_MAX_RANKS));
    HR_CUDA(ctx, cudaMemset(p->sync_ticks, 0, sizeof(int) * 2 * HR_MAX_RANKS));
    HR_CUDA(ctx, cudaHostAlloc((void**)&p->sync_error, sizeof(int), cudaHostAllocMapped));
    *p->sync_error = 0;
    return HR_OK;
}

} // namespace

void hr_peer_register(hr_pass* p, void* const* imgs, int n)
{
    p->n_hist = n;
    for (int k = 0; k < n; k++) p->hist_local[k] = imgs[k];
}

// Collective over the NCCL communicator: all-gather the CUDA IPC handles of the `n` allocations local[] of every rank and map the
// peers': out[r * n + k] = rank r's allocation k in this process (local[k] for r == self).
static int ipc_exchange(hr_ctx* ctx, void* const* local, int n, void** out, cudaStream_t st)
{
    NcclApi&     N = nccl();
    const int    world = ctx->world;
    const size_t mine  = sizeof(cudaIpcMemHandle_t) * n;
    std::vector<cudaIpcMemHandle_t> h(n), all((size_t)n * world);
    for (int k = 0; k < n; k++) HR_CUDA(ctx, cudaIpcGetMemHandle(&h[k], local[k]));
    char *d_send = nullptr, *d_recv = nullptr;
    HR_CUDA(ctx, cudaMalloc((void**)&d_send, mine));
    HR_CUDA(ctx, cudaMalloc((void**)&d_recv, mine * world));
    HR_CUDA(ctx, cudaMemcpyAsync(d_send, h.data(), mine, cudaMemcpyHostToDevice, st));
    HR_NCCL(ctx, N.AllGather(d_send, d_recv, mine, ncclUint8, (ncclComm_t)ctx->nccl_comm, st));
    HR_CUDA(ctx, cudaMemcpyAsync(all.data(), d_recv, mine * world, cudaMemcpyDeviceToHost, st));
    HR_CUDA(ctx, cudaStreamSynchronize(st));
    cudaFree(d_send);
    cudaFree(d_recv);
    for (int r = 0; r < world; r++)
        for (int k = 0; k < n; k++)
        {
            void*& m = out[(size_t)r * n + k];
            if (r == ctx->rank) m = local[k];
            else HR_CUDA(ctx, cudaIpcOpenMemHandle(&m, all[(size_t)r * n + k], cudaIpcMemLazyEnablePeerAccess));
        }
    return HR_OK;
}

// Collective: map every peer's shared images and tick array.  Called from the first sharded render of the pass (all ranks render their
// passes in the same order).
int hr_peer_link_ipc(hr_pass* p, cudaStream_t st)
{
    hr_ctx* ctx = p->ctx;
    if (p->peers_linked || ctx->world <= 1 || !ctx->nccl_comm || p->n_hist == 0) return HR_OK;
    int rc = peer_alloc_ticks(p);
    if (rc == HR_OK) rc = rt_alloc_counts(p);
    if (rc != HR_OK) return rc;
    const int nh = p->n_hist + 1;
    void*     local[HR_MAX_SHARED + 1];
    void*     all[HR_MAX_RANKS * (HR_MAX_SHARED + 1)];
    for (int k = 0; k < p->n_hist; k++) local[k] = p->hist_local[k];
    local[p->n_hist] = p->sync_ticks;
    if ((rc = ipc_exchange(ctx, local, nh, all, st)) != HR_OK) return rc;
    for (int r = 0; r < ctx->world; r++)
    {
        for (int k = 0; k < p->n_hist; k++) p->hist_peer[r][k] = all[r * nh + k];
        p->peer_ticks[r] = static_cast<int*>(all[r * nh + p->n_hist]);
    }
    if (p->rt_bounds) { rc = rt_init_bounds(p); if (rc != HR_OK) return rc; }
    p->peers_linked = true;
    p->peers_ipc    = true;
    return HR_OK;
}

void hr_peer_unlink(hr_pass* p)
{
    hr_ddgi_unmap(p);
    if (p->peers_ipc)
        for (int r = 0; r < HR_MAX_RANKS; r++)
        {
            if (r == p->ctx->rank) continue;
            for (int k = 0; k < p->n_hist; k++)
                if (p->hist_peer[r][k]) cudaIpcCloseMemHandle(p->hist_peer[r][k]);
            if (p->peer_ticks[r]) cudaIpcCloseMemHandle(p->peer_ticks[r]);
        }
    p->peers_linked = p->peers_ipc = false;
    if (p->sync_ticks) cudaFree(p->sync_ticks);
    if (p->sync_error) cudaFreeHost(p->sync_error);
    p->sync_ticks = nullptr;
    p->sync_error = nullptr;
}

// History table for the reprojection kernel: images `img_k` / `aux_k` of every rank, rows split like hr_shard_rows(H).
void hr_peer_hist(const hr_pass* p, int img_k, int aux_k, int H, bool no_history, HistPeers* out)
{
    const hr_ctx* ctx = p->ctx;
    HistPeers     hp {};
    hp.no_history = no_history ? 1 : 0;
    if (hr_peer_linked(p))
    {
        hp.world = ctx->world;
        hp.self  = ctx->rank;
        for (int r = 0; r < ctx->world; r++)
        {
            int b, e;
            hr_shard_rows(H, r, ctx->world, &b, &e);
            hp.img[r]      = p->hist_peer[r][img_k];
            hp.aux[r]      = p->hist_peer[r][aux_k];
            hp.band_end[r] = e;
        }
    }
    else
    { // single GPU, or band emulation where the caller moves the bands itself (hr_shard_config + hr_pass_upload)
        hp.world       = 1;
        hp.self        = 0;
        hp.img[0]      = p->hist_local[img_k];
        hp.aux[0]      = p->hist_local[aux_k];
        hp.band_end[0] = H;
    }
    *out = hp;
}

// The device address of the time-out flag of the wait kernels, or the error of an earlier wait that timed out.
static int sync_error_ptr(hr_pass* p, int** d_err)
{
    hr_ctx* ctx = p->ctx;
    if (p->sync_error && *p->sync_error)
    {
        hr_set_error(ctx, "peer sync: timed out waiting for rank %d's frame tick (peer stopped, or ranks rendered different frame counts)", *p->sync_error - 1);
        return HR_ERR_NCCL;
    }
    HR_CUDA(ctx, cudaHostGetDevicePointer((void**)d_err, p->sync_error, 0));
    return HR_OK;
}

int hr_peer_wait(hr_pass* p, int slot, int tick, cudaStream_t st)
{
    if (!hr_peer_linked(p) || tick <= 0) return HR_OK;
    int* d_err = nullptr;
    int  rc    = sync_error_ptr(p, &d_err);
    if (rc != HR_OK) return rc;
    k_peer_wait<<<1, 32, 0, st>>>(p->sync_ticks + slot * HR_MAX_RANKS, p->ctx->world, p->ctx->rank, tick, d_err);
    p->ctx->launches++;
    return HR_OK;
}

int hr_peer_signal(hr_pass* p, int slot, int tick, cudaStream_t st)
{
    if (!hr_peer_linked(p)) return HR_OK;
    k_peer_signal<<<1, 32, 0, st>>>(peer_tick_ptrs(p), p->ctx->world, p->ctx->rank, slot, tick);
    p->ctx->launches++;
    return HR_OK;
}

int hr_push_chunks(hr_pass* p, int img, int tick, const int* need0, const int* need1, cudaStream_t st)
{
    hr_ctx*  ctx = p->ctx;
    NeedRows nd {};
    for (int r = 0; r < ctx->world; r++)
    {
        nd.r0[r] = need0[r];
        nd.r1[r] = need1[r];
    }
    const int mine = RowSet::interleave(ctx->rank, ctx->world).chunks(p->H);
    k_rt_push_chunks<<<(mine > 0 ? mine : 1) * PUSH_SPLIT, 256, 0, st>>>(peer_image_ptrs<uint2>(p, img), nd, peer_tick_ptrs(p), p->rt_bounds, ctx->world, ctx->rank,
                                                                        p->W, p->H, tick);
    ctx->launches++;
    return HR_OK;
}

// ---- DDGI atlases -----------------------------------------------------------------------------------------------------
// Linked DDGI passes split the probe stages by z-slices (hr_api_gi.inc).  The slices of a rank are one contiguous row range of each
// atlas, which the rank stores into every peer's atlas of this frame's ping-pong after its K19/K20 (k_ddgi_push), so every rank
// holds the complete atlases without a collective on the render stream.  The atlases are allocated when the grid is (re)initialised,
// after the passes were linked, so the push reads the peers' addresses at run time from this rank's table (SHARED_DDGI_TAB,
// [rank][irradiance 0, irradiance 1, depth 0, depth 1]):
//   * same-process ranks render one after another from one thread, so rank 0 enqueues the push of a re-initialisation frame before
//     rank 1 has allocated its new atlases.  After a (re)initialisation every rank writes its addresses into its peers' tables on
//     its stream and then publishes its ready tick (TICK_DDGI_READY) = that render's frame tick (k_ddgi_publish); in that render the push
//     is preceded by a one-warp wait until every peer's ready tick reached it (hr_api_gi.inc).
//   * IPC ranks re-initialise in the same render (they render the same scene with the same parameters): they exchange the new
//     atlases' IPC handles in a collective and write the mapped addresses into their own table; the push waits for nothing.
// One frame tick (TICK_ATLAS) orders the stores: a rank publishes tick N after its frame-N stores (last block of k_ddgi_push) and waits,
// before its K21, until every peer's tick reached N.
//   * Write before read: K21 and the reflections of frame N read atlas[mp] after that wait, so it is complete.
//   * Read before write: the frame-N stores go into atlas[mp], which a peer last read in frame N-1 (K18's infinite bounce, every
//     probe; K19's hysteresis, its slices) and, before that, in frame N-2 (its K21 and reflections).  This rank's frame-N push runs
//     after its frame N-1 wait saw that peer's tick N-1, which the peer published after its frame N-1 K18 and K19 and, in stream
//     order, after its frame N-2 consumers — as long as every consumer of the atlas runs on the render stream.
namespace {

struct AtlasSet { void* a[4]; };

__global__ void k_ddgi_publish(PeerPtrs<void*> tabs, PeerPtrs<int> ticks, AtlasSet mine, int world, int self, int tick)
{
    const int r = threadIdx.x;
    if (r >= world || r == self || !tabs.p[r] || !ticks.p[r]) return;
    for (int k = 0; k < 4; k++) tabs.p[r][self * 4 + k] = mine.a[k];
    __threadfence_system();
    st_release_sys(ticks.p[r] + TICK_DDGI_READY * HR_MAX_RANKS + self, tick);
}

// Bytes [i0, i1) of the irradiance atlas and [d0, d1) of the depth atlas (ping-pong mp) into every peer's atlas, at the addresses in
// this rank's table; the last block publishes the atlas tick.
__global__ void __launch_bounds__(256) k_ddgi_push(void* const* tab, const uint8_t* __restrict__ irr, const uint8_t* __restrict__ dep, size_t i0, size_t i1, size_t d0,
                                                   size_t d1, int mp, PeerPtrs<int> ticks, int* __restrict__ ctl, int world, int self, int tick)
{
    __shared__ uint8_t* s_dst[2][HR_MAX_RANKS];
    const int r = threadIdx.x;
    if (r < HR_MAX_RANKS)
    { // written by the peer before its ready tick (same process), or by this rank's host at the grid's initialisation (IPC)
        const bool peer = r < world && r != self;
        s_dst[0][r] = peer ? static_cast<uint8_t*>(*reinterpret_cast<void* const volatile*>(tab + r * 4 + mp)) : nullptr;
        s_dst[1][r] = peer ? static_cast<uint8_t*>(*reinterpret_cast<void* const volatile*>(tab + r * 4 + 2 + mp)) : nullptr;
    }
    __syncthreads();
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)gridDim.x * blockDim.x;
    push_bytes(irr, s_dst[0], world, self, i0, i1, tid, nthr);
    push_bytes(dep, s_dst[1], world, self, d0, d1, tid, nthr);
    publish_when_grid_done(ctl, ticks, world, self, TICK_ATLAS, tick);
}

} // namespace

void hr_ddgi_unmap(hr_pass* p)
{
    for (int r = 0; r < HR_MAX_RANKS; r++)
        for (int k = 0; k < 4; k++)
            if (p->ddgi_mapped[r][k])
            {
                cudaIpcCloseMemHandle(p->ddgi_mapped[r][k]);
                p->ddgi_mapped[r][k] = nullptr;
            }
}

int hr_ddgi_publish(hr_pass* p, int tick, cudaStream_t st)
{
    hr_ctx* ctx  = p->ctx;
    AtlasSet mine { { p->ddgi_irr[0], p->ddgi_irr[1], p->ddgi_depth[0], p->ddgi_depth[1] } };
    if (p->peers_ipc)
    {
        void* all[HR_MAX_RANKS * 4];
        int   rc = ipc_exchange(ctx, mine.a, 4, all, st);
        if (rc != HR_OK) return rc;
        for (int r = 0; r < ctx->world; r++)
            for (int k = 0; k < 4 && r != ctx->rank; k++) p->ddgi_mapped[r][k] = all[r * 4 + k];
        HR_CUDA(ctx, cudaMemcpyAsync(p->ddgi_tab, all, sizeof(void*) * 4 * ctx->world, cudaMemcpyHostToDevice, st));
        HR_CUDA(ctx, cudaStreamSynchronize(st));
        // The replaced atlases: every peer's stores into them completed before this render (this rank's stream passed its last atlas
        // wait, which saw every peer's tick published after its stores, and was synchronised at the re-initialisation), and every peer
        // closed its mappings of them before it entered the exchange above (hr_ddgi_unmap at its re-initialisation).
        for (void* a : p->ddgi_retired) cudaFree(a);
        p->ddgi_retired.clear();
    }
    else
    {
        k_ddgi_publish<<<1, 32, 0, st>>>(peer_image_ptrs<void*>(p, SHARED_DDGI_TAB), peer_tick_ptrs(p), mine, ctx->world, ctx->rank, tick);
        ctx->launches++;
    }
    p->ddgi_ready = tick;
    return HR_OK;
}

int hr_ddgi_push(hr_pass* p, int mp, size_t i0, size_t i1, size_t d0, size_t d1, int tick, cudaStream_t st)
{
    hr_ctx* ctx = p->ctx;
    k_ddgi_push<<<ctx->sm_count, 256, 0, st>>>(p->ddgi_tab, (const uint8_t*)p->ddgi_irr[mp], (const uint8_t*)p->ddgi_depth[mp], i0, i1, d0, d1, mp, peer_tick_ptrs(p),
                                               p->rt_bounds, ctx->world, ctx->rank, tick);
    ctx->launches++;
    return HR_OK;
}

// ---- shared ray mask + cost-balanced partition ------------------------------------------------------------------------
static int rt_init_bounds(hr_pass* p)
{ // first frame: uniform split of the mask rows
    hr_ctx*   ctx = p->ctx;
    const int MH = (p->H + 3) / 4, world = ctx->world;
    int       h[HR_MAX_RANKS + 1];
    for (int k = 0; k <= world; k++) h[k] = (int)(((long long)MH * k) / world);
    HR_CUDA(ctx, cudaMemcpy(p->rt_bounds, h, sizeof(int) * (world + 1), cudaMemcpyHostToDevice));
    return HR_OK;
}

bool hr_rt_share(hr_pass* p, int parity, RtShare* out)
{
    hr_ctx* ctx = p->ctx;
    if (!hr_peer_linked(p) || (p->kind != PASS_SHADOWS && p->kind != PASS_AO)) return false;
    RtShare sh {};
    sh.mask_local = static_cast<uint32_t*>(p->hist_local[SHARED_MASK + parity]);
    sh.bounds     = p->rt_bounds;
    sh.cost_acc   = p->rt_cost_acc;
    sh.world      = ctx->world;
    sh.self       = ctx->rank;
    *out          = sh;
    return true;
}

int hr_rt_share_finish(hr_pass* p, int parity, int tick, bool count, cudaStream_t st)
{
    hr_ctx*   ctx = p->ctx;
    const int MH = (p->H + 3) / 4;
    // mask row: one row of 4 * MW bytes; count image: 4 rows of W bytes, 8x the bytes of a mask row, so more blocks for the wider copy
    const int    blocks = count ? 128 : 32, rows = count ? 4 : 1, height = count ? p->H : MH;
    const size_t row_bytes = count ? (size_t)p->W : (size_t)4 * ((p->W + 7) / 8);
    k_rt_push<<<blocks, 256, 0, st>>>(peer_image_ptrs<uint8_t>(p, (count ? SHARED_COUNT : SHARED_MASK) + parity), peer_image_ptrs<uint32_t>(p, SHARED_COST), p->rt_bounds,
                                      p->rt_cost_acc, peer_tick_ptrs(p), ctx->world, ctx->rank, parity, MH, row_bytes, rows, height, tick);
    ctx->launches++;
    return HR_OK;
}

int hr_rt_wait_partition(hr_pass* p, int parity, int rt_tick, int hist_tick, cudaStream_t st)
{
    hr_ctx*   ctx = p->ctx;
    const int MH  = (p->H + 3) / 4;
    int*      d_err = nullptr;
    int       rc    = sync_error_ptr(p, &d_err);
    if (rc != HR_OK) return rc;
    k_rt_wait_partition<<<1, 32, 0, st>>>(p->sync_ticks, rt_tick, hist_tick, d_err, p->rt_cost_all + (size_t)parity * MH, MH, ctx->world, ctx->rank,
                                         hr_rt_share_cap(MH, ctx->world), p->rt_bounds);
    ctx->launches++;
    return HR_OK;
}

extern "C" {

int hr_shard_unique_id(void* out_128_bytes)
{
    if (!out_128_bytes) return HR_ERR_INVALID_ARG;
    NcclApi& N = nccl();
    if (!N.ok) { hr_set_error(nullptr, "hr_shard_unique_id: libnccl.so.2 could not be loaded"); return HR_ERR_NCCL; }
    ncclUniqueId id;
    if (N.GetUniqueId(&id) != ncclSuccess) { hr_set_error(nullptr, "ncclGetUniqueId failed"); return HR_ERR_NCCL; }
    memcpy(out_128_bytes, &id, sizeof(id));
    return HR_OK;
}

int hr_shard_init(hr_ctx* ctx, int rank, int world, const void* unique_id_128_bytes)
{
    HR_REQUIRE(ctx, ctx && world >= 1 && rank >= 0 && rank < world, HR_ERR_INVALID_ARG, "hr_shard_init: bad rank/world");
    HR_REQUIRE(ctx, world <= HR_MAX_RANKS, HR_ERR_UNSUPPORTED, "hr_shard_init: at most 8 ranks — one process per GPU of ONE box (peer history uses CUDA IPC mappings)");
    ctx->rank  = rank;
    ctx->world = world;
    if (world == 1) return HR_OK;
    HR_REQUIRE(ctx, unique_id_128_bytes, HR_ERR_INVALID_ARG, "hr_shard_init: unique id required for world > 1");
    NcclApi& N = nccl();
    HR_REQUIRE(ctx, N.ok, HR_ERR_NCCL, "hr_shard_init: libnccl.so.2 could not be loaded");
    HR_CUDA(ctx, cudaSetDevice(ctx->device));
    ncclUniqueId id;
    memcpy(&id, unique_id_128_bytes, sizeof(id));
    ncclComm_t comm;
    HR_NCCL(ctx, N.CommInitRank(&comm, world, id, rank));
    ctx->nccl_comm = comm;
    return HR_OK;
}

// Same-process DDGI ranks allocate their grids from a pool of their own, in stream order (hr_api_gi.inc).  `pass`'s rank stores into `peer`'s
// atlases, so a peer on another device grants this rank's device access to its pool (pool memory is not covered by peer access).
static int ddgi_pool_create(hr_pass* p)
{
    if (p->ddgi_pool) return HR_OK;
    cudaMemPoolProps props {};
    props.allocType     = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id   = p->ctx->device;
    HR_CUDA(p->ctx, cudaMemPoolCreate(&p->ddgi_pool, &props));
    return HR_OK;
}

static int ddgi_pool_link(hr_pass* pass, hr_pass* peer)
{
    int rc = ddgi_pool_create(pass);
    if (rc == HR_OK) rc = ddgi_pool_create(peer);
    if (rc != HR_OK || pass->ctx->device == peer->ctx->device) return rc;
    cudaMemAccessDesc a {};
    a.location.type = cudaMemLocationTypeDevice;
    a.location.id   = pass->ctx->device;
    a.flags         = cudaMemAccessFlagsProtReadWrite;
    HR_CUDA(pass->ctx, cudaMemPoolSetAccess(peer->ddgi_pool, &a, 1));
    return HR_OK;
}

// Same-process peers (N ranks emulated on one GPU, or a multi-GPU single-process host): rank `rank`'s history lives in
// `peer`'s images.  Every pass of the group must be linked with every other before the first sharded render.
int hr_shard_link_local(hr_pass* pass, int rank, hr_pass* peer)
{
    if (!pass || !peer) return HR_ERR_INVALID_ARG;
    hr_ctx* ctx = pass->ctx;
    HR_REQUIRE(ctx, rank >= 0 && rank < ctx->world && rank < HR_MAX_RANKS && pass->kind == peer->kind && pass->n_hist == peer->n_hist && pass->n_hist > 0 &&
                        pass->W == peer->W && pass->H == peer->H && !pass->peers_ipc,
               HR_ERR_INVALID_ARG, "hr_shard_link_local: passes do not match (kind / size / rank) or the pass has no peer history");
    int rc = peer_alloc_ticks(pass);
    if (rc == HR_OK) rc = peer_alloc_ticks(peer);
    if (rc == HR_OK) rc = rt_alloc_counts(pass);
    if (rc == HR_OK) rc = rt_alloc_counts(peer);
    if (rc == HR_OK && pass->kind == PASS_DDGI) rc = ddgi_pool_link(pass, peer);
    if (rc != HR_OK) return rc;
    for (int k = 0; k < pass->n_hist; k++) pass->hist_peer[rank][k] = peer->hist_local[k];
    pass->peer_ticks[rank] = peer->sync_ticks;
    for (int k = 0; k < pass->n_hist; k++) pass->hist_peer[ctx->rank][k] = pass->hist_local[k];
    pass->peer_ticks[ctx->rank] = pass->sync_ticks;
    bool all = true;
    for (int r = 0; r < ctx->world; r++) all = all && pass->peer_ticks[r] != nullptr;
    pass->peers_linked = all;
    if (all && pass->rt_bounds) return rt_init_bounds(pass);
    return HR_OK;
}

int hr_shard_set_gather(hr_ctx* ctx, int gather_final_output)
{
    if (!ctx) return HR_ERR_INVALID_ARG;
    ctx->gather_final = gather_final_output != 0;
    return HR_OK;
}

int hr_shard_shutdown(hr_ctx* ctx)
{
    if (!ctx) return HR_ERR_INVALID_ARG;
    if (ctx->nccl_comm) { nccl().CommDestroy((ncclComm_t)ctx->nccl_comm); ctx->nccl_comm = nullptr; }
    ctx->rank  = 0;
    ctx->world = 1;
    return HR_OK;
}

} // extern "C"
