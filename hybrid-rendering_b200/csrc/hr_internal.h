// hr_internal.h — internal types of libhr_b200 (not part of the ABI).
#pragma once
#include "../../include/hr_api.h"
#include "tex_px.cuh"
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <string>
#include <vector>

#define HR_VERSION 100

// ---- error plumbing -------------------------------------------------------------------------------
void        hr_set_error(hr_ctx* ctx, const char* fmt, ...);
#define HR_CUDA(ctx, expr)                                                                                         \
    do {                                                                                                           \
        cudaError_t _e = (expr);                                                                                   \
        if (_e != cudaSuccess) {                                                                                   \
            hr_set_error((ctx), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__);       \
            return _e == cudaErrorMemoryAllocation ? HR_ERR_OUT_OF_MEMORY : HR_ERR_CUDA;                           \
        }                                                                                                          \
    } while (0)
#define HR_CHECK_LAUNCH(ctx) HR_CUDA(ctx, cudaGetLastError())
#define HR_REQUIRE(ctx, cond, code, msg)                                   \
    do {                                                                   \
        if (!(cond)) { hr_set_error((ctx), "%s", (msg)); return (code); } \
    } while (0)

// ---- device-side views ----------------------------------------------------------------------------
struct GBufLevelDev {          // one mip of one G-buffer slot
    int            W, H;
    const uint2*   gb2;        // RGBA16F as 4 halves = uint2
    const uint2*   gb3;        // RGBA16F
    const float*   depth;      // D32
    const uint32_t* gb1;       // RGBA8 (may be null)
};

struct BvhDev {                // traversal view of hr_scene
    const float4* nodes;       // 4 x float4 per node (see bvh_build.cu)
    const float4* tris;        // 3 x float4 per triangle in leaf order: (v0,prim) (e1,0) (e2,0)
    const float4* wnodes;      // 4-wide nodes, 8 x float4 each, indexed like `nodes` (bvh_build.cu k_widen); per-lane traversal
    int           root_is_valid;
};

struct FrameConsts {           // what kernels need from hr_frame (passed by value as a kernel param)
    float    view_proj_inverse[16];
    float    prev_view_proj[16];
    float    cam_pos[4];
    hr_light light;
    float    z_buffer_params[4];
    float    camera_delta[3];
    uint32_t num_frames;
    unsigned long long* ray_ctr; // per-pass ray counters (hr_pass_get_stats): [kind][HR_RAY_CTR_SLOTS] spread over 32-byte slots; may be null
};
#define HR_RAY_CTR_SLOTS 32
#define HR_RAY_CTR_STRIDE 4 // unsigned long longs between slots (32 bytes: one sector each)

// ---- objects ----------------------------------------------------------------------------------------
#define HR_MAX_RANKS 8
#define HR_MAX_SHARED 8

// Temporal history as the reprojection kernels see it (shard.cu, "peer history").  Row y of the previous frame's history
// images lives on the rank that owns y (band_end[r] = first row NOT owned by ranks 0..r); img[r] / aux[r] are that rank's
// full-size images — this GPU's own for r == self, NVLink peer mappings (CUDA IPC) otherwise.  Single GPU: world = 1.
// no_history: first frame after creation / hr_pass_reset_history — every history texel reads as 0 (cleared images).
struct HistPeers {
    const void* img[HR_MAX_RANKS];
    const void* aux[HR_MAX_RANKS];
    int         band_end[HR_MAX_RANKS];
    int         world, self, no_history;
};

struct GBufSlot {
    void*  gb1[HR_MAX_MIPS]   = {};
    void*  gb2[HR_MAX_MIPS]   = {};
    void*  gb3[HR_MAX_MIPS]   = {};
    float* depth[HR_MAX_MIPS] = {};
    bool   owns_mip0          = true; // false when bound zero-copy
    bool   valid              = false;
};

struct hr_ctx {
    int          device = 0;
    std::string  last_error;
    // blue noise (device)
    uint8_t*     d_sobol    = nullptr; // 256*4
    uint8_t*     d_scr_rank = nullptr; // 128*128*4
    uint8_t*     d_scr_rank_slot[9] = {}; // per sample count (BlueNoiseSpp): [0] aliases d_scr_rank
    bool         bn_set     = false;
    // g-buffer
    int          gb_w = 0, gb_h = 0;
    GBufSlot     slot[2];
    void*        owned_mip0[2][4] = {}; // library-owned mip0 storage (gb1,gb2,gb3,depth) kept when a slot is bound zero-copy
    // streaming host frames: a third mip0 surface receives frame N+1 over PCIe (upload_stream) while frame N renders;
    // hr_gbuffer_commit_staged swaps it with a slot's storage (no copy)
    void*        staging_mip0[4] = {};
    bool         staging_has_gb1 = false, staged_pending = false;
    cudaStream_t upload_stream = nullptr;
    cudaEvent_t  ev_staged = nullptr, ev_storage_free = nullptr;
    bool         storage_free_recorded = false;
    // scene
    hr_scene*    scene = nullptr;
    // sharding
    int          rank = 0, world = 1;
    void*        nccl_comm = nullptr; // ncclComm_t when hr_shard_init was called (NCCL is dlopen'ed lazily, see shard.cu)
    bool         gather_final = true;   // all-gather every pass's final output after the render (hr_shard_set_gather)
    cudaStream_t comm_stream = nullptr; // band exchanges run here, overlapped with the next pass / next frame's ray trace
    // profiling
    bool         profiling = false;
    uint64_t     launches  = 0;
    int          sm_count  = 132;
    cudaStream_t build_stream = nullptr;
    uint32_t*    d_brdf_lut = nullptr;  // 512 x 512 RG16F split-sum LUT (hr_brdf_lut_set); null: the IBL specular terms are 0
    unsigned long long* gbuf_ray_ctr = nullptr; // primary rays of hr_gbuffer_render (same slot layout as hr_pass::ray_ctr)
};

struct hr_scene {
    hr_ctx*  ctx     = nullptr;
    uint32_t n_tris  = 0;
    uint32_t n_nodes = 0;
    // inputs kept on device for rebuilds
    float*    d_tri_verts = nullptr; // n*9 world-space
    uint32_t* d_prim_inst = nullptr; // instance (= mesh id) per primitive
    // build scratch
    uint64_t* d_keys = nullptr, *d_keys_sorted = nullptr;
    uint32_t* d_vals = nullptr, *d_vals_sorted = nullptr;
    float*    d_tri_aabb = nullptr;  // n*6
    int*      d_bounds_i = nullptr;  // 6 ordered-int min/max
    int2*     d_children = nullptr;  // n-1
    int2*     d_ranges   = nullptr;  // n-1 (first,last)
    int*      d_parent   = nullptr;  // 2n-1
    float*    d_node_aabb = nullptr; // (n-1)*6
    int*      d_flags    = nullptr;  // n-1
    void*     d_sort_tmp = nullptr;
    size_t    sort_tmp_bytes = 0;
    void*     d_ploc = nullptr;      // PLOC builder scratch (cluster ping-pong, nearest neighbours, scan)
    size_t    ploc_bytes = 0;
    // outputs
    float4*   d_nodes = nullptr;     // n_nodes*4
    float4*   d_wnodes = nullptr;    // n_nodes*8: 4-wide nodes (k_widen)
    int*      d_depth = nullptr;     // height of the binary tree (k_depth)
    float4*   d_tris  = nullptr;     // n*3
    // shading data (reflections / ddgi hit shading)
    float4*   d_vnormals = nullptr;  // n*3 world-space vertex normals in primitive order
    uint32_t* d_prim_mat = nullptr;  // material index per primitive
    hr_material* d_materials = nullptr;
    uint32_t  n_materials = 0;
    // material textures (hr_scene_set_textures): per-primitive texture coordinates are kept on the host by hr_scene_build and only uploaded when
    // textures are bound; `tex` is what the TEX instantiations of the shading kernels receive (n_textures == 0: the untextured kernels run)
    std::vector<float> h_vuv;        // 6 per primitive
    std::vector<float> h_vtb;        // 18 per primitive: world-space unit tangents of the three corners, then bitangents (normal maps)
    float*         d_vuv = nullptr;
    float*         d_vtb = nullptr;
    uint32_t*      d_texels = nullptr;
    tex::TexDesc*  d_tex_desc = nullptr;
    tex::MatTex*   d_mat_tex = nullptr;
    float*         d_srgb_lut = nullptr;
    tex::TexDev    tex {};
    hr_scene_info info {};
};

enum PassKind { PASS_SHADOWS = 1, PASS_AO = 2, PASS_REFLECTIONS = 3, PASS_DDGI = 4, PASS_DEFERRED = 5, PASS_TAA = 6, PASS_TONEMAP = 7, PASS_PATH_TRACER = 8 };

struct StageTimer { // one Rec per profiled render; hr_pass_stage_times averages and recycles them
    struct Rec { std::vector<std::string> names; std::vector<cudaEvent_t> ev; };
    std::vector<Rec>         recs;
    std::vector<cudaEvent_t> pool;
    std::vector<std::string> last_names;
};

struct hr_pass {
    hr_ctx* ctx  = nullptr;
    int     kind = 0;
    int     W = 0, H = 0;      // pass resolution
    int     W0 = 0, H0 = 0;    // full resolution
    int     scale = 0;         // = g_buffer_mip
    bool    first = true;      // own m_first_frame (ray_traced_ao.cpp:829)
    int     final_which = 0;
    // generic image table: which -> (ptr, w, h, format)
    struct Img { void* p = nullptr; int w = 0, h = 0, fmt = 0; };
    Img     img[16];
    Img     out_view[128];     // indexed by `which` (filled per render)
    Img     hist_view[8][2];   // history surfaces by `which` (< 8) and frame parity, known from creation: hr_pass_upload before the first render
    // shadows
    uint32_t* mask = nullptr;
    uint8_t*  count = nullptr;       // spp > 1: unoccluded rays per pixel (allocated on first use)
    __half2*  temporal_out = nullptr;
    uint2*    moments[2] = { nullptr, nullptr };
    __half2*  prev_image[2] = { nullptr, nullptr }; // [ping_pong]: written by frame N's feedback iteration, read by frame N+1's temporal
    __half2*  atrous[2] = { nullptr, nullptr };
    uint8_t*  tile_flags = nullptr;
    __half*   upsample_out = nullptr;
    // ao
    __half*   ao_color[2] = { nullptr, nullptr };
    __half*   ao_len[2] = { nullptr, nullptr };
    __half*   ao_blur[2] = { nullptr, nullptr };
    // reflections (RGBA16F images as uint2)
    uint2*    refl_rt = nullptr;
    uint2*    refl_rt_pp[2] = { nullptr, nullptr };   // ray-trace output by frame parity when the ranks trace cooperatively (refl_rt_pp[0] == refl_rt)
    unsigned int* work_counters = nullptr;             // tile / job counters of this pass's persistent kernels
    float4*   refl_hits = nullptr;                     // wavefront K12: one hit record (t, primitive, u, v) per pixel
    uint2*    refl_temporal[2] = { nullptr, nullptr }; // current_output[pp] (also the history of the next frame)
    uint2*    refl_moments[2] = { nullptr, nullptr };
    uint2*    refl_prev = nullptr;                     // prev_image (blur_as_input)
    uint2*    refl_atrous[2] = { nullptr, nullptr };
    uint2*    refl_upsample = nullptr;
    // ddgi
    hr_ddgi_uniforms ddgi_u {};
    bool      ddgi_grid_valid = false;
    const void* ddgi_scene = nullptr;
    float     ddgi_key[4] = { 0, 0, 0, 0 };            // probe_distance, irradiance_oct, depth_oct, rays_per_probe
    int       ddgi_mp = 0;                             // m_ping_pong (ddgi.cpp:103)
    bool      ddgi_first = true;
    uint2*    ddgi_radiance = nullptr;
    uint2*    ddgi_dirdepth = nullptr;
    uint2*    ddgi_irr[2] = { nullptr, nullptr };
    uint32_t* ddgi_depth[2] = { nullptr, nullptr };
    uint2*    ddgi_sample = nullptr;
    uint2*    deferred_out = nullptr;                  // deferred shading combine: RGBA16F (Lo, 1)
    uint2*    post_img[2] = { nullptr, nullptr };      // TAA: m_image[2] (temporal_aa.cpp:196-212); path tracer: images[2]; [0] = tone map RGBA8
    uint32_t* pt_prim = nullptr;                       // path tracer: primitive hit by the last frame's primary ray (0xFFFFFFFF = sky)
    uint32_t  pt_frame_idx = 0;                        // GroundTruthPathTracer::m_frame_idx
    int       pt_ping_pong = 0;                        // GroundTruthPathTracer::m_ping_pong
    std::vector<void*> ddgi_grid_allocs;
    // asynchronous band exchange (shard.cu): ev_ready = pass kernels done on the caller's stream, ev_done = exchange done on
    // ctx->comm_stream.  Whoever next touches an exchanged image (next frame's temporal stage, hr_pass_output/download)
    // first makes its stream wait on ev_done (hr_wait_exchange).
    cudaEvent_t ev_ready = nullptr, ev_done = nullptr;
    bool        xchg_pending = false;
    // peer history (shard.cu): the history images of every rank mapped into this process, and the frame ticks that order
    // "rank q finished writing frame N's history" before "rank r's frame N+1 reprojection reads it"
    bool        peers_linked = false, peers_ipc = false;
    int         n_hist = 0;                          // shared images: 0-3 history (shadows: prev_image[2], moments[2]; AO: colour[2], length[2]),
                                                     // 4-5 ray mask [frame parity], 6 ray-trace cost table [2][mask rows]
    void*       hist_local[HR_MAX_SHARED] = {};
    void*       hist_peer[HR_MAX_RANKS][HR_MAX_SHARED] = {}; // [rank][image]; own rank = hist_local
    int*        sync_ticks = nullptr;                // [2][HR_MAX_RANKS] ticks written by the peers into THIS rank's memory: [0] history, [1] ray trace
    uint32_t*   mask_pp[2] = { nullptr, nullptr };   // ray mask by frame parity (mask_pp[0] == mask); peers push their rows into both copies' owner
    uint32_t*   rt_cost_all = nullptr;               // [2][MH] per-mask-row trace cost of the frame (all ranks' rows, pushed by their owners)
    uint32_t*   rt_cost_acc = nullptr;               // [MH] this rank's accumulation scratch (atomicAdd per warp), drained by the push kernel
    int*        rt_bounds = nullptr;                 // [world+1] mask-row partition of the NEXT frame's ray trace (device side, cost balanced); [HR_MAX_RANKS+1] = job counter, [+2] = push blocks done
    int*        peer_ticks[HR_MAX_RANKS] = {};       // the peers' tick arrays (we write slot [self])
    int*        sync_error = nullptr;                // set by the wait kernel on time-out
    int         epoch = 0;                           // renders of this pass so far
    unsigned long long* ray_ctr = nullptr;           // [2 kinds][HR_RAY_CTR_SLOTS * HR_RAY_CTR_STRIDE]: primary / secondary rays traced since the last hr_pass_get_stats
    uint64_t    n_renders = 0;                       // renders since the last hr_pass_get_stats
    int         last_rows[2] = { 0, 0 };             // rows [r0, r1) the last render's denoise stages covered (tile statistics)
    StageTimer timer;
    std::vector<void*> allocs;
};

// rt_shade.cu / ddgi_update.cu / svgf_reflections.cu
void launch_ddgi_ray_trace(const hr_scene* sc, const hr_ddgi_uniforms& d, const void* irr_prev, const void* depth_prev, const hr_light& light, const float* rot16,
                           uint32_t num_frames, uint32_t infinite_bounces, float gi_intensity, const float* sky3, int probe0, int probe1, void* radiance,
                           void* dirdepth, unsigned long long* ray_ctr, cudaStream_t st);
void launch_ddgi_probe_update(const hr_ddgi_uniforms& d, const void* radiance, const void* dirdepth, const void* prev_irr, const void* prev_depth, void* out_irr,
                              void* out_depth, int first_frame, int probe0, int probe1, cudaStream_t st);
void launch_ddgi_sample_probe_grid(const GBufLevelDev& g, const FrameConsts& fc, const hr_ddgi_uniforms& d, const void* irr, const void* depth, float gi_intensity,
                                   void* out, int row0, int row1, cudaStream_t st);
void launch_reflections_ray_trace(const hr_scene* sc, const GBufLevelDev& g, const FrameConsts& fc, const hr_ddgi_uniforms* d, const void* irr, const void* depth,
                                  float bias, float trim, int sample_gi, int approximate_with_ddgi, float gi_intensity, float rough_ddgi_intensity, const float* sky3,
                                  const uint8_t* sobol, const uint8_t* srk, void* out, void* hits, int row0, int row1, int chunk_first, int chunk_stride,
                                  int spp, const void* brdf_lut, float ibl_intensity, cudaStream_t st); // chunk_stride > 1: only the 8-row chunks c = chunk_first + i * chunk_stride (rows are ignored)
void launch_reflections_temporal(const GBufLevelDev& cur, const GBufLevelDev& prev, const void* input, const HistPeers& hist, const FrameConsts& fc, float alpha,
                                 float moments_alpha, int approximate_with_ddgi, void* out, void* mom_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st);
int  launch_reflections_atrous(const GBufLevelDev& g, const void* in, const uint8_t* tile_flags, int radius, int step, float phi_color, float phi_normal,
                               float sigma_depth, int approximate_with_ddgi, void* out, int row0, int row1, unsigned int* counters, cudaStream_t st);
void launch_upsample_vec4(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, void* out, int row0, int row1, cudaStream_t st);

// ---- row-band sharding (shard.cu) ---------------------------------------------------------------------
// An image whose rows are owned band-wise by the ranks.  The band partition is defined on the PASS height `H`
// (hr_shard_rows); the image's own rows are band << shift (full-res upsample outputs) or band / div (ray masks),
// clamped to `rows` (the image's real height).
struct ExchangeItem { void* base; size_t row_bytes; int H; int shift; int div; int rows; };
// peer history (shard.cu)
void hr_peer_register(hr_pass* p, void* const* imgs, int n);
int  hr_peer_link_ipc(hr_pass* p, cudaStream_t st);
void hr_peer_unlink(hr_pass* p);
void hr_peer_hist(const hr_pass* p, int img_k, int aux_k, int H, bool no_history, HistPeers* out);
int  hr_peer_wait(hr_pass* p, int which, int tick, cudaStream_t st);   // which: 0 history ticks, 1 ray-trace ticks
int  hr_peer_signal(hr_pass* p, int which, int tick, cudaStream_t st);
// Cost-balanced ray trace over the whole image with the masks pushed to every peer (trace.cu / shard.cu).
struct RtShare {
    uint32_t*     mask_local; // this rank's mask image of this frame's parity (k_rt_push copies the share to the peers)
    const int*    bounds;     // [world+1] mask-row partition (device)
    uint32_t*     cost_acc;   // [MH] local cost accumulation
    int           world, self;
};
// most mask rows one rank may be handed: twice the uniform share (+4); the whole image for world <= 2
inline int hr_rt_share_cap(int MH, int world) { const int c = 2 * ((MH + world - 1) / world) + 4; return c < MH ? c : MH; }
bool hr_rt_share(hr_pass* p, int parity, RtShare* out); // false when the pass is not linked to peers
int  hr_rt_share_finish(hr_pass* p, int parity, int tick, cudaStream_t st); // push costs, signal the ray-trace tick
int  hr_rt_wait_partition(hr_pass* p, int parity, int rt_tick, int hist_tick, cudaStream_t st); // wait for the peers' ticks, then next frame's bounds
void launch_shadows_ray_trace_shared(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float bias, const uint8_t* sobol, const uint8_t* sr,
                                     const RtShare& sh, cudaStream_t st);
void launch_ao_ray_trace_shared(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float ray_length, float bias, const uint8_t* sobol,
                                const uint8_t* sr, const RtShare& sh, cudaStream_t st);
// Interleaved cooperative ray trace of the reflections pass (shard.cu): rank r traces the 8-row chunks c with c % world == r of the
// WHOLE image into its own image and copies every chunk to the ranks whose denoise stages read it (rows [need0[q], need1[q]));
// the last block publishes the ray-trace tick.
int hr_refl_push_chunks(hr_pass* p, int parity, int tick, const int* need0, const int* need1, cudaStream_t st);
// Rows of an image of height H owned by this context's rank (all rows when world == 1).
void hr_band(const hr_ctx* ctx, int H, int* b0, int* b1);
// [b0 - halo, b1 + halo) clamped to [0, H); halo must be a multiple of 8 so tile alignment is kept.
inline void hr_extend(int b0, int b1, int halo, int H, int* e0, int* e1)
{
    *e0 = b0 - halo < 0 ? 0 : b0 - halo;
    *e1 = b1 + halo > H ? H : b1 + halo;
}
// Make every rank's copy of each image complete: rank r broadcasts its band of every item (one NCCL group).
// Asynchronous: enqueued on ctx->comm_stream after everything already enqueued on `st`; completion is p->ev_done.
int hr_shard_exchange(hr_pass* p, const ExchangeItem* items, int n, cudaStream_t st);
// Same, with explicit per-rank row ranges [row0[r], row1[r]) (rank r broadcasts its rows of every item): DDGI atlases split by
// probe z-slices.  SYNCHRONOUS with respect to `st`: the exchange is enqueued on `st` itself.
struct RowRangeItem { void* base; size_t row_bytes; };
int hr_shard_exchange_rows(hr_pass* p, const RowRangeItem* items, int n, const int* row0, const int* row1, cudaStream_t st);
// Make `st` wait for the pass's pending exchange (no-op when nothing is pending).
void hr_wait_exchange(hr_pass* p, cudaStream_t st);

// ---- kernel launchers (defined in the .cu files) -----------------------------------------------------
void launch_gbuffer_render(const hr_scene* sc, const hr_frame* f, int W, int H, int row0, int row1, int chunk_first, int chunk_stride, void* gb1, void* gb2, void* gb3,
                           float* depth, unsigned long long* ray_ctr, cudaStream_t st); // gbuffer.cu
void launch_deferred(const GBufLevelDev& g, const FrameConsts& fc, const void* shadow, int shadow_channels, const void* ao, const void* reflections, const void* gi,
                     const float* env3, const void* brdf_lut, void* out, int row0, int row1, cudaStream_t st); // deferred.cu
// rt_shade.cu: ground-truth path tracer
void launch_path_trace(const hr_scene* sc, const hr_frame* f, int W, int H, uint32_t num_frames, uint32_t max_ray_bounces, float roughness_multiplier, const float* sky3,
                       const void* prev, void* out, uint32_t* out_prim, unsigned long long* ray_ctr, cudaStream_t st);
// post.cu
void launch_taa(const GBufLevelDev& g, const void* current, int current_channels, const void* history, const float* jitter_xy, float feedback_min, float feedback_max,
                int sharpen, void* out, cudaStream_t st);
void launch_blit_rgba16f(const void* src, int channels, int W, int H, void* out, cudaStream_t st);
void launch_tonemap(const void* src, int channels, int W, int H, float exposure, int single_channel, void* out_rgba8, cudaStream_t st);
// stats.cu (measurement helpers, not on the frame path)
void launch_tile_stats(const uint8_t* flags, int TW, int t0, int t1, unsigned long long* d_out, cudaStream_t st);
void launch_drain_ray_counters(unsigned long long* ctr, unsigned long long* d_out, cudaStream_t st);
void launch_checksum(const void* base, size_t byte0, size_t byte1, unsigned long long* d_out, cudaStream_t st);
int hr_launch_build_mips(hr_ctx* ctx, GBufSlot& s, int W, int H, cudaStream_t st);
int hr_bvh_build(hr_scene* sc, cudaStream_t st);
BvhDev hr_bvh_view(const hr_scene* sc);

// Function attributes (opt-in shared memory sizes) are per device: launchers keep one flag per device, not per process, so
// a process that drives several GPUs configures each of them.  Returns true the first time it is called for the current
// device with this flag array.
inline bool hr_once_per_device(bool (&done)[64])
{
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (done[dev]) return false;
    done[dev] = true;
    return true;
}


void launch_shadows_ray_trace(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float bias, const uint8_t* sobol, const uint8_t* sr,
                              uint32_t* mask, int row0, int row1, cudaStream_t st);
void launch_ao_ray_trace(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float ray_length, float bias, const uint8_t* sobol,
                         const uint8_t* sr, uint32_t* mask, int row0, int row1, cudaStream_t st);
void launch_shadows_ray_trace_count(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float bias, const uint8_t* sobol, const uint8_t* sr,
                                    uint8_t* count, int spp, int row0, int row1, cudaStream_t st);
void launch_ao_ray_trace_count(const GBufLevelDev& g, const BvhDev& bvh, const FrameConsts& fc, float ray_length, float bias, const uint8_t* sobol,
                               const uint8_t* sr, uint8_t* count, int spp, int row0, int row1, cudaStream_t st);
void launch_shadows_temporal_count(const GBufLevelDev& cur, const GBufLevelDev& prev, const uint8_t* count, int spp, const HistPeers& hist, const FrameConsts& fc,
                                   float alpha, float moments_alpha, __half2* out, uint2* moments_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st);
void launch_ao_temporal_count(const GBufLevelDev& cur, const GBufLevelDev& prev, const uint8_t* count, int spp, const HistPeers& hist, const FrameConsts& fc,
                              float alpha, __half* out, __half* len_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st);
void launch_trace_any(const BvhDev& bvh, const float* rays, size_t n, uint32_t* out, cudaStream_t st);
void launch_trace_closest(const BvhDev& bvh, const float* rays, size_t n, float* out_t, uint32_t* out_prim, float* out_uv, cudaStream_t st);

void launch_shadows_temporal(const GBufLevelDev& cur, const GBufLevelDev& prev, const uint32_t* mask, const HistPeers& hist,
                             const FrameConsts& fc, float alpha, float moments_alpha, __half2* out, uint2* moments_out, uint8_t* tile_flags,
                             int row0, int row1, cudaStream_t st);
void launch_shadows_atrous(const GBufLevelDev& g, const __half2* in, const uint8_t* tile_flags, int radius, int step, float phi_vis, float phi_n,
                           float sigma_z, float power, __half2* out, int row0, int row1, cudaStream_t st);
void launch_upsample_scalar(const GBufLevelDev& g0, const GBufLevelDev& gm, const void* in, int in_channels, float sky_value, float power,
                            __half* out, int row0, int row1, cudaStream_t st);
void launch_ao_temporal(const GBufLevelDev& cur, const GBufLevelDev& prev, const uint32_t* mask, const HistPeers& hist,
                        const FrameConsts& fc, float alpha, __half* out, __half* len_out, uint8_t* tile_flags, int row0, int row1, cudaStream_t st);
void launch_ao_blur(const GBufLevelDev& g, const __half* in, const uint8_t* tile_flags, const float* zbp, int dirx, int diry, int radius, __half* out,
                    int row0, int row1, cudaStream_t st);
