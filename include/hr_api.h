/*
 * hr_api.h — C ABI of the H100-native ray-trace + SVGF hot path.
 *
 * This is the drop-in boundary for the four render passes of diharaw/hybrid-rendering
 * (RayTracedShadows, RayTracedAO, RayTracedReflections, DDGI) and the stages either side of them
 * (G-buffer producer; DeferredShading, TemporalAA, ToneMap, GroundTruthPathTracer).  The reference has no
 * FFI of its own; its seam is the C++ pass-class interface
 *     Pass(backend, CommonResources*, GBuffer*, RayTraceScale)   src/ray_traced_shadows.h:23
 *     void render(cmd_buf)                                       src/ray_traced_shadows.h:26
 *     DescriptorSet::Ptr output_ds()                             src/ray_traced_shadows.h:28
 * and each entry point below cites the reference interface it replaces.
 *
 * Conventions: every function returns 0 (HR_OK) or a negative hr_status; the message
 * is available from hr_last_error().  All pointers are plain; "device" pointers are CUDA
 * device addresses on the context's GPU.  All work is enqueued on the caller's stream
 * (a cudaStream_t passed as void*); no hidden synchronisation except where documented
 * (hr_*_download, hr_scene_build).  One hr_ctx per GPU; a ctx is not thread-safe.
 * No torch / C++ types cross this boundary.
 */
#ifndef HR_API_H
#define HR_API_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HR_API __attribute__((visibility("default")))

typedef enum hr_status {
    HR_OK                = 0,
    HR_ERR_INVALID_ARG   = -1,
    HR_ERR_CUDA          = -2,
    HR_ERR_OUT_OF_MEMORY = -3,
    HR_ERR_NOT_READY     = -4, /* e.g. render before scene / g-buffer / blue-noise were set */
    HR_ERR_UNSUPPORTED   = -5,
    HR_ERR_NCCL          = -6
} hr_status;

typedef struct hr_ctx   hr_ctx;   /* CommonResources + Backend equivalent, one per GPU (src/common.h:181-243) */
typedef struct hr_scene hr_scene; /* RayTracedScene equivalent: device LBVH instead of BLAS/TLAS            */
typedef struct hr_pass  hr_pass;  /* one of the four pass objects                                           */

/* ------------------------------------------------------------------------------------------------
 * Plain-data mirrors of the reference's per-frame constants
 * ---------------------------------------------------------------------------------------------- */

/* struct Light, src/common.h:106-158: data0 = dir.xyz|intensity, data1 = pos.xyz|radius,
 * data2 = color.rgb, data3 = type|cos_outer|cos_inner.  data0.xyz points TOWARDS the light
 * (src/main.cpp:963). */
typedef struct hr_light {
    float data0[4];
    float data1[4];
    float data2[4];
    float data3[4];
} hr_light;

enum { HR_LIGHT_DIRECTIONAL = 0, HR_LIGHT_POINT = 1, HR_LIGHT_SPOT = 2 }; /* src/shaders/common.glsl:23-25 */

/* struct UBO, src/common.h:161-179 (416 bytes).  Matrices are column-major like glm. */
typedef struct hr_ubo {
    float    view_inverse[16];
    float    proj_inverse[16];
    float    view_proj_inverse[16];
    float    prev_view_proj[16];
    float    view_proj[16];
    float    cam_pos[4];
    float    current_prev_jitter[4];
    hr_light light;
} hr_ubo;

/* The CommonResources fields a pass pulls every frame (src/common.h:186-191). */
typedef struct hr_frame {
    hr_ubo   ubo;
    uint32_t num_frames;         /* CommonResources::num_frames; blue-noise sample index            */
    int32_t  ping_pong;          /* CommonResources::ping_pong; selects current/history G-buffer    */
    int32_t  first_frame;        /* CommonResources::first_frame                                    */
    float    z_buffer_params[4]; /* src/main.cpp:253-254                                            */
    float    camera_delta[3];    /* CommonResources::camera_delta (reflections temporal)            */
    float    frame_time;         /* CommonResources::frame_time                                     */
} hr_frame;

/* RayTraceScale, src/common.h:39-44 */
enum { HR_SCALE_FULL = 0, HR_SCALE_HALF = 1, HR_SCALE_QUARTER = 2 };

/* ------------------------------------------------------------------------------------------------
 * Context  (replaces dw::vk::Backend + CommonResources construction, src/common.cpp:302-322)
 * ---------------------------------------------------------------------------------------------- */
HR_API int         hr_init(int device, hr_ctx** out);
HR_API int         hr_shutdown(hr_ctx* ctx);
HR_API const char* hr_last_error(hr_ctx* ctx); /* ctx may be NULL: returns the last global error */
HR_API int         hr_version(void);

/* Blue-noise tables (src/blue_noise.cpp:5-33, sampled by src/shaders/bnd_sampler.glsl:4-24).
 * sobol: 256 x RGBA8 (sobol_256_4d.png); scrambling_ranking: 128 x 128 x RGBA8 (…_1spp.png). Host pointers. */
HR_API int hr_bluenoise_set(hr_ctx* ctx, const uint8_t* sobol_256x4, const uint8_t* scrambling_ranking_128x128x4);
/* The reference loads nine scrambling / ranking tables, one per sample count (BlueNoiseSpp, src/blue_noise.h:5-16;
 * scrambling_ranking_128x128_2d_{1,2,4,...,256}spp.png, src/blue_noise.cpp:9-19) and binds the 1-spp one to every pass.  slot =
 * log2(spp) in 0..8.  A pass rendered with spp = 2^slot > 1 samples the table of its slot when one was set, the 1-spp table
 * (hr_bluenoise_set, = slot 0) otherwise. */
HR_API int hr_bluenoise_set_slot(hr_ctx* ctx, int slot, const uint8_t* scrambling_ranking_128x128x4);

/* Split-sum BRDF LUT (dw::BRDFIntegrateLUT: textures/brdf_lut.bin, 512 x 512 RG16F, extras/brdf_preintegrate_lut.cpp:8-31; bound
 * with the bilinear CLAMP_TO_EDGE sampler, src/common.cpp:814-816).  Host pointer to 512 * 512 * 2 halves.  Until it is set the IBL
 * specular terms (reflections_ray_trace.rchit:97-104, deferred.frag:167-170) are 0.  The sky / prefiltered environment cubemaps
 * are replaced by the constant colour passed in the pass parameters (sky_color). */
HR_API int hr_brdf_lut_set(hr_ctx* ctx, const uint16_t* rg16f_512x512);

/* ------------------------------------------------------------------------------------------------
 * Scene  (replaces dw::RayTracedScene + driver BLAS/TLAS build,
 *         external/dwSampleFramework/extras/ray_traced_scene.cpp:196-248, src/mesh.cpp:169-231)
 * ---------------------------------------------------------------------------------------------- */

/* dw::Vertex, external/dwSampleFramework/include/mesh.h:16-23 (80 bytes) */
typedef struct hr_vertex {
    float position[4];
    float tex_coord[4];
    float normal[4];
    float tangent[4];
    float bitangent[4];
} hr_vertex;

/* Material constants used when no textures are bound (src/shaders/scene_descriptor_set.glsl:180-229). */
typedef struct hr_material {
    float albedo[4];   /* linear rgb, a */
    float emissive[4];
    float roughness;
    float metallic;
    float _pad[2];
} hr_material;

/* One (instance, sub-mesh) draw range: model matrix + index range + material.
 * ray_traced_scene.cpp:573-613 (instance data), mesh.h SubMesh. */
typedef struct hr_instance {
    float    model[16]; /* column-major */
    uint32_t first_index;
    uint32_t index_count;
    uint32_t base_vertex;
    uint32_t material_idx;
} hr_instance;

/* Builds the device BVH over all instances' world-space triangles: 63-bit Morton codes + radix sort, then PLOC
 * agglomerative clustering with treelet restructuring for the surface-area cost (default) or the Karras radix tree + bottom-up
 * fit (hr_debug_set key 3), collapsed into <= 2-triangle leaves and packed into 64-byte two-child nodes.  Host pointers in; synchronises the context's build
 * stream before returning.  Fails with HR_ERR_UNSUPPORTED when the tree is deeper than the traversal stack (64).  Every
 * built scene gets a new process-wide serial number; a DDGI pass re-initialises its probe grid when it next renders a scene
 * with another serial, even one allocated at a destroyed scene's address. */
HR_API int hr_scene_build(hr_ctx* ctx, const hr_vertex* vertices, size_t n_vertices, const uint32_t* indices, size_t n_indices,
                          const hr_instance* instances, size_t n_instances, const hr_material* materials, size_t n_materials,
                          hr_scene** out);
HR_API int hr_scene_destroy(hr_scene* scene);
HR_API int hr_scene_set_current(hr_ctx* ctx, hr_scene* scene); /* CommonResources::current_scene() */
/* Build statistics / debug: n_tris, n_nodes, build time of the last build in ms. */
typedef struct hr_scene_info {
    uint64_t n_triangles;
    uint64_t n_nodes;
    float    bounds_min[3];
    float    bounds_max[3];
    float    build_ms;
    uint32_t depth;        /* height of the binary tree (edges root -> deepest triangle); the traversal stacks hold HR_BVH_MAX_DEPTH pending nodes */
} hr_scene_info;
#define HR_BVH_MAX_DEPTH 63 /* a deeper tree is refused by hr_scene_build / hr_scene_rebuild (HR_ERR_UNSUPPORTED), never traversed lossily */
HR_API int hr_scene_get_info(hr_scene* scene, hr_scene_info* out);
/* Re-run only the device build (the reference rebuilds its TLAS every frame, src/main.cpp:74). */
HR_API int hr_scene_rebuild(hr_scene* scene, void* stream);
/* Read-only copy of the built tree to host memory, for measuring its quality: the traversal layout of bvh_build.cu, n_nodes
 * nodes of 4 float4 (both child boxes, then the child links; child < 0 is a leaf ~((first << 3) | (count - 1))) and n_triangles
 * triangles of 3 float4 (v0 with the primitive index's bits in w, e1, e2) in leaf order.  nodes_bytes must be n_nodes * 64 and
 * tris_bytes n_triangles * 48; a NULL destination is skipped.  Synchronises the device. */
HR_API int hr_scene_download_bvh(hr_scene* scene, void* nodes, size_t nodes_bytes, void* tris, size_t tris_bytes);

/* Material textures (Material::load + the bindless s_Textures array, extras/ray_traced_scene.cpp:345-420, scene_descriptor_set.glsl:84-93,180-218).
 * textures: 8-bit images, 1, 2 or 4 channels (what Image::create_from_file produces: RGB files arrive as RGBA), host pointers, copied;
 * srgb = 1 for albedo images (material.cpp:114).  bindings: one entry per material of the scene (n_materials must equal the scene's):
 * texture index or -1 = use the hr_material constant; *_channel selects the component of the roughness / metallic image (glTF: 1 / 2).
 * Sampled at every hit of the reflections / DDGI / path-tracer shading and by hr_gbuffer_render (albedo, metallic, roughness, normal map)
 * at mip 0 with bilinear filtering and REPEAT addressing.  Emissive maps are accepted and unused (no shader of the reference reads them).
 * n_textures = 0 removes them.  Not to be called while work that uses the scene is in flight. */
typedef struct hr_texture {
    int32_t        width, height;
    int32_t        channels; /* 1, 2 or 4 */
    int32_t        srgb;
    const uint8_t* data;     /* width * height * channels bytes, rows top to bottom */
} hr_texture;
typedef struct hr_material_textures {
    int32_t albedo, normal, roughness, roughness_channel, metallic, metallic_channel, emissive;
} hr_material_textures;
HR_API int hr_scene_set_textures(hr_scene* scene, const hr_texture* textures, size_t n_textures, const hr_material_textures* bindings, size_t n_materials);

/* Generic ray query against the current scene, for tests of the traversal kernel.
 * rays: n x 8 floats {ox,oy,oz,tmin, dx,dy,dz,tmax} (device).  any-hit: out_hit[n] uint32 (1 = hit).
 * closest: out_t[n] float (tmax if miss), out_prim[n] uint32 (0xFFFFFFFF if miss), out_uv[n*2]. */
HR_API int hr_trace_any(hr_ctx* ctx, const float* d_rays, size_t n, uint32_t* d_out_hit, void* stream);
HR_API int hr_trace_closest(hr_ctx* ctx, const float* d_rays, size_t n, float* d_out_t, uint32_t* d_out_prim, float* d_out_uv, void* stream);

/* ------------------------------------------------------------------------------------------------
 * G-buffer  (replaces GBuffer::output_ds()/history_ds(), src/g_buffer.cpp:201-211; formats :254-263)
 *   gb1   RGBA8   albedo.rgb | metallic
 *   gb2   RGBA16F oct normal.xy | motion.xy (prev_uv - cur_uv)
 *   gb3   RGBA16F roughness | curvature | mesh id | linear z (view-space w; -1 = sky)
 *   depth D32     z_clip / w_clip, 1.0 = sky
 * Two slots mirror the reference's double buffering: slot[frame.ping_pong] is "current",
 * slot[!frame.ping_pong] is "history".
 * ---------------------------------------------------------------------------------------------- */
#define HR_MAX_MIPS 3

typedef struct hr_gbuffer_desc {
    int32_t     width, height; /* mip 0 */
    const void* gb1;           /* may be NULL (not read on the hot path) */
    const void* gb2;
    const void* gb3;
    const void* depth;
} hr_gbuffer_desc;

/* Allocate library-owned device storage for both slots (mips 0..HR_MAX_MIPS-1). */
HR_API int hr_gbuffer_create(hr_ctx* ctx, int width, int height);
/* Host -> device copy of mip 0 into slot, then NEAREST mip chain on device (g_buffer.cpp:236-244). Async on stream. */
HR_API int hr_gbuffer_upload(hr_ctx* ctx, int slot, const hr_gbuffer_desc* host_mip0, void* stream);
/* Streaming host frames (copy / compute overlap).  hr_gbuffer_stage_upload starts the host -> device copy of the NEXT
 * frame's mip 0 into a third, library-owned surface on the library's own upload stream and returns immediately (pinned
 * host memory required for the copy to be asynchronous; the host buffers must stay untouched until the frame was
 * committed and `stream` reached that point).  hr_gbuffer_commit_staged makes `stream` wait for that copy, swaps the
 * staged surface into `slot` (pointer swap, no copy) and builds the mip chain on `stream` — afterwards the slot behaves
 * exactly as after hr_gbuffer_upload.  One staged frame at a time: stage, commit, stage, commit ... */
HR_API int hr_gbuffer_stage_upload(hr_ctx* ctx, const hr_gbuffer_desc* host_mip0);
HR_API int hr_gbuffer_commit_staged(hr_ctx* ctx, int slot, void* stream);
/* Device -> device variant (inputs already resident in HBM). */
HR_API int hr_gbuffer_copy_from_device(hr_ctx* ctx, int slot, const hr_gbuffer_desc* dev_mip0, void* stream);
/* Zero-copy: bind caller-owned device mip-0 images as slot; the library only builds mips 1.. from them. */
HR_API int hr_gbuffer_bind_device(hr_ctx* ctx, int slot, const hr_gbuffer_desc* dev_mip0, void* stream);
/* G-buffer producer on the device (SURVEY.md §8 f1): replaces the reference's raster G-buffer pass (src/g_buffer.cpp:100-263,
 * src/shaders/g_buffer.{vert,frag}) with a primary-visibility ray cast over the current scene's BVH — depth, octahedral
 * normal, motion vector from frame->ubo.prev_view_proj, curvature from the 2x2-quad normal differences, mesh id, linear z,
 * albedo / metallic — into the library-owned storage of `slot`, then the NEAREST mip chain.  A headless frame then needs
 * only the 496-byte hr_frame from the host instead of a 24 B/pixel upload.  rows [row0, row1) (multiples of 8, or the image
 * height; row1 <= 0 = the whole image) let a sharded rank produce just the rows it consumes.  Async on `stream`.  The CPU
 * statement oracle/orc_gbuffer.cpp produces the same bits. */
HR_API int hr_gbuffer_render(hr_ctx* ctx, int slot, const hr_frame* frame, int row0, int row1, void* stream);
/* Sharded variant: only the rows this rank's full-resolution passes consume — its band +- halo_rows (temporal / a-trous stages;
 * pass the recompute halo + the reprojection reach the camera motion needs) and the 8-row chunks it traces in the interleaved
 * cooperative ray trace.  The other rows of the slot keep their old contents.  world == 1: the whole image. */
HR_API int hr_gbuffer_render_sharded(hr_ctx* ctx, int slot, const hr_frame* frame, int halo_rows, void* stream);
/* Pipelined variant: the ray cast for the NEXT frame runs on the library's side stream into a third surface while the caller's
 * stream still renders the current frame (whose passes read both slots); hr_gbuffer_commit_staged(slot, stream) then swaps it in.
 * Same protocol as hr_gbuffer_stage_upload: stage, commit, stage, commit ... */
HR_API int hr_gbuffer_stage_render(hr_ctx* ctx, const hr_frame* frame);
/* Read back one mip of a slot (tests). which: 1,2,3 = gb1..3, 0 = depth. Synchronous. */
HR_API int hr_gbuffer_download(hr_ctx* ctx, int slot, int mip, int which, void* host_dst, size_t bytes);

/* ------------------------------------------------------------------------------------------------
 * Pass outputs
 * ---------------------------------------------------------------------------------------------- */
typedef enum hr_format { HR_FMT_R32_UINT = 1, HR_FMT_R16F = 2, HR_FMT_RG16F = 3, HR_FMT_RGBA16F = 4, HR_FMT_R8_UINT = 5, HR_FMT_RGBA8 = 6 } hr_format;

typedef struct hr_image {
    void*   data; /* device pointer, dense rows (pitch = width * texel size) */
    int32_t width, height;
    int32_t format; /* hr_format */
} hr_image;

/* ------------------------------------------------------------------------------------------------
 * Ray-traced shadows  (src/ray_traced_shadows.{h,cpp}; shaders/shadows/ *)
 * ---------------------------------------------------------------------------------------------- */
typedef struct hr_shadows_params { /* defaults: src/ray_traced_shadows.h:50-115 */
    float   bias;               /* 0.5  */
    float   alpha;              /* 0.01 */
    float   moments_alpha;      /* 0.2  */
    float   phi_visibility;     /* 10   */
    float   phi_normal;         /* 32   */
    float   sigma_depth;        /* 1    */
    float   power;              /* 1.2  */
    int32_t radius;             /* 1    */
    int32_t filter_iterations;  /* 4    */
    int32_t feedback_iteration; /* 1    */
    int32_t denoise;            /* 1    */
    int32_t spp;                /* 1: the reference's single ray per pixel.  > 1 (SURVEY.md §8d configs 4-5, not in the reference):
                                 * spp rays per pixel, sample index num_frames * spp + s; output 0 becomes an R8_UINT W x H image
                                 * of unoccluded-ray counts, the temporal stage uses visibility = count / spp.  Linked ranks
                                 * (hr_shard_init, or hr_shard_config + hr_shard_link_local) trace the count image cooperatively
                                 * like the 1-spp mask: each traces a cost-balanced share of the rows and pushes it to every peer,
                                 * so output 0 is complete on every rank; results are bit-identical to one GPU.  A linked shadows /
                                 * AO pass holds two W x H count images from link time (2 B per pass pixel: 16.6 MB at 3840 x 2160);
                                 * 0 is read as 1; at most 255 */
} hr_shadows_params;

/* OutputType, src/ray_traced_shadows.h:10-16 (+ internals for tests) */
enum {
    HR_SHADOWS_OUT_RAY_TRACE             = 0, /* R32_UINT mask ceil(W/8) x ceil(H/4) */
    HR_SHADOWS_OUT_TEMPORAL_ACCUMULATION = 1, /* RG16F (visibility, variance) */
    HR_SHADOWS_OUT_ATROUS                = 2, /* RG16F */
    HR_SHADOWS_OUT_UPSAMPLE              = 3, /* R16F full-res (scale != FULL) */
    HR_SHADOWS_OUT_MOMENTS               = 4, /* RGBA16F (m1, m2, history length, 0) of this frame */
    HR_SHADOWS_OUT_PREV_IMAGE            = 5, /* RG16F history image (a-trous output after feedback_iteration) */
    HR_SHADOWS_OUT_TILE_FLAGS            = 6, /* R8_UINT per 8x8 tile: 1 = denoise list, 0 = shadow list */
    HR_SHADOWS_OUT_FINAL                 = 100 /* what output_ds() returns (src/ray_traced_shadows.cpp:135-155) */
};

HR_API void hr_shadows_default_params(hr_shadows_params* p);
HR_API int  hr_shadows_create(hr_ctx* ctx, int width, int height, int scale, hr_pass** out); /* ctor, ray_traced_shadows.cpp:60-96 */
HR_API int  hr_shadows_render(hr_pass* pass, const hr_frame* frame, const hr_shadows_params* params, void* stream); /* render(), :100-116 */

/* ------------------------------------------------------------------------------------------------
 * Ray-traced ambient occlusion  (src/ray_traced_ao.{h,cpp}; shaders/ao/ *)
 * ---------------------------------------------------------------------------------------------- */
typedef struct hr_ao_params { /* defaults: src/ray_traced_ao.h:51-110 */
    float   ray_length;  /* 7.0  */
    float   bias;        /* 0.3  */
    float   alpha;       /* 0.01 */
    float   power;       /* 1.2  */
    int32_t blur_radius; /* 4    */
    int32_t denoise;     /* 1    */
    int32_t spp;         /* 1; > 1: see hr_shadows_params.spp (count image, cooperative trace on linked ranks) */
} hr_ao_params;

enum {
    HR_AO_OUT_RAY_TRACE             = 0, /* R32_UINT mask */
    HR_AO_OUT_TEMPORAL_ACCUMULATION = 1, /* R16F */
    HR_AO_OUT_BILATERAL_BLUR        = 2, /* R16F */
    HR_AO_OUT_UPSAMPLE              = 3, /* R16F full-res */
    HR_AO_OUT_HISTORY_LENGTH        = 4, /* R16F */
    HR_AO_OUT_TILE_FLAGS            = 6, /* R8_UINT */
    HR_AO_OUT_FINAL                 = 100
};

HR_API void hr_ao_default_params(hr_ao_params* p);
HR_API int  hr_ao_create(hr_ctx* ctx, int width, int height, int scale, hr_pass** out);               /* ray_traced_ao.cpp:71-90 */
HR_API int  hr_ao_render(hr_pass* pass, const hr_frame* frame, const hr_ao_params* params, void* stream); /* :98-112 */

/* ------------------------------------------------------------------------------------------------
 * DDGI  (src/ddgi.{h,cpp}; shaders/gi/ *)
 * ---------------------------------------------------------------------------------------------- */
/* DDGIUniforms, src/ddgi.cpp:14-32 <-> gi_common.glsl:10-28 (scalar layout, 88 bytes) */
typedef struct hr_ddgi_uniforms {
    float   grid_start_position[3];
    float   grid_step[3];
    int32_t probe_counts[3];
    float   max_distance;
    float   depth_sharpness;
    float   hysteresis;
    float   normal_bias;
    float   energy_preservation;
    int32_t irradiance_probe_side_length;
    int32_t irradiance_texture_width;
    int32_t irradiance_texture_height;
    int32_t depth_probe_side_length;
    int32_t depth_texture_width;
    int32_t depth_texture_height;
    int32_t rays_per_probe;
    int32_t visibility_test;
} hr_ddgi_uniforms;

typedef struct hr_ddgi_params { /* defaults: src/ddgi.h:52-115; per-scene overrides src/main.cpp:1084-1145 */
    int32_t infinite_bounces;          /* 1    */
    float   infinite_bounce_intensity; /* 1.7  */
    int32_t rays_per_probe;            /* 256  */
    int32_t visibility_test;           /* 1    */
    float   probe_distance;            /* 1.0 (4.0 test scenes, 50.0 Sponza) */
    float   recursive_energy_preservation; /* 0.85 */
    int32_t irradiance_oct_size;       /* 8    */
    int32_t depth_oct_size;            /* 16   */
    float   hysteresis;                /* 0.98 */
    float   depth_sharpness;           /* 50   */
    float   normal_bias;               /* 0.25 */
    float   gi_intensity;              /* 1.0 (sample_probe_grid) */
    float   sky_color[3];              /* constant-colour environment replacing the sky cubemap (ENVIRONMENT "None" = 0) */
} hr_ddgi_params;

enum {
    HR_DDGI_OUT_RADIANCE        = 0, /* RGBA16F rays_per_probe x num_probes  (gi_ray_trace.rgen:98) */
    HR_DDGI_OUT_DIRECTION_DEPTH = 1, /* RGBA16F rays_per_probe x num_probes  (:99) */
    HR_DDGI_OUT_IRRADIANCE      = 2, /* RGBA16F atlas written this frame */
    HR_DDGI_OUT_DEPTH           = 3, /* RG16F atlas written this frame */
    HR_DDGI_OUT_SAMPLE          = 4, /* RGBA16F per-pixel irradiance (gi_sample_probe_grid.comp) */
    HR_DDGI_OUT_FINAL           = 100
};

HR_API void hr_ddgi_default_params(hr_ddgi_params* p);
HR_API int  hr_ddgi_create(hr_ctx* ctx, int width, int height, int scale, hr_pass** out); /* ddgi.cpp:60-76 */
/* render(), ddgi.cpp:89-104.  random_orientation: column-major mat4 (the reference draws it from std::mt19937 seeded by
 * std::random_device, ddgi.cpp:73,788 — non-deterministic; the caller supplies it).  The probe grid is (re)initialised from
 * the current scene's bounds on the first render, when the current scene is another hr_scene_build's (even at a reused address),
 * when probe_distance / irradiance_oct_size / depth_oct_size / rays_per_probe change, and after a failed initialisation
 * (ddgi.cpp:150-169).  A re-initialised grid starts like the first frame: zero atlases, no hysteresis, no infinite bounce.  The
 * other parameters are applied every frame.  Out-of-range parameters return HR_ERR_INVALID_ARG and change nothing; a grid of
 * more than 2^20 probes returns HR_ERR_UNSUPPORTED and leaves the pass without a grid (the next render initialises one).
 * Sharded (world > 1): linked to its peers (hr_shard_init, or hr_shard_link_local for ranks of one process) rank r traces and updates
 * the probes of the z-slices [cz * r / world, cz * (r + 1) / world) and stores their atlas rows into every peer's atlases, so outputs 2
 * and 3 are complete on every rank once the stream passes the render; the per-pixel sample (output 4 / 100) covers the rank's band.
 * Consumers of the atlases (hr_reflections_render, downloads) must run on the render stream, and all ranks must re-initialise their
 * grids in the same render; the replaced grid is freed in that render (same-process ranks: in stream order on the render stream), so
 * re-initialisations do not accumulate memory.  Not linked (hr_shard_config only): every probe on every rank.  Outputs 0 and 1 hold the
 * rank's probes. */
HR_API int hr_ddgi_render(hr_pass* pass, const hr_frame* frame, const hr_ddgi_params* params, const float* random_orientation16, void* stream);
/* The uniforms of the current grid; HR_ERR_NOT_READY before the first render and after a failed grid initialisation. */
HR_API int hr_ddgi_get_uniforms(hr_pass* pass, hr_ddgi_uniforms* out);

/* ------------------------------------------------------------------------------------------------
 * Ray-traced reflections  (src/ray_traced_reflections.{h,cpp}; shaders/reflections/ *)
 * ---------------------------------------------------------------------------------------------- */
typedef struct hr_reflections_params { /* defaults: src/ray_traced_reflections.h:51-123 */
    float   bias;                  /* 0.5  */
    float   trim;                  /* 0.8  */
    int32_t sample_gi;             /* 1    */
    int32_t approximate_with_ddgi; /* 1    */
    float   gi_intensity;          /* 0.5  */
    float   rough_ddgi_intensity;  /* 0.5  */
    float   ibl_indirect_specular_intensity; /* 0.05; needs prefiltered environment + BRDF LUT assets: term is 0 here */
    float   alpha;                 /* 0.01 */
    float   moments_alpha;         /* 0.2  */
    int32_t blur_as_input;         /* 0    */
    float   phi_color;             /* 10   */
    float   phi_normal;            /* 32   */
    float   sigma_depth;           /* 1    */
    int32_t radius;                /* 1    */
    int32_t filter_iterations;     /* 4    */
    int32_t feedback_iteration;    /* 1    */
    int32_t denoise;               /* 1    */
    float   sky_color[3];          /* miss colour (skybox cubemap replaced by a constant) */
    int32_t spp;                   /* 1: the reference's single ray per pixel.  > 1 (SURVEY.md §8d configs 4-5, not in the reference): the GGX
                                    * lobe draws spp directions (sample index num_frames * spp + s) and stores the mean of the clamped
                                    * radiance; the ray length is the first sample's; 0 is read as 1.  Linked ranks trace the
                                    * interleaved 8-row chunks at every spp (DESIGN.md §9), bit-identical to one GPU */
} hr_reflections_params;

enum {
    HR_REFLECTIONS_OUT_RAY_TRACE             = 0, /* RGBA16F (rgb clamped to 0.7, a = ray length or -1) */
    HR_REFLECTIONS_OUT_TEMPORAL_ACCUMULATION = 1, /* RGBA16F (rgb, variance) */
    HR_REFLECTIONS_OUT_ATROUS                = 2, /* RGBA16F */
    HR_REFLECTIONS_OUT_UPSAMPLE              = 3, /* RGBA16F full-res */
    HR_REFLECTIONS_OUT_MOMENTS               = 4, /* RGBA16F (m1, m2, history length, 0) */
    HR_REFLECTIONS_OUT_TILE_FLAGS            = 6, /* R8_UINT: 1 = denoise list, 0 = copy list */
    HR_REFLECTIONS_OUT_FINAL                 = 100
};

HR_API void hr_reflections_default_params(hr_reflections_params* p);
HR_API int  hr_reflections_create(hr_ctx* ctx, int width, int height, int scale, hr_pass** out); /* ray_traced_reflections.cpp:67-103 */
/* render(cmd_buf, DDGI*), ray_traced_reflections.cpp:107-123; ddgi may be NULL (then sample_gi / approximate_with_ddgi are off). */
HR_API int hr_reflections_render(hr_pass* pass, const hr_frame* frame, const hr_reflections_params* params, hr_pass* ddgi, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Deferred shading combine  (SURVEY.md §8 f2: src/deferred_shading.{h,cpp}; shaders/deferred.frag:146-205)
 * Lo = direct_lighting * shadows.r + indirect_lighting(DDGI irradiance, reflections, BRDF LUT) * AO  ->  RGBA16F (Lo, 1), full res;
 * pixels at the G-buffer's clear depth (1.0) show the sky box = env_color (render_skybox, deferred_shading.cpp:69, skybox.frag).
 * Any of the four passes may be NULL (the reference's push constants shadow / ao / reflections / gi = 0: visibility 1, AO 1, the
 * environment colour as prefiltered reflection / irradiance).  Reads GB1 (albedo, metallic): bind or render it.
 * ---------------------------------------------------------------------------------------------- */
typedef struct hr_deferred_params {
    float env_color[3]; /* constant environment: evaluate_sh9_irradiance / prefiltered cubemap value */
} hr_deferred_params;
HR_API int hr_deferred_create(hr_ctx* ctx, int width, int height, hr_pass** out);
HR_API int hr_deferred_render(hr_pass* pass, const hr_frame* frame, const hr_deferred_params* params, hr_pass* shadows, hr_pass* ao, hr_pass* reflections, hr_pass* ddgi,
                              void* stream); /* output: hr_pass_output(pass, HR_..._OUT_FINAL = 100) */

/* ------------------------------------------------------------------------------------------------
 * Post-processing  (SURVEY.md §8 f4: src/temporal_aa.{h,cpp} + shaders/taa.comp; src/tone_map.{h,cpp} + shaders/tone_map.frag)
 * Both passes read the FINAL output (which = 100) of any other pass at full resolution — the reference binds the deferred,
 * shadows, AO, reflections or DDGI output by visualisation type (temporal_aa.cpp:136-147, tone_map.cpp:106-125); R16F / RG16F
 * inputs are read as (r, 0, 0, 1) / (r, g, 0, 1) like a sampler does.
 * Sharded (world > 1): each rank resolves / maps its band hr_shard_rows(H).  TAA reads the input's 3x3 neighbourhood one row beyond
 * the band and its own previous output wherever the motion vector reprojects it, so it needs complete inputs: the input pass's
 * gathered final output, the G-buffer rows of the band + 2 (the sharded G-buffer's halo covers them) and its own output, which it
 * gathers after every render (8 B/px).  With world > 1 and the gather off (hr_shard_set_gather(ctx, 0)) hr_taa_render returns
 * HR_ERR_UNSUPPORTED and changes nothing.  Its reset blit copies the whole gathered input on every rank.  The tone map reads only its
 * band of the input and gathers its RGBA8 output (4 B/px) when the gather is on; with the gather off each rank holds its band only.
 * ---------------------------------------------------------------------------------------------- */
typedef struct hr_taa_params { /* defaults: src/temporal_aa.h:54-59 */
    float   feedback_min;      /* 0.88 */
    float   feedback_max;      /* 0.97 */
    int32_t sharpen;           /* 1    */
    int32_t reset_every_frame; /* 1 = the reference as written: m_reset is initialised true and never cleared (temporal_aa.cpp:112,
                                * temporal_aa.h:57), so every frame first overwrites the history image with the current input and the
                                * resolve blends the frame with itself.  0 = what the code evidently intends: the blit happens on the
                                * first render (and after hr_pass_reset_history) only and the history accumulates */
} hr_taa_params;
HR_API void hr_taa_default_params(hr_taa_params* p);
/* TemporalAA::update (temporal_aa.cpp:66-81): the sub-pixel jitter of frame `num_frames` — Halton(2, 3) sample
 * (num_frames % 16) + 1 mapped to [-1, 1), divided by (width, height).  The caller multiplies its projection by
 * translate(jitter.xy, 0) and stores (current, previous) in hr_frame.ubo.current_prev_jitter (main.cpp:941-957).  Pure function. */
HR_API void hr_taa_jitter(uint32_t num_frames, int width, int height, float out_xy[2]);
HR_API int  hr_taa_create(hr_ctx* ctx, int width, int height, hr_pass** out); /* temporal_aa.cpp:44-56: two RGBA16F images */
/* TemporalAA::render (temporal_aa.cpp:83-172): resolves `input`'s final output against this pass's previous output using the
 * current G-buffer slot's depth and motion vectors and frame->ubo.current_prev_jitter.xy; writes image[frame->ping_pong] (RGBA16F,
 * rgb clamped to [0, 1], a = 1), which = 100.  Bit-specified (oracle/orc_post.cpp). */
HR_API int hr_taa_render(hr_pass* pass, const hr_frame* frame, const hr_taa_params* params, hr_pass* input, void* stream);

typedef struct hr_tonemap_params { /* tone_map.h:41, push constants tone_map.frag:24-29 */
    float   exposure;       /* 1.0 */
    int32_t single_channel; /* 0; 1 = grey-scale visualisation of a one-channel pass (.rrr), no curve */
} hr_tonemap_params;
HR_API void hr_tonemap_default_params(hr_tonemap_params* p);
HR_API int  hr_tonemap_create(hr_ctx* ctx, int width, int height, hr_pass** out);
/* ToneMap::render (tone_map.cpp:44-150): exposure, ACES film curve, gamma 1 / 2.2 -> RGBA8 UNORM image of the input's size
 * (the reference renders into the swap chain; row y of the output is row y of the input), which = 100. */
HR_API int hr_tonemap_render(hr_pass* pass, const hr_tonemap_params* params, hr_pass* input, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Ground-truth progressive path tracer  (SURVEY.md §8 f4: src/ground_truth_path_tracer.{h,cpp}; shaders/ground_truth/ *)
 * One jittered primary ray per pixel per render; first hit shaded with the soft-shadowed punctual light and one cosine-lobe sky
 * sample (each with its shadow ray); running average over renders.  As written in the reference the indirect bounce is disabled
 * (its traceRayEXT is commented out, ground_truth_path_trace.rchit:92-104), so max_ray_bounces changes nothing unless trace_indirect
 * is 1.  Needs only the
 * scene and frame->ubo.{view_inverse, proj_inverse, light}: no G-buffer.
 * Sharded (world > 1): linked to its peers (hr_shard_init, or hr_shard_link_local for ranks of one process) rank r traces the 8-row
 * chunks c with c % world == r of the whole image; with only hr_shard_config it traces its band hr_shard_rows(H).  A rank's running
 * average covers its own rows, which are bit for bit the single-GPU rows; its ray counters (hr_pass_get_stats) count its own rows, the
 * ranks' counts sum to the single-GPU counts.  With the gather on (the default) a linked rank pushes its chunks into every peer's
 * image and its render ends with a wait on `stream` for every peer's chunks of that render: FINAL / COLOR are then complete on every
 * rank.  Consumers of the output must run on the render stream.  The gather needs an even width: an odd one returns HR_ERR_UNSUPPORTED
 * and changes nothing.  With the gather off FINAL / COLOR hold the rank's own rows only; PRIMITIVE and PATH_HASH always do.
 * hr_pass_reset_history must be called on all ranks together.
 * ---------------------------------------------------------------------------------------------- */
typedef struct hr_path_tracer_params {
    int32_t max_ray_bounces;      /* 2 (ground_truth_path_tracer.h:28; the ctor overwrites it with the device's recursion limit) */
    float   roughness_multiplier; /* 1.0 (CommonResources::roughness_multiplier, common.h:193) */
    float   sky_color[3];         /* constant-colour environment replacing the sky cubemap */
    int32_t trace_indirect;       /* 0 = the reference as written (default): one path vertex, direct light + one sky sample.  1 = what the
                                   * code evidently intends (max_ray_bounces, RAY_THROUGHPUT, the environment added at depth 0 only): each
                                   * vertex adds direct_lighting weighted by the path throughput, then samples the GGX or the diffuse lobe
                                   * and traces the bounce, up to max_ray_bounces vertices (1 = direct light only, bit for bit the image of
                                   * 0; 2 = one indirect bounce).  Requires 1 <= max_ray_bounces <= 31 (the recursion limit the reference
                                   * reads on NVIDIA devices).  No Russian roulette; estimator in DESIGN.md §7 */
} hr_path_tracer_params;
enum {
    HR_PATH_TRACER_OUT_COLOR     = 0,  /* RGBA16F running average (rgb clamped to 1 per sample, a = 1) */
    HR_PATH_TRACER_OUT_PRIMITIVE = 1,  /* R32_UINT primitive hit by the last render's primary ray, 0xFFFFFFFF = sky (tests) */
    HR_PATH_TRACER_OUT_PATH_HASH = 2,  /* R32_UINT, trace_indirect = 1 renders only (tests): FNV-1a, h = (h ^ w) * 16777619 from 2166136261,
                                        * over the primitive hit by every path segment in order (primary included), then one end code:
                                        * 0xFFFFFFFF the last ray missed, 0xFFFFFFFE the sampled direction was below the horizon,
                                        * 0xFFFFFFFD the path reached max_ray_bounces */
    HR_PATH_TRACER_OUT_FINAL     = 100
};
HR_API void hr_path_tracer_default_params(hr_path_tracer_params* p);
HR_API int  hr_path_tracer_create(hr_ctx* ctx, int width, int height, hr_pass** out);
/* render(), ground_truth_path_tracer.cpp:44-113: the sample index is the pass's own counter (m_frame_idx, push constant num_frames),
 * restarted by hr_pass_reset_history (restart_accumulation(), ground_truth_path_tracer.h:17). */
HR_API int  hr_path_tracer_render(hr_pass* pass, const hr_frame* frame, const hr_path_tracer_params* params, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Converged references of the shadows, AO and reflections signals (reference.cu, DESIGN.md §8)
 *
 * A reference pass estimates the signal its target pass denoises: the same G-buffer, the same per-ray function (K1's soft-shadow
 * ray, K7's cosine-lobe ray, K12's mirror / DDGI / GGX sample with its shading and its 0.7 clamp) and the same parameters, averaged
 * over many independent rays per pixel instead of denoised from one.  The difference between the target's FINAL output and the
 * reference's MEAN is then the error of the denoise chain alone.
 *
 * Only the random numbers differ from the target's ray trace: (r0, r1) of sample k at pixel (x, y) are the first two next_float of
 * the xoroshiro64* stream of the path tracer seeded with rng_init(x, y, k) (random.glsl), not the 256-periodic blue noise.  Sample
 * k is the k-th sample the pass has accumulated, so any split of the samples over renders traces the same rays: shadows and AO
 * counts are identical, reflection sums equal up to float64 rounding.
 *
 * Output at the target's FINAL resolution (the full resolution, whatever the target's scale), the signal alone:
 *   HR_REFERENCE_OUT_MEAN    R16F (shadows, AO) or RGBA16F (rgb, 1) (reflections): the accumulated mean passed through the per-pixel
 *                            transform the target's FINAL applies after filtering, read from the parameters: shadows raise it to
 *                            `power` when denoise is on and filter_iterations >= 1 (the last a-trous iteration), AO when denoise is
 *                            on and the target's scale is not FULL (the upsample); reflections apply none.  Sky pixels (depth 1)
 *                            hold the FINAL's sky value: 0 for shadows, 1 for AO, (0, 0, 0, 1) for reflections.
 *   HR_REFERENCE_OUT_STDERR  same format: the standard error of the untransformed mean per channel, sqrt(s^2 / N) with the unbiased
 *                            sample variance s^2 of the N samples (0 for N = 1 and at sky pixels).  Mirror and DDGI-branch reflection
 *                            pixels do not depend on the sample: their STDERR is 0.
 * A shadows target at full resolution has an RG16F FINAL (visibility, variance): compare its r channel, copied into an R16F
 * image, with MEAN (hr_image_compare takes images of one format).
 *
 * Accumulation: one sample counter N for the rendered rows (uint32, restarted by hr_pass_reset_history, which the caller calls when the
 * view, the scene or the light changes: the reference does no reprojection).  Shadows and AO keep a uint32 count of unoccluded rays
 * per pixel, reflections float64 sums of the value and of its square per channel.  hr_pass_get_stats counts the rays traced (the
 * mirror and DDGI-branch samples are evaluated once per render); hr_pass_output, the downloads, the checksum and hr_pass_destroy
 * work as for any pass.  The target must outlive its reference.
 * ---------------------------------------------------------------------------------------------- */
enum { HR_REFERENCE_OUT_STDERR = 1, HR_REFERENCE_OUT_MEAN = 100 };
/* A reference of `target` (a shadows, AO or reflections pass); HR_ERR_INVALID_ARG for a pass of another kind. */
HR_API int hr_reference_create(hr_pass* target, hr_pass** out);
/* Adds `samples` (1..65536) rays per pixel on rows [row0, row1) (row1 <= 0: to the last row) of the current G-buffer slot
 * (frame->ping_pong) at mip 0, then writes MEAN and STDERR of those rows; the other rows are left as they are.  The one sample
 * counter N counts the samples of these rows, so every render between two resets covers the same rows: a render over other rows
 * than the first one after the reset is refused.  A sharded rank renders its band and the 5 rows beyond it that the SSIM window
 * of hr_image_compare reads.
 * params: the target's parameter block (hr_shadows_params, hr_ao_params or hr_reflections_params).  ddgi: reflections only, may be
 * NULL; the DDGI and IBL terms are switched on exactly as hr_reflections_render decides for the target's next render with that
 * DDGI pass (off on the target's first frame, so render the reference before the target in that frame).
 * HR_ERR_INVALID_ARG, changing nothing: NULL pointers, a bad sample count or row range, rows other than those of the first render
 * since the reset, N passing 2^32 - 1, non-finite parameters, or a DDGI pass of another context. */
HR_API int hr_reference_render(hr_pass* ref, const hr_frame* frame, const void* params, hr_pass* ddgi, int samples, int row0, int row1, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Common pass functions
 * ---------------------------------------------------------------------------------------------- */
/* output_ds() equivalent: borrowed device image, valid until the next render/destroy of this pass. */
HR_API int hr_pass_output(hr_pass* pass, int which, hr_image* out);
/* Synchronous device->host copy of an output on `stream` (waits for it). bytes must equal w*h*texel. */
HR_API int hr_pass_download(hr_pass* pass, int which, void* host_dst, size_t bytes, void* stream);
/* Same copy enqueued on `stream` without the host synchronisation (pinned host_dst, or a device pointer: the copy kind is
 * inferred, so a caller may stage the image on the device and run the PCIe copy on its own stream; the caller synchronises). */
HR_API int hr_pass_download_async(hr_pass* pass, int which, void* host_dst, size_t bytes, void* stream);
/* Rows [row0,row1) only — e.g. a rank's own band (hr_shard_rows, scaled to the image) of an output left distributed. */
HR_API int hr_pass_download_rows_async(hr_pass* pass, int which, int row0, int row1, void* host_dst, size_t bytes, void* stream);
/* Checkpoint / resume of temporal history: hr_pass_download saves an image, hr_pass_upload restores it (synchronous). */
HR_API int hr_pass_upload(hr_pass* pass, int which, const void* host_src, size_t bytes, void* stream);
/* restart_accumulation() / clear_images() equivalent: next render behaves like first_frame for this pass's history. */
HR_API int hr_pass_reset_history(hr_pass* pass);
HR_API int hr_pass_destroy(hr_pass* pass);
/* Per-stage GPU timings in ms (DW_SCOPED_SAMPLE equivalent, profiler.cpp:83-181) of the renders profiled since the previous call
 * (at most the last 1024): one entry per stage name, in the order the names first occurred, each the mean over the renders that
 * recorded that stage.  Enable with hr_ctx_set_profiling(ctx,1); names/ms arrays of capacity cap; returns count via *n.
 * Synchronises. */
HR_API int hr_ctx_set_profiling(hr_ctx* ctx, int enabled);
HR_API int hr_pass_stage_times(hr_pass* pass, const char** names, float* ms, int cap, int* n);
/* Test hook, process-wide.  key 1 = shadows a-trous implementation (0 naive global-memory kernel, 1 shared-memory tiled kernel,
 * 3 packed fp32x2 pixel-pair kernel = default); key 3 = BVH topology used by the next hr_scene_build / hr_scene_rebuild (0 Karras radix tree,
 * 1 PLOC agglomerative clustering = default); key 6 = reflections a-trous (0 scalar kernel, 2 packed fp32x2 pixel pairs with plain staging,
 * 3 = 2 + TMA-staged persistent kernel for step 1 = default).  Any other key, or a value its key does not list, returns
 * HR_ERR_INVALID_ARG and changes nothing.  None of them changes a result bit of the visibility masks; key 6 values 2 and 3 agree to
 * the last fp16 bit. */
HR_API int hr_debug_set(int key, int value);
/* Number of kernels this library launched since the context was created (bench.py gpu_launches).  Each kernel counts once.
 * Earlier versions counted the reflections ray trace (K12) as two launches, a leftover of a removed two-kernel form, so config 3's
 * gpu_launches was one per frame higher.  tests/test_gpu_launch_count.py checks the count against the kernels torch.profiler
 * records for every pass. */
HR_API uint64_t hr_ctx_launch_count(hr_ctx* ctx);

/* Work actually done by a pass (bench.py: roofline on processed bytes, Mrays/s on counted rays; SURVEY.md §8d).
 * Ray counts accumulate on the device since the previous hr_pass_get_stats call (warp-aggregated atomics inside the trace
 * kernels), which drains them to 0; `renders` counts the same way.  The tile counts describe the last render only: the 8x8 tiles
 * of the rows this rank's denoise stages covered (its band +- the denoise halo of hr_shard_halo_rows, the whole pass at world 1),
 * and how many of them were on the denoise list (the others take the reference's copy / zero-fill path).  A render with
 * denoise = 0 covers no rows: tiles_total, tiles_denoise and pixels_total are then 0.  Passes without tile flags (DDGI and the
 * post passes) report 0 for them.  Synchronises `stream`. */
typedef struct hr_pass_stats {
    uint64_t rays_primary;   /* K1/K7: pixels that traced a ray; K12: reflection rays; K18: probe rays                     */
    uint64_t rays_secondary; /* shadow / sky-light rays of the hit shading (K12, K18)                                      */
    uint64_t tiles_total;    /* 8x8 tiles in the rows covered by the last render's denoise stages                          */
    uint64_t tiles_denoise;  /* of those, tiles on the denoise list (tile flag = 1)                                        */
    uint64_t pixels_total;   /* pixels in those rows                                                                       */
    uint64_t renders;        /* renders since the previous call                                                           */
} hr_pass_stats;
HR_API int hr_pass_get_stats(hr_pass* pass, hr_pass_stats* out, void* stream);
/* Order-independent 64-bit checksum of an output image computed on the device, over rows [row0,row1) (row1 <= 0 = the whole
 * image; any other range outside [0, height] or with row1 < row0 returns HR_ERR_INVALID_ARG):
 *     sum mod 2^64 over the texels i of those rows of  mix(mix(i + 0x9E3779B97F4A7C15) ^ v_i)
 * where i = y * width + x is the texel's row-major index from the image's first texel, v_i its 1, 2, 4 or 8 bytes (R8_UINT;
 * R16F; R32_UINT, RG16F, RGBA8; RGBA16F) read as a little-endian unsigned integer, and mix the splitmix64 finaliser
 *     z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;  mix(z) = z ^ (z >> 31).
 * So the checksums of any split of the rows add up (mod 2^64) to the whole image's: the ranks of a sharded run can each sum their
 * own rows.  bench.py uses it to show that an N-GPU frame equals the single-GPU frame without moving the images.  Synchronises
 * `stream`. */
HR_API int hr_pass_output_checksum(hr_pass* pass, int which, int row0, int row1, uint64_t* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Image comparison (not in the reference, whose judge is a person flipping between the "Ground Truth" view and the hybrid frame):
 * error sums and SSIM of a test image against a reference image, e.g. the deferred combine's FINAL output against the path tracer's,
 * computed on the device.  The per-pixel terms are bit-specified (DESIGN.md §5, restated in tests/image_compare.py):
 *   t, r = the pixel's C channels as float (RGBA16F and RGBA8: rgb, alpha ignored, RGBA8 as b / 255; RG16F: r, g; R16F: r); d = t - r;
 *   se = (sum d^2) / C,  ae = (sum |d|) / C,  rel = (sum d^2 / (r^2 + relmse_eps)) / C, each channel sum in channel order;
 *   a pixel with a NaN or infinite channel in t (r) counts in nonfinite_test (nonfinite_ref) and is left out of every sum;
 *   luminance Y = (0.299 c0 + 0.587 c1) + 0.114 c2 of the channels clamped to [0, 1] (one channel: clamp(c0); two: c2 = 0), 0 in both
 *   images at a left-out pixel; SSIM over the 11-tap Gaussian window (sigma 1.5, float weights of the normalised double Gaussian),
 *   rows first, then columns, taps clamped to the image:
 *   ssim = ((2 mu_t mu_r + ssim_c1)(2 cov + ssim_c2)) / ((mu_t^2 + mu_r^2 + ssim_c1)(var_t + var_r + ssim_c2)).
 * Each term x enters its sum as round-to-nearest-even(x * 2^32), x clamped to [-2^63, 2^63] (NaN, possible only with zero
 * parameters: 0).  The sums are integers, so they do not depend on the launch and the sums of any row split (one per rank of a
 * sharded run) add up to the whole image's.
 * ---------------------------------------------------------------------------------------------- */
typedef struct hr_compare_params {
    float relmse_eps; /* 0.01: relMSE term d^2 / (r^2 + eps) */
    float ssim_c1;    /* 1e-4 = (0.01 * 1)^2 */
    float ssim_c2;    /* 9e-4 = (0.03 * 1)^2 */
} hr_compare_params;
HR_API void hr_compare_default_params(hr_compare_params* p);

typedef struct hr_compare_sums {   /* integers: order-independent; the sums of any row split add up to the whole image's */
    uint64_t pixels;               /* pixels summed (both texels finite)                                                  */
    uint64_t nonfinite_test, nonfinite_ref;
    uint64_t sq_err[2], abs_err[2], rel_err[2]; /* unsigned 128-bit (lo, hi), fixed point 2^-32                           */
    uint64_t ssim[2];              /* signed 128-bit two's complement, fixed point 2^-32                                  */
    uint32_t max_abs_err;          /* float bits of the largest per-pixel channel |d| (max of non-negative floats = max of their bits) */
    uint32_t _pad;
} hr_compare_sums;
/* Pure: acc += s (128-bit adds wrapping mod 2^128, counts added, max_abs_err the larger). */
HR_API void hr_compare_sums_add(hr_compare_sums* acc, const hr_compare_sums* s);

typedef struct hr_compare_result {
    double   mse, rmse, psnr, relmse, mean_abs, max_abs, ssim;
    uint64_t pixels, nonfinite_test, nonfinite_ref;
} hr_compare_result;
/* Pure: the means of the sums, each (double)(sum) * 2^-32 / (double)pixels (the 128-bit integer rounded once to double); rmse =
 * sqrt(mse); psnr = 10 log10(1 / mse), +inf at mse 0; max_abs = the float of max_abs_err.  No pixel summed: the means are NaN. */
HR_API void hr_compare_finish(const hr_compare_sums* s, hr_compare_result* out);

/* test, ref: device images of equal size and format (hr_pass_output of two passes, or caller memory).  Rows [row0, row1) are summed
 * (row1 <= 0 = whole image; any other range outside [0, height] or with row1 < row0 returns HR_ERR_INVALID_ARG).  SSIM windows read
 * 5 rows beyond the range (clamped to the image), so those rows must be valid: gathered FINAL outputs are.  error_map: optional caller
 * device RGBA16F W x H image that receives (ae, se, rel, ssim) rounded to fp16 for the pixels of the range's rows (a left-out pixel:
 * four quiet NaNs, 0x7E00); its other rows are not written.  R32_UINT and R8_UINT images return HR_ERR_UNSUPPORTED; a size or format
 * mismatch, a NULL argument, a bad row range, an error map of another size or format or whose bytes overlap test's or ref's, or a negative
 * or non-finite parameter returns
 * HR_ERR_INVALID_ARG.  A refused call writes nothing to `out` or `error_map`.  Two kernels (per-tile sums, then their total; none for
 * an empty range).  Synchronises `stream`. */
HR_API int hr_image_compare(hr_ctx* ctx, const hr_image* test, const hr_image* ref, const hr_compare_params* params, int row0, int row1,
                            hr_compare_sums* out, hr_image* error_map, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Screen-space row-band sharding across GPUs (new; SURVEY.md §8e).  rank owns pass rows
 * [row_begin, row_end) aligned to 8; the other rows are skipped by every stage except a halo.
 * ---------------------------------------------------------------------------------------------- */
HR_API int hr_shard_config(hr_ctx* ctx, int rank, int world); /* band assignment only (world <= 8); the caller exchanges bands itself */
/* NCCL-backed sharding: rank 0 obtains a 128-byte ncclUniqueId, every rank calls hr_shard_init with it (one process per
 * GPU of ONE box, world <= 8: the peer mappings are CUDA IPC).  The temporal history stays distributed (see below); the
 * only per-frame collective is the optional all-gather of each pass's final output on the library's side stream. */
HR_API int hr_shard_unique_id(void* out_128_bytes);
HR_API int hr_shard_init(hr_ctx* ctx, int rank, int world, const void* unique_id_128_bytes);
HR_API int hr_shard_shutdown(hr_ctx* ctx);
/* After hr_shard_init the shadows / AO temporal history stays distributed: every rank keeps the rows of its band and the
 * reprojection kernel reads a history texel from the GPU that owns its row (peer mappings over NVLink, set up on the
 * first render of each pass — all ranks must create and render their passes in the same order, and call
 * hr_pass_reset_history together).  hr_pass_output / hr_pass_download of history and intermediate images are therefore
 * valid on the rank's own band only.  The FINAL output (which = 100) of every pass is all-gathered after each render
 * unless this is switched off (gather_final_output = 0: every rank keeps just its band of the frame). */
HR_API int hr_shard_set_gather(hr_ctx* ctx, int gather_final_output);
/* Pure query (no context, no GPU): the rows beyond its band a sharded rank recomputes, derived from the pass parameters — the
 * denoise stages (temporal + a-trous chain: sum(radius << i) + 1 rounded up to 8; AO: 8 + blur_radius rounded up to 8) and the
 * ray-trace output the temporal stage's 17x17 statistics read (8 more).  pass_kind: 1 shadows, 2 AO, 3 reflections. */
#define HR_PASS_KIND_SHADOWS 1
#define HR_PASS_KIND_AO 2
#define HR_PASS_KIND_REFLECTIONS 3
HR_API int hr_shard_halo_rows(int pass_kind, int radius, int filter_iterations, int blur_radius, int* denoise_halo, int* ray_trace_halo);
/* Same-process peers (N ranks emulated on one GPU with hr_shard_config, or several GPUs driven by one process): declare
 * that rank `rank`'s band of this pass's history lives in `peer` (DDGI: that `peer` receives this rank's probe slices).  Passes of
 * another kind or size are refused.  Link every pass with every other rank's pass before
 * the first render, give every rank its own stream (the ranks wait for each other's ray masks inside a frame, so their
 * kernels must be able to run concurrently) and run the process with CUDA_MODULE_LOADING=EAGER (a lazily loaded kernel's
 * first launch synchronises the context, which stalls until the peer time-out while another rank's wait kernel spins). */
HR_API int hr_shard_link_local(hr_pass* pass, int rank, hr_pass* peer);
/* Row range (at pass resolution, height H) owned by rank. */
HR_API int hr_shard_rows(int height, int rank, int world, int* row_begin, int* row_end);

#ifdef __cplusplus
}
#endif
#endif /* HR_API_H */
