/*
 * synth.h — headless input producers for the hot path (C interface, host only).
 *
 * The reference feeds its RT passes from a Vulkan raster G-buffer (src/g_buffer.cpp, shaders/g_buffer.{vert,frag}),
 * scenes loaded through assimp (src/common.cpp:340-534) and blue-noise PNGs (src/blue_noise.cpp:5-19); none of the
 * assets are in the repository.  Per BASELINE.json's north_star the raster stage is replaced by this CPU-side
 * synthetic G-buffer writer: it ray-casts primary visibility through the same camera and emits the reference's
 * G-buffer encodings (g_buffer.frag:86-112; clears g_buffer.cpp:72-96).
 */
#ifndef HR_SYNTH_H
#define HR_SYNTH_H
#include "../../include/hr_api.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct hrs_scene hrs_scene;

enum {
    HRS_SCENE_SINGLE_TRIANGLE = 0, /* BASELINE config 1 occluder: (-4,3,-4),(4,3,-4),(0,3,4)                    */
    HRS_SCENE_GROUND_PLANE    = 1, /* BASELINE config 1 visible surface: y = 0 plane, mesh id 0, roughness 0.5   */
    HRS_SCENE_SHADOWS_TEST    = 2, /* floor + boxes + pillars (a few thousand triangles), like common.cpp:340-430 */
    HRS_SCENE_ARCADE          = 3  /* "Sponza-scale" two-storey arcade, tessellated to ~target_tris               */
};

HR_API hrs_scene* hrs_scene_create(int kind, int target_tris, uint32_t seed);
HR_API void       hrs_scene_destroy(hrs_scene* s);
HR_API void       hrs_scene_counts(const hrs_scene* s, uint64_t* n_vertices, uint64_t* n_indices, uint64_t* n_instances, uint64_t* n_materials);
HR_API const hr_vertex*   hrs_scene_vertices(const hrs_scene* s);
HR_API const uint32_t*    hrs_scene_indices(const hrs_scene* s);
HR_API const hr_instance* hrs_scene_instances(const hrs_scene* s);
HR_API const hr_material* hrs_scene_materials(const hrs_scene* s);
HR_API void               hrs_scene_bounds(const hrs_scene* s, float mn[3], float mx[3]);
/* World-space triangle soup, 9 floats per triangle, in the primitive order hr_scene_build uses
 * (instances in order, triangles in index order).  prim_instance (optional): instance index per triangle. */
HR_API void hrs_scene_world_triangles(const hrs_scene* s, float* out9, uint32_t* prim_instance);
/* World-space unit vertex normals (9 floats per triangle) and material index per triangle, same primitive order. */
HR_API void hrs_scene_world_normals(const hrs_scene* s, float* out9, uint32_t* prim_material);

/* Fill hr_frame like HybridRendering::update_uniforms (src/main.cpp:937-972) + create_camera (:248-255):
 * perspective(60 deg, W/H, 1, 1000), jitter 0.  prev == NULL => first frame (prev_view_proj = identity, first_frame = 1). */
typedef struct hrs_light_desc {
    int32_t type;             /* HR_LIGHT_*                                                      */
    float   rot_y_deg, rot_x_deg; /* m_light_transform = rotY * rotX (main.cpp:787); dir = mat3 * (0,-1,0) */
    float   position[3];
    float   radius, intensity;
    float   color[3];
    float   cone_inner_deg, cone_outer_deg;
} hrs_light_desc;
HR_API void hrs_default_light(hrs_light_desc* l); /* shadows-test directional preset, main.cpp:782-787 */
HR_API void hrs_make_frame(hr_frame* out, const float cam_pos[3], const float cam_target[3], int width, int height,
                           const hrs_light_desc* light, const hr_frame* prev, uint32_t num_frames);
/* hrs_make_frame with any camera: look_at(cam_pos, cam_target, cam_up) and perspective(fovy_deg, W/H, z_near, z_far);
 * z_buffer_params follow z_near / z_far.  hrs_make_frame is this with up (0, 1, 0), 60 degrees, near 1, far 1000. */
HR_API void hrs_make_frame_ex(hr_frame* out, const float cam_pos[3], const float cam_target[3], const float cam_up[3], float fovy_deg,
                              float z_near, float z_far, int width, int height, const hrs_light_desc* light, const hr_frame* prev,
                              uint32_t num_frames);

/* Ray-cast the visible scene through frame->ubo and write mip 0 of the G-buffer (host memory):
 * gb1 RGBA8 (may be NULL), gb2/gb3 RGBA16F, depth float. */
HR_API void hrs_write_gbuffer(const hrs_scene* visible, const hr_frame* frame, int width, int height,
                              uint8_t* gb1, uint16_t* gb2, uint16_t* gb3, float* depth);

/* Substitute blue-noise tables (the Heitz'19 PNGs are release-zip assets, SURVEY.md §8c):
 * 8-bit Sobol' points dims 0..3 from the Joe-Kuo direction numbers; seeded-PRNG scramble/rank tile. */
HR_API void hrs_blue_noise(uint32_t seed, uint8_t* sobol_256x4, uint8_t* scrambling_ranking_128x128x4);

/* synthetic stand-in for textures/brdf_lut.bin: 512 x 512 RG16F split-sum LUT */
HR_API void hrs_brdf_lut(int samples, uint16_t* out_512x512x2);

#ifdef __cplusplus
}
#endif
#endif
