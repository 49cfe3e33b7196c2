// mask_px.cuh — the per-ray function of K1 (shadows) and K7 (AO), shared by their ray traces (trace.cu) and the converged references
// (reference.cu).  Compile with -fmad=false: the ray is part of the deterministic chain (det_math.cuh).
#pragma once
#include "traverse.cuh"

namespace {

// MODE 0 = K1 (p0 = bias): the soft-shadow ray toward the light (shadows_ray_trace.comp:89-132); MODE 1 = K7 (p0 = ray length, p1 = bias):
// the cosine-lobe ray (ao_ray_trace.comp:90-126), at surface point P with normal N from the random pair (r0, r1).  false: K1 traces no
// ray (the light's attenuation is 0); true: the caller traces r with trace_any, the ray is unoccluded when it hits nothing.
template <int MODE>
__device__ __forceinline__ bool mask_ray(const FrameConsts& fc, det::V3 P, det::V3 N, float p0, float p1, float r0, float r1, trv::Ray& r)
{
    r.tmin = 0.01f;
    if (MODE == 0)
    {
        r.o = det::add(P, det::scale(N, p0)); // bias
        float att;
        det::fetch_light_properties_shadow(fc.light, P, N, r0, r1, r.d, r.tmax, att);
        return att > 0.0f;
    }
    r.o    = det::add(P, det::scale(N, p1)); // bias
    r.d    = det::sample_cosine_lobe(N, r0, r1);
    r.tmax = p0; // ray_length
    return true;
}

} // namespace
