#!/usr/bin/env python
"""make_ref_constants.py — extract every literal table / constant the reference holds IN SOURCE for the hot path and
write them to tests/golden/ref_constants.json.

The reference (diharaw/hybrid-rendering) ships no tests, golden vectors or fixtures; the only reference-held data that
can pin the oracle are the literals inside its shaders and headers.  This script parses them (nothing is typed in by
hand) from a checkout of the reference and records the file:line each value came from.  The reference is not part of
this repository, so the JSON is committed and tests/test_ref_constants.py checks the oracle (and, on the GPU, the CUDA
kernels) against it.

    python tests/golden/make_ref_constants.py REFERENCE_CHECKOUT
"""
import json
import os
import re
import sys

if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
SH = os.path.join(REF, "src", "shaders")
SRC = os.path.join(REF, "src")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_constants.json")


def read(path):
    with open(path) as f:
        return f.read()


def line_of(text, pos):
    return text.count("\n", 0, pos) + 1


def num(s):
    """GLSL / C++ numeric literal or simple constant expression (a / b) -> python number."""
    s = s.strip().rstrip(";").strip()
    s = re.sub(r"(?<=[0-9.])[fFuU]\b", "", s)
    if re.fullmatch(r"0[xX][0-9a-fA-F]+", s):
        return int(s, 16)
    if re.fullmatch(r"[-+]?\d+", s):
        return int(s)
    if re.fullmatch(r"[-+0-9.eE/* ()]+", s):
        return float(eval(s))  # only digits and arithmetic survive the regex above
    if s in ("true", "false"):
        return s == "true"
    raise ValueError(f"cannot parse literal {s!r}")


def define(text, name, rel):
    m = re.search(rf"^\s*#define\s+{name}\s+(.+?)\s*$", text, re.M)
    if not m:
        raise KeyError(f"#define {name} not found in {rel}")
    return {"value": num(m.group(1)), "src": f"{rel}:{line_of(text, m.start(1))}"}


def member_default(text, name, rel, nth=0):
    ms = list(re.finditer(rf"\b(?:float|int32_t|uint32_t|bool)\s+{name}\s*=\s*([^;]+);", text))
    if len(ms) <= nth:
        raise KeyError(f"member {name} (#{nth}) not found in {rel}")
    m = ms[nth]
    return {"value": num(m.group(1)), "src": f"{rel}:{line_of(text, m.start())}"}


def main():
    out = {"_generated_by": "tests/golden/make_ref_constants.py", "_reference": "diharaw/hybrid-rendering (/root/reference)"}

    # ---- DDGI border copy tables, gi/gi_border_update.glsl:35-143 ------------------------------------------------------
    rel = "src/shaders/gi/gi_border_update.glsl"
    t = read(os.path.join(SH, "gi", "gi_border_update.glsl"))
    tables = {}
    for m in re.finditer(r"const\s+ivec4\s+g_offsets\[(\d+)\]\s*=\s*ivec4\[\]\((.*?)\);", t, re.S):
        n = int(m.group(1))
        rows = [[int(v) for v in r] for r in re.findall(r"ivec4\(\s*(-?\d+)\s*,\s*(-?\d+)\s*,\s*(-?\d+)\s*,\s*(-?\d+)\s*\)", m.group(2))]
        assert len(rows) == n, (n, len(rows))
        tables[n] = {"rows": rows, "src": f"{rel}:{line_of(t, m.start())}-{line_of(t, m.end())}"}
    assert set(tables) == {68, 36}, sorted(tables)
    out["gi_border_offsets_depth_16"] = tables[68]
    out["gi_border_offsets_irradiance_8"] = tables[36]

    # ---- a-trous kernels, shadows_denoise_atrous.comp:69-72,99-100 (+ reflections twin) --------------------------------
    for key, sub in (("shadows", "shadows/shadows_denoise_atrous.comp"), ("reflections", "reflections/reflections_denoise_atrous.comp")):
        rel = f"src/shaders/{sub}"
        t = read(os.path.join(SH, sub))
        m = re.search(r"const\s+float\s+kernel\[2\]\[2\]\s*=\s*\{\s*\{([^}]*)\}\s*,\s*\{([^}]*)\}\s*\}", t)
        out[f"{key}_atrous_variance_kernel"] = {"value": [[num(v) for v in m.group(1).split(",")], [num(v) for v in m.group(2).split(",")]],
                                                "src": f"{rel}:{line_of(t, m.start())}"}
        m = re.search(r"const\s+float\s+kernel_weights\[3\]\s*=\s*\{([^}]*)\}", t)
        out[f"{key}_atrous_kernel_weights"] = {"value": [num(v) for v in m.group(1).split(",")], "src": f"{rel}:{line_of(t, m.start())}"}
        m = re.search(r"const\s+float\s+eps_variance\s*=\s*([^;]+);", t)
        out[f"{key}_atrous_eps_variance"] = {"value": num(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}

    # ---- RNG, random.glsl:17-56 -----------------------------------------------------------------------------------------
    rel = "src/shaders/random.glsl"
    t = read(os.path.join(SH, "random.glsl"))
    rng = {}
    m = re.search(r"uint\s+result\s*=\s*rng\.s\.x\s*\*\s*(0x[0-9a-fA-F]+)", t)
    rng["star_multiplier"] = {"value": num(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}
    m = re.search(r"rng\.s\.x\s*=\s*rng_rotl\(rng\.s\.x,\s*(\d+)\)\s*\^\s*rng\.s\.y\s*\^\s*\(rng\.s\.y\s*<<\s*(\d+)\)", t)
    rng["rotl_a"] = {"value": int(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}
    rng["shift_b"] = {"value": int(m.group(2)), "src": f"{rel}:{line_of(t, m.start())}"}
    m = re.search(r"rng\.s\.y\s*=\s*rng_rotl\(rng\.s\.y,\s*(\d+)\)", t)
    rng["rotl_c"] = {"value": int(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}
    m = re.search(r"seed\s*=\s*\(seed\s*\^\s*(\d+)\)\s*\^\s*\(seed\s*>>\s*(\d+)\);\s*seed\s*\*=\s*(\d+);\s*seed\s*=\s*seed\s*\^\s*\(seed\s*>>\s*(\d+)\);\s*"
                  r"seed\s*\*=\s*(0x[0-9a-fA-F]+);\s*seed\s*=\s*seed\s*\^\s*\(seed\s*>>\s*(\d+)\);", t)
    rng["hash"] = {"value": [num(m.group(i)) for i in range(1, 7)], "src": f"{rel}:{line_of(t, m.start())}-{line_of(t, m.end())}",
                   "meaning": "xor0, shr0, mul0, shr1, mul1, shr2 of the Wang hash"}
    m = re.search(r"uint\s+s0\s*=\s*\(id\.x\s*<<\s*(\d+)\)\s*\|\s*id\.y", t)
    rng["seed_shift"] = {"value": int(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}
    m = re.search(r"uint\s+u\s*=\s*(0x[0-9a-fA-F]+)\s*\|\s*\(rng_next\(rng\)\s*>>\s*(\d+)\)", t)
    rng["float_bits"] = {"value": [num(m.group(1)), int(m.group(2))], "src": f"{rel}:{line_of(t, m.start())}"}
    out["rng"] = rng

    # ---- thresholds ------------------------------------------------------------------------------------------------------
    rel = "src/shaders/common.glsl"
    t = read(os.path.join(SH, "common.glsl"))
    for name in ("M_PI", "EPSILON", "MIRROR_REFLECTIONS_ROUGHNESS_THRESHOLD", "DDGI_REFLECTIONS_ROUGHNESS_THRESHOLD", "LIGHT_TYPE_DIRECTIONAL", "LIGHT_TYPE_POINT",
                 "LIGHT_TYPE_SPOT"):
        out[name] = define(t, name, rel)
    rel = "src/shaders/reprojection.glsl"
    t = read(os.path.join(SH, "reprojection.glsl"))
    for name in ("NORMAL_DISTANCE", "PLANE_DISTANCE"):
        out[name] = define(t, name, rel)
    rel = "src/shaders/scene_descriptor_set.glsl"
    t = read(os.path.join(SH, "scene_descriptor_set.glsl"))
    out["MIN_ROUGHNESS"] = define(t, "MIN_ROUGHNESS", rel)
    rel = "src/common.h"
    t = read(os.path.join(SRC, "common.h"))
    for name in ("CAMERA_NEAR_PLANE", "CAMERA_FAR_PLANE"):
        try:
            out[name] = define(t, name, rel)
        except KeyError:
            pass

    # ---- pass defaults (struct initialisers) ----------------------------------------------------------------------------
    defaults = {}
    rel = "src/ray_traced_shadows.h"
    t = read(os.path.join(SRC, "ray_traced_shadows.h"))
    defaults["shadows"] = {k: member_default(t, k, rel) for k in ("bias", "alpha", "moments_alpha", "phi_visibility", "phi_normal", "sigma_depth", "power", "radius",
                                                                  "filter_iterations", "feedback_iteration")}
    rel = "src/ray_traced_ao.h"
    t = read(os.path.join(SRC, "ray_traced_ao.h"))
    defaults["ao"] = {k: member_default(t, k, rel) for k in ("ray_length", "bias", "alpha", "blur_radius", "power")}
    rel = "src/ray_traced_reflections.h"
    t = read(os.path.join(SRC, "ray_traced_reflections.h"))
    defaults["reflections"] = {k: member_default(t, k, rel) for k in ("sample_gi", "approximate_with_ddgi", "gi_intensity", "rough_ddgi_intensity",
                                                                      "ibl_indirect_specular_intensity", "bias", "trim", "alpha", "moments_alpha", "blur_as_input",
                                                                      "phi_color", "phi_normal", "sigma_depth", "radius", "filter_iterations", "feedback_iteration")}
    rel = "src/ddgi.h"
    t = read(os.path.join(SRC, "ddgi.h"))
    defaults["ddgi"] = {k: member_default(t, k, rel) for k in ("infinite_bounces", "infinite_bounce_intensity", "rays_per_probe", "visibility_test", "probe_distance",
                                                               "recursive_energy_preservation", "irradiance_oct_size", "depth_oct_size", "hysteresis", "depth_sharpness",
                                                               "normal_bias", "gi_intensity")}
    # ---- post-processing (SURVEY.md section 8 f4): taa.comp, temporal_aa.{h,cpp}, tone_map.{frag,h} ---------------------------------
    rel = "src/shaders/taa.comp"
    t = read(os.path.join(SH, "taa.comp"))
    taa = {}
    m = re.search(r"const\s+float\s+FLT_EPS\s*=\s*([^;]+);", t)
    taa["FLT_EPS"] = {"value": num(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}
    # the feature switches that select which branches of the shader exist (only un-commented, top-level #define lines)
    defs = [(mm.group(1), line_of(t, mm.start())) for mm in re.finditer(r"^#define\s+(\w+)\s*(?:\d+)?\s*$", t, re.M)]
    taa["defines"] = {"value": [d for d, _ in defs], "src": f"{rel}:{defs[0][1]}-{defs[-1][1]}"}
    m = re.search(r"max\(lum0,\s*max\(lum1,\s*([0-9.]+)\)\)", t)
    taa["luminance_floor"] = {"value": num(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}
    m = re.search(r"sum \+= ([-0-9.]+) \* cml;\s*sum \+= ([-0-9.]+) \* ctc;\s*sum \+= ([-0-9.]+) \* texel0;\s*sum \+= ([-0-9.]+) \* cbc;\s*sum \+= ([-0-9.]+) \* cmr;", t)
    taa["sharpen_weights"] = {"value": [num(m.group(i)) for i in range(1, 6)], "src": f"{rel}:{line_of(t, m.start())}-{line_of(t, m.end())}", "meaning": "cml, ctc, texel0, cbc, cmr"}
    rel = "src/temporal_aa.cpp"
    t = read(os.path.join(SRC, "temporal_aa.cpp"))
    taa["HALTON_SAMPLES"] = define(t, "HALTON_SAMPLES", rel)
    out["taa"] = taa
    rel = "src/temporal_aa.h"
    t = read(os.path.join(SRC, "temporal_aa.h"))
    defaults["taa"] = {k: member_default(t, k, rel) for k in ("m_enabled", "m_sharpen", "m_reset", "m_feedback_min", "m_feedback_max")}
    rel = "src/shaders/tone_map.frag"
    t = read(os.path.join(SH, "tone_map.frag"))
    aces = {}
    for k in "abcde":
        m = re.search(rf"float\s+{k}\s*=\s*([^;]+);", t)
        aces[k] = num(m.group(1))
    m0 = re.search(r"vec3\s+aces_film", t)
    m = re.search(r"pow\(color,\s*vec3\(([^)]+)\)\)", t)
    out["tone_map"] = {"aces": {"value": aces, "src": f"{rel}:{line_of(t, m0.start())}"}, "gamma_exponent": {"value": num(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}}
    rel = "src/tone_map.h"
    t = read(os.path.join(SRC, "tone_map.h"))
    defaults["tone_map"] = {"m_exposure": member_default(t, "m_exposure", rel)}

    # ---- ground-truth path tracer: ground_truth_path_trace.{rgen,rchit}, ground_truth_path_tracer.h, common.glsl, lighting.glsl -------
    pt = {}
    rel = "src/shaders/ground_truth/ground_truth_path_trace.rgen"
    t = read(os.path.join(SH, "ground_truth", "ground_truth_path_trace.rgen"))
    m = re.search(r"float\s+tmin\s*=\s*([^;]+);\s*float\s+tmax\s*=\s*([^;]+);", t)
    pt["primary_tmin_tmax"] = {"value": [num(m.group(1)), num(m.group(2))], "src": f"{rel}:{line_of(t, m.start())}"}
    rel = "src/shaders/common.glsl"
    t = read(os.path.join(SH, "common.glsl"))
    m = re.search(r"#define\s+RADIANCE_CLAMP_COLOR\s+vec3\(([^)]+)\)", t)
    pt["RADIANCE_CLAMP_COLOR"] = {"value": num(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}
    rel = "src/shaders/lighting.glsl"
    t = read(os.path.join(SH, "lighting.glsl"))
    m = re.search(r"vec3\s+ray_origin\s*=\s*P\s*\+\s*N\s*\*\s*([^;]+);", t)
    pt["shadow_ray_origin_offset"] = {"value": num(m.group(1)), "src": f"{rel}:{line_of(t, m.start())}"}
    rel = "src/shaders/ray_query.glsl"
    t = read(os.path.join(SH, "ray_query.glsl"))
    m = re.search(r"float\s+query_distance\(.*?float\s+t_min\s*=\s*([^;]+);", t, re.S)
    pt["query_distance_t_min"] = {"value": num(m.group(1)), "src": f"{rel}:{line_of(t, m.start(1))}"}
    rel = "src/shaders/ground_truth/ground_truth_path_trace.rchit"
    t = read(os.path.join(SH, "ground_truth", "ground_truth_path_trace.rchit"))
    m = re.search(r"^\s*//\s*traceRayEXT\(u_TopLevelAS", t, re.M)
    pt["indirect_trace_is_commented_out"] = {"value": bool(m) and not re.search(r"^\s*traceRayEXT\(", t, re.M), "src": f"{rel}:{line_of(t, m.start()) if m else 0}"}
    pt["rchit_defines"] = {"value": re.findall(r"^#define\s+(\w+)\s*$", t, re.M), "src": rel}
    rel = "src/ground_truth_path_tracer.h"
    t = read(os.path.join(SRC, "ground_truth_path_tracer.h"))
    defaults["path_tracer"] = {"max_ray_bounces": member_default(t, "max_ray_bounces", rel)}
    out["path_tracer"] = pt

    out["defaults"] = defaults

    # ---- struct sizes the ABI mirrors (counted from the member lists) ---------------------------------------------------
    rel = "src/common.h"
    t = read(os.path.join(SRC, "common.h"))
    m = re.search(r"struct\s+UBO\s*\{(.*?)\};", t, re.S)
    body = m.group(1)
    n_mat4 = len(re.findall(r"\bglm::mat4\b|DW_ALIGNED\(16\)\s*glm::mat4", body))
    n_vec4 = len(re.findall(r"\bglm::vec4\b", body))
    n_light = len(re.findall(r"\bLight\b", body))
    out["ubo_layout"] = {"mat4": n_mat4, "vec4": n_vec4, "light": n_light, "bytes": n_mat4 * 64 + n_vec4 * 16 + n_light * 64,
                         "src": f"{rel}:{line_of(t, m.start())}-{line_of(t, m.end())}"}

    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {OUT}: {len(out)} entries")


if __name__ == "__main__":
    main()
