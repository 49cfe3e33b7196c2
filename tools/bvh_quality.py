"""BVH quality of the device-built tree: its SAH cost and the work of the traversal walks on config 3's reflection rays.

    python tools/bvh_quality.py [--width 600] [--height 338] [--tris 262144] [--treelet-rounds R] [--json PATH]

Builds the arcade of bench.py config 3 on cuda:0, downloads the packed tree (hr_scene_download_bvh) and reports
  sah          the tree's SAH cost per ray, in the units of the build's cost model: a node step (both child boxes) costs
               SAH_CI = 75 and a triangle test SAH_CT = 80 issued instructions (csrc/bvh_build.cu), each weighted by the
               area of the box that leads to it over the root's area;
  node_steps / tri_tests per ray of the reflection trace (K12's closest-hit walk) and of its shadow rays (any-hit walk).
The rays: primary rays of the bench view (camera, 60 degree field of view) at the reduced size --width x --height find their
first hit, the mirror reflection about the hit triangle's face normal is the reflection ray (the centre of the GGX lobe K12
samples), and the reflection ray's hit casts a shadow ray toward the directional light.  The walker follows the kernels'
rules exactly (trv::node_test in fp32 without contraction, near child first, TRV_WIDEN, the closest hit shrinking tmax,
traverse.cuh), so the counts are the ones the device walks make on the same rays.  --treelet-rounds sets the build's
restructuring rounds (0 = plain PLOC) through the library's test hook.  Not part of bench.py: it measures the tree, not time.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SAH_CI, SAH_CT = 75.0, 80.0
TRV_WIDEN = np.float32(1.0000019073486328125)
SENTINEL = 0x7FFFFFFF
F32 = np.float32


def unpack(nodes, tris):
    """packed layout -> (lo0, hi0, lo1, hi1) child boxes (N, 3) each, child links (N, 2) int32, triangles (T, 3, 4)"""
    nodes = np.asarray(nodes, np.float32).reshape(-1, 4, 4)
    n0, n1, nz = nodes[:, 0], nodes[:, 1], nodes[:, 2]
    lo0 = np.stack([n0[:, 0], n0[:, 2], nz[:, 0]], 1)
    hi0 = np.stack([n0[:, 1], n0[:, 3], nz[:, 1]], 1)
    lo1 = np.stack([n1[:, 0], n1[:, 2], nz[:, 2]], 1)
    hi1 = np.stack([n1[:, 1], n1[:, 3], nz[:, 3]], 1)
    ch = np.ascontiguousarray(nodes[:, 3, :2]).view(np.int32)
    return lo0, hi0, lo1, hi1, ch, np.asarray(tris, np.float32).reshape(-1, 3, 4)


def half_area(lo, hi):
    d = (hi - lo).astype(np.float64)
    return d[..., 0] * d[..., 1] + d[..., 1] * d[..., 2] + d[..., 2] * d[..., 0]


def sah_cost(nodes, tris):
    """SAH cost per ray of the packed tree reachable from node 0, with the build's node and triangle costs"""
    lo0, hi0, lo1, hi1, ch, _ = unpack(nodes, tris)
    a = np.stack([half_area(lo0, hi0), half_area(lo1, hi1)], 1)
    root = half_area(np.minimum(lo0[0], lo1[0]), np.maximum(hi0[0], hi1[0]))
    total = SAH_CI * root
    frontier = np.array([0])
    while frontier.size:
        c = ch[frontier]                      # (m, 2)
        ar = a[frontier]
        leaf = c < 0
        cnt = (~c & 7) + 1
        total += SAH_CT * float(np.sum(ar[leaf] * cnt[leaf])) + SAH_CI * float(np.sum(ar[~leaf]))
        frontier = c[~leaf]
    return total / root


def _tri_test(T, idx, o, d, tmin, tmax):
    """trv::ray_triangle in fp32, fixed operation order; returns (hit, t)"""
    v0, e1, e2 = T[idx, 0, :3], T[idx, 1, :3], T[idx, 2, :3]

    def cross(a, b):
        return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)

    def dot(a, b):
        return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]

    p = cross(d, e2)
    dt = dot(e1, p)
    ok = dt != 0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inv = F32(1.0) / dt
        tv = o - v0
        u = dot(tv, p) * inv
        q = cross(tv, e1)
        v = dot(d, q) * inv
        t = dot(e2, q) * inv
        hit = ok & (u >= 0) & (u <= 1) & (v >= 0) & (u + v <= 1) & (t > tmin) & (t < tmax)
    return hit, t


def walk(nodes, tris, rays, closest):
    """Lock-step numpy form of trv::trace_closest / trace_any over rays (n, 8) {o, tmin, d, tmax}.
    Returns (hit, t, prim, node_steps, tri_tests) per ray; t = tmax and prim = 0xFFFFFFFF on a miss."""
    lo0, hi0, lo1, hi1, ch, T = unpack(nodes, tris)
    prim_of = np.ascontiguousarray(T[:, 0, 3]).view(np.uint32)
    rays = np.asarray(rays, np.float32)
    n = rays.shape[0]
    o, d, tmin = rays[:, 0:3], rays[:, 4:7], rays[:, 3].copy()
    best_t, best_p = rays[:, 7].copy(), np.full(n, 0xFFFFFFFF, np.uint32)
    with np.errstate(divide="ignore"):
        dd = np.where(np.abs(d) > F32(1e-18), d, np.copysign(F32(1e-18), d)).astype(np.float32)
        inv = (F32(1.0) / dd).astype(np.float32)
    stack = np.empty((n, 66), np.int32)
    stack[:, 0] = SENTINEL
    sp = np.ones(n, np.int32)
    node = np.zeros(n, np.int32)
    steps, tests = np.zeros(n, np.int64), np.zeros(n, np.int64)
    found = np.zeros(n, bool)

    def slab(r, lo, hi):
        a = (lo - o[r]) * inv[r]
        b = (hi - o[r]) * inv[r]
        tn = np.maximum(np.maximum(np.minimum(a[:, 0], b[:, 0]), np.minimum(a[:, 1], b[:, 1])), np.maximum(np.minimum(a[:, 2], b[:, 2]), tmin[r]))
        tf = np.minimum(np.minimum(np.maximum(a[:, 0], b[:, 0]), np.maximum(a[:, 1], b[:, 1])), np.minimum(np.maximum(a[:, 2], b[:, 2]), best_t[r]))
        return tn <= tf * TRV_WIDEN, tn

    def pop(r):
        sp[r] -= 1
        node[r] = stack[r, sp[r]]

    live = np.arange(n)
    while live.size:
        r = live[node[live] >= 0]
        if r.size:
            nd = node[r]
            steps[r] += 1
            h0, t0 = slab(r, lo0[nd], hi0[nd])
            h1, t1 = slab(r, lo1[nd], hi1[nd])
            c0, c1 = ch[nd, 0], ch[nd, 1]
            none = ~h0 & ~h1
            pop(r[none])
            both = h0 & h1
            nxt = np.where(h0, c0, c1)
            far = c1.copy()
            sw = both & (t1 < t0)
            nxt[sw], far[sw] = c1[sw], c0[sw]
            rb = r[both]
            stack[rb, sp[rb]] = far[both]
            sp[rb] += 1
            go = ~none
            node[r[go]] = nxt[go]
        r = live[node[live] < 0]
        r = r[node[r] != SENTINEL]
        if r.size:
            leaf = ~node[r]
            first, cnt = leaf >> 3, (leaf & 7) + 1
            stop = np.zeros(r.size, bool)
            for k in range(int(cnt.max())):
                m = (k < cnt) & ~stop
                rk = r[m]
                tests[rk] += 1
                hit, t = _tri_test(T, first[m] + k, o[rk], d[rk], tmin[rk], best_t[rk])
                if closest:
                    p = prim_of[first[m] + k]
                    upd = hit & ((t < best_t[rk]) | ((t == best_t[rk]) & (p < best_p[rk])))
                    ru = rk[upd]
                    best_t[ru], best_p[ru] = t[upd], p[upd]
                else:
                    found[rk[hit]] = True
                    stop[np.flatnonzero(m)[hit]] = True
            if closest:
                pop(r)
            else:
                node[r[stop]] = SENTINEL
                pop(r[~stop])
        live = live[node[live] != SENTINEL]
    if closest:
        found = best_p != 0xFFFFFFFF
    return found, best_t, best_p, steps, tests


def brute_closest(tris_verts, rays):
    """closest hit over every triangle (same fp32 test, ties -> lowest primitive): (t, prim)"""
    tv = np.asarray(tris_verts, np.float32).reshape(-1, 9)
    T = np.zeros((tv.shape[0], 3, 4), np.float32)
    T[:, 0, :3] = tv[:, 0:3]
    T[:, 1, :3] = tv[:, 3:6] - tv[:, 0:3]
    T[:, 2, :3] = tv[:, 6:9] - tv[:, 0:3]
    rays = np.asarray(rays, np.float32)
    n = rays.shape[0]
    best_t, best_p = rays[:, 7].copy(), np.full(n, 0xFFFFFFFF, np.uint32)
    for k in range(tv.shape[0]):
        hit, t = _tri_test(T, np.full(n, k), rays[:, 0:3], rays[:, 4:7], rays[:, 3], best_t)
        upd = hit & ((t < best_t) | ((t == best_t) & (k < best_p)))
        best_t[upd], best_p[upd] = t[upd], k
    return best_t, best_p


def bench_rays(tri_verts, nodes, tris, W, H, cam, tgt, light_dir, fovy_deg=60.0):
    """config-3 reflection rays and their shadow rays (see the module docstring): (reflection rays, shadow rays)"""
    cam, tgt = np.array(cam, np.float64), np.array(tgt, np.float64)
    fwd = (tgt - cam) / np.linalg.norm(tgt - cam)
    right = np.cross(fwd, (0.0, 1.0, 0.0))
    right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    th = np.tan(np.radians(fovy_deg) / 2)
    ys, xs = np.mgrid[0:H, 0:W]
    sx = ((xs + 0.5) / W * 2 - 1) * th * W / H
    sy = (1 - (ys + 0.5) / H * 2) * th
    d = fwd + sx[..., None] * right + sy[..., None] * up
    d = (d / np.linalg.norm(d, axis=-1, keepdims=True)).reshape(-1, 3)
    prim_rays = np.zeros((d.shape[0], 8), np.float32)
    prim_rays[:, 0:3], prim_rays[:, 3], prim_rays[:, 4:7], prim_rays[:, 7] = cam, 0.0, d, 1e4
    hit, t, prim, _, _ = walk(nodes, tris, prim_rays, True)
    tv = np.asarray(tri_verts, np.float64).reshape(-1, 3, 3)[prim[hit]]
    nrm = np.cross(tv[:, 1] - tv[:, 0], tv[:, 2] - tv[:, 0])
    nrm /= np.maximum(np.linalg.norm(nrm, axis=1, keepdims=True), 1e-30)
    di = d[hit]
    nrm *= -np.sign(np.sum(nrm * di, axis=1, keepdims=True) + 1e-30)
    p = cam + di * t[hit, None].astype(np.float64)
    rd = di - 2 * np.sum(di * nrm, axis=1, keepdims=True) * nrm
    refl = np.zeros((rd.shape[0], 8), np.float32)
    refl[:, 0:3], refl[:, 3], refl[:, 4:7], refl[:, 7] = p + nrm * 1e-3, 0.0, rd, 1e4
    rhit, rt, _, _, _ = walk(nodes, tris, refl, True)
    q = refl[rhit, 0:3].astype(np.float64) + refl[rhit, 4:7] * rt[rhit, None]
    shadow = np.zeros((q.shape[0], 8), np.float32)
    shadow[:, 0:3], shadow[:, 3], shadow[:, 4:7], shadow[:, 7] = q - refl[rhit, 4:7] * 1e-3, 0.0, light_dir, 1e4
    return refl, shadow


def measure(nodes, tris, refl, shadow):
    _, _, _, s, k = walk(nodes, tris, refl, True)
    _, _, _, ss, sk = walk(nodes, tris, shadow, False)
    return dict(sah=sah_cost(nodes, tris), rays=int(refl.shape[0]), shadow_rays=int(shadow.shape[0]),
                node_steps_per_ray=float(s.mean()), tri_tests_per_ray=float(k.mean()),
                shadow_node_steps_per_ray=float(ss.mean()), shadow_tri_tests_per_ray=float(sk.mean()))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--width", type=int, default=600)
    ap.add_argument("--height", type=int, default=338)
    ap.add_argument("--tris", type=int, default=262144)
    ap.add_argument("--treelet-rounds", type=int, nargs="*", default=[0, 3], help="build each of these and report every tree")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.ensure_built()
    import pyhr
    import bench

    sc = pyhr.SynthScene(pyhr.SCENE_ARCADE, a.tris)
    tri, _ = sc.world_triangles()
    f = pyhr.make_frame(bench.CAM_POS, bench.CAM_TGT, a.width, a.height, light=pyhr.default_light(rot_x_deg=bench.LIGHT_ROT_X))
    ld = np.array(f.ubo.light.data0[:3], np.float64)
    ld = -ld / np.linalg.norm(ld)
    if ld[1] < 0:
        ld = -ld  # toward the light, which shines from above
    ctx = pyhr.Context(0)
    hook = ctx.lib.hr_internal_bvh_treelet_rounds
    hook.argtypes = [C.c_int]
    default_rounds = hook(-1)
    trees = {}
    try:
        for r in a.treelet_rounds:
            hook(r)
            h = ctx.build_scene(sc)
            trees[r] = (ctx.download_bvh(h), ctx.scene_info(h))
            ctx.lib.hr_scene_destroy(h)
    finally:
        hook(default_rounds)
        ctx.close()
    # the same rays for every tree: generated on the first one (hits do not depend on the topology)
    (nodes, tris), _ = trees[a.treelet_rounds[0]]
    refl, shadow = bench_rays(tri, nodes, tris, a.width, a.height, bench.CAM_POS, bench.CAM_TGT, ld.astype(np.float32))
    out = {}
    for r, ((nodes, tris), info) in trees.items():
        m = measure(nodes, tris, refl, shadow)
        m["depth"] = int(info.depth)
        out[f"treelet_rounds={r}"] = m
        print(f"treelet rounds {r}: " + ", ".join(f"{k} {v:.4g}" if isinstance(v, float) else f"{k} {v}" for k, v in m.items()), flush=True)
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
