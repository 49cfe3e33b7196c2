"""Adversarial triangle soups and ray sets for BVH traversal tests (numpy only, no GPU).

Every scene is an (n, 9) float32 soup (three vertices per row).  Every ray set is an (n, 8) float32 array in the layout of
hr_trace_any / hr_trace_closest: origin xyz, t_min, direction xyz, t_max.  The ground truth is always the oracle's
brute-force loop over all triangles (oracle.Scene(tri, brute=True)); these inputs target what a BVH walk can get wrong:
the box test near shared edges and vertices, ties between coincident triangles, degenerate boxes, identical Morton codes,
coordinates far from the origin, and interval ends exactly at a hit.
"""
import numpy as np

F32 = np.float32
T_FAR = F32(3.0e38)
LEAF_MAX = 2  # hybrid-rendering_b200/csrc/bvh_build.cu
MAX_DEPTH = 63  # HR_BVH_MAX_DEPTH, include/hr_api.h


def _f32(a):
    # + 0.0 turns -0.0 into +0.0: hr_scene_build applies the instance transform (x * 1 + 0), which does the same
    return (np.asarray(a, np.float64).astype(F32) + F32(0.0)).astype(F32)


def grid(nx=8, offset=(0.0, 0.0, 0.0), scale=1.0):
    """nx x nx unit quads in the plane y = offset.y, two triangles each: every interior edge and vertex is shared"""
    ox, oy, oz = offset
    out = []
    for i in range(nx):
        for j in range(nx):
            x0, x1 = ox + scale * i, ox + scale * (i + 1)
            z0, z1 = oz + scale * j, oz + scale * (j + 1)
            out.append([x0, oy, z0, x1, oy, z0, x1, oy, z1])
            out.append([x0, oy, z0, x1, oy, z1, x0, oy, z1])
    return _f32(out)


def duplicates(seed=0):
    """the 8x8 grid with every triangle repeated 2-4 times, some copies with reversed winding, rows shuffled"""
    rng = np.random.default_rng(seed)
    base = grid(8)
    rows = []
    for t in base:
        for k in range(int(rng.integers(2, 5))):
            rows.append(t if k % 2 == 0 else t.reshape(3, 3)[[0, 2, 1]].reshape(9))
    rows = np.array(rows, F32)
    return np.ascontiguousarray(rows[rng.permutation(len(rows))])


def degenerate(seed=0):
    """a 4x4 grid mixed with zero-area triangles: three collinear vertices on a line parallel to an axis, or three equal
    vertices.  For both the ray/triangle determinant is exactly 0 in fp32, so no ray hits them, but their boxes (zero
    thickness in two or three axes) sit on the grid's edges and vertices.
    Thin slivers and collinear triangles on other lines are left out on purpose: Moeller-Trumbore is ill-conditioned on
    them and reports hits off the triangle, outside any box of its vertices, so no conservative box test agrees with it."""
    rng = np.random.default_rng(seed)
    g = grid(4)
    extra = []
    for _ in range(32):
        c = rng.integers(0, 16, 3) * [0.25, 0, 0.25] + [0, 0.25 * int(rng.integers(-4, 5)), 0]
        e = np.eye(3)[int(rng.integers(0, 3))] * 0.25 * int(rng.integers(1, 5))
        extra.append(np.concatenate([c, c + e, c + 3 * e]))                       # collinear along an axis
        p = rng.integers(0, 17, 3) * [0.25, 0, 0.25] + [0, 0.25 * int(rng.integers(-4, 5)), 0]
        extra.append(np.concatenate([p, p, p]))                                  # a point
    soup = np.concatenate([g, _f32(extra)])
    return np.ascontiguousarray(soup[rng.permutation(len(soup))])


def same_centroid(n=48, centre=(1.0, 2.0, 3.0)):
    """nested, scaled triangles whose boxes all have the same centre: every Morton code is equal"""
    c = np.array(centre)
    out = []
    for k in range(n):
        s = 0.25 * (k + 1)  # exact in fp32, so every box centre is exactly `centre`
        a, b, d = np.array([-s, -s, 0.0]), np.array([s, -s, 0.0]), np.array([0.0, s, 0.0])
        perm = [[0, 1, 2], [2, 0, 1], [1, 2, 0]][k % 3]  # the triangle in the xy, zx or yz plane
        out.append(np.concatenate([(c + a[perm]), (c + b[perm]), (c + d[perm])]))
    return _f32(out)


def flat_sheets():
    """4x4 grids in the planes x = 0, y = 0 and z = 0 (each box has zero thickness before padding), moved apart"""
    g = grid(4).reshape(-1, 3, 3)
    xy = g[..., [0, 2, 1]] + [0.0, 0.0, 0.0]        # z = 0
    yz = g[..., [1, 0, 2]] + [6.0, 0.0, 0.0]        # x = 6
    zx = g + [0.0, 0.0, 6.0]                         # y = 0
    return _f32(np.concatenate([xy, yz, zx]).reshape(-1, 9))


def tiny(n):
    """n triangles: n <= LEAF_MAX is the single-node tree with one leaf (and a dummy second child)"""
    base = [[0, 0, 0, 1, 0, 0, 0, 0, 1], [1, 0, 0, 1, 0, 1, 0, 0, 1], [0, 1, 0, 1, 1, 0, 0, 1, 1], [2, 0, 0, 3, 0, 0, 2, 1, 0]]
    return _f32(base[:n])


def chain(n):
    """n triangles in planes x = 2^k (k < n), each crossing the x axis: the builders' tree is a chain of height n - 1.
    PLOC merges one pair per round (the smallest union is always the cluster of the lowest triangles and the next one)."""
    out = []
    for k in range(n):
        x = 2.0 ** k
        out.append([x, -1.0, -1.0, x, 2.0, -1.0, x, -1.0, 2.0])
    return _f32(out)


def random_soup(n, seed=0, extent=10.0, size=1.0):
    """n triangles of random orientation and size up to `size`, centred uniformly in a cube of side `extent`"""
    rng = np.random.default_rng(seed)
    c = rng.uniform(0.0, extent, (n, 1, 3))
    return _f32((c + rng.uniform(-0.5, 0.5, (n, 3, 3)) * size * rng.uniform(0.05, 1.0, (n, 1, 1))).reshape(n, 9))


def clustered(n_clusters=8, per=64, seed=0):
    """Gaussian clusters of small triangles, cluster sizes and spreads varying, far apart from each other"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_clusters):
        c = rng.uniform(0.0, 100.0, 3)
        s = 10.0 ** rng.uniform(-1, 1)
        out.append(c + rng.normal(0.0, s, (per, 1, 3)) + rng.uniform(-0.2, 0.2, (per, 3, 3)) * s)
    return _f32(np.concatenate(out).reshape(-1, 9))


def strip(quads=512):
    """a long planar strip of unit quads along x in the plane y = 0, two triangles each"""
    out = []
    for i in range(quads):
        out.append([i, 0, 0, i + 1, 0, 0, i + 1, 0, 1])
        out.append([i, 0, 0, i + 1, 0, 1, i, 0, 1])
    return _f32(out)


def far_pairs(n, size=0.01, spacing=100.0):
    """n // 2 pairs of small triangles (side `size`), the two of a pair about a unit apart and the pairs `spacing` apart
    (plus one more triangle for odd n): the cheapest trees keep a pair as an internal node over two one-triangle leaves,
    since one leaf of both would be tested by every ray that enters the pair's long box"""
    tri = np.array([0.0, 0.0, 0.0, size, 0.0, 0.0, 0.0, size, size])
    return _f32([tri + np.tile([spacing * (k // 2) + (k % 2), 0.5 * (k % 2), 0.25 * (k % 2)], 3) for k in range(n)])


def points_and_segments(n, seed=0):
    """zero-area boxes: points (three equal vertices, every other one twice) and segments along an axis, at random places.
    Two copies of a point cost 0 as one leaf and 0 as an inner node: the build packs them as a leaf (ties go to the leaf)."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        p = out[-2][:3] if k % 4 == 2 else rng.uniform(0.0, 8.0, 3)
        if k % 2 == 0:
            out.append(np.concatenate([p, p, p]))
        else:
            e = np.eye(3)[int(rng.integers(0, 3))] * rng.uniform(0.1, 3.0)
            out.append(np.concatenate([p, p + e, p + 0.5 * e]))
    return _f32(out)


def deep_chain_cluster():
    """chain(62) and five small triangles among its lowest ones, found by a search with the treelet restatement
    (bvh_treelet.py): plain PLOC builds it exactly MAX_DEPTH deep (DEEP_CHAIN_CLUSTER_PLOC), and the cheapest treelet at the
    chain's bottom would take a triangle one level deeper, so the restructuring's depth guard has to refuse it"""
    cluster = [
        [0.6619769930839539, -0.43171611428260803, 1.9393442869186401, 0.5848695039749146, -0.4460156559944153, 1.896966814994812,
         0.599098801612854, -0.550525963306427, 1.941376805305481],
        [2.0024828910827637, 0.25815069675445557, 0.11551348865032196, 2.6716103553771973, 0.07642986625432968, 0.5076364278793335,
         2.725355625152588, 0.25231078267097473, 0.3219222128391266],
        [2.295197010040283, 1.3277125358581543, 0.004972369875758886, 1.9215171337127686, 1.5196951627731323, 0.023755604401230812,
         2.0728631019592285, 1.2457642555236816, -0.11852587759494781],
        [1.1302663087844849, -0.001505021471530199, -0.006700961850583553, 1.1840806007385254, 0.08699750900268555,
         -0.015070694498717785, 1.2224746942520142, -0.05395051836967468, 0.12170501053333282],
        [0.6048675179481506, 1.1207380294799805, 0.28542760014533997, 0.6170430779457092, 1.113888144493103, 0.2835697531700134,
         0.6057540774345398, 1.1093798875808716, 0.28516000509262085],
    ]
    return np.ascontiguousarray(np.concatenate([chain(62), _f32(cluster)]))


def _deep_chain_cluster_ploc():
    t = (((("leaf", 65, 66), 62), 0), ((("leaf", 63, 64), 1), 2))
    for k in range(3, 62):
        t = (t, k)
    return t


# plain PLOC's tree of deep_chain_cluster() in bvh_treelet.ordered form (primitive ids; ("leaf", a, b) is a packed leaf)
DEEP_CHAIN_CLUSTER_PLOC = _deep_chain_cluster_ploc()


def scene_bounds(tri):
    v = tri.reshape(-1, 3).astype(np.float64)
    return v.min(0), v.max(0)


def _unit(d):
    d = np.asarray(d, np.float64)
    return d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-300)


def _rays(o, d, tmin, tmax):
    n = len(o)
    r = np.zeros((n, 8), F32)
    r[:, 0:3] = np.asarray(o, np.float64).astype(F32)
    r[:, 3] = tmin
    r[:, 4:7] = np.asarray(d, np.float64).astype(F32)
    r[:, 7] = tmax
    return r


def edge_vertex_targets(tri, rng, n):
    """points on the soup's vertices, edge midpoints and random points along edges (rounded to fp32)"""
    v = tri.reshape(-1, 3, 3).astype(np.float64)
    k = rng.integers(0, len(v), n)
    e = rng.integers(0, 3, n)
    a, b = v[k, e], v[k, (e + 1) % 3]
    w = rng.choice([0.0, 0.5, 1.0, -1.0], n)
    w = np.where(w < 0, rng.uniform(0, 1, n), w)
    return (a + w[:, None] * (b - a)).astype(F32).astype(np.float64)


def aimed(tri, rng, n, dist):
    """rays aimed at vertices and edges from `dist` times the scene extent, from random directions on both sides"""
    lo, hi = scene_bounds(tri)
    ext = max(float((hi - lo).max()), 1e-30)
    p = edge_vertex_targets(tri, rng, n)
    u = _unit(rng.normal(size=(n, 3)))
    o = (p + u * (dist * ext)).astype(F32).astype(np.float64)
    return _rays(o, _unit(p - o), 0.0, T_FAR)


def grazing(tri, rng, n, axis=1):
    """rays 1e-6 to 1e-3 (times the extent) out of the plane coordinate[axis] = that of the first vertex, aimed at edges and
    vertices from outside the scene's box, nearly parallel to the plane"""
    lo, hi = scene_bounds(tri)
    ext = max(float((hi - lo).max()), 1e-30)
    plane = float(tri[0, axis])
    p = edge_vertex_targets(tri, rng, n)
    p[:, axis] = plane
    u = rng.normal(size=(n, 3))
    u[:, axis] = 0.0
    u = _unit(u)
    h = 10.0 ** rng.uniform(-6, -3, n) * ext * rng.choice([-1.0, 1.0], n)
    o = p + u * (1.5 * ext)
    o[:, axis] = plane + h
    o = o.astype(F32).astype(np.float64)
    d = _unit(p - o)
    return _rays(o, d, 0.0, T_FAR)


def axis_aligned(tri, rng, n):
    """rays along the coordinate axes through edge / vertex targets, with exact 0.0 and -0.0 in the other components"""
    lo, hi = scene_bounds(tri)
    ext = max(float((hi - lo).max()), 1e-30)
    p = edge_vertex_targets(tri, rng, n)
    ax = rng.integers(0, 3, n)
    sgn = rng.choice([-1.0, 1.0], n)
    d = np.zeros((n, 3))
    d[np.arange(n), ax] = sgn
    o = p - d * (2.0 * ext)
    r = _rays(o, d, 0.0, T_FAR)
    neg = rng.random((n, 3)) < 0.5
    r[:, 4:7] = np.where((r[:, 4:7] == 0) & neg, F32(-0.0), r[:, 4:7])
    return r


def tiny_components(tri, rng, n):
    """like axis_aligned, but the other two components are between 1e-18 (the slab setup's clamp) and 1e-6, either sign"""
    r = axis_aligned(tri, rng, n)
    d = r[:, 4:7].astype(np.float64)
    small = 10.0 ** rng.uniform(-18, -6, (n, 3)) * rng.choice([-1.0, 1.0], (n, 3))
    d = np.where(d == 0, small, d)
    r[:, 4:7] = d.astype(F32)
    return r


def from_surface(tri, rng, n):
    """rays starting on a triangle (random barycentrics) or at a vertex, t_min = 0, random directions"""
    v = tri.reshape(-1, 3, 3).astype(np.float64)
    k = rng.integers(0, len(v), n)
    b = rng.dirichlet([1, 1, 1], n)
    b[: n // 4] = np.eye(3)[rng.integers(0, 3, n // 4)]
    o = np.einsum("ni,nij->nj", b, v[k])
    return _rays(o, _unit(rng.normal(size=(n, 3))), 0.0, T_FAR)


def interval_ends(rays, t_hit, hit):
    """for rays with a closest hit at t: t_max = t (the hit is excluded: t < t_max is strict), t_max = nextafter(t, inf)
    (included), t_min = t (excluded: t > t_min is strict) and t_min = nextafter(t, -inf) (included)"""
    r, t = rays[hit], t_hit[hit]
    out = []
    for tmin, tmax in ((r[:, 3], t), (r[:, 3], np.nextafter(t, F32(np.inf))), (t, r[:, 7]), (np.nextafter(t, F32(-np.inf)), r[:, 7])):
        q = r.copy()
        q[:, 3], q[:, 7] = tmin, tmax
        out.append(q)
    return np.concatenate(out) if out else rays[:0]


# scene name -> soup; the grid also moved and scaled
SCENES = {
    "grid": lambda: grid(8),
    "grid_off1e3": lambda: grid(8, (1e3, 0.0, 1e3)),
    "grid_off2e4": lambda: grid(8, (2e4, 50.0, -2e4)),
    "grid_off1e5": lambda: grid(8, (1e5, 0.0, 0.0)),
    "grid_scale1e-3": lambda: grid(8, (0.0, 0.0, 0.0), 1e-3),
    "grid_scale1e3": lambda: grid(8, (0.0, 0.0, 0.0), 1e3),
    "duplicates": duplicates,
    "degenerate": degenerate,
    "same_centroid": same_centroid,
    "flat_sheets": flat_sheets,
    "tiny1": lambda: tiny(1),
    "tiny2": lambda: tiny(2),
    "tiny3": lambda: tiny(3),
    "tiny4": lambda: tiny(LEAF_MAX + 2),
}


def ray_families(tri, seed=0, n=4000, with_dist=(5.0, 1e3, 1e4)):
    """name -> ray set (without the interval-end rays, which need the brute-force hits: see interval_ends)"""
    rng = np.random.default_rng(seed)
    fam = {}
    for dist in with_dist:
        fam[f"aimed_{dist:g}x"] = aimed(tri, rng, n, dist)
    fam["grazing"] = np.concatenate([grazing(tri, rng, n // 3, a) for a in range(3)])
    fam["axis_aligned"] = axis_aligned(tri, rng, n)
    fam["tiny_components"] = tiny_components(tri, rng, n)
    fam["from_surface"] = from_surface(tri, rng, n)
    return fam
