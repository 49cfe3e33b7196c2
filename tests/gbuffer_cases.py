"""Hand-built G-buffers at the inputs where the screen-space passes make a decision, shared by tests/test_gpu_adversarial_gbuffer.py
(device vs oracle) and tests/test_gbuffer_cases_cpu.py (the cases are well formed and the oracle reaches them).  numpy only, seeded.

Every other test feeds the passes G-buffers a renderer wrote, whose plane distances, normal dots and history coordinates sit far
from the thresholds of is_reprojection_valid (reprojection.glsl:52-67).  A case here is a short list of frames, each a hand-built
G-buffer (pyhr.GBufferHost, fp16 fields written as fp16 bits) and its hr_frame; the previous G-buffer of frame i is frame i - 1's.
The camera is static, so every motion vector is the case's own.  Threshold cases are LADDERS: pixels whose decisive value runs
through consecutive representable values on both sides of the threshold.

`targets` are reprojection branches ("kernel:branch", test_gpu_camera.Reach / oracle.ReprojectCodes) the case reaches in at least
MIN_PIXELS pixels of some frame that reads history.  `ladders` maps a ladder's name to the float64 signed distance of each of its
pixels from its threshold (> 0: the side the test rejects or flags), computed from the stored inputs.  `tame()` builds the frames of
the case's twin with the ladder moved off its threshold (or the decisive input made ordinary), whose oracle outputs must differ.
`prev`: the G-buffer that precedes the first frame (None: the all-zero start-up slot).  `plant`: histories planted through
hr_pass_upload, {"sh" | "ao" | "rf": (frame index, image, aux)}: before that frame's render, the image and the aux image (moments or
history length) that frame reads as history; at frame 0 through the cold-start path (before the pass's first render).
"""
from collections import namedtuple

import numpy as np

import pyhr

SIZES = ((128, 72), (97, 53))  # one size divisible by 8, one ragged (97 % 8 = 1, 53 % 8 = 5)
MIN_PIXELS = 20
PLANE_DISTANCE, NORMAL_DISTANCE = 5.0, 0.1
MESH = 3.0
# a generic view of the plane z = 0 (the plane is not perpendicular to the view: its depth varies per pixel), and a view straight
# down -z, where the plane's depth is the same at every pixel (ties in every depth comparison)
CAM = ((1.3, 4.1, 7.2), (0.2, 2.9, -0.4))
CAM_STRAIGHT = ((0.0, 3.0, 6.0), (0.0, 3.0, 0.0))

Case = namedtuple("Case", "id W H frames targets ladders tame resets prev plant", defaults=((), None, None))


def h16(a):
    """float64 / float32 values -> fp16 bits"""
    return np.asarray(a, np.float64).astype(np.float16).view(np.uint16)


def f16(bits):
    return np.asarray(bits, np.uint16).view(np.float16).astype(np.float64)


def frames(W, H, n, cam=CAM):
    out, f = [], None
    for i in range(n):
        f = pyhr.make_frame(cam[0], cam[1], W, H, prev=f, num_frames=i)
        out.append(f)
    return out


def _m(a):
    """column-major float[16] -> float64 4x4 acting on column vectors"""
    return np.array(a[:], np.float64).reshape(4, 4).T


def _tex(W, H):
    y, x = np.mgrid[0:H, 0:W]
    return (np.float32(x) + np.float32(0.5)) / np.float32(W), (np.float32(y) + np.float32(0.5)) / np.float32(H)


def world_pos(f, u, v, d):
    """world_position_from_depth in float64 of float32 inputs"""
    M = _m(f.ubo.view_proj_inverse)
    ndc = np.stack([np.float64(u) * 2 - 1, np.float64(v) * 2 - 1, np.asarray(d, np.float64), np.ones(np.shape(d))], -1)
    w = ndc @ M.T
    return w[..., :3] / w[..., 3:4]


def depth_on_plane(f, W, H, z):
    """float64 NDC depth of the point where each pixel's ray meets the plane world z = `z` (z may be per pixel)"""
    u, v = _tex(W, H)
    M = _m(f.ubo.view_proj_inverse)
    sx, sy = np.float64(u) * 2 - 1, np.float64(v) * 2 - 1
    # wz(d) / ww(d) = z, both affine in d
    az = M[2, 0] * sx + M[2, 1] * sy + M[2, 3]
    aw = M[3, 0] * sx + M[3, 1] * sy + M[3, 3]
    return (z * aw - az) / (M[2, 2] - z * M[3, 2])


def clip_z(f, P):
    c = np.concatenate([P, np.ones(P.shape[:-1] + (1,))], -1) @ _m(f.ubo.view_proj).T
    return c[..., 2]


def ulp_steps(d64, k):
    """float32 nearest d64, moved k float32 steps (k per pixel)"""
    d = np.float32(d64)
    k = np.broadcast_to(k, d.shape)
    out = d.copy()
    for s in range(1, int(np.abs(k).max()) + 1):
        out = np.where(k >= s, np.nextafter(out, np.float32(np.inf)), out)
        out = np.where(k <= -s, np.nextafter(out, np.float32(-np.inf)), out)
    return out.astype(np.float32)


def plane(f, W, H, z=0.0, depth=None, oct_xy=(0.0, 0.0), mesh=MESH, roughness=0.3, metallic=0, sky=None, motion=(0.0, 0.0)):
    """a G-buffer of the plane world z = `z` (or of `depth`, float32 per pixel), normal from the octahedral pair oct_xy (per pixel
    arrays or scalars), mesh id, roughness and motion per pixel or scalar; sky: bool mask of sky pixels (the clear values).
    Curvature is 0 on even rows and 0.25 on odd ones, so the reflections reprojection takes both its virtual-point and its
    motion-vector path."""
    g = pyhr.GBufferHost(W, H)
    d = np.float32(depth_on_plane(f, W, H, z)) if depth is None else np.asarray(depth, np.float32)
    u, v = _tex(W, H)
    P = world_pos(f, u, v, d)
    g.depth[:] = d
    g.gb2[..., 0] = h16(np.broadcast_to(oct_xy[0], (H, W)))
    g.gb2[..., 1] = h16(np.broadcast_to(oct_xy[1], (H, W)))
    g.gb2[..., 2] = h16(np.broadcast_to(motion[0], (H, W)))
    g.gb2[..., 3] = h16(np.broadcast_to(motion[1], (H, W)))
    g.gb3[..., 0] = h16(np.broadcast_to(roughness, (H, W)))
    g.gb3[..., 1] = h16(np.where(np.arange(H)[:, None] % 2 == 1, 0.25, 0.0) * np.ones((1, W)))
    g.gb3[..., 2] = h16(np.broadcast_to(mesh, (H, W)))
    g.gb3[..., 3] = h16(clip_z(f, P))
    g.gb1[..., 0], g.gb1[..., 1], g.gb1[..., 2] = 200, 140, 90
    g.gb1[..., 3] = np.broadcast_to(metallic, (H, W))
    if sky is not None:
        g.depth[sky] = 1.0
        g.gb2[sky] = 0
        g.gb3[sky] = 0
        g.gb3[..., 3][sky] = h16(-1.0)
        g.gb1[sky] = 0
    return g


def _pattern(W, H, n):
    """a per-pixel index 0 .. n-1 that changes from each pixel to its neighbours"""
    y, x = np.mgrid[0:H, 0:W]
    return (x * 7 + y * 3) % n


# ---------------------------------------------------------------------------------------------- plane distance
LADDER_K = 4  # float32 steps either side


def _plane_distance(W, H, tame=False):
    """the plane z = 0 and, behind it, the plane moved 5.0 along its normal (+z) with a ladder of float32 depth steps around
    exactly 5.0: frames far, far, near, far, near, so the history is long when the ladder decides, in both directions"""
    fs = frames(W, H, 5)
    f = fs[0]
    u, v = _tex(W, H)
    near = plane(f, W, H, 0.0)
    cz = world_pos(f, u, v, near.depth)[..., 2]
    d64 = depth_on_plane(f, W, H, cz - (4.0 if tame else PLANE_DISTANCE))
    k = _pattern(W, H, 2 * LADDER_K + 1) - LADDER_K
    far = plane(f, W, H, depth=ulp_steps(d64, k))
    dist = np.abs(cz - world_pos(f, u, v, far.depth)[..., 2])
    seq = [far, far, near, far, near]
    return list(zip(seq, fs)), {"plane distance": dist - PLANE_DISTANCE}


# ---------------------------------------------------------------------------------------------- normal distance
def oct_decode(ex, ey):
    """octohedral_to_direction in float64"""
    ex, ey = np.asarray(ex, np.float64), np.asarray(ey, np.float64)
    z = 1 - np.abs(ex) - np.abs(ey)
    x = np.where(z < 0, (1 - np.abs(ey)) * np.where(ex < 0, -1.0, 1.0), ex)
    y = np.where(z < 0, (1 - np.abs(ex)) * np.where(ey < 0, -1.0, 1.0), ey)
    v = np.stack([x, y, z], -1)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


_NORMAL_PAIRS = None


def normal_ladder(n=48):
    """fp16 octohedral pairs (ex, ey) whose normal's dot with (0, 0, 1), squared, lies nearest NORMAL_DISTANCE: the n nearest above
    and the n nearest below, from a float64 search over the fp16 grid (for every fp16 ex in (0, 1), the fp16 neighbours of the ey
    that puts dot^2 on the threshold), both signs of each component"""
    global _NORMAL_PAIRS
    if _NORMAL_PAIRS is None:
        ex = np.arange(0x1400, 0x3C00, dtype=np.uint16).view(np.float16).astype(np.float64)  # fp16 values in [2^-10, 1)
        lo, hi = np.zeros_like(ex), 1 - ex
        for _ in range(80):  # dot^2 = z^2 / (ex^2 + ey^2 + z^2) falls as ey grows
            mid = (lo + hi) / 2
            above = oct_decode(ex, mid)[..., 2] ** 2 > NORMAL_DISTANCE
            lo, hi = np.where(above, mid, lo), np.where(above, hi, mid)
        ey0 = lo.astype(np.float16)
        cand = []
        for ey in (ey0, np.nextafter(ey0, np.float16(1)), np.nextafter(ey0, np.float16(0))):
            cand.append(np.stack([ex, ey.astype(np.float64)], -1))
        c = np.concatenate(cand)
        r = oct_decode(c[:, 0], c[:, 1])[..., 2] ** 2 - NORMAL_DISTANCE
        ia, ib = np.where(r > 0)[0], np.where(r < 0)[0]
        pick = np.concatenate([ia[np.argsort(r[ia])[:n]], ib[np.argsort(-r[ib])[:n]]])
        _NORMAL_PAIRS = c[pick]
    return _NORMAL_PAIRS


def _normal_distance(W, H, tame=False):
    """the plane z = 0, frames with normal oct (0, 0) = (0, 0, 1) alternating with frames whose normals are the fp16 ladder around
    dot^2 = 0.1 (signs of ex / ey varied over the pixels); same depth and mesh id, so only the normal test decides"""
    fs = frames(W, H, 5)
    f = fs[0]
    pairs = normal_ladder()
    idx = _pattern(W, H, len(pairs))
    sgn = np.array([(1, 1), (-1, 1), (1, -1), (-1, -1)], np.float64)[np.arange(H) % 4][:, None, :]  # row r: the signs of row r % 4
    ex, ey = pairs[idx, 0] * sgn[..., 0], pairs[idx, 1] * sgn[..., 1]
    if tame:
        ex, ey = ex * 0.5, ey * 0.5
    flat, tilted = plane(f, W, H), plane(f, W, H, oct_xy=(ex, ey))
    r = oct_decode(f16(tilted.gb2[..., 0]), f16(tilted.gb2[..., 1]))[..., 2] ** 2
    seq = [flat, flat, tilted, flat, tilted]
    return list(zip(seq, fs)), {"normal dot^2": NORMAL_DISTANCE - r}


# ---------------------------------------------------------------------------------------------- frame edges
def edge_motion(x, t, n, side):
    """the fp16 motion m whose history_coord_floor rn(rn(m * n) + x) (float32, as the kernels and the oracle round it) is exactly t,
    else the nearest one below (side < 0) or above (side > 0) t"""
    m0 = np.float16((t - x) / n)
    steps = np.arange(-256, 257)
    c = (np.full(steps.shape, m0).view(np.uint16).astype(np.int32) + np.where(m0 < 0, -steps, steps)).astype(np.uint16).view(np.float16)
    c = c[np.isfinite(c)]
    h = np.float32(c.astype(np.float32) * np.float32(n)) + np.float32(x)
    if (h == np.float32(t)).any():
        return c[h == np.float32(t)][0]
    pick = h < t if side < 0 else h > t
    d = np.abs(h.astype(np.float64) - t)
    return c[pick][np.argmin(d[pick])]


def _edges(W, H, tame=False):
    """motion vectors that put history_coord_floor at -1.5, -1, -0.5, -2^-10, 0, W-1, W-0.5, W-2^-8, W (and the same in y) from the
    pixels of the two border columns / rows, exactly where an fp16 motion reaches it, else at the nearest values on both sides
    (fp16 motions found by search); motion of +-0.0, and motion larger than the frame"""
    fs = frames(W, H, 4)
    f = fs[0]
    y, x = np.mgrid[0:H, 0:W]
    mx = np.where(x % 2 == 0, -0.0, 0.0)  # +-0.0 everywhere else
    my = np.where(y % 2 == 0, -0.0, 0.0)
    reached = {}
    for axis, n, a, b in (("x", W, x, y), ("y", H, y, x)):
        targets = np.array([-1.5, -1.0, -0.5, -2.0 ** -10, 0.0, n - 1.0, n - 0.5, n - 2.0 ** -8, float(n)])
        m = mx if axis == "x" else my
        for p in (0, 1, n - 2, n - 1):
            for ti, t in enumerate(targets):
                for side in (-1, 1):
                    sel = (a == p) & ((b + p) % 18 == 2 * ti + (side > 0))
                    mv = edge_motion(p, t, n, side)
                    m = np.where(sel, np.float64(mv), m)
                    reached.setdefault(f"{axis} {t:g}", []).append(float(np.float32(np.float32(mv) * np.float32(n)) + np.float32(p)) - t)
        if axis == "x":
            mx = m
        else:
            my = m
    big = (x % 11 == 5) & (y % 7 == 3)
    mx = np.where(big, np.where(x % 2 == 0, 1.5, -1.25), mx)
    if tame:
        mx, my = mx * 0.0, my * 0.0
    g = plane(f, W, H, motion=(mx, my))
    seq = [plane(f, W, H), plane(f, W, H), g, g]
    # per target: the reached history_coord_floor minus the target (0: hit exactly)
    return list(zip(seq, fs)), {}, {k: np.array(v) for k, v in reached.items()}


# ---------------------------------------------------------------------------------------------- sumw
def _sumw(W, H, tame=False):
    """history meshes match only on even (x, y) texels, and in rows y % 4 == 0 also on the texel right of them.  Pixels on even
    texels move by (fx, fy) = (f, f), f an fp16 ladder around 0.9, so their only valid bilinear tap has weight (1 - f)^2 around
    0.01, or (rows y % 4 == 0, f around 0.93) two valid taps, (1 - f)^2 + f (1 - f) around 0.01: a sum of two products, which a
    contracted kernel would fuse; pixels on odd columns do not move (fx = 0), so their valid right-hand tap has weight exactly 0"""
    fs = frames(W, H, 4)
    f = fs[0]
    y, x = np.mgrid[0:H, 0:W]
    two = (y % 4 == 0)
    hist_mesh = np.where(((x % 2 == 0) | (two & (x % 2 == 1))) & (y % 2 == 0), MESH, MESH + 2)
    target = 0.0 if tame else 0.9
    # fp16 motion m with m * W (and m * H) stepping through the values around `target` texels
    k = _pattern(W, H, 2 * LADDER_K + 1) - LADDER_K
    # two valid taps (1 - fx)(1 - fy) + fx (1 - fy) = 1 - fy: fy around 0.99, fx anywhere (0.5)
    mx = np.where(two, np.float16(0.0 if tame else 0.5 / W), np.float16(target / W)).astype(np.float16)
    my = np.where(two, np.float16(0.0 if tame else 0.99 / H), np.float16(target / H)).astype(np.float16)
    for s in range(1, LADDER_K + 1):
        mx = np.where(k >= s, np.nextafter(mx, np.float16(1)), np.where(k <= -s, np.nextafter(mx, np.float16(-1)), mx))
        my = np.where(k >= s, np.nextafter(my, np.float16(1)), np.where(k <= -s, np.nextafter(my, np.float16(-1)), my))
    even = (x % 2 == 0) & (y % 2 == 0)
    mx, my = np.where(even, mx, 0.0), np.where(even, my, 0.0)
    hist = plane(f, W, H, mesh=hist_mesh)
    g = plane(f, W, H, motion=(mx, my))
    fx = (np.float32(f16(g.gb2[..., 2])) * np.float32(W) + np.float32(x)) - x
    fy = (np.float32(f16(g.gb2[..., 3])) * np.float32(H) + np.float32(y)) - y
    w0 = (1 - np.float64(fx)) * (1 - np.float64(fy))
    w01 = w0 + np.float64(fx) * (1 - np.float64(fy))
    seq = [hist, hist, g, hist]
    inner = even & (y < H - 1) & (x < W - 1)
    return list(zip(seq, fs)), {"sumw, one tap": (0.01 - w0)[inner & ~two], "sumw, two taps": (0.01 - w01)[inner & two]}


# ---------------------------------------------------------------------------------------------- mesh ids
def _mesh_ids(W, H, tame=False):
    """fx = fy = 0.5: all four bilinear taps weigh 0.25, and one of them (in turn) carries another mesh id; mesh ids 2047 against
    2048 (one fp16 step), 2049 (stored as 2048) against 2048; mesh id 0 against the all-zero texel outside the frame"""
    fs = frames(W, H, 4)
    f = fs[0]
    y, x = np.mgrid[0:H, 0:W]
    cur_mesh = np.full((H, W), 2048.0)
    cur_mesh[:, ::3] = 2049.0
    hist_mesh = np.full((H, W), 2048.0)
    if not tame:
        hist_mesh[(x % 4 == 1) & (y % 3 == 0)] = 2047.0
        hist_mesh[(x % 5 == 2) & (y % 3 == 1)] = 2047.0
        hist_mesh[(x % 3 == 0) & (y % 4 == 2)] = 7.0
    cur_mesh[:, -2:] = 0.0  # the right border moves out of the frame: mesh id 0 meets the zero texel
    mx = np.where(x >= W - 2, 2.0 / W, 0.5 / W)
    g = plane(f, W, H, mesh=cur_mesh, motion=(mx, 0.5 / H))
    hist = plane(f, W, H, mesh=np.where(x >= W - 2, 0.0, hist_mesh))
    seq = [hist, hist, g, hist]
    return list(zip(seq, fs)), {}


# ---------------------------------------------------------------------------------------------- depth: sky, 0, nextafter(1, 0)
def _depth(W, H, tame=False):
    """sky / geometry checkerboards, single-pixel islands, fully-sky 8x8 tiles and tiles with one geometry pixel (on the ragged
    border too); depth nextafter(1, 0) next to sky (1.0), and depth 0"""
    fs = frames(W, H, 4)
    f = fs[0]
    y, x = np.mgrid[0:H, 0:W]
    ty, tx = y // 8, x // 8
    sky = np.zeros((H, W), bool)
    sky |= (tx % 4 == 0) & ((x + y) % 2 == 0)              # checkerboard tiles
    sky |= (tx % 4 == 1) & ~((x % 5 == 2) & (y % 5 == 2))  # single-pixel islands
    sky |= (tx % 4 == 2) & (ty % 2 == 0)                   # fully-sky tiles
    one = (tx % 4 == 3) | (tx == (W - 1) // 8) | (ty == (H - 1) // 8)
    sky |= one & ~((x % 8 == 3) & (y % 8 == 4)) & (ty % 2 == 1)  # one geometry pixel per tile, the border tiles included
    if tame:
        sky[:] = False
    base = plane(f, W, H)
    d = base.depth.copy()
    d[(x % 13 == 6) & (y % 9 == 4)] = np.nextafter(np.float32(1), np.float32(0))
    d[(x % 17 == 8) & (y % 11 == 5)] = 0.0
    g = plane(f, W, H, depth=d, sky=sky)
    g2 = plane(f, W, H, depth=d, sky=np.roll(sky, 1, axis=1))
    seq = [g, g, g2, g]
    return list(zip(seq, fs)), {}


# ---------------------------------------------------------------------------------------------- normals
def _normals(W, H, tame=False):
    """octahedral encodings on the fold lines |x| + |y| = 1, at the corners (+-1, +-1), (+-1, 0), (0, +-1), and with +-0.0
    components, the same in both frames and against the flat normal"""
    fs = frames(W, H, 4)
    f = fs[0]
    t = np.array([0.0, 0.125, 0.25, 0.375, 0.5, 0.625, 0.75, 0.875, 1.0])
    pts = [(a, 1 - a) for a in t] + [(1.0, 1.0), (1.0, 0.0), (0.0, 1.0), (-0.0, 0.5), (0.5, -0.0), (-0.0, -0.0), (-0.0, 1.0), (0.25, 0.25)]
    pts = [(sx * a, sy * b) for a, b in pts for sx in (1, -1) for sy in (1, -1)]
    pts = np.array(pts, np.float64)
    idx = _pattern(W, H, len(pts))
    ex, ey = pts[idx, 0], pts[idx, 1]
    if tame:
        ex, ey = ex * 0.0 + 0.25, ey * 0.0 + 0.25
    g = plane(f, W, H, oct_xy=(ex, ey))
    seq = [g, g, plane(f, W, H), g]
    return list(zip(seq, fs)), {}


# ---------------------------------------------------------------------------------------------- roughness / metallic
def fp16_around(v, k=LADDER_K):
    """the fp16 values nearest v: k below and k at or above"""
    h = np.float16(v)
    below = [h if np.float64(h) < v else np.nextafter(h, np.float16(-1))]
    above = [h if np.float64(h) >= v else np.nextafter(h, np.float16(1))]
    for _ in range(k - 1):
        below.append(np.nextafter(below[-1], np.float16(-1)))
        above.append(np.nextafter(above[-1], np.float16(1)))
    return np.array(below[::-1] + above, np.float64)


def _roughness(W, H, tame=False):
    """roughness ladders over the fp16 values around 0.05 (fp16(0.05) < 0.05f) and 0.75, roughness 0 (mirror) and 1, metallic 0
    and 1, and grazing normals (K12's reflected ray tangent to the surface)"""
    fs = frames(W, H, 4)
    f = fs[0]
    lo, hi = fp16_around(0.05), fp16_around(0.75)
    vals = np.concatenate([lo, hi, [0.0, 1.0]])
    if tame:
        vals = np.full_like(vals, 0.3)
    y, x = np.mgrid[0:H, 0:W]
    idx = ((x // 8) * 5 + (y // 8) * 3) % len(vals)  # one value per 8x8 tile: the tile flag reads the whole tile
    r = vals[idx]
    metallic = np.where((x // 2 + y) % 2 == 0, 0, 255).astype(np.uint8)
    # grazing: normal perpendicular to the view direction in some columns (oct encoding of a direction in the view plane)
    cam, tgt = np.array(CAM[0]), np.array(CAM[1])
    vd = (tgt - cam) / np.linalg.norm(tgt - cam)
    n = np.cross(vd, (0.0, 1.0, 0.0))
    n /= np.abs(n).sum()
    graze = (x % 9 == 4)
    ex = np.where(graze, n[0], 0.0)
    ey = np.where(graze, n[1], 0.0)
    g = plane(f, W, H, roughness=r, metallic=metallic, oct_xy=(ex, ey))
    seq = [g, g, g, g]
    return list(zip(seq, fs)), {"roughness 0.05": 0.05 - lo, "roughness 0.75": hi - 0.75}


# ---------------------------------------------------------------------------------------------- ties
def _ties(W, H, tame=False):
    """the plane straight in front of the camera: every pixel has the same depth, so every upsample footprint and every TAA 3x3
    neighbourhood compares equal depths and only the tie order picks the texel.  Each texel of a 3x3 neighbourhood carries another
    small motion vector (TAA fetches its history at the chosen texel's motion) and another normal (the upsample's candidates
    differ), so the texel the tie order picks shows in the output"""
    cam = CAM if tame else CAM_STRAIGHT
    fs = frames(W, H, 4, cam)
    y, x = np.mgrid[0:H, 0:W]
    k = (x % 3) + 3 * (y % 3)  # 0 .. 8 over every 3x3 neighbourhood
    mx, my = (k - 4) * 2.0 ** -9, ((k * 5) % 9 - 4) * 2.0 ** -9
    ex, ey = (k % 3 - 1) * 0.0625, (k // 3 - 1) * 0.0625
    g0 = plane(fs[0], W, H, oct_xy=(ex, ey))
    g = plane(fs[0], W, H, oct_xy=(ex, ey), motion=(mx, my))
    return list(zip([g0, g0, g, g], fs)), {}


# ---------------------------------------------------------------------------------------------- planted histories
def _tiles(W, H, vals):
    """one of `vals` per 8x8 tile (the tile classification reads whole tiles)"""
    y, x = np.mgrid[0:H, 0:W]
    return np.asarray(vals, np.float64)[((x // 8) * 3 + (y // 8)) % len(vals)]


def _planted(W, H, tame=False):
    """a static plane whose first frame reads a planted history: shadows and AO through the cold-start path, the reflections after
    their first frame.  History colours exactly 0, 1, one fp16 step below 1 and 0.5 per 8x8 tile (the tile classification compares
    the blended colour with 0 / 1), history lengths 0, 1, 30, 31 and 32 (the cap) per pixel, second moments up to 16"""
    fs = frames(W, H, 3)
    g = plane(fs[0], W, H)
    if tame:
        return list(zip([g] * 3, fs)), {}, g, None
    y, x = np.mgrid[0:H, 0:W]
    cols = (0.0, 1.0, 1.0 - 2.0 ** -11, 0.5)
    lens = np.array([0.0, 1.0, 30.0, 31.0, 32.0])
    AW, AH = max(W // 2, 1), max(H // 2, 1)
    ln, aln = lens[(x * 3 + y) % 5], lens[(np.mgrid[0:AH, 0:AW][1] * 3 + np.mgrid[0:AH, 0:AW][0]) % 5]
    c = _tiles(W, H, cols)
    m2 = np.array([0.0, 1.0, 16.0])[(x + y) % 3]
    sh_img = h16(np.stack([c, np.zeros_like(c)], -1))
    sh_mom = h16(np.stack([c, np.maximum(m2, c * c), ln, np.zeros_like(c)], -1))
    ao_col, ao_len = h16(_tiles(AW, AH, cols)), h16(aln)
    rgb = np.stack([c, _tiles(W, H, cols[::-1]), np.full_like(c, 0.5)], -1)
    rf_img = h16(np.concatenate([rgb, np.zeros_like(c)[..., None]], -1))
    rf_mom = h16(np.stack([c, np.maximum(m2, c * c), ln, np.zeros_like(c)], -1))
    plant = {"sh": (0, sh_img, sh_mom), "ao": (0, ao_col, ao_len), "rf": (1, rf_img, rf_mom)}
    return list(zip([g] * 3, fs)), {"history length 32": ln - 31.5}, g, plant


def plant_device(case, i, sh=None, ao=None, rf=None):
    """hr_pass_upload the histories case.plant plants before frame i: shadows (prev image 5, moments 4), AO (temporal 1, length 4),
    reflections (temporal 1, moments 4)"""
    for key, p in (("sh", sh), ("ao", ao), ("rf", rf)):
        if p is not None and case.plant and case.plant[key][0] == i:
            _, img, aux = case.plant[key]
            p.upload(5 if key == "sh" else 1, img)
            p.upload(4, aux)


def plant_oracle(case, i, f, osh=None, oao=None, orf=None):
    """the same histories in the oracle passes: the images frame i reads (parity 1 - f.ping_pong), and no first-frame clear"""
    if not case.plant:
        return
    q = 1 - f.ping_pong
    if osh is not None and case.plant["sh"][0] == i:
        osh.prev_image[:], osh.moments[q][:] = case.plant["sh"][1:]
        osh.first = False
    if oao is not None and case.plant["ao"][0] == i:
        oao.color[q][:], oao.length[q][:] = case.plant["ao"][1:]
        oao.first = False
    if orf is not None and case.plant["rf"][0] == i:
        orf.temporal[q][:], orf.moments[q][:] = case.plant["rf"][1:]
        orf.first = False


def plant_hist(case, i, hist, keys):
    """the planted histories as the isolated stages read them (test_gpu_camera's after.hist)"""
    for k in keys:
        if case.plant and case.plant[k][0] == i:
            hist[k] = tuple(np.ascontiguousarray(a) for a in case.plant[k][1:])


# ---------------------------------------------------------------------------------------------- DDGI probe-cell planes
DDGI_PROBE_DISTANCE = 4.0  # test_gpu_ragged.run_gi_refl's grid on the shadows-test scene


def _ddgi_cells(W, H, tame=False):
    """world positions on the probe-cell plane z = start.z + 7 * step (gi_common.cuh: the cell index is (P - start) / step,
    truncated): a depth ladder of float32 steps puts P.z on both sides of the plane; the plane reaches below the grid's first y
    plane and above its last (outside the grid in y)"""
    fs = frames(W, H, 4)
    f = fs[0]
    mn, mx = pyhr.SynthScene(pyhr.SCENE_SHADOWS_TEST).bounds()
    zc = float(np.float32(mn[2]) + np.float32(7 * DDGI_PROBE_DISTANCE)) + (0.5 if tame else 0.0)
    ny = int(np.float32(np.float32(mx[1]) - np.float32(mn[1])) / np.float32(DDGI_PROBE_DISTANCE)) + 2
    ytop = float(mn[1]) + (ny - 1) * DDGI_PROBE_DISTANCE
    k = _pattern(W, H, 2 * LADDER_K + 1) - LADDER_K
    d = ulp_steps(depth_on_plane(f, W, H, zc), k)
    g = plane(f, W, H, depth=d)
    u, v = _tex(W, H)
    P = world_pos(f, u, v, d)
    return list(zip([g] * 4, fs)), {"cell plane z": P[..., 2] - zc, "grid y min": float(mn[1]) - P[..., 1], "grid y max": P[..., 1] - ytop}


BUILDERS = {
    "plane_distance": (_plane_distance, ("K3:sumw", "K3:fallback", "K14:fallback", "K14:invalid")),
    "normal_distance": (_normal_distance, ("K3:invalid", "K3:fallback", "K9:invalid", "K14:invalid")),
    "edges": (_edges, ("K3:out", "K3:trunc", "K9:out", "K14:out")),
    "sumw": (_sumw, ("K3:sumw", "K3:fallback")),
    "mesh_ids": (_mesh_ids, ("K3:invalid", "K9:invalid")),
    "depth": (_depth, ("K3:fallback", "K9:invalid", "K14:fallback")),
    "normals": (_normals, ("K3:invalid",)),
    "roughness": (_roughness, ()),
    "ties": (_ties, ()),
    "planted": (_planted, ()),
    "ddgi_cells": (_ddgi_cells, ()),
}


def build(name, W, H):
    """the case; a builder returns (frames, ladders), (frames, ladders, reached edge offsets) or (frames, ladders, prev, plant)"""
    fn, targets = BUILDERS[name]
    r = fn(W, H)
    prev, plant = (r[2], r[3]) if len(r) == 4 else (None, None)
    ladders = r[1]
    c = Case(f"{name}@{W}x{H}", W, H, r[0], targets, ladders, lambda: fn(W, H, tame=True)[0], (), prev, plant)
    if len(r) == 3:
        EDGE_REACH[c.id] = r[2]
    return c


EDGE_REACH = {}  # case id -> {"x -0.5": reached history_coord_floor - target per border pixel group, ...}


CASE_IDS = [f"{n}@{W}x{H}" for n in BUILDERS for W, H in SIZES]


def case(cid):
    name, size = cid.split("@")
    W, H = (int(v) for v in size.split("x"))
    return build(name, W, H)
