"""The PLOC build's treelet restructuring (k_treelet / treelet_node, csrc/bvh_build.cu) against the float64 yardsticks of
bvh_treelet.py: the exact SAH optimum of small soups, the restatement of the rounds on the device's own plain PLOC tree,
the depth guard, every adversarial scene at several round counts, and determinism of hr_scene_build / hr_scene_rebuild.

The round count (hr_internal_bvh_treelet_rounds) and the topology (hr_debug_set key 3) are process-wide; every test sets
them for its builds only and restores them on the way out.
"""
import ctypes as C

import numpy as np
import pytest

import bvh_cases as B
import bvh_treelet as T
import pyhr
from bvh_gpu import bad_entries, build, chain_rays, check_scene, gpu_trace, switches

pytestmark = pytest.mark.gpu

ARCADE_TRIS = 262144      # bench.py configs 2-4
NEAR_TIE = 1e-4           # below this relative decision margin the device's fp32 choice may differ from the float64 one
SAH_SLACK = 2e-5          # the device's rewiring needs a 1e-5 gain, and it adds its costs in fp32


class rounds:
    """hr_internal_bvh_treelet_rounds(r) for the builds inside, the previous count restored on exit"""

    def __init__(self, lib, r):
        self.hook, self.r = lib.hr_internal_bvh_treelet_rounds, r
        self.hook.argtypes = [C.c_int]

    def __enter__(self):
        self.prev = self.hook(self.r)
        return self

    def __exit__(self, *exc):
        self.hook(self.prev)
        return False


@pytest.fixture(scope="module")
def ctx():
    c = pyhr.Context(0)
    c.set_bluenoise(*pyhr.blue_noise())
    yield c
    c.close()


@pytest.fixture(scope="module")
def default_rounds(ctx):
    with rounds(ctx.lib, -1) as r:
        return r.prev


def device_tree(ctx, tri, r, topology=1):
    """(nodes, tris, depth) of the tree built for the soup with r restructuring rounds"""
    with switches(ctx.lib, k3=topology), rounds(ctx.lib, r):
        rc, h, _ = build(ctx, tri)
    ctx.check(rc, "hr_scene_build")
    try:
        nodes, tris = ctx.download_bvh(h)
        return nodes, tris, int(ctx.scene_info(h).depth)
    finally:
        ctx.lib.hr_scene_destroy(h)


def device_sah(ctx, tri, r):
    nodes, tris, _ = device_tree(ctx, tri, r)
    T.check_packed(nodes, tris)
    tree = T.tree_from_packed(nodes, tris)
    return T.sah(tree, T.tri_boxes(tri)), tree


# ---------------------------------------------------------------------------------------------- a. the global optimum
def small_soups(n):
    out = {f"random{s}": B.random_soup(n, 100 * n + s) for s in range(30)}
    dup = B.random_soup(2, n)
    out["duplicates"] = dup[np.arange(n) % 2]
    out["same_centroid"] = B.same_centroid(n)
    out["points_and_segments"] = B.points_and_segments(n, n)
    out["chain"] = B.chain(n)
    out["far_pairs"] = B.far_pairs(n)
    return out


def inner_pairs(t):
    """number of inner nodes over exactly two triangles that are not packed as one leaf"""
    if isinstance(t, int) or t[0] == "leaf":
        return 0
    return int(all(isinstance(c, int) for c in t)) + inner_pairs(t[0]) + inner_pairs(t[1])


@pytest.mark.parametrize("n", [3, 4, 5, 6, 7])
def test_small_soups_reach_the_global_optimum(ctx, default_rounds, n):
    """up to TREELET_LEAVES triangles the root's treelet holds all of them, so the device tree is an optimal one"""
    bad = []
    for name, tri in small_soups(n).items():
        opt = T.optimal_sah(T.tri_boxes(tri))
        for r in sorted({1, default_rounds}):
            got, tree = device_sah(ctx, tri, r)
            if got > opt * (1 + SAH_SLACK):
                bad.append(f"{name} rounds {r}: sah {got:.9g} vs optimum {opt:.9g} ({got / opt - 1:.3g})")
            if name == "far_pairs":
                # the optimum keeps two-triangle subtrees as inner nodes over one-triangle leaves (as_leaf = 0)
                assert inner_pairs(T.ordered(tree)) > 0, (r, T.ordered(tree))
    assert not bad, bad


@pytest.mark.parametrize("n", [8, 10, 12])
def test_small_soups_lie_between_the_optimum_and_plain_ploc(ctx, default_rounds, n):
    for s in range(6):
        tri = B.random_soup(n, 7 * n + s)
        opt = T.optimal_sah(T.tri_boxes(tri))
        plain, _ = device_sah(ctx, tri, 0)
        got, _ = device_sah(ctx, tri, default_rounds)
        assert opt * (1 - 1e-9) <= got <= plain * (1 + 1e-6), (s, opt, got, plain)


# ---------------------------------------------------------------------------------------------- b. the restatement
RESTATED = {
    "random8": lambda: B.random_soup(8, 8),
    "random9": lambda: B.random_soup(9, 9),
    "random33": lambda: B.random_soup(33, 33),
    "random257": lambda: B.random_soup(257, 257),
    "random4096": lambda: B.random_soup(4096, 4096, extent=40.0),
    "clustered": lambda: B.clustered(8, 64, 1),
    "strip": lambda: B.strip(512),
    "points_and_segments": lambda: B.points_and_segments(96, 5),
}
RESTATED_ROUNDS = (1, 2, 3, 5)


@pytest.fixture(scope="module")
def restated(ctx):
    """case -> [(rounds, device sah, reference sah, margin, same ordered topology, device sah of the previous count,
    reference topology, device node bytes)]"""
    out = {}
    for case, make in RESTATED.items():
        tri = make()
        boxes = T.tri_boxes(tri)
        nodes, tris, _ = device_tree(ctx, tri, 0)
        ref = T.tree_from_packed(nodes, tris)
        prev_dev = T.sah(ref, boxes)
        margin, done, rows = np.inf, 0, []
        for r in RESTATED_ROUNDS:
            ref, m = T.treelet_rounds(ref, boxes, r - done)
            done, margin = r, min(margin, m)
            nodes, tris, depth = device_tree(ctx, tri, r)
            T.check_packed(nodes, tris)
            dev = T.tree_from_packed(nodes, tris)
            rows.append((r, T.sah(dev, boxes), T.sah(ref, boxes), margin, T.ordered(dev) == T.ordered(ref), prev_dev,
                         T.ordered(ref), nodes.tobytes()))
            prev_dev = rows[-1][1]
        out[case] = rows
    return out


@pytest.mark.parametrize("case", sorted(RESTATED))
def test_rounds_match_the_restatement(restated, case):
    for r, dev, ref, margin, same, prev, _, _ in restated[case]:
        print(f"{case} rounds {r}: device sah {dev:.9g}, restatement {ref:.9g} ({dev / ref - 1:+.2e}), margin {margin:.2e}, "
              f"same topology {same}")
        assert dev <= prev * (1 + 1e-6), f"rounds {r}: sah {dev} after {prev} one round count lower"
        if margin >= NEAR_TIE:
            assert same, f"rounds {r}: no decision within {NEAR_TIE} of a tie, yet the topology differs (sah {dev} vs {ref})"
        assert dev == pytest.approx(ref, rel=1e-4), f"rounds {r}"


def test_converged_rounds_leave_the_nodes_unchanged(restated):
    """Once the restatement stops changing the tree (rounds 3 and 5 alike, no near-tie), the device's further rounds rewire
    nothing: every treelet keeps its nodes unless the new cost is below ACCEPT x the old one, which fp32 rounding of one
    cost summed in two orders never reaches.  Rewiring to an equally cheap tree would renumber the nodes."""
    converged = 0
    for case, rows in restated.items():
        by_r = {row[0]: row for row in rows}
        if by_r[3][6] == by_r[5][6] and by_r[5][3] >= NEAR_TIE:
            converged += 1
            assert by_r[3][7] == by_r[5][7], f"{case}: the packed nodes changed between rounds 3 and 5"
    assert converged >= 2


def test_most_restated_cases_are_free_of_near_ties(restated):
    """otherwise the topology comparison above would check nothing"""
    rows = [row for v in restated.values() for row in v]
    free = sum(row[3] >= NEAR_TIE for row in rows)
    assert 2 * free >= len(rows), f"{free} of {len(rows)} (case, rounds) pairs free of near-ties"


# ---------------------------------------------------------------------------------------------- c. the depth limit
@pytest.mark.parametrize("r", [1, 2, 3, 4, 5, 6])
def test_chain_at_the_depth_limit_after_restructuring(ctx, r):
    n = B.MAX_DEPTH + 1
    tri = B.chain(n)
    with rounds(ctx.lib, r):
        rc, h, _ = build(ctx, tri)
    ctx.check(rc, "hr_scene_build")
    try:
        assert ctx.scene_info(h).depth <= B.MAX_DEPTH
        ctx.check(ctx.lib.hr_scene_set_current(ctx.h, h), "hr_scene_set_current")
        rays, x = chain_rays(n)
        a, t, p, _ = gpu_trace(ctx, rays)
        assert np.array_equal(p, np.arange(n, dtype=np.uint32)) and np.array_equal(t, x) and np.all(a == 1)
    finally:
        ctx.lib.hr_scene_destroy(h)


@pytest.mark.parametrize("r", [1, 2, 3])
def test_depth_guard_keeps_the_deep_scene_within_the_limit(ctx, r):
    """bvh_cases.deep_chain_cluster: the restatement without the guard takes a triangle below depth 63"""
    tri = B.deep_chain_cluster()
    boxes = T.tri_boxes(tri)
    nodes, tris, depth0 = device_tree(ctx, tri, 0)
    plain = T.tree_from_packed(nodes, tris)
    assert T.ordered(plain) == B.DEEP_CHAIN_CLUSTER_PLOC, "the plain PLOC tree the guard case was found on"
    assert depth0 <= B.MAX_DEPTH
    want, margin = T.treelet_rounds(plain, boxes, r, guard=True)
    assert margin >= NEAR_TIE
    nodes, tris, depth = device_tree(ctx, tri, r)
    T.check_packed(nodes, tris)
    assert depth <= B.MAX_DEPTH
    assert T.ordered(T.tree_from_packed(nodes, tris)) == T.ordered(want)


# ---------------------------------------------------------------------------------------------- d. every adversarial scene
ADVERSARIAL = dict(B.SCENES, far_pairs=lambda: B.far_pairs(7))


@pytest.mark.parametrize("r", [1, 2, 5, 8])
@pytest.mark.parametrize("scene", sorted(ADVERSARIAL))
def test_adversarial_scene_after_restructuring(ctx, scene, r):
    tri = ADVERSARIAL[scene]()
    if len(tri) > T.LEAF_MAX:
        nodes, tris, depth = device_tree(ctx, tri, r)
        T.check_packed(nodes, tris)
    with rounds(ctx.lib, r):
        report, hits = check_scene(ctx, tri, n=1500)
    if scene == "far_pairs":
        # Moeller-Trumbore's error in t grows with the square of the distance over the triangle's size; on these small
        # triangles a hit seen from 5 scene extents and more lies outside the padded box by more than the pad, so an interval
        # that starts or ends exactly at such a hit is not reproduced by the walk on any tree (the plain one included)
        report = {k: v for k, v in report.items() if not k.endswith("+ends")}
    assert hits > 0
    assert not bad_entries(report), f"{scene} / rounds {r}: rays that differ from brute force (any, closest): {bad_entries(report)}"


# ---------------------------------------------------------------------------------------------- e. determinism and rebuilds
def download(ctx, h):
    nodes, tris = ctx.download_bvh(h)
    return nodes.tobytes(), tris.tobytes(), int(ctx.scene_info(h).depth)


def rebuild(ctx, h):
    ctx.check(ctx.lib.hr_scene_rebuild(h, None), "hr_scene_rebuild")
    return download(ctx, h)


def test_builds_and_rebuilds_of_the_arcade_are_identical(ctx, default_rounds):
    sc = pyhr.SynthScene(pyhr.SCENE_ARCADE, ARCADE_TRIS)
    fresh = {}
    handles = []
    try:
        for key, (r, q) in {"ploc": (default_rounds, 1), "plain": (0, 1), "karras": (default_rounds, 0)}.items():
            with rounds(ctx.lib, r), switches(ctx.lib, k3=q):
                h = ctx.build_scene(sc)
                handles.append(h)
                fresh[key] = download(ctx, h)
        with rounds(ctx.lib, default_rounds):
            h2 = ctx.build_scene(sc)
            handles.append(h2)
            assert download(ctx, h2)[:2] == fresh["ploc"][:2], "two builds differ"
            h = handles[0]
            assert rebuild(ctx, h)[:2] == fresh["ploc"][:2], "a rebuild differs from the build"
        with rounds(ctx.lib, 0):
            assert rebuild(ctx, h)[:2] == fresh["plain"][:2], "rebuild with 0 rounds"
        with rounds(ctx.lib, default_rounds):
            assert rebuild(ctx, h)[:2] == fresh["ploc"][:2], "rebuild back at the default rounds"
            with switches(ctx.lib, k3=0):
                assert rebuild(ctx, h)[:2] == fresh["karras"][:2], "rebuild with the radix tree"
            assert rebuild(ctx, h)[:2] == fresh["ploc"][:2], "rebuild back with PLOC"
            ctx.set_profiling(True)
            try:
                assert rebuild(ctx, h)[2] == fresh["ploc"][2], "depth reported by a profiled rebuild"
            finally:
                ctx.set_profiling(False)
        assert fresh["ploc"][0] != fresh["plain"][0]
    finally:
        for h in handles:
            ctx.lib.hr_scene_destroy(h)
