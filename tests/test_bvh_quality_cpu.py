"""CPU tests of tools/bvh_quality.py on hand-built trees in the packed traversal layout: the walker's hits equal brute force,
its node-step and triangle-test counts match a hand count, and the SAH cost matches the cost model by hand."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import bvh_quality as Q  # noqa: E402


def pack(tri_verts, leaf_max=2, pad=0.0):
    """median-split binary tree over the triangles, packed like k_pack_nodes (boxes padded by `pad`, leaves of <= leaf_max)"""
    tv = np.asarray(tri_verts, np.float32).reshape(-1, 3, 3)
    nodes, order = [], []

    def box(ids):
        v = tv[ids].reshape(-1, 3)
        return v.min(0) - pad, v.max(0) + pad

    def child(ids):
        if len(ids) <= leaf_max:
            first = len(order)
            order.extend(ids)
            return ~((first << 3) | (len(ids) - 1))
        return build(ids)

    def build(ids):
        i = len(nodes)
        nodes.append(None)
        c = tv[ids].mean(1)
        ax = int(np.argmax(c.max(0) - c.min(0)))
        ids = [ids[k] for k in np.argsort(c[:, ax], kind="stable")]
        halves = ids[: len(ids) // 2], ids[len(ids) // 2:]
        links = [child(h) for h in halves]
        (l0, h0), (l1, h1) = box(halves[0]), box(halves[1])
        nodes[i] = np.array([[l0[0], h0[0], l0[1], h0[1]], [l1[0], h1[0], l1[1], h1[1]], [l0[2], h0[2], l1[2], h1[2]],
                             np.array([links[0], links[1], 0, 0], np.int32).view(np.float32)], np.float32)
        return i

    build(list(range(tv.shape[0])))
    tris = np.zeros((len(order), 3, 4), np.float32)
    for k, p in enumerate(order):
        tris[k, 0, :3], tris[k, 1, :3], tris[k, 2, :3] = tv[p, 0], tv[p, 1] - tv[p, 0], tv[p, 2] - tv[p, 0]
        tris[k, 0, 3] = np.array([p], np.uint32).view(np.float32)[0]
    return np.stack(nodes), tris


def quad_row():
    """three unit triangles in the plane z = 0 at x = 0, 2, 4 (tree: root -> (leaf {0}, node -> (leaf {1}, leaf {2})))"""
    return np.array([[x, 0, 0, x + 1, 0, 0, x, 1, 0] for x in (0.0, 2.0, 4.0)], np.float32)


def test_walker_counts_by_hand():
    nodes, tris = pack(quad_row(), leaf_max=1, pad=0.01)
    assert nodes.shape[0] == 2
    rays = np.array([[0.25, 0.25, 1.0, 0.0, 0.0, 0.0, -1.0, 100.0],   # hits triangle 0 only: root step, one test
                     [4.25, 0.25, 1.0, 0.0, 0.0, 0.0, -1.0, 100.0],   # triangle 2: root step, inner step, one test
                     # in the row's plane through all three padded boxes: root step, leaf {0}, pop the inner node (step),
                     # leaf {1} and the pushed leaf {2}: every triangle test fails (the ray is parallel to them)
                     [-5.0, 0.25, 0.0, 0.0, 1.0, 0.0, 0.0, 100.0],
                     [0.5, 5.0, 1.0, 0.0, 0.0, 0.0, -1.0, 100.0]],    # misses the root's children: one step
                    np.float32)
    hit, t, prim, steps, tests = Q.walk(nodes, tris, rays, True)
    assert hit.tolist() == [True, True, False, False]
    assert prim[:2].tolist() == [0, 2] and t[:2].tolist() == [1.0, 1.0]
    assert steps.tolist() == [1, 2, 2, 1]
    assert tests.tolist() == [1, 1, 3, 0]
    ahit, _, _, asteps, atests = Q.walk(nodes, tris, rays, False)
    assert ahit.tolist() == [True, True, False, False]
    assert asteps.tolist() == [1, 2, 2, 1] and atests.tolist() == [1, 1, 3, 0]


def test_closest_hit_shrinks_the_walk():
    """four stacked triangles under one ray (z = 0, -1, -9, -10; tree root -> (node {-10, -9}, node {-1, 0})): the near node is
    walked first (step 2), its near leaf hits at t = 1, the pushed leaf {-1} is tested without a box test like the kernel's
    pop, and the pushed node {-10, -9} is stepped (3) but both its boxes now lie beyond the closest hit"""
    tri = np.array([[0, 0, z, 1, 0, z, 0, 1, z] for z in (0.0, -1.0, -9.0, -10.0)], np.float32)
    nodes, tris = pack(tri, leaf_max=1)
    ray = np.array([[0.25, 0.25, 1.0, 0.0, 0.0, 0.0, -1.0, 100.0]], np.float32)
    hit, t, prim, steps, tests = Q.walk(nodes, tris, ray, True)
    assert prim.tolist() == [0] and t.tolist() == [1.0]
    assert steps.tolist() == [3] and tests.tolist() == [2]
    _, _, _, asteps, atests = Q.walk(nodes, tris, ray, False)
    assert asteps.tolist() == [2] and atests.tolist() == [1]


def test_walker_matches_brute_force():
    rng = np.random.default_rng(5)
    n = 300
    c = rng.uniform(-10, 10, (n, 1, 3))
    tri = (c + rng.normal(0, 0.8, (n, 3, 3))).astype(np.float32).reshape(n, 9)
    nodes, tris = pack(tri)
    m = 2000
    o = rng.uniform(-14, 14, (m, 3))
    tgt = tri.reshape(n, 3, 3)[rng.integers(0, n, m)].mean(1) + rng.normal(0, 0.3, (m, 3))
    d = tgt - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays = np.zeros((m, 8), np.float32)
    rays[:, 0:3], rays[:, 4:7], rays[:, 7] = o, d, rng.uniform(5, 40, m)
    bt, bp = Q.brute_closest(tri, rays)
    hit, t, prim, steps, tests = Q.walk(nodes, tris, rays, True)
    assert np.array_equal(prim, bp) and np.array_equal(t, bt)
    assert hit.sum() > m // 4
    ahit, _, _, asteps, atests = Q.walk(nodes, tris, rays, False)
    assert np.array_equal(ahit, bp != 0xFFFFFFFF)
    assert np.all(asteps <= steps) and np.all(atests <= tests)


def test_sah_cost_by_hand():
    nodes, tris = pack(quad_row(), leaf_max=1)
    # root box [0,5]x[0,1]x[0,0]: half area 5; leaf {0}: 1; inner node [2,5]x[0,1]: 3, its leaves {1}, {2}: 1 each
    want = (Q.SAH_CI * 5 + Q.SAH_CT * 1 + Q.SAH_CI * 3 + Q.SAH_CT * 1 + Q.SAH_CT * 1) / 5
    assert abs(Q.sah_cost(nodes, tris) - want) < 1e-9
    two = pack(quad_row()[:2])
    # n <= LEAF_MAX triangles in one node: both children are single-triangle leaves here (median split of two)
    assert abs(Q.sah_cost(*two) - (Q.SAH_CI * 3 + 2 * Q.SAH_CT) / 3) < 1e-9
