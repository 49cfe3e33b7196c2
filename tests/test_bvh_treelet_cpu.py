"""The float64 treelet restatement and tree-quality yardsticks of bvh_treelet.py, checked on their own (no GPU): the subset
program against every topology, the rounds' monotone cost and small-tree optimality, the depth guard, and the packer."""
import itertools

import numpy as np
import pytest

import bvh_cases as B
import bvh_treelet as T


def random_tree(ids, rng):
    """a random full binary tree over ids (nested tuples, every two-triangle node left as an inner node)"""
    if len(ids) == 1:
        return int(ids[0])
    k = int(rng.integers(1, len(ids)))
    return (random_tree(ids[:k], rng), random_tree(ids[k:], rng))


def all_topologies(ids):
    """every full binary tree over ids, up to child order: (2n - 3)!! of them"""
    if len(ids) == 1:
        yield ids[0]
        return
    first, rest = ids[0], ids[1:]
    for k in range(len(rest)):
        for other in itertools.combinations(rest, k):
            left = (first,) + other
            right = tuple(x for x in rest if x not in other)
            for a in all_topologies(left):
                for b in all_topologies(right):
                    yield (a, b)


def pair_nodes(t):
    """the inner nodes over exactly two triangles, which may each be packed as one leaf"""
    if isinstance(t, int):
        return []
    if isinstance(t[0], int) and isinstance(t[1], int):
        return [t]
    return pair_nodes(t[0]) + pair_nodes(t[1])


def with_leaves(t, leaves):
    if isinstance(t, int):
        return t
    if t in leaves:
        return ("leaf",) + t
    return (with_leaves(t[0], leaves), with_leaves(t[1], leaves))


def brute_force_sah(boxes):
    n = len(boxes)
    best, count = np.inf, 0
    for t in all_topologies(tuple(range(n))):
        count += 1
        pairs = pair_nodes(t)
        for k in range(len(pairs) + 1):
            for leaves in itertools.combinations(pairs, k):
                best = min(best, T.sah(T.from_ordered(with_leaves(t, set(leaves))), boxes))
    return best, count


def soups_for(n, seed):
    rng = np.random.default_rng(seed)
    yield "random", B.random_soup(n, seed)
    yield "far_pairs", B.far_pairs(n)
    yield "points_and_segments", B.points_and_segments(n, seed)
    yield "same_centroid", B.same_centroid(n)
    dup = B.random_soup(2, seed)
    yield "duplicates", dup[rng.integers(0, 2, n)]
    yield "chain", B.chain(n)


@pytest.mark.parametrize("n", [2, 3, 4, 5, 6])
def test_optimal_sah_equals_brute_force_over_every_topology(n):
    counts = set()
    for seed in range(3):
        for name, tri in soups_for(n, seed):
            boxes = T.tri_boxes(tri)
            want, count = brute_force_sah(boxes)
            counts.add(count)
            got = T.optimal_sah(boxes)
            assert got == pytest.approx(want, rel=1e-12), f"{name} seed {seed}: {got} vs {want}"
    assert counts == {[1, 1, 3, 15, 105, 945][n - 1]}


def test_optimal_tree_of_far_pairs_keeps_each_pair_an_inner_node():
    """the cheapest tree over two far-apart pairs costs less than any tree that packs a pair as one leaf"""
    boxes = T.tri_boxes(B.far_pairs(4))
    opt = T.optimal_sah(boxes)
    assert opt == pytest.approx(T.sah(T.from_ordered(((0, 1), (2, 3))), boxes), rel=1e-12)
    assert opt < T.sah(T.from_ordered((("leaf", 0, 1), (2, 3))), boxes) * 0.99


@pytest.mark.parametrize("n", [8, 20, 64, 300])
def test_rounds_never_increase_the_cost(n):
    rng = np.random.default_rng(n)
    for tri in (B.random_soup(n, n), B.clustered(4, n // 4 + 1, n)):
        boxes = T.tri_boxes(tri)
        tree = T.from_ordered(random_tree(rng.permutation(len(tri)), rng))
        prev = T.sah(tree, boxes)
        for _ in range(4):
            tree, _ = T.treelet_rounds(tree, boxes, 1)
            cur = T.sah(tree, boxes)
            assert cur <= prev * (1 + 1e-12), (prev, cur)
            prev = cur


@pytest.mark.parametrize("n", [3, 4, 5, 6, 7])
def test_one_round_reaches_the_optimum_up_to_seven_triangles(n):
    """the root's treelet holds every triangle, so its program is the exact optimum (a rewiring needs a 1e-5 gain)"""
    rng = np.random.default_rng(n)
    for seed in range(6):
        for name, tri in soups_for(n, seed):
            boxes = T.tri_boxes(tri)
            opt = T.optimal_sah(boxes)
            start = T.from_ordered(random_tree(rng.permutation(n), rng))
            got = T.sah(T.treelet_rounds(start, boxes, 1)[0], boxes)
            assert opt * (1 - 1e-12) <= got <= opt * (1 + 1.001e-5), f"{name} seed {seed}: {got} vs optimum {opt}"


def test_leaf_choice_follows_the_cost():
    """far pairs stay inner nodes, touching pairs become one leaf"""
    boxes = T.tri_boxes(B.far_pairs(4))
    tree, _ = T.treelet_rounds(T.from_ordered(((0, 2), (1, 3))), boxes, 1)
    assert T.canonical(tree) == T.canonical(T.from_ordered(((0, 1), (2, 3))))
    tri = np.concatenate([B.grid(1), B.grid(1, (5.0, 0.0, 0.0))])
    tree, _ = T.treelet_rounds(T.from_ordered(((0, 2), (1, 3))), T.tri_boxes(tri), 1)
    assert T.ordered(tree) == (("leaf", 0, 1), ("leaf", 2, 3))


def test_chain_is_left_at_its_height():
    tri = B.chain(B.MAX_DEPTH + 1)
    boxes = T.tri_boxes(tri)
    tree = T.from_ordered(chain_tree(len(tri)))
    assert T.height(tree) == B.MAX_DEPTH
    for r in range(1, 4):
        out, _ = T.treelet_rounds(tree, boxes, r)
        assert T.height(out) <= B.MAX_DEPTH


@pytest.mark.parametrize("r", [1, 2, 3])
def test_depth_guard_binds_in_the_deep_chain_cluster(r):
    tri = B.deep_chain_cluster()
    boxes = T.tri_boxes(tri)
    plain = T.from_ordered(B.DEEP_CHAIN_CLUSTER_PLOC)
    assert T.height(plain) == B.MAX_DEPTH
    free, _ = T.treelet_rounds(plain, boxes, r, guard=False)
    kept, margin = T.treelet_rounds(plain, boxes, r, guard=True)
    assert T.height(free) > B.MAX_DEPTH, "without the guard the cheapest treelets go below the limit"
    assert T.height(kept) <= B.MAX_DEPTH
    assert T.sah(kept, boxes) <= T.sah(plain, boxes) and T.ordered(kept) != T.ordered(plain), "the other treelets still restructure"
    assert margin >= 1e-4, "no near-tie: the device must take the same decisions (tests/test_gpu_bvh_treelet.py)"


def chain_tree(n):
    """PLOC's tree of bvh_cases.chain(n): one merge per level, the lowest pair packed as a leaf"""
    t = ("leaf", 0, 1)
    for k in range(2, n):
        t = (t, k)
    return t


@pytest.mark.parametrize("n", [3, 5, 17, 100])
def test_packer_round_trips_through_tree_from_packed(n):
    rng = np.random.default_rng(n)
    tri = B.random_soup(n, n)
    for _ in range(5):
        tree = T.from_ordered(random_tree(rng.permutation(n), rng))
        S = T.node_boxes(tree, T.tri_boxes(tri))[1]
        tree.as_leaf = (S[: n - 1] <= T.LEAF_MAX) & (rng.random(n - 1) < 0.5)
        nodes, tris = T.pack(tree, tri, 1e-4)
        T.check_packed(nodes, tris)
        back = T.tree_from_packed(nodes, tris)
        assert T.ordered(back) == T.ordered(tree)
        assert T.canonical(back) == T.canonical(tree)
        assert T.sah(back, T.tri_boxes(tri)) == pytest.approx(T.sah(tree, T.tri_boxes(tri)), rel=1e-12)

