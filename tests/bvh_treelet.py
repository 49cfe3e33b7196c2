"""A float64 numpy restatement of the BVH build's treelet restructuring (k_treelet / treelet_node, csrc/bvh_build.cu) and
the tree-quality yardsticks it is held to (no GPU).

Trees are binary trees over primitive ids.  A Tree holds n - 1 internal nodes (id 0 is the root) and n triangles with the ids
n - 1 + prim, the same numbering as the build; children[i] keeps the child order, and as_leaf[i] marks an internal node of at
most LEAF_MAX triangles that is packed as one leaf.

    tree_from_packed   hr_scene_download_bvh's traversal layout -> Tree
    pack               Tree -> traversal layout, following k_pack_nodes / encode_child / k_pack_tris
    sah                the build's cost model (node step SAH_CI, triangle test SAH_CT, area-weighted) over the root's area
    optimal_sah        the exact minimum of sah over every tree of a few triangles (dynamic program over subsets)
    treelet_rounds     the kernel's rounds on a Tree, with the smallest relative margin of any decision it took
    check_packed       validity walk of a packed tree: every triangle once, boxes nest, depth bound
    canonical          the set of triangle sets of every node (topology equality regardless of child order)
    ordered            the tree as nested tuples in child order (topology and layout equality)

Triangle boxes come from the input soup (tri_boxes), unpadded like k_tri_bounds: the packed boxes carry box_pad and the
triangles' edges v - v0 are rounded, so neither gives the build's costs.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import bvh_quality as Q  # noqa: E402

SAH_CI, SAH_CT = Q.SAH_CI, Q.SAH_CT
LEAF_MAX = 2          # csrc/bvh_build.cu
TREELET_LEAVES = 7    # csrc/bvh_build.cu
MAX_DEPTH = 63        # HR_BVH_MAX_DEPTH, include/hr_api.h
ACCEPT = 1.0 - 1e-5   # a treelet is rewired only when its new cost is below ACCEPT * its old cost


class Tree:
    def __init__(self, children, as_leaf=None):
        self.children = np.array(children, np.int64).reshape(-1, 2)
        self.n = self.children.shape[0] + 1
        self.as_leaf = np.zeros(self.n - 1, bool) if as_leaf is None else np.array(as_leaf, bool)


def tri_boxes(tri):
    """(n, 9) soup -> (n, 6) float64 boxes (lo xyz, hi xyz), exactly the fp32 min / max of the vertices"""
    v = np.asarray(tri, np.float32).reshape(-1, 3, 3)
    return np.concatenate([v.min(1), v.max(1)], 1).astype(np.float64)


def half_area(b):
    d = b[..., 3:6] - b[..., 0:3]
    return d[..., 0] * d[..., 1] + d[..., 1] * d[..., 2] + d[..., 2] * d[..., 0]


def rel(a, b):
    """relative difference of two costs; two exact zeros (areas of boxes without extent, zero in any arithmetic) are no
    near-tie: both sides compare equal on every device and the same side wins"""
    m = max(abs(a), abs(b))
    return abs(a - b) / m if m > 0 else np.inf


# ------------------------------------------------------------------------------------------------ tree <-> traversal layout
def tree_from_packed(nodes, tris):
    """packed tree -> Tree.  A leaf of two triangles becomes an internal node (as_leaf) over its triangles in leaf order,
    which is the depth-first order of the build's tree, so a 0-round build is recovered exactly."""
    _, _, _, _, ch, T = Q.unpack(nodes, tris)
    prim = np.ascontiguousarray(T[:, 0, 3]).view(np.uint32).astype(np.int64)
    n = len(prim)
    if n <= LEAF_MAX:
        raise ValueError("a tree of at most LEAF_MAX triangles is a single leaf")
    children, as_leaf = [], []

    def new_node():
        children.append([0, 0])
        as_leaf.append(False)
        return len(children) - 1

    def child(c):
        if c >= 0:
            return visit(int(c))
        first, cnt = (~c) >> 3, ((~c) & 7) + 1
        if cnt == 1:
            return n - 1 + int(prim[first])
        assert cnt == 2, cnt
        i = new_node()
        children[i] = [n - 1 + int(prim[first]), n - 1 + int(prim[first + 1])]
        as_leaf[i] = True
        return i

    def visit(k):
        i = new_node()
        a = child(int(ch[k, 0]))
        b = child(int(ch[k, 1]))
        children[i] = [a, b]
        return i

    visit(0)
    assert len(children) == n - 1, "every internal node once"
    return Tree(children, as_leaf)


def _dfs_order(tree):
    """internal node ids in pre-order (root first)"""
    out, stack, n = [], [0], tree.n
    while stack:
        i = stack.pop()
        out.append(i)
        for c in tree.children[i][::-1]:
            if c < n - 1:
                stack.append(int(c))
    return out


def node_boxes(tree, boxes):
    """(2n - 1, 6) boxes and (2n - 1,) triangle counts of every node id (triangles at n - 1 + prim)"""
    n = tree.n
    B = np.empty((2 * n - 1, 6))
    S = np.ones(2 * n - 1, np.int64)
    B[n - 1:] = boxes
    for i in reversed(_dfs_order(tree)):
        a, b = tree.children[i]
        B[i, :3] = np.minimum(B[a, :3], B[b, :3])
        B[i, 3:] = np.maximum(B[a, 3:], B[b, 3:])
        S[i] = S[a] + S[b]
    return B, S


def pack(tree, tri, pad):
    """Tree + (n, 9) soup -> (nodes (n - 1, 4, 4), tris (n, 3, 4)) in the traversal layout, as k_pack_nodes writes it for
    the build's node ids: triangles in depth-first order, a child of <= LEAF_MAX triangles marked as_leaf is one leaf."""
    n = tree.n
    tri = np.asarray(tri, np.float32).reshape(-1, 9)
    B, S = node_boxes(tree, tri_boxes(tri))
    first = np.zeros(2 * n - 1, np.int64)
    order = []
    for i in _dfs_order(tree):                                 # pre-order: a node's first slot is known before its children
        a, b = tree.children[i]
        first[a] = first[i]
        first[b] = first[i] + S[a]
        order += [int(c) - (n - 1) for c in (a, b) if c >= n - 1]
    leaf_prim = np.zeros(n, np.int64)
    leaf_prim[first[n - 1:]] = np.arange(n)
    assert sorted(order) == list(range(n))

    def encode(c):
        if c >= n - 1:
            return ~(int(first[c]) << 3)
        if S[c] <= LEAF_MAX and tree.as_leaf[c]:
            return ~((int(first[c]) << 3) | (int(S[c]) - 1))
        return int(c)

    f32 = np.float32
    nodes = np.zeros((n - 1, 4, 4), f32)
    lo = (B[:, :3].astype(f32) - f32(pad)).astype(f32)
    hi = (B[:, 3:].astype(f32) + f32(pad)).astype(f32)
    c0, c1 = tree.children[:, 0], tree.children[:, 1]
    nodes[:, 0] = np.stack([lo[c0, 0], hi[c0, 0], lo[c0, 1], hi[c0, 1]], 1)
    nodes[:, 1] = np.stack([lo[c1, 0], hi[c1, 0], lo[c1, 1], hi[c1, 1]], 1)
    nodes[:, 2] = np.stack([lo[c0, 2], hi[c0, 2], lo[c1, 2], hi[c1, 2]], 1)
    links = np.array([[encode(a), encode(b)] for a, b in tree.children], np.int32)
    nodes[:, 3, :2] = links.view(f32)
    v = tri[leaf_prim].reshape(-1, 3, 3)
    tris = np.zeros((n, 3, 4), f32)
    tris[:, 0, :3] = v[:, 0]
    tris[:, 0, 3] = leaf_prim.astype(np.uint32).view(f32)
    tris[:, 1, :3] = v[:, 1] - v[:, 0]
    tris[:, 2, :3] = v[:, 2] - v[:, 0]
    return nodes, tris


# ------------------------------------------------------------------------------------------------ topology forms and checks
def ordered(tree):
    """nested tuples in child order: a triangle is its primitive id, a packed leaf ("leaf", a, b), an inner node (c0, c1)"""
    n = tree.n

    def f(i):
        if i >= n - 1:
            return i - (n - 1)
        a, b = tree.children[i]
        if tree.as_leaf[i] and a >= n - 1 and b >= n - 1:
            return ("leaf", int(a) - (n - 1), int(b) - (n - 1))
        return (f(int(a)), f(int(b)))

    return f(0)


def from_ordered(t):
    """the inverse of ordered: nested tuples over the primitive ids 0..n-1 -> Tree (node ids in pre-order)"""
    prims = []

    def count(t):
        if isinstance(t, (int, np.integer)):
            prims.append(int(t))
        else:
            for c in (t[1:] if t[0] == "leaf" else t):
                count(c)

    count(t)
    n = len(prims)
    assert sorted(prims) == list(range(n))
    children, as_leaf = [], []

    def f(t):
        if isinstance(t, (int, np.integer)):
            return n - 1 + int(t)
        i = len(children)
        children.append([0, 0])
        as_leaf.append(t[0] == "leaf")
        children[i] = [f(c) for c in (t[1:] if t[0] == "leaf" else t)]
        return i

    f(t)
    return Tree(children, as_leaf)


def canonical(tree):
    """frozenset of the triangle sets of every node; a packed leaf's triangles are not nodes of their own"""
    out = set()

    def f(t):
        if isinstance(t, int):
            s = frozenset([t])
        elif t[0] == "leaf":
            s = frozenset(t[1:])
        else:
            s = f(t[0]) | f(t[1])
        out.add(s)
        return s

    f(ordered(tree))
    return frozenset(out)


def check_packed(nodes, tris, max_depth=MAX_DEPTH):
    """Walks a packed tree from node 0: every triangle is in exactly one reachable leaf of <= LEAF_MAX triangles, an internal
    child's box holds both of its children's boxes, a leaf's box holds its triangles' vertices, the tree is at most max_depth
    node levels deep and the triangle array holds every primitive once.  Returns the number of node levels walked."""
    lo0, hi0, lo1, hi1, ch, T = Q.unpack(nodes, tris)
    n = T.shape[0]
    prim = np.ascontiguousarray(T[:, 0, 3]).view(np.uint32)
    assert np.array_equal(np.sort(prim), np.arange(n, dtype=np.uint32)), "every triangle once in the triangle array"
    seen = np.zeros(n, np.int64)
    frontier, depth = np.array([0]), 0
    tv = T[:, 0, :3], T[:, 0, :3] + T[:, 1, :3], T[:, 0, :3] + T[:, 2, :3]
    while frontier.size:
        assert depth <= max_depth, f"deeper than {max_depth}"
        for s, (lo, hi) in enumerate(((lo0, hi0), (lo1, hi1))):
            c = ch[frontier, s]
            blo, bhi = lo[frontier], hi[frontier]
            inner = c >= 0
            ci = c[inner]
            for clo, chi in ((lo0, hi0), (lo1, hi1)):
                assert np.all(blo[inner] <= clo[ci]) and np.all(bhi[inner] >= chi[ci]), "an internal child's box holds its children's"
            leaf = ~c[~inner]
            first, cnt = leaf >> 3, (leaf & 7) + 1
            assert np.all(cnt <= LEAF_MAX)
            for k in range(LEAF_MAX):
                m = k < cnt
                idx = first[m] + k
                np.add.at(seen, idx, 1)
                for v in tv:
                    assert np.all(blo[~inner][m] <= v[idx]) and np.all(bhi[~inner][m] >= v[idx]), "a leaf's box holds its triangles"
        frontier = np.concatenate([ch[frontier, 0][ch[frontier, 0] >= 0], ch[frontier, 1][ch[frontier, 1] >= 0]])
        depth += 1
    assert np.all(seen == 1), "every triangle in exactly one reachable leaf"
    return depth


def height(tree):
    """edges from the root to the deepest triangle (hr_scene_info.depth)"""
    n, h = tree.n, np.zeros(2 * tree.n - 1, np.int64)
    for i in reversed(_dfs_order(tree)):
        h[i] = 1 + max(h[tree.children[i, 0]], h[tree.children[i, 1]])
    return int(h[0])


# ------------------------------------------------------------------------------------------------ cost
def sah(tree, boxes):
    """the build's cost of the packed tree over the root's area: an internal node SAH_CI x its area, a leaf SAH_CT x its
    triangle count x its area (a node marked as_leaf is a leaf)"""
    B, S = node_boxes(tree, boxes)
    n = tree.n
    A = half_area(B)
    cost = np.empty(2 * n - 1)
    cost[n - 1:] = SAH_CT * A[n - 1:]
    for i in reversed(_dfs_order(tree)):
        a, b = tree.children[i]
        cost[i] = SAH_CT * S[i] * A[i] if tree.as_leaf[i] and S[i] <= LEAF_MAX else SAH_CI * A[i] + cost[a] + cost[b]
    assert A[0] > 0, "sah is relative to the root's area"
    return float(cost[0] / A[0])


_TABLES = {}


def _tables(L):
    """per subset size k >= 2: the subsets of L slots (M) and, row by row, their splits p (holding the lowest slot, p != m)
    in the kernel's enumeration order, so exact ties resolve alike"""
    if L not in _TABLES:
        out = []
        for k in range(2, L + 1):
            M = [m for m in range(1, 1 << L) if bin(m).count("1") == k]
            P = []
            for m in M:
                low = m & -m
                rest = m ^ low
                q, row = rest, []
                while True:
                    q = (q - 1) & rest
                    row.append(low | q)
                    if q == 0:
                        break
                P.append(row)
            out.append((k, np.array(M, np.int64), np.array(P, np.int64)))
        _TABLES[L] = out
    return _TABLES[L]


def subset_dp(box, size, cost):
    """The kernel's dynamic program over the subsets of L slots (box (L, 6), triangle count and subtree cost per slot).
    Returns per subset mask: area, best cost, best split (part), leaf choice, and the second-best split's cost."""
    L = len(size)
    F = 1 << L
    lo = np.full((F, 3), np.inf)
    hi = np.full((F, 3), -np.inf)
    sz = np.zeros(F, np.int64)
    for b in range(L):  # masks in [2^b, 2^(b+1)) are the masks below 2^b plus slot b
        s = slice(1 << b, 2 << b)
        lo[s] = np.minimum(lo[: 1 << b], box[b, :3])
        hi[s] = np.maximum(hi[: 1 << b], box[b, 3:])
        sz[s] = sz[: 1 << b] + size[b]
    area = np.zeros(F)
    area[1:] = half_area(np.concatenate([lo[1:], hi[1:]], 1))
    pc = np.array([bin(m).count("1") for m in range(F)])
    best_cost = np.where((pc >= 2) & (sz <= LEAF_MAX), SAH_CT * sz * area, np.inf)
    for b in range(L):
        best_cost[1 << b] = cost[b]
    part = np.zeros(F, np.int64)
    leaf = np.zeros(F, bool)
    inner = np.full(F, np.inf)
    second = np.full(F, np.inf)
    split = np.full(F, np.inf)
    for k, M, P in _tables(L):
        c = best_cost[P] + best_cost[M[:, None] ^ P]
        bi = np.argmin(c, 1)
        best = c[np.arange(len(M)), bi]
        if P.shape[1] > 1:
            second[M] = np.partition(c, 1, 1)[:, 1]
        split[M] = best
        part[M] = P[np.arange(len(M)), bi]
        inner[M] = SAH_CI * area[M] + best
        leafc = best_cost[M]
        leaf[M] = leafc <= inner[M]
        best_cost[M] = np.minimum(leafc, inner[M])
    return dict(area=area, cost=best_cost, part=part, leaf=leaf, inner=inner, split=split, second=second, size=sz)


def optimal_sah(boxes):
    """the least sah over every full binary tree of the triangles (any subset of <= LEAF_MAX triangles may be one leaf)"""
    boxes = np.asarray(boxes, np.float64)
    n = len(boxes)
    assert 2 <= n <= 14
    d = subset_dp(boxes, np.ones(n, np.int64), SAH_CT * half_area(boxes))
    full = (1 << n) - 1
    return float(d["cost"][full] / d["area"][full])


# ------------------------------------------------------------------------------------------------ treelet restructuring
def _post_order(tree):
    return _dfs_order(tree)[::-1]


def _depths(tree):
    d = np.zeros(tree.n - 1, np.int64)
    for i in _dfs_order(tree):
        for c in tree.children[i]:
            if c < tree.n - 1:
                d[c] = d[i] + 1
    return d


def _round(tree, boxes, max_depth, guard):
    """one k_treelet round: every internal node, children before parents, as the root of a treelet over its final subtree"""
    n = tree.n
    ch = tree.children.copy()
    as_leaf = np.zeros(n - 1, bool)
    B, S = node_boxes(tree, boxes)
    A = half_area(B)
    cost = np.empty(2 * n - 1)
    cost[n - 1:] = SAH_CT * A[n - 1:]
    hgt = np.zeros(2 * n - 1, np.int64)
    depth = _depths(tree)   # at the start of the round, as k_node_depth
    margin = np.inf
    for root in _post_order(tree):
        # grow: open the treelet leaf of largest area (internal nodes only, the first slot wins a tie)
        leaf = [int(ch[root, 0]), int(ch[root, 1])]
        inner = [root]
        while len(leaf) < TREELET_LEAVES:
            cand = [(A[x], s) for s, x in enumerate(leaf) if x < n - 1]
            if not cand:
                break
            best = max(a for a, _ in cand)
            open_ = next(s for a, s in cand if a == best)
            if len(cand) > 1:
                margin = min(margin, rel(best, max(a for a, s in cand if s != open_)))
            x = leaf[open_]
            inner.append(x)
            leaf[open_] = int(ch[x, 0])
            leaf.append(int(ch[x, 1]))
        L = len(leaf)
        d = subset_dp(B[leaf], S[leaf], cost[leaf])
        full = (1 << L) - 1
        c0, c1 = ch[root]
        old_inner = SAH_CI * d["area"][full] + cost[c0] + cost[c1]
        old_leaf = SAH_CT * S[root] * d["area"][full] if S[root] <= LEAF_MAX else np.inf
        old_c = min(old_inner, old_leaf)
        keep = True
        if L > 2 and rel(d["cost"][full], old_c) > 1e-9:
            # (when the program finds the input's own cost again, both sides are one sum in two orders, which fp32 rounds
            # far less than ACCEPT's 1e-5: the treelet is kept on any device)
            margin = min(margin, rel(d["cost"][full], old_c * ACCEPT))
        if L > 2 and d["cost"][full] < old_c * ACCEPT:
            om, ref = [full], []
            i = 0
            while i < len(om):
                r = []
                for side in (d["part"][om[i]], om[i] ^ d["part"][om[i]]):
                    if bin(side).count("1") == 1:
                        r.append(~(int(side).bit_length() - 1))
                    else:
                        r.append(len(om))
                        om.append(int(side))
                ref.append(r)
                i += 1
            nh = [0] * len(om)
            for i in range(len(om) - 1, -1, -1):
                nh[i] = 1 + max(nh[r] if r >= 0 else hgt[leaf[~r]] for r in ref[i])
            if not guard or nh[0] <= max_depth - depth[root]:
                keep = False
                for i in reversed(range(len(om))):  # children before parents
                    m, nid = om[i], inner[i]
                    ids = [inner[r] if r >= 0 else leaf[~r] for r in ref[i]]
                    ch[nid] = ids
                    B[nid, :3] = np.minimum(B[ids[0], :3], B[ids[1], :3])
                    B[nid, 3:] = np.maximum(B[ids[0], 3:], B[ids[1], 3:])
                    A[nid] = half_area(B[nid])
                    S[nid] = S[ids[0]] + S[ids[1]]
                    cost[nid] = d["cost"][m]
                    hgt[nid] = nh[i]
                    as_leaf[nid] = d["leaf"][m]
                    if np.isfinite(d["second"][m]):
                        margin = min(margin, rel(d["split"][m], d["second"][m]))
                    if S[nid] <= LEAF_MAX:
                        margin = min(margin, rel(SAH_CT * S[nid] * d["area"][m], d["inner"][m]))
        if keep:
            cost[root] = old_c
            hgt[root] = 1 + max(hgt[c0], hgt[c1])
            as_leaf[root] = old_leaf <= old_inner
            if S[root] <= LEAF_MAX:
                margin = min(margin, rel(old_leaf, old_inner))
    return Tree(ch, as_leaf), margin


def treelet_rounds(tree, boxes, rounds, max_depth=MAX_DEPTH, guard=True):
    """The build's treelet restructuring on tree for `rounds` rounds -> (tree, margin).  margin is the smallest relative
    difference met in any decision taken: the growth choice (largest area vs the next), the acceptance (new cost vs
    ACCEPT x old), and for every node of the result the best split vs the second best and leaf vs inner.  The device
    computes in fp32 with contraction, so below a small margin its choice may differ and only the costs are comparable.
    guard=False drops the depth guard (a treelet whose new height would take a triangle below max_depth keeps its input)."""
    boxes = np.asarray(boxes, np.float64)
    margin = np.inf
    for _ in range(rounds):
        tree, m = _round(tree, boxes, max_depth, guard)
        margin = min(margin, m)
    return tree, margin
