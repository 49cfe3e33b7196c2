"""The PLOC tree after treelet restructuring, built on the device for the bench's arcade: a lower SAH cost than plain PLOC
(the same build with 0 restructuring rounds, set through the library's test hook), and a valid tree in the traversal layout."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import pyhr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import bvh_quality as Q  # noqa: E402

pytestmark = pytest.mark.gpu

ARCADE_TRIS = 262144  # bench.py configs 2-4 (the generator rounds the count up to whole meshes)


@pytest.fixture(scope="module")
def trees():
    ctx = pyhr.Context(0)
    hook = ctx.lib.hr_internal_bvh_treelet_rounds
    hook.argtypes = [C.c_int]
    default = hook(-1)
    sc = pyhr.SynthScene(pyhr.SCENE_ARCADE, ARCADE_TRIS)
    out = {}
    try:
        for rounds in (0, default):
            hook(rounds)
            h = ctx.build_scene(sc)
            out[rounds] = (ctx.download_bvh(h), ctx.scene_info(h))
            ctx.lib.hr_scene_destroy(h)
    finally:
        hook(default)
        ctx.close()
    return default, out


def test_restructured_tree_has_lower_sah_than_plain_ploc(trees):
    default, out = trees
    assert default > 0
    plain, opt = Q.sah_cost(*out[0][0]), Q.sah_cost(*out[default][0])
    assert opt < plain * 0.99, f"SAH cost {opt:.1f} after {default} restructuring rounds vs {plain:.1f} for plain PLOC"


@pytest.mark.parametrize("which", ["plain", "restructured"])
def test_tree_is_valid(trees, which):
    default, out = trees
    (nodes, tris), info = out[0 if which == "plain" else default]
    n = tris.shape[0]
    assert n == info.n_triangles >= ARCADE_TRIS and info.depth <= 63  # HR_BVH_MAX_DEPTH
    lo0, hi0, lo1, hi1, ch, _ = Q.unpack(nodes, tris)
    prim = np.ascontiguousarray(tris[:, 0, 3]).view(np.uint32)
    assert np.array_equal(np.sort(prim), np.arange(n, dtype=np.uint32)), "every triangle once in the triangle array"
    seen = np.zeros(n, np.int64)
    frontier, depth = np.array([0]), 0
    tv = tris[:, 0, :3], tris[:, 0, :3] + tris[:, 1, :3], tris[:, 0, :3] + tris[:, 2, :3]
    while frontier.size:
        assert depth <= 63
        for s, (lo, hi) in enumerate(((lo0, hi0), (lo1, hi1))):
            c = ch[frontier, s]
            blo, bhi = lo[frontier], hi[frontier]
            inner = c >= 0
            ci = c[inner]
            # an internal child's box holds both of its children's boxes
            for clo, chi in ((lo0, hi0), (lo1, hi1)):
                assert np.all(blo[inner] <= clo[ci]) and np.all(bhi[inner] >= chi[ci])
            leaf = ~c[~inner]
            first, cnt = leaf >> 3, (leaf & 7) + 1
            assert np.all(cnt <= 2)
            for k in range(2):
                m = k < cnt
                idx = first[m] + k
                np.add.at(seen, idx, 1)
                for v in tv:  # a leaf's box holds its triangles' vertices
                    assert np.all(blo[~inner][m] <= v[idx]) and np.all(bhi[~inner][m] >= v[idx])
        frontier = np.concatenate([ch[frontier, 0][ch[frontier, 0] >= 0], ch[frontier, 1][ch[frontier, 1] >= 0]])
        depth += 1
    assert np.all(seen == 1), "every triangle in exactly one reachable leaf"
