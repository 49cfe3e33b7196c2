"""The PLOC tree after treelet restructuring, built on the device for the bench's arcade: a lower SAH cost than plain PLOC
(the same build with 0 restructuring rounds, set through the library's test hook), and a valid tree in the traversal layout."""
import ctypes as C
import os
import sys

import pytest

import pyhr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import bvh_quality as Q  # noqa: E402
import bvh_treelet as T  # noqa: E402

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
    assert tris.shape[0] == info.n_triangles >= ARCADE_TRIS and info.depth <= 63  # HR_BVH_MAX_DEPTH
    T.check_packed(nodes, tris)
