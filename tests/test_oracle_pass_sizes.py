"""Every oracle pass sizes its images like the C ABI: hr_*_create halves the frame once per RayTraceScale level and clamps each
dimension to 1 (hr_api.cu pass_common_create), which is also how the G-buffer mip chain is built.  A plain shift (W0 >> scale)
agrees with that rule until a dimension reaches 1 and then gives 0, so the sizes below include 1-pixel frames."""
import numpy as np
import pytest

import oracle as O
import pyhr


def abi_pass_size(W0, H0, scale):
    """restated from pass_common_create: w = w / 2 > 0 ? w / 2 : 1 per level"""
    w, h = W0, H0
    for _ in range(scale):
        w = w // 2 if w // 2 > 0 else 1
        h = h // 2 if h // 2 > 0 else 1
    return w, h


def _ddgi_params():
    P = pyhr.hr_ddgi_params()
    P.rays_per_probe, P.probe_distance, P.irradiance_oct_size, P.depth_oct_size = 8, 4.0, 6, 14
    return P


@pytest.mark.parametrize("W0,H0", [(1, 1), (7, 3), (251, 141)])
@pytest.mark.parametrize("scale", [0, 1, 2])
def test_oracle_pass_size_matches_the_abi(W0, H0, scale):
    W, H = abi_pass_size(W0, H0, scale)
    assert W >= 1 and H >= 1
    assert O.pass_size(W0, H0, scale) == (W, H)
    sh, ao = O.ShadowsOracle(W0, H0, scale), O.AOOracle(W0, H0, scale)
    dd = O.DDGIOracle(W0, H0, scale, _ddgi_params(), np.zeros(3, np.float32), np.full(3, 8.0, np.float32))
    rf = O.ReflectionsOracle(W0, H0, scale, None)
    for o in (sh, ao, dd, rf):
        assert (o.W, o.H) == (W, H), type(o).__name__
    # the images each oracle writes have the pass size (mask: 8x4 pixels per word, tile flags: 8x8 tiles)
    assert sh.temporal.shape[:2] == ao.color[0].shape == rf.rt.shape[:2] == dd.sample.shape[:2] == (H, W)
    assert sh.mask.shape == ao.mask.shape == ((H + 3) // 4, (W + 7) // 8)
    assert sh.tile_flags.shape == ao.tile_flags.shape == rf.tile_flags.shape == ((H + 7) // 8, (W + 7) // 8)
    for o in (sh, ao, rf):
        assert (o.upsample is None) == (scale == 0)
        if scale:
            assert o.upsample.shape[:2] == (H0, W0)
    # ... and the G-buffer mip the pass reads is that size too
    assert O.zero_gbuf_mips(W0, H0).size(scale) == (W, H)
