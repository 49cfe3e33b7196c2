"""CPU checks of the host restatements in measurement_hooks.py: the checksum formula of hr_api.h (known splitmix64 values, exact
uint64 arithmetic, additivity over any row split, sensitivity to a bit flip, a texel swap and +0 / -0), the tile counts and the
stage-list helpers.  No GPU."""
import numpy as np
import pytest

import measurement_hooks as MH

# splitmix64 from state 0 (Vigna's reference generator): its n-th output is the finaliser of n * 0x9E3779B97F4A7C15
SPLITMIX64_SEED0 = [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F, 0xF88BB8A8724C81EC]


def test_mix64_is_the_splitmix64_finaliser():
    for n, want in enumerate(SPLITMIX64_SEED0, 1):
        z = (n * MH.GOLDEN) & MH.M64
        assert MH.mix64_int(z) == want
        assert int(MH.mix64(np.array([z], np.uint64))[0]) == want
    assert MH.mix64_int(0) == 0
    rng = np.random.default_rng(5)
    z = rng.integers(0, 2**63, size=2000, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=2000, dtype=np.uint64)
    assert [int(v) for v in MH.mix64(z)] == [MH.mix64_int(int(v)) for v in z]


# one image per format a pass exposes: (dtype, channels) of R32_UINT, R8_UINT, R16F, RG16F, RGBA16F, RGBA8
FORMATS = {"r32u": (np.uint32, 1), "r8u": (np.uint8, 1), "r16f": (np.uint16, 1), "rg16f": (np.uint16, 2), "rgba16f": (np.uint16, 4),
           "rgba8": (np.uint8, 4)}
SIZES = [(1, 1), (1, 5), (3, 7), (4, 251), (5, 250), (6, 1)]


def image(rng, fmt, H, W):
    dt, ch = FORMATS[fmt]
    shape = (H, W) if ch == 1 else (H, W, ch)
    return rng.integers(0, np.iinfo(dt).max, size=shape, endpoint=True, dtype=dt)


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_checksum_equals_texel_by_texel_sum(fmt):
    rng = np.random.default_rng(11)
    for H, W in SIZES:
        a = image(rng, fmt, H, W)
        assert MH.checksum(a) == MH.checksum_ref(a)
        for y in range(H):
            assert MH.checksum(a, y, y + 1) == MH.checksum_ref(a, y, y + 1)


def test_texel_value_is_little_endian():
    a = np.array([[[0x0102, 0x0304, 0x0506, 0x0708]]], np.uint16)  # one RGBA16F texel
    assert int(MH.texel_values(a)[0, 0]) == 0x0708050603040102
    b = np.array([[[1, 2, 3, 4]]], np.uint8)  # one RGBA8 texel
    assert int(MH.texel_values(b)[0, 0]) == 0x04030201


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_checksum_adds_up_over_any_row_split(fmt):
    """every single row, every two-way split and random k-way splits (empty ranges included) sum to the whole mod 2^64; the
    odd-width R16F and one-byte-wide R8 images are the shapes a word-wise hash could not split"""
    rng = np.random.default_rng(12)
    for H, W in SIZES + [(17, 1), (9, 251), (8, 3)]:
        a = image(rng, fmt, H, W)
        whole = MH.checksum(a)
        assert MH.split_sum(a, list(range(H + 1))) == whole
        for c in range(H + 1):
            assert MH.split_sum(a, [0, c, H]) == whole
        for k in (2, 3, 5, 9):
            assert MH.split_sum(a, MH.random_cuts(rng, H, k)) == whole
        assert all(MH.checksum(a, c, c) == 0 for c in range(1, H + 1))  # empty ranges (row1 = 0 is the whole image)


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_checksum_sees_one_bit_flip(fmt):
    rng = np.random.default_rng(13)
    a = image(rng, fmt, 5, 13)
    whole = MH.checksum(a)
    flat = a.view(np.uint8).reshape(-1)
    for byte in range(flat.size):
        for bit in range(8):
            b = a.copy()
            b.view(np.uint8).reshape(-1)[byte] ^= np.uint8(1 << bit)
            assert MH.checksum(b) != whole, f"flipping bit {bit} of byte {byte} does not change the checksum"


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_checksum_sees_two_texels_swapped(fmt):
    rng = np.random.default_rng(14)
    a = image(rng, fmt, 4, 9)
    whole = MH.checksum(a)
    v = MH.texel_values(a).reshape(-1)
    for i, j in [(0, 1), (0, 35), (8, 9), (9, 18), (17, 30)]:
        if v[i] == v[j]:
            continue
        b = a.reshape(a.shape[0] * a.shape[1], -1).copy()
        b[[i, j]] = b[[j, i]]
        assert MH.checksum(b.reshape(a.shape)) != whole, f"swapping texels {i} and {j} does not change the checksum"


def test_checksum_sees_signed_zero():
    """+0.0 and -0.0 compare equal as floats; the checksum hashes bits, so it tells them apart in every half-float format"""
    for shape in [(3, 5), (3, 5, 2), (3, 5, 4)]:
        a = np.zeros(shape, np.float16)
        b = a.copy()
        b.reshape(-1)[7] = -0.0
        assert np.array_equal(a, b)  # equal as numbers
        assert MH.checksum(a.view(np.uint16)) != MH.checksum(b.view(np.uint16))


def test_checksum_row_range_semantics():
    a = image(np.random.default_rng(15), "r16f", 6, 7)
    assert MH.checksum(a, 0, 0) == MH.checksum(a) == MH.checksum(a, 3, -1)  # row1 <= 0: the whole image
    assert MH.checksum(a, 2, 5) == (MH.checksum(a, 2, 3) + MH.checksum(a, 3, 5)) & MH.M64


def test_tile_counts():
    W, H = 250, 141
    flags = np.zeros(((H + 7) // 8, (W + 7) // 8), np.uint8)
    flags[0, :3] = 1
    flags[5, 7] = 1
    flags[-1, -1] = 1
    assert MH.tile_counts(flags, W, H) == (18 * 32, 5, W * H)
    assert MH.tile_counts(flags, W, H, 40, 64) == (3 * 32, 1, 24 * W)
    assert MH.tile_counts(flags, W, H, 136, 141) == (32, 1, 5 * W)
    assert MH.tile_counts(flags, W, H, 0, 0) == (0, 0, 0)


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("H", [141, 144, 35, 3, 1])
def test_own_rows_partition_the_image(H, world):
    """the ranks' own rows cover the pass rows, and the upsampled rows of a half / quarter-resolution pass the full-resolution rows,
    exactly once"""
    rows = [MH.own_rows(H, r, world) for r in range(world)]
    assert rows[0][0] == 0 and rows[-1][1] == H
    assert all(a[1] == b[0] for a, b in zip(rows[:-1], rows[1:]))
    for scale, H0 in ((1, 2 * H + 1), (2, 4 * H + 3)):
        up = [MH.own_rows(H, r, world, scale, H0) for r in range(world)]
        assert up[0][0] == 0 and up[-1][1] == H0
        assert all(a[1] == b[0] for a, b in zip(up[:-1], up[1:]))


def test_stage_lists():
    assert MH.shadows_stages(4, scale=1) == ["Ray Trace", "Temporal Accumulation", "A-Trous 0", "A-Trous 1", "A-Trous 2", "A-Trous 3", "Upsample"]
    assert MH.shadows_stages(0, denoise=0, exchange=True) == ["Ray Trace", "Exchange"]
    assert MH.shadows_stages(2, linked=True, denoise=0, exchange=True) == ["Ray Trace", "Mask Exchange Wait"]
    assert MH.ao_stages(scale=2) == ["Ray Trace", "Temporal Accumulation", "Bilateral Blur", "Upsample"]
    assert MH.union_names([MH.taa_stages(False), MH.taa_stages(True)]) == ["TAA", "Reset Blit"]
    assert MH.union_names([MH.reflections_stages(1, scale=1), MH.reflections_stages(3, scale=1)]) == \
        ["Ray Trace", "Temporal Accumulation", "A-Trous 0", "Upsample", "A-Trous 1", "A-Trous 2"]
