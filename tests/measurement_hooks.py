"""Host restatements of the measurement hooks bench.py reports from (hr_api.h): the device checksum
(hr_pass_output_checksum), the tile / pixel counts of hr_pass_get_stats and the stage lists of hr_pass_stage_times.
No GPU and no CUDA library needed; the GPU side is tests/test_gpu_measurement_hooks.py, the CPU checks of this file
tests/test_measurement_hooks_cpu.py.
"""
import numpy as np

M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15  # splitmix64's increment
_MIX1, _MIX2 = np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)


def mix64(z):
    """splitmix64 finaliser over uint64 arrays (wrapping arithmetic)"""
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * _MIX1
        z = (z ^ (z >> np.uint64(27))) * _MIX2
    return z ^ (z >> np.uint64(31))


def mix64_int(z):
    """the same finaliser on one Python integer, with exact big-integer arithmetic reduced mod 2^64"""
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def texel_values(img):
    """(H, W) or (H, W, C) image as the device holds it -> (H, W) uint64: each texel's bytes as a little-endian unsigned integer"""
    a = np.ascontiguousarray(img)
    H, W = a.shape[:2]
    n = a.nbytes // (H * W) if H * W else 1
    assert n in (1, 2, 4, 8), f"texel of {n} bytes"
    return a.view(np.uint8).reshape(H, W, n).copy().view(f"<u{n}").reshape(H, W).astype(np.uint64)


def texel_terms(img):
    """(H, W) uint64: texel i's term mix(mix(i + GOLDEN) ^ v_i), i = y * W + x (hr_pass_output_checksum)"""
    v = texel_values(img)
    H, W = v.shape
    with np.errstate(over="ignore"):
        i = np.arange(H * W, dtype=np.uint64).reshape(H, W) + np.uint64(GOLDEN)
    return mix64(mix64(i) ^ v)


def checksum(img, row0=0, row1=0):
    """hr_pass_output_checksum of rows [row0, row1) of `img` (row1 <= 0: the whole image), exact mod 2^64"""
    if row1 <= 0:
        row0, row1 = 0, img.shape[0]
    t = texel_terms(img)[row0:row1]
    return int(np.sum(t, dtype=np.uint64)) if t.size else 0  # uint64 sums wrap: the sum mod 2^64


def checksum_ref(img, row0=0, row1=0):
    """the same sum texel by texel with Python integers (slow: small images only), for checking checksum() itself"""
    v = texel_values(img)
    H, W = v.shape
    if row1 <= 0:
        row0, row1 = 0, H
    acc = 0
    for y in range(row0, row1):
        for x in range(W):
            acc += mix64_int(mix64_int(y * W + x + GOLDEN) ^ int(v[y, x]))
    return acc & M64


def split_sum(img, cuts):
    """sum mod 2^64 of the checksums of the row ranges between consecutive cuts (0 and H included by the caller)"""
    return sum(checksum(img, a, b) for a, b in zip(cuts[:-1], cuts[1:]) if b > a) & M64


def random_cuts(rng, H, k):
    """0 = c0 <= c1 <= ... <= ck = H, with repeated cuts (empty ranges) allowed"""
    return [0] + sorted(int(c) for c in rng.integers(0, H + 1, size=k - 1)) + [H]


# ---------------------------------------------------------------------------------------------- tile and pixel counts
def tile_counts(flags, W, H, row0=0, row1=None):
    """(tiles_total, tiles_denoise, pixels_total) of hr_pass_get_stats for a render whose denoise stages covered pass rows
    [row0, row1) of a W x H pass with tile-flag image `flags` (ceil(H/8) x ceil(W/8)); row1 None = H"""
    row1 = H if row1 is None else row1
    if row1 <= row0:
        return 0, 0, 0
    t0, t1 = row0 // 8, (row1 + 7) // 8
    TW = (W + 7) // 8
    return (t1 - t0) * TW, int(np.count_nonzero(flags[t0:t1])), (row1 - row0) * W


def own_rows(H, rank, world, scale=0, H0=None):
    """rows of a pass's final output that rank owns: its band hr_shard_rows(H) at pass resolution, or, for an upsampled final of
    full-resolution height H0, the band's full-resolution rows b0 << scale .. b1 << scale (H0 for the last band).  A rank left
    without a band (fewer 8-row tiles than ranks) owns no rows"""
    tiles = (H + 7) // 8
    base, rem = divmod(tiles, world)
    t0 = rank * base + min(rank, rem)
    t1 = t0 + base + (1 if rank < rem else 0)
    b0, b1 = min(t0 * 8, H), min(t1 * 8, H)
    if scale:
        return (H0, H0) if b1 <= b0 else (b0 << scale, H0 if b1 >= H else b1 << scale)
    return b0, b1


def denoise_rows(H, rank, world, halo):
    """rows a sharded rank's denoise stages cover: its band +- halo, clamped to the pass"""
    b0, b1 = own_rows(H, rank, world)
    if world <= 1:
        return 0, H
    return max(b0 - halo, 0), min(b1 + halo, H)


# ---------------------------------------------------------------------------------------------- stage lists
def atrous(n):
    return [f"A-Trous {i}" for i in range(n)]


def shadows_stages(filter_iterations=4, denoise=1, scale=0, linked=False, exchange=False):
    """hr_shadows_render's stage list; linked: cooperative ray trace (hr_shard_link_local / hr_shard_init); exchange: world > 1 with
    the gather on (the mark follows the NCCL exchange, which is skipped when there is no communicator)"""
    s = ["Ray Trace"] + (["Mask Exchange Wait"] if linked else [])
    if denoise:
        s += ["Temporal Accumulation"] + atrous(filter_iterations) + (["Upsample"] if scale else [])
    if exchange and not (linked and not denoise):
        s += ["Exchange"]
    return s


def ao_stages(denoise=1, scale=0, linked=False, exchange=False):
    s = ["Ray Trace"] + (["Mask Exchange Wait"] if linked else [])
    if denoise:
        s += ["Temporal Accumulation", "Bilateral Blur"] + (["Upsample"] if scale else [])
    if exchange and not (linked and not denoise):
        s += ["Exchange"]
    return s


def reflections_stages(filter_iterations=4, denoise=1, scale=0):
    """single GPU"""
    s = ["Ray Trace"]
    if denoise:
        s += ["Temporal Accumulation"] + atrous(filter_iterations) + (["Upsample"] if scale else [])
    return s


def ddgi_stages(linked=False, world=1):
    s = (["Atlas Publish"] if linked else []) + ["Ray Trace", "Probe Update"]
    if linked:
        s += ["Atlas Ready Wait", "Atlas Store", "Atlas Wait"]
    return s + ["Sample Probe Grid"] + (["Exchange"] if world > 1 else [])


def taa_stages(blit):
    return (["Reset Blit"] if blit else []) + ["TAA"]


DEFERRED_STAGES = ["Deferred"]
TONEMAP_STAGES = ["Tone Map"]


def path_tracer_stages(gather_wait=False):
    return ["Ground Truth Path Trace"] + (["Gather Wait"] if gather_wait else [])


def union_names(lists):
    """the names hr_pass_stage_times reports for a window of renders with these stage lists: each name once, in first-seen order"""
    out = []
    for names in lists:
        out += [n for n in names if n not in out]
    return out
