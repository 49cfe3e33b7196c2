"""Counter cases shared by tests/test_gpu_counters.py (device vs oracle) and tests/test_counters_cpu.py (the oracle's side of the
same cases).  Numbers, frame sequences and host-side measures only, no GPU.

Three counters feed every temporal pass and are otherwise only run at small values:
- `spp` (shadows, AO, reflections): the API accepts 1..255.  visibility = count / spp and the 17x17 box mean = window count /
  (289 spp) are exact quotients (DESIGN.md §7); away from powers of two a multiply by a rounded reciprocal is not: count == spp
  gives 0.99999994 at 38 of the counts (41, 47, 55, ...), an all-open window a mean one ulp off 1 at 36 (3, 6, 7, ...).
  SPP_SH_AO covers both, 128 (the largest blue-noise slot, 7) and 255.
- the history length (K3, K9, K14: fminf(32, length + 1)), which saturates at 32 after 31 frames of valid history.
- hr_frame::num_frames: the blue-noise sample index is (num_frames * spp + s) mod 256 over the unsigned counter (DESIGN.md §7),
  K18 / K12 seed their RNG with it and TAA jitters by num_frames % 16.  COUNTER_STARTS cross the 256 wrap, 2^31, 2^32 and, for spp
  255 and 4, the point where num_frames * spp crosses 2^31.
"""
import numpy as np

import pyhr

CAM = ((0.0, 14.0, 34.0), (0.0, 3.0, 0.0))  # the shadows-test scene's default camera
PAN = 0.05  # world units a frame, sideways
CUT_AT, CUT_JUMP = 3, 1.5  # frame of the cut (the camera jumps sideways, the passes' histories are reset)

# shadows + AO: (spp, W, H); 128 x 72 for spp >= 128 keeps the oracle at a few seconds a frame
SPP_SH_AO = [(3, 256, 144), (6, 256, 144), (7, 256, 144), (41, 256, 144), (47, 256, 144), (128, 128, 72), (255, 128, 72)]
SCALES_SH_AO = [(0, 1), (1, 2)]
SPP_REFL = [(3, 128, 72), (41, 128, 72), (255, 128, 72)]
SPP_LINKED = [3, 255]

HIST_CAP = 32
LONG_STATIC = 300  # static frames of the long run (64 x 48)

# (id, first num_frames, spp): 5-frame sequences across each wrap
COUNTER_STARTS = [
    ("wrap256", 250, 1),
    ("2^31-3", 2**31 - 3, 1),
    ("2^32-3", 2**32 - 3, 1),
    ("spp255_2^31", 8421502, 255),  # 8421504 * 255 + 128 = 2^31
    ("spp4_2^31", 2**29 - 2, 4),
]
# (spp, num_frames) whose mask / count image must equal the one at num_frames mod 256 (static camera); each read outside the
# sobol table before the oracle computed the index unsigned
MOD256 = [(1, 2**31 + 1), (1, 2**31 + 77), (1, 2**32 - 1), (255, 8421505), (4, 2**29 + 3)]


def frames(W, H, n, start=0, pan=(), cut=None, cam=CAM):
    """(i, frame) for i < n with num_frames = (start + i) mod 2^32; the camera moves PAN sideways on each frame in `pan` and jumps
    CUT_JUMP at frame `cut` (the caller resets the histories there)"""
    (px, py, pz), (tx, ty, tz) = cam
    f, dx = None, 0.0
    for i in range(n):
        if i in pan:
            dx += PAN
        if i == cut:
            dx += CUT_JUMP
        f = pyhr.make_frame((px + dx, py, pz), (tx + dx, ty, tz), W, H, prev=f, num_frames=(start + i) & 0xFFFFFFFF)
        yield i, f


def spp_frames(W, H, start=0):
    """the 5 frames of an spp case: static, static, pan, cut, pan.  Frames 0, 1, 3 and 4 blend with alpha >= 0.5"""
    return frames(W, H, 5, start, pan=(2, 4), cut=CUT_AT)


def history_frames(W, H, n=48):
    """static until frame 35 (the history length saturates at frame 31), a pan over frames 36..41, static again"""
    return frames(W, H, n, pan=range(36, 42))


def tile_all(pred, valid, t=8):
    """per t x t tile: pred holds on every pixel where `valid` does, and `valid` holds somewhere"""
    H, W = pred.shape
    TH, TW = -(-H // t), -(-W // t)
    out = np.zeros((TH, TW), bool)
    for ty in range(TH):
        for tx in range(TW):
            v, p = valid[ty * t:(ty + 1) * t, tx * t:(tx + 1) * t], pred[ty * t:(ty + 1) * t, tx * t:(tx + 1) * t]
            out[ty, tx] = v.any() and p[v].all()
    return out


def tile_any(pred, t=8):
    """per t x t tile: pred holds somewhere (a temporal stage's tile flag from its per-pixel flags)"""
    return ~tile_all(~pred, np.ones_like(pred), t)


def full_count_tiles(count, depth, hist_len, spp):
    """AO tiles in which every geometry pixel has count == spp and blends with alpha >= 0.5 (history length <= 2): there a
    visibility of 0.99999994 in place of 1 flags the tile"""
    geo = depth != 1.0
    return int(tile_all((count == spp) & (hist_len <= 2.0), geo).sum())


def open_windows(count, spp):
    """17x17 windows inside the image whose every pixel has count == spp"""
    full = (count == spp).astype(np.int64)
    c = np.pad(full.cumsum(0).cumsum(1), ((1, 0), (1, 0)))
    s = c[17:, 17:] - c[:-17, 17:] - c[17:, :-17] + c[:-17, :-17]
    return int((s == 289).sum())
