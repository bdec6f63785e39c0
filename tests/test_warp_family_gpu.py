"""The antialiased sampler (csrc/warp.cu) against float64, over its launch plans.

  warp_compose_fwd_kernel<T, MIP, MODE>   one 32 x 8 output tile of one image per CTA; the tile's coordinates and an
                                          84-slot halo ring (halo_slot, replicate-clamped to the image) in shared memory
                                          feed the level of detail.  MODE 0 reads a grid (gg_mipmap_warp_forward), 1
                                          generates an affine grid and 2 a composed flow (gg_stn_sample_forward), 3 lerps
                                          two grids for T weights (gg_mipmap_warp_lerp_forward; CTA image tn = frame N + n)
  warp_lerp_mean_kernel<T, MIP, C>        the per-frame sums over the batch of MODE 3's frames, 8 frames per CTA row
                                          (gg_mipmap_warp_lerp_mean)
  warp_bwd_kernel<T, MIP>                 one thread per output pixel, grid-stride: grad_src / grad_pyramid by atomics,
                                          grad_grid gathered from the neighbours whose level-of-detail arg-max it is
                                          (gg_mipmap_warp_backward)
  sample_indices_kernel                   the integer work (x0, y0, l0, l1) of the same device functions

This file restates the host-side plans in Python and labels every case with the routes it takes (CPU tests assert that
the cases reach every label), then checks every output against float64 evaluated on the exact operands the launch reads
(warp_reference.py: the source, the STORED fp32 pyramid, and the caller's grid or the grid the kernel wrote), with a
bound derived from the kernel's order of operations (oracle/rounding.py):
    fp32 value     |y - ref| <= c * 2^-24 * A + extra                (assert_fp32_sum)
    stored half    |y - ref| <= 1/2 ulp + c * 2^-24 * A + extra      (assert_rounded_once with k = c)
A is the same float64 evaluation on magnitudes, `extra` an explicit float64 allowance for the fp32 level of detail (eps_L
times the output's slope in the level) and, where the grid is not dyadic, for the fp32 source coordinate.

Dyadic grids: entries are multiples of 2^-12 with |g + 1| < 4, so ((g + 1) size - 1) / 2, the bilinear fractions, the
up-sampling weights and the level-of-detail coordinate differences are exact in fp32 for sources up to 1024 px a side
(the numerator (g + 1) 2^12 stays below 2^14 and the size at most 2^10: the product fits in 24 bits).  Every forward
output is continuous across the discrete choices (corner floor, level floor / ceil, clamps, the arg-max: a max), so the
forward checks exempt no pixel.  The backward cases have margins on all of those choices, asserted up front, and also
exempt no pixel.

The kernel's correction for a level-of-detail arg-max clamped onto the pixel itself never changes a result: such a
neighbour is the pixel, its squared distance is 0 < 1, and a pixel whose arg-max lies below the clamp(min=1) passes no
level-of-detail gradient.  The backward cases still reach that arg-max ("bwd: arg-max clamped onto the pixel itself").

Every check prints its worst observed k / c (`[contract] ...` lines with `pytest -s`), and the module prints the worst per
path when it finishes.
"""
import math
import re

import pytest
import torch

from fp64_contract import (BF16, CODE, DEV, F16, F32, H100_SMS, SHORT, TNAME, Worst, assert_routes_reached, ceil_div, f32,
                           grid_for, launched, library, nan_at, run_fresh, seeded)
from oracle import sampling as S
from oracle.rounding import assert_fp32_sum, assert_rounded_once
from warp_reference import (LN2, _edge_grid, _take, argmax_targets, bilinear_slopes, blend, blend_abs, build_stack,
                            coordinate_error, forward_c, level_error, level_slope, levels64, neighbour_sq,
                            pad_geometry, sample_stack, split_pyramid, undecided_pixels)

TILE_X, TILE_Y = 32, 8                     # warp.cu kTileX, kTileY
RING = 2 * (TILE_X + 2) + 2 * TILE_Y       # kRing: 84 halo slots
MEAN_FRAMES = 8                            # kMeanFrames
PAD_MODES = S.PAD_MODES
PAD_CODE = {"zeros": 0, "border": 1, "reflection": 2}
DTYPES = (F32, F16, BF16)


# ======================================================================================== planner restatement (no GPU)
def forward_plan(n, ho, wo, mode, frames=1):
    """sample_forward: (tiles_x, tiles_y, CTAs); mode 3 launches a CTA row per frame."""
    tx, ty = ceil_div(wo, TILE_X), ceil_div(ho, TILE_Y)
    return tx, ty, n * tx * ty * (frames if mode == 3 else 1)


def cta_tile(cta, tiles_x, tiles_y, n, mode):
    """warp_compose_fwd_kernel's CTA -> (bx, by, output image tn, source sample, frame)."""
    bx, by, tn = cta % tiles_x, (cta // tiles_x) % tiles_y, cta // (tiles_x * tiles_y)
    return bx, by, tn, (tn % n if mode == 3 else tn), (tn // n if mode == 3 else 0)


def halo_slot(r):
    """Halo position (hy, hx) in tile coordinates of ring slot r: the row above, the row below, the left and right
    columns."""
    if r < TILE_X + 2:
        return -1, r - 1
    if r < 2 * (TILE_X + 2):
        return TILE_Y, r - (TILE_X + 2) - 1
    if r < 2 * (TILE_X + 2) + TILE_Y:
        return r - 2 * (TILE_X + 2), -1
    return r - 2 * (TILE_X + 2) - TILE_Y, TILE_X


def mean_plan(ho, wo, frames):
    """gg_mipmap_warp_lerp_mean: grid (tiles, chunks), and the frames nf of each chunk (the last one may hold fewer)."""
    tiles = ceil_div(wo, TILE_X) * ceil_div(ho, TILE_Y)
    chunks = ceil_div(frames, MEAN_FRAMES)
    return (tiles, chunks), [min(MEAN_FRAMES, frames - MEAN_FRAMES * k) for k in range(chunks)]


def trips(total, sms):
    """Grid-stride trips of a grid_for(total, 256) launch."""
    return ceil_div(total, grid_for(total, sms) * 256)


def trip_batch(ho, wo, sms):
    """fp64_contract.grid_stride_batch for `sms` SMs."""
    return grid_for(1 << 62, sms) * 256 // (ho * wo) + 2


# ------------------------------------------------------------------------------------------------------------ grids
def dyadic_random(n, ho, wo, hs, ws, seed, steps, noise=2, exact=()):
    """Dyadic grids (k / 4096, |k| <= 5120): per sample an affine grid whose neighbours sit about steps[i] px apart in
    level-of-detail coordinates, slightly rotated, plus integer noise of up to `noise` on half the entries; samples in
    `exact` take the axis-aligned grid without noise (exact ties, and an exact level where steps[i] is a power of two and
    (size - 1) / 2 divides the step's k)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(ho, dtype=torch.float64), torch.arange(wo, dtype=torch.float64), indexing="ij")
    out = []
    for i in range(n):
        st = steps[i % len(steps)]
        kx_step, ky_step = round(st * 8192 / max(ws - 1, 1)), round(st * 8192 / max(hs - 1, 1))
        rot = 0 if i in exact else 0.15 * (i + 1)
        kx = kx_step * (xx - (wo - 1) / 2) + rot * ky_step * (yy - (ho - 1) / 2)
        ky = ky_step * (yy - (ho - 1) / 2) - rot * kx_step * (xx - (wo - 1) / 2)
        k = torch.stack([kx, ky], -1).round()
        if i not in exact:
            k += torch.randint(-noise, noise + 1, k.shape, generator=g) * (torch.rand(k.shape, generator=g) < 0.5)
        out.append(k.clamp(-5120, 5120))
    return (torch.stack(out) / 4096.0).float()


def seam_grid(n, ho, wo, seed):
    """Dyadic grids over several tiles whose columns 32j - 1 | 32j and rows 8j - 1 | 8j sit ~4 px apart (level 2) while
    every other neighbour is ~0.7 px away: the pixels on each side of every tile seam take their arg-max neighbour from
    the other tile, i.e. from the halo ring, and it moves their level by two."""
    g = torch.Generator().manual_seed(seed)
    sx = torch.tensor([70, 90, 110])[torch.randint(0, 3, (n, wo), generator=g)]
    sy = torch.tensor([70, 90, 110])[torch.randint(0, 3, (n, ho), generator=g)]
    sx[:, ::TILE_X] = 520
    sy[:, ::TILE_Y] = 520
    sx[:, 0] = sy[:, 0] = 0
    kx, ky = sx.cumsum(1), sy.cumsum(1)
    kx, ky = kx - kx[:, -1:] // 2, ky - ky[:, -1:] // 2
    yy, xx = torch.meshgrid(torch.arange(ho), torch.arange(wo), indexing="ij")
    k = torch.stack([kx[:, None, :] + 7 * yy, ky[:, :, None] + 5 * xx], -1)
    return (k.clamp(-5120, 5120).double() / 4096.0).float()


def is_dyadic(grid):
    k = grid.double() * 4096.0
    return bool((k == k.round()).all() and ((grid.double() + 1.0).abs() < 4).all())


# ------------------------------------------------------------------------------------------------------------- cases
# forward, mode 0: (name, dtype, E, N, C, hs, ws, ho, wo, max_level, min_level)
MODE0 = [
    ("seams", F32, 4, 2, 3, 64, 64, 24, 96, 4.0, 0.0),
    ("padded", F16, 5, 3, 2, 194, 450, 13, 45, 4.5, 0.5),
    ("single-tile", BF16, 4, 3, 3, 65, 65, 6, 20, 3.0, 0.0),
    ("row", F32, 3, 3, 1, 64, 64, 1, 33, 3.0, 0.0),
    ("column", BF16, 3, 3, 1, 64, 64, 17, 1, 2.5, 0.0),
    ("pixel", F16, 2, 3, 2, 32, 32, 1, 1, 2.0, 0.0),
    ("plain", F32, 0, 2, 3, 40, 56, 16, 64, 0.0, 0.0),
    ("plain-row", F16, 0, 2, 2, 40, 56, 1, 40, 0.0, 0.0),
    ("plain-column", BF16, 0, 2, 2, 40, 56, 9, 1, 0.0, 0.0),
    ("plain-pixel", BF16, 0, 1, 1, 40, 56, 1, 1, 0.0, 0.0),
]
STEPS = (0.7, 1.6, 3.1, 6.5, 13.0, 2.0)       # px between neighbours: levels 0 (clamped), 0.7, 1.6, 2.7, 3.7, 1
STEPS_OF = {"padded": (3.1, 13.0, 22.0)}      # up to level 4.46


def mode0_grid(case):
    name, dtype, extra, n, c, hs, ws, ho, wo, max_level, min_level = case
    if name == "seams":
        return seam_grid(n, ho, wo, 11)
    # on the 65 px source (size - 1) / 2 = 32 divides k: the first sample's 2 px steps give level 1 exactly
    steps = STEPS_OF.get(name, STEPS)
    return dyadic_random(n, ho, wo, hs, ws, sum(map(ord, name)), (2.0,) + steps if hs == 65 else steps,
                         exact=(0,) if hs == 65 else ())


# mode 1: (dtype, E, N, C, hs, ws, ho, wo);  mode 2: ... + (lh, lw, s, base warp, alpha);  mode 3: ... + (T, broadcast base)
MODE1 = [(F32, 3, 2, 3, 64, 64, 24, 70), (F16, 3, 2, 2, 65, 65, 17, 33), (BF16, 2, 3, 1, 32, 32, 8, 32),
         (F32, 0, 2, 3, 64, 64, 9, 40), (F16, 0, 2, 2, 64, 64, 8, 64), (BF16, 0, 1, 1, 32, 32, 1, 1)]
MODE2 = [(F32, 3, 2, 3, 64, 64, 4, 12, 3, True, "n"), (F16, 3, 2, 2, 64, 64, 9, 40, 1, False, None),
         (BF16, 2, 2, 1, 32, 32, 6, 11, 3, True, "1"), (F32, 0, 2, 3, 64, 64, 10, 35, 1, False, "n"),
         (F16, 0, 2, 2, 64, 64, 3, 11, 3, True, None), (BF16, 0, 2, 1, 32, 32, 5, 7, 1, False, "1")]
MODE3 = [(F32, 3, 2, 3, 64, 64, 12, 40, 3, False), (F16, 3, 3, 2, 65, 65, 9, 33, 2, True),
         (BF16, 2, 2, 1, 32, 32, 8, 32, 4, False), (F32, 0, 2, 2, 64, 64, 12, 40, 2, True),
         (F16, 0, 2, 2, 64, 64, 7, 31, 3, False), (BF16, 0, 3, 1, 32, 32, 9, 9, 2, True)]
# lerp weights on both sides of |w| = 0.5, with full mantissas; 1 - w rounds for -0.65 and 1.3
ALPHAS = [0.3, 0.7, -0.65, 0.2, 1.3, 0.15, 0.85, -0.2]
# frame mean: every dtype x MIP x C, cycling T, accumulate and N
MEAN = [(dt, e, c, (1, 8, 9, 17)[i % 4], i % 2, (0, 1, 5)[i % 3])
        for i, (dt, e, c) in enumerate((dt, e, c) for dt in DTYPES for e in (0, 2) for c in (1, 2, 3, 4))]
# backward: (grid, dtype, MIP); the trip case takes grid_stride_batch samples
BWD = [("pinch", F32, True), ("ties", F16, True), ("clamps", BF16, True), ("clamps_min", F32, True),
       ("borders", F32, True), ("trips", F32, True), ("ties", F32, False), ("borders", F16, False),
       ("pinch", BF16, False)]
SUBSETS = ("grad_src", "grad_grid", "both")


def trip_grid(n):
    """A dyadic affine grid over a 16 px source (level-of-detail scale 7.5 px per unit): left / right neighbours 2.217 px
    apart, up / down 2.098 px, so every level is 1.149 (exact left / right ties, clear of every integer and clamp)."""
    yy, xx = torch.meshgrid(torch.arange(16), torch.arange(16), indexing="ij")
    k = torch.stack([150 * xx + 30 * yy - 1300, -20 * xx + 140 * yy - 1100], -1)
    return (k.double() / 512.0).float()[None].expand(n, -1, -1, -1).contiguous()


def bwd_setup(case, sms=H100_SMS):
    """-> (grid (N, Ho, Wo, 2), hs, ws, C, E, max_level, min_level)."""
    name, dtype, mip = case
    if name == "trips":
        return trip_grid(trip_batch(16, 16, sms)), 16, 16, 1, 2, 2.0, 0.0
    grid, size, num_levels, min_level = _edge_grid(name)
    extra = min(num_levels - 1, 6)                 # a 64 px source hosts 6 levels beyond the source
    if not mip:
        return grid, size, size, 3, 0, 0.0, 0.0
    return grid, size, size, 3, extra, float(extra), min_level


# ------------------------------------------------------------------------------------------------------------ labels
def tile_labels(ho, wo):
    labels = {"tiles: wo %% 32 %s 0" % ("==" if wo % TILE_X == 0 else "!="),
              "tiles: ho %% 8 %s 0" % ("==" if ho % TILE_Y == 0 else "!=")}
    tx, ty, _ = forward_plan(1, ho, wo, 0)
    if tx == ty == 1:
        labels.add("tiles: a single tile")
    if tx >= 2 and ty >= 2:
        labels.add("tiles: >= 2 tiles on both axes")
    if (ho, wo) == (1, 1):
        labels.add("tiles: 1 x 1")
    elif ho == 1:
        labels.add("tiles: ho = 1")
    elif wo == 1:
        labels.add("tiles: wo = 1")
    return labels


def level_labels(grid, hs, ws, extra, max_level, min_level):
    labels = set()
    lp = pad_geometry(hs, ws)[0]
    labels.add("pyramid: power-of-two source (lp = 0)" if lp == 0 else "pyramid: width-padded source (lp > 0)")
    if min_level > 0:
        labels.add("pyramid: min_level > 0")
    if max_level != math.floor(max_level):
        labels.add("pyramid: max_level fractional")
    if max_level == extra:
        labels.add("pyramid: max_level at extra")
    lv = levels64(grid.double(), hs, ws, f32(max_level), f32(min_level))
    for k in range(extra):
        if bool(((lv > k) & (lv < k + 1)).any()):
            labels.add("levels in (%d, %d), w != 0" % (k, k + 1))
    if bool(((lv == lv.floor()) & (lv >= 1)).any()):
        labels.add("levels: an exact integer level >= 1 (l0 = l1)")
    # tile seams: a pixel next to a seam whose arg-max neighbour lies across it, in the halo, and moves its level
    arg, _, _ = argmax_targets(grid, hs, ws)
    n, ho, wo = arg.shape
    x = torch.arange(wo)[None, None, :].expand(n, ho, wo)
    y = torch.arange(ho)[None, :, None].expand(n, ho, wo)
    live = lv > 0
    for what, sel in (("x = 32j, arg-max left", (x % TILE_X == 0) & (x > 0) & (arg == 0)),
                      ("x = 32j - 1, arg-max right", (x % TILE_X == TILE_X - 1) & (x < wo - 1) & (arg == 1)),
                      ("y = 8j, arg-max up", (y % TILE_Y == 0) & (y > 0) & (arg == 2)),
                      ("y = 8j - 1, arg-max down", (y % TILE_Y == TILE_Y - 1) & (y < ho - 1) & (arg == 3))):
        if bool((sel & live).any()):
            labels.add("seam: %s in the halo, level > 0" % what)
    return labels


def mode0_labels(case):
    name, dtype, extra, n, c, hs, ws, ho, wo, max_level, min_level = case
    labels = {"fwd: %s MIP=%d mode 0" % (SHORT[dtype], extra > 0)} | tile_labels(ho, wo)
    labels |= {"pad: %s" % m for m in PAD_MODES} | {"levels_out: null", "levels_out: written"}
    if extra:
        labels |= level_labels(mode0_grid(case), hs, ws, extra, max_level, min_level)
    return labels


def mode_labels(mode, case):
    dtype, extra, n, c, hs, ws = case[:6]
    labels = {"fwd: %s MIP=%d mode %d" % (SHORT[dtype], extra > 0, mode), "grid_out: null", "grid_out: written"}
    if mode == 2:
        lh, lw, s, base, alpha = case[6:]
        labels |= {"delta_out: null", "delta_out: written", "flow: %s base warp" % ("with" if base else "no"),
                   "flow: %s alpha" % ("with" if alpha else "no"), "flow: s = %d" % s}
        labels |= tile_labels(lh * s, lw * s)
        if s > 1 and (lw * s) > TILE_X and TILE_X % s:
            labels.add("flow: s-blocks straddle a tile seam")
    if mode == 3:
        ho, wo, frames, bcast = case[6:]
        labels |= tile_labels(ho, wo)
        labels.add("lerp: base_stride %s" % ("0 (one broadcast base)" if bcast else "full"))
        if n >= 2 and frames >= 2:
            labels.add("lerp: N >= 2 and T >= 2")
        al = ALPHAS[:frames]
        labels |= {"lerp: |w| < 0.5" for a in al if abs(a) < 0.5} | {"lerp: |w| >= 0.5" for a in al if abs(a) >= 0.5}
    if mode == 1:
        labels |= tile_labels(*case[6:8])
    return labels


def mean_labels(case):
    dtype, extra, c, frames, acc, n = case
    labels = {"mean: %s MIP=%d C=%d" % (SHORT[dtype], extra > 0, c), "mean: T = %d" % frames,
              "mean: accumulate %d" % acc, "mean: N = %d" % n}
    _, nf = mean_plan(12, 40, frames)
    if nf[-1] < MEAN_FRAMES:
        labels.add("mean: a last chunk of nf < 8 frames")
    if len(nf) >= 2:
        labels.add("mean: several frame chunks")
    return labels


def bwd_labels(case, sms=H100_SMS):
    name, dtype, mip = case
    grid, hs, ws, c, extra, max_level, min_level = bwd_setup(case, sms)
    n, ho, wo = grid.shape[:3]
    labels = {"bwd: %s MIP=%d %s" % (SHORT[dtype], mip, s) for s in SUBSETS}
    labels.add("bwd: %s" % ("one trip" if trips(n * ho * wo, sms) == 1 else "a second trip"))
    if not mip:
        return labels
    sq = neighbour_sq(grid.double(), hs, ws)
    arg, ty, tx = argmax_targets(grid, hs, ws)
    sq_arg = sq.gather(0, arg[None])[0]
    yy = torch.arange(ho)[None, :, None].expand(n, ho, wo)
    xx = torch.arange(wo)[None, None, :].expand(n, ho, wo)
    self_t = (ty == yy) & (tx == xx)
    if bool(self_t.any()):
        labels.add("bwd: arg-max clamped onto the pixel itself")
    live = (sq_arg >= 1) & ~self_t
    hits = torch.zeros(n, ho, wo, dtype=torch.long)
    ni = torch.arange(n)[:, None, None].expand(n, ho, wo)
    hits.index_put_((ni[live], ty[live], tx[live]), torch.ones(int(live.sum()), dtype=torch.long), accumulate=True)
    for k in (2, 3, 4):
        if bool((hits == k).any()):
            labels.add("bwd: a pixel targeted by %d neighbours" % k)
    top = sq.clamp(min=1.0).sqrt().topk(2, dim=0).values
    if bool(((top[0] == top[1]) & (top[0] > 1)).any()):
        labels.add("bwd: exact arg-max ties")
    if bool((sq.max(dim=0).values == 1).any()):
        labels.add("bwd: sq == 1")
    lv = levels64(grid.double(), hs, ws, max_level, min_level)
    for what, v in (("0", 0.0), ("min_level > 0", min_level), ("max_level", max_level)):
        if (what == "0" or v > 0) and bool((lv == v).any()):
            labels.add("bwd: levels exactly at %s" % what)
    return labels


REQUIRED = (
    ["fwd: %s MIP=%d mode %d" % (SHORT[d], m, k) for d in DTYPES for m in (0, 1) for k in range(4)]
    + ["pad: %s" % m for m in PAD_MODES]
    + ["tiles: wo % 32 == 0", "tiles: wo % 32 != 0", "tiles: ho % 8 == 0", "tiles: ho % 8 != 0", "tiles: a single tile",
       "tiles: ho = 1", "tiles: wo = 1", "tiles: 1 x 1", "tiles: >= 2 tiles on both axes"]
    + ["seam: %s in the halo, level > 0" % w for w in ("x = 32j, arg-max left", "x = 32j - 1, arg-max right",
                                                        "y = 8j, arg-max up", "y = 8j - 1, arg-max down")]
    + ["pyramid: power-of-two source (lp = 0)", "pyramid: width-padded source (lp > 0)", "pyramid: min_level > 0",
       "pyramid: max_level fractional", "pyramid: max_level at extra"]
    + ["levels in (%d, %d), w != 0" % (k, k + 1) for k in range(5)]
    + ["levels: an exact integer level >= 1 (l0 = l1)", "levels_out: null", "levels_out: written", "grid_out: null",
       "grid_out: written", "delta_out: null", "delta_out: written"]
    + ["flow: with base warp", "flow: no base warp", "flow: with alpha", "flow: no alpha", "flow: s = 1", "flow: s = 3",
       "flow: s-blocks straddle a tile seam"]
    + ["lerp: N >= 2 and T >= 2", "lerp: base_stride 0 (one broadcast base)", "lerp: base_stride full",
       "lerp: |w| < 0.5", "lerp: |w| >= 0.5"]
    + ["mean: %s MIP=%d C=%d" % (SHORT[d], m, c) for d in DTYPES for m in (0, 1) for c in (1, 2, 3, 4)]
    + ["mean: T = %d" % t for t in (1, 8, 9, 17)] + ["mean: accumulate 0", "mean: accumulate 1"]
    + ["mean: N = %d" % n for n in (0, 1, 5)] + ["mean: a last chunk of nf < 8 frames", "mean: several frame chunks"]
    + ["bwd: %s MIP=%d %s" % (SHORT[d], m, s) for d in DTYPES for m in (0, 1) for s in SUBSETS]
    + ["bwd: one trip", "bwd: a second trip", "bwd: a pixel targeted by 2 neighbours",
       "bwd: a pixel targeted by 3 neighbours", "bwd: a pixel targeted by 4 neighbours",
       "bwd: arg-max clamped onto the pixel itself", "bwd: exact arg-max ties", "bwd: sq == 1",
       "bwd: levels exactly at 0", "bwd: levels exactly at min_level > 0", "bwd: levels exactly at max_level"]
)


def all_labels(sms=H100_SMS):
    reached = set()
    for cs in MODE0:
        reached |= mode0_labels(cs)
    for mode, cases in ((1, MODE1), (2, MODE2), (3, MODE3)):
        for cs in cases:
            reached |= mode_labels(mode, cs)
    for cs in MEAN:
        reached |= mean_labels(cs)
    for cs in BWD:
        reached |= bwd_labels(cs, sms)
    return reached


def test_cases_reach_every_route():
    """Coverage of the cases below, by the restatement planned for 132 SMs: every forward instantiation (dtype x MIP x
    MODE) and padding mode, the tile shapes, the four tile seams read from the halo, the pyramid shapes and level ranges,
    every optional output null and written, the flow and lerp variants, every frame-mean instantiation with T, accumulate
    and N, and every backward instantiation and output subset, with both grid-stride trip counts and the gather's edges."""
    assert_routes_reached(REQUIRED, all_labels())


def test_restated_plans_cover_every_pixel_once():
    """The restated CTA -> (tile, image) map covers every output pixel of every forward case exactly once (mode 3: frame
    tn / N of sample tn % N); the 84 halo slots are the 84 distinct positions around a 32 x 8 tile; the frame chunks of
    the mean partition 0..T-1; the backward's grid-stride trips cover N Ho Wo."""
    ring = {halo_slot(r) for r in range(RING)}
    around = {(y, x) for y in range(-1, TILE_Y + 1) for x in range(-1, TILE_X + 1)
              if y in (-1, TILE_Y) or x in (-1, TILE_X)}
    assert ring == around and len(around) == RING
    shapes = [(0, cs[3], cs[7], cs[8], 1) for cs in MODE0] + [(1, cs[2], cs[6], cs[7], 1) for cs in MODE1]
    shapes += [(2, cs[2], cs[6] * cs[8], cs[7] * cs[8], 1) for cs in MODE2] + [(3, cs[2], cs[6], cs[7], cs[8]) for cs in MODE3]
    for mode, n, ho, wo, frames in shapes:
        tx, ty, ctas = forward_plan(n, ho, wo, mode, frames)
        seen = {}
        for cta in range(ctas):
            bx, by, tn, src, frame = cta_tile(cta, tx, ty, n, mode)
            assert src < n and frame < frames and tn == frame * n + src
            for py in range(by * TILE_Y, min(by * TILE_Y + TILE_Y, ho)):
                for px in range(bx * TILE_X, min(bx * TILE_X + TILE_X, wo)):
                    seen[(tn, py, px)] = seen.get((tn, py, px), 0) + 1
        assert len(seen) == n * frames * ho * wo and set(seen.values()) == {1}, (mode, n, ho, wo)
    for frames in (1, 7, 8, 9, 16, 17, 100):
        (_, chunks), nf = mean_plan(12, 40, frames)
        assert sum(nf) == frames and all(1 <= f <= MEAN_FRAMES for f in nf) and chunks == len(nf)
    for total in (1, 256, 540672, 540673, 10 ** 7):
        assert grid_for(total, H100_SMS) * 256 * trips(total, H100_SMS) >= total
    assert trips(trip_batch(16, 16, H100_SMS) * 256, H100_SMS) == 2


def test_every_case_is_feasible():
    """Every case's pyramid is one the library builds, and every grid the bounds call dyadic is."""
    from gangealing_b200 import _lib
    lib = _lib.load()
    for cs in MODE0:
        name, dtype, extra, n, c, hs, ws, ho, wo, max_level, min_level = cs
        assert lib.gg_mipmap_pyramid_elems(n * c, hs, ws, extra) >= 0 and max_level <= extra
        assert is_dyadic(mode0_grid(cs)), name
    for cases in (MODE1, MODE2, MODE3):
        for cs in cases:
            assert lib.gg_mipmap_pyramid_elems(cs[2] * cs[3], cs[4], cs[5], cs[1]) >= 0
    for cs in BWD:
        grid, hs, ws, c, extra, max_level, min_level = bwd_setup(cs)
        assert lib.gg_mipmap_pyramid_elems(c, hs, ws, extra) >= 0 and is_dyadic(grid), cs


# ======================================================================================================== GPU checks
WORST = Worst("k / c per path", "%-56s %.2f")
_report_worst = WORST.fixture()


def check(y, ref, a, c, path, what, extra=None):
    """fp32: |y - ref| <= c u A + extra; fp16 / bf16: 1/2 ulp + c u A + extra."""
    y = y.detach().cpu()
    if y.dtype in (F16, BF16):
        _, obs = assert_rounded_once(y, ref, a, c, "%s: %s" % (path, what), extra)
    else:
        obs = assert_fp32_sum(y, ref, a, c, "%s: %s" % (path, what), extra)
    WORST.note(path, obs)
    print("[contract] %s: %s: obs=%.2f (c=%d)" % (path, what, obs, c))


def pyramid_of(x, extra):
    from gangealing_b200.stn.sampling import _pyramid
    return _pyramid(x, extra)


def stored_levels(pyr, n, c, hs, ws, extra):
    return [] if not extra else [t.double() for t in split_pyramid(pyr.cpu(), n, c, hs, ws, extra)]


def forward_reference(x, pyr, grid, extra, max_level, min_level, mode, dyadic):
    """-> (ref, A, extra allowance, float64 levels or None, eps_L or None) of one forward output on the grid `grid`."""
    n, c, hs, ws = x.shape
    x64, g64 = x.double().cpu(), grid.double().cpu()
    levs = stored_levels(pyr, n, c, hs, ws, extra)
    stack = build_stack(x64, levs, hs, ws)
    smp = sample_stack(stack, g64, mode)
    smp_abs = sample_stack(build_stack(x64.abs(), [t.abs() for t in levs], hs, ws), g64, mode)
    if extra:
        lv = levels64(g64, hs, ws, f32(max_level), f32(min_level))
        eps = level_error(g64, hs, ws, dyadic)
        # A where the fp32 level may fall on the other side of an integer: the larger blend of |values|
        a = torch.stack([blend_abs(smp_abs, (lv + s * eps).clamp(0, extra)) for s in (-1, 0, 1)]).max(dim=0).values
        allow = eps[:, None] * level_slope(smp, lv, extra)
    else:
        lv = eps = None
        a, allow = blend_abs(smp_abs, None), torch.zeros(n, c, *g64.shape[1:3], dtype=torch.float64)
    if not dyadic:
        ex, ey = coordinate_error(g64, hs, ws, mode)
        kx, ky = bilinear_slopes(stack, g64, mode)
        allow = allow + (ex[:, None, None] * kx + ey[:, None, None] * ky).max(dim=2).values
    return blend(smp, lv), a, allow, lv, eps


def check_forward(out, x, pyr, grid, extra, max_level, min_level, mode, path, what, dyadic, levels_out=None):
    ref, a, allow, lv, eps = forward_reference(x, pyr, grid, extra, max_level, min_level, mode, dyadic)
    check(out, ref, a, forward_c(extra), path, what, allow)
    if levels_out is not None:
        err = (levels_out.double().cpu() - lv).abs()
        bad = err > eps
        assert not bool(bad.any()), "%s: %s: %d levels off by more than eps_L (worst %.3g, eps_L %.3g)" % (
            path, what, int(bad.sum()), float(err.max()), float(eps[bad].max()))
        WORST.note("levels_out (|error| / eps_L)", float((err / eps).max()))


def call_forward(x, pyr, grid, extra, max_level, min_level, mode, with_levels=True):
    lib = library()
    n, c, hs, ws = x.shape
    ho, wo = grid.shape[1:3]
    out = nan_at((n, c, ho, wo), x.dtype)
    lv = nan_at((n, ho, wo), F32) if with_levels and extra else None
    rc = lib.load().gg_mipmap_warp_forward(out.data_ptr(), lib.ptr(lv), x.data_ptr(), lib.ptr(pyr), grid.data_ptr(),
                                           CODE[x.dtype], n, c, hs, ws, ho, wo, extra, max_level, min_level,
                                           PAD_CODE[mode], lib.stream())
    lib.check(rc, "gg_mipmap_warp_forward")
    return out, lv


def _fwd_id(cs):
    return "%s-%s-E%d" % (cs[0], SHORT[cs[1]], cs[2])


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODE0, ids=_fwd_id)
def test_forward_on_a_read_grid(case):
    """Mode 0 on dyadic grids, every padding mode, with and without levels_out: the output against the float64 blend of
    the stored pyramid's stack within forward_c (no pixel exempt), levels_out within eps_L, and the output without
    levels_out bitwise the same."""
    name, dtype, extra, n, c, hs, ws, ho, wo, max_level, min_level = case
    x = torch.randn(n, c, hs, ws, generator=seeded(hs + ws + n), device=DEV).to(dtype)
    pyr = pyramid_of(x, extra)
    grid = mode0_grid(case).to(DEV)
    for mode in PAD_MODES:
        out, lv = call_forward(x, pyr, grid, extra, max_level, min_level, mode)
        check_forward(out, x, pyr, grid, extra, max_level, min_level, mode, "fwd mode 0, %s" % SHORT[dtype],
                      "%s %s" % (name, mode), True, lv)
        out2, _ = call_forward(x, pyr, grid, extra, max_level, min_level, mode, with_levels=False)
        assert torch.equal(out2, out), "%s %s: the output depends on levels_out" % (name, mode)


def affine_inputs(case, seed):
    dtype, extra, n, c, hs, ws, ho, wo = case[:8]
    g = torch.Generator().manual_seed(seed)
    theta = torch.eye(2, 3)[None] * (0.6 + 1.8 * torch.rand(n, 1, 1, generator=g)) + 0.2 * torch.randn(n, 2, 3, generator=g)
    x = torch.randn(n, c, hs, ws, generator=g).to(dtype)
    return x.to(DEV), theta.to(DEV)


def stn_call(x, pyr, mode, extra, max_level, min_level, pad, ho, wo, theta=None, low=None, mask=None, ident=None,
             alpha=None, s=1, grid_out=True, delta_out=True, with_levels=True):
    lib = library()
    n, c, hs, ws = x.shape
    out = nan_at((n, c, ho, wo), x.dtype)
    g = nan_at((n, ho, wo, 2), F32) if grid_out else None
    d = nan_at((n, ho, wo, 2), F32) if (delta_out and mode == 2) else None
    lv = nan_at((n, ho, wo), F32) if (with_levels and extra) else None
    lh, lw = (low.shape[1], low.shape[2]) if low is not None else (0, 0)
    rc = lib.load().gg_stn_sample_forward(out.data_ptr(), lib.ptr(g), lib.ptr(d), lib.ptr(lv), x.data_ptr(), lib.ptr(pyr),
                                          lib.ptr(theta), lib.ptr(low), lib.ptr(mask), lib.ptr(ident), lib.ptr(alpha),
                                          mode, CODE[x.dtype], n, c, hs, ws, ho, wo, lh, lw, s, extra, max_level,
                                          min_level, PAD_CODE[pad], lib.stream())
    lib.check(rc, "gg_stn_sample_forward")
    return out, g, d, lv


# The affine grid: bx = (2x + 1) / wo - 1 rounds in the division and the subtraction, u (|bx + 1| + |bx|) together (the
# same for by); g = fmaf(M0, bx, fmaf(M1, by, M2)) rounds once per fmaf, u |M1 by + M2| and u |g|; one more for the
# products of two roundings.
AFFINE_C = 2


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODE1, ids=lambda cs: "%s-E%d-%dx%d" % (SHORT[cs[0]], cs[1], cs[6], cs[7]))
def test_affine_sampler(case):
    """Mode 1: the written grid against the float64 affine grid within AFFINE_C, then the samples against float64 on
    that written grid, with the fp32 source coordinate's error times the bilinear slope as an allowance."""
    dtype, extra, n, c, hs, ws, ho, wo = case
    x, theta = affine_inputs(case, ho * 100 + wo)
    pyr = pyramid_of(x, extra)
    max_level = float(extra)
    th = theta.double().cpu()
    bx = (2 * torch.arange(wo, dtype=torch.float64) + 1) / wo - 1
    by = (2 * torch.arange(ho, dtype=torch.float64) + 1) / ho - 1
    for pad in PAD_MODES:
        out, grid, _, lv = stn_call(x, pyr, 1, extra, max_level, 0.0, pad, ho, wo, theta=theta)
        ref = S.affine_grid_ref(th, (n, c, ho, wo))
        inner = (th[:, None, None, :, 1] * by[None, :, None, None] + th[:, None, None, :, 2]).abs()
        a = (inner + ref.abs() + th[:, None, None, :, 0].abs() * ((bx + 1).abs() + bx.abs())[None, None, :, None]
             + th[:, None, None, :, 1].abs() * ((by + 1).abs() + by.abs())[None, :, None, None])
        check(grid, ref, a, AFFINE_C, "mode 1 grid", "%s %s" % (SHORT[dtype], pad))
        check_forward(out, x, pyr, grid, extra, max_level, 0.0, pad, "fwd mode 1, %s" % SHORT[dtype],
                      "%dx%d %s" % (ho, wo, pad), False, lv)
        out2, g2, _, _ = stn_call(x, pyr, 1, extra, max_level, 0.0, pad, ho, wo, theta=theta, grid_out=False,
                                  with_levels=False)
        assert g2 is None and torch.equal(out2, out)


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODE2, ids=lambda cs: "%s-E%d-%dx%d-s%d" % (SHORT[cs[0]], cs[1], cs[6], cs[7], cs[8]))
def test_flow_sampler(case):
    """Mode 2: grid and delta bitwise the stand-alone flow_compose's, the samples against float64 on that grid (with the
    coordinate allowance), and the output the same with grid_out / delta_out / levels_out null."""
    from gangealing_b200.stn import flow as GF
    dtype, extra, n, c, hs, ws, lh, lw, s, with_base, alpha_kind = case
    g = torch.Generator().manual_seed(lh * 100 + lw + s)
    ho, wo = lh * s, lw * s
    x = torch.randn(n, c, hs, ws, generator=g).to(dtype).to(DEV)
    low = ((0.1 / s) * torch.randn(n, lh, lw, 2, generator=g)).to(DEV)
    mask = (2.0 * torch.randn(n, 9 * s * s, lh, lw, generator=g)).to(DEV)
    base = (torch.eye(2, 3)[None] * 1.4 + 0.1 * torch.randn(n, 2, 3, generator=g)).to(DEV) if with_base else None
    alpha = {None: None, "n": torch.rand(n, generator=g), "1": torch.rand(1, generator=g)}[alpha_kind]
    alpha = None if alpha is None else alpha.to(DEV)
    ident = S.affine_grid_ref(torch.eye(2, 3)[None], (1, 1, ho, wo)).to(DEV)
    pyr = pyramid_of(x, extra)
    max_level = float(extra)
    delta_c, flow_c = GF.flow_compose(low, mask, ident, base, alpha, s)
    alpha = None if alpha is None else alpha.expand(n).contiguous()     # the entry reads alpha[n] (flow_inputs expands)
    for pad in PAD_MODES:
        out, flow, delta, lv = stn_call(x, pyr, 2, extra, max_level, 0.0, pad, ho, wo, theta=base, low=low, mask=mask,
                                        ident=ident, alpha=alpha, s=s)
        assert torch.equal(flow, flow_c) and torch.equal(delta, delta_c), "mode 2 grid / delta vs flow_compose"
        check_forward(out, x, pyr, flow, extra, max_level, 0.0, pad, "fwd mode 2, %s" % SHORT[dtype],
                      "%dx%d s=%d %s" % (ho, wo, s, pad), False, lv)
        out2, _, _, _ = stn_call(x, pyr, 2, extra, max_level, 0.0, pad, ho, wo, theta=base, low=low, mask=mask,
                                 ident=ident, alpha=alpha, s=s, grid_out=False, delta_out=False, with_levels=False)
        assert torch.equal(out2, out)


def lerp_operands(n, ho, wo, hs, ws, bcast, seed):
    """Base and target grids off the dyadic lattice: on it b - a and a + w (b - a) are exact for most weights, and the two
    branches of torch.lerp would round the same exact value."""
    g = torch.Generator().manual_seed(seed)
    base = dyadic_random(1 if bcast else n, ho, wo, hs, ws, seed, (1.2, 3.0))
    target = dyadic_random(n, ho, wo, hs, ws, seed + 1, (0.8, 5.0, 2.5))
    base = base + 1e-3 * torch.randn(base.shape, generator=g)
    target = target + 1e-3 * torch.randn(target.shape, generator=g)
    return base.to(DEV), target.to(DEV)


def lerp_call(x, pyr, base, target, alphas, extra, max_level, min_level, pad, grid_out=True):
    lib = library()
    n, c, hs, ws = x.shape
    ho, wo = target.shape[1:3]
    t = alphas.numel()
    stride = 0 if (base.shape[0] == 1 and n != 1) else ho * wo * 2
    out = nan_at((t, n, c, ho, wo), x.dtype)
    grids = nan_at((t, n, ho, wo, 2), F32) if grid_out else None
    rc = lib.load().gg_mipmap_warp_lerp_forward(out.data_ptr(), lib.ptr(grids), x.data_ptr(), lib.ptr(pyr), base.data_ptr(),
                                                stride, target.data_ptr(), alphas.data_ptr(), t, CODE[x.dtype], n, c, hs,
                                                ws, ho, wo, extra, max_level, min_level, PAD_CODE[pad], lib.stream())
    lib.check(rc, "gg_mipmap_warp_lerp_forward")
    return out, grids


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODE3, ids=lambda cs: "%s-E%d-N%d-T%d-%s" % (SHORT[cs[0]], cs[1], cs[2], cs[8],
                                                                              "bcast" if cs[9] else "full"))
def test_lerp_sampler(case):
    """Mode 3: every written grid bitwise torch.lerp(base[n], target[n], alphas[t]) (both of its branches), every frame
    against float64 on its grid, and the frames the same without grid_out."""
    dtype, extra, n, c, hs, ws, ho, wo, frames, bcast = case
    x = torch.randn(n, c, hs, ws, generator=seeded(ho + wo + frames), device=DEV).to(dtype)
    base, target = lerp_operands(n, ho, wo, hs, ws, bcast, ho * 7 + wo)
    alphas = torch.tensor(ALPHAS[:frames], device=DEV)
    pyr = pyramid_of(x, extra)
    max_level = float(extra)
    for pad in PAD_MODES:
        out, grids = lerp_call(x, pyr, base, target, alphas, extra, max_level, 0.0, pad)
        for t in range(frames):
            want = torch.lerp(base.expand(n, -1, -1, -1), target, float(alphas[t]))
            assert torch.equal(grids[t], want), "frame %d (alpha %g): grid is not torch.lerp's" % (t, ALPHAS[t])
            check_forward(out[t], x, pyr, grids[t], extra, max_level, 0.0, pad, "fwd mode 3, %s" % SHORT[dtype],
                          "frame %d %s" % (t, pad), False)
        out2, _ = lerp_call(x, pyr, base, target, alphas, extra, max_level, 0.0, pad, grid_out=False)
        assert torch.equal(out2, out)


@pytest.mark.gpu
@pytest.mark.parametrize("case", MEAN, ids=lambda cs: "%s-E%d-C%d-T%d-acc%d-N%d" % (SHORT[cs[0]], *cs[1:]))
def test_frame_mean(case):
    """The frame sums are bitwise the sequential fp32 sum over the batch of gg_mipmap_warp_lerp_forward's stored frames
    (acc + s under accumulate) and bitwise repeatable; the frames past T, in a guard region behind acc, stay untouched,
    and so do alphas past T (a guard the kernel would read into frames that do not exist).  The float64 contract of each
    frame is test_lerp_sampler's."""
    dtype, extra, c, frames, accumulate, n = case
    lib = library()
    hs = ws = 32
    ho, wo = 12, 40
    x = torch.randn(n, c, hs, ws, generator=seeded(c * 10 + frames), device=DEV).to(dtype)
    base, target = lerp_operands(max(n, 1), ho, wo, hs, ws, False, c + frames)
    base, target = base[:n].contiguous(), target[:n].contiguous()
    alpha_buf = torch.full((frames + MEAN_FRAMES,), 0.375, device=DEV)
    alpha_buf[:frames] = torch.tensor((ALPHAS * 3)[:frames], device=DEV)
    alphas = alpha_buf[:frames]
    plane = c * ho * wo
    pyr = pyramid_of(x, extra) if n else None
    max_level = float(extra)
    for pad in PAD_MODES:
        if n:
            frames_out, _ = lerp_call(x, pyr, base, target, alphas, extra, max_level, 0.0, pad, grid_out=False)
        want = torch.zeros(frames, c, ho, wo, device=DEV)
        for i in range(n):
            want = want + frames_out[:, i].float()
        acc0 = torch.randn(frames, c, ho, wo, generator=seeded(frames), device=DEV)
        if accumulate:
            want = acc0 + want
        results = []
        for _ in range(2):
            buf = torch.full((frames * plane + MEAN_FRAMES * plane,), 1234.5, device=DEV)
            acc = buf[:frames * plane].view(frames, c, ho, wo)
            acc.copy_(acc0)
            rc = lib.load().gg_mipmap_warp_lerp_mean(acc.data_ptr(), x.data_ptr(), lib.ptr(pyr),
                                                     base.data_ptr() if n else alphas.data_ptr(), ho * wo * 2,
                                                     target.data_ptr() if n else alphas.data_ptr(), alphas.data_ptr(),
                                                     frames, CODE[dtype], n, c, hs, ws, ho, wo, extra, max_level, 0.0,
                                                     PAD_CODE[pad], accumulate, lib.stream())
            lib.check(rc, "gg_mipmap_warp_lerp_mean")
            assert bool((buf[frames * plane:] == 1234.5).all()), "%s: frames past T were written" % pad
            assert torch.equal(acc, want), "%s: %d sums differ from the sequential fp32 sum of the frames" % (
                pad, int((acc != want).sum()))
            results.append(acc.clone())
        assert torch.equal(results[0], results[1])
    assert bool((alpha_buf[frames:] == 0.375).all())


# ------------------------------------------------------------------------------------------------------------ backward
def upsample_taps(d, lev, size):
    """warp.cu upsample_index for destination d of a level of `size` at scale 2^lev: (i0, i1)."""
    src = ((d.double() + 0.5) * 2.0 ** -lev - 0.5).clamp(min=0)
    i0 = src.floor().long()
    return i0, i0 + (i0 < size - 1).long()


def fan_in(grid, hs, ws, mode, lv, extra, n):
    """The largest number of atomicAdds into one element of grad_src (index 0) and of each pyramid level: every in-bounds
    corner of every pixel that uses the level, four up-sampling taps per corner on levels >= 1 (zero weights included)."""
    g = grid.double()
    ix, iy = S.source_index(g[..., 0], ws, mode), S.source_index(g[..., 1], hs, mode)
    x0, y0 = ix.floor().long(), iy.floor().long()
    l0 = lv.floor().long() if extra else torch.zeros_like(x0)
    l1 = lv.ceil().long() if extra else l0
    lp, hp, wp = pad_geometry(hs, ws)
    ni = torch.arange(n)[:, None, None].expand_as(x0)
    out = []
    for lev in range(extra + 1):
        h, w = (hs, ws) if lev == 0 else (hp >> lev, wp >> lev)
        cnt = torch.zeros(n, h, w, dtype=torch.long)
        uses = (l0 == lev) | ((l1 == lev) & (l1 != l0))
        for a in (0, 1):
            for b in (0, 1):
                y, x = y0 + a, x0 + b
                ok = uses & (y >= 0) & (y < hs) & (x >= 0) & (x < ws)
                if lev == 0:
                    idx = [(y, x)]
                else:
                    ya, yb = upsample_taps(y + lp, lev, h)
                    xa, xb = upsample_taps(x + lp, lev, w)
                    idx = [(ya, xa), (ya, xb), (yb, xa), (yb, xb)]
                for yy, xx in idx:
                    cnt.index_put_((ni[ok], yy[ok], xx[ok]), torch.ones(int(ok.sum()), dtype=torch.long), accumulate=True)
        out.append(int(cnt.max()))
    return out


# grad_src / grad_pyramid: a term is g = go (1 - w) (the subtraction and the product: 2), times wy * wx (2 more); a level
# >= 1 term then times uy.l and ux.l (2 more); F atomicAdds onto zero add F roundings of partial sums bounded by the sum of
# |terms|; one more for the products of two roundings.
def scatter_c(level, fan):
    return 4 + (2 if level > 0 else 0) + fan + 1


# grad_grid: per channel, a level's dix = -v00 wy0 + v01 wy0 - v10 wy1 + v11 wy1 is 4 products and 3 additions on values
# that carry corner_c(l) - 5 roundings of their own (4 on levels >= 1): 8; (1 - w) dx0 + w dx1 adds 4 (1 - w, two
# products, a sum), go * (...) 1, the sum over C channels C, times mult 1: 14 + C.  The level-of-detail term: glevel sums
# go (o1 - o0) over C (o: corner_c = 9, the difference and the product: 11 + C); g_sq = glevel / (dmax ln2f) (0.5 / dmax)
# with dmax carrying 3 roundings (sq: 2, sqrtf: 1 -- dyadic coordinates are exact), the fp32 ln 2 1, and 2 products, a
# division and 0.5 / dmax 1 more each: 11; gox = 2 dx g_sq sx (2 dx and sx exact): 2 more: 24 + C.  A pixel's value adds
# its own term, its own level-of-detail share and up to 4 gathered neighbour shares: 6 additions; one more for the
# products of two roundings.
def grid_c(c):
    return max(14 + c, 24 + c) + 6 + 1


def corners_abs(s, ix, iy):
    """|values| (N, C, Ho, Wo) at the four corners of each pixel (zero outside the image) and the bilinear weights."""
    n, c, h, w = s.shape
    x0, y0 = ix.floor(), iy.floor()
    wx1, wy1 = ix - x0, iy - y0
    x0, y0 = x0.long(), y0.long()
    flat = s.abs().reshape(n, c, h * w)
    v = []
    for a in (0, 1):
        for b in (0, 1):
            y, x = y0 + a, x0 + b
            ok = (y >= 0) & (y < h) & (x >= 0) & (x < w)
            idx = (y.clamp(0, h - 1) * w + x.clamp(0, w - 1)).reshape(n, 1, -1).expand(n, c, -1)
            v.append(torch.gather(flat, 2, idx).reshape(n, c, *ix.shape[1:]) * ok[:, None])
    return v, 1 - wx1, wx1, 1 - wy1, wy1


def backward_reference(x, pyr, grid, go, extra, max_level, min_level, mode):
    """float64 autograd with x, each stored level and the grid as leaves, and the magnitudes and allowances of every
    gradient -> dict."""
    n, c, hs, ws = x.shape
    levs32 = stored_levels(pyr, n, c, hs, ws, extra)
    x64 = x.double().cpu().requires_grad_(True)
    leaves = [t.clone().requires_grad_(True) for t in levs32]
    g64 = grid.double().cpu().requires_grad_(True)
    go64 = go.double().cpu()
    smp = sample_stack(build_stack(x64, leaves, hs, ws), g64, mode)
    lv = levels64(g64, hs, ws, f32(max_level), f32(min_level)) if extra else None
    grads = torch.autograd.grad(blend(smp, lv), [x64, *leaves, g64], go64)
    gd = g64.detach()
    lvd = None if lv is None else lv.detach()
    eps = level_error(gd, hs, ws, True) if extra else torch.zeros(gd.shape[:3], dtype=torch.float64)
    # magnitudes of the scatter: the same blend of |values| (its weights are >= 0) against |go|; the allowance for the
    # fp32 (1 - w) / w: eps_L times the scatter of |go| into both levels at full weight
    xa = x64.detach().abs().requires_grad_(True)
    la = [t.detach().abs().requires_grad_(True) for t in levs32]
    smp_a = sample_stack(build_stack(xa, la, hs, ws), gd, mode)
    a_src = torch.autograd.grad(blend(smp_a, lvd), [xa, *la], go64.abs(), retain_graph=True)
    if extra:
        l0, l1 = lvd.floor().long(), lvd.ceil().long()
        both = (eps[:, None] * go64.abs() * (_take(smp_a, l0) + _take(smp_a, l1))).sum()
        allow_src = torch.autograd.grad(both, [xa, *la])
    else:
        allow_src = [torch.zeros_like(t) for t in [xa, *la]]
    # magnitudes of the grid gradient
    stack_abs = [t.detach() for t in build_stack(x64.detach().abs(), [t.abs() for t in levs32], hs, ws)]
    ix, iy = S.source_index(gd[..., 0], ws, mode), S.source_index(gd[..., 1], hs, mode)
    per = []
    for s in stack_abs:
        (v00, v01, v10, v11), wx0, wx1, wy0, wy1 = corners_abs(s, ix, iy)
        wx0, wx1, wy0, wy1 = (t[:, None] for t in (wx0, wx1, wy0, wy1))
        per.append(((v00 + v01) * wy0 + (v10 + v11) * wy1, (v00 + v10) * wx0 + (v01 + v11) * wx1,
                    v00 * wx0 * wy0 + v01 * wx1 * wy0 + v10 * wx0 * wy1 + v11 * wx1 * wy1))
    dix, diy, oab = (torch.stack([p[i] for p in per], dim=2) for i in range(3))
    ga = go64.abs()
    if extra:
        two = (l1 != l0).double()
        w = (lvd - l0)[:, None]
        k0 = 1 - w * two[:, None]
        bil_x = (ga * (k0 * _take(dix, l0) + two[:, None] * w * _take(dix, l1))).sum(1) * ws / 2
        bil_y = (ga * (k0 * _take(diy, l0) + two[:, None] * w * _take(diy, l1))).sum(1) * hs / 2
        allow_x = eps * (ga * (_take(dix, l0) + _take(dix, l1))).sum(1) * two * ws / 2
        allow_y = eps * (ga * (_take(diy, l0) + _take(diy, l1))).sum(1) * two * hs / 2
        glevel = (ga * (_take(oab, l0) + _take(oab, l1))).sum(1) * two
        sq = neighbour_sq(gd, hs, ws)
        arg, ty, tx = argmax_targets(gd, hs, ws)
        sq_arg = sq.gather(0, arg[None])[0]
        c_ = S.lod_coordinates(gd, hs, ws)
        cp = torch.nn.functional.pad(c_.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="replicate").permute(0, 2, 3, 1)
        neigh = torch.stack([cp[:, 1:-1, :-2], cp[:, 1:-1, 2:], cp[:, :-2, 1:-1], cp[:, 2:, 1:-1]])
        d_arg = neigh.gather(0, arg[None, ..., None].expand(1, *arg.shape, 2))[0] - c_
        raw = 0.5 * torch.log2(sq.max(dim=0).values)
        lvl = raw.clamp(0, f32(max_level))
        live = (raw >= 0) & (raw <= f32(max_level)) & (lvl >= f32(min_level)) & (sq_arg >= 1)
        fac = live.double() * glevel / (sq_arg.clamp(min=1.0) * LN2)
        lod_x = fac * d_arg[..., 0].abs() * (ws - 1) / 2
        lod_y = fac * d_arg[..., 1].abs() * (hs - 1) / 2
        ni = torch.arange(n)[:, None, None].expand_as(arg)
        a_x, a_y = bil_x + lod_x, bil_y + lod_y
        a_x = a_x.index_put((ni, ty, tx), lod_x, accumulate=True)
        a_y = a_y.index_put((ni, ty, tx), lod_y, accumulate=True)
    else:
        bil_x = (ga * dix[:, :, 0]).sum(1) * ws / 2
        bil_y = (ga * diy[:, :, 0]).sum(1) * hs / 2
        a_x, a_y = bil_x, bil_y
        allow_x = allow_y = torch.zeros_like(a_x)
    return dict(grad_src=grads[0], grad_levels=list(grads[1:1 + extra]), grad_grid=grads[-1], a_src=a_src[0],
                a_levels=list(a_src[1:]), allow_src=allow_src[0], allow_levels=list(allow_src[1:]),
                a_grid=torch.stack([a_x, a_y], -1), allow_grid=torch.stack([allow_x, allow_y], -1), levels=lvd)


def call_backward(x, pyr, grid, go, extra, max_level, min_level, pad, subset):
    lib = library()
    n, c, hs, ws = x.shape
    ho, wo = grid.shape[1:3]
    want_src, want_grid = subset in ("grad_src", "both"), subset in ("grad_grid", "both")
    gsrc = torch.zeros(n, c, hs, ws, device=DEV) if want_src else None
    gpyr = torch.zeros_like(pyr) if (want_src and pyr is not None) else None
    ggrid = nan_at((n, ho, wo, 2), F32) if want_grid else None
    rc = lib.load().gg_mipmap_warp_backward(lib.ptr(gsrc), lib.ptr(gpyr), lib.ptr(ggrid), go.data_ptr(), x.data_ptr(),
                                            lib.ptr(pyr), grid.data_ptr(), CODE[x.dtype], n, c, hs, ws, ho, wo, extra,
                                            max_level, min_level, PAD_CODE[pad], lib.stream())
    lib.check(rc, "gg_mipmap_warp_backward")
    return gsrc, gpyr, ggrid


def _bwd_id(cs):
    return "%s-%s-%s" % (cs[0], SHORT[cs[1]], "mip" if cs[2] else "plain")


@pytest.mark.gpu
@pytest.mark.parametrize("case", BWD, ids=_bwd_id)
def test_backward(case):
    """gg_mipmap_warp_backward on dyadic grids with margins on every decision (asserted first), each output subset, every
    padding mode: grad_src and every grad_pyramid level (before the pyramid's adjoint) within scatter_c with the fan-in
    counted from the reference, grad_grid within grid_c (level-of-detail gather included), no pixel exempt; and
    gg_warp_sample_indices returns the reference's (x0, y0, l0, l1) on every pixel."""
    lib = library()
    name, dtype, mip = case
    grid, hs, ws, c, extra, max_level, min_level = bwd_setup(case, lib.sm_count())
    n, ho, wo = grid.shape[:3]
    x = torch.randn(n, c, hs, ws, generator=seeded(n + hs), device=DEV).to(dtype)
    go = torch.randn(n, c, ho, wo, generator=seeded(n + ho + 1), device=DEV).to(dtype)
    pyr = pyramid_of(x, extra)
    grid_d = grid.to(DEV)
    path = "bwd %s %s" % (SHORT[dtype], "mip" if mip else "plain")
    for pad in PAD_MODES:
        exempt = undecided_pixels(grid, hs, ws, pad, max_level if extra else None, min_level)
        assert int(exempt.sum()) == 0, "%s %s: %d pixels lack the decision margin: change the grid" % (name, pad,
                                                                                                     int(exempt.sum()))
        ref = backward_reference(x, pyr, grid_d, go, extra, max_level, min_level, pad)
        idx = torch.empty(n, ho, wo, 4, dtype=torch.int32, device=DEV)
        rc = lib.load().gg_warp_sample_indices(idx.data_ptr(), grid_d.data_ptr(), n, hs, ws, ho, wo, max_level,
                                               min_level, PAD_CODE[pad], lib.stream())
        lib.check(rc, "gg_warp_sample_indices")
        idx = idx.cpu().long()
        g64 = grid.double()
        assert torch.equal(idx[..., 0], S.source_index(g64[..., 0], ws, pad).floor().long()), "x0"
        assert torch.equal(idx[..., 1], S.source_index(g64[..., 1], hs, pad).floor().long()), "y0"
        if extra:
            assert torch.equal(idx[..., 2], ref["levels"].floor().long()) and \
                torch.equal(idx[..., 3], ref["levels"].ceil().long()), "l0 / l1"
        else:
            assert bool((idx[..., 2:] == 0).all()), "l0 / l1 with max_level = 0"
        fans = fan_in(grid, hs, ws, pad, ref["levels"], extra, n)
        for subset in SUBSETS:
            gsrc, gpyr, ggrid = call_backward(x, pyr, grid_d, go, extra, max_level, min_level, pad, subset)
            what = "%s %s %s" % (name, pad, subset)
            if gsrc is not None:
                check(gsrc, ref["grad_src"], ref["a_src"], scatter_c(0, fans[0]), path + " grad_src", what,
                      ref["allow_src"])
                got = split_pyramid(gpyr, n, c, hs, ws, extra) if extra else []
                for i in range(extra):
                    check(got[i], ref["grad_levels"][i], ref["a_levels"][i], scatter_c(i + 1, fans[i + 1]),
                          path + " grad_pyramid", "%s level %d" % (what, i + 1), ref["allow_levels"][i])
            if ggrid is not None:
                check(ggrid, ref["grad_grid"], ref["a_grid"], grid_c(c), path + " grad_grid", what, ref["allow_grid"])


# ------------------------------------------------------------------------------------------------------------ launches
KERNELS = re.compile(r"(warp_compose_fwd_kernel|warp_lerp_mean_kernel|warp_bwd_kernel)<[^>]*>|sample_indices_kernel")


def _tb(flag):
    return "true" if flag else "false"


@pytest.mark.gpu
def test_each_entry_launches_its_labelled_instantiation():
    """Each entry launches exactly the instantiation its case is labelled with: warp_compose_fwd_kernel<T, MIP, MODE>,
    warp_lerp_mean_kernel<T, MIP, C>, warp_bwd_kernel<T, MIP> and sample_indices_kernel (one profiler session per
    dtype x MIP, the calls in order)."""
    run_fresh("test_warp_family_gpu", "check_launches")


def check_launches():
    """The body of test_each_entry_launches_its_labelled_instantiation (raises AssertionError on a mismatch)."""
    lib = library()
    checked = 0
    grid = dyadic_random(2, 9, 40, 32, 32, 1, (1.5, 3.0)).to(DEV)
    theta = torch.eye(2, 3, device=DEV)[None].repeat(2, 1, 1)
    low = torch.zeros(2, 3, 8, 2, device=DEV)
    mask = torch.zeros(2, 9 * 25, 3, 8, device=DEV)
    ident = S.affine_grid_ref(torch.eye(2, 3)[None], (1, 1, 15, 40)).to(DEV)
    alphas = torch.tensor([0.25, 0.75], device=DEV)
    for dtype in DTYPES:
        for extra in (0, 2):
            x = torch.randn(2, 3, 32, 32, device=DEV).to(dtype)
            pyr = pyramid_of(x, extra)
            go = torch.randn(2, 3, 9, 40, device=DEV).to(dtype)
            xs = [x[:, :1].repeat(1, c, 1, 1).contiguous() for c in (1, 2, 3, 4)]
            pyrs = [pyramid_of(xc, extra) for xc in xs]
            accs = [torch.zeros(2, c, 9, 40, device=DEV) for c in (1, 2, 3, 4)]
            mip, t = _tb(extra > 0), TNAME[dtype]

            def calls():
                call_forward(x, pyr, grid, extra, float(extra), 0.0, "border")
                stn_call(x, pyr, 1, extra, float(extra), 0.0, "border", 9, 40, theta=theta)
                stn_call(x, pyr, 2, extra, float(extra), 0.0, "border", 15, 40, low=low, mask=mask, ident=ident, s=5)
                lerp_call(x, pyr, grid, grid, alphas, extra, float(extra), 0.0, "border")
                for sub in SUBSETS:
                    call_backward(x, pyr, grid, go, extra, float(extra), 0.0, "border", sub)
                for c, xc, pc, acc in zip((1, 2, 3, 4), xs, pyrs, accs):
                    rc = lib.load().gg_mipmap_warp_lerp_mean(acc.data_ptr(), xc.data_ptr(), lib.ptr(pc), grid.data_ptr(),
                                                             9 * 40 * 2, grid.data_ptr(), alphas.data_ptr(), 2,
                                                             CODE[dtype], 2, c, 32, 32, 9, 40, extra, float(extra), 0.0,
                                                             1, 0, lib.stream())
                    lib.check(rc, "gg_mipmap_warp_lerp_mean")

            want = ["warp_compose_fwd_kernel<%s, %s, %d>" % (t, mip, m) for m in range(4)]
            want += ["warp_bwd_kernel<%s, %s>" % (t, mip)] * len(SUBSETS)
            want += ["warp_lerp_mean_kernel<%s, %s, %d>" % (t, mip, c) for c in (1, 2, 3, 4)]
            got = launched(calls, KERNELS)
            assert got == want, "launched %s, the cases are labelled %s" % (got, want)
            checked += len(want)
    idx = torch.empty(2, 9, 40, 4, dtype=torch.int32, device=DEV)
    got = launched(lambda: lib.check(lib.load().gg_warp_sample_indices(idx.data_ptr(), grid.data_ptr(), 2, 32, 32, 9, 40,
                                                                       2.0, 0.0, 1, lib.stream()), "indices"), KERNELS)
    assert got == ["sample_indices_kernel"], got
    print("[launch] %d entry calls launched their labelled instantiation" % (checked + 1))
