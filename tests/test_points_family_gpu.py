"""The nearest-neighbour search, the point tracker and the PCK-Transfer kernels (csrc/points.cu, csrc/pck.cu), over their
launch plans.  These kernels decide integers: a wrong index moves a point to another pixel or changes a PCK count.

  nn_init_kernel / nn_argmin_kernel / nn_unpack_kernel
        nn_argmin_search: grid (pblocks = ceil(P / 256), splits, N); the HW grid entries are cut into `splits` ranges of
        per = ceil(HW / splits) entries, splits = clamp(ceil(2 SMs / (pblocks N)), 1, min(ceil(HW / 1024), 65535)); a CTA
        scans its range in 1024-entry shared-memory tiles, one thread per point, and the splits meet in one 64-bit
        atomicMin on order_bits(d) << 32 | index.  gg_nn_argmin: init, search, unpack.
  pck_query_kernel
        grid-stride over min(ceil(total / 256), 8 SMs) CTAs, total = B P (+ B F F 2 with a flow): the query threads
        (normalise, analytic inverse similarity, the flow STN's round trip), then the nn_grid = delta + identity threads.
  pck_score_kernel
        ceil(B P / 256) CTAs: unravel the packed index, bilinear 'border' lookup in the destination grid + unnormalise (or
        the closed-form similarity), err <= alpha * thresh per alpha (A <= 8), warp sums, integer atomics.
  track_points_kernel
        128-thread CTAs, one thread per point for all T frames: the patch x patch window of pad_grid(lerp(base, target,
        w_t)), Unfold's zero candidates beyond the ring, the flat-index unravel with floor division.

This file restates the three host plans (planned for 132 SMs), labels every case with the routes it takes and asserts on
a machine without a GPU that the cases reach every label.  The GPU half calls gg_nn_argmin, gg_pck_transfer and
gg_track_points_lerp through the C ABI, with outputs filled with NaN or a sentinel and a guard past every output and
workspace, and checks:

  indices, bitwise     the search and the tracker evaluate d = (|p|^2 + |g|^2) - 2 g.p with __fmul_rn / __fadd_rn /
                       __fsub_rn only, so separate fp32 torch ops reproduce every distance bit; the first minimum of
                       those (torch.argmin's rule: the first NaN wins, an all-+inf row gives 0) must be the kernel's
                       index, with no tie exempt.  The tracker's lerp_aten uses fmaf, emulated exactly (exact float64
                       product, TwoSum, round to odd, one rounding to fp32).  The packed keys in the workspace must
                       carry the restated distance's bits.
  placed ties          duplicate entries straddling a split boundary and a tile seam, identical queries either side of
                       a point-block boundary, mirror entries +-g about a query on the axis (bitwise equal distances),
                       queries on clustered entries where the expanded distance rounds negative, in different splits:
                       the smaller index wins.
  against float64      e_j = 5 * 2^-24 * M_j bounds |d_fp32 - d| for candidate j, M = |p|^2 + |g|^2 + 2 (|gx px| +
                       |gy py|): three roundings each for |p|^2, |g|^2 and g.p (two are needed, the third absorbs the
                       second-order terms), the add and the subtract.  Where every other candidate's d - e exceeds the
                       float64 best's d + e the index is the float64 argmin; everywhere the picked d lies within
                       e_pick + e_best of the float64 minimum.
  PCK-Transfer         stage by stage from one call whose workspace is read back: nn_grid bitwise delta + identity; the
                       query within its derived bound of float64 congeal_query_ref (the analytic double inverse is
                       DESIGN.md section 2 deviation (11)); nn_index bitwise the restated argmin over the kernel's own
                       query and nn_grid; est within its derived bound of float64 lookup + unnormalise at the kernel's
                       own index (bitwise the closed form without a flow); counts exactly the fp32 restatement of
                       vis && sqrt(dx dx + dy dy) <= alpha * thresh on the kernel's own est, and equal across two calls.
  non-finite rows      a NaN query, a NaN entry in a later split than a finite minimum, an all-NaN grid, |p|^2 = +inf:
                       argmin's index, always in [0, HW); the tracker picks the first NaN candidate.

Every bound check prints its worst observed ratio (`[contract] ...` lines with `pytest -s`), and the module prints the
worst per check when it finishes.
"""
import math
import re
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fp64_contract import (DEV, H100_SMS, Worst, assert_routes_reached, ceil_div, f32, launched, library, run_fresh)
from oracle import pck as OP
from oracle import vis as OV
from oracle.rounding import U32, assert_fp32_sum

NN_THREADS, NN_TILE = 256, 1024          # points.cu kNNThreads, kNNTile
PCK_THREADS, MAX_ALPHAS = 256, 8         # pck.cu kPckThreads, kMaxAlphas
TRACK_THREADS = 128                      # track_points_kernel's launch bounds
GUARD = 1024                             # elements past every output and workspace that no launch may write
SENTINEL = -7                            # integer outputs start as this
K_D = 5                                  # roundings of the expanded distance, relative to M
HIGHER = 1 + 2.0 ** -20                  # second-order terms of the first-order bounds below
CHUNK = 1 << 23                          # distance elements per chunk (N x points x candidates)


# ======================================================================================== planner restatements (no GPU)
def nn_plan(n, p, hw, sms):
    """nn_argmin_search: point blocks, splits, each split's [e0, e1) and its 1024-entry tiles."""
    pblocks = ceil_div(p, NN_THREADS)
    splits = ceil_div(2 * sms, pblocks * n)
    splits = min(splits, ceil_div(hw, NN_TILE))
    splits = min(max(splits, 1), 65535)
    per = ceil_div(hw, splits)
    ranges = [(s * per, min(s * per + per, hw)) for s in range(splits)]
    return dict(pblocks=pblocks, splits=splits, per=per, ranges=ranges,
                tiles=[ceil_div(e1 - e0, NN_TILE) for e0, e1 in ranges])


def pck_plan(b, p, f, flow, sms):
    """gg_pck_transfer: the query grid and its trips, the score grid and the workspace layout in bytes."""
    npts = b * p
    total = npts + (b * f * f * 2 if flow else 0)
    qgrid = min(ceil_div(total, PCK_THREADS), 8 * sms)
    ws = npts * 16 + (b * f * f * 8 if flow else 0)
    return dict(total=total, qgrid=qgrid, trips=ceil_div(total, qgrid * PCK_THREADS), sgrid=ceil_div(npts, PCK_THREADS),
                ws=ws, best=(0, 8 * npts), query=(8 * npts, 16 * npts), nn_grid=(16 * npts, ws))


def track_plan(n, p):
    return dict(grid=ceil_div(n * p, TRACK_THREADS))


# ------------------------------------------------------------------------------------------------------------- cases
# nn: (name, N, P, HW, kind); kind "random" or "placed" (ties placed at the plan's split boundaries and tile seams)
NN_CASES = [
    ("one-split", 2, 33900, 2500, "placed"),          # pblocks 133, N pblocks = 266 >= 264: one split of 3 tiles
    ("splits-off-1024", 1, 300, 10000, "placed"),     # 10 splits of 1000 entries
    ("tiles-per-split", 2, 12800, 5000, "placed"),    # N pblocks = 100: 3 splits of 1667 entries, 2 tiles each
    ("hw-37", 3, 37, 37, "random"),
    ("hw-1024", 1, 500, 1024, "random"),
    ("hw-1025", 2, 257, 1025, "placed"),              # 2 splits of 513 entries
    ("hw-1", 2, 70, 1, "random"),
    ("grid-128x128", 1, 3000, 128 * 128, "placed"),   # 16 splits of 1024 entries: boundaries on multiples of 1024
]
# nn on sampling-grid-like inputs: (N, H, W, P) jittered lattices over [-1, 1]^2, and an all-zero 4 x 4 grid where all 16
# distances to the origin are 0 and the first entry wins
LATTICE_CASES = [(2, 16, 16, 37), (1, 128, 128, 3000), (3, 24, 40, 1)]
# pck: (name, B, P, A, S, F (0: similarity-only), visible, outputs)  outputs: "all" or "counts" (est_out, nn_index null)
PCK_CASES = [
    ("flow-one-trip", 3, 300, 5, 128, 64, True, "all"),
    ("flow-two-trips", 4, 37, 8, 256, 192, False, "all"),
    ("flow-a1-counts-only", 2, 17, 1, 128, 48, True, "counts"),
    ("flow-B12xP1", 12, 1, 3, 128, 32, True, "all"),
    ("similarity", 6, 300, 3, 128, 0, True, "all"),
    ("similarity-a8-no-visible", 12, 1, 8, 64, 0, False, "all"),
    ("similarity-counts-only", 2, 17, 2, 128, 0, True, "counts"),
]
# track: (name, N, P, H, patch, alphas)
ALPHAS = (0.0, 0.5, 1.0, 0.3, 0.75, -0.2)
TRACK_CASES = [
    ("patch1", 3, 300, 24, 1, ALPHAS),
    ("patch3", 3, 300, 24, 3, ALPHAS),
    ("patch7", 2, 100, 16, 7, ALPHAS[:3]),
    ("patch9", 3, 300, 24, 9, ALPHAS),
    ("patch37-beyond-every-border", 3, 300, 24, 37, ALPHAS),
    ("single-frame-small", 1, 5, 2, 3, (0.4,)),
]


def nn_labels(case, sms=H100_SMS):
    name, n, p, hw, kind = case
    pl = nn_plan(n, p, hw, sms)
    labels = set()
    if n * pl["pblocks"] >= 2 * sms:
        labels.add("nn: one split because N pblocks >= 2 SMs")
    if pl["splits"] > 1 and any(e0 % NN_TILE for e0, _ in pl["ranges"]):
        labels.add("nn: several splits, boundaries off multiples of 1024")
    if pl["splits"] > 1 and not any(e0 % NN_TILE for e0, _ in pl["ranges"]):
        labels.add("nn: several splits, boundaries on multiples of 1024")
    if any(t > 1 and (e1 - e0) % NN_TILE for (e0, e1), t in zip(pl["ranges"], pl["tiles"])):
        labels.add("nn: several tiles in a split, partial last tile")
    if hw < NN_TILE:
        labels.add("nn: HW < 1024")
    if hw in (1, NN_TILE, NN_TILE + 1):
        labels.add("nn: HW = %d" % hw)
    if p % NN_THREADS:
        labels.add("nn: partial last point block")
    if n > 1:
        labels.add("nn: N > 1 (blockIdx.z)")
    if kind == "placed" and pl["splits"] > 1:
        labels.add("nn: placed ties across a split boundary")
    if kind == "placed" and any(t > 1 for t in pl["tiles"]):
        labels.add("nn: placed ties across a tile seam")
    if kind == "placed" and p > NN_THREADS:
        labels.add("nn: identical queries either side of a point-block boundary")
    return labels


def pck_labels(case, sms=H100_SMS):
    name, b, p, a, s, f, visible, outputs = case
    pl = pck_plan(b, p, f, f > 0, sms)
    labels = {"pck_query: one trip" if pl["trips"] == 1 else "pck_query: >= 2 trips"}
    if f and (b * p) % 32:
        labels.add("pck_query: query / nn_grid boundary inside a warp")
    if not f:
        labels.add("pck_query: similarity-only (no nn_grid)")
    if a in (1, MAX_ALPHAS):
        labels.add("pck_score: A = %d" % a)
    if not visible:
        labels.add("pck_score: visible null")
    if outputs == "counts":
        labels.add("pck_score: est_out and nn_index null")
    if (b * p) % PCK_THREADS:
        labels.add("pck_score: B P not a multiple of 256")
    return labels


def track_frame0(case):
    """The case's inputs on the CPU (deterministic): base, target (N, H, H, 2), points (N, P, 2), centres (N, P, 2),
    alphas (T,).  The first points sit at (0, 0) with their centres at the corners, so that a zero candidate beyond the
    padded grid is nearest and the unravel wraps."""
    name, n, p, h, patch, alphas = case
    g = torch.Generator().manual_seed(sum(map(ord, name)) + p)
    eye = torch.eye(2, 3).unsqueeze(0).repeat(n, 1, 1)
    base = F.affine_grid(eye, (n, 1, h, h), align_corners=False) + 0.02 * torch.randn(n, h, h, 2, generator=g)
    theta = eye * 0.7
    theta[:, :, 2] = 0.25 * torch.randn(n, 2, generator=g)
    target = F.affine_grid(theta, (n, 1, h, h), align_corners=False) + 0.02 * torch.randn(n, h, h, 2, generator=g)
    points = torch.rand(n, p, 2, generator=g) * 2.4 - 1.2
    centers = torch.randint(-1, h + 1, (n, p, 2), generator=g)
    corners = torch.tensor([[-1, -1], [h, h], [-1, h], [h, -1]])
    k = min(4, p)
    centers[:, :k] = corners[:k]
    points[:, :k] = 0.0
    return base, target, points, centers, torch.tensor(alphas, dtype=torch.float32)


def window_positions(centers, h, patch):
    """Padded-grid positions (qy, qx) of every window candidate (N, P, patch^2) and the flat centre."""
    hp = wp = h + 2
    r = patch // 2
    flat = (centers[..., 0] + 1) + hp * (centers[..., 1] + 1)
    ly, lx = torch.div(flat, wp, rounding_mode="floor"), torch.remainder(flat, wp)
    k = torch.arange(patch * patch, device=centers.device)
    qy = ly.unsqueeze(-1) + torch.div(k, patch, rounding_mode="floor") - r
    qx = lx.unsqueeze(-1) + k % patch - r
    return qy, qx, flat


def track_labels(case):
    name, n, p, h, patch, alphas = case
    _, _, _, centers, al = track_frame0(case)
    labels = {"track: patch %d" % patch} if patch in (1, 3, 7) else set()
    qy, qx, _ = window_positions(centers, h, patch)
    inside = (qy >= 0) & (qy < h + 2) & (qx >= 0) & (qx < h + 2)
    ring = inside & ((qy == 0) | (qy == h + 1) | (qx == 0) | (qx == h + 1))
    if bool(ring.any()):
        labels.add("track: windows reach the extrapolation ring")
    if bool((~inside).any()):
        labels.add("track: windows beyond the ring (Unfold's zero candidates)")
    if patch > 1 and p >= 4:
        labels.add("track: flat-index wrap (a zero candidate beyond the padded grid is nearest)")
    if bool((centers == -1).any()) and bool((centers == h).any()):
        labels.add("track: centres at -1 and H")
    if bool((al.abs() < 0.5).any()):
        labels.add("track: lerp |w| < 0.5")
    if bool((al.abs() >= 0.5).any()):
        labels.add("track: lerp |w| >= 0.5")
    if all(bool((al == v).any()) for v in (0.0, 0.5, 1.0)):
        labels.add("track: w = 0, 0.5 and 1")
    if len(alphas) >= 3:
        labels.add("track: T >= 3 frames carrying centres")
    if track_plan(n, p)["grid"] > 1 and (n * p) % TRACK_THREADS:
        labels.add("track: N P > 128 with a partial CTA")
    return labels


REQUIRED = ["nn: one split because N pblocks >= 2 SMs", "nn: several splits, boundaries off multiples of 1024",
            "nn: several splits, boundaries on multiples of 1024",
            "nn: several tiles in a split, partial last tile", "nn: HW < 1024", "nn: HW = 1024", "nn: HW = 1025",
            "nn: partial last point block", "nn: N > 1 (blockIdx.z)", "nn: HW = 1",
            "nn: placed ties across a split boundary", "nn: placed ties across a tile seam",
            "nn: identical queries either side of a point-block boundary",
            "pck_query: one trip", "pck_query: >= 2 trips", "pck_query: query / nn_grid boundary inside a warp",
            "pck_query: similarity-only (no nn_grid)", "pck_score: A = 1", "pck_score: A = 8",
            "pck_score: visible null", "pck_score: est_out and nn_index null", "pck_score: B P not a multiple of 256",
            "track: patch 1", "track: patch 3", "track: patch 7", "track: windows reach the extrapolation ring",
            "track: windows beyond the ring (Unfold's zero candidates)",
            "track: flat-index wrap (a zero candidate beyond the padded grid is nearest)", "track: centres at -1 and H",
            "track: lerp |w| < 0.5", "track: lerp |w| >= 0.5", "track: w = 0, 0.5 and 1",
            "track: T >= 3 frames carrying centres", "track: N P > 128 with a partial CTA"]
UNREACHED = ["nn: splits capped at 65535 (splits never exceed 2 SMs: a device with more than 32767 SMs)"]


def test_cases_reach_every_route():
    reached = set()
    for case in NN_CASES + [("lattice", n, p, h * w, "random") for n, h, w, p in LATTICE_CASES]:
        reached |= nn_labels(case)
    for case in PCK_CASES:
        reached |= pck_labels(case)
    for case in TRACK_CASES:
        reached |= track_labels(case)
    assert_routes_reached(REQUIRED, reached, UNREACHED)


def test_planner_restatements():
    """The split arithmetic at its edges, every split non-empty, and the workspace formulas against the library's."""
    assert nn_plan(1, 264 * 256, 5000, H100_SMS)["splits"] == 1
    assert nn_plan(1, 1, 1, H100_SMS)["splits"] == 1 and nn_plan(1, 1, 1025, H100_SMS)["splits"] == 2
    assert nn_plan(1, 1, 10 ** 9, H100_SMS)["splits"] == 2 * H100_SMS
    for n, p, hw in ((1, 1, 1), (1, 300, 10000), (2, 12800, 5000), (1, 1, 2 * H100_SMS * NN_TILE + 1), (3, 5, 999999)):
        pl = nn_plan(n, p, hw, H100_SMS)
        assert all(e0 < e1 for e0, e1 in pl["ranges"]) and pl["ranges"][-1][1] == hw
    pl = pck_plan(4, 37, 192, True, H100_SMS)
    assert pl["qgrid"] == 8 * H100_SMS and pl["trips"] == 2 and pl["sgrid"] == 1
    lib = library().load()
    for b, p, f in ((2, 5, 64), (3, 300, 0), (4, 37, 192)):
        assert lib.gg_pck_transfer_workspace(b, p, f) == pck_plan(b, p, f, f > 0, H100_SMS)["ws"]
    assert lib.gg_nn_argmin_workspace(3, 7) == 3 * 7 * 8


# ============================================================================================ fp32 restatements (CPU/GPU)
def first_min(d):
    """torch.argmin's rule over the last dimension, stated explicitly: the first NaN if there is one, else the first
    minimum (an all-+inf row gives 0).  -> (index, minimum with NaN rows NaN)."""
    hw = d.shape[-1]
    idx = torch.arange(hw, device=d.device)
    nan = torch.isnan(d)
    m = torch.where(nan, torch.full_like(d, math.inf), d).amin(-1, keepdim=True)
    first_nan = torch.where(nan, idx, hw).amin(-1)
    first_m = torch.where(d == m, idx, hw).amin(-1)
    has_nan = nan.any(-1)
    return torch.where(has_nan, first_nan, first_m), torch.where(has_nan, math.nan, m.squeeze(-1))


def test_first_min_is_torch_argmin():
    """The restated rule is torch.argmin's on the CPU: NaN first (either sign), all +inf -> 0, ties -> first, -0.0 == 0.0."""
    nan, inf = math.nan, math.inf
    rows = [[1., nan, 0., nan], [inf, inf, inf], [3., -nan, 2., nan], [0., -0., -0.], [2., 1., 1., -inf, -inf],
            [-1e-7, 0., -1e-7], [inf, 5., inf], [nan, nan]]
    for r in rows:
        t = torch.tensor(r, dtype=torch.float32)
        assert int(first_min(t)[0]) == int(t.argmin()), r


def dist32(gx, gy, px, py):
    """The kernels' expanded distance, every op a separate fp32 torch op rounded once (no contraction)."""
    pp = px * px + py * py
    gg = gx * gx + gy * gy
    sim = gx * px + gy * py
    return (pp + gg) - 2 * sim


def dist64(gx, gy, px, py):
    """float64 |p - g|^2 of the fp32 operands and M = |p|^2 + |g|^2 + 2 (|gx px| + |gy py|)."""
    gx, gy, px, py = (t.double() for t in (gx, gy, px, py))
    d = (px - gx) ** 2 + (py - gy) ** 2
    m = px * px + py * py + gx * gx + gy * gy + 2 * ((gx * px).abs() + (gy * py).abs())
    return d, m


def order_bits(d):
    """points.cu order_bits as int64: the monotone map of an fp32 distance to 32 bits, every NaN to 0."""
    u = d.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    key = torch.where((u & 0x80000000) != 0, (~u) & 0xFFFFFFFF, u | 0x80000000)
    return torch.where(torch.isnan(d), torch.zeros_like(key), key)


# ======================================================================================================== GPU checks
WORST = Worst("ratio to the derived bound", "%-64s %.3f", kind_suffix=False)
_report_worst = WORST.fixture()


def check_bound(y, ref, bound, key, what):
    """|y - ref| <= bound per element (bound in float64); records the worst |y - ref| / bound."""
    obs = assert_fp32_sum(y, ref, bound / U32, 1, "%s: %s" % (key, what))
    WORST.note(key, obs)
    print("[contract] %s: %s: %.3f of the bound" % (key, what, obs))


def guarded(shape, dtype, fill):
    """An output of `shape` filled with `fill`, followed by GUARD elements of the same fill: (view, whole buffer)."""
    buf = torch.full((math.prod(shape) + GUARD,), fill, dtype=dtype, device=DEV)
    return buf[:math.prod(shape)].view(shape), buf


def assert_guard(buf, n, fill, what):
    tail = buf[n:]
    ok = tail.isnan().all() if isinstance(fill, float) and math.isnan(fill) else (tail == fill).all()
    assert bool(ok), "%s: a launch wrote past the end" % what


def pick_ratio(d64, e, pick, best):
    """(d_pick - d_best) / (e_pick + e_best) per row: at most 1 where the fp32 pick is within the bound of the float64
    minimum; 0 where the pick is the minimum (also where both bounds are 0: a zero candidate at a query on the origin)."""
    diff = (d64.gather(-1, pick.unsqueeze(-1)) - d64.gather(-1, best)).squeeze(-1)
    den = (e.gather(-1, pick.unsqueeze(-1)) + e.gather(-1, best)).squeeze(-1)
    return torch.where(diff == 0, 0.0, diff / den)


def check_search(grid, pts, idx, keys, what, key="nn_argmin"):
    """grid (N, HW, 2), pts (N, P, 2) fp32 on the device, idx (N, P) the kernel's indices, keys (N, P) int64 its packed
    keys or None.  Bitwise against the fp32 restatement; the float64 bound checks on finite rows.  -> restated minima."""
    n, hw, _ = grid.shape
    p = pts.shape[1]
    step = max(1, CHUNK // (n * hw))
    decided, rows, mins = 0, 0, []
    for c0 in range(0, p, step):
        q = pts[:, c0:c0 + step].unsqueeze(2)                      # (N, C, 1, 2)
        g = grid.unsqueeze(1)                                       # (N, 1, HW, 2)
        d32 = dist32(g[..., 0], g[..., 1], q[..., 0], q[..., 1])
        k32, m32 = first_min(d32)
        got = idx[:, c0:c0 + step]
        bad = got != k32
        if bool(bad.any()):
            i = torch.nonzero(bad)[0].tolist()
            raise AssertionError("%s: %d of %d indices differ from the fp32 restatement's argmin; first at (n, p) = (%d, %d): "
                                 "kernel %d, restatement %d" % (what, int(bad.sum()), bad.numel(), i[0], c0 + i[1],
                                                                int(got[i[0], i[1]]), int(k32[i[0], i[1]])))
        if keys is not None:
            kk = keys[:, c0:c0 + step]
            assert torch.equal((kk >> 32) & 0xFFFFFFFF, order_bits(m32)), "%s: a packed key's distance bits" % what
            assert torch.equal(kk & 0xFFFFFFFF, k32), "%s: a packed key's index" % what
        mins.append(m32)
        finite = torch.isfinite(d32).all(-1)
        if not bool(finite.any()):
            continue
        d64, m64 = dist64(g[..., 0], g[..., 1], q[..., 0], q[..., 1])
        e = K_D * U32 * m64 * HIGHER
        k64 = d64.argmin(-1, keepdim=True)                           # float64 ties are measure-zero here
        d_best, e_best = d64.gather(-1, k64), e.gather(-1, k64)
        ratio = torch.where(finite, pick_ratio(d64, e, got, k64), 0.0)
        assert bool((ratio <= 1).all()), "%s: a picked distance lies %.3f bounds above the float64 minimum" % (
            what, float(ratio.max()))
        lower = (d64 - e).scatter(-1, k64, math.inf).amin(-1, keepdim=True)
        dec = (lower > d_best + e_best).squeeze(-1) & finite
        assert torch.equal(got[dec], k64.squeeze(-1)[dec]), "%s: a decided row picks another entry than float64" % what
        decided += int(dec.sum())
        rows += int(finite.sum())
        WORST.note(key + ": (d_pick - d_min) / (e_pick + e_min)", float(ratio.max()))
    if rows:
        print("[contract] %s: %s: %d of %d finite rows decided by float64" % (key, what, decided, rows))
    return torch.cat(mins, 1)


def run_nn(grid, pts):
    """gg_nn_argmin with a sentinel-filled index and a NaN-filled workspace, both guarded: (index, packed keys)."""
    lib = library()
    n, hw, _ = grid.shape
    p = pts.shape[1]
    index, ibuf = guarded((n, p), torch.int64, SENTINEL)
    nbytes = lib.load().gg_nn_argmin_workspace(n, p)
    ws, wbuf = guarded((nbytes // 4,), torch.float32, math.nan)
    rc = lib.load().gg_nn_argmin(index.data_ptr(), ws.data_ptr(), grid.data_ptr(), pts.data_ptr(), n, p, hw, lib.stream())
    lib.check(rc, "gg_nn_argmin")
    torch.cuda.synchronize()
    assert_guard(ibuf, n * p, SENTINEL, "gg_nn_argmin index")
    assert_guard(wbuf, nbytes // 4, math.nan, "gg_nn_argmin workspace")
    return index, ws.view(torch.int64).view(n, p)


def nn_inputs(case, sms):
    """(grid (N, HW, 2), points (N, P, 2), placed) on the CPU; placed: [(what, n, point rows, expected index)]."""
    name, n, p, hw, kind = case
    g = torch.Generator().manual_seed(sum(map(ord, name)) + hw)
    grid = torch.rand(n, hw, 2, generator=g) * 2 - 1
    pts = torch.rand(n, p, 2, generator=g) * 2.2 - 1.1
    placed = []
    if kind != "placed":
        return grid, pts, placed
    pl = nn_plan(n, p, hw, sms)
    seams = [(e0, "split boundary") for e0, _ in pl["ranges"][1:]]
    seams += [(e0 + t * NN_TILE, "tile seam") for (e0, _), nt in zip(pl["ranges"], pl["tiles"]) for t in range(1, nt)]
    row = 0
    for j, (at, what) in enumerate(seams[:6]):
        v = torch.tensor([-0.9 + 0.3 * j, 0.8 - 0.25 * j])
        clear(grid, v, 0.02)
        grid[:, at - 1] = grid[:, at] = v                       # duplicates either side of the seam
        if row + 2 <= p:
            pts[:, row] = v + torch.tensor([1e-3, -2e-3])
            pts[:, row + 1] = v
            placed.append(("duplicates across a %s" % what, list(range(n)), [row, row + 1], at - 1))
            row += 2
    if pl["splits"] > 1 and row + 1 <= p:
        # mirror entries (+-a, b) about a query on the y axis: bitwise equal distances in two splits
        (e0a, _), (e0b, _) = pl["ranges"][0], pl["ranges"][-1]
        v = torch.tensor([0.0, -0.45])
        clear(grid, v, 0.05)
        grid[:, e0a + 3] = torch.tensor([-0.004, -0.447])
        grid[:, e0b + 1] = torch.tensor([0.004, -0.447])
        pts[:, row] = v
        placed.append(("mirror entries +-g in two splits", list(range(n)), [row], e0a + 3))
        row += 1
        # queries on clustered entries, one entry per split: the expanded distance rounds negative
        c = torch.tensor([0.61, 0.73])
        clear(grid, c, 0.05)
        at = [e0 + 5 + i for e0, _ in pl["ranges"][:8] for i in range(3)]
        for j, a in enumerate(at):
            grid[:, a] = c + torch.tensor([(j * 7 % 11) * 1e-5, -(j * 5 % 13) * 1e-5])
            if row < p:
                pts[:, row] = grid[0, a]
                row += 1
        placed.append(("queries on clustered entries across splits (negative distances)", list(range(n)),
                       list(range(row - len(at), row)), None))
    if p > NN_THREADS:
        pts[:, NN_THREADS] = pts[:, NN_THREADS - 1]             # identical queries either side of a point-block boundary
        placed.append(("identical queries either side of a point-block boundary", list(range(n)),
                       [NN_THREADS - 1, NN_THREADS], "same"))
    return grid, pts, placed


def clear(grid, v, radius):
    """Move every entry within `radius` of v out to distance >= 3 radius, so that placed entries near v stand alone."""
    off = grid - v
    near = off.norm(dim=-1) < radius
    grid[near] = v + torch.tensor([3 * radius, 3 * radius])


@pytest.mark.gpu
@pytest.mark.parametrize("case", NN_CASES, ids=lambda c: c[0])
def test_nn_argmin(case):
    name, n, p, hw, kind = case
    sms = library().sm_count()
    grid, pts, placed = (t.to(DEV) if torch.is_tensor(t) else t for t in nn_inputs(case, sms))
    idx, keys = run_nn(grid, pts)
    assert bool(((idx >= 0) & (idx < hw)).all())
    mins = check_search(grid, pts, idx, keys, name)
    for what, ns, rows, want in placed:
        got = idx[ns][:, rows]
        if want == "same":
            assert bool((got[:, 0] == got[:, 1]).all()), "%s: %s" % (name, what)
        elif want is None:
            m = mins[ns][:, rows]
            assert bool((m < 0).any()), "%s: %s: no distance rounded negative" % (name, what)
            assert bool((got >= nn_plan(n, p, hw, sms)["per"]).any()), "%s: %s: no pick outside split 0" % (name, what)
        else:
            assert bool((got == want).all()), "%s: %s: picked %s, the first entry is %d" % (name, what, got.tolist(), want)
        print("[placed] %s: %s: indices %s" % (name, what, sorted(set(got.flatten().tolist()))))


@pytest.mark.gpu
def test_nn_argmin_on_jittered_lattices():
    """congeal_points' search on what it is given in use: sampling grids near a lattice over [-1, 1]^2 (16 x 16, 128 x 128
    in 16 splits, 24 x 40 with one point per sample), bitwise against the fp32 restatement and within the float64 bound;
    and an all-zero 4 x 4 grid, where every distance to the origin is 0 and index 0 wins."""
    g = torch.Generator().manual_seed(8)
    for n, h, w, p in LATTICE_CASES:
        ys, xs = torch.meshgrid(torch.linspace(-1, 1, h), torch.linspace(-1, 1, w), indexing="ij")
        grid = torch.stack([xs, ys], -1)[None].repeat(n, 1, 1, 1) + 0.05 * torch.randn(n, h, w, 2, generator=g)
        pts = torch.rand(n, p, 2, generator=g) * 2 - 1
        grid, pts = grid.reshape(n, h * w, 2).contiguous().to(DEV), pts.to(DEV)
        idx, keys = run_nn(grid, pts)
        check_search(grid, pts, idx, keys, "lattice %dx%d, N = %d, P = %d" % (h, w, n, p))
    idx, keys = run_nn(torch.zeros(1, 16, 2, device=DEV), torch.zeros(1, 1, 2, device=DEV))
    assert idx.tolist() == [[0]] and int(keys[0, 0]) & 0xFFFFFFFF == 0


@pytest.mark.gpu
def test_nn_argmin_non_finite_rows_follow_argmin():
    """A NaN query, a point with |p|^2 = +inf, NaN entries (either sign) in later splits than a finite minimum, an all-NaN
    grid: each index equals argmin of the restated distances and lies in [0, HW)."""
    n, p, hw = 3, 40, 3000                                 # 3 splits of 1000 entries
    g = torch.Generator().manual_seed(5)
    grid = torch.rand(n, hw, 2, generator=g) * 2 - 1
    pts = torch.rand(n, p, 2, generator=g) * 2 - 1
    nan = float("nan")
    pts[0, 3] = torch.tensor([nan, 0.2])
    pts[0, 4] = torch.tensor([0.1, nan])
    pts[0, 5] = torch.tensor([1e20, 0.3])                  # |p|^2 = +inf: every distance +inf -> index 0
    grid[1, 2500] = torch.tensor([0.3, nan])
    grid[1, 1200] = -torch.tensor([nan, nan])              # a negative NaN, earlier: it wins
    grid[2] = nan
    grid, pts = grid.to(DEV), pts.to(DEV)
    idx, keys = run_nn(grid, pts)
    assert bool(((idx >= 0) & (idx < hw)).all()), "an index outside [0, HW): %s" % idx[(idx < 0) | (idx >= hw)].tolist()
    check_search(grid, pts, idx, keys, "non-finite rows")
    assert idx[0, 3:6].tolist() == [0, 0, 0] and bool((idx[1] == 1200).all()) and bool((idx[2] == 0).all())


# ------------------------------------------------------------------------------------------------------- PCK-Transfer
def pck_inputs(case):
    """Seeded inputs of one gg_pck_transfer call on the CPU: smooth random flows around the identity, random similarity
    matrices; row i's destination is row i + 1's source."""
    name, b, p, a, s, f, visible, outputs = case
    g = torch.Generator().manual_seed(sum(map(ord, name)) + b * p)
    ang = (torch.rand(b, generator=g) - 0.5) * 1.0
    sc = torch.rand(b, generator=g) * 0.5 + 0.8
    m = torch.stack([sc * torch.cos(ang), -sc * torch.sin(ang), (torch.rand(b, generator=g) - 0.5) * 0.3,
                     sc * torch.sin(ang), sc * torch.cos(ang), (torch.rand(b, generator=g) - 0.5) * 0.3], 1).view(b, 2, 3)
    pts = torch.rand(b, p, 2, generator=g) * (s - 9) + 4
    gt = pts + torch.randn(b, p, 2, generator=g) * 8
    vis = (torch.rand(b, p, generator=g) > 0.25).float() if visible else None
    thresh = torch.rand(b, generator=g) * 60 + 40
    alphas = torch.tensor([0.1, 0.05, 0.01, 0.2, 0.15, 0.3, 0.02, 0.5])[:a]
    kw = dict(matrix_dst=torch.roll(m, 1, 0).contiguous())
    if f:
        ident = F.affine_grid(torch.eye(2, 3)[None], (1, 1, f, f), align_corners=False)
        low = torch.randn(b, 2, 8, 8, generator=g) * 0.06
        delta = F.interpolate(low, size=(f, f), mode="bicubic", align_corners=False).permute(0, 2, 3, 1)
        grid_dst = torch.roll(delta, 1, 0) + F.affine_grid(torch.roll(m, 1, 0), (b, 1, f, f), align_corners=False)
        kw = dict(delta_src=delta.contiguous(), identity=ident.contiguous(), grid_dst=grid_dst.contiguous())
    return dict(points=pts, gt=gt, visible=vis, thresh=thresh, alphas=alphas, matrix_src=m.contiguous(), size=s, **kw)


def run_pck(inp, with_outputs=True):
    """gg_pck_transfer with guarded outputs and a NaN-filled guarded workspace: (counts, est, nn_index, workspace)."""
    lib = library()
    pts = inp["points"]
    b, p = pts.shape[:2]
    a = inp["alphas"].numel()
    delta = inp.get("delta_src")
    f = delta.shape[1] if delta is not None else 0
    counts, cbuf = guarded((a,), torch.int64, 0)
    est, ebuf = guarded((b, p, 2), torch.float32, math.nan)
    nn, nbuf = guarded((b, p), torch.int64, SENTINEL)
    nbytes = lib.load().gg_pck_transfer_workspace(b, p, f)
    ws, wbuf = guarded((nbytes // 4,), torch.float32, math.nan)
    ptr = lib.ptr
    rc = lib.load().gg_pck_transfer(counts.data_ptr(), est.data_ptr() if with_outputs else None,
                                    nn.data_ptr() if with_outputs and f else None, ws.data_ptr(), pts.data_ptr(),
                                    inp["gt"].data_ptr(), ptr(inp["visible"]), inp["thresh"].data_ptr(),
                                    inp["alphas"].data_ptr(), inp["matrix_src"].data_ptr(), ptr(inp.get("matrix_dst")),
                                    ptr(delta), ptr(inp.get("identity")), ptr(inp.get("grid_dst")), b, p, a, inp["size"],
                                    f, f, f, lib.stream())
    lib.check(rc, "gg_pck_transfer")
    torch.cuda.synchronize()
    assert_guard(cbuf, a, 0, "counts")
    assert_guard(ebuf, b * p * 2, math.nan, "est_points")
    assert_guard(nbuf, b * p if with_outputs and f else 0, SENTINEL, "nn_index")
    assert_guard(wbuf, nbytes // 4, math.nan, "workspace")
    if not (with_outputs and f):
        assert bool((nn == SENTINEL).all()), "nn_index written although null or similarity-only"
    if not with_outputs:
        assert bool(est.isnan().all()), "est_points written although null"
    return counts, est, nn, ws


def workspace_parts(ws, b, p, f):
    pl = pck_plan(b, p, f, f > 0, H100_SMS)
    raw = ws.view(torch.uint8)
    part = lambda k: raw[pl[k][0]:pl[k][1]]
    keys = part("best").view(torch.int64).view(b, p)
    query = part("query").view(torch.float32).view(b, p, 2)
    nn_grid = part("nn_grid").view(torch.float32).view(b, f * f, 2) if f else None
    return keys, query, nn_grid


def normalize32(v, res_m1, k):
    """pck.cu normalize1 in numpy fp32: v.div(res - 1).add(-0.5).mul(2).mul(k), each op rounded once."""
    v = np.asarray(v, dtype=np.float32)
    return ((v / np.float32(res_m1) + np.float32(-0.5)) * np.float32(2)) * np.float32(k)


def unnormalize32(v, k, res_m1):
    """pck.cu unnormalize1 in numpy fp32: v.div(k).div(2).add(0.5).mul(res - 1)."""
    v = np.asarray(v, dtype=np.float32)
    return ((v / np.float32(k)) / np.float32(2) + np.float32(0.5)) * np.float32(res_m1)


def query_bound(points, m, s, flow):
    """float64 congeal_query_ref and the bound on the kernel's fp32 query, first order in u = 2^-24 (x HIGHER):
      normalize1   x = ((v / (S-1) - 0.5) 2) k_32: u (2k |t| + 2k |t - 0.5| + |x|), t = v / (S-1), and u |x| more for
                   k_32 = fl((S-1)/S) against the float64 (S-1)/S;
      the inverse  each entry of the double 2x2 inverse rounded once to fp32, u |I|, plus 2^-48 (sum of the |products|) |r|
                   for the double arithmetic (contracted or not: DESIGN.md section 2 deviation (11) states why the kernel
                   forms the inverse analytically and where that differs from the reference's fp32 torch.inverse);
      the apply    (x i00 + y i01) + i02: u (3 |x i00| + 3 |y i01| + |i02|) and the propagated input errors;
      flow         the un-normalise / normalise round trip (identity in exact arithmetic with the same k_32 both ways):
                   u (6 |w| + 3 k) at w."""
    k = (s - 1) / s
    v = points.double()
    ref = OP.congeal_query_ref(v, m.double(), s, flow)
    t = v / (s - 1)
    x = (t - 0.5) * 2 * k
    dx = U32 * (2 * k * (t.abs() + (t - 0.5).abs()) + 2 * x.abs())
    md = m.double()
    a_, b_, c_, d_, e_, f_ = (md[:, 0, 0], md[:, 0, 1], md[:, 0, 2], md[:, 1, 0], md[:, 1, 1], md[:, 1, 2])
    r = 1 / (a_ * e_ - b_ * d_)
    inv = torch.stack([torch.stack([e_ * r, -b_ * r, (b_ * f_ - e_ * c_) * r], -1),
                       torch.stack([-d_ * r, a_ * r, (d_ * c_ - a_ * f_) * r], -1)], 1)        # (B, 2, 3)
    eps = 2.0 ** -48 * (a_.abs() * e_.abs() + b_.abs() * d_.abs() + (b_ * f_).abs() + (e_ * c_).abs() + (d_ * c_).abs()
                        + (a_ * f_).abs() + a_.abs() + b_.abs() + d_.abs() + e_.abs()) * r.abs()
    dinv = U32 * inv.abs() + eps.view(-1, 1, 1)
    bounds = []
    for row in range(2):
        i0, i1, i2 = (inv[:, row, j].view(-1, 1) for j in range(3))
        d0, d1, d2 = (dinv[:, row, j].view(-1, 1) for j in range(3))
        x0, x1 = x[..., 0], x[..., 1]
        w = x0 * i0 + x1 * i1 + i2
        bd = (i0.abs() * dx[..., 0] + i1.abs() * dx[..., 1] + x0.abs() * d0 + x1.abs() * d1 + d2
              + U32 * (3 * (x0 * i0).abs() + 3 * (x1 * i1).abs() + i2.abs()))
        if flow:
            bd = bd + U32 * (6 * w.abs() + 3 * k)
        bounds.append(bd * HIGHER + 2.0 ** -50 * (w.abs() + 1))          # + the float64 reference's own rounding
    return ref, torch.stack(bounds, -1)


def lookup_bound(grid, qn, k, m):
    """float64 lookup_point (grid_sample 'border', align_corners=False + unnormalise with the fp32 k and m) at the fp32
    query qn (B, P, 2), and its bound on the kernel's fp32 evaluation, first order (x HIGHER):
      ix = ((q + 1) gw - 1) / 2 rounds at most three times (the multiply-subtract may contract): |dix| <= u (gw |q + 1| +
      |ix|); the lookup is Lipschitz in ix with the sample's largest neighbour difference L; the weights carry <= 3
      roundings (one in (fx + 1) - ix, one in the product; ix - fx is exact), the 4-term fma chain 4: 7 u sum |v| w;
      unnormalise adds u m (|o| / (2k) + 0.5) for each of / k, + 0.5, * m and scales the lookup's error by m / (2k)."""
    b, gh, gw, _ = grid.shape
    g64 = grid.double()
    q = qn.double()
    res, mags = [], []
    for gv in (g64, g64.abs()):
        o = F.grid_sample(gv.permute(0, 3, 1, 2), q.unsqueeze(2), padding_mode="border", align_corners=False)
        res.append(o.squeeze(3).permute(0, 2, 1))
    o, oa = res
    est = ((o / k) / 2 + 0.5) * m
    lx = (g64[:, :, 1:] - g64[:, :, :-1]).abs().amax((1, 2)).view(b, 1, 2)
    ly = (g64[:, 1:] - g64[:, :-1]).abs().amax((1, 2)).view(b, 1, 2)
    ix = (((q[..., 0] + 1) * gw - 1) / 2).clamp(0, gw - 1)
    iy = (((q[..., 1] + 1) * gh - 1) / 2).clamp(0, gh - 1)
    dix = U32 * (gw * (q[..., 0] + 1).abs() + ix)
    diy = U32 * (gh * (q[..., 1] + 1).abs() + iy)
    do = 7 * U32 * oa + lx * dix.unsqueeze(-1) + ly * diy.unsqueeze(-1)
    bound = (m / (2 * k) * do + 3 * U32 * m * (o.abs() / (2 * k) + 0.5)) * HIGHER
    return est, bound


def counts32(est, gt, visible, thresh, alphas):
    """pck_score's test in numpy fp32 on the kernel's est: vis && sqrt(dx dx + dy dy) <= alpha * thresh per alpha."""
    est, gt = est.cpu().numpy(), gt.cpu().numpy()
    dx, dy = est[..., 0] - gt[..., 0], est[..., 1] - gt[..., 1]
    err = np.sqrt(dx * dx + dy * dy)
    vis = np.ones(err.shape, bool) if visible is None else visible.cpu().numpy() != 0
    th = thresh.cpu().numpy()
    out = []
    for a in alphas.cpu().numpy():
        thr = (np.float32(a) * th).astype(np.float32)
        out.append(int((vis & (err <= thr[:, None])).sum()))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", PCK_CASES, ids=lambda c: c[0])
def test_pck_transfer(case):
    name, b, p, a, s, f, visible, outputs = case
    inp = {k: v.to(DEV) if torch.is_tensor(v) else v for k, v in pck_inputs(case).items()}
    counts, est, nn, ws = run_pck(inp)
    keys, query, nn_grid = workspace_parts(ws, b, p, f)
    ks = f32((s - 1) / s)
    # query, against float64
    ref, bound = query_bound(inp["points"].cpu(), inp["matrix_src"].cpu(), s, f > 0)
    check_bound(query.cpu(), ref, bound, "pck query (flow)" if f else "pck query (similarity)", name)
    if f:
        assert torch.equal(nn_grid, (inp["delta_src"] + inp["identity"]).view(b, f * f, 2)), "%s: nn_grid" % name
        assert bool(((nn >= 0) & (nn < f * f)).all())
        check_search(nn_grid, query, nn, keys, name, key="pck nn_index")
        ix = (nn % f).cpu().numpy().astype(np.float32)
        iy = (nn // f).cpu().numpy().astype(np.float32)
        qn = torch.from_numpy(np.stack([normalize32(ix, f - 1, ks), normalize32(iy, f - 1, ks)], -1))
        e64, eb = lookup_bound(inp["grid_dst"].cpu(), qn, ks, float(s - 1))
        check_bound(est.cpu(), e64, eb, "pck est (flow lookup)", name)
    else:
        assert bool(keys.view(torch.float32).isnan().all()), "%s: the search's workspace was written" % name
        q = query.cpu().numpy()
        md = inp["matrix_dst"].cpu().numpy()
        want = np.empty_like(q)
        for j in range(2):
            lin = (q[..., 0] * md[:, j, 0:1] + q[..., 1] * md[:, j, 1:2]) + md[:, j, 2:3]
            want[..., j] = unnormalize32(lin, ks, s - 1)
        assert np.array_equal(est.cpu().numpy(), want), "%s: est differs from the closed form on the kernel's query" % name
    want = counts32(est, inp["gt"], inp["visible"], inp["thresh"], inp["alphas"])
    assert counts.tolist() == want, "%s: counts %s, fp32 restatement %s" % (name, counts.tolist(), want)
    print("[pck] %s: counts %s of %d points" % (name, want, b * p))
    again = run_pck(inp, with_outputs=outputs == "all")
    assert torch.equal(again[0], counts), "%s: counts differ between two calls" % name
    if outputs == "all":
        assert torch.equal(again[1], est) and torch.equal(again[2], nn)


@pytest.mark.gpu
def test_pck_transfer_never_returns_a_negative_index():
    """Non-finite queries and grids through pck_transfer_points: a NaN source point, a NaN flow entry, a source point so
    large that |q|^2 overflows.  nn_index is argmin of the restated distances, in [0, F^2)."""
    from gangealing_b200.evaluation.ops import pck_transfer_points
    case = ("non-finite", 3, 20, 3, 128, 32, True, "all")
    inp = pck_inputs(case)
    inp["points"][0, 2] = float("nan")
    inp["points"][1, 3] = 1e37
    inp["delta_src"][2, 20, 5, 0] = float("nan")
    inp = {k: v.to(DEV) if torch.is_tensor(v) else v for k, v in inp.items()}
    counts, est, nn = pck_transfer_points(**inp)
    assert bool(((nn >= 0) & (nn < 32 * 32)).all()), nn[(nn < 0) | (nn >= 32 * 32)].tolist()
    _, _, _, ws = run_pck(inp)
    keys, query, nn_grid = workspace_parts(ws, 3, 20, 32)
    check_search(nn_grid, query, nn, keys, "non-finite", key="pck nn_index")
    assert int(nn[2, 0]) == 20 * 32 + 5


# -------------------------------------------------------------------------------------------------------------- tracker
def fma32(a, b, c):
    """fmaf(a, b, c) on fp32 tensors, exactly: the float64 product of two fp32 values is exact; the sum by TwoSum,
    rounded to odd in float64 (53 >= 24 + 2 bits), then rounded once to fp32."""
    pr = a.double() * b.double()
    cd = c.double()
    s = pr + cd
    bb = s - pr
    err = (pr - (s - bb)) + (cd - bb)
    inexact = (err != 0) & torch.isfinite(s)
    even = (s.view(torch.int64) & 1) == 0
    odd = torch.nextafter(s, torch.where(err > 0, math.inf, -math.inf))
    return torch.where(inexact & even, odd, s).float()


def round32(q):
    """The fp32 value nearest the Fraction q, ties to even."""
    lo = np.float32(float(q))
    cands = [lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))]
    return min(cands, key=lambda v: (abs(Fraction(float(v)) - q), int(np.float32(v).view(np.int32)) & 1))


def test_fma32_rounds_once():
    """fmaf's single rounding, where a float64 multiply-add rounded to fp32 rounds twice: (1 + 2^-12)^2 + 2^-80 is
    1 + 2^-11 + 2^-24 + 2^-80, just above the midpoint of two fp32 values, but its float64 sum is the midpoint itself and
    then rounds to even, one ulp low.  And random operands against exact rational arithmetic."""
    a = torch.tensor([1 + 2.0 ** -12], dtype=torch.float32)
    c = torch.tensor([2.0 ** -80], dtype=torch.float32)
    assert float(fma32(a, a, c)) == 1 + 2.0 ** -11 + 2.0 ** -23
    assert float((a.double() * a.double() + c.double()).float()) == 1 + 2.0 ** -11        # the double rounding
    rng = np.random.default_rng(3)
    x, y = (torch.from_numpy(rng.standard_normal(4000).astype(np.float32)) for _ in range(2))
    z = torch.from_numpy((rng.standard_normal(4000) * 10.0 ** rng.integers(-8, 2, 4000)).astype(np.float32))
    got = fma32(x, y, z)
    for i in range(4000):
        q = Fraction(float(x[i])) * Fraction(float(y[i])) + Fraction(float(z[i]))
        assert float(got[i]) == float(round32(q)), i


def lerp32(a, b, w):
    """points.cu lerp_aten: d = b - a; |w| < 0.5 ? fmaf(w, d, a) : fmaf(-d, 1 - w, b), w an fp32 scalar tensor."""
    d = b - a
    wt = torch.full_like(a, float(w))
    return torch.where(wt.abs() < 0.5, fma32(wt, d, a), fma32(-d, 1 - wt, b))


def track_step32(base, target, w, points, centers, patch):
    """One frame of track_points_kernel restated in fp32 from the given centres: the candidates' distances (N, P, K)
    bitwise the kernel's, the first minimum and the next centres with the wrap."""
    n, h, _, _ = base.shape
    hp = wp = h + 2
    r = patch // 2
    grid = OV.pad_grid(lerp32(base, target, w))                       # 2 a - b: the product exact, the difference rounded
    qy, qx, flat = window_positions(centers, h, patch)
    inside = (qy >= 0) & (qy < hp) & (qx >= 0) & (qx < wp)
    lin = (qy.clamp(0, hp - 1) * wp + qx.clamp(0, wp - 1)).view(n, -1)
    cand = grid.reshape(n, hp * wp, 2).gather(1, lin.unsqueeze(-1).expand(-1, -1, 2)).view(*qy.shape, 2)
    cand = torch.where(inside.unsqueeze(-1), cand, torch.zeros_like(cand))    # Unfold's zero padding
    px, py = points[..., 0:1], points[..., 1:2]
    d = dist32(cand[..., 0], cand[..., 1], px, py)
    k, _ = first_min(d)
    out = flat + (k % patch - r) + hp * (torch.div(k, patch, rounding_mode="floor") - r)
    nxt = torch.stack([torch.remainder(out, wp) - 1,
                       torch.remainder(torch.div(out, wp, rounding_mode="floor"), hp) - 1], -1)
    return nxt, k, d, cand, out


def run_track(base, target, alphas, points, centers, patch):
    lib = library()
    t, (n, p) = alphas.numel(), points.shape[:2]
    h = base.shape[1]
    track, tbuf = guarded((t, n, p, 2), torch.int64, SENTINEL)
    c, cb = guarded((n, p, 2), torch.int64, SENTINEL)
    c.copy_(centers)
    rc = lib.load().gg_track_points_lerp(track.data_ptr(), c.data_ptr(), base.data_ptr(), target.data_ptr(),
                                         alphas.data_ptr(), points.data_ptr(), t, n, p, h, h, patch, lib.stream())
    lib.check(rc, "gg_track_points_lerp")
    torch.cuda.synchronize()
    assert_guard(tbuf, t * n * p * 2, SENTINEL, "track")
    assert_guard(cb, n * p * 2, SENTINEL, "centers")
    return track, c


def check_track(case, base, target, alphas, points, centers, track, c_out, what):
    name, n, p, h, patch, _ = case
    prev = centers
    wraps = 0
    for t in range(alphas.numel()):
        nxt, k, d, cand, out = track_step32(base, target, float(alphas[t]), points, prev, patch)
        bad = (track[t] != nxt).any(-1)
        if bool(bad.any()):
            i = torch.nonzero(bad)[0].tolist()
            raise AssertionError("%s frame %d: %d of %d points differ from the fp32 restatement; first (n, p) = %s: kernel %s,"
                                 " restatement %s" % (what, t, int(bad.sum()), bad.numel(), i, track[t][i[0], i[1]].tolist(),
                                                      nxt[i[0], i[1]].tolist()))
        wraps += int(((out < 0) | (out >= (h + 2) ** 2)).sum())
        finite = torch.isfinite(d).all(-1)
        d64, m64 = dist64(cand[..., 0], cand[..., 1], points[..., 0:1], points[..., 1:2])
        e = K_D * U32 * m64 * HIGHER
        ratio = torch.where(finite, pick_ratio(d64, e, k, d64.argmin(-1, keepdim=True)), 0.0)
        assert bool((ratio <= 1).all()), "%s frame %d: a picked distance %.3f bounds above the float64 minimum" % (
            what, t, float(ratio.max()))
        WORST.note("track: (d_pick - d_min) / (e_pick + e_min)", float(ratio.max()))
        prev = track[t]
    assert torch.equal(c_out, track[-1]), "%s: the returned centres are not the last frame's" % what
    return wraps


@pytest.mark.gpu
@pytest.mark.parametrize("case", TRACK_CASES, ids=lambda c: c[0])
def test_track_points(case):
    """Every frame of two stages (the centres carried from the first to the second), bitwise against the fp32
    restatement from the kernel's own previous centres."""
    name, n, p, h, patch, _ = case
    base, target, points, centers, alphas = (t.to(DEV) for t in track_frame0(case))
    stage2 = (target + 0.05 * torch.randn(target.shape, generator=torch.Generator().manual_seed(9)).to(DEV)).contiguous()
    wraps = 0
    c = centers
    for b, tg in ((base, target), (target, stage2)):
        track, c_out = run_track(b, tg, alphas, points, c, patch)
        wraps += check_track(case, b, tg, alphas, points, c, track, c_out, name)
        c = c_out
    if patch > 1 and p >= 4:
        assert wraps > 0, "%s: no frame wrapped the flat index" % name
    print("[track] %s: %d wrapped picks" % (name, wraps))


@pytest.mark.gpu
def test_track_points_non_finite_candidates_follow_argmin():
    """A NaN grid entry inside a window is picked as argmin picks the first NaN (the rest of the window finite); a NaN
    point picks the first candidate; a point with |p|^2 = +inf picks the first candidate."""
    case = ("non-finite", 2, 40, 12, 5, (0.0, 0.3, 0.8))
    base, target, points, centers, alphas = track_frame0(case)
    base[0, 5, 6] = float("nan")                       # padded position (6, 7)
    target[0, 5, 6] = float("nan")
    centers[0, 10:20] = torch.tensor([6, 5])           # windows around padded (6, 7) -> (y, x) = (6, 7)
    points[1, 7] = torch.tensor([float("nan"), 0.1])
    points[1, 8] = torch.tensor([3e19, 0.1])
    base, target, points, centers, alphas = (t.to(DEV) for t in (base, target, points, centers, alphas))
    track, c_out = run_track(base, target, alphas, points, centers, 5)
    check_track(case, base, target, alphas, points, centers, track, c_out, "non-finite")
    assert bool((track[0, 0, 10:20] == torch.tensor([6, 5], device=DEV)).all()), track[0, 0, 10:20].tolist()


# ------------------------------------------------------------------------------------------------------------ launches
KERNELS = re.compile(r"nn_init_kernel|nn_argmin_kernel|nn_unpack_kernel|pck_query_kernel|pck_score_kernel|"
                     r"track_points_kernel")


@pytest.mark.gpu
def test_each_entry_launches_its_kernels():
    """gg_nn_argmin: init, search, unpack; gg_pck_transfer: query, init, search, score with a flow and query, score
    without; gg_track_points_lerp: the tracker."""
    run_fresh("test_points_family_gpu", "check_launches")


def check_launches():
    lib = library()
    grid, pts = torch.zeros(1, 100, 2, device=DEV), torch.zeros(1, 10, 2, device=DEV)
    idx = torch.empty(1, 10, dtype=torch.int64, device=DEV)
    ws = torch.empty(10, dtype=torch.int64, device=DEV)
    calls = [("gg_nn_argmin", lambda: lib.check(lib.load().gg_nn_argmin(idx.data_ptr(), ws.data_ptr(), grid.data_ptr(),
                                                                         pts.data_ptr(), 1, 10, 100, lib.stream()), "nn"),
              ["nn_init_kernel", "nn_argmin_kernel", "nn_unpack_kernel"])]
    for case, want in ((PCK_CASES[0], ["pck_query_kernel", "nn_init_kernel", "nn_argmin_kernel", "pck_score_kernel"]),
                       (PCK_CASES[4], ["pck_query_kernel", "pck_score_kernel"])):
        inp = {k: v.to(DEV) if torch.is_tensor(v) else v for k, v in pck_inputs(case).items()}
        calls.append(("gg_pck_transfer %s" % case[0], lambda inp=inp: run_pck(inp), want))
    tc = TRACK_CASES[1]
    b, tg, pt, ce, al = (t.to(DEV) for t in track_frame0(tc))
    calls.append(("gg_track_points_lerp", lambda: run_track(b, tg, al, pt, ce, tc[4]), ["track_points_kernel"]))
    for what, fn, want in calls:
        got = launched(fn, KERNELS)
        assert got == want, "%s launched %s, expected %s" % (what, got, want)
    print("[launch] %d entries launched exactly their kernels" % len(calls))
