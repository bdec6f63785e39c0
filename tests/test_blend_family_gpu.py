"""Laplacian blending (csrc/blend.cu) against float64, over its launch plans.

  blend_level_kernel<NC, MODE>   one 32 x 64 output tile of one sample per CTA, grid (ceil(W/32), ceil(H/64), N); NC =
                                 ceil(width / 8) pads the taps to P = 8 NC (zero taps).  Per plane (mask, then A_c, B_c):
                                 stage the tile and a P-1 halo in shared memory (clamped for MODE 0 / 1, zero-padded for
                                 MODE 2), a horizontal pass of 8 columns per thread, a vertical pass of 8 rows per thread,
                                 then the level's epilogue.  MODE 0 (BL_FWD) adds the level's lerp to `out`; MODE 1
                                 (BL_BWD_SWEEP) keeps the mask stack and the mask's direct gradient d_l; MODE 2 (BL_ADJ) is
                                 one Horner step of the adjoint, with the border fold (tap prefix sums) on the first and
                                 last row / column.  Past 48 KB of shared memory (NC >= 6) the launch sets the opt-in
                                 attribute.
  blend_adj_init_kernel          U_{L-1} = g c_{L-1}
  blend_lerp_kernel              levels == 1: out = lerp(img0, img1, mask)
  blend_lerp_bwd_kernel          levels == 1: g (1 - m), g m and sum_c g (b - a)

This file restates the host plan in Python (launch_level's instantiation, level_smem_bytes, the grid, both entries'
ping-pong buffers and workspace formulas), labels every case with the routes it takes and asserts on a machine without a
GPU that the cases reach every label.  The GPU half calls the two entries through the C ABI with NaN-filled outputs and a
NaN guard past the workspace, and checks every element against float64 evaluated with the STORED fp32 taps (the float64
reference of oracle/blend.py and its autograd):
    |y - ref| <= c * 2^-24 * A                                   (assert_fp32_sum)
A is the same computation on magnitudes (stacks of |img0|, |img1|, the mask's lerp weights bounded by 1, |g|), and c is
derived next to each check from the kernel's order of operations.  The taps are positive, so a blur is non-expansive on
magnitudes and an error made at one level reaches the next at most as large, relative to the magnitude stack.  No pixel is
exempt and borders take no scale of their own.  levels == 1 is checked bitwise.

Every check prints its worst observed c (`[contract] ...` lines with `pytest -s`), and the module prints the worst per
path when it finishes.
"""
import re

import pytest
import torch

from fp64_contract import (DEV, Worst, assert_routes_reached, ceil_div, launched, library, nan_at, run_fresh)
from oracle import blend as OB

TW, TH = 32, 64                  # blend.cu kTW, kTH
MAX_WIDTH = 63                   # kMaxWidth
STATIC_SMEM = 48 * 1024
GUARD = 1024                     # NaN floats past the workspace
BL_FWD, BL_SWEEP, BL_ADJ = 0, 1, 2
MODE_NAME = {BL_FWD: "fwd", BL_SWEEP: "sweep", BL_ADJ: "adj"}


# ======================================================================================== planner restatement (no GPU)
def nc_of(width):
    """launch_level's switch: the tap count padded to P = 8 NC."""
    return min(ceil_div(width, 8), 8)


def level_smem_bytes(nc):
    p = 8 * nc
    hrows = TH + p - 1
    return 4 * (hrows * (TW + p) + hrows * TW + p)


def level_grid(n, h, w):
    return ceil_div(w, TW), ceil_div(h, TH), n


def workspace_bytes(n, c, h, w, levels, backward):
    """gg_laplacian_blend_workspace."""
    if n <= 0 or c <= 0 or h <= 0 or w <= 0 or levels <= 1:
        return 0
    plane = n * h * w
    if not backward:
        return 4 * 2 * (2 * c + 1) * plane
    return 4 * (4 * c * plane + (2 * levels - 1) * plane)


def forward_buffers(n, c, h, w, levels):
    """The workspace ranges (first float, floats) each forward launch writes, in launch order: pa / pb / pm[l & 1]."""
    total, plane = n * c * h * w, n * h * w
    pa, pb, pm = [0, total], [2 * total, 3 * total], [4 * total, 4 * total + plane]
    out = []
    for l in range(levels - 1):
        out += [(pa[l & 1], total), (pb[l & 1], total), (pm[l & 1], plane)]
        if l:
            out += [(pa[(l - 1) & 1], total), (pb[(l - 1) & 1], total), (pm[(l - 1) & 1], plane)]
    return out


def backward_buffers(n, c, h, w, levels):
    """The workspace ranges the backward's sweep, adjoint init and Horner steps address."""
    total, plane = n * c * h * w, n * h * w
    pa, pb = [0, total], [2 * total, 3 * total]
    mstack = 4 * total
    dstack = mstack + (levels - 1) * plane
    out = []
    for l in range(levels - 1):
        out += [(pa[l & 1], total), (pb[l & 1], total), (mstack + l * plane, plane), (dstack + l * plane, plane),
                (dstack + (levels - 1) * plane, plane)]
        if l:
            out += [(pa[(l - 1) & 1], total), (pb[(l - 1) & 1], total), (mstack + (l - 1) * plane, plane)]
    out += [(pa[0], total), (pb[0], total)]
    cur = 0
    for l in range(levels - 2, -1, -1):
        out += [(pa[cur], total), (pb[cur], total), (dstack + (l + 1) * plane, plane), (dstack + l * plane, plane)]
        if l:
            out += [(pa[cur ^ 1], total), (pb[cur ^ 1], total)]
        cur ^= 1
    return out


def launches(levels, width, backward):
    """Kernel names one entry call launches, in order."""
    if levels == 1:
        return ["blend_lerp_bwd_kernel" if backward else "blend_lerp_kernel"]
    nc = nc_of(width)
    if not backward:
        return ["blend_level_kernel<%d, %d>" % (nc, BL_FWD)] * (levels - 1)
    return (["blend_level_kernel<%d, %d>" % (nc, BL_SWEEP)] * (levels - 1) + ["blend_adj_init_kernel"]
            + ["blend_level_kernel<%d, %d>" % (nc, BL_ADJ)] * (levels - 1))


# ------------------------------------------------------------------------------------------------------------- cases
# (levels, width, sigma, level_sigma_multiplier, N, C, H, W); the taps are the product's level_taps(levels, width, sigma,
# 0, multiplier).  The old presets first: laplacian, laplacian_light, and the custom (width 11 + adder 2 = 13, sigma
# multiplier 1.5) configuration, over the shapes the forward and gradient sweeps of test_laplacian_blend.py used.
OLD_CONFIGS = {"laplacian": (5, 45, 1.0, 2.0), "laplacian_light": (3, 11, 0.5, 2.0), "custom": (4, 13, 1.0, 1.5),
               "single_level": (1, 45, 1.0, 2.0)}
OLD_SHAPES = [(2, 3, 40, 56), (1, 3, 144, 201), (2, 3, 512, 512), (1, 3, 1024, 1024), (2, 1, 40, 56), (1, 1, 144, 201),
              (1, 1, 70, 33), (2, 3, 1, 9), (1, 2, 5, 1)]
CASES = [cfg + shape for cfg in OLD_CONFIGS.values() for shape in OLD_SHAPES]
CASES += [
    (3, 1, 1.0, 2.0, 1, 1, 1, 1),          # NC 1, width 1: every band is exactly zero; W == H == 1
    (4, 7, 1.0, 1.5, 2, 3, 65, 33),        # NC 1 at 7; y and x tile seams + 1
    (5, 9, 1.5, 1.5, 1, 4, 64, 32),        # NC 2 at 9; seams, C = 4, both ping-pong parities
    (3, 15, 2.0, 1.5, 1, 3, 129, 65),
    (2, 17, 2.5, 2.0, 1, 1, 40, 56),       # NC 3
    (4, 23, 3.0, 1.5, 2, 1, 70, 40),       # right fold with W - 1 = 39, 7 (mod 8), in the tile's middle group
    (4, 25, 3.0, 1.5, 1, 2, 5, 1),         # NC 4: W == 1, H shorter than the radius
    (3, 31, 4.0, 1.5, 1, 3, 144, 201),
    (5, 33, 4.0, 1.5, 1, 1, 1, 9),         # NC 5: H == 1, W narrower than the radius
    (2, 39, 5.0, 2.0, 2, 3, 128, 64),
    (3, 41, 5.0, 1.5, 1, 4, 96, 96),       # NC 6: opt-in shared memory; W - 1 = 95, 7 (mod 8), in the last group
    (3, 47, 6.0, 1.5, 1, 3, 97, 95),
    (3, 49, 6.0, 1.5, 1, 1, 65, 129),      # NC 7
    (2, 55, 7.0, 2.0, 2, 2, 30, 20),       # W and H narrower than the radius 27
    (3, 57, 7.0, 1.5, 1, 3, 128, 88),      # NC 8
    (2, 63, 8.0, 2.0, 1, 1, 20, 70),       # the cap, H shorter than the radius 31
    (4, 63, 8.0, 1.5, 1, 2, 129, 257),
    (1, 1, 1.0, 2.0, 2, 3, 37, 45),        # levels 1: elementwise kernels
    (1, 1, 1.0, 2.0, 1, 1, 8, 8),
]


def _id(case):
    L, w, s, m, n, c, h, wd = case
    return "L%d-w%d-s%g-m%g-%dx%dx%dx%d" % (L, w, s, m, n, c, h, wd)


def case_labels(case):
    L, w, _, _, n, c, h, wd = case
    r = w // 2
    labels = set()
    if L == 1:
        return {"levels = 1 (lerp kernels)", "C = %d" % c if c in (1, 4) else "C other", "N > 1" if n > 1 else "N = 1"}
    nc = nc_of(w)
    labels |= {"%s NC=%d" % (MODE_NAME[m], nc) for m in (BL_FWD, BL_SWEEP, BL_ADJ)}
    labels.add("width %d (NC=%d, %s)" % (w, nc, "width = 1" if w == 1 else "width = 8 NC - 7" if w % 8 == 1
                                           else "width = 8 NC - 1" if w % 8 == 7 else "other width"))
    if L == 2:
        labels.add("levels = 2 (first == last, adjoint init from the input mask)")
    if L >= 4:
        labels.add("levels >= 4 (both ping-pong parities twice)")
    if wd > TW and wd % TW in (0, 1):
        labels.add("x tile seam (W = 32k%s)" % ("" if wd % TW == 0 else " + 1"))
    if h > TH and h % TH in (0, 1):
        labels.add("y tile seam (H = 64k%s)" % ("" if h % TH == 0 else " + 1"))
    if wd > 1:
        last = (wd - 1) % TW
        labels.add("right fold in a tile's %s 8-group" % ("last" if last >= TW - 8 else "middle"))
        labels.add("right fold with W - 1 %s 7 (mod 8)" % ("=" if (wd - 1) % 8 == 7 else "!="))
        labels.add("left fold")
    if h > 1:
        labels.add("top fold")
        labels.add("bottom fold")
    if wd > 1 and r > wd - 1:
        labels.add("fold with min(r, W - 1) = W - 1")
    if h > 1 and r > h - 1:
        labels.add("fold with min(r, H - 1) = H - 1")
    if wd == 1:
        labels.add("W == 1 (wsum)")
    if h == 1:
        labels.add("H == 1 (wsum)")
    if c in (1, 4):
        labels.add("C = %d" % c)
    if n > 1:
        labels.add("N > 1 (blockIdx.z)")
    if level_smem_bytes(nc) > STATIC_SMEM:
        labels.add("shared memory past 48 KB (opt-in attribute)")
    return labels


REQUIRED = (["%s NC=%d" % (m, k) for m in ("fwd", "sweep", "adj") for k in range(1, 9)]
            + ["width 1 (NC=1, width = 1)", "width 63 (NC=8, width = 8 NC - 1)"]
            + ["width %d (NC=%d, width = 8 NC - 7)" % (8 * k - 7, k) for k in range(2, 9)]
            + ["width %d (NC=%d, width = 8 NC - 1)" % (8 * k - 1, k) for k in range(1, 9)]
            + ["levels = 1 (lerp kernels)", "levels = 2 (first == last, adjoint init from the input mask)",
               "levels >= 4 (both ping-pong parities twice)",
               "x tile seam (W = 32k)", "x tile seam (W = 32k + 1)", "y tile seam (H = 64k)", "y tile seam (H = 64k + 1)",
               "right fold in a tile's last 8-group", "right fold in a tile's middle 8-group",
               "right fold with W - 1 = 7 (mod 8)", "right fold with W - 1 != 7 (mod 8)", "left fold", "top fold",
               "bottom fold", "fold with min(r, W - 1) = W - 1", "fold with min(r, H - 1) = H - 1", "W == 1 (wsum)",
               "H == 1 (wsum)", "C = 1", "C = 4", "N > 1 (blockIdx.z)", "shared memory past 48 KB (opt-in attribute)"])


def test_cases_reach_every_route():
    """Every instantiation {fwd, sweep, adj} x NC = 1..8 at both padding extremes of its NC, levels 1, 2 and >= 4, both
    tile seams and one past them, the right fold in a tile's last and in a middle 8-group with W - 1 = 7 and != 7 (mod 8),
    folds clipped by a plane narrower or shorter than the radius, W == 1 and H == 1, C = 1 and 4, N > 1 and the opt-in
    shared memory."""
    reached = set()
    for case in CASES:
        reached |= case_labels(case)
    assert_routes_reached(REQUIRED, reached)


def test_every_case_is_legal():
    for L, w, _, _, n, c, h, wd in CASES:
        assert L >= 1 and 1 <= w <= MAX_WIDTH and w % 2 == 1 and 1 <= n <= 65535 and h <= 65535 * TH, (L, w, n, h)


def test_static_shared_memory_reads_stay_inside_the_tiles():
    """For every NC, the horizontal pass's float4 reads s_in[q][xg + i + u] (xg <= 24, i < P + 8 in steps of 4, u < 4)
    stay below the staged row stride SWI = 32 + P, the vertical pass's s_h rows vy + i (vy <= 56, i < P + 7) below HROWS =
    64 + P - 1, the epilogue's centre tap s_in[vy + k + r][vx + r] inside the staged tile, and the border folds' columns /
    rows (W - 1 - x0) + r - i and (H - 1 - y0) + r - i inside [0, SWI) / [0, HROWS) for every width of that NC."""
    for nc in range(1, 9):
        p = 8 * nc
        swi, hrows = TW + p, TH + p - 1
        assert max(xg + i + u for xg in range(0, TW, 8) for i in range(0, p + 8, 4) for u in range(4)) < swi
        assert max(vy + i for vy in range(0, TH, 8) for i in range(p + 7)) < hrows
        for w in range(8 * nc - 7, 8 * nc + 1, 2):
            r = w // 2
            assert 2 * r <= p - 1
            assert (TH - 8) + 7 + r < hrows and (TW - 1) + r < swi        # the epilogue's centre tap
            assert 2 * r < swi and 2 * r < hrows                            # left / top fold: r + i, i <= r
            assert (TW - 1) + r < swi and (TH - 1) + r < hrows              # right / bottom fold: (n - 1 - x0) + r - i
    # the static layout fits the opt-in limit (227 KB) at the largest P
    assert level_smem_bytes(8) <= 227 * 1024


def test_workspace_covers_every_address_the_launches_use():
    """The ping-pong A / B / M buffers of the forward and the A / B ping-pong, mask stack M_1..M_{L-1} and d_0..d_{L-1}
    of the backward lie inside gg_laplacian_blend_workspace(...) at levels 1..6, and the restated formula equals the
    library's."""
    lib = library().load()
    for n, c, h, w in [(1, 1, 1, 1), (2, 3, 40, 56), (1, 4, 65, 33), (3, 2, 7, 129)]:
        for levels in range(1, 7):
            for backward in (0, 1):
                ws = lib.gg_laplacian_blend_workspace(n, c, h, w, levels, backward)
                assert ws == workspace_bytes(n, c, h, w, levels, backward), (n, c, h, w, levels, backward)
                if levels == 1:
                    assert ws == 0
                    continue
                ranges = (backward_buffers if backward else forward_buffers)(n, c, h, w, levels)
                assert min(s for s, _ in ranges) == 0
                assert max(s + k for s, k in ranges) <= ws // 4, (n, c, h, w, levels, backward)
                if levels >= 3:                                    # both ping-pong halves in use: no float is spare
                    assert max(s + k for s, k in ranges) == ws // 4


def test_product_taps_are_bitwise_symmetric():
    """The adjoint runs the forward's tiled kernel on zero-padded input, which is the transpose only for symmetric taps."""
    from gangealing_b200.splat2d.blend import level_taps
    cfgs = {(L, w, s, m) for L, w, s, m, *_ in CASES if L > 1}
    cfgs |= {(5, 45, 1, 2), (3, 11, 0.5, 2), (6, 63, 0.3, 3.0), (6, 3, 10.0, 0.5)}
    for L, w, s, m in sorted(cfgs):
        t = level_taps(L, w, s, 0, m, device="cpu")
        assert t.shape == (L - 1, w)
        assert torch.equal(t, t.flip(1)), (L, w, s, m)
        assert bool((t >= 0).all()), "non-negative taps: the blur is non-expansive on magnitudes"


def test_plan_matches_the_launch_names():
    for L, w, *_ in CASES:
        for bwd in (0, 1):
            names = launches(L, w, bwd)
            assert len(names) == (1 if L == 1 else (L - 1) * (2 if bwd else 1) + bwd)
    assert launches(5, 45, 0) == ["blend_level_kernel<6, 0>"] * 4
    assert level_grid(2, 65, 33) == (2, 2, 2)


# ======================================================================================================== GPU checks
WORST = Worst("c per path", "%-56s %.2f")
_report_worst = WORST.fixture()


def _inputs(case):
    L, w, s, m, n, c, h, wd = case
    img0, img1, mask, gout = OB.fixture_inputs(w * 31 + h + wd, n, c, h, wd)
    mask = mask.clone()
    mask.view(-1)[::7] = 0.5                              # the lerp's branch point
    return [t.to(DEV) for t in (img0, img1, mask, gout)]


def _guarded(nbytes):
    buf = torch.full((nbytes // 4 + GUARD,), float("nan"), device=DEV)
    return buf


def _guard_intact(buf, nbytes, what):
    torch.cuda.synchronize()
    assert bool(buf[nbytes // 4:].isnan().all()), "%s: the launches wrote past the workspace" % what


def stack64(x, taps, levels):
    out = [x]
    for l in range(levels - 1):
        out.append(OB.blur_ref(out[-1], taps[l]))
    return out


def blur_t(u, taps_l):
    """float64 transpose of one level's blur."""
    z = torch.zeros_like(u, requires_grad=True)
    return torch.autograd.grad(OB.blur_ref(z, taps_l), z, u)[0]


def c_stack(w, l):
    """A stored level-l plane: two fma chains of `width` non-zero taps per level (the padding taps are exact zeros),
    plus the error of level l - 1 carried through the non-expansive blur."""
    return 2 * w * l


def c_forward(w, L):
    """The planes of level l + 1 carry c_stack(L - 1) at most; the mask's error times |b - a| counts as much again;
    then the two differences, the lerp's difference and its fma (4), and the running sum over L terms (L - 1)."""
    return 2 * c_stack(w, L - 1) + 4 + L - 1


def c_transpose(w, h, wd):
    """One level of T^T: interior two fma chains of `width` taps; a border value is a fold over min(r, n - 1) + 1 terms
    with prefix sums rounded once (W == 1 / H == 1: the product with the rounded tap sum)."""
    r = w // 2
    return max(w, min(r, wd - 1) + 2) + max(w, min(r, h - 1) + 2)


def _run_forward(case, img0, img1, mask, taps):
    lib = library()
    L, w, s, m, n, c, h, wd = case
    out = nan_at((n, c, h, wd), torch.float32)
    nbytes = lib.load().gg_laplacian_blend_workspace(n, c, h, wd, L, 0)
    ws = _guarded(nbytes)
    rc = lib.load().gg_laplacian_blend_forward(out.data_ptr(), ws.data_ptr(), img0.data_ptr(), img1.data_ptr(),
                                               mask.data_ptr(), taps.data_ptr() if L > 1 else None, n, c, h, wd, L, w,
                                               lib.stream())
    lib.check(rc, "gg_laplacian_blend_forward")
    _guard_intact(ws, nbytes, "forward")
    return out, ws


def _run_backward(case, gout, img0, img1, mask, taps):
    lib = library()
    L, w, s, m, n, c, h, wd = case
    g0, g1 = nan_at((n, c, h, wd), torch.float32), nan_at((n, c, h, wd), torch.float32)
    gm = nan_at((n, 1, h, wd), torch.float32)
    nbytes = lib.load().gg_laplacian_blend_workspace(n, c, h, wd, L, 1)
    ws = _guarded(nbytes)
    rc = lib.load().gg_laplacian_blend_backward(g0.data_ptr(), g1.data_ptr(), gm.data_ptr(), ws.data_ptr(),
                                                gout.data_ptr(), img0.data_ptr(), img1.data_ptr(), mask.data_ptr(),
                                                taps.data_ptr() if L > 1 else None, n, c, h, wd, L, w, lib.stream())
    lib.check(rc, "gg_laplacian_blend_backward")
    _guard_intact(ws, nbytes, "backward")
    return g0, g1, gm, ws


MULTI = [cs for cs in CASES if cs[0] > 1]


@pytest.mark.gpu
@pytest.mark.parametrize("case", MULTI, ids=_id)
def test_forward_and_gradients(case):
    from gangealing_b200.splat2d.blend import level_taps
    L, w, s, m, n, c, h, wd = case
    nc = nc_of(w)
    img0, img1, mask, gout = _inputs(case)
    taps = level_taps(L, w, s, 0, m, device=DEV)
    t64 = taps.double()
    x0, x1, mk, g = (t.double() for t in (img0, img1, mask, gout))
    A, B, M = stack64(x0, t64, L), stack64(x1, t64, L), stack64(mk, t64, L)
    Aa, Ba = stack64(x0.abs(), t64, L), stack64(x1.abs(), t64, L)
    total, plane = n * c * h * wd, n * h * wd

    # ---- forward: every output element, then the last two levels the workspace holds
    out, ws = _run_forward(case, img0, img1, mask, taps)
    ref = OB.laplacian_blend_ref(x0, x1, mk, L, w, s, taps=t64)
    mag = sum(Aa[l] + Aa[l + 1] + Ba[l] + Ba[l + 1] for l in range(L - 1)) + Aa[L - 1] + Ba[L - 1]
    WORST.check_sum(out, ref, mag, c_forward(w, L), "forward, NC=%d" % nc, _id(case))
    for l in range(max(1, L - 2), L):
        slot = (l - 1) & 1
        a_l = ws[slot * total:(slot + 1) * total].view(n, c, h, wd)
        b_l = ws[(2 + slot) * total:(3 + slot) * total].view(n, c, h, wd)
        m_l = ws[4 * total + slot * plane:4 * total + (slot + 1) * plane].view(n, 1, h, wd)
        for name, y, r64, a64 in (("A", a_l, A[l], Aa[l]), ("B", b_l, B[l], Ba[l]), ("M", m_l, M[l], M[l])):
            WORST.check_stored(y, r64, a64, c_stack(w, l), "forward stack, NC=%d" % nc, "%s %s_%d" % (_id(case), name, l))

    # ---- backward
    g0, g1, gm, wsb = _run_backward(case, gout, img0, img1, mask, taps)
    mstack = wsb[4 * total:4 * total + (L - 1) * plane].view(L - 1, n, 1, h, wd)
    for l in range(1, L):                                   # the sweep's mask stack, as stored values
        WORST.check_stored(mstack[l - 1], M[l], M[l], c_stack(w, l), "sweep mask stack, NC=%d" % nc,
                           "%s M_%d" % (_id(case), l))
    Ms = [mk] + [mstack[l - 1].double() for l in range(1, L)]   # the operands the adjoint reads
    cA = [1 - Ms[0]] + [Ms[l - 1] - Ms[l] for l in range(1, L)]
    cT = c_transpose(w, h, wd)
    # U_{L-1} = g c_{L-1} (coefficient and product: 2); each Horner step adds T^T, the coefficient and the fma
    c_img = 2 + (L - 1) * (cT + 2)
    cB = [Ms[0]] + [-cA[l] for l in range(1, L)]
    for name, y, coef in (("grad_img0", g0, cA), ("grad_img1", g1, cB)):
        u = g * coef[L - 1]
        ua = u.abs()
        for l in range(L - 2, -1, -1):
            u = g * coef[l] + blur_t(u, t64[l])
            ua = (g * coef[l]).abs() + blur_t(ua, t64[l])
        WORST.check_sum(y, u, ua, c_img, "adjoint, NC=%d" % nc, "%s %s" % (_id(case), name))
    # grad_mask: float64 autograd; its terms d_l carry the fp32 A / B stacks of the sweep
    args = [t.clone().requires_grad_(True) for t in (x0, x1, mk)]
    ref_gm = torch.autograd.grad(OB.laplacian_blend_ref(*args, L, w, s, taps=t64), args[2], g)[0]
    gabs = g.abs()
    D = [(gabs * (Aa[l] + Aa[l + 1] + Ba[l] + Ba[l + 1])).sum(1, keepdim=True) for l in range(L - 1)]
    D.append((gabs * (Aa[L - 1] + Ba[L - 1])).sum(1, keepdim=True))
    um = D[L - 1]
    for l in range(L - 2, -1, -1):
        um = D[l] + blur_t(um, t64[l])
    c_d = c_stack(w, L - 1) + 4 + (c - 1)       # the stack planes (level <= L - 1), 4 roundings per term, the sum over C
    c_mask = c_d + (L - 1) * (cT + 1)
    WORST.check_sum(gm, ref_gm, um, c_mask, "adjoint, NC=%d" % nc, "%s grad_mask" % _id(case))


LERP_CASES = [cs for cs in CASES if cs[0] == 1]


def _lerp_inputs(case, seed):
    """Operands off the dyadic lattice (randn: full mantissas, mixed binades) and masks with exact 0, 0.5, 1 and
    arbitrary values in between."""
    _, _, _, _, n, c, h, wd = case
    gen = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(n, c, h, wd, generator=gen, device=DEV) * 3
    b = torch.randn(n, c, h, wd, generator=gen, device=DEV)
    u = torch.rand(n, 1, h, wd, generator=gen, device=DEV)
    pick = torch.randint(0, 4, (n, 1, h, wd), generator=gen, device=DEV)
    mask = torch.where(pick == 0, torch.zeros_like(u), torch.where(pick == 1, torch.full_like(u, 0.5),
                                                                   torch.where(pick == 2, torch.ones_like(u), u)))
    mask.view(-1)[:3] = torch.tensor([0.0, 0.5, 1.0], device=DEV)
    g = torch.randn(n, c, h, wd, generator=gen, device=DEV)
    return a, b, mask, g


@pytest.mark.gpu
@pytest.mark.parametrize("case", LERP_CASES, ids=_id)
def test_single_level_is_bitwise(case):
    """levels == 1: the forward is torch.lerp(img0, img1, mask); grad_img0 = g * (1 - m) and grad_img1 = g * m, each
    rounded as written; grad_mask is the sequential fp32 sum over c of g * (b - a).  For the sum the gradient takes powers
    of two, so that each product is exact and the sum's roundings are the additions alone."""
    _, w, _, _, n, c, h, wd = case
    a, b, mask, g = _lerp_inputs(case, h * wd + c)
    assert bool((mask == 0.5).any() and (mask == 0).any() and (mask == 1).any())
    out, _ = _run_forward(case, a, b, mask, None)
    assert torch.equal(out, torch.lerp(a, b, mask)), "forward != torch.lerp"
    g0, g1, gm, _ = _run_backward(case, g, a, b, mask, None)
    assert torch.equal(g0, g * (1 - mask)), "grad_img0 != g * (1 - m)"
    assert torch.equal(g1, g * mask), "grad_img1 != g * m"
    gp = torch.ldexp(torch.sign(g) + (g == 0), torch.randint(-3, 4, g.shape, device=DEV).float())   # +-2^k
    _, _, gm, _ = _run_backward(case, gp, a, b, mask, None)
    s = gp[:, 0:1] * (b[:, 0:1] - a[:, 0:1])
    for ch in range(1, c):
        s = s + gp[:, ch:ch + 1] * (b[:, ch:ch + 1] - a[:, ch:ch + 1])
    assert torch.equal(gm, s), "grad_mask != the sequential fp32 sum over channels"
    print("[contract] levels = 1: %s bitwise" % _id(case))


@pytest.mark.gpu
def test_entries_refuse_a_grid_taller_than_the_y_dimension():
    """H > 65535 * 64 row tiles cannot be launched (grid.y): both entries return GG_ERR_UNSUPPORTED before any device
    work, on real buffers (one 4 194 241 x 1 plane each), and leave the outputs as they were."""
    lib = library()
    h = 65535 * TH + 1
    img = torch.zeros(1, 1, h, 1, device=DEV)
    taps = torch.ones(1, 1, device=DEV)
    out = nan_at((1, 1, h, 1), torch.float32)
    ws = torch.zeros(max(lib.load().gg_laplacian_blend_workspace(1, 1, h, 1, 2, 1),
                         lib.load().gg_laplacian_blend_workspace(1, 1, h, 1, 2, 0)) // 4, device=DEV)
    rc = lib.load().gg_laplacian_blend_forward(out.data_ptr(), ws.data_ptr(), img.data_ptr(), img.data_ptr(),
                                               img.data_ptr(), taps.data_ptr(), 1, 1, h, 1, 2, 1, lib.stream())
    assert rc == -2 and b"height" in lib.load().gg_last_error(), (rc, lib.load().gg_last_error())
    g1, gm = nan_at((1, 1, h, 1), torch.float32), nan_at((1, 1, h, 1), torch.float32)
    rc = lib.load().gg_laplacian_blend_backward(out.data_ptr(), g1.data_ptr(), gm.data_ptr(), ws.data_ptr(), img.data_ptr(),
                                                img.data_ptr(), img.data_ptr(), img.data_ptr(), taps.data_ptr(), 1, 1, h,
                                                1, 2, 1, lib.stream())
    assert rc == -2 and b"height" in lib.load().gg_last_error(), (rc, lib.load().gg_last_error())
    torch.cuda.synchronize()
    assert bool(out.isnan().all() and g1.isnan().all() and gm.isnan().all())
    # one row tile less is legal and runs
    h2 = 65535 * TH
    rc = lib.load().gg_laplacian_blend_forward(out.data_ptr(), ws.data_ptr(), img.data_ptr(), img.data_ptr(),
                                               img.data_ptr(), taps.data_ptr(), 1, 1, h2, 1, 2, 1, lib.stream())
    lib.check(rc, "gg_laplacian_blend_forward at 65535 row tiles")
    torch.cuda.synchronize()
    assert bool((out.view(-1)[:h2] == 0).all())


# ------------------------------------------------------------------------------------------------------------ launches
KERNELS = re.compile(r"blend_level_kernel<\d+, \d+>|blend_adj_init_kernel|blend_lerp_bwd_kernel|blend_lerp_kernel")


@pytest.mark.gpu
def test_each_entry_launches_its_labelled_instantiation():
    """Each entry launches exactly the blend_level_kernel<NC, MODE> its case is labelled with, one per level in level
    order (and the adjoint init between the sweep and the Horner steps; the lerp kernels at one level)."""
    run_fresh("test_blend_family_gpu", "check_launches")


def check_launches():
    from gangealing_b200.splat2d.blend import level_taps
    lib = library()
    checked = 0
    for case in CASES:
        L, w, s, m, n, c, h, wd = case
        z = torch.zeros(n, c, h, wd, device=DEV)
        zm = torch.zeros(n, 1, h, wd, device=DEV)
        taps = level_taps(L, w, s, 0, m, device=DEV) if L > 1 else None
        for bwd in (0, 1):
            ws = torch.empty(max(1, lib.load().gg_laplacian_blend_workspace(n, c, h, wd, L, bwd) // 4), device=DEV)
            if bwd:
                def call():
                    lib.check(lib.load().gg_laplacian_blend_backward(z.data_ptr(), z.data_ptr(), zm.data_ptr(), ws.data_ptr(),
                                                                     z.data_ptr(), z.data_ptr(), z.data_ptr(), zm.data_ptr(),
                                                                     lib.ptr(taps), n, c, h, wd, L, w, lib.stream()), "bwd")
            else:
                def call():
                    lib.check(lib.load().gg_laplacian_blend_forward(z.data_ptr(), ws.data_ptr(), z.data_ptr(), z.data_ptr(),
                                                                    zm.data_ptr(), lib.ptr(taps), n, c, h, wd, L, w,
                                                                    lib.stream()), "fwd")
            got = launched(call, KERNELS)
            want = launches(L, w, bwd)
            assert got == want, "%s %s: launched %s, the case is labelled %s" % (_id(case), "bwd" if bwd else "fwd", got, want)
            checked += 1
    print("[launch] %d entry calls launched their labelled instantiations" % checked)
