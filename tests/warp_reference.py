"""The antialiased sampler's float64 reference, its decision margins and constructed edge grids (not collected: the name
does not match test_*.py).  test_sampling_gpu.py checks the sampler end to end against the reference model's semantics;
test_warp_family_gpu.py checks each kernel of csrc/warp.cu against float64 evaluated on the exact operands a launch reads.

Operands.  The float64 stack is built from the source and the STORED fp32 pyramid (each level up-sampled by 2^i and
cropped by the power-of-two padding lp, oracle/sampling.py upsample_bilinear), so the pyramid's own rounding, which
test_pyramid_tent_family_gpu.py bounds, does not enter these bounds.  Sampling and the level of detail follow
oracle/sampling.py grid_sample_bilinear and mipmap_levels.

Level of detail.  The fp32 level differs from the float64 one by at most eps_L (level_error): the rounding of the
coordinates (none on dyadic grids), of sq = dx^2 + dy^2, of sqrtf (correctly rounded: the library is built without
fast-math) and log2f (at most 1 ulp, CUDA C Programming Guide, table of single-precision functions).  The sampled value
is continuous in the level, so that error reaches an output as eps_L times the slope between the adjacent levels.
"""
import math

import torch
import torch.nn.functional as F

from oracle import sampling as S
from oracle.rounding import U32

F64 = torch.float64
LN2 = math.log(2.0)


# ------------------------------------------------------------------------------------------------ "decided" pixels
# The sampler makes discrete choices: the bilinear corner floor(c), the mip levels floor / ceil(level), the arg-max
# neighbour of the level of detail and the clamps of both.  Where the oracle's value sits within rounding noise of such a
# boundary, the last ulp of the fp32 evaluation order decides the choice (on the GPU as in ATen's own CUDA kernel), and the
# grid gradient jumps there.  The level thresholds are those of the fp32 level of detail (level_atol): level_atol of a
# level, half of it relative between the two largest neighbour distances.
def level_atol(size):
    """levels vs the float64 oracle: the level of detail is log2 of a difference of fp32 coordinates of up to ~size px,
    which cancellation leaves with ~ulp(coordinate) / distance relative error: measured 3e-5 (128 px source) and 1.6e-4
    (512 px) in log2 units at 1-2 px distances."""
    return 1e-4 * max(1.0, size / 200.0)


def coordinate_decided(c, size, mode, exact_integers=False):
    """floor(c) is decided: c is not within 1e-4 px of an integer -- or pinned to a border pixel by the clamp of the border /
    reflection modes (an exact constant on both sides).  `exact_integers`: c is the float64 image of fp32 arithmetic that is
    exact on both sides (dyadic grids; float64 of fp32 inputs, where an exact integer is an exact integer in fp32 too)."""
    off = (c - c.round()).abs()
    ok = off > 1e-4
    if exact_integers:
        ok |= off == 0
    if mode != "zeros":
        ok |= (c == 0) | (c == size - 1)
    return ok


def level_decided(lv):
    """floor / ceil of a level of detail are decided: not within 1e-5 of an integer -- or exactly 0, the clamp of a
    distance <= 1 px (an exact constant on both sides)."""
    return ((lv - lv.round()).abs() > 1e-5) | (lv == 0)


def neighbour_sq(grid, hs, ws):
    """(4, N, Ho, Wo) squared distances, in level-of-detail coordinates, to the left / right / up / down neighbour
    (replicate-clamped at the image border), unclamped -- the oracle's max_coord_distance before its clamp(min=1)."""
    c = S.lod_coordinates(grid, hs, ws)
    p = F.pad(c.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="replicate").permute(0, 2, 3, 1)
    neigh = [p[:, 1:-1, :-2], p[:, 1:-1, 2:], p[:, :-2, 1:-1], p[:, 2:, 1:-1]]
    return torch.stack([((o - c) ** 2).sum(dim=3) for o in neigh])


def argmax_targets(grid, hs, ws):
    """The level-of-detail arg-max neighbour of every pixel (first maximum of the clamped distances, order left, right,
    up, down) -> (arg, ty, tx), each (N, Ho, Wo), the target replicate-clamped to the image."""
    sq = neighbour_sq(grid.double(), hs, ws)
    arg = sq.clamp(min=1.0).sqrt().max(dim=0).indices
    n, ho, wo = arg.shape
    ty = (torch.arange(ho)[None, :, None] + torch.tensor([0, 0, -1, 1])[arg]).clamp(0, ho - 1)
    tx = (torch.arange(wo)[None, None, :] + torch.tensor([-1, 1, 0, 0])[arg]).clamp(0, wo - 1)
    return arg, ty, tx


def _mark_targets(bad, nb_idx, sel):
    """bad |= the neighbours nb_idx (0 left, 1 right, 2 up, 3 down; replicate-clamped) of the pixels `sel`."""
    n, ho, wo = bad.shape
    ni, yi, xi = torch.meshgrid(torch.arange(n), torch.arange(ho), torch.arange(wo), indexing="ij")
    ty = (yi + torch.tensor([0, 0, -1, 1])[nb_idx]).clamp(0, ho - 1)
    tx = (xi + torch.tensor([-1, 1, 0, 0])[nb_idx]).clamp(0, wo - 1)
    bad[ni[sel], ty[sel], tx[sel]] = True


def undecided_pixels(grid, hs, ws, mode, max_level=None, min_level=0.0, grid_gradient=True):
    """(N, Ho, Wo) bool, from the float64 grid: a bilinear coordinate within 1e-4 px of an integer, or (mip sampling,
    `max_level` not None) the level within level_atol of an integer or of a clamp, or the top two neighbour distances within
    half of that relative, or (border / reflection) the coordinate within 1e-4 px of the clip.  Exactly-on values are
    decided: the float64 images of fp32 inputs are exact, and so are their ties.
    `grid_gradient`: a pixel also receives the level-of-detail term of every neighbour that targets it, so an undecided
    level or arg-max also marks every neighbour that may be the arg-max (a corner index only moves the
    pixel's own terms: the level-of-detail term is continuous in it)."""
    g = grid.double()
    bad = torch.zeros(g.shape[:3], dtype=torch.bool)
    for k, size in ((0, ws), (1, hs)):
        bad |= ~coordinate_decided(S.source_index(g[..., k], size, mode), size, mode, True)
        if mode != "zeros":     # the clip itself: a coordinate at the border is clamped (gradient 0) on one side only
            raw = ((g[..., k] + 1.0) * size - 1.0) / 2.0
            raw = S._reflect(raw, -1, 2 * size - 1) if mode == "reflection" else raw
            for edge in (0.0, size - 1.0):
                bad |= ((raw - edge).abs() <= 1e-4) & (raw != edge)
    if max_level is None:
        return bad
    sq = neighbour_sq(g, hs, ws)
    raw = 0.5 * torch.log2(sq.max(dim=0).values)          # unclamped level; -inf where every neighbour coincides
    off = (raw - raw.round()).abs()
    tol = level_atol(max(hs, ws))
    level_bad = (off > 0) & (off <= tol) & (raw >= -tol) & (raw <= max_level + tol)
    for clamp in (max_level, min_level):
        level_bad |= (raw != clamp) & ((raw - clamp).abs() <= tol)
    top = sq.clamp(min=1.0).sqrt().topk(2, dim=0)
    gap = top.values[0] - top.values[1]
    tie_bad = (gap > 0) & (gap <= 0.5 * tol * top.values[0])
    bad |= level_bad | tie_bad
    if grid_gradient:
        # the kernel's arg-max may be ANY neighbour whose distance lies within the rounding band of the largest (three of them
        # can be that close), judged by the UNCLAMPED distance: below 1 px the clamp ties them all, the rounding does not
        band = sq >= sq.max(dim=0).values * (1.0 - tol)
        for k in range(4):
            _mark_targets(bad, torch.full(bad.shape, k), (level_bad | tie_bad) & band[k])
    return bad


# ------------------------------------------------------------------------------------------------ constructed grids
def _dyadic(k):
    return k.double() / 512.0


def _edge_grid(case):
    """Constructed grids (N, Ho, Wo, 2), source size and sampler settings for the edges of the grid-gradient gather."""
    yy, xx = torch.meshgrid(torch.arange(16), torch.arange(16), indexing="ij")
    if case == "pinch":
        # a zoomed-out dyadic affine grid (~4 px between neighbours) with three points displaced ~20 px: every neighbour of
        # the displaced interior point (4), edge point (3) and corner point (2) takes it as its arg-max neighbour
        k = torch.stack([64 * xx + 9 * yy - 540, -6 * xx + 60 * yy - 480], dim=-1)
        for y, x in ((8, 8), (0, 5), (15, 15)):
            k[y, x] += torch.tensor([256, -205])
        return _dyadic(k[None]).float(), 64, 8, 0.0
    if case == "ties":
        # dyadic affine grid (k/512): left/right and up/down distances tie EXACTLY (in fp32 too), half the pixels nudged by
        # +-1/512 so that some ties break; "first maximum, order left, right, up, down" = torch.max(dim=0)'s first index
        g = torch.Generator().manual_seed(5)
        kx = 40 * xx + 13 * yy - 300
        ky = -11 * xx + 37 * yy - 280
        k = torch.stack([kx, ky], dim=-1) + torch.randint(-1, 2, (16, 16, 2), generator=g) * (torch.rand(16, 16, 1, generator=g) < 0.5)
        return _dyadic(k[None]).float(), 64, 8, 0.0
    if case.startswith("clamps"):
        # 65 px source: level-of-detail coordinates are k/16 + 32, so steps of 16, 24, 32, 48, 64, 128 (/512) are distances
        # of exactly 1 (sq == 1: level 0 at the clamp), 1.5, 2, 3, 4 (level 2 = min_level of "clamps_min") and 8 px
        # (level 3 = max_level); a corner patch has unit steps only, the
        # crossing of rows and columns 10..13 4 px steps only
        g = torch.Generator().manual_seed(6)
        steps = torch.tensor([16, 24, 32, 48, 64, 128])
        sx, sy = steps[torch.randint(0, 6, (16, 16), generator=g)], steps[torch.randint(0, 6, (16, 16), generator=g)]
        sx[:4, :4] = sy[:4, :4] = 16
        sx[10:14, :] = 64
        sy[:, 10:14] = 64
        kx, ky = sx.cumsum(1), sy.cumsum(0)
        k = torch.stack([kx - kx[8, 8], ky - ky[8, 8]], dim=-1)
        return _dyadic(k[None]).float(), 65, 4, (2.0 if case == "clamps_min" else 0.0)
    # "borders": source coordinates exactly on (and just inside / outside of) both borders: k = -504 / 504 is c = 0 / 63
    # on a 64 px source, k = -512 / 512 the edges of the normalised range (reflection folds them onto the borders)
    kx = torch.where(xx < 8, -528 + 4 * xx, 488 + 4 * (xx - 8))
    ky = -504 + 84 * yy
    return _dyadic(torch.stack([kx, ky], dim=-1)[None]).float(), 64, 8, 0.0


# ------------------------------------------------------------------------------------------------ the float64 reference
def pad_geometry(hs, ws):
    """warp.cu make_pyramid: (lp, hp, wp) -- the width decides the reflect padding to a power of two, both axes take it."""
    lp, rp = S.pow2_padding(ws)
    return lp, hs + lp + rp, ws + lp + rp


def split_pyramid(flat, n, c, hs, ws, extra):
    """Levels 1..E of the library's flat fp32 pyramid as (N, C, h_i, w_i) views, at make_pyramid's offsets."""
    _, hp, wp = pad_geometry(hs, ws)
    out, off = [], 0
    for i in range(1, extra + 1):
        h, w = hp >> i, wp >> i
        out.append(flat[off:off + n * c * h * w].view(n, c, h, w))
        off += n * c * h * w
    return out


def build_stack(x64, levels64, hs, ws):
    """[the source] + each stored level up-sampled by 2^i (F.interpolate, bilinear, align_corners=False) and cropped by lp:
    the Gaussian stack the kernel reads through level_value, (N, C, hs, ws) per level."""
    lp = pad_geometry(hs, ws)[0]
    return [x64] + [S.upsample_bilinear(lv, 2 ** i)[:, :, lp:lp + hs, lp:lp + ws] for i, lv in enumerate(levels64, 1)]


def sample_stack(stack, grid64, mode):
    """(N, C, K, Ho, Wo): the bilinear sample of every stack level."""
    return torch.stack([S.grid_sample_bilinear(s, grid64, mode)[0] for s in stack], dim=2)


def _take(samples, idx):
    """samples (N, C, K, Ho, Wo) at the per-pixel level index idx (N, Ho, Wo)."""
    n, c = samples.shape[:2]
    return torch.gather(samples, 2, idx[:, None, None].expand(n, c, 1, *idx.shape[1:]))[:, :, 0]


def blend(samples, level):
    """o0 + w (o1 - o0) at levels floor / ceil (antialiased_sampling.py:227-237); level None: level 0 alone."""
    if level is None:
        return samples[:, :, 0]
    l0, l1 = level.floor().long(), level.ceil().long()
    o0 = _take(samples, l0)
    return o0 + (level - l0)[:, None] * (_take(samples, l1) - o0)


def blend_abs(samples_abs, level):
    """A = A0 + w (A0 + A1): the magnitudes the fp32 blend o0 + w (o1 - o0) rounds (the difference may cancel)."""
    if level is None:
        return samples_abs[:, :, 0]
    l0, l1 = level.floor().long(), level.ceil().long()
    a0 = _take(samples_abs, l0)
    return a0 + (level - l0)[:, None] * (a0 + _take(samples_abs, l1))


def levels64(grid64, hs, ws, max_level, min_level):
    """The float64 level of detail with the fp32 clamps a launch holds."""
    return S.mipmap_levels(grid64, hs, ws, max_level + 1.0, min_level)


def ulp32(v):
    """Spacing of fp32 in the binade of |v| (float64 tensor), the subnormal spacing below the normal range."""
    _, e = torch.frexp(v.abs())
    e = torch.where(v == 0, torch.full_like(e, -125), e)
    return torch.ldexp(torch.ones_like(v), (torch.clamp(e - 1, min=-126) - 23).to(v.dtype))


def level_error(grid, hs, ws, dyadic):
    """eps_L (N, Ho, Wo): |fp32 level - float64 level| for the grid the kernel reads (fp32 values, exact in float64).
      coordinates  c = (size - 1) (g + 1) / 2: g + 1 and the product round (u |(size-1)(g+1)| together), the halving is
                   exact; on dyadic grids (multiples of 2^-12, |g + 1| < 4, size <= 1024) all of it is exact
      dx = o - c   one rounding of |dx| plus both coordinates' errors (exact on dyadic grids: both lie on the 2^-13 lattice)
      sq           dx*dx + dy*dy: up to three roundings (a contracted multiply-add counts as two): 3 u sq
      d            sqrtf(fmaxf(sq, 1)): |d(sq)| <= |d sq| / (2 sqrt(max(1, sq - |d sq|))), plus its own rounding u d
      dmax         a max of the four: off by at most the largest of their errors
      level        log2f(dmax): the error of dmax over dmax ln 2 (dmax >= 1), plus 1 ulp of the result; the clamps are
                   exact and 1-Lipschitz."""
    g = grid.double()
    c = S.lod_coordinates(g, hs, ws)
    scale = torch.tensor([ws - 1.0, hs - 1.0], dtype=F64)
    dc = torch.zeros_like(c) if dyadic else U32 * (scale * (g + 1.0)).abs()

    def neighbours(t):
        p = F.pad(t.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="replicate").permute(0, 2, 3, 1)
        return [p[:, 1:-1, :-2], p[:, 1:-1, 2:], p[:, :-2, 1:-1], p[:, 2:, 1:-1]]

    dk, ek = [], []
    for o, do in zip(neighbours(c), neighbours(dc)):
        d = o - c
        dd = torch.zeros_like(d) if dyadic else do + dc + U32 * d.abs()
        sq = (d * d).sum(dim=3)
        dsq = (2.0 * d.abs() * dd).sum(dim=3) + 3.0 * U32 * sq
        dist = sq.clamp(min=1.0).sqrt()
        dk.append(dist)
        ek.append(dsq / (2.0 * (sq - dsq).clamp(min=1.0).sqrt()) + U32 * dist)
    dmax = torch.stack(dk).max(dim=0).values
    err = torch.stack(ek).max(dim=0).values
    raw = torch.log2(dmax)
    return err / ((dmax - err).clamp(min=1.0) * LN2) + ulp32(raw + err / LN2)


def level_slope(samples, level, extra):
    """max |S(l+1) - S(l)| over the level segments next to the pixel's level (l = l0 - 1, l0, l1): the output's slope in
    the level on either side of the float64 level.  (N, C, Ho, Wo); zero without mip levels."""
    if level is None or extra == 0:
        return torch.zeros_like(samples[:, :, 0])
    diff = (samples[:, :, 1:] - samples[:, :, :-1]).abs()
    l0, l1 = level.floor().long(), level.ceil().long()
    return torch.stack([_take(diff, l.clamp(0, extra - 1)) for l in (l0 - 1, l0, l1)]).max(dim=0).values


def coordinate_error(grid, hs, ws, mode):
    """(dx, dy) (N, Ho, Wo): |fp32 - float64| of the bilinear source coordinate for a grid that is not dyadic.
    ((g + 1) size - 1) / 2: g + 1, the product and the subtraction round (a contracted multiply-add counts as two), the
    halving is exact; reflection adds three more (in - mn, span - extra, + mn; fmodf is exact).  Each rounding is at most
    u times the largest intermediate, |g + 1| size + size + 1; the border clip is exact and 1-Lipschitz."""
    g = grid.double()
    k = 3 + (3 if mode == "reflection" else 0)
    return [k * U32 * ((g[..., i] + 1.0).abs() * size + size + 1.0) for i, size in ((0, ws), (1, hs))]


def _window_max(t, kh, kw, y0, x0):
    """max of t (N, C, H', W') over the window of kh x kw anchored at (y0, x0) (N, Ho, Wo) -> (N, C, Ho, Wo)."""
    pooled = F.max_pool2d(t, (kh, kw), stride=1)
    n, c, ph, pw = pooled.shape
    idx = (y0.clamp(0, ph - 1) * pw + x0.clamp(0, pw - 1)).reshape(n, 1, -1).expand(n, c, -1)
    return torch.gather(pooled.reshape(n, c, -1), 2, idx).reshape(n, c, *y0.shape[1:])


def bilinear_slopes(stack, grid, mode):
    """(Kx, Ky) per level, each (N, C, K, Ho, Wo): a Lipschitz constant of the bilinear interpolant of each stack level, in
    x and in y, over the cells around the pixel's coordinate (rows y0 - 1 .. y0 + 2, columns x0 - 1 .. x0 + 2), so it holds
    on both sides of the coordinate for any move under a pixel.  Zero padding (zeros mode) or replicate padding (the
    clipped modes) stands for what the sampler reads beyond the image."""
    g = grid.double()
    hs, ws = stack[0].shape[2:]
    x0 = S.source_index(g[..., 0], ws, mode).floor().long()
    y0 = S.source_index(g[..., 1], hs, mode).floor().long()
    kx, ky = [], []
    for s in stack:
        p = F.pad(s, (2, 2, 2, 2)) if mode == "zeros" else F.pad(s, (2, 2, 2, 2), mode="replicate")
        dx = (p[..., :, 1:] - p[..., :, :-1]).abs()
        dy = (p[..., 1:, :] - p[..., :-1, :]).abs()
        # padded row r + 2 holds row r: the window rows y0 - 1 .. y0 + 2 start at y0 + 1, columns x0 - 1 .. x0 + 1 at x0 + 1
        kx.append(_window_max(dx, 4, 3, y0 + 1, x0 + 1))
        ky.append(_window_max(dy, 3, 4, y0 + 1, x0 + 1))
    return torch.stack(kx, dim=2), torch.stack(ky, dim=2)


def corner_c(level):
    """fp32 roundings of one level's bilinear sample, relative to the same sample of |values|: the sum over 4 corners of
    v * (wx * wy) is 2 products and 3 additions (5); a level >= 1 value is itself a bilinear up-sampling with exact weights,
    uy.l0 * (ux.l0 v00 + ux.l1 v01) + ..., a product, an addition, a product, an addition per term (4 more)."""
    return 5 + (4 if level > 0 else 0)


def forward_c(extra):
    """The blend o0 + w (o1 - o0): the difference, the product and the sum (a contraction counts as two: three), over
    A = A0 + w (A0 + A1), on top of the worse of the two levels' corner_c, and one for the products of two roundings."""
    return corner_c(extra) + 3 + 1 if extra > 0 else corner_c(0)
