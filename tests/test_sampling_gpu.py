"""GPU parity of the fused antialiased sampler (csrc/warp.cu) against the reference fixtures and the oracle."""
import pytest
import torch
import torch.nn.functional as F

from conftest import assert_close, golden_cases, load_golden
from fp64_contract import grid_stride_batch
from oracle import sampling as S
from warp_reference import _edge_grid, coordinate_decided, level_atol, level_decided, neighbour_sq, undecided_pixels

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _stn():
    from gangealing_b200 import stn
    return stn


# out / grad_x vs the float64 oracle, relative to the largest entry.  fp32: the source coordinate ((g + 1) * size - 1) / 2
# rounds at ulp(2) * size / 2 (6e-5 px on a 512 px source), which a random image's slopes of a few units per px turn into
# ~1e-4 of the output's magnitude; half precision: the output is rounded to the source's type.
LOW_PRECISION_TOL = {torch.float32: 3e-4, torch.float16: 1e-3, torch.bfloat16: 8e-3}


# level_atol, the "decided" pixels (coordinate_decided, level_decided, undecided_pixels), neighbour_sq and the constructed
# edge grids (_edge_grid) live in warp_reference.py, which test_warp_family_gpu.py shares.
def warp_oracle(x, grid, go, num_levels, min_level, mode):
    """float64 autograd of the oracle on the kernel's inputs (x, grid, go as the kernel sees them) ->
    out, levels, grad_x, grad_grid, and grad_grid with the levels detached (the bilinear part alone)."""
    xd = x.double().requires_grad_(True)
    gd = grid.double().requires_grad_(True)
    out, aux = S.mipmap_warp_ref(xd, gd, num_levels, min_level, mode, return_aux=True)
    gx, gg = torch.autograd.grad(out, [xd, gd], go.double())
    gd2 = grid.double().requires_grad_(True)
    (gg_det,) = torch.autograd.grad(S.mipmap_warp_ref(x.double(), gd2, num_levels, min_level, mode, detach_levels=True),
                                    gd2, go.double())
    return out.detach(), aux["levels"], gx, gg, gg_det


def check_grid_grad(gg, gg_o, gg_det, exempt, rtol, lod_rtol, what, need_lod=True):
    """The kernel's grid gradient vs the float64 oracle on the decided pixels (tolerance relative to its largest entry);
    then its level-of-detail share alone -- kernel minus the oracle with levels detached, vs the oracle's live minus
    detached -- on THAT share's own scale, over the whole grid and over the pixels of the four output borders (where the
    neighbour gather meets the clamps), so that an error in a term much smaller than the bilinear part still shows."""
    gg = gg.detach().double().cpu()
    keep = ~exempt[..., None].expand_as(gg)
    assert_close(gg[keep], gg_o[keep], rtol=rtol, what=what + " grad_grid")
    lod_o, lod_k = gg_o - gg_det, gg - gg_det
    if need_lod:
        assert lod_o[keep].abs().max() > 0, what + ": no level-of-detail gradient to check"
    if lod_o[keep].abs().max() == 0:     # every level clamped: the share is zero, and the check above covers the rest
        return
    assert_close(lod_k[keep], lod_o[keep], rtol=lod_rtol, what=what + " level-of-detail share")
    border = torch.zeros(exempt.shape, dtype=torch.bool)
    border[:, 0] = border[:, -1] = True
    border[:, :, 0] = border[:, :, -1] = True
    keep_b = keep & border[..., None]
    if lod_o[keep_b].abs().max() > 0:
        assert_close(lod_k[keep_b], lod_o[keep_b], rtol=lod_rtol, what=what + " level-of-detail share at the borders")


def test_mipmap_warp_golden_forward_backward_and_levels():
    stn = _stn()
    blob = load_golden("mipmap_warp")
    mw = stn.MipmapWarp(3.5).to(DEV)
    for name in golden_cases(blob):
        mode = S.PAD_MODES[int(blob[name + ".mode"])]
        x = blob[name + ".x"].to(DEV).requires_grad_(True)
        grid = blob[name + ".grid"].to(DEV).requires_grad_(True)
        y = mw(x, grid, padding_mode=mode)
        assert_close(y, blob[name + ".y"], rtol=1e-4, what=name + " fwd")
        gx, gg = torch.autograd.grad(y, [x, grid], blob[name + ".go"].to(DEV))
        assert_close(gx, blob[name + ".gx"], rtol=1e-4, what=name + " gx")
        assert_close(gg, blob[name + ".ggrid"], rtol=1e-3, what=name + " ggrid")
        lv = (mw.levels_map * 2.5).cpu()
        ref_lv = blob[name + ".levels"]
        assert_close(lv, ref_lv, atol=2e-6, what=name + " levels")
        # integer level indices: exact wherever the level is not within float noise of an integer
        safe = (ref_lv - ref_lv.round()).abs() > 1e-5
        assert torch.equal(lv.floor()[safe], ref_lv.floor()[safe]) and torch.equal(lv.ceil()[safe], ref_lv.ceil()[safe])
        # plain Warp
        w = stn.Warp()
        x2 = blob[name + ".x"].to(DEV).requires_grad_(True)
        g2 = blob[name + ".grid"].to(DEV).requires_grad_(True)
        yw = w(x2, g2, padding_mode=mode)
        assert_close(yw, blob[name + ".warp_y"], rtol=1e-5, what=name + " warp fwd")
        gxw, ggw = torch.autograd.grad(yw, [x2, g2], blob[name + ".go"].to(DEV))
        assert_close(gxw, blob[name + ".warp_gx"], rtol=1e-4, what=name + " warp gx")
        assert_close(ggw, blob[name + ".warp_ggrid"], rtol=1e-3, what=name + " warp ggrid")


@pytest.mark.parametrize("size,res,mode", [(128, 128, "border"), (256, 128, "reflection"), (450, 128, "border"),
                                           (512, 512, "border"), (64, 96, "zeros")])
def test_mipmap_warp_vs_oracle_training_shapes(size, res, mode):
    """Forward, levels, grad_x (scatter + pyramid adjoint) and grad_grid (bilinear part + the level-of-detail gather) vs
    float64 autograd of the oracle at the STN's shapes."""
    _check_training_shape(size, res, mode, torch.float32)


@pytest.mark.parametrize("size,res,mode,dtype", [(256, 128, "reflection", torch.float16), (450, 128, "border", torch.bfloat16),
                                                 (64, 96, "zeros", torch.float16), (128, 128, "border", torch.bfloat16)])
def test_mipmap_warp_vs_oracle_half_precision_sources(size, res, mode, dtype):
    """The same with fp16 / bf16 sources: the oracle gets the same rounded source and output gradient (the kernel reads them
    as they are and computes in fp32); out and grad_x are rounded to the source's type, grad_grid is fp32."""
    _check_training_shape(size, res, mode, dtype)


def _check_training_shape(size, res, mode, dtype):
    stn = _stn()
    g = torch.Generator().manual_seed(size + res)
    n = 3
    x = torch.randn(n, 3, size, size, generator=g).to(dtype)
    theta = torch.tensor([[1.0, 0.0, 0.0, 0.0, 1.0, 0.0], [1.9, 0.6, 0.1, -0.6, 1.9, -0.1], [3.0, 0.0, 0.2, 0.0, 3.0, 0.0]]).reshape(3, 2, 3)
    coarse = torch.randn(n, 2, 6, 6, generator=g)
    grid = F.affine_grid(theta, (n, 3, res, res), align_corners=False) + \
        0.08 * F.interpolate(coarse, size=(res, res), mode="bicubic", align_corners=False).permute(0, 2, 3, 1)
    go = torch.randn(n, 3, res, res, generator=g).to(dtype)
    yo, lv_o, gx_o, gg_o, gg_det = warp_oracle(x, grid, go, 3.5, 0.0, mode)
    mw = stn.MipmapWarp(3.5).to(DEV)
    xg, gr = x.to(DEV).requires_grad_(True), grid.to(DEV).requires_grad_(True)
    y = mw(xg, gr, padding_mode=mode)
    assert y.dtype == dtype
    tol = LOW_PRECISION_TOL[dtype]
    assert_close(y, yo, rtol=tol, what="fwd")
    assert_close(mw.levels_map.cpu() * 2.5, lv_o, atol=level_atol(size), what="levels")
    gx, gg = torch.autograd.grad(y, [xg, gr], go.to(DEV))
    assert gx.dtype == dtype and gg.dtype == torch.float32
    assert_close(gx, gx_o, rtol=tol, what="grad_x")
    exempt = undecided_pixels(grid, size, size, mode, 2.5)
    # these grids are affine plus a smooth perturbation: a pixel's left and right (up and down) distances differ only by the
    # perturbation's second difference, so 1-2 % of the pixels hold their top distances within the rounding of the fp32
    # level-of-detail coordinates (5 % on the 512 px source, whose coordinates are larger)
    assert exempt.float().mean() < (0.06 if size >= 512 else 0.03)
    check_grid_grad(gg, gg_o, gg_det, exempt, GRID_RTOL, LOD_RTOL, "%d->%d %s" % (size, res, mode))


# grid-gradient tolerances, relative to the largest entry of the whole gradient / of its level-of-detail share
GRID_RTOL, LOD_RTOL = 1e-4, 1e-4


@pytest.mark.parametrize("mode", S.PAD_MODES)
@pytest.mark.parametrize("case", ["pinch", "ties", "clamps", "clamps_min", "borders"])
def test_mipmap_warp_grid_gradient_edges(case, mode):
    """The gathered grid gradient (csrc/warp.cu warp_bwd_kernel) on constructed grids: one target shared by 2, 3 and 4
    neighbours, exact arg-max ties, distances and levels exactly at their clamps, source coordinates exactly on the
    borders -- vs float64 autograd of the oracle, with its level-of-detail share checked on its own scale."""
    stn = _stn()
    grid, size, num_levels, min_level = _edge_grid(case)
    g = torch.Generator().manual_seed(7)
    n, ho, wo = grid.shape[:3]
    x = torch.randn(n, 3, size, size, generator=g)
    go = torch.randn(n, 3, ho, wo, generator=g)
    max_level = min(num_levels - 1.0, float(stn.sampling.feasible_levels(size, size, num_levels - 1)))
    sq = neighbour_sq(grid.double(), size, size)
    arg = sq.clamp(min=1.0).sqrt().max(dim=0).indices[0]
    if case == "pinch":
        # how many neighbours pick each pixel as their arg-max target
        ty = (torch.arange(ho)[:, None] + torch.tensor([0, 0, -1, 1])[arg]).clamp(0, ho - 1)
        tx = (torch.arange(wo)[None, :] + torch.tensor([-1, 1, 0, 0])[arg]).clamp(0, wo - 1)
        hits = torch.zeros(ho, wo, dtype=torch.long).index_put_((ty.flatten(), tx.flatten()), torch.ones(ho * wo, dtype=torch.long),
                                                                accumulate=True)
        assert hits[8, 8] == 4 and hits[0, 5] == 3 and hits[15, 15] == 2
    if case != "pinch":
        top = sq.clamp(min=1.0).sqrt().topk(2, dim=0).values
        assert ((top[0] == top[1]) & (top[0] > 1)).sum() >= 3           # exact ties with a live gradient
    if case.startswith("clamps"):
        sq_max = sq.max(dim=0).values
        assert (sq_max == 1).any() and (sq_max == 64).any() and (sq_max == 16).any()
    yo, lv_o, gx_o, gg_o, gg_det = warp_oracle(x, grid, go, num_levels, min_level, mode)
    mw = stn.MipmapWarp(num_levels).to(DEV)
    xg, gr = x.to(DEV).requires_grad_(True), grid.to(DEV).requires_grad_(True)
    y = mw(xg, gr, min_level=min_level, padding_mode=mode)
    assert_close(y, yo, rtol=LOW_PRECISION_TOL[torch.float32], what="fwd")
    assert_close(mw.levels_map.cpu() * (num_levels - 1.0), lv_o, atol=level_atol(size), what="levels")
    gx, gg = torch.autograd.grad(y, [xg, gr], go.to(DEV))
    assert_close(gx, gx_o, rtol=1e-4, what="grad_x")
    exempt = undecided_pixels(grid, size, size, mode, max_level, min_level)
    # the dyadic grids are exact in fp32: every pixel is decided, ties and clamps included
    assert exempt.sum() == 0
    check_grid_grad(gg, gg_o, gg_det, exempt, GRID_RTOL, LOD_RTOL, "%s %s" % (case, mode))


def test_mipmap_warp_min_level_and_warp_match_torch_grid_sample():
    stn = _stn()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 5, 32, 40, generator=g)  # non-square, 5 channels: plain Warp only
    grid = torch.rand(2, 17, 23, 2, generator=g) * 2.6 - 1.3
    for mode in S.PAD_MODES:
        y = stn.Warp()(x.to(DEV), grid.to(DEV), padding_mode=mode)
        assert_close(y, F.grid_sample(x, grid, padding_mode=mode, align_corners=False), rtol=1e-5, what=mode)
    x = torch.randn(2, 3, 64, 64, generator=g)
    grid = F.affine_grid(torch.eye(2, 3)[None].repeat(2, 1, 1) * 1.7, (2, 3, 32, 32), align_corners=False)
    mw = stn.MipmapWarp(3.5).to(DEV)
    for min_level in (0.5, 2.0):
        y = mw(x.to(DEV), grid.to(DEV), min_level=min_level)
        assert_close(y, S.mipmap_warp_ref(x, grid, 3.5, min_level, "border"), rtol=1e-4, what="min_level %g" % min_level)


def test_mipmap_warp_low_precision_and_errors():
    stn = _stn()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 3, 64, 64, generator=g)
    grid = F.affine_grid(torch.tensor([[[2.0, 0.1, 0.0], [-0.1, 2.0, 0.0]]]).repeat(2, 1, 1), (2, 3, 32, 32), align_corners=False)
    yo = S.mipmap_warp_ref(x.bfloat16().float(), grid, 3.5, 0.0, "border")
    y = stn.MipmapWarp(3.5).to(DEV)(x.bfloat16().to(DEV), grid.to(DEV))
    assert y.dtype == torch.bfloat16
    assert_close(y, yo, rtol=1.6e-2)
    with pytest.raises(RuntimeError):
        stn.MipmapWarp(3.5)(x, grid)  # CPU tensors
    with pytest.raises(RuntimeError):
        stn.Warp()(x.to(DEV), grid.to(DEV), padding_mode="wrap")
    with pytest.raises(RuntimeError):
        stn.Warp()(x.to(DEV), grid[:1].to(DEV))


def test_bilinear_downsample_golden():
    stn = _stn()
    blob = load_golden("bilinear_downsample")
    for stride in (2, 4):
        y = stn.BilinearDownsample(stride, 3).to(DEV)(blob["x"].to(DEV))
        assert_close(y, blob["s%d.y" % stride], rtol=1e-5)


@pytest.mark.parametrize("shape,stride", [((2, 3, 32, 32), 2), ((1, 3, 33, 29), 2), ((2, 3, 64, 48), 4), ((1, 2, 40, 40), 8),
                                          ((2, 3, 9, 7), 1), ((1, 3, 21, 30), 3), ((4, 3, 256, 256), 2)])
def test_bilinear_downsample_forward_and_adjoint(shape, stride):
    """One-kernel BilinearDownsample vs the oracle (reference antialiased_sampling.py:241-256): forward, and the
    gather-form backward against autograd of the reference formulation."""
    stn = _stn()
    g = torch.Generator().manual_seed(shape[2] * 7 + stride)
    x = torch.randn(*shape, generator=g)
    xo = x.clone().requires_grad_(True)
    yo = S.bilinear_downsample_ref(xo, stride)
    go = torch.randn(yo.shape, generator=g)
    (gxo,) = torch.autograd.grad(yo, xo, go)
    mod = stn.BilinearDownsample(stride, shape[1]).to(DEV)
    xg = x.to(DEV).requires_grad_(True)
    y = mod(xg)
    assert y.shape == yo.shape
    assert_close(y, yo, rtol=1e-5, what="forward")
    (gx,) = torch.autograd.grad(y, xg, go.to(DEV))
    assert_close(gx, gxo, rtol=1e-5, what="backward")
    lhs = (y.detach().double() * go.to(DEV).double()).sum()
    rhs = (xg.detach().double() * gx.double()).sum()
    assert abs(lhs - rhs) <= 1e-6 * (y.detach().double() * go.to(DEV).double()).abs().sum()


def test_bilinear_downsample_errors():
    stn = _stn()
    with pytest.raises(RuntimeError):
        stn.BilinearDownsample(2, 3)(torch.zeros(1, 3, 8, 8))             # CPU tensor: no fallback
    with pytest.raises(RuntimeError):
        stn.BilinearDownsample(4, 3).to(DEV)(torch.zeros(1, 3, 2, 2, device=DEV))   # plane not larger than stride/2
    y = stn.BilinearDownsample(2, 3).to(DEV)(torch.zeros(0, 3, 8, 8, device=DEV))
    assert y.shape == (0, 3, 4, 4)


@pytest.mark.parametrize("mode", ["zeros", "border", "reflection"])
@pytest.mark.parametrize("hs,ws", [(128, 128), (64, 256)])
def test_sampler_integer_work_is_bit_exact(mode, hs, ws):
    """The sampler's INTEGER work compared as integers (north_star: "bit-exact for sampling-grid integer/index work"):
    bilinear corner indices (x0, y0) after the padding-mode transform and the floor / ceil level indices, exported by
    gg_warp_sample_indices from the device functions the sampling kernels call, vs the oracle's
    (oracle/sampling.py grid_sample_bilinear / mipmap_levels = ATen grid_sampler + antialiased_sampling.py:197-229).

    (a) DYADIC grid: every coordinate k/512 -- all of ((g+1)*size-1)/2, the reflection fold and the floor are exact in
        fp32 on both sides (no rounding, so FMA contraction cannot matter): ALL pixels must agree, including the exact
        ties where the source coordinate IS an integer and the far out-of-range coordinates of every padding mode.
    (b) random smooth grid: exact wherever the oracle's coordinate is not within 1e-4 px of an integer (there the last
        ulp of the fp32 evaluation order decides, on the GPU as in ATen's own CUDA kernel); that exempt set must be tiny."""
    from gangealing_b200.stn import sampling as GS
    g = torch.Generator().manual_seed(hs + ws)
    n, ho, wo = 2, 96, 80
    k = torch.randint(-900, 900, (n, ho, wo, 2), generator=g)
    k[0, :8, :8] = torch.tensor([4, -4])                 # exact ties: coordinate lands on an integer pixel
    k[0, 8:16, :8] = torch.tensor([-512, 512])           # the two borders of the normalised range
    dyadic = k.float() / 512.0
    theta = torch.tensor([[[0.9, 0.2, 0.05], [-0.15, 1.3, -0.1]], [[2.2, 0.0, 0.3], [0.1, 1.9, 0.0]]])
    smooth = F.affine_grid(theta, (n, 1, ho, wo), align_corners=False) + 0.03 * torch.randn(n, ho, wo, 2, generator=g)
    img = torch.zeros(n, 1, hs, ws)
    for name, grid in (("dyadic", dyadic), ("smooth", smooth)):
        got = GS.sample_indices(grid.to(DEV), (hs, ws), 3.5, 0.0, mode).cpu()
        _, (x0, y0) = S.grid_sample_bilinear(img, grid, mode)
        lv = S.mipmap_levels(grid, hs, ws, 3.5)
        ix = S.source_index(grid[..., 0], ws, mode)
        iy = S.source_index(grid[..., 1], hs, mode)
        if name == "dyadic":
            corner_ok = torch.ones_like(x0, dtype=torch.bool)
        else:
            corner_ok = coordinate_decided(ix, ws, mode) & coordinate_decided(iy, hs, mode)
            assert corner_ok.float().mean() > 0.995
        assert torch.equal(got[..., 0][corner_ok].long(), x0[corner_ok]), name + " x0"
        assert torch.equal(got[..., 1][corner_ok].long(), y0[corner_ok]), name + " y0"
        level_ok = level_decided(lv)
        assert level_ok.float().mean() > 0.995
        assert torch.equal(got[..., 2][level_ok].long(), lv.floor().long()[level_ok]), name + " floor(level)"
        assert torch.equal(got[..., 3][level_ok].long(), lv.ceil().long()[level_ok]), name + " ceil(level)"


# ------------------------------------------------------------------------------------------------ one-pass STN sampler
def _kernel_grid_grad(x, grid, go, levels, mode):
    """The sampler's own backward (the kernel stn_sample_* call) on a given grid: its gradient w.r.t. the grid."""
    from gangealing_b200.stn import sampling as GS
    gk = grid.detach().requires_grad_(True)
    if levels is None:
        y = GS.grid_sample_bilinear(x, gk, mode)
    else:
        y = GS.mipmap_warp(x, gk, levels, 0.0, mode)[0]
    return torch.autograd.grad(y, gk, go)[0].double().cpu()


def _sampler_oracle(x, grid, go, levels, mode, hs, ws, affine):
    """The sampling stage of stn_sample_* on the grid the kernel generated (`grid`, returned by it; checked against the
    oracle's generator by the caller) -> float64 oracle out, levels, grad_x, and the kernel's own per-pixel grid gradient
    (its sampler backward on that grid), checked per pixel against the oracle's on the decided pixels.  The caller checks
    the grid generator's backward against float64 autograd of the oracle's generator fed with THAT gradient: a sum over
    pixels (g_theta, g_base, g_low) would otherwise inherit the O(1) jumps of the few undecided pixels.
    `affine` with levels: an affine grid has equal left / right (and up / down) neighbour distances at every pixel, so
    rounding picks the level-of-detail arg-max everywhere and no pixel is decided; the per-pixel grid gradient is left to the
    MipmapWarp tests above (non-affine grids, and exact ties on dyadic grids).  g_theta does not depend on that choice."""
    xd = x.double().requires_grad_(True)
    gl = grid.detach().double().cpu().requires_grad_(True)
    if levels is None:
        out, lv, gg_det = S.warp_ref(xd, gl, mode), None, None
    else:
        out, aux = S.mipmap_warp_ref(xd, gl, levels, 0.0, mode, return_aux=True)
        lv = aux["levels"]
        gd2 = gl.detach().clone().requires_grad_(True)
        (gg_det,) = torch.autograd.grad(S.mipmap_warp_ref(x.double(), gd2, levels, 0.0, mode, detach_levels=True), gd2, go.double())
    gx, gg = torch.autograd.grad(out, [xd, gl], go.double())
    gg_k = _kernel_grid_grad(x.to(DEV), grid, go.to(DEV), levels, mode)
    if not (affine and levels is not None):
        exempt = undecided_pixels(gl.detach(), hs, ws, mode, None if levels is None else levels - 1.0)
        assert exempt.float().mean() < 0.005
        if levels is None:
            keep = ~exempt[..., None].expand_as(gg)
            assert_close(gg_k[keep], gg[keep], rtol=GRID_RTOL, what="sampler grid gradient")
        else:
            check_grid_grad(gg_k, gg, gg_det, exempt, GRID_RTOL, LOD_RTOL, "sampler", need_lod=False)
    return out.detach(), lv, gx, gg_k


def _check_stn_affine(n, out_hw, levels, mode, dtype, seed=0):
    from gangealing_b200.stn import sampling as GS
    g = torch.Generator().manual_seed(seed + out_hw[0] * 1000 + out_hw[1])
    hs = ws = 128
    ho, wo = out_hw
    x = torch.randn(n, 3, hs, ws, generator=g).to(dtype)
    # zoom in and out, rotation / shear, translation
    theta = torch.eye(2, 3)[None] * (0.5 + 1.5 * torch.rand(n, 1, 1, generator=g)) + 0.15 * torch.randn(n, 2, 3, generator=g)
    go = torch.randn(n, 3, ho, wo, generator=g).to(dtype)
    g_grid = torch.randn(n, ho, wo, 2, generator=g)          # the caller also uses the returned grid
    x_dev, go_dev = x.to(DEV), go.to(DEV)
    xg, tg = x_dev.clone().requires_grad_(True), theta.to(DEV).requires_grad_(True)
    out, grid, lv = GS.stn_sample_affine(xg, tg, out_hw, levels, 0.0, mode)
    gx, gth = torch.autograd.grad((out.float() * go_dev.float()).sum() + (grid * g_grid.to(DEV)).sum(), [xg, tg])
    # oracle
    th = theta.double().requires_grad_(True)
    grid_o = S.affine_grid_ref(th, (n, 3, ho, wo))
    assert_close(grid, grid_o, rtol=1e-6, what="grid")
    out_o, lv_o, gx_o, gg_k = _sampler_oracle(x, grid, go, levels, mode, hs, ws, affine=True)
    tol = LOW_PRECISION_TOL[dtype]
    assert out.dtype == dtype and gx.dtype == dtype
    assert_close(out, out_o, rtol=tol, what="out")
    if levels is None:
        assert lv is None
    else:
        assert_close(lv, lv_o, atol=level_atol(hs), what="levels")
    assert_close(gx, gx_o, rtol=tol, what="grad_x")
    (gth_o,) = torch.autograd.grad(grid_o, th, gg_k + g_grid.double())
    assert_close(gth, gth_o, rtol=1e-4, what="g_theta")


@pytest.mark.parametrize("mode", S.PAD_MODES)
@pytest.mark.parametrize("levels", [None, 4])
@pytest.mark.parametrize("out_hw", [(128, 128), (100, 60), (7, 300), (1, 1)])
def test_stn_sample_affine_vs_oracle(out_hw, levels, mode):
    """The one-pass sampler (csrc/warp.cu warp_compose_fwd_kernel: affine grid generated in 32x8 tiles with a clamped halo)
    and its hand-written backward (stn/sampling.py _StnSample) vs affine_grid_ref + mipmap_warp_ref in float64: out, the
    returned grid and levels, grad_x and g_theta.  Output sizes: training, tiles overhanging the image, a single pixel
    (every neighbour clamps onto itself)."""
    _check_stn_affine(3, out_hw, levels, mode, torch.float32)


FLOW_CASES = [  # low h, w, s, base warp, alpha, max_num_levels, padding mode
    (16, 16, 8, True, None, 4, "border"), (16, 16, 8, False, "n", 4, "reflection"), (16, 16, 8, True, "1", None, "zeros"),
    (12, 20, 4, True, "1", 4, "zeros"), (12, 20, 4, False, None, None, "border"), (12, 20, 4, True, "n", 4, "reflection"),
    (7, 9, 1, True, "n", 4, "reflection"), (7, 9, 1, False, "1", None, "zeros"), (7, 9, 1, False, None, 4, "border")]


def _check_stn_flow(n, lh, lw, s, with_base, alpha_kind, levels, mode, dtype, seed=0):
    from gangealing_b200.stn import sampling as GS
    from oracle import flow as FL
    g = torch.Generator().manual_seed(seed + lh * 100 + lw + s)
    ho, wo = lh * s, lw * s
    hs = ws = 128 if s > 1 else 32
    x = torch.randn(n, 3, hs, ws, generator=g).to(dtype)
    low = (0.1 / s) * torch.randn(n, lh, lw, 2, generator=g)
    mask = 2.0 * torch.randn(n, 9 * s * s, lh, lw, generator=g)
    base = (torch.eye(2, 3)[None] * 1.4 + 0.1 * torch.randn(n, 2, 3, generator=g)) if with_base else None
    alpha = {None: None, "n": torch.rand(n, generator=g), "1": torch.rand(1, generator=g)}[alpha_kind]
    ident = S.affine_grid_ref(torch.eye(2, 3)[None], (1, 1, ho, wo))
    go = torch.randn(n, 3, ho, wo, generator=g).to(dtype)
    g_flow, g_delta = torch.randn(n, ho, wo, 2, generator=g), torch.randn(n, ho, wo, 2, generator=g)   # the TV loss's use
    x_dev, go_dev = x.to(DEV), go.to(DEV)
    leaves = [t.to(DEV).requires_grad_(True) for t in ([low, mask] + ([base] if with_base else []))]
    out, flow, delta, lv = GS.stn_sample_flow(x_dev, leaves[0], leaves[1], ident.to(DEV), leaves[2] if with_base else None,
                                              None if alpha is None else alpha.to(DEV), s, levels, 0.0, mode)
    loss = (out.float() * go_dev.float()).sum() + (flow * g_flow.to(DEV)).sum() + (delta * g_delta.to(DEV)).sum()
    grads = torch.autograd.grad(loss, leaves)
    # oracle
    leaves_o = [t.double().requires_grad_(True) for t in ([low, mask] + ([base] if with_base else []))]
    delta_o, flow_o = FL.flow_compose_ref(leaves_o[0], leaves_o[1], ident.double(), leaves_o[2] if with_base else None,
                                          None if alpha is None else alpha.double(), s)
    assert_close(delta, delta_o, rtol=1e-5, what="delta")
    assert_close(flow, flow_o, rtol=1e-5, what="flow")
    out_o, lv_o, _, gg_k = _sampler_oracle(x, flow, go, levels, mode, hs, ws, affine=False)
    assert out.dtype == dtype
    assert_close(out, out_o, rtol=LOW_PRECISION_TOL[dtype], what="out")
    if levels is None:
        assert lv is None
    else:
        assert_close(lv, lv_o, atol=level_atol(hs), what="levels")
    grads_o = torch.autograd.grad([flow_o, delta_o], leaves_o, [gg_k + g_flow.double(), g_delta.double()])
    for a, e, nm in zip(grads, grads_o, ("g_low", "g_mask", "g_base")):
        assert_close(a, e, rtol=1e-4, what=nm)


@pytest.mark.parametrize("lh,lw,s,with_base,alpha,levels,mode", FLOW_CASES)
def test_stn_sample_flow_vs_oracle(lh, lw, s, with_base, alpha, levels, mode):
    """The one-pass flow sampler (RAFT convex up-sampling + identity + base warp + alpha generated inside the sampler) and
    its backward (sampler backward, then csrc/flow.cu) vs flow_compose_ref + mipmap_warp_ref in float64, with a loss that
    also uses the returned flow and delta (as the TV loss does): out, flow, delta, levels, g_low, g_mask, g_base.
    Low-res sizes: training (16x16, s=8), non-square with 80 columns (not a multiple of the 32-wide tile), s=1."""
    _check_stn_flow(3, lh, lw, s, with_base, alpha, levels, mode, torch.float32)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_stn_sample_low_precision_sources(dtype):
    """Half-precision sources: the kernels read them as they are and compute in fp32; the oracle gets the same rounded
    source and output gradient, so g_theta / g_low / g_mask / g_base keep the fp32 bound and only `out` is rounded."""
    _check_stn_affine(3, (128, 128), 4, "border", dtype)
    _check_stn_flow(3, 16, 16, 8, True, "n", 4, "reflection", dtype)


def test_stn_sample_beyond_the_grid_stride_cap():
    """Batch-32-and-up sampling at 128^2: more output pixels than the capped grids have threads, so the backward kernels
    (warp_bwd_kernel, flow_compose_bwd_kernel) make a second trip through their grid-stride loops."""
    n = grid_stride_batch(128, 128)
    _check_stn_affine(n, (128, 128), 4, "border", torch.float32, seed=1)
    _check_stn_flow(n, 16, 16, 8, True, "n", 4, "border", torch.float32, seed=1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", S.PAD_MODES)
@pytest.mark.parametrize("levels", [None, 4])
@pytest.mark.parametrize("out_hw", [(128, 128), (100, 60), (7, 300), (1, 1)])
def test_one_sampler_for_given_and_generated_grids(out_hw, levels, mode, dtype):
    """One forward kernel samples every grid: mipmap_warp (Warp and grid_sample_bilinear without levels) on the grid that
    stn_sample_affine generated reproduce its output and level map bit for bit.  The odd sizes overhang the 32x8 tiles of
    a read grid, and (1, 1) clamps every neighbour onto the pixel itself."""
    stn = _stn()
    from gangealing_b200.stn import sampling as GS
    g = torch.Generator().manual_seed(out_hw[0] * 1000 + out_hw[1])
    n = 3
    x = torch.randn(n, 3, 128, 128, generator=g).to(dtype).to(DEV)
    theta = torch.eye(2, 3)[None] * (0.5 + 1.5 * torch.rand(n, 1, 1, generator=g)) + 0.15 * torch.randn(n, 2, 3, generator=g)
    with torch.no_grad():
        out, grid, lv = GS.stn_sample_affine(x, theta.to(DEV), out_hw, levels, 0.0, mode)
        if levels is None:
            assert torch.equal(stn.Warp()(x, grid, mode), out)
            assert torch.equal(GS.grid_sample_bilinear(x, grid, mode), out)
        else:
            out_g, lv_g = GS.mipmap_warp(x, grid, levels, 0.0, mode)
            assert torch.equal(out_g, out)
            assert torch.equal(lv_g, lv)


@pytest.mark.parametrize("lh,lw,s,with_base,alpha,levels,mode", FLOW_CASES)
def test_one_flow_composition_for_op_and_sampler(lh, lw, s, with_base, alpha, levels, mode):
    """The stand-alone flow_compose and the one-pass flow sampler compose the same grid bit for bit, and sampling that grid
    with mipmap_warp (grid_sample_bilinear without levels) reproduces the one-pass output and level map."""
    from gangealing_b200.stn import flow as GF
    from gangealing_b200.stn import sampling as GS
    g = torch.Generator().manual_seed(lh * 100 + lw + s)
    n = 3
    ho, wo = lh * s, lw * s
    hs = ws = 128 if s > 1 else 32
    x = torch.randn(n, 3, hs, ws, generator=g).to(DEV)
    low = ((0.1 / s) * torch.randn(n, lh, lw, 2, generator=g)).to(DEV)
    mask = (2.0 * torch.randn(n, 9 * s * s, lh, lw, generator=g)).to(DEV)
    base = (torch.eye(2, 3)[None] * 1.4 + 0.1 * torch.randn(n, 2, 3, generator=g)).to(DEV) if with_base else None
    alpha = {None: None, "n": torch.rand(n, generator=g), "1": torch.rand(1, generator=g)}[alpha]
    alpha = None if alpha is None else alpha.to(DEV)
    ident = S.affine_grid_ref(torch.eye(2, 3)[None], (1, 1, ho, wo)).to(DEV)
    with torch.no_grad():
        out, flow, delta, lv = GS.stn_sample_flow(x, low, mask, ident, base, alpha, s, levels, 0.0, mode)
        delta_c, flow_c = GF.flow_compose(low, mask, ident, base, alpha, s)
        assert torch.equal(delta_c, delta)
        assert torch.equal(flow_c, flow)
        if levels is None:
            assert torch.equal(GS.grid_sample_bilinear(x, flow, mode), out)
        else:
            out_g, lv_g = GS.mipmap_warp(x, flow, levels, 0.0, mode)
            assert torch.equal(out_g, out)
            assert torch.equal(lv_g, lv)
