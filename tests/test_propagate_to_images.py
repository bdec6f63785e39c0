"""Dense labels and edits on real images (gangealing_b200.evaluation.propagate, ComposedSTN.congeal_and_grid and the fused
lookup-splat-composite grid op, csrc/splat.cu) against the reference fixture (oracle/make_golden_propagate.py), the
reference's composition on the device and the float64 restatement (oracle/propagate.py).

uint8 grids are compared value by value: the STN here and the reference's round their convolutions in different orders,
so a value near a quantisation step may round the other way.  At most 0.5 % of the stored values may differ, each by 1."""
import math

import numpy as np
import pytest
import torch
from PIL import Image
from torchvision.utils import make_grid, save_image

from conftest import load_golden
from oracle import make_golden_propagate as GPR
from oracle import opset
from oracle import propagate as OPR
from vis_reference import fp32_stn

DEV = "cuda"
CASES = [c[0] for c in GPR.CASES]
DIFFER_BOUND = 0.005
GRIDS = ("input_images", "congealed_images", "propagated", "average_annotated")


def _mirror(ops, **kw):
    from gangealing_b200.stn import get_stn
    return opset.fill_parameters(get_stn(["similarity", "flow"], ops=ops, **{**GPR.STN_KW, **kw}).eval(), GPR.WEIGHT_SEED,
                                 gain=GPR.WEIGHT_GAIN)


def _count_images(t):
    seen = [0]
    handle = t.stns[-1].register_forward_hook(lambda m, inp, out: seen.__setitem__(0, seen[0] + inp[0].size(0)))
    return seen, handle


def _label(blob, name, tmp_path, device):
    from gangealing_b200.evaluation import load_dense_label
    n, seed, objects, iters, resolution, png_size, n_mean = blob[name + ".cfg"].tolist()
    path = str(tmp_path / ("%s.png" % name))
    Image.fromarray(blob[name + ".label"].numpy()).save(path)
    points, colors, alpha = load_dense_label(path, resolution=resolution, load_colors=bool(objects), device=device)
    return points, colors, alpha


def _run(ops, blob, name, tmp_path, device="cpu", individual=False):
    from gangealing_b200.evaluation import average_congealed_image, average_png, propagate_to_images
    n, seed, objects, iters, resolution, png_size, n_mean = blob[name + ".cfg"].tolist()
    points, colors, alpha = _label(blob, name, tmp_path, device)
    if not objects:
        colors, alpha = blob[name + ".colors"].to(device), None
    t = _mirror(ops).to(device)
    images = GPR.case_images(seed, n).to(device)
    png = average = None
    with torch.no_grad():
        if n_mean > 0:
            batches = [GPR.case_images(seed + 1000 + i, 4).to(device) for i in range(3)]
            mean = average_congealed_image(t, batches, n_mean, output_resolution=GPR.SIZE, iters=iters)
            png, average = average_png(mean, ops)
        res = propagate_to_images(t, images, points[0], colors, alpha, GPR.SIGMA, GPR.OPACITY, resolution=resolution,
                                  output_resolution=GPR.SIZE, average_image=average, iters=iters, individual=individual)
    return res, png


def _compare(got, want, what, step=1):
    """At most DIFFER_BOUND of the values differ, each by at most `step`."""
    got = got.cpu()
    assert got.shape == want.shape, "%s: shape %s vs %s" % (what, tuple(got.shape), tuple(want.shape))
    d = (got.int() - want.int()).abs()
    differ = int((d > 0).sum())
    assert int(d.max()) <= step and differ <= DIFFER_BOUND * want.numel(), "%s: %d of %d values differ (max %d)" % (
        what, differ, want.numel(), int(d.max()))
    return differ


def _check_fixture(blob, name, res, png):
    """With iters > 1 the similarity STN warps its own output again and the two STNs' rounding compounds (make_golden_vis
    allows 5x the one-pass tolerance): a propagated value where a splat edge is steep may then move by 2."""
    assert torch.equal(res["flips"].cpu(), blob[name + ".flips"]), name
    step = 1 if blob[name + ".cfg"][3].item() == 1 else 2
    for g in GRIDS:
        key = "%s.%s" % (name, g)
        if key in blob:
            differ = _compare(res[g], blob[key], key, step)
            print("%s: %d of %d values differ from the reference" % (key, differ, blob[key].numel()))
        else:
            assert g not in res
    if png is not None:
        _compare(png, blob[name + ".average_png"], name + " average.png")
    err = (res["correspondences"].cpu() - blob[name + ".correspondences"]).abs().max().item()
    assert err <= 2e-3, "%s: correspondences differ by %.2e pixels" % (name, err)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", CASES)
def test_api_on_the_oracle_reproduces_the_reference_fixture(name, tmp_path):
    """propagate_to_images (and average_png) on oracle.propagate.cpu_ops(): the script's four grids, average.png, the
    flips and the correspondences; the STN sees every image twice."""
    blob = load_golden("propagate_to_images")
    _check_fixture(blob, name, *_run(OPR.cpu_ops(), blob, name, tmp_path))


@pytest.mark.parametrize("name", CASES)
def test_load_dense_label_equals_the_reference_loader(name, tmp_path):
    """Point order, colours and alpha exactly as helpers.load_dense_label returns them (the resize quirk included)."""
    blob = load_golden("propagate_to_images")
    points, colors, alpha = _label(blob, name, tmp_path, "cpu")
    assert torch.equal(points, blob[name + ".label_points"])
    assert torch.equal(alpha, blob[name + ".label_alpha"])
    if name + ".label_colors" in blob:
        assert torch.equal(colors, blob[name + ".label_colors"])
    else:
        assert colors is None


@pytest.mark.parametrize("n", [2, 4, 5])
def test_pad_value_minus_one_stores_the_bytes_of_pad_value_zero(n, tmp_path):
    """write()'s save_image(normalize=True, range=(-1, 1), padding=3, pad_value=-1) stores the same PNG bytes as the pad
    value 0 the grid kernels write: the pad is not normalised, and -1 * 255 + 0.5 clamps to 0 as 0 * 255 + 0.5 truncates."""
    g = torch.Generator().manual_seed(n)
    images = torch.randn(n, 3, 11, 11, generator=g) * 1.2
    nrow = int(math.sqrt(n))
    save_image(images, str(tmp_path / "a.png"), nrow=nrow, padding=3, pad_value=-1.0, normalize=True, value_range=(-1, 1))
    zero = make_grid(images, nrow=nrow, padding=3, pad_value=0, normalize=True, value_range=(-1, 1))
    zero = zero.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)
    assert np.array_equal(np.asarray(Image.open(str(tmp_path / "a.png"))), zero.numpy())


@pytest.mark.parametrize("no_flip_inference", [False, True])
def test_one_stn_pass_per_batch(no_flip_inference):
    """The flip, the congealed images and the grid come from one forward: 2N images through the flow STN with flip
    inference, N without (the reference runs 4N)."""
    from gangealing_b200.evaluation import propagate_to_images
    t = _mirror(OPR.cpu_ops(), flow_size=64, supersize=128)
    images = GPR.case_images(5, 3)[..., ::2, ::2].contiguous()
    label = torch.tensor([[3, 4], [10, 20], [31, 0]])
    seen, handle = _count_images(t)
    res = propagate_to_images(t, images, label, torch.zeros(1, 3, 3), resolution=32, no_flip_inference=no_flip_inference)
    handle.remove()
    assert seen[0] == (1 if no_flip_inference else 2) * images.size(0)
    assert res["propagated"].shape == res["input_images"].shape and res["correspondences"].shape == (3, 3, 2)
    if no_flip_inference:
        assert not bool(res["flips"].any())


def test_abi_rejects_bad_arguments():
    """Validation runs before any device work; a non-null dummy pointer is never dereferenced."""
    from gangealing_b200 import _lib
    dll = _lib.load()
    one = 16

    def err():
        return dll.gg_last_error().decode()

    def call(out=one, pts=one, ws=one, ws_bytes=1 << 20, images=one, grid=one, query=one, flip=one, colors=one, alpha=one,
             sigma=1.3, opacity=0.75, N=4, P=5, query_n=1, C=3, R=8, gh=4, gw=4, nrow=2, padding=3, colors_n=1, alpha_n=4):
        return dll.gg_splat_lookup_composite_grid(out, pts, ws, ws_bytes, images, grid, query, flip, colors, alpha, sigma,
                                                  opacity, N, P, query_n, C, R, gh, gw, nrow, padding, colors_n, alpha_n,
                                                  None)

    assert call(out=None) == -1 and "null" in err()
    assert call(images=None) == -1 and "null" in err()
    for k in ("grid", "query", "colors", "ws"):
        assert call(**{k: None}) == -1 and "null" in err(), k
    assert call(sigma=0.0) == -1 and "sigma" in err()
    assert call(sigma=float("nan")) == -1 and "sigma" in err()
    assert call(opacity=1.5) == -1 and "opacity" in err()
    assert call(C=4) == -1 and "C must be 3" in err()
    assert call(ws=one + 4) == -1 and "16-byte" in err()
    for k in ("query", "grid", "pts"):
        assert call(**{k: one + 4}) == -1 and "8-byte" in err(), k
    assert call(ws_bytes=100) == -1 and "workspace" in err()
    assert call(query_n=2) == -1 and "query_n" in err()
    assert call(colors_n=3) == -1 and "colors_n" in err()
    assert call(alpha_n=2) == -1 and "alpha_n" in err()
    assert call(N=0) == -1 and call(R=0) == -1 and call(nrow=0) == -1 and call(P=-1) == -1
    assert call(gh=0) == -1 and call(gw=0) == -1 and call(padding=-1) == -1
    assert call(R=40000, N=2, P=0) == -1 and "2^31" in err()
    assert call(N=1 << 20, P=1 << 12, R=1, alpha_n=1) == -1 and "2^31" in err()


# ------------------------------------------------------------------------------------------------ GPU
def _grid_inputs(g, n, r, gs, p):
    """Smooth sampling grids (N, gs, gs, 2) near the identity and queries (1, P, 2) in [-1, 1]."""
    import torch.nn.functional as F
    ident = F.affine_grid(torch.eye(2, 3).unsqueeze(0).repeat(n, 1, 1), (n, 3, gs, gs), align_corners=False)
    grid = ident * 0.9 + F.interpolate(torch.randn(n, 2, 4, 4, generator=g) * 0.05, size=(gs, gs), mode="bilinear",
                                       align_corners=False).permute(0, 2, 3, 1)
    query = torch.rand(1, p, 2, generator=g) * 2.2 - 1.1
    return grid, query


@pytest.mark.gpu
@pytest.mark.parametrize("with_flip", [False, True])
def test_points_out_is_the_fused_lookup_then_the_flip(with_flip):
    """points_out equals splat2d_lookup's points bitwise, mirrored by torch's (R - 1) - x where flipped."""
    from gangealing_b200.splat2d import splat2d_lookup, splat_lookup_composite_grid
    g = torch.Generator().manual_seed(800 + with_flip)
    n, r, gs, p = 4, 96, 48, 3000
    grid, query = _grid_inputs(g, n, r, gs, p)
    flip = torch.tensor([False, True, True, False]) if with_flip else None
    images = (torch.randn(n, 3, r, r, generator=g) * 0.7).to(DEV)
    colors = (torch.rand(1, p, 3, generator=g) * 2 - 1).to(DEV)
    _, got = splat_lookup_composite_grid(images, grid.to(DEV), query.to(DEV), None if flip is None else flip.to(DEV),
                                         colors, None, 1.3, 0.75, 2, padding=3)
    _, want = splat2d_lookup(torch.zeros(n, 3, r, r, device=DEV), grid.to(DEV), query.expand(n, p, 2).contiguous().to(DEV),
                             colors.expand(n, p, 3).contiguous(), torch.full((n,), 1.3, device=DEV), r, r)
    if flip is not None:
        want[:, :, 0] = torch.where(flip.to(DEV).view(-1, 1), r - 1 - want[:, :, 0], want[:, :, 0])
    assert torch.equal(got, want)


def _device_composition(images, grid, query, flip, colors, alpha, sigma, opacity, nrow):
    """The reference's composition on the device: uncongeal_points' lookup (the fused splat2d_lookup's points, which
    test_splat.py holds to grid_sample + unnormalize), torch's flip, splat_points' two splat2d calls, the alpha blend and
    write()'s make_grid(pad_value=-1) + quantisation."""
    from gangealing_b200.opset import cuda_ops
    from gangealing_b200.splat2d import splat2d_lookup
    ops = cuda_ops()
    n, _, r, _ = images.shape
    p = query.size(1)
    sig = torch.full((n,), sigma, device=DEV)
    _, pts = splat2d_lookup(torch.zeros(n, 3, r, r, device=DEV), grid, query.expand(n, p, 2).contiguous(),
                            colors.expand(n, p, 3).contiguous(), sig, r, r)
    if flip is not None:
        pts[:, :, 0] = torch.where(flip.view(-1, 1), r - 1 - pts[:, :, 0], pts[:, :, 0])
    al = torch.ones(n, p, 1, device=DEV) if alpha is None else alpha.expand(n, p, 1).contiguous()
    obj = ops.splat2d(torch.zeros(n, 3, r, r, device=DEV), pts, colors.expand(n, p, 3).contiguous(), sig, False)
    mask = ops.splat2d(torch.zeros(n, 1, r, r, device=DEV), pts, al, sig, True) * opacity
    out = mask * obj + (1 - mask) * images
    grid_img = make_grid(out, nrow=nrow, padding=3, pad_value=-1.0, normalize=True, value_range=(-1, 1))
    return grid_img.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8), pts


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(3))
def test_sparse_label_is_bitwise_the_device_composition(case):
    """Queries that land at most two per pixel neighbourhood (a 12-pixel lattice of identity-grid lookups, pairs within
    0.8 pixels): the grid equals uncongeal_points + the flip + two splat2d calls + the blend + make_grid, bitwise."""
    import torch.nn.functional as F
    from gangealing_b200.splat2d import splat_lookup_composite_grid
    n, r, with_alpha = [(4, 96, True), (3, 130, False), (1, 96, False)][case]
    g = torch.Generator().manual_seed(900 + case)
    ident = F.affine_grid(torch.eye(2, 3).unsqueeze(0).repeat(n, 1, 1), (n, 3, r, r), align_corners=False)
    ys, xs = torch.meshgrid(torch.arange(4, r - 3, 12).float(), torch.arange(4, r - 3, 12).float(), indexing="ij")
    sites = torch.stack([xs.flatten(), ys.flatten()], -1) + torch.rand(xs.numel(), 2, generator=g) * 2 - 1
    pix = torch.cat([sites, sites + torch.rand(sites.shape, generator=g) * 1.6 - 0.8], 0)
    query = ((pix + 0.5) / r * 2 - 1).unsqueeze(0)     # identity-grid pixel centres
    p = query.size(1)
    flip = (torch.arange(n) % 2 == 1).to(DEV)
    images = (torch.randn(n, 3, r, r, generator=g) * 0.8).to(DEV)
    colors = (torch.rand(n, p, 3, generator=g) * 2.4 - 1.2).to(DEV)
    alpha = torch.rand(1, p, 1, generator=g).to(DEV) if with_alpha else None
    got, got_pts = splat_lookup_composite_grid(images, ident.to(DEV), query.to(DEV), flip, colors, alpha, 1.3, 0.75,
                                               int(n ** 0.5), padding=3)
    want, pts = _device_composition(images, ident.to(DEV), query.to(DEV), flip, colors, alpha, 1.3, 0.75, int(n ** 0.5))
    assert torch.equal(got_pts, pts)
    assert torch.equal(got, want), "%d of %d values differ" % (int((got != want).sum()), got.numel())


@pytest.mark.gpu
def test_dense_label_vs_float64_oracle():
    """A dense label (every query of a 160^2 lattice, overlapping footprints): every value equals the float64
    restatement's, or differs by 1 where its v * 255 + 0.5 lies within 1e-3 of an integer."""
    from gangealing_b200.splat2d import splat_lookup_composite_grid
    g = torch.Generator().manual_seed(1000)
    n, r, gs = 4, 128, 64
    grid, _ = _grid_inputs(g, n, r, gs, 1)
    ys, xs = torch.meshgrid(torch.linspace(-0.8, 0.8, 160), torch.linspace(-0.8, 0.8, 160), indexing="ij")
    query = torch.stack([xs.flatten(), ys.flatten()], -1).unsqueeze(0)
    p = query.size(1)
    flip = torch.tensor([True, False, False, True])
    images = torch.randn(n, 3, r, r, generator=g) * 0.8
    colors = torch.rand(1, p, 3, generator=g) * 2 - 1
    alpha = torch.rand(1, p, 1, generator=g)
    got, pts = splat_lookup_composite_grid(images.to(DEV), grid.to(DEV), query.to(DEV), flip.to(DEV), colors.to(DEV),
                                           alpha.to(DEV), 1.3, 0.75, 2, padding=3)
    # the float64 composite at the kernel's own points (the lookup is held to torch's bitwise above)
    from oracle import labels as OL
    want, values = OL.splat_composite_grid_ref(images.double().unsqueeze(0), pts.cpu().unsqueeze(0), colors, alpha, 1.3, 0.75,
                                               2, padding=3, return_values=True)
    d = (got.cpu().int() - want[0].int()).abs()
    tie = (values[0] - values[0].round()).abs() <= 1e-3
    assert bool((d <= 1).all()) and bool(tie[d == 1].all()), "%d values differ without a tie" % int(
        ((d == 1) & ~tie).sum() + (d > 1).sum())
    print("dense label, %d points: %d of %d values differ by 1 at ties" % (p, int(d.sum()), d.numel()))


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [1, 3])
def test_one_pass_equals_determine_flips_t_and_uncongeal_points(iters):
    """congeal_and_grid's flips, congealed images (output resolution 256, flow 128) and grids equal determine_flips +
    t(flipped) + uncongeal_points' grid on cuda_ops, within the convolutions' rounding at batch 2N versus N."""
    from gangealing_b200.evaluation import determine_flips
    from gangealing_b200.opset import cuda_ops
    t = _mirror(cuda_ops()).to(DEV)
    images = GPR.case_images(70 + iters, 6).to(DEV)
    with torch.no_grad(), fp32_stn():
        flip, congealed, grid = t.congeal_and_grid(images, True, GPR.SIZE, iters)
        flipped, want_flip, policy = determine_flips(t, None, images, iters=iters)
        want_img = t(flipped, warp_policy=policy, iters=iters, output_resolution=GPR.SIZE)
        _, want_grid = t(flipped, return_warp=True, warp_policy=policy, iters=iters)
    assert torch.equal(flip, want_flip.view(-1)), (flip, want_flip.view(-1))
    assert (congealed - want_img).abs().max().item() <= 1e-4 * want_img.abs().max().item()
    assert (grid - want_grid).abs().max().item() <= 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_api_on_the_gpu_reproduces_the_fixture(name, tmp_path):
    """The whole API on cuda_ops with the STN's convolutions in fp32 against the CPU fixture, and its individual images
    against the grid cells."""
    from gangealing_b200.evaluation import save_propagation
    from gangealing_b200.opset import cuda_ops
    blob = load_golden("propagate_to_images")
    with fp32_stn():
        res, png = _run(cuda_ops(), blob, name, tmp_path, DEV, individual=True)
    assert all(res[g].is_cuda and res[g].dtype == torch.uint8 for g in GRIDS if g in res)
    _check_fixture(blob, name, res, png)
    n = blob[name + ".cfg"][0].item()
    pad = 3
    xmaps = int(math.sqrt(n))
    for g, cells in res["individual"].items():
        r = cells.size(1)
        for k in range(n):
            y, x = pad + (k // xmaps) * (r + pad), pad + (k % xmaps) * (r + pad)
            assert torch.equal(cells[k], res[g][y:y + r, x:x + r]), (g, k)
    paths = save_propagation(res, str(tmp_path / "out"))
    assert np.array_equal(np.asarray(Image.open(paths[0])), res["input_images"].cpu().numpy())


class _Classifier:
    """A cluster classifier's flip decision (run_flip_target): image n is flipped where n is odd."""

    def run_flip_target(self, x, cluster):
        flip = (torch.arange(x.size(0), device=x.device) % 2 == 1).view(-1, 1, 1, 1)
        return torch.where(flip, x.flip(3), x), flip


@pytest.mark.gpu
def test_classifier_path_with_two_heads_and_a_cluster():
    """num_heads = 2 with a cluster: the classifier decides the flips, the STN runs once over N images with that
    cluster's head, and the grid equals the device composition at those points."""
    from gangealing_b200.evaluation import propagate_to_images
    from gangealing_b200.opset import cuda_ops
    t = _mirror(cuda_ops(), num_heads=2).to(DEV)
    images = GPR.case_images(80, 4).to(DEV)
    label = torch.tensor([[5, 6], [30, 40], [63, 63], [0, 10]])
    colors = torch.rand(1, 4, 3, generator=torch.Generator().manual_seed(1)).to(DEV) * 2 - 1
    seen, handle = _count_images(t)
    with torch.no_grad():
        res = propagate_to_images(t, images, label, colors, resolution=64, classifier=_Classifier(), cluster=1,
                                  num_heads=2)
    handle.remove()
    assert seen[0] == images.size(0)
    assert res["flips"].tolist() == [False, True, False, True]
    with torch.no_grad():
        flipped = torch.where(res["flips"].view(-1, 1, 1, 1), images.flip(3), images)
        policy = torch.eye(2, device=DEV)[torch.ones(4, dtype=torch.long, device=DEV)]
        _, grid = t(flipped, return_warp=True, warp_policy=policy)
    from gangealing_b200.evaluation.propagate import label_queries
    queries, _ = label_queries(label.to(DEV), 64, images.size(-1))
    want, pts = _device_composition(images, grid, queries, res["flips"], colors, None, 1.3, 0.75, 2)
    assert torch.equal(res["correspondences"], pts)
    differ = int((res["propagated"] != want).sum())
    assert differ <= DIFFER_BOUND * want.numel(), differ
