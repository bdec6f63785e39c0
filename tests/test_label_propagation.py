"""Labelled videos (gangealing_b200.evaluation: label_propagation_frames, smooth_correspondence, labeled_average_frames) and
the fused splat-and-composite grid op (splat_composite_grid, csrc/splat.cu) against the reference fixture
(oracle/make_golden_labels.py), the reference's composition on the device and the float64 restatement (oracle/labels.py).

uint8 frames are compared pixel by pixel: the STN here and the reference's round their convolutions in different orders,
so a tracked point may move (see test_congealing_vis.py) and a value near a quantisation step may round the other way.
At most 0.5 % of the stored pixels may differ, and the count is reported."""
import pytest
import torch
from torchvision.utils import make_grid

from conftest import load_golden
from oracle import labels as OL
from oracle import make_golden_labels as GL
from oracle import make_golden_pck as GP
from oracle import make_golden_vis as GV
from oracle import opset
from vis_reference import fp32_stn

DEV = "cuda"
CASES = [c[0] for c in GL.LABEL_CASES]
DIFFER_BOUND = 0.005


def _mirror(ops):
    from gangealing_b200.stn import get_stn
    return opset.fill_parameters(get_stn(["similarity", "flow"], ops=ops, **GP.STN_KW).eval(), GP.WEIGHT_SEED,
                                 gain=GP.WEIGHT_GAIN)


def images2grid(images, nrow):
    """utils/vis_tools/helpers.py:39-43 with make_grid(normalize=True, range=(-1, 1)), left on the images' device."""
    grid = make_grid(images, nrow=nrow, normalize=True, value_range=(-1, 1))
    return grid.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)


def _label(blob, with_alpha):
    return GV.label_points(), blob["colors"], (blob["alpha"] if with_alpha else None)


def _compare(got, blob, key, kept):
    """Frame count and per-channel sums of every frame, and the stored frames pixel by pixel -> differing pixels."""
    sums = blob[key + ".sums"]
    got = got.cpu()
    assert got.size(0) == sums.size(0), "%s: %d frames, the reference has %d" % (key, got.size(0), sums.size(0))
    want = blob[key + ".kept"]
    assert got.shape[1:] == want.shape[1:], "%s: frame shape %s vs %s" % (key, tuple(got.shape[1:]), tuple(want.shape[1:]))
    differ = int((got[kept] != want).sum())
    assert differ <= DIFFER_BOUND * want.numel(), "%s: %d of %d pixels differ" % (key, differ, want.numel())
    pixels = got.size(1) * got.size(2)
    sum_err = (got.long().sum((1, 2)) - sums).abs().max().item()
    assert sum_err <= DIFFER_BOUND * 255 * pixels, "%s: per-frame sums differ by %d" % (key, sum_err)
    return differ, want.numel()


def _videos(ops, blob, name, device="cpu"):
    from gangealing_b200.evaluation import smooth_correspondence
    smooth, n, with_alpha = blob[name + ".cfg"].tolist()
    _, stages, stage_flip, length, flip_length, iters, seed = GV.SMOOTH_CASES[smooth]
    pts, colors, alpha = _label(blob, with_alpha)
    t = _mirror(ops).to(device)
    data = GV.case_batches(seed, 1)[0][:n].to(device)
    with torch.no_grad():
        return smooth_correspondence(t, data, pts, colors.to(device), None if alpha is None else alpha.to(device),
                                     GL.SIGMA, GL.OPACITY, resolution=GV.RESOLUTION, length=length,
                                     flip_length=flip_length, vis_in_stages=bool(stages), stage_flip=bool(stage_flip),
                                     output_resolution=GV.RES, iters=iters)


def _check_videos(blob, name, videos):
    counts = {v: blob["%s.%s.sums" % (name, v)].size(0) for v in GL.VIDEOS}
    for video in GL.VIDEOS:
        differ, total = _compare(videos[video], blob, "%s.%s" % (name, video), GL.kept_frames(video, counts))
        print("%s %s: %d of %d stored pixels differ from the reference" % (name, video, differ, total))


def _average(ops, blob, device="cpu"):
    from gangealing_b200.evaluation import congealing_average_frames, labeled_average_frames
    avg, with_alpha = blob["labeled_average.cfg"].tolist()
    _, stages, stage_flip, length, flip_length, iters, n_mean, seed = GV.AVG_CASES[avg]
    pts, colors, alpha = _label(blob, with_alpha)
    t = _mirror(ops).to(device)
    batches = [b.to(device) for b in GV.case_batches(seed)]
    with torch.no_grad():
        frames = congealing_average_frames(t, batches, n_mean, length=length, flip_length=flip_length,
                                           vis_in_stages=bool(stages), stage_flip=bool(stage_flip),
                                           output_resolution=GV.RES, iters=iters)
        return labeled_average_frames(frames, pts, colors.to(device), None if alpha is None else alpha.to(device),
                                      GL.SIGMA, GL.OPACITY, resolution=GV.RESOLUTION, ops=ops)


def _check_average(blob, got):
    f = blob["labeled_average.sums"].size(0)
    differ, total = _compare(got, blob, "labeled_average", [f - 126, f - 35, f - 1])
    print("labeled_average: %d of %d stored pixels differ from the reference" % (differ, total))


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", CASES)
def test_videos_reproduce_the_reference_fixture(name):
    """smooth_correspondence on the oracle op set: the congealing, propagation and correspondence videos of the
    reference's smoothly_congeal_and_propagate, frame counts and shapes exact."""
    blob = load_golden("label_propagation")
    _check_videos(blob, name, _videos(OL.cpu_ops(), blob, name))


def test_labeled_average_reproduces_the_reference_fixture():
    """congealing_average_frames + labeled_average_frames on the oracle op set: average_and_congeal's video."""
    blob = load_golden("label_propagation")
    _check_average(blob, _average(OL.cpu_ops(), blob))


@pytest.mark.parametrize("n", [1, 3, 4, 5])
def test_restatement_without_points_is_images2grid(n):
    """P = 0 (points None or an empty label) is images2grid of every frame, bitwise; N = 1 has no padding."""
    g = torch.Generator().manual_seed(n)
    frames = torch.randn(3, n, 3, 20, 20, generator=g) * 1.3
    want = torch.stack([images2grid(f, int(n ** 0.5)) for f in frames])
    got = OL.splat_composite_grid_ref(frames, None, None, None, 1.2, 0.7, int(n ** 0.5))
    empty = OL.splat_composite_grid_ref(frames, torch.zeros(3, n, 0, 2), torch.zeros(1, 0, 3), None, 1.2, 0.7, int(n ** 0.5))
    assert torch.equal(got, want) and torch.equal(empty, want)
    if n == 1:
        assert got.shape == (3, 20, 20, 3)


def test_abi_rejects_bad_arguments():
    """Validation runs before any device work; a non-null dummy pointer is never dereferenced."""
    from gangealing_b200 import _lib
    dll = _lib.load()
    one = 16

    def err():
        return dll.gg_last_error().decode()

    def call(out=one, ws=one, ws_bytes=1 << 20, images=one, points=one, colors=one, alpha=one, sigma=1.2, opacity=0.7,
             T=2, N=4, P=5, C=3, R=8, nrow=2, padding=2, colors_n=1, alpha_n=4):
        return dll.gg_splat_composite_grid(out, ws, ws_bytes, images, points, colors, alpha, sigma, opacity, T, N, P, C, R,
                                           nrow, padding, colors_n, alpha_n, None)

    assert call(out=None) == -1 and "null" in err()
    assert call(images=None) == -1 and "null" in err()
    assert call(points=None) == -1 and "null" in err()
    assert call(colors=None) == -1 and "null" in err()
    assert call(ws=None) == -1 and "null" in err()
    assert call(sigma=0.0) == -1 and "sigma" in err()
    assert call(sigma=float("nan")) == -1 and "sigma" in err()
    assert call(opacity=1.5) == -1 and "opacity" in err()
    assert call(opacity=-0.1) == -1 and "opacity" in err()
    assert call(C=4) == -1 and "C must be 3" in err()
    assert call(ws=one + 4) == -1 and "16-byte" in err()
    assert call(points=one + 4) == -1 and "8-byte" in err()
    assert call(ws_bytes=100) == -1 and "workspace" in err()
    assert call(colors_n=3) == -1 and "colors_n" in err()
    assert call(alpha_n=2) == -1 and "alpha_n" in err()
    assert call(N=0) == -1 and call(R=0) == -1 and call(nrow=0) == -1 and call(T=-1) == -1
    assert call(R=40000, N=2, P=0) == -1 and "2^31" in err()
    assert call(N=1 << 20, P=1 << 12, R=1, alpha_n=1) == -1 and "2^31" in err()
    assert dll.gg_splat_composite_grid_workspace(3, 4, 8, 1) == 3 * 4 * 64 * 32
    assert dll.gg_splat_composite_grid_workspace(3, 4, 8, 0) == 3 * 4 * 64 * 16


# ------------------------------------------------------------------------------------------------ GPU
def _device_reference(images, points, colors, alpha, sigma, opacity, nrow):
    """The reference's composition on the device: cuda_ops().splat2d twice (splat_points), the alpha composite, make_grid
    and images2grid's quantisation, frame by frame."""
    from gangealing_b200.opset import cuda_ops
    ops = cuda_ops()
    t, n, _, r, _ = images.shape
    p = points.size(2)
    col = colors.expand(n, p, 3).contiguous()
    al = torch.ones(n, p, 1, device=DEV) if alpha is None else alpha.expand(n, p, 1).contiguous()
    sig = torch.tensor(sigma, device=DEV, dtype=torch.float).view(1).repeat(n)
    out = []
    for i in range(t):
        obj = ops.splat2d(torch.zeros(n, 3, r, r, device=DEV), points[i].contiguous(), col, sig, False)
        mask = ops.splat2d(torch.zeros(n, 1, r, r, device=DEV), points[i].contiguous(), al, sig, True) * opacity
        out.append(images2grid(mask * obj + (1 - mask) * images[i], nrow))
    return torch.stack(out)


def _sparse_points(g, t, n, r):
    """Pairs of points around the sites of a 12-pixel lattice (footprints of sigma 1.2 span at most 7 pixels), so that no
    pixel receives more than two contributions and the fp32 sums do not depend on their order; plus points outside the
    image, which are skipped."""
    ys, xs = torch.meshgrid(torch.arange(4, r - 3, 12).float(), torch.arange(4, r - 3, 12).float(), indexing="ij")
    sites = torch.stack([xs.flatten(), ys.flatten()], -1)
    sites = sites.view(1, 1, -1, 2).repeat(t, n, 1, 1) + torch.rand(t, n, sites.size(0), 2, generator=g) * 2 - 1
    pair = sites + torch.rand(sites.shape, generator=g) * 1.6 - 0.8
    outside = torch.tensor([[-0.5, 3.0], [3.0, float(r)], [float(r) + 0.2, 5.0], [-3.0, -3.0]]).view(1, 1, 4, 2).repeat(t, n, 1, 1)
    return torch.cat([sites, pair, outside], 2)


SPARSE_CASES = [   # N, R, alpha channel, opacity, per-image colours, frames per chunk
    (1, 96, True, 0.7, False, 2),
    (3, 130, False, 1.0, True, 5),
    (4, 96, False, 0.7, False, 2),
    (5, 130, True, 1.0, True, 3),
    (4, 130, True, 0.7, True, 5),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(SPARSE_CASES)))
def test_sparse_label_is_bitwise_the_device_composition(case):
    """With at most two contributions per pixel the op equals, bitwise, splat2d twice + the composite + make_grid +
    images2grid's quantisation on the device; T = 5 frames in chunks that do not divide it evenly."""
    from gangealing_b200.splat2d import splat_composite_grid
    n, r, with_alpha, opacity, per_image, chunk = SPARSE_CASES[case]
    g = torch.Generator().manual_seed(500 + case)
    t = 5
    points = _sparse_points(g, t, n, r)
    p = points.size(2)
    images = (torch.randn(t, n, 3, r, r, generator=g) * 0.8).to(DEV)
    colors = (torch.rand(n if per_image else 1, p, 3, generator=g) * 2.4 - 1.2).to(DEV)
    alpha = torch.rand(n if per_image else 1, p, 1, generator=g).to(DEV) if with_alpha else None
    frame_bytes = n * r * r * (32 if with_alpha else 16)
    got = splat_composite_grid(images, points.to(DEV), colors, alpha, 1.2, opacity, int(n ** 0.5),
                               max_workspace_bytes=chunk * frame_bytes)
    want = _device_reference(images, points.to(DEV), colors, alpha, 1.2, opacity, int(n ** 0.5))
    assert got.shape == want.shape and got.dtype == torch.uint8
    assert torch.equal(got, want), "%d of %d values differ" % (int((got != want).sum()), got.numel())


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 4])
def test_no_points_is_images2grid_bitwise(n):
    from gangealing_b200.splat2d import splat_composite_grid
    g = torch.Generator().manual_seed(600 + n)
    frames = (torch.randn(7, n, 3, 45, 45, generator=g) * 1.3).to(DEV)
    got = splat_composite_grid(frames, None, None, None, 1.2, 0.7, int(n ** 0.5))
    want = torch.stack([images2grid(f, int(n ** 0.5)) for f in frames])
    assert torch.equal(got, want)


@pytest.mark.gpu
def test_dense_tracked_label_vs_float64_oracle():
    """A dense label (every pixel of a 40^2 block at resolution 64, overlapping footprints) tracked by smooth_congealing:
    every uint8 value equals the float64 restatement's, or differs by 1 where its v * 255 + 0.5 lies within 1e-3 of an
    integer (a tie that fp32 sums in another order may round either way)."""
    from gangealing_b200.evaluation import smooth_congealing
    from gangealing_b200.opset import cuda_ops
    from gangealing_b200.splat2d import splat_composite_grid
    _, stages, stage_flip, length, flip_length, iters, seed = GV.SMOOTH_CASES[0]
    ys, xs = torch.meshgrid(torch.arange(12, 52), torch.arange(12, 52), indexing="ij")
    label = torch.stack([xs.flatten(), ys.flatten()], -1)
    g = torch.Generator().manual_seed(700)
    colors = torch.rand(1, label.size(0), 3, generator=g) * 2 - 1
    alpha = torch.rand(1, label.size(0), 1, generator=g)
    t = _mirror(cuda_ops()).to(DEV)
    data = GV.case_batches(seed, 1)[0].to(DEV)
    with torch.no_grad(), fp32_stn():
        frames, points, _ = smooth_congealing(t, data, label, GV.RESOLUTION, length, flip_length, bool(stages),
                                              bool(stage_flip), GV.RES, iters=iters)
    frames, points = frames[flip_length::12], points[::12]
    got = splat_composite_grid(frames, points, colors.to(DEV), alpha.to(DEV), GL.SIGMA, GL.OPACITY, 2).cpu()
    want, values = OL.splat_composite_grid_ref(frames.cpu().double(), points.cpu(), colors, alpha, GL.SIGMA, GL.OPACITY, 2,
                                               return_values=True)
    d = (got.int() - want.int()).abs()
    tie = (values - values.round()).abs() <= 1e-3
    assert bool((d <= 1).all()) and bool(tie[d == 1].all()), "%d values differ without a tie" % int(((d == 1) & ~tie).sum() + (d > 1).sum())
    print("dense label, %d points, %d frames: %d of %d values differ by 1 at ties" % (label.size(0), frames.size(0),
                                                                                        int(d.sum()), d.numel()))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_videos_on_the_gpu_reproduce_the_fixture(name):
    from gangealing_b200.opset import cuda_ops
    blob = load_golden("label_propagation")
    with fp32_stn():
        videos = _videos(cuda_ops(), blob, name, DEV)
    assert all(v.is_cuda and v.dtype == torch.uint8 for v in videos.values())
    _check_videos(blob, name, videos)


@pytest.mark.gpu
def test_labeled_average_on_the_gpu_reproduces_the_fixture():
    from gangealing_b200.opset import cuda_ops
    blob = load_golden("label_propagation")
    with fp32_stn():
        got = _average(cuda_ops(), blob, DEV)
    _check_average(blob, got)
