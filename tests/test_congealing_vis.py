"""Congealing visualisations (gangealing_b200.evaluation.visuals): the average-image animation, the average congealed image
and the congealing animation with dense point tracking, against the reference fixture (oracle/make_golden_vis.py), the
float64 oracle (oracle/vis.py) and the reference's per-frame composition; the lerped-grid sampler and its frame-mean kernel
against torch and float64; a 2-rank gloo run; the C ABI's argument checks.  The windowed point tracker's kernel is checked
over its launch plan in test_points_family_gpu.py."""
import pytest
import torch

from conftest import load_golden
from oracle import make_golden_pck as GP
from oracle import make_golden_vis as GV
from oracle import opset
from oracle import vis as OV
from ranks import run_ranks
from vis_reference import fp32_stn

DEV = "cuda"
AVG = [c[0] for c in GV.AVG_CASES]
SMOOTH = [c[0] for c in GV.SMOOTH_CASES]


def _mirror(ops):
    from gangealing_b200.stn import get_stn
    return opset.fill_parameters(get_stn(["similarity", "flow"], ops=ops, **GP.STN_KW).eval(), GP.WEIGHT_SEED,
                                 gain=GP.WEIGHT_GAIN)


def _avg_cfg(blob, name):
    stages, flip, length, flip_length, iters, n_mean, seed = blob[name + ".cfg"].tolist()
    return dict(length=length, flip_length=flip_length, vis_in_stages=bool(stages), stage_flip=bool(flip),
                output_resolution=GV.RES, iters=iters), n_mean, seed


def _smooth_cfg(blob, name):
    stages, flip, length, flip_length, iters, seed = blob[name + ".cfg"].tolist()
    return dict(resolution=GV.RESOLUTION, length=length, flip_length=flip_length, vis_in_stages=bool(stages),
                stage_flip=bool(flip), output_resolution=GV.RES, iters=iters), seed


def _rel(a, b, scale=None):
    """Relative error.  With `scale` (averages: their images' magnitude): the largest difference over scale.  Otherwise
    max(|a - b|_2 / |b|_2, largest |a - b| / (10 max|b|)): compared with tol, the norm within tol and every element within
    10 tol -- two STNs that compute the grids in different orders may move a pixel where the image is steep by more than
    the norm."""
    d = a.double().cpu() - b.double().cpu()
    if scale is not None:
        return (d.abs().max() / float(scale)).item()
    return max((d.norm() / b.double().norm().clamp_min(1e-12)).item(),
               (d.abs().max() / b.double().abs().max().clamp_min(1e-12)).item() / 10)


def _scale(batches):
    return max(float(b.abs().max()) for b in batches)


def _check_smooth(blob, name, frames, points, unaligned, rtol):
    kept = [f for f in blob["kept_frames"].tolist() if f < frames.size(0)]
    assert _rel(frames[kept, :2], blob[name + ".frames_kept"]) <= rtol
    assert _rel(frames.double().sum((3, 4)), blob[name + ".frame_sums"]) <= rtol
    assert _rel(unaligned, blob[name + ".unaligned"]) <= rtol
    return int((points.cpu() != blob[name + ".points"]).any(-1).sum())


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", AVG)
def test_average_frames_reproduce_the_reference_fixture(name):
    """The API and the oracle's per-frame composition on the oracle op set: the reference's frames within
    GV.tolerance(iters) (1e-5 for one STN pass)."""
    from gangealing_b200.evaluation import congealing_average_frames
    blob = load_golden("congealing_vis")
    kw, n_mean, seed = _avg_cfg(blob, name)
    t = _mirror(OV.cpu_ops())
    batches = GV.case_batches(seed)
    with torch.no_grad():
        got = congealing_average_frames(t, batches, n_mean, **kw)
        oracle = OV.average_frames_ref(t, batches, n_mean, **kw)
    assert got.shape == blob[name + ".frames"].shape
    tol = GV.tolerance(kw["iters"])
    assert _rel(got, blob[name + ".frames"], _scale(batches)) <= tol
    assert _rel(oracle, blob[name + ".frames"], _scale(batches)) <= tol


@pytest.mark.parametrize("name", SMOOTH)
def test_smooth_congealing_reproduces_the_reference_fixture(name):
    """Frames within GV.tolerance(iters) (1e-5 for one STN pass); tracked points equal to the reference's except where the mirror STN's rounding turns a near-tie
    of the window search (the count is reported; at most 1 % of the (frame, image, point) positions)."""
    from gangealing_b200.evaluation import smooth_congealing
    blob = load_golden("congealing_vis")
    kw, seed = _smooth_cfg(blob, name)
    t = _mirror(OV.cpu_ops())
    data = GV.case_batches(seed, 1)[0]
    with torch.no_grad():
        frames, points, unaligned = smooth_congealing(t, data, blob["label_points"], **kw)
    differ = _check_smooth(blob, name, frames, points, unaligned, GV.tolerance(kw["iters"]))
    print("%s: %d of %d tracked points differ" % (name, differ, points[..., 0].numel()))
    assert differ <= 0.01 * points[..., 0].numel()


def test_average_congealed_image_reproduces_the_reference_fixture():
    """propagate_to_images.average: whole batches until n_mean // world images are seen (6 asked, 8 used)."""
    from gangealing_b200.evaluation import average_congealed_image
    blob = load_golden("congealing_vis")
    n_mean, iters, seed = blob["average.cfg"].tolist()
    t = _mirror(OV.cpu_ops())
    batches = GV.case_batches(seed)
    with torch.no_grad():
        got = average_congealed_image(t, batches, n_mean, output_resolution=GV.RES, iters=iters)
        oracle = OV.average_ref(t, batches, n_mean, GV.RES, iters)
    assert got.shape == (1,) + tuple(blob["average.image"].shape)
    assert _rel(got[0], blob["average.image"], _scale(batches)) <= GV.tolerance(iters)
    assert _rel(oracle, blob["average.image"], _scale(batches)) <= GV.tolerance(iters)


def _gloo_worker(rank, world, ret):
    from gangealing_b200.evaluation import average_congealed_image, congealing_average_frames
    t = _mirror(OV.cpu_ops())
    batches = GV.case_batches(GV.AVG_CASES[0][-1])
    with torch.no_grad():
        frames = congealing_average_frames(t, batches[rank:rank + 1], 8, length=3, flip_length=3, vis_in_stages=True,
                                           stage_flip=True, output_resolution=GV.RES)
        avg = average_congealed_image(t, batches[rank:rank + 1], 8, output_resolution=GV.RES)
    if rank == 0:
        ret["frames"], ret["avg"] = frames, avg


@pytest.mark.timeout(900)
def test_two_rank_gloo_run_equals_the_single_process_result():
    """Rank r congeals batch r; the single process both batches in order."""
    from gangealing_b200.evaluation import average_congealed_image, congealing_average_frames
    t = _mirror(OV.cpu_ops())
    batches = GV.case_batches(GV.AVG_CASES[0][-1])
    with torch.no_grad():
        frames = congealing_average_frames(t, batches, 8, length=3, flip_length=3, vis_in_stages=True, stage_flip=True,
                                           output_resolution=GV.RES)
        avg = average_congealed_image(t, batches, 8, output_resolution=GV.RES)
    ret = run_ranks(_gloo_worker, 860)
    assert _rel(ret["frames"], frames) <= 1e-6, _rel(ret["frames"], frames)
    assert _rel(ret["avg"], avg) <= 1e-6


def test_reference_assertions_raise_value_error():
    from gangealing_b200.evaluation import congealing_average_frames, smooth_congealing
    t = _mirror(OV.cpu_ops())
    batches = GV.case_batches(1)
    with pytest.raises(ValueError, match="evenly divide"):            # :340-341
        congealing_average_frames(t, batches, 6, length=3, output_resolution=32)
    with pytest.raises(ValueError, match="needed 12"):                 # :377
        congealing_average_frames(t, batches, 12, length=3, output_resolution=32)
    with pytest.raises(ValueError, match="length"):
        smooth_congealing(t, batches[0], length=1, output_resolution=32)


def test_abi_rejects_bad_arguments():
    """Validation runs before any device work; a non-null dummy pointer is never dereferenced."""
    from gangealing_b200 import _lib
    dll = _lib.load()
    one = 16

    def err():
        return dll.gg_last_error().decode()

    track = lambda T=2, H=8, W=8, patch=9, ptr=one: dll.gg_track_points_lerp(ptr, one, one, one, one, one, T, 1, 5, H, W, patch, None)
    assert track(patch=8) == -1 and "odd" in err()
    assert track(W=9) == -1 and "H == W" in err()
    assert track(T=0) == -1 and "T" in err()
    assert track(ptr=None) == -1 and "null" in err()
    mean = lambda C=3, T=2, acc=one, base=one: dll.gg_mipmap_warp_lerp_mean(acc, one, one, base, 0, one, one, T, 0, 2, C, 16,
                                                                         16, 8, 8, 1, 1.0, 0.0, 1, 0, None)
    assert mean(C=5) == -2 and "C <= 4" in err()
    assert mean(T=0) == -1 and "T" in err()
    assert mean(acc=None) == -1 and "null" in err()
    assert mean(base=None) == -1 and "null" in err()
    fwd = lambda T=2, stride=0, target=one: dll.gg_mipmap_warp_lerp_forward(one, None, one, one, one, stride, target, one, T,
                                                                            0, 2, 3, 16, 16, 8, 8, 1, 1.0, 0.0, 1, None)
    assert fwd(T=0) == -1 and "T" in err()
    assert fwd(stride=7) == -1 and "base_stride" in err()
    assert fwd(target=None) == -1 and "null" in err()


# ------------------------------------------------------------------------------------------------ GPU
def _grids(g, n, ho, wo, broadcast):
    base = torch.nn.functional.affine_grid(torch.eye(2, 3).unsqueeze(0).repeat(1 if broadcast else n, 1, 1), (1 if broadcast else n, 1, ho, wo),
                                           align_corners=False)
    if not broadcast:
        base = base + 0.05 * torch.randn(base.shape, generator=g)
    theta = torch.eye(2, 3).unsqueeze(0) * (0.6 + 0.8 * torch.rand(n, 1, 1, generator=g))
    theta[:, :, 2] = 0.3 * torch.randn(n, 2, generator=g)
    target = torch.nn.functional.affine_grid(theta, (n, 1, ho, wo), align_corners=False) + 0.03 * torch.randn(n, ho, wo, 2, generator=g)
    return base, target


LERP_CASES = [  # dtype, padding, broadcast base, (hs, ws), (ho, wo), T
    (torch.float32, "border", True, (64, 64), (96, 96), 7),
    (torch.float32, "zeros", False, (48, 80), (37, 45), 9),
    (torch.float32, "reflection", False, (128, 128), (40, 70), 3),
    (torch.bfloat16, "border", False, (64, 64), (33, 65), 5),
    (torch.bfloat16, "reflection", True, (96, 96), (96, 96), 8),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(LERP_CASES)))
def test_mipmap_warp_lerp_is_bitwise_the_per_frame_warp(case):
    from gangealing_b200.stn.sampling import mipmap_warp, mipmap_warp_lerp
    dtype, pad, broadcast, (hs, ws), (ho, wo), T = LERP_CASES[case]
    g = torch.Generator().manual_seed(100 + case)
    n = 3
    src = torch.randn(n, 3, hs, ws, generator=g).to(DEV, dtype)
    base, target = [x.to(DEV) for x in _grids(g, n, ho, wo, broadcast)]
    alphas = torch.cat([torch.tensor([0.0, 1.0, 0.5]), torch.rand(T - 3, generator=g)]).to(DEV)
    out, grids = mipmap_warp_lerp(src, base, target, alphas, 3.5, padding_mode=pad)
    for t in range(T):
        want_grid = torch.lerp(base, target, alphas[t].view(1, 1, 1, 1))
        assert torch.equal(grids[t], want_grid.expand_as(grids[t])), "frame %d: grid differs from torch.lerp" % t
        assert torch.equal(out[t], mipmap_warp(src, grids[t], 3.5, padding_mode=pad)[0]), "frame %d: warp differs" % t


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(LERP_CASES)))
def test_mipmap_warp_lerp_mean_is_the_sequential_sum(case):
    """Bitwise a sequential fp32 sum of the per-sample frames (with and without accumulate), bitwise repeatable, and within
    N * max|src| * (1e-4 + the source dtype's rounding, 2^-8 for bf16) of the float64 oracle (each sample's value is stored
    in the source dtype)."""
    from gangealing_b200.stn.sampling import mipmap_warp_lerp, mipmap_warp_lerp_mean
    dtype, pad, broadcast, (hs, ws), (ho, wo), T = LERP_CASES[case]
    g = torch.Generator().manual_seed(200 + case)
    n = 5
    src = torch.randn(n, 3, hs, ws, generator=g).to(DEV, dtype)
    base, target = [x.to(DEV) for x in _grids(g, n, ho, wo, broadcast)]
    alphas = torch.rand(T, generator=g).to(DEV)
    frames, _ = mipmap_warp_lerp(src, base, target, alphas, 3.5, padding_mode=pad)
    seq = torch.zeros(T, 3, ho, wo, device=DEV)
    for i in range(n):
        seq = seq + frames[:, i].float()
    got = mipmap_warp_lerp_mean(src, base, target, alphas, None, 3.5, padding_mode=pad)
    assert torch.equal(got, seq)
    again = mipmap_warp_lerp_mean(src, base, target, alphas, None, 3.5, padding_mode=pad)
    assert torch.equal(got, again)
    prior = torch.randn(T, 3, ho, wo, generator=g).to(DEV)
    acc = mipmap_warp_lerp_mean(src, base, target, alphas, prior.clone(), 3.5, padding_mode=pad)
    assert torch.equal(acc, prior + seq)
    ref = OV.mipmap_warp_lerp_mean_ref(src.double().cpu(), base.double().cpu(), target.double().cpu(), alphas.double().cpu(),
                                       None, 3.5, padding_mode=pad)
    err = (got.double().cpu() - ref).abs().max().item()
    bound = n * src.float().abs().max().item() * (1e-4 + (2.0 ** -8 if dtype == torch.bfloat16 else 0.0))
    print("case %d: |mean - float64| = %.2e (bound %.2e)" % (case, err, bound))
    assert err <= bound


def _count_images(t):
    seen = [0]
    handle = t.stns[-1].register_forward_hook(lambda m, inp, out: seen.__setitem__(0, seen[0] + inp[0].size(0)))
    return seen, handle


@pytest.mark.gpu
@pytest.mark.parametrize("name", AVG)
def test_average_frames_on_the_gpu(name):
    """The API equals the reference's per-frame composition on cuda_ops (fp32 reordering tolerance) and the fixture; the
    STN sees every image 3 times, whatever the length."""
    from gangealing_b200.evaluation import congealing_average_frames
    from gangealing_b200.opset import cuda_ops
    blob = load_golden("congealing_vis")
    kw, n_mean, seed = _avg_cfg(blob, name)
    t = _mirror(cuda_ops()).to(DEV)
    batches = [b.to(DEV) for b in GV.case_batches(seed)]
    with torch.no_grad(), fp32_stn():
        seen, handle = _count_images(t)
        got = congealing_average_frames(t, batches, n_mean, **kw)
        handle.remove()
        assert seen[0] == 3 * n_mean
        ref = OV.average_frames_ref(t, batches, n_mean, **kw)
    assert _rel(got, ref, _scale(batches)) <= 1e-5, _rel(got, ref, _scale(batches))
    assert _rel(got, blob[name + ".frames"], _scale(batches)) <= 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("name", SMOOTH)
def test_smooth_congealing_on_the_gpu(name):
    """The API equals the reference's per-frame composition on cuda_ops (frames to fp32 reordering, at least 99 % of the
    tracked positions equal) and the CPU fixture; the STN sees every image 3 times."""
    from gangealing_b200.evaluation import smooth_congealing
    from gangealing_b200.opset import cuda_ops
    blob = load_golden("congealing_vis")
    kw, seed = _smooth_cfg(blob, name)
    t = _mirror(cuda_ops()).to(DEV)
    data = GV.case_batches(seed, 1)[0].to(DEV)
    with torch.no_grad(), fp32_stn():
        seen, handle = _count_images(t)
        frames, points, unaligned = smooth_congealing(t, data, blob["label_points"], **kw)
        handle.remove()
        assert seen[0] == 3 * data.size(0)
        rf, rp, ru = OV.smooth_congealing_ref(t, data, blob["label_points"].to(DEV), **kw)
    assert _rel(frames, rf) <= 2e-5 and _rel(unaligned, ru) <= 1e-5
    same = (points == rp).all(-1).float().mean().item()
    fixture_differ = _check_smooth(blob, name, frames, points, unaligned, 1e-3)
    print("%s: %.4f of the points equal the per-frame composition; %d differ from the CPU fixture" % (name, same, fixture_differ))
    assert same >= 0.99
    assert fixture_differ <= 0.01 * points[..., 0].numel()
