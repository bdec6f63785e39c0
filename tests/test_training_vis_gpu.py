"""Training visuals on the H100: the three trainvis.cu entries against their restatements (oracle/training_vis.py), the
API against the CPU op set, and the visuals run between replays of a captured training step."""
import pytest
import torch

from oracle import make_golden_training_vis as GT
from oracle import training_vis as OT
from vis_reference import case_grids, compare_to_fixture, mirror_models

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _lib():
    from gangealing_b200 import _lib
    return _lib.load()


# ------------------------------------------------------------------------------------------------ cluster_accumulate
ROUTE_PLAN = [   # K, flips (S = K or 2K), N per call, calls, n_keep, C, H, W
    (1, False, 1, 1, 4, 3, 7, 9),
    (3, False, 17, 2, 2, 3, 5, 11),
    (2, True, 33, 3, 40, 3, 13, 13),        # n_keep larger than any cluster's count
    (4, True, 250, 2, 8, 3, 16, 16),
    (2, True, 1100, 1, 3, 1, 3, 5),         # more images than one shared-memory chunk of selections
]


@pytest.mark.parametrize("k,flips,n,calls,n_keep,c,h,w", ROUTE_PLAN)
def test_cluster_accumulate_is_the_sequential_sum(k, flips, n, calls, n_keep, c, h, w):
    from gangealing_b200.op.grids import cluster_accumulate
    g = torch.Generator().manual_seed(n + k)
    f = 2 if flips else 1
    sums, counts, keep = torch.zeros(k, c, h, w, device=DEV), torch.zeros(k, dtype=torch.int64, device=DEV), \
        torch.zeros(k, n_keep, c, h, w, device=DEV)
    rs, rc, rk = sums.cpu(), counts.cpu(), keep.cpu()
    for _ in range(calls):
        flat = torch.randn(f * n * k, c, h, w, generator=g) * 3
        sel = torch.randint(0, f * k, (n,), generator=g)
        view = flat.view(f, n, k, c, h, w)
        cluster_accumulate(sums, counts, keep, view.to(DEV), sel.to(DEV))
        OT.cluster_accumulate_ref(rs, rc, rk, view, sel)       # one fp32 add per image, in order
    torch.cuda.synchronize()
    assert torch.equal(counts.cpu(), rc)
    assert torch.equal(sums.cpu(), rs), "sums are not bitwise the sequential fp32 sum"
    assert torch.equal(keep.cpu(), rk)


def test_cluster_accumulate_reads_strided_and_broadcast_views():
    from gangealing_b200.op.grids import cluster_accumulate
    g = torch.Generator().manual_seed(5)
    x = torch.randn(6, 3, 9, 9, generator=g).to(DEV).to(memory_format=torch.channels_last)
    sel = torch.tensor([3, 0, 1, 2, 3, 1], device=DEV)
    view = x[None, :, None].expand(2, -1, 2, -1, -1, -1)      # real_cluster_congeal: one image whatever the slot
    sums, counts, keep = torch.zeros(2, 3, 9, 9, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV), \
        torch.zeros(2, 2, 3, 9, 9, device=DEV)
    cluster_accumulate(sums, counts, keep, view, sel)
    rs, rc, rk = sums.cpu() * 0, counts.cpu() * 0, keep.cpu() * 0
    OT.cluster_accumulate_ref(rs, rc, rk, view.cpu(), sel.cpu())
    assert torch.equal(sums.cpu(), rs) and torch.equal(counts.cpu(), rc) and torch.equal(keep.cpu(), rk)


# ---------------------------------------------------------------------------------------------------- image_grid
def _device_images2grid(images, nrow, value_range, scale_each):
    from torchvision.utils import make_grid
    grid = make_grid(images, nrow=nrow, padding=2, pad_value=0, normalize=True, value_range=value_range, scale_each=scale_each)
    return grid.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)


@pytest.mark.parametrize("n,nrow,value_range,scale_each", [(1, 1, None, True), (5, 2, None, True), (3, 8, None, True),
                                                           (7, 2, None, False), (4, 2, (0, 1), False),
                                                           (6, 3, (-1, 1), False)])
def test_image_grid_is_make_grid_on_the_device(n, nrow, value_range, scale_each):
    from gangealing_b200.training.visuals import image_grid
    g = torch.Generator().manual_seed(n * 7 + nrow)
    images = (torch.randn(n, 3, 13, 11, generator=g) * torch.linspace(0.01, 2, n).view(n, 1, 1, 1)).to(DEV)
    got = image_grid(images, nrow, value_range, scale_each)
    assert torch.equal(got, _device_images2grid(images, nrow, value_range, scale_each))


# ----------------------------------------------------------------------------------------------- flow_image_grid
@pytest.mark.parametrize("n,h,w,nrow,scale", [(1, 17, 17, 1, 0.1), (4, 64, 64, 2, 0.05), (5, 31, 29, 2, 1.0),
                                              (3, 128, 128, 8, 0.01)])
def test_flow_image_grid_matches_the_restatement(n, h, w, nrow, scale):
    from gangealing_b200.op.grids import flow_image_grid
    g = torch.Generator().manual_seed(n * h)
    flow = torch.randn(n, h, w, 2, generator=g) * scale
    flow[0, 0, 0] = 0.0
    got = flow_image_grid(flow.to(DEV), nrow).cpu()
    want = OT.flow_image_grid_ref(flow, nrow)
    assert got.shape == want.shape
    d = (got.long() - want.long()).abs()
    differ = int((d > 0).sum())
    print("flow_image_grid %s: %d of %d values differ (max %d)" % ((n, h, w), differ, d.numel(), int(d.max())))
    if differ:
        # a difference is allowed only where numpy's float32 arctan2 and the correctly rounded one give a different fk
        # (a neighbouring wheel bin, or a shifted mix), or where 255 * col lies within 1e-3 of an integer step
        explained = OT.flow_explained(flow.numpy())
        single = OT.flow_image_grid_ref(flow, nrow).clone()
        mask = torch.from_numpy(explained).to(torch.uint8) * 255
        cells = OT.images2grid(mask.permute(0, 3, 1, 2).float() / 255.0, nrow, (0, 1)) > 127
        bad = (d > 0) & ~cells
        assert not bool(bad.any()), "%d differences not explained by an atan2 ulp or a step tie" % int(bad.sum())


def test_flow_to_image_is_the_reference_float_image():
    from gangealing_b200.training.visuals import flow_to_image
    g = torch.Generator().manual_seed(9)
    flow = torch.randn(3, 20, 20, 2, generator=g) * 0.2
    got = flow_to_image(flow.to(DEV)).cpu()
    want = torch.from_numpy(OT.flow_colors(flow.numpy())).float().div(255.0).permute(0, 3, 1, 2)
    assert got.shape == want.shape and (got != want).sum() <= 3


# ------------------------------------------------------------------------------------------------- bad arguments
def test_entries_refuse_bad_arguments_before_device_work():
    lib = _lib()
    out = torch.zeros(64, dtype=torch.uint8, device=DEV)
    buf = torch.zeros(64, device=DEV)
    i64 = torch.zeros(4, dtype=torch.int64, device=DEV)
    p, s = out.data_ptr(), torch.cuda.current_stream().cuda_stream
    assert lib.gg_flow_image_grid(p, buf.data_ptr(), buf.data_ptr(), 0, 2, 2, 1, 2, s) == -1
    assert lib.gg_flow_image_grid(p, None, buf.data_ptr(), 1, 2, 2, 1, 2, s) == -1
    assert lib.gg_flow_image_grid(p, buf.data_ptr(), buf.data_ptr() + 4, 1, 2, 2, 1, 2, s) == -1
    assert lib.gg_image_grid(p, buf.data_ptr(), buf.data_ptr(), 1, 2, 2, 0, 2, s) == -1
    assert lib.gg_image_grid(p, buf.data_ptr(), buf.data_ptr() + 4, 1, 2, 2, 1, 2, s) == -1
    assert lib.gg_image_grid(None, buf.data_ptr(), buf.data_ptr(), 1, 2, 2, 1, 2, s) == -1
    args = [buf.data_ptr(), i64.data_ptr(), buf.data_ptr(), buf.data_ptr(), i64.data_ptr()]
    ok = [1, 2, 2, 1, 2, 2, 0, 0, 0, 4, 2, 1, 1]
    assert lib.gg_cluster_accumulate(*args, *ok, s) == 0
    for i, v in ((1, 3), (2, 0), (1, 1), (6, -1), (12, -1), (0, -1)):     # S not a multiple of K, K = 0, S < K, ...
        bad = list(ok)
        bad[i] = v
        if i == 1 and v == 1:
            bad[2] = 2
        assert lib.gg_cluster_accumulate(*args, *bad, s) == -1, "accepted %s" % bad
    assert lib.gg_cluster_accumulate(args[0], None, *args[2:], *ok, s) == -1
    torch.cuda.synchronize()
    assert (buf == 0).all()


# ------------------------------------------------------------------------------------------- end to end and graphs
def _cfg(k, flips, dtype="f32"):
    from gangealing_b200.training import TrainConfig
    return TrainConfig(gen_size=64, flow_size=64, dim_latent=16, n_mlp=1, batch=2, inject=3, num_heads=k, flips=flips, ndirs=2,
                       stn_channel_multiplier=0.25, gen_channel_multiplier=1, padding_mode="reflection", dtype=dtype)


def _inputs(device, seed=1):
    g = torch.Generator().manual_seed(seed)
    z, big_z = torch.randn(4, 16, generator=g), torch.randn(7, 16, generator=g)
    reals = torch.randn(4, 3, 64, 64, generator=g)
    loader = [torch.randn(3, 3, 64, 64, generator=g) for _ in range(3)]
    return z.to(device), big_z.to(device), reals.to(device), [x.to(device) for x in loader]


@pytest.fixture
def fp32_convolutions():
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = False, False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags


@pytest.fixture
def cpu_noise(monkeypatch):
    """The generator's noise drawn from the CPU generator in the reference's order, then moved: the fixture's fakes."""
    from gangealing_b200.stylegan2.networks import NoiseInjection
    monkeypatch.setattr(NoiseInjection, "sample", staticmethod(
        lambda batch, h, w, like: torch.empty(batch, 1, h, w).normal_().to(like.device, like.dtype)))


@pytest.mark.parametrize("case", GT.CASES, ids=[c[0] for c in GT.CASES])
def test_visuals_reproduce_the_reference_grids_on_the_gpu(case, fp32_convolutions, cpu_noise):
    """training_visuals / classifier_visuals on the sm_90a op set, the convolutions in fp32, against the reference's own
    grids: at most 0.5 % of the stored values differ, each by one step.  The assignments of every batch of fakes are
    compared with the reference's: a difference is allowed only at a near-tie (the two best losses within 1e-4
    relative), and the counts are reported."""
    from conftest import load_golden
    blob = load_golden("training_vis")
    name, k, flips = case[:3]
    differ, total = compare_to_fixture(case_grids(None, case, DEV), blob, name)
    print("%s on the GPU: %d of %d stored values differ" % (name, differ, total))
    if not any(key.startswith(name + ".assign") for key in blob):
        return
    from gangealing_b200.training import assign_fake_images_to_clusters
    trainer, _ = mirror_models(None, k, flips, DEV)
    _, big_z, _, _ = GT.inputs()
    torch.manual_seed(GT.NOISE_SEED)
    vb = case[4] // k
    mismatched = near_ties = compared = 0
    with torch.no_grad():
        for i in range(-(-big_z.size(0) // vb)):
            z_in = big_z[i * vb:(i + 1) * vb].to(DEV)
            a, _, _, _, _, dist = assign_fake_images_to_clusters(
                trainer.generator, trainer.t_ema, trainer.ll, trainer.loss_fn, trainer.resize_fake2stn, GT.PSI, z_in.size(0),
                None, True, k, flips, DEV, sample_from_full_res=True, z=z_in, padding_mode=GT.PADDING)
            want, ref_dist = blob["%s.assign%d" % (name, i)], blob["%s.dist%d" % (name, i)]
            best = ref_dist.sort(dim=1).values
            tie = (best[:, 1] - best[:, 0]) <= 1e-4 * best[:, 0].abs().clamp_min(1e-12)
            bad = a.indices.cpu() != want
            mismatched += int(bad.sum())
            near_ties += int(tie.sum())
            compared += want.numel()
            assert not bool((bad & ~tie).any()), "batch %d: assignments %s, the reference's %s" % (i, a.indices.tolist(),
                                                                                                 want.tolist())
    print("%s: %d of %d assignments differ from the reference's, %d near-ties" % (name, mismatched, compared, near_ties))


def _state(trainer):
    sd = trainer.checkpoint()
    flat = {}
    for key in ("t", "t_ema", "ll"):
        for n, v in sd[key].items():
            flat[key + "." + n] = v.detach().clone()
    return flat


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("k,flips", [(1, False), (2, True)])
def test_visuals_between_replays_leave_the_training_state_unchanged(dtype, k, flips):
    """Visuals between replays of a captured step: the training state is byte-identical just before and just after them,
    and k replays, visuals, k replays end byte-identical to 2k replays.  cuDNN runs deterministic algorithms here: at this
    size the fp32 single-head step was seen to differ from run to run without any visuals."""
    from gangealing_b200.training import Trainer
    from gangealing_b200.training import visuals as V
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        results = []
        for with_visuals in (False, True):
            torch.manual_seed(0)
            tr = Trainer(_cfg(k, flips, dtype), DEV)
            tr.capture(warmup=2)
            for _ in range(3):
                tr.step()
            if with_visuals:
                torch.cuda.synchronize()
                before = _state(tr)
                V.training_visuals(tr, *_inputs(DEV), n_mean=7, n_sample=4, vis_batch_size=6)
                torch.cuda.synchronize()
                _equal_states(before, _state(tr))
            for _ in range(3):
                tr.step()
            torch.cuda.synchronize()
            results.append(_state(tr))
            tr.release_graph()
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags
    _equal_states(*results)


def _equal_states(a, b):
    assert a.keys() == b.keys()
    for n in a:
        x, y = a[n].contiguous().reshape(-1), b[n].contiguous().reshape(-1)
        assert torch.equal(x.view(torch.uint8) if x.is_floating_point() else x,
                           y.view(torch.uint8) if y.is_floating_point() else y), n
