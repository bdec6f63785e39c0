"""Training visuals (gangealing_b200.training.visuals) on the CPU restatement (oracle/training_vis.py): the restated ops
against torchvision's make_grid and float64, and the API's grids against the reference's host formulation of the
per-cluster averages (host lists, pad_heads, accumulate_means) restated here."""
import os
import sys

import pytest
import torch

from oracle import make_golden_training_vis as GT
from oracle import opset
from oracle import training_vis as OT
from ranks import run_ranks
from vis_reference import DIFFER_BOUND, case_grids, compare_to_fixture, mirror_models

CPU = opset.cpu_ops()
OPS = OT.cpu_ops()


def _cfg(k, flips):
    from gangealing_b200.training import TrainConfig
    return TrainConfig(gen_size=64, flow_size=64, dim_latent=16, n_mlp=1, batch=2, inject=3, num_heads=k, flips=flips, ndirs=2,
                       stn_channel_multiplier=0.25, gen_channel_multiplier=1, padding_mode="reflection")


def _inputs(seed=1):
    g = torch.Generator().manual_seed(seed)
    z, big_z = torch.randn(4, 16, generator=g), torch.randn(7, 16, generator=g)
    reals = torch.randn(4, 3, 64, 64, generator=g)
    loader = [torch.randn(3, 3, 64, 64, generator=g) for _ in range(3)]
    return z, big_z, reals, loader


def test_color_wheel_entries():
    w = OT.color_wheel()
    assert w.shape == (55, 3) and w.min() == 0 and w.max() == 255
    assert (w[0] == [255, 0, 0]).all() and (w[15] == [255, 255, 0]).all() and (w[21] == [0, 255, 0]).all()
    assert (w[25] == [0, 255, 255]).all() and (w[36] == [0, 0, 255]).all() and (w[49] == [255, 0, 255]).all()


def test_flow_colors_zero_flow_is_white_and_layout_is_make_grid():
    flow = torch.zeros(3, 9, 7, 2)
    flow[1, 4, 3] = torch.tensor([0.5, -0.25])
    col = OT.flow_colors(flow.numpy())
    assert (col[0] == 255).all() and (col[2] == 255).all()
    assert (col[1, 4, 3] != 255).any()
    grid = OT.flow_image_grid_ref(flow, nrow=2)
    assert tuple(grid.shape) == (2 * 11 + 2, 2 * 9 + 2, 3)
    assert torch.equal(grid[2:11, 2:9], torch.from_numpy(col[0]))
    assert torch.equal(grid[13:22, 2:9], torch.from_numpy(col[2]))
    assert (grid[13:22, 11:18] == 0).all()          # the empty fourth cell holds the pad value
    single = OT.flow_image_grid_ref(flow[1:2], nrow=8)
    assert torch.equal(single, torch.from_numpy(OT.flow_colors(flow[1:2].numpy())[0]))   # N = 1: the bare image


@pytest.mark.parametrize("n,nrow", [(1, 1), (5, 2), (3, 8)])
def test_image_grid_ref_is_make_grid_scale_each(n, nrow):
    g = torch.Generator().manual_seed(n)
    images = torch.randn(n, 3, 11, 13, generator=g) * torch.linspace(0.1, 3, n).view(n, 1, 1, 1)
    ranges = torch.stack([images.amin(dim=(1, 2, 3)), images.amax(dim=(1, 2, 3))], 1)
    assert torch.equal(OT.image_grid_ref(images, ranges, nrow), OT.images2grid(images, nrow, None, scale_each=True))


def test_cluster_accumulate_ref_routes_in_order():
    g = torch.Generator().manual_seed(3)
    k, n = 3, 10
    images = torch.randn(2, n, k, 3, 5, 7, generator=g)
    sel = torch.randint(0, 2 * k, (n,), generator=g)
    sums, counts, keep = torch.zeros(k, 3, 5, 7), torch.zeros(k, dtype=torch.int64), torch.zeros(k, 2, 3, 5, 7)
    OT.cluster_accumulate_ref(sums, counts, keep, images, sel)
    s64, c64 = OT.routed_sums_f64(images, sel, k)
    assert torch.equal(counts, c64)
    assert torch.allclose(sums.double(), s64, atol=1e-5)
    for c in range(k):
        idx = [i for i, s in enumerate(sel.tolist()) if s % k == c][:2]
        for j, i in enumerate(idx):
            s = int(sel[i])
            assert torch.equal(keep[c, j], images[s // k, i, s % k])


def _reference_cluster_means(trainer, big_z, n_mean, n_sample, vis_batch_size):
    """generate_cluster_congeal + pad_heads + accumulate_means as the reference computes them (host lists, one rank)."""
    from gangealing_b200.training import assign_fake_images_to_clusters
    cfg = trainer.cfg
    k = cfg.num_heads
    heads = [[] for _ in range(k)]
    total = 0
    while True:
        z_in = big_z[total:total + vis_batch_size]
        a, aligned, _, _, _, _ = assign_fake_images_to_clusters(
            trainer.generator, trainer.t_ema, trainer.ll_module, trainer.loss_fn, trainer.resize_fake2stn, trainer.psi_t,
            z_in.size(0), None, True, k, cfg.flips, "cpu", sample_from_full_res=True, z=z_in, padding_mode=cfg.padding_mode)
        chw = aligned.shape[1:]
        if cfg.flips:
            aligned = aligned.reshape(2, z_in.size(0), k, *chw).permute(1, 0, 2, 3, 4, 5).reshape(z_in.size(0), 2 * k, *chw)
        else:
            aligned = aligned.view(z_in.size(0), k, *chw)
        for warp, c in zip(aligned[torch.arange(z_in.size(0)), a.indices], a.indices):
            heads[c.item() % k].append(warp)
        total += z_in.size(0)
        if total >= n_mean:
            break
    counts = [len(h) for h in heads]
    for h in heads:
        h.extend([torch.zeros(*chw)] * max(0, n_sample - len(h)))
    stacked = [torch.stack(h, 0) for h in heads]
    means = torch.stack([h.sum(0) for h in stacked]) / torch.tensor([float(h.size(0)) for h in stacked]).view(k, 1, 1, 1)
    return stacked, means, counts


def test_training_visuals_cluster_means_keep_the_pad_count_quirk():
    """K = 2 with flips: 7 fakes in batches of 3 (vis_batch_size 6 // K): a cluster with fewer than n_sample = 4 fakes
    is divided by n_sample and its grid ends in zero images, as pad_heads + accumulate_means do."""
    from gangealing_b200.training import Trainer
    from gangealing_b200.training import visuals as V
    tr = Trainer(_cfg(2, True), "cpu", ops=CPU)
    z, big_z, reals, loader = _inputs()
    grids = V.training_visuals(tr, z, big_z, None, loader, n_mean=7, n_sample=4, vis_batch_size=6, ops=OPS)
    stacked, means, counts = _reference_cluster_means(tr, big_z, 7, 4, 3)
    assert min(counts) < 4, "the case must leave a cluster with fewer than n_sample fakes (counts %s)" % counts
    want = OT.images2grid(means, 1, None, scale_each=True)
    got = grids["mean_generated_EMA_transformed_assigned"]
    assert (got.long() - want.long()).abs().max() <= 1 and (got != want).float().mean() <= 0.005
    for h in range(2):
        assert torch.equal(grids["generated_EMA_assigned_head_%d" % h], OT.images2grid(stacked[h][:4], 2, (-1, 1)))
    expected = {"mean_EMA_transformed_real_sample", "EMA_transformed_real_sample", "EMA_head_0", "EMA_head_1",
                "mean_generated_EMA_transformed_assigned", "generated_EMA_assigned_head_0", "generated_EMA_assigned_head_1",
                "sample", "mean_sample", "truncated_sample", "mean_truncated_sample", "transformed_sample",
                "mean_transformed_sample"}
    assert set(grids) == expected


def test_training_visuals_unimodal_grids_match_the_reference_formulation():
    from gangealing_b200.training import Trainer, sample_gan_supervised_pairs
    from gangealing_b200.training import visuals as V
    tr = Trainer(_cfg(1, False), "cpu", ops=CPU)
    z, _, reals, loader = _inputs(2)
    grids = V.training_visuals(tr, z, None, reals, loader, n_mean=7, n_sample=4, ops=OPS)
    # run_loader_mean: whole batches until n_mean // world = 7 images are seen -> 9 images
    congealed = torch.cat([tr.t_ema(x, unfold=True, padding_mode="reflection") for x in loader], 0)
    mean = congealed.reshape(9, -1, 3, 64, 64).sum(0) / 9
    want = OT.images2grid(mean, 1, None, scale_each=True)
    got = grids["mean_EMA_transformed_real_sample"]
    assert (got.long() - want.long()).abs().max() <= 1 and (got != want).float().mean() <= 0.005
    out, flow = tr.t_ema(reals, return_flow=True, padding_mode="reflection")
    assert torch.equal(grids["EMA_transformed_real_sample"], OT.images2grid(out, 2, (-1, 1)))
    assert torch.equal(grids["flow_real"], OT.flow_image_grid_ref(flow, 2))
    sample, truncated = sample_gan_supervised_pairs(tr.generator, tr.ll, lambda x: x, tr.psi_t, 4, None, True, "cpu", z=z)
    assert torch.equal(grids["sample"], OT.images2grid(sample, 2, (-1, 1)))
    assert torch.equal(grids["truncated_sample"], OT.images2grid(truncated, 2, (-1, 1)))
    assert torch.equal(grids["mean_sample"], OT.images2grid(sample.mean(0, keepdim=True), 1, None, scale_each=True))


def test_classifier_visuals_route_real_images_by_the_classifier():
    from gangealing_b200.training import ClassifierTrainer, Trainer
    from gangealing_b200.training import visuals as V
    tr = Trainer(_cfg(2, True), "cpu", ops=CPU)
    ct = ClassifierTrainer(tr, ops=CPU)
    _, _, _, loader = _inputs(3)
    grids = V.classifier_visuals(ct, loader, n_mean=5, n_sample=4, ops=OPS)
    assert set(grids) == {"mean_EMA_transformed_assigned", "EMA_assigned_head_0", "EMA_assigned_head_1"}
    heads, total = [[], []], 0
    for x in loader:                                      # real_cluster_congeal's host loop
        total += x.size(0)
        preds = ct.classifier(x)
        classes = preds.argmax(dim=1)
        x = torch.where((classes >= 2).view(-1, 1, 1, 1), x.flip(3), x)
        for img, c in zip(tr.t_ema(x, warp_policy=preds, padding_mode="reflection"), classes):
            heads[c.item() % 2].append(img)
        if total >= 5:
            break
    for h in range(2):
        shown = torch.stack((heads[h] + [torch.zeros(3, 64, 64)] * 4)[:4])
        assert torch.equal(grids["EMA_assigned_head_%d" % h], OT.images2grid(shown, 2, (-1, 1)))


def test_save_grids_writes_the_reference_file_names(tmp_path):
    from gangealing_b200.training.visuals import save_grids
    grids = {"sample": torch.randint(0, 255, (10, 12, 3), dtype=torch.uint8), "flow_real": torch.zeros(4, 4, 3, dtype=torch.uint8)}
    paths = save_grids(grids, str(tmp_path), 1500)
    assert sorted(os.path.basename(p) for p in paths) == ["flow_real_0001500.png", "sample_0001500.png"]
    from PIL import Image
    import numpy as np
    assert (np.asarray(Image.open(tmp_path / "sample_0001500.png")) == grids["sample"].numpy()).all()


def test_compat_registers_flow_to_image():
    from gangealing_b200 import compat
    from gangealing_b200.training import visuals
    saved = sys.modules.pop("utils.vis_tools.flow_vis", None)
    try:
        compat.install()
        assert sys.modules["utils.vis_tools.flow_vis"].flow_to_image is visuals.flow_to_image
    finally:
        if saved is not None:
            sys.modules["utils.vis_tools.flow_vis"] = saved


# ------------------------------------------------------------------------------------ the reference's own grids
@pytest.mark.parametrize("case", GT.CASES, ids=[c[0] for c in GT.CASES])
def test_api_reproduces_the_reference_grids_on_the_cpu_op_set(case):
    from conftest import load_golden
    blob = load_golden("training_vis")
    differ, total = compare_to_fixture(case_grids(CPU, case, vis_ops=OPS), blob, case[0])
    print("%s: %d of %d stored values differ" % (case[0], differ, total))


def test_oracle_restatements_reproduce_the_reference_flow_and_mean_grids():
    """The restated colour wheel and normalised grid applied to the reference's own inputs of those grids (the mirror
    STN's flow and mean images on the fixture's models) reproduce the captured grids."""
    from conftest import load_golden
    blob = load_golden("training_vis")
    trainer, _ = mirror_models(CPU, 1, False)
    _, _, reals, _ = GT.inputs()
    with torch.no_grad():
        _, flow = trainer.t_ema(reals, return_flow=True, padding_mode=GT.PADDING)
    got = OT.flow_image_grid_ref(flow, 2)
    d = (got.long() - blob["unimodal.flow_real"].long()).abs()
    assert int(d.max()) <= 1 and int((d > 0).sum()) <= DIFFER_BOUND * d.numel()


# --------------------------------------------------------------------------------------------- two ranks over gloo
def _worker_two_ranks(rank, world, ret):
    from gangealing_b200.training import Trainer
    from gangealing_b200.training import distributed as gdist
    from gangealing_b200.training import visuals as V
    tr = Trainer(_cfg(2, True), "cpu", ops=CPU)
    z, big_z, _, loader = _inputs(10 + rank)               # each rank its own fakes and real batches
    big_z = big_z[:4]                                       # n_mean // world = 4 fakes per rank, batches of 3: 3 + 1
    grids = V.training_visuals(tr, z, big_z, None, loader, n_mean=8, n_sample=4, vis_batch_size=6, ops=OPS)
    # the reference's formulas on this rank's host lists: pad_heads + accumulate_means, run_loader_mean + all_reduce
    stacked, _, counts = _reference_cluster_means(tr, big_z, 4, 4, 3)
    fake_sums = torch.stack([h.sum(0) for h in stacked])
    fake_num = torch.tensor([float(h.size(0)) for h in stacked])
    real, seen = [], 0
    for x in loader:
        real.append(tr.t_ema(x, unfold=True, padding_mode="reflection"))
        seen += x.size(0)
        if seen >= 8 // world:
            break
    real = torch.cat(real, 0)
    g_fake, g_num = gdist.all_gather(fake_sums[None]), gdist.all_gather(fake_num[None])
    g_real = gdist.all_gather(real.sum(0, keepdim=True))
    g_seen = gdist.all_gather(torch.tensor([float(real.size(0))]))
    if rank == 0:
        ret["grids"] = {k: v.clone() for k, v in grids.items()}
        ret["fake_means"] = g_fake.sum(0) / g_num.sum(0).view(-1, 1, 1, 1)
        ret["real_means"] = g_real.sum(0) / g_seen.sum()
        ret["counts"] = counts
    else:
        ret["rank1_grids"] = len(grids)


@pytest.mark.timeout(600)
def test_two_rank_means_follow_the_reference_formulas_gloo():
    """world 2: the per-cluster means divide the ranks' summed sums by the ranks' summed max(count, n_sample), the real
    means by all images seen on both ranks; rank 0 returns the grids, rank 1 none."""
    ret = run_ranks(_worker_two_ranks, 560)
    grids = ret["grids"]
    assert ret["rank1_grids"] == 0
    assert min(ret["counts"]) < 4
    for name, means in (("mean_generated_EMA_transformed_assigned", ret["fake_means"]),
                        ("mean_EMA_transformed_real_sample", ret["real_means"])):
        want = OT.images2grid(means, 1, None, scale_each=True)
        d = (grids[name].long() - want.long()).abs()
        assert int(d.max()) <= 1 and int((d > 0).sum()) <= DIFFER_BOUND * d.numel(), name
