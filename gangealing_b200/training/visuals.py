"""Training visuals (reference utils/vis_tools/training_vis.py, written every vis_every steps by train.py:80-87,160-170):
congealed real and fake samples with their means, the STN's flows as colour-wheel images and, for clustering models, the
per-head grids and per-cluster averages of assigned images.  Every grid is a uint8 (Hg, Wg, 3) tensor in the layout of
GANgealingWriter._log_image_grid (make_grid with nrow = int(sqrt(N)), padding 2, pad value 0).

The reference keeps every congealed real image on the host (run_loader_mean), moves every assigned fake to the host with
its own .cpu() (generate_cluster_congeal) and colours flows in numpy.  Here the sums stay on the device: real images add
into a running batch sum (evaluation.average_congealed_image), assigned images are routed to their clusters by the op
set's `cluster_accumulate` (sums in order, the first n_sample of each cluster kept), and every grid is written by one
launch (`splat_composite_grid` for the (-1, 1) grids, `image_grid` for the min/max-normalised means, `flow_image_grid`).

Quirks of the reference kept here:
  * pad_heads appends zero images up to n_sample per cluster on each rank and accumulate_means counts them: a cluster
    with fewer than n_sample assigned images on a rank is divided by max(count_r, n_sample), summed over the ranks, and
    its grid shows the zero images after the assigned ones;
  * the loops stop once n_mean // world images have been seen, so the real loops may use more than n_mean;
  * real_cluster_congeal passes the classifier's logits to the STN as warp_policy;
  * the real-image sample grids are rank 0's images; only rank 0 returns grids (the others return {} after taking part
    in the collectives);
  * a single-image grid is the bare image, without padding.
Visuals run the EMA STN, the generator, the latent learner and (for clustering) VGG eagerly under no_grad; they read the
training state and write none of it, and they draw their random numbers (the generator's noise) from a fork of the RNG
state, so they may run between replays of a captured training step and leave the training run exactly as it would be
without them.
"""
import functools
import os

import torch

from ..evaluation.visuals import average_congealed_image
from . import distributed as dist
from .losses import assign_fake_images_to_clusters, sample_gan_supervised_pairs


def _ops_or_cuda(ops):
    if ops is not None:
        return ops
    from ..opset import cuda_ops
    return cuda_ops()


def _forked_rng(fn):
    """Run fn on a fork of the CPU and current-device RNG states: the training run's random stream is left as it was."""
    @functools.wraps(fn)
    def run(*a, **k):
        devices = [torch.cuda.current_device()] if torch.cuda.is_available() and torch.cuda.is_initialized() else []
        with torch.random.fork_rng(devices=devices):
            return fn(*a, **k)
    return run


def _nrow(n):
    return max(1, int(n ** 0.5))     # GANgealingWriter._log_image_grid


@torch.no_grad()
def flow_to_image(flow_uv, clip_flow=None, convert_to_bgr=False):
    """utils/vis_tools/flow_vis.py:flow_to_image on the device: flow (N, H, W, 2) -> float (N, 3, H, W) in [0, 1], the
    colour-wheel image divided by 255, the same values as the reference's (one `flow_image_grid` launch pair)."""
    if clip_flow is not None:
        raise NotImplementedError("flow_to_image: clip_flow is not supported (train.py does not use it)")
    if flow_uv.dim() != 4 or flow_uv.size(3) != 2:
        raise AssertionError("input flow must have shape [N,H,W,2]")
    from ..op.grids import flow_image_grid
    n, h, w = flow_uv.shape[:3]
    img = flow_image_grid(flow_uv, nrow=1, padding=0).view(n, h, w, 3)    # one column, no padding: the images themselves
    if convert_to_bgr:
        img = img.flip(3)
    img = img.permute(0, 3, 1, 2).float()
    return img / torch.full_like(img, 255.0)     # an elementwise division, rounded as numpy's (not a reciprocal product)


@torch.no_grad()
def image_grid(images, nrow=None, value_range=(-1, 1), scale_each=False, ops=None):
    """images2grid(images, nrow, padding=2, pad_value=0, normalize=True, range=value_range, scale_each) -> uint8
    (Hg, Wg, 3).  value_range None: the batch's (min, max), or each image's with scale_each; nrow None: int(sqrt(N))."""
    ops = _ops_or_cuda(ops)
    images = images.float()
    nrow = _nrow(images.size(0)) if nrow is None else nrow
    if value_range is not None and tuple(value_range) == (-1, 1) and images.size(2) == images.size(3):
        return ops.splat_composite_grid(images.unsqueeze(0), None, None, None, 1.0, 1.0, nrow)[0]
    n = images.size(0)
    if value_range is not None:
        ranges = torch.tensor([[float(value_range[0]), float(value_range[1])]], device=images.device).expand(n, 2)
    elif scale_each:
        ranges = torch.stack([images.amin(dim=(1, 2, 3)), images.amax(dim=(1, 2, 3))], 1)
    else:
        ranges = torch.stack([images.amin(), images.amax()]).view(1, 2).expand(n, 2)
    return ops.image_grid(images, ranges.contiguous(), nrow)


def _log(grids, images, name, n_sample, ops, log_mean_img=True, range=(-1, 1), scale_each=False):
    """GANgealingWriter.log_image_grid with num_heads=1: the first n_sample images and, with log_mean_img, the mean of all
    of them as `mean_<name>` (range None, scale_each)."""
    shown = images[:n_sample]
    grids[name] = image_grid(shown, _nrow(shown.size(0)), range, scale_each, ops)
    if log_mean_img:
        grids["mean_" + name] = image_grid(images.float().mean(dim=0, keepdim=True), 1, None, True, ops)


def _stn_kw(trainer):
    return dict(padding_mode=trainer.cfg.padding_mode)


def _fake_visuals(grids, trainer, z, n_sample, ops):
    """create_fake_visuals (training_vis.py:111-119): generated, truncated and congealed fake samples with their means."""
    ll = getattr(trainer, "ll_module", trainer.ll)
    sample, truncated = sample_gan_supervised_pairs(trainer.generator, ll, lambda x: x, trainer.psi_t, n_sample, None, True,
                                                    trainer.device, z=z)
    transformed = trainer.t_ema(trainer.resize_fake2stn(sample), **_stn_kw(trainer))
    _log(grids, sample, "sample", n_sample, ops)
    _log(grids, transformed, "transformed_sample", n_sample, ops)
    _log(grids, truncated, "truncated_sample", n_sample, ops)


def _cluster_means(sums, counts, n_sample):
    """accumulate_means after pad_heads: per-cluster sums over the ranks divided by the ranks' max(count, n_sample)."""
    num = counts.clamp_min(n_sample).float().view(1, -1)
    k = sums.size(0)
    means = dist.all_gather(sums.unsqueeze(0)).sum(dim=0)
    return means.div(dist.all_gather(num).sum(dim=0).view(k, 1, 1, 1))


def _cluster_buffers(k, c, h, w, n_sample, device):
    return (torch.zeros((k, c, h, w), dtype=torch.float32, device=device), torch.zeros(k, dtype=torch.int64, device=device),
            torch.zeros((k, n_sample, c, h, w), dtype=torch.float32, device=device))


@torch.no_grad()
def generate_cluster_congeal(trainer, big_z, n_mean, n_sample, vis_batch_size, ops):
    """generate_cluster_congeal (training_vis.py:57-88): the fakes of big_z in batches of vis_batch_size, congealed by
    every head (and mirrored, with flips), each routed by its assignment to cluster index % K on the device.
    -> (kept (K, n_sample, C, R, R): the first n_sample of each cluster then zeros, means (K, C, R, R))."""
    cfg = trainer.cfg
    k = cfg.num_heads
    ll = getattr(trainer, "ll_module", trainer.ll)
    sums = counts = keep = None
    total = 0
    while True:
        z_in = big_z[total:total + vis_batch_size]
        b = z_in.size(0)
        assignments, aligned, _, _, _, _ = assign_fake_images_to_clusters(
            trainer.generator, trainer.t_ema, ll, trainer.loss_fn, trainer.resize_fake2stn, trainer.psi_t, b, None, True, k,
            cfg.flips, trainer.device, sample_from_full_res=True, z=z_in, **_stn_kw(trainer))
        chw = aligned.shape[1:]
        if sums is None:
            sums, counts, keep = _cluster_buffers(k, *chw, n_sample, aligned.device)
        view = aligned.float().view(1 + int(cfg.flips), b, k, *chw)     # slot s: flip s // K, head s % K (loss.py:52)
        ops.cluster_accumulate(sums, counts, keep, view, assignments.indices)
        total += b
        if total >= n_mean // dist.get_world_size():
            break
    return keep, _cluster_means(sums, counts, n_sample)


@torch.no_grad()
def real_cluster_congeal(t_ema, classifier, loader, num_heads, n_mean, n_sample, ops, **stn_kwargs):
    """real_cluster_congeal (training_vis.py:90-109): each real image is mirrored when the classifier's argmax says so,
    congealed with the logits as warp_policy and routed to argmax % K.  -> (kept, means) as generate_cluster_congeal."""
    sums = counts = keep = None
    total = 0
    for x in loader:
        total += x.size(0)
        preds = classifier(x)
        classes = preds.argmax(dim=1)
        flip = classes >= num_heads
        x = torch.where(flip.reshape(x.size(0), 1, 1, 1), x.flip(3), x)
        congealed = t_ema(x, warp_policy=preds, **stn_kwargs).float()
        if sums is None:
            sums, counts, keep = _cluster_buffers(num_heads, *congealed.shape[1:], n_sample, congealed.device)
        slots = 2 * num_heads if classifier_slots(preds, num_heads) else num_heads
        view = congealed[None, :, None].expand(slots // num_heads, -1, num_heads, -1, -1, -1)
        ops.cluster_accumulate(sums, counts, keep, view, classes)
        if total >= n_mean // dist.get_world_size():
            break
    if sums is None:
        raise ValueError("real_cluster_congeal: the loader yielded no images")
    return keep, _cluster_means(sums, counts, n_sample)


def classifier_slots(preds, num_heads):
    """True when the classifier also predicts flips (2K logits)."""
    return preds.size(1) > num_heads


def _real_means(trainer, loader, n_mean, n_sample):
    """run_loader_mean(unfold=True) + all_reduce: the per-head means (K, C, R, R) and this rank's first n_sample
    congealed images (unfolded: (n, K, C, R, R) for K > 1)."""
    k = trainer.cfg.num_heads
    out = average_congealed_image(trainer.t_ema, loader, n_mean, no_flip_inference=True, unfold=True, keep=n_sample,
                                  padding_mode=trainer.cfg.padding_mode)
    mean, kept = out if n_sample > 0 else (out, None)
    return mean.reshape(k, *mean.shape[-3:]), kept


@_forked_rng
@torch.no_grad()
def training_visuals(trainer, z, big_z=None, reals=None, loader=None, n_mean=8000, n_sample=64, vis_batch_size=250,
                     ops=None):
    """The reference's training visuals of one round (train.py:160-170): create_training_cluster_visuals when
    trainer.cfg.num_heads > 1, else create_training_visuals.  z: (n_sample, dim_latent) fixed latents of the fake grids;
    big_z: (n_mean // world, dim_latent) latents of the per-cluster averages (clustering); reals: (n, C, H, W) real
    images of the unimodal grids (train.py's sample_reals); loader: an iterable of real (B, C, H, W) batches on the
    device, or None.  vis_batch_size is divided by the number of heads, as train.py does before its loop.
    -> {logging name: uint8 (Hg, Wg, 3) grid} on rank 0, {} on the other ranks."""
    ops = _ops_or_cuda(ops)
    cfg = trainer.cfg
    k = cfg.num_heads
    grids = {}
    primary = dist.primary()
    if k > 1:
        if big_z is None:
            raise ValueError("training_visuals: a clustering model needs big_z")
        if loader is not None:
            mean, local = _real_means(trainer, loader, n_mean, n_sample)
            if primary:
                grids["mean_EMA_transformed_real_sample"] = image_grid(mean, _nrow(k), None, True, ops)
                flat = local.reshape(-1, *local.shape[2:])[:n_sample]
                grids["EMA_transformed_real_sample"] = image_grid(flat, _nrow(flat.size(0)), ops=ops)
                for h in range(k):
                    head = local[:, h][:n_sample]
                    grids["EMA_head_%d" % h] = image_grid(head, _nrow(head.size(0)), ops=ops)
        kept, means = generate_cluster_congeal(trainer, big_z, n_mean, n_sample, max(1, vis_batch_size // k), ops)
        if primary:
            grids["mean_generated_EMA_transformed_assigned"] = image_grid(means, _nrow(k), None, True, ops)
            for h in range(k):
                grids["generated_EMA_assigned_head_%d" % h] = image_grid(kept[h], _nrow(n_sample), ops=ops)
            _fake_visuals(grids, trainer, z, n_sample, ops)
        return grids
    if loader is not None:
        mean, _ = _real_means(trainer, loader, n_mean, 0)
        if primary:
            grids["mean_EMA_transformed_real_sample"] = image_grid(mean, 1, None, True, ops)
            transformed, flow = trainer.t_ema(reals, return_flow=True, **_stn_kw(trainer))
            shown = transformed[:n_sample]
            grids["EMA_transformed_real_sample"] = image_grid(shown, _nrow(shown.size(0)), ops=ops)
            if trainer.t_ema.is_flow:      # the radius is normalised over all of `reals`, the grid shows n_sample
                if flow.size(0) <= n_sample:
                    grids["flow_real"] = ops.flow_image_grid(flow, _nrow(flow.size(0)))
                else:
                    grids["flow_real"] = image_grid(flow_to_image(flow)[:n_sample], _nrow(n_sample), (0, 1), ops=ops)
    if primary:
        _fake_visuals(grids, trainer, z, n_sample, ops)
    return grids


@_forked_rng
@torch.no_grad()
def classifier_visuals(classifier_trainer, loader, n_mean=8000, n_sample=64, ops=None):
    """create_training_cluster_classifier_visuals (training_vis.py:175-187): real images routed to the cluster the
    classifier predicts -> {mean_EMA_transformed_assigned, EMA_assigned_head_k} on rank 0, {} elsewhere."""
    ops = _ops_or_cuda(ops)
    t = classifier_trainer.trainer
    k = t.cfg.num_heads
    kept, means = real_cluster_congeal(t.t_ema, classifier_trainer.classifier, loader, k, n_mean, n_sample, ops,
                                       padding_mode=t.cfg.padding_mode)
    grids = {}
    if dist.primary():
        grids["mean_EMA_transformed_assigned"] = image_grid(means, _nrow(k), None, True, ops)
        for h in range(k):
            grids["EMA_assigned_head_%d" % h] = image_grid(kept[h], _nrow(n_sample), ops=ops)
    return grids


def save_grids(grids, results_path, itr):
    """GANgealingWriter._log_image_grid's files: `{results_path}/{name}_{itr:07}.png` for every grid (PIL).
    -> the paths written."""
    from PIL import Image
    os.makedirs(results_path, exist_ok=True)
    paths = []
    for name, grid in grids.items():
        path = os.path.join(results_path, "%s_%s.png" % (name, str(itr).zfill(7)))
        Image.fromarray(grid.cpu().numpy()).save(path)
        paths.append(path)
    return paths
