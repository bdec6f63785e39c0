"""Congealing visualisations: the average congealed image, the average-image animation and the congealing animation of a
few images with their dense labels tracked (reference applications/vis_correspondence.py and
applications/propagate_to_images.py:81-104).  The reference's `args` fields are keyword arguments here, as in flips.py.

The reference re-runs the flip inference and the STN for every frame of the average-image animation, although only the
lerp weight changes from one frame to the next.  Here every image runs through the STN three times in all (twice for the
flip decision, once for the grids of every stage) and every stage's frames come from one call per batch of the op set's
`mipmap_warp_lerp_mean` (sums over the batch, no per-sample frames written) or `mipmap_warp_lerp` (the congealed frames),
and the label points of a stage are tracked by one `track_points_lerp` launch instead of one Unfold per frame.

Quirks of the reference that published visuals come from, kept here:
  * without `vis_in_stages`, the average-image animation (`congealing_average_frames`) animates grids[0], the similarity
    stage, while the congealing animation (`smooth_congealing`) animates grids[-1], the full warp;
  * `average_congealed_image` averages whole batches until at least n_mean // world images are seen (run_loader_mean),
    so it may use more than n_mean images; it samples the flipped images, while the animations sample the unflipped
    images on flipped grids (create_average_image, smoothly_sample_image);
  * the point tracker's window positions beyond pad_grid's ring are Unfold's (0, 0) zero padding and stay candidates, and
    a window that leaves the padded grid wraps around in the flat index (see track_points_lerp).
"""
import math

import torch
import torch.nn.functional as F

from ..training import distributed as dist
from .flips import determine_flips

WARP_LEVELS = 3.5   # the reference's warper: MipmapWarp(3.5), border padding


def cosine_alphas(length, device):
    """The lerp weight of every frame, with the reference's float32 expression (vis_correspondence.py:192, :409)."""
    if length < 2:
        raise ValueError("an animation needs length >= 2 frames (the reference divides by length - 1), got %d" % length)
    a = [1 - 0.5 * (1 + torch.cos(torch.tensor(math.pi * i / (length - 1)))) for i in range(length)]
    return torch.stack(a).to(device)


def flip_grid(grid, flip_indices):
    """vis_correspondence.py:166-169: negate x where the image was flipped."""
    grid = grid.clone()
    grid[..., 0] = torch.where(flip_indices.view(1, -1, 1, 1), -grid[..., 0], grid[..., 0])
    return grid


def get_patch_size(length):
    """vis_correspondence.py:172-180: the tracking window grows as the animation gets shorter."""
    patch_size = math.ceil(9 * max(1, 240 / length))
    return patch_size + 1 if patch_size % 2 == 0 else patch_size


def _resize(grid, res):
    if res == grid.size(1):
        return grid
    return F.interpolate(grid.permute(0, 3, 1, 2), scale_factor=res / grid.size(1), mode="bilinear").permute(0, 2, 3, 1)


def _identity(n, res, like):
    """F.affine_grid of the identity, built on the CPU and moved as the reference does."""
    return F.affine_grid(torch.eye(2, 3).unsqueeze(0).repeat(n, 1, 1), (n, 3, res, res), align_corners=False).to(like)


def _flips(t, data, classifier, cluster, num_heads, no_flip_inference, iters, padding_mode):
    return determine_flips(t, classifier, data, cluster=cluster, num_heads=num_heads, no_flip_inference=no_flip_inference,
                           iters=iters, padding_mode=padding_mode)


def _num_stages(t, vis_in_stages):
    return len(t.stns) if hasattr(t, "stns") and vis_in_stages else 1


@torch.no_grad()
def average_congealed_image(t, loader, n_mean, classifier=None, cluster=None, num_heads=1, no_flip_inference=False,
                            output_resolution=None, iters=1, padding_mode="border", unfold=False, keep=0):
    """propagate_to_images.average + run_loader_mean + utils/distributed.all_reduce: the mean of the congealed (flipped)
    images of whole batches until this rank has seen at least n_mean // world images, over all ranks.  The sum is kept
    on the device instead of a host-side list of every congealed image.  -> (1, C, R, R).
    unfold=True: every head congeals every image (the STN's (N, K, C, R, R) output) and the result is the per-head means
    (K, C, R, R), as training_vis.run_loader_mean(unfold=True) returns them.  keep > 0: also return this rank's first
    `keep` congealed images (the STN's output rows, in loader order) -> (mean, kept)."""
    world = dist.get_world_size()
    acc, total, kept = None, 0, []
    for x in loader:
        flipped, _, policy = _flips(t, x, classifier, cluster, num_heads, no_flip_inference, iters, padding_mode)
        out = t(flipped, warp_policy=policy, unfold=unfold, iters=iters, padding_mode=padding_mode,
                output_resolution=output_resolution)
        if sum(k.size(0) for k in kept) < keep:
            kept.append(out[:keep - sum(k.size(0) for k in kept)])
        s = out.float().sum(dim=0, keepdim=True)
        acc = s if acc is None else acc + s
        total += x.size(0)
        if total >= n_mean // world:
            break
    if acc is None:
        raise ValueError("average_congealed_image: the loader yielded no images")
    num = dist.all_gather(torch.tensor([float(total)], device=acc.device)).sum()
    mean = dist.all_gather(acc).sum(dim=0, keepdim=not unfold) / num
    return (mean, torch.cat(kept, 0)) if keep > 0 else mean


@torch.no_grad()
def congealing_average_frames(t, loader, n_mean, length=240, flip_length=40, vis_in_stages=False, stage_flip=False,
                              output_resolution=None, classifier=None, cluster=None, num_heads=1, no_flip_inference=False,
                              iters=1, padding_mode="border"):
    """The frames of average_and_congeal (vis_correspondence.py:384-419) before its `normalize`: frame t of a stage is
    the mean over n_mean images of the image warped by lerp(base, grid, alpha_t).  Stages: the flip (with stage_flip;
    flip_length frames, the identity lerped to the flipped identity), then every STN stage with vis_in_stages or else
    grids[0] alone (the similarity stage: the reference's quirk), length frames each, from the previous stage's grid (the
    identity for the first).  Every batch runs the flip decision and the STN once; each stage's frames are one
    `mipmap_warp_lerp_mean` call into a (F, C, R, R) sum, divided by n_mean // world and averaged over ranks.
    The loader yields (N, C, H, W) batches in a fixed order; output_resolution None: the images' size.  -> (F, C, R, R)."""
    world = dist.get_world_size()
    per_rank = n_mean // world
    if per_rank * world != n_mean:
        raise ValueError("n_mean (%d) must be divisible by the number of processes (%d)" % (n_mean, world))
    ops = t.ops
    num_stages = _num_stages(t, vis_in_stages) + int(stage_flip)
    lengths = [flip_length if (stage_flip and i == 0) else length for i in range(num_stages)]
    acc, alphas, identity, total = None, None, None, 0
    for data in loader:
        n_batch = data.size(0)
        if acc is None:
            if per_rank // n_batch != per_rank / n_batch:
                raise ValueError("the batch size (%d) must evenly divide the images each process needs (%d)" % (n_batch, per_rank))
            res = output_resolution or data.size(-1)
            acc = torch.zeros((sum(lengths), data.size(1), res, res), dtype=torch.float32, device=data.device)
            alphas = [cosine_alphas(n, data.device) for n in lengths]
            identity = _identity(1, res, data)
        flipped, flip_indices, policy = _flips(t, data, classifier, cluster, num_heads, no_flip_inference, iters, padding_mode)
        _, grids = t(flipped, warp_policy=policy, return_intermediates=True, iters=iters, padding_mode=padding_mode)
        n = min(n_batch, per_rank - total)
        f0 = 0
        for i in range(num_stages):
            warp_index = i - int(stage_flip)
            if warp_index >= 0:
                target = flip_grid(grids[warp_index], flip_indices)
                base = identity.repeat(n_batch, 1, 1, 1) if warp_index == 0 else grids[warp_index - 1]
                base = _resize(flip_grid(base, flip_indices), res)[:n]
            else:
                target = flip_grid(identity.repeat(n_batch, 1, 1, 1), flip_indices)
                base = identity
            target = _resize(target, res)[:n]
            ops.mipmap_warp_lerp_mean(data[:n], base, target, alphas[i], acc[f0:f0 + lengths[i]], WARP_LEVELS)
            f0 += lengths[i]
        total += n
        if total >= per_rank:
            break
    if total != per_rank:
        raise ValueError("needed %d images per process but the loader gave %d" % (per_rank, total))
    dist.synchronize()
    return torch.stack(dist.all_gather(acc / per_rank, cat=False), 0).mean(dim=0)


@torch.no_grad()
def smooth_congealing(t, data, label_points=None, resolution=256, length=240, flip_length=40, vis_in_stages=False,
                      stage_flip=False, output_resolution=None, classifier=None, cluster=None, num_heads=1,
                      no_flip_inference=False, iters=1, padding_mode="border"):
    """smoothly_congeal_and_propagate (vis_correspondence.py:208-298) with sample_images_and_points' label handling
    (:48-54): the congealing animation of `data` (N, C, H, W) and the dense label tracked through it.
    label_points: (P, 2) integer (x, y) pixel coordinates of the label in the congealed frame at `resolution`, or None.
    Stages: the flip (with stage_flip), then every STN stage with vis_in_stages or else grids[-1] alone (the full warp).
    The unflipped images are sampled on flipped grids.  The points are tracked forward from where the label lands in each
    image, then backward from the label itself, and the two runs are blended as the reference does (:279-287).
    -> (frames (F, N, C, R, R); points (stages * length, N, P, 2) fp32 pixel positions in the frames, or None;
        the label's unaligned-space pixel positions (N, P, 2) that the flip stage's splat uses, or None)."""
    return _smooth_congealing(t, data, label_points, resolution, length, flip_length, vis_in_stages, stage_flip,
                              output_resolution, classifier, cluster, num_heads, no_flip_inference, iters, padding_mode)[:3]


def _smooth_congealing(t, data, label_points, resolution, length, flip_length, vis_in_stages, stage_flip, output_resolution,
                       classifier, cluster, num_heads, no_flip_inference, iters, padding_mode):
    """smooth_congealing's results and the flip decision (N,) bool."""
    ops = t.ops
    res = output_resolution or data.size(-1)
    n = data.size(0)
    flipped, flip_indices, policy = _flips(t, data, classifier, cluster, num_heads, no_flip_inference, iters, padding_mode)
    _, grids = t(flipped, return_intermediates=True, warp_policy=policy, padding_mode=padding_mode, iters=iters)
    if not vis_in_stages:
        grids = [grids[-1]]
    grids = flip_grid(torch.stack(grids), flip_indices.view(1, -1, 1, 1))
    flow_size = grids.size(2)
    if res != flow_size:
        g = grids.reshape(-1, flow_size, flow_size, 2)
        g = F.interpolate(g.permute(0, 3, 1, 2), scale_factor=res / flow_size, mode="bilinear").permute(0, 2, 3, 1)
        grids = g.reshape(-1, n, res, res, 2)
    identity = _identity(n, res, data)
    num_stages = grids.size(0)
    flipping = flip_grid(identity, flip_indices)
    grids = torch.cat([flipping.unsqueeze(0), grids], 0)
    alphas = cosine_alphas(length, data.device)
    frames = []
    if stage_flip:
        frames.append(ops.mipmap_warp_lerp(data, identity, flipping, cosine_alphas(flip_length, data.device), WARP_LEVELS)[0])
    for i in range(num_stages):
        frames.append(ops.mipmap_warp_lerp(data, grids[i], grids[i + 1], alphas, WARP_LEVELS)[0])
    frames = torch.cat(frames, 0)
    if label_points is None:
        return frames, None, None, flip_indices
    # sample_images_and_points (:48-54) and :240-253
    points = label_points.to(data.device).unsqueeze(0).repeat(n, 1, 1)
    points_normalized = _normalize(points, res, resolution)
    if resolution != res:
        points = _unnormalize(_normalize(points, res, resolution), res, res).round().long()
    lookup = ops.grid_sample(grids[-1].permute(0, 3, 1, 2).contiguous(), points_normalized.unsqueeze(2).float().contiguous(),
                             "border")
    normalized_unaligned = lookup.squeeze(3).permute(0, 2, 1).contiguous()
    unaligned = _unnormalize(normalized_unaligned, res, res)
    centers = unaligned.round().long().clamp(0, res - 1)
    centers[..., 0] = torch.where(flip_indices.view(-1, 1), res - 1 - centers[..., 0], centers[..., 0])
    patch = get_patch_size(length)
    propagated = []
    for i in range(num_stages):
        track, centers = ops.track_points_lerp(grids[i], grids[i + 1], alphas, normalized_unaligned, centers, patch)
        propagated.append(track.float())
    congealed_centers = points.long()
    blend = torch.linspace(0, 1, steps=length, device=data.device).view(length, 1, 1, 1)
    for i in range(num_stages):     # the reverse pass, congealed -> unaligned (:279-287)
        rev, congealed_centers = ops.track_points_lerp(grids[-i - 1], grids[-i - 2], alphas, normalized_unaligned,
                                                       congealed_centers, patch)
        propagated[-i - 1].lerp_(rev.float().flip(0), blend)
    return frames, torch.cat(propagated, 0), unaligned, flip_indices


def _normalize(points, res, out_res):
    return points.div(out_res - 1).add(-0.5).mul(2).mul((res - 1) / res)


def _unnormalize(points, res, out_res):
    return points.div((res - 1) / res).div(2).add(0.5).mul(out_res - 1)


# ------------------------------------------------------------------------------------------------ labelled videos
# The label-propagation, correspondence and labelled average-image videos of vis_correspondence.py as uint8 frames
# (F, H, W, 3), the frames its save_video receives; encoding them is left to the caller.  Colours are required: the
# reference's default Plotly colour scales (get_plotly_colors) are not reproduced here.
PAUSE_STEPS, INTERP_STEPS, END_PAUSE_STEPS = 60, 60, 5    # visualize_correspondence (:121-123), average_and_congeal (:428-433)


def _ops_or_cuda(ops):
    if ops is not None:
        return ops
    from ..opset import cuda_ops
    return cuda_ops()


def _label_inputs(colors, alpha_channel):
    colors = colors.unsqueeze(0) if colors.dim() == 2 else colors
    if alpha_channel is not None and alpha_channel.dim() == 2:
        alpha_channel = alpha_channel.unsqueeze(0)
    return colors, alpha_channel


def _splat_points(ops, images, points, colors, alpha_channel, sigma, opacity):
    """splat_points (helpers.py:134-194, alpha blending) on the op set's splat2d: points (N, P, 2) pixels, colors and
    alpha_channel (N or 1, P, C)."""
    n, _, h, w = images.shape
    p = points.size(1)
    if alpha_channel is None:
        alpha_channel = torch.ones(n, p, 1, device=images.device)
    sig = torch.full((n,), float(sigma), device=images.device)
    obj = ops.splat2d(torch.zeros(n, 3, h, w, device=images.device), points.float().contiguous(),
                      colors.expand(n, p, 3).float().contiguous(), sig, False)
    mask = ops.splat2d(torch.zeros(n, 1, h, w, device=images.device), points.float().contiguous(),
                       alpha_channel.expand(n, p, 1).float().contiguous(), sig, True) * opacity
    return mask * obj + (1 - mask) * images


@torch.no_grad()
def label_propagation_frames(frames, points, colors, alpha_channel=None, sigma=1.2, opacity=0.7, initial_frames=None,
                             ops=None):
    """visualize_label_propagation (vis_correspondence.py:133-158): the label splatted at its tracked points onto every
    tracked frame, each frame's images laid out by images2grid with nrow = int(sqrt(N)), `initial_frames` first, and the
    whole video reversed.  frames (T, N, 3, R, R): smooth_congealing's frames without the flip stage's first
    flip_length; points (T, N, P, 2): smooth_congealing's tracked points; colors (N or 1, P, 3) in [-1, 1] (required)
    and alpha_channel (N or 1, P, 1) or None; initial_frames (F0, Hg, Wg, 3) uint8 or None.  One splat_composite_grid
    call of the op set (cuda_ops() by default).  -> (F0 + T, Hg, Wg, 3) uint8."""
    ops = _ops_or_cuda(ops)
    colors, alpha_channel = _label_inputs(colors, alpha_channel)
    nrow = int(math.sqrt(frames.size(1)))
    out = ops.splat_composite_grid(frames, points, colors, alpha_channel, sigma, opacity, nrow)
    if initial_frames is not None:
        out = torch.cat([initial_frames.to(out.device), out], 0)
    return out.flip(0)


@torch.no_grad()
def smooth_correspondence(t, data, label_points, colors, alpha_channel=None, sigma=1.2, opacity=0.7,
                          **smooth_congealing_kwargs):
    """smoothly_congeal_and_propagate's three videos (vis_correspondence.py:208-298, :118-130): the congealing
    animation of `data`, the propagation of the dense label (label_points (P, 2) at `resolution`, as smooth_congealing)
    and the correspondence video that joins them.  With stage_flip, the propagation starts with the label splatted at its
    unclamped unaligned points onto the images sampled on the identity grid, flipped as the images are (:263-271).
    The correspondence video is the congealing frames, 60 pauses on the last one, 60 frames blending it into the first
    propagation frame (float lerp, clamp(0, 255), round, on the host as the reference does), the propagation frames and 5
    pauses on the last one.  Every grid comes from the op set's splat_composite_grid.  colors (N or 1, P, 3) are
    required; alpha_channel (N or 1, P, 1) or None.  smooth_congealing_kwargs: smooth_congealing's keyword arguments.
    -> dict of uint8 (F, Hg, Wg, 3) tensors on data's device: congealing, propagation, correspondence."""
    kw = dict(resolution=256, length=240, flip_length=40, vis_in_stages=False, stage_flip=False, output_resolution=None,
              classifier=None, cluster=None, num_heads=1, no_flip_inference=False, iters=1, padding_mode="border")
    unknown = set(smooth_congealing_kwargs) - set(kw)
    if unknown:
        raise TypeError("smooth_correspondence: unexpected keyword arguments %s" % sorted(unknown))
    kw.update(smooth_congealing_kwargs)
    ops = t.ops
    colors, alpha_channel = _label_inputs(colors, alpha_channel)
    frames, points, unaligned, flip_indices = _smooth_congealing(t, data, label_points, **kw)
    n, res = data.size(0), frames.size(-1)
    nrow = int(math.sqrt(n))
    congealing = ops.splat_composite_grid(frames, None, None, None, sigma, opacity, nrow)
    initial, tracked = None, frames
    if kw["stage_flip"]:
        tracked = frames[kw["flip_length"]:]
        identity = _identity(n, res, data)
        images = ops.mipmap_warp(data, identity, WARP_LEVELS)[0]
        splatted = _splat_points(ops, images, unaligned, colors, alpha_channel, sigma, opacity)
        flipped = ops.mipmap_warp_lerp(splatted, identity, flip_grid(identity, flip_indices),
                                       cosine_alphas(kw["flip_length"], data.device), WARP_LEVELS)[0]
        initial = ops.splat_composite_grid(flipped, None, None, None, sigma, opacity, nrow)
    propagation = label_propagation_frames(tracked, points, colors, alpha_channel, sigma, opacity, initial, ops=ops)
    blend = torch.linspace(0, 1, steps=INTERP_STEPS).view(INTERP_STEPS, 1, 1, 1)
    interp = congealing[-1:].cpu().float().lerp(propagation[:1].cpu().float(), blend).clamp(0, 255).round().to(torch.uint8)
    correspondence = torch.cat([congealing, congealing[-1:].expand(PAUSE_STEPS, -1, -1, -1), interp.to(congealing.device),
                                propagation, propagation[-1:].expand(END_PAUSE_STEPS, -1, -1, -1)], 0)
    return {"congealing": congealing, "propagation": propagation, "correspondence": correspondence}


def _minmax_normalize(images, amin=None, amax=None):
    """utils/vis_tools/helpers.py:26-36 `normalize`: per-image min/max, or clamp to the given range."""
    if amin is None:
        amin, amax = images.amin(dim=(1, 2, 3), keepdim=True), images.amax(dim=(1, 2, 3), keepdim=True)
    else:
        amin, amax = torch.tensor(amin, device=images.device), torch.tensor(amax, device=images.device)
        images = images.clamp(amin, amax)
    return images.sub(amin).div(torch.maximum(amax - amin, torch.tensor(1e-5, device=images.device)))


@torch.no_grad()
def labeled_average_frames(average_frames, label_points, colors, alpha_channel=None, sigma=1.2, opacity=0.7,
                           resolution=256, ops=None):
    """The average-image video of average_and_congeal with its labelled tail (vis_correspondence.py:420-437): the frames
    min/max-normalised one by one; the label splatted onto the last frame (splat_points on the op set's splat2d); 60
    pauses on the last frame, 60 frames blending it into the labelled frame, 5 pauses on that; then mul(255).round().
    average_frames (F, 3, R, R): congealing_average_frames' frames; label_points (P, 2) integer pixels at `resolution`
    (converted to R and rounded as sample_images_and_points does); colors (1, P, 3) in [-1, 1] (required) and
    alpha_channel (1, P, 1) or None.  The op set is cuda_ops() by default.  -> (F + 125, R, R, 3) uint8."""
    ops = _ops_or_cuda(ops)
    colors, alpha_channel = _label_inputs(colors, alpha_channel)
    frames = _minmax_normalize(average_frames.float())
    res = frames.size(-1)
    points = label_points.to(frames.device)
    if resolution != res:
        points = _unnormalize(_normalize(points, res, resolution), res, res).round().long()
    last = frames[-1:].mul(2).add(-1)
    labeled = _splat_points(ops, last, points.float().unsqueeze(0), colors, alpha_channel, sigma, opacity)
    blend = torch.linspace(0, 1, steps=INTERP_STEPS, device=frames.device).view(INTERP_STEPS, 1, 1, 1)
    interp = _minmax_normalize(last.lerp(labeled, blend), -1, 1)
    frames = torch.cat([frames, frames[-1:].repeat(PAUSE_STEPS, 1, 1, 1), interp,
                        interp[-1:].repeat(END_PAUSE_STEPS, 1, 1, 1)], 0)
    return frames.mul(255.0).round().permute(0, 2, 3, 1).to(torch.uint8)
