"""Torch restatement of the congealing visualisations (test infrastructure -- see oracle/__init__.py).

Reference: applications/vis_correspondence.py:59-114 (`pad_grid`, `nearest_neighbor_within_patch`), :166-205
(`flip_grid`, `get_patch_size`, `smoothly_sample_image`), :208-298 (`smoothly_congeal_and_propagate`), :335-437
(`create_average_image`, `average_and_congeal`) and applications/propagate_to_images.py:81-104 (`average`, with
utils/vis_tools/training_vis.py:15-28 `run_loader_mean` and utils/distributed.py:125-131 `all_reduce`).

Every function runs in the dtype and on the device of its inputs, so in float64 it is the accuracy reference of the CUDA
ops.  `average_frames_ref`, `smooth_congealing_ref` and `average_ref` are the reference's own per-frame compositions (the
flip inference and the STN run again for every frame) written against the mirror STN, so they run on any op set.
"""
import math
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

from .pck import determine_flips_ref, normalize, unnormalize, unravel_index


def pad_grid(grid):
    """(N, H, W, 2) -> (N, H+2, W+2, 2): replicate padding, then the ring replaced by linear extrapolations (:59-76)."""
    grid = F.pad(grid.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="replicate").permute(0, 2, 3, 1)
    right = 2 * grid[:, :, -2] - grid[:, :, -3]
    left = 2 * grid[:, :, 1] - grid[:, :, 2]
    bottom = 2 * grid[:, -2] - grid[:, -3]
    top = 2 * grid[:, 1] - grid[:, 2]
    grid = grid.clone()
    grid[:, 0] = top
    grid[:, -1] = bottom
    grid[:, :, 0] = left
    grid[:, :, -1] = right
    return grid


def nearest_neighbor_within_patch(grid, points, patch_centers, patch_size):
    """:79-114 line by line (the Unfold of the padded grid, the expanded distance, first minimum, index wrap)."""
    n, p = grid.size(0), points.size(1)
    unfold = nn.Unfold(patch_size, padding=patch_size // 2)
    grid = pad_grid(grid)
    padded = patch_centers + 1
    flat_centers = padded[..., 0] + grid.size(1) * padded[..., 1]
    patches = unfold(grid.permute(0, 3, 1, 2))
    patches = patches.gather(dim=2, index=flat_centers.view(n, 1, p).repeat(1, patches.size(1), 1))
    patches = patches.reshape(n, 2, patch_size, patch_size, p).permute(0, 2, 3, 4, 1).reshape(n, patch_size, patch_size, p, 1, 2)
    pts = points.reshape(n, 1, 1, p, 2, 1)
    sim = (patches @ pts)[..., 0, 0]
    dist = pts.pow(2).squeeze(-1).sum(dim=-1) + patches.pow(2).sum(dim=-1).squeeze(-1) - 2 * sim
    nearest = dist.reshape(n, patch_size * patch_size, p).argmin(dim=1)
    diff = unravel_index(nearest, (patch_size, patch_size)) - patch_size // 2
    out = flat_centers + diff[..., 0] + grid.size(1) * diff[..., 1]
    return unravel_index(out, (grid.size(1), grid.size(2))) - 1


def window_distances(grid, points, patch_centers, patch_size):
    """(N, P, patch^2) float64 exact distances |p - g|^2 of every window candidate (zero padding included): the tie rule
    of the tracking tests compares the candidates two trackers picked with these."""
    n, p = grid.size(0), points.size(1)
    g = pad_grid(grid.double())
    unfold = nn.Unfold(patch_size, padding=patch_size // 2)
    flat = (patch_centers[..., 0] + 1) + g.size(1) * (patch_centers[..., 1] + 1)
    patches = unfold(g.permute(0, 3, 1, 2)).gather(2, flat.view(n, 1, p).repeat(1, 2 * patch_size ** 2, 1))
    patches = patches.reshape(n, 2, patch_size * patch_size, p).permute(0, 3, 2, 1)       # (N, P, K, 2)
    return (patches - points.double().unsqueeze(2)).pow(2).sum(-1)


def flip_grid(grid, flip_indices):
    grid = grid.clone()
    grid[..., 0] = torch.where(flip_indices.view(1, -1, 1, 1), -grid[..., 0], grid[..., 0])
    return grid


def get_patch_size(length):
    patch_size = math.ceil(9 * max(1, 240 / length))
    return patch_size + 1 if patch_size % 2 == 0 else patch_size


def cosine_alpha(frame_ix, length):
    """:192 / :409, the reference's float32 expression."""
    return 1 - 0.5 * (1 + torch.cos(torch.tensor(math.pi * frame_ix / (length - 1))))


# ------------------------------------------------------------------------------------------------ the op set's three ops
def mipmap_warp_lerp_ref(inputs, base, target, alphas, max_num_levels=8, min_level=0.0, padding_mode="border"):
    from .sampling import mipmap_warp_ref
    grids = torch.stack([base.lerp(target, a.view(1, 1, 1, 1).to(base.dtype)) for a in alphas], 0)
    out = torch.stack([mipmap_warp_ref(inputs, g, max_num_levels, min_level, padding_mode) for g in grids], 0)
    return out, grids


def mipmap_warp_lerp_mean_ref(inputs, base, target, alphas, acc=None, max_num_levels=8, min_level=0.0,
                              padding_mode="border"):
    frames, _ = mipmap_warp_lerp_ref(inputs, base, target, alphas, max_num_levels, min_level, padding_mode)
    s = torch.zeros_like(frames[:, 0], dtype=torch.promote_types(frames.dtype, torch.float32))
    for i in range(frames.size(1)):
        s = s + frames[:, i]
    return s if acc is None else acc.copy_(acc + s)


def track_points_lerp_ref(base, target, alphas, points, centers, patch_size):
    track, c = [], centers.long()
    for a in alphas:
        c = nearest_neighbor_within_patch(base.lerp(target, a.view(1, 1, 1, 1).to(base.dtype)), points, c, patch_size)
        track.append(c)
    return torch.stack(track, 0), c


def cpu_ops():
    """oracle.pck.cpu_ops() plus the congealing-animation ops: the op set that runs gangealing_b200.evaluation.visuals
    on the CPU restatement."""
    from . import pck
    return types.SimpleNamespace(**vars(pck.cpu_ops()), mipmap_warp_lerp=mipmap_warp_lerp_ref,
                                 mipmap_warp_lerp_mean=mipmap_warp_lerp_mean_ref, track_points_lerp=track_points_lerp_ref)


# ------------------------------------------------------------------------------------------------ per-frame compositions
def _warper(t):
    from gangealing_b200.stn.sampling import MipmapWarp
    return MipmapWarp(3.5, ops=t.ops)


def _resize(grid, res):
    if res == grid.size(1):
        return grid
    return F.interpolate(grid.permute(0, 3, 1, 2), scale_factor=res / grid.size(1), mode="bilinear").permute(0, 2, 3, 1)


def create_average_image_ref(t, loader, warper, alpha, n_mean, output_resolution, warp_index, identity_grid, iters=1,
                             padding_mode="border"):
    """:335-380 on one process (no classifier): the flips and the STN run again for this frame."""
    average_image, total = 0, 0
    for data in loader:
        data_flipped, flip_indices = determine_flips_ref(t, data, iters, padding_mode)
        if warp_index >= 0:
            _, grids = t(data_flipped, warp_policy="cartesian", return_intermediates=True, iters=iters, padding_mode=padding_mode)
            grid = flip_grid(grids[warp_index], flip_indices)
            base = identity_grid.repeat(data.size(0), 1, 1, 1) if warp_index == 0 else grids[warp_index - 1]
            base = flip_grid(base, flip_indices)
        else:
            grid = flip_grid(identity_grid.repeat(data.size(0), 1, 1, 1), flip_indices)
            base = identity_grid
        grid = _resize(grid, output_resolution)
        base = _resize(base, output_resolution)
        congealed = warper(data, base.lerp(grid, alpha))
        n = congealed.size(0)
        if total + n > n_mean:
            n = n_mean - total
        average_image = average_image + congealed[:n].sum(dim=0, keepdim=True)
        total += n
        if total >= n_mean:
            break
    return (average_image / n_mean).mean(dim=0)


def average_frames_ref(t, batches, n_mean, length=240, flip_length=40, vis_in_stages=False, stage_flip=False,
                       output_resolution=None, iters=1, padding_mode="border"):
    """average_and_congeal's frames (:384-419) before `normalize`: -> (F, C, R, R)."""
    res = output_resolution or batches[0].size(-1)
    num_stages = (len(t.stns) if hasattr(t, "stns") and vis_in_stages else 1) + int(stage_flip)
    identity_grid = F.affine_grid(torch.eye(2, 3).unsqueeze(0), (1, 3, res, res)).to(batches[0])
    warper = _warper(t)
    frames = []
    for i in range(num_stages):
        n_frames = length if not stage_flip or i > 0 else flip_length
        for frame_ix in range(n_frames):
            alpha = cosine_alpha(frame_ix, n_frames).to(batches[0])
            frames.append(create_average_image_ref(t, batches, warper, alpha, n_mean, res, i - int(stage_flip), identity_grid,
                                                   iters, padding_mode))
    return torch.stack(frames, 0)


def average_ref(t, batches, n_mean, output_resolution=None, iters=1, padding_mode="border"):
    """propagate_to_images.average (:81-104) + run_loader_mean(unfold=False) + all_reduce on one process: -> (C, R, R)."""
    out, total = [], 0
    for x in batches:
        flipped, _ = determine_flips_ref(t, x, iters, padding_mode)
        out.append(t(flipped, warp_policy="cartesian", unfold=False, iters=iters, padding_mode=padding_mode,
                     output_resolution=output_resolution))
        total += x.size(0)
        if total >= n_mean:
            break
    out = torch.cat(out, 0)
    return out.sum(dim=0) / out.size(0)


def smooth_congealing_ref(t, data, label_points=None, resolution=256, length=240, flip_length=40, vis_in_stages=False,
                          stage_flip=False, output_resolution=None, iters=1, padding_mode="border"):
    """smoothly_congeal_and_propagate (:208-298) with sample_images_and_points' point handling (:48-54), frame by frame.
    -> (frames (F, N, C, R, R), points (stages * length, N, P, 2) float or None, unaligned-space points (N, P, 2) or None)."""
    res = output_resolution or data.size(-1)
    data_flipped, flip_indices = determine_flips_ref(t, data, iters, padding_mode)
    _, grids = t(data_flipped, return_intermediates=True, warp_policy="cartesian", padding_mode=padding_mode, iters=iters)
    if not vis_in_stages:
        grids = [grids[-1]]
    grids = flip_grid(torch.stack(grids), flip_indices.view(1, -1, 1, 1))
    flow_size = grids.size(2)
    if res != flow_size:
        g = grids.reshape(-1, flow_size, flow_size, 2)
        g = F.interpolate(g.permute(0, 3, 1, 2), scale_factor=res / flow_size, mode="bilinear").permute(0, 2, 3, 1)
        grids = g.reshape(-1, data.size(0), res, res, 2)
    identity_grid = F.affine_grid(torch.eye(2, 3).unsqueeze(0).repeat(data.size(0), 1, 1), (data.size(0), 3, res, res)).to(data)
    num_stages = grids.size(0)
    flipping_grid = flip_grid(identity_grid, flip_indices)
    grids = torch.cat([flipping_grid.unsqueeze(0), grids], 0)
    warper = _warper(t)
    n = data.size(0)
    normalized_unaligned = unaligned = centers = congealed_centers = None
    if label_points is not None:
        points = label_points.unsqueeze(0).repeat(n, 1, 1)
        points_normalized = normalize(points, res, resolution)
        if resolution != res:
            points = unnormalize(normalize(points, res, resolution), res, res).round().long()
        normalized_unaligned = F.grid_sample(grids[-1].permute(0, 3, 1, 2), points_normalized.unsqueeze(2).to(data.dtype),
                                             padding_mode="border", align_corners=False).squeeze(3).permute(0, 2, 1)
        unaligned = unnormalize(normalized_unaligned, res, res)
        centers = unaligned.round().long().clamp(0, res - 1)
        centers[..., 0] = torch.where(flip_indices.view(-1, 1), res - 1 - centers[..., 0], centers[..., 0])
        congealed_centers = points

    def run(target, base, n_frames, pts=None, c=None):
        imgs, track = [], []
        ps = get_patch_size(n_frames)
        for frame_ix in range(n_frames):
            grid_t = base.lerp(target, cosine_alpha(frame_ix, n_frames).to(data).view(1, 1, 1, 1))
            imgs.append(warper(data, grid_t))
            if pts is not None:
                c = nearest_neighbor_within_patch(grid_t, pts, c, ps)
                track.append(c.to(data.dtype))
        return torch.stack(imgs, 0), (torch.stack(track, 0) if track else None), c

    frames = []
    if stage_flip:
        frames.append(run(flipping_grid, identity_grid, flip_length)[0])
    propagated = []
    for i in range(num_stages):
        imgs, track, centers = run(grids[i + 1], grids[i], length, normalized_unaligned, centers)
        frames.append(imgs)
        propagated.append(track)
    if label_points is None:
        return torch.cat(frames, 0), None, None
    for i in range(num_stages):
        alpha = torch.linspace(0, 1, steps=length, device=data.device, dtype=data.dtype).view(length, 1, 1, 1)
        _, rev, congealed_centers = run(grids[-i - 2], grids[-i - 1], length, normalized_unaligned, congealed_centers)
        propagated[-i - 1].lerp_(rev.flip(0), alpha)
    return torch.cat(frames, 0), torch.cat(propagated, 0), unaligned
