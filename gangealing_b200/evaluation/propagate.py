"""Dense labels and edits put on real images (reference applications/propagate_to_images.py:29-104, with
utils/vis_tools/helpers.py:49-55 `load_pil`, :79-108 `load_dense_label` and applications/vis_correspondence.py:48-54, the
label handling of `sample_images_and_points`).

The reference runs the STN four times over the N images of a batch (determine_flips' forward_with_flip twice,
t(reals_flipped) once, uncongeal_points once) and puts every output through make_grid and a uint8 cast on the host.
`propagate_to_images` runs it once over the images and their mirrors (ComposedSTN.congeal_and_grid: 2N images, or N
when a cluster classifier or no_flip_inference decides the flips), and writes every grid as uint8 on the device: the
input and congealed grids through the op set's splat_composite_grid without points, the propagated grid through one
splat_lookup_composite_grid call (lookup, flip, splat, composite and grid in one scatter and one composite launch).
Colours are required: the reference's Plotly colour scales are not reproduced.
"""
import math
import os

import torch
import torch.nn.functional as F

from .flips import determine_flips
from .visuals import _label_inputs, _normalize, _unnormalize

GRID_PADDING = 3   # write(): save_image(nrow=int(sqrt(N)), padding=3, pad_value=-1); -1 and 0 both store byte 0


def grid_cells(grid, n, r, nrow, padding=GRID_PADDING):
    """The n images of a make_grid layout, (Hg, Wg, 3) -> (n, r, r, 3): what write(save_individual_images) stores."""
    xmaps = min(nrow, n)
    pad = 0 if n == 1 else padding
    cells = []
    for k in range(n):
        y, x = pad + (k // xmaps) * (r + pad), pad + (k % xmaps) * (r + pad)
        cells.append(grid[y:y + r, x:x + r])
    return torch.stack(cells, 0)


def label_queries(label_points, resolution, output_resolution):
    """sample_images_and_points (vis_correspondence.py:48-54): label pixels (P, 2) at `resolution` -> (the normalised
    congealed-frame queries (1, P, 2) uncongeal_points reads, the label's pixels at output_resolution (1, P, 2): converted
    and rounded when the resolutions differ)."""
    points = label_points.unsqueeze(0)
    queries = _normalize(points, output_resolution, resolution)
    if resolution != output_resolution:
        points = _unnormalize(_normalize(points, output_resolution, resolution), output_resolution,
                              output_resolution).round().long()
    return queries, points


@torch.no_grad()
def propagate_to_images(t, images, label_points=None, colors=None, alpha_channel=None, sigma=1.3, opacity=0.75,
                        resolution=256, output_resolution=None, average_image=None, classifier=None, cluster=None,
                        num_heads=1, no_flip_inference=False, iters=1, padding_mode="border", individual=False):
    """make_visuals (propagate_to_images.py:44-78) on the images (N, 3, R, R) in [-1, 1] the caller selected.
    label_points: (P, 2) integer (x, y) pixels of the label in the congealed frame at `resolution`, or None; colors
    (1 or N, P, 3) in [-1, 1] (required with a label) and alpha_channel (1 or N, P, 1) or None (opaque);
    output_resolution: the congealed images' size (None: R, as the script's default); average_image (1, 3, R, R) in
    [-1, 1] (average_png's image) or None.  The flip comes from the one STN pass, or from determine_flips with a cluster
    classifier (cluster, num_heads) or no_flip_inference.  All grids are make_grid(nrow=int(sqrt(N)), padding=3,
    normalize=True, range=(-1, 1)) as uint8 (Hg, Wg, 3) on the device, as write() saves them.
    -> dict: input_images, congealed_images, flips (N,) bool; with a label propagated and correspondences (N, P, 2), the
    label's pixels on the unflipped images; with a label and average_image average_annotated (R, R, 3); with individual,
    `individual`: {grid name: (N, R', R', 3) uint8}, the cells of each grid."""
    ops = t.ops
    n, r = images.size(0), images.size(-1)
    out_res = output_resolution or r
    nrow = int(math.sqrt(n))
    if classifier is None and not no_flip_inference:
        flip, congealed, grid = t.congeal_and_grid(images, True, out_res, iters, padding_mode)
    else:
        flipped, flip, policy = determine_flips(t, classifier, images, cluster=cluster, num_heads=num_heads,
                                                no_flip_inference=no_flip_inference, iters=iters, padding_mode=padding_mode)
        _, congealed, grid = t.congeal_and_grid(flipped, False, out_res, iters, padding_mode, warp_policy=policy)
        flip = flip.reshape(n).bool()

    def plain_grid(x):
        return ops.splat_composite_grid(x.unsqueeze(0), None, None, None, sigma, opacity, nrow, padding=GRID_PADDING)[0]

    results = {"flips": flip, "input_images": plain_grid(images), "congealed_images": plain_grid(congealed)}
    sizes = {"input_images": r, "congealed_images": congealed.size(-1)}
    if label_points is not None:
        if colors is None:
            raise ValueError("propagate_to_images: colors are required with a label (plotly colour scales are not supported)")
        colors, alpha_channel = _label_inputs(colors.to(images.device),
                                              None if alpha_channel is None else alpha_channel.to(images.device))
        queries, points = label_queries(label_points.to(images.device), resolution, out_res)
        results["propagated"], results["correspondences"] = ops.splat_lookup_composite_grid(
            images, grid, queries, flip, colors, alpha_channel, sigma, opacity, nrow, padding=GRID_PADDING)
        sizes["propagated"] = r
        if average_image is not None:   # :70-73: the label's own pixels on the average image, a single image
            results["average_annotated"] = ops.splat_composite_grid(
                average_image.float().unsqueeze(0), points.float().unsqueeze(0), colors[0:1],
                None if alpha_channel is None else alpha_channel[0:1], sigma, opacity, 1, padding=GRID_PADDING)[0]
    if individual:
        results["individual"] = {name: grid_cells(results[name], n, size, nrow) for name, size in sizes.items()}
    return results


@torch.no_grad()
def average_png(mean, ops=None):
    """average() (propagate_to_images.py:81-104): save_image(mean, normalize=True, range=None) -- the image scaled by its
    own min and max -- through the op set's image_grid, and the [-1, 1] image load_pil reads back from that PNG
    (helpers.py:49-55; PIL's resize to the same size is a copy, another size is the caller's business).
    mean: (1, 3, R, R) or (3, R, R), average_congealed_image's result.  -> ((R, R, 3) uint8, (1, 3, R, R) fp32)."""
    if ops is None:
        from ..opset import cuda_ops
        ops = cuda_ops()
    m = mean.reshape(-1, *mean.shape[-3:])[:1].float().contiguous()
    ranges = torch.stack([m.min(), m.max()]).view(1, 2)
    png = ops.image_grid(m, ranges, 1)
    return png, png.permute(2, 0, 1).unsqueeze(0).float().div(255.0).add(-0.5).mul(2)


@torch.no_grad()
def load_dense_label(path, resolution=None, load_colors=False, device="cuda"):
    """helpers.py:79-108: the pixels of an RGBA image with alpha > 0, in row-major order, as (1, P, 2) integer (x, y);
    with load_colors their colours (1, P, 3) in [-1, 1] and alphas (1, P, 1) in [0, 1], else (None, ones).  The
    reference's quirk is kept: `resolution != label.size(0)` compares with the batch dimension (1), so any given
    resolution resizes the label with bilinear interpolate(scale_factor=resolution / W).  -> (points, colors, alpha)."""
    import numpy as np
    from PIL import Image
    label = torch.from_numpy(np.array(Image.open(path))).to(device)
    label = label.permute(2, 0, 1).unsqueeze(0)
    if resolution is not None and resolution != label.size(0):
        label = F.interpolate(label.float(), scale_factor=resolution / label.size(2), mode="bilinear")
    if label.size(1) != 4:
        raise ValueError("load_dense_label: %s is not an RGBA image" % path)
    i, j = torch.where(label[0, 3] > 0)
    points = torch.stack([j, i], -1).unsqueeze(0)
    if load_colors:
        image = label.float().div(255.0)
        alpha_channel = image[:, 3:4, i, j].permute(0, 2, 1)
        colors = image[:, :3, i, j].add(-0.5).mul(2.0).permute(0, 2, 1)
    else:
        alpha_channel = torch.ones(1, points.size(1), 1, device=device, dtype=torch.float)
        colors = None
    return points, colors, alpha_channel


def save_propagation(results, out):
    """write() (propagate_to_images.py:29-37) of propagate_to_images' grids with PIL: `{out}/{name}_grid.png` for every
    grid and, with individual images, `{out}/{name}/{i:03}.png`.  -> the paths written."""
    from PIL import Image
    os.makedirs(out, exist_ok=True)
    paths = []
    for name in ("input_images", "congealed_images", "propagated", "average_annotated"):
        if name in results:
            paths.append(os.path.join(out, "%s_grid.png" % name))
            Image.fromarray(results[name].cpu().numpy()).save(paths[-1])
    for name, cells in results.get("individual", {}).items():
        os.makedirs(os.path.join(out, name), exist_ok=True)
        for i, cell in enumerate(cells.cpu().numpy()):
            paths.append(os.path.join(out, name, "%03d.png" % i))
            Image.fromarray(cell).save(paths[-1])
    return paths
