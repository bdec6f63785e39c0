"""Restatements of the training visuals' ops (test infrastructure -- see oracle/__init__.py).

Reference: utils/vis_tools/flow_vis.py (the colour wheel, with numpy's precision as the reference runs it), torchvision
make_grid(normalize=True) + utils/vis_tools/helpers.py:39-43 images2grid (the normalised grid), and
utils/vis_tools/training_vis.py:57-109 (the routed per-cluster sums).  `cpu_ops()` is oracle.labels.cpu_ops() plus the
three entries, so gangealing_b200.training.visuals runs end to end on the CPU restatement.
"""
import types

import numpy as np
import torch
from torchvision.utils import make_grid

from . import labels as _labels

RY, YG, GC, CB, BM, MR = 15, 6, 4, 11, 13, 6
NCOLS = RY + YG + GC + CB + BM + MR


def color_wheel():
    """(55, 3) float64: Baker et al.'s wheel, each entry floor(255 * i / n) of its ramp."""
    ramps = [(RY, (255, "up", 0)), (YG, ("down", 255, 0)), (GC, (0, 255, "up")), (CB, (0, "down", 255)),
             (BM, ("up", 0, 255)), (MR, (255, 0, "down"))]
    rows = []
    for n, spec in ramps:
        up = np.floor(255 * np.arange(n) / n)
        rows.append(np.stack([up if s == "up" else 255 - up if s == "down" else np.full(n, float(s)) for s in spec], 1))
    return np.concatenate(rows, 0)


def flow_colors(flow):
    """flow (N, H, W, 2) float32 -> (N, H, W, 3) uint8 floor(255 * col): float32 up to fk, float64 from f = fk - k0 on
    (numpy's promotion of float32 - int32), as flow_to_image runs in the reference."""
    f = np.asarray(flow, dtype=np.float32) * np.float32(flow.shape[1] - 1)
    u, v = f[..., 0], f[..., 1]
    rad_max = np.max(np.sqrt(np.square(u) + np.square(v)))
    den = np.float32(rad_max + np.float32(1e-5))
    u, v = u / den, v / den
    rad = np.sqrt(np.square(u) + np.square(v))
    a = np.arctan2(-v, -u) / np.float32(np.pi)
    fk = (a + np.float32(1)) / np.float32(2) * np.float32(NCOLS - 1)
    k0 = np.floor(fk).astype(np.int32)
    k1 = k0 + 1
    k1[k1 == NCOLS] = 0
    fr = fk.astype(np.float64) - k0
    wheel = color_wheel()
    out = np.zeros(u.shape + (3,), np.uint8)
    for i in range(3):
        col = (1 - fr) * (wheel[k0, i] / 255.0) + fr * (wheel[k1, i] / 255.0)
        inside = rad <= 1
        col = np.where(inside, 1 - rad.astype(np.float64) * (1 - col), col * 0.75)
        out[..., i] = np.floor(255 * col)
    return out


def flow_explained(flow):
    """(N, H, W, 3) bool: where a port may differ from flow_colors by an atan2 ulp or a step tie -- numpy's float32
    arctan2 and the correctly rounded float32 atan2 give different fk, or 255 * col lies within 1e-3 of an integer."""
    f = np.asarray(flow, dtype=np.float32) * np.float32(flow.shape[1] - 1)
    u, v = f[..., 0], f[..., 1]
    den = np.float32(np.max(np.sqrt(np.square(u) + np.square(v))) + np.float32(1e-5))
    u, v = u / den, v / den
    a32 = np.arctan2(-v, -u)
    a64 = np.arctan2(-v.astype(np.float64), -u.astype(np.float64)).astype(np.float32)
    ulp = a32 != a64
    rad = np.sqrt(np.square(u) + np.square(v)).astype(np.float64)
    fk = ((a32 / np.float32(np.pi) + np.float32(1)) / np.float32(2) * np.float32(NCOLS - 1))
    k0 = np.floor(fk).astype(np.int32)
    k1 = np.where(k0 + 1 == NCOLS, 0, k0 + 1)
    fr = fk.astype(np.float64) - k0
    wheel = color_wheel()
    out = np.zeros(u.shape + (3,), bool)
    for i in range(3):
        col = (1 - fr) * (wheel[k0, i] / 255.0) + fr * (wheel[k1, i] / 255.0)
        col = np.where(rad <= 1, 1 - rad * (1 - col), col * 0.75) * 255
        out[..., i] = ulp | (np.abs(col - np.round(col)) < 1e-3)
    return out


def images2grid(images, nrow, value_range, scale_each=False, padding=2):
    """GANgealingWriter._log_image_grid's array: make_grid(normalize=True, value_range, scale_each) then mul(255),
    add(0.5), clamp(0, 255), uint8 -> (Hg, Wg, 3)."""
    grid = make_grid(images.float(), nrow=nrow, padding=padding, pad_value=0, normalize=True, value_range=value_range,
                     scale_each=scale_each)
    return grid.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)


def flow_image_grid_ref(flow, nrow, padding=2):
    """The op set's flow_image_grid: the reference's flow_to_image (/ 255) through images2grid(range=(0, 1))."""
    colors = torch.from_numpy(flow_colors(flow.detach().cpu().float().numpy())).float().div(255.0).permute(0, 3, 1, 2)
    return images2grid(colors, nrow, (0, 1), padding=padding).to(flow.device)


def image_grid_ref(images, ranges, nrow, padding=2):
    """The op set's image_grid: every image normalised by its own (lo, hi) as make_grid's norm_ip does."""
    shown = []
    for img, (lo, hi) in zip(images.float(), ranges.tolist()):
        x = img.clamp(min=lo, max=hi)
        shown.append(x.sub(lo).div(max(hi - lo, 1e-5)))
    return images2grid(torch.stack(shown), nrow, (0, 1), padding=padding)


def cluster_accumulate_ref(sums, counts, keep, images, sel):
    """The op set's cluster_accumulate, image by image as generate_cluster_congeal's host loop does (in place)."""
    k = images.size(2)
    for n, s in enumerate(sel.tolist()):
        c = s % k
        img = images[s // k, n, c].float()
        if keep is not None and counts[c] < keep.size(1):
            keep[c, counts[c]] = img
        sums[c] += img
        counts[c] += 1


def routed_sums_f64(images, sel, num_heads):
    """float64 per-cluster sums and counts of the routed images (the accuracy reference of the sums)."""
    chw = images.shape[3:]
    sums = torch.zeros((num_heads,) + tuple(chw), dtype=torch.float64)
    counts = torch.zeros(num_heads, dtype=torch.int64)
    for n, s in enumerate(sel.tolist()):
        sums[s % num_heads] += images[s // num_heads, n, s % num_heads].double().cpu()
        counts[s % num_heads] += 1
    return sums, counts


def cpu_ops():
    """oracle.labels.cpu_ops() plus flow_image_grid, image_grid and cluster_accumulate."""
    return types.SimpleNamespace(**vars(_labels.cpu_ops()), flow_image_grid=flow_image_grid_ref, image_grid=image_grid_ref,
                                 cluster_accumulate=cluster_accumulate_ref)
