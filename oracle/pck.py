"""Torch restatement of PCK-Transfer evaluation (test infrastructure -- see oracle/__init__.py).

Reference: applications/pck.py:103-175 (`pck_transfer`), models/spatial_transformers/spatial_transformer.py:242-295
(`match_flows`), :159-198 + :617-672 (the composed `transfer_points`), applications/__init__.py:57-84 (`determine_flips`),
applications/flow_scores.py:25-47 and models/losses/loss.py:4-12 (`total_variation_loss(reduce_batch=False)`).

Every function runs in the dtype and on the device of its inputs, so in float64 it is the accuracy reference of the CUDA
ops.  `pck_transfer_ref` is the reference's own composition -- `match_flows`, then `transfer_points` once per direction,
8N STN forwards per batch -- written against the mirror STN, so it runs on any op set.
"""
import types

import torch
import torch.nn.functional as F

ALPHAS = [0.1, 0.05, 0.01]       # run_pck_transfer's default --alphas


def tv_per_sample_ref(flow):
    """total_variation_loss(flow, reduce_batch=False): mean huber |d/dx| + mean huber |d/dy| per sample."""
    def huber(a):
        return torch.where(a <= 1.0, 0.5 * a.pow(2), a - 0.5).mean(dim=(1, 2, 3))
    dy = huber((flow[:, :-1] - flow[:, 1:]).abs())
    dx = huber((flow[:, :, :-1] - flow[:, :, 1:]).abs())
    return dx + dy


def normalize(points, res, out_res):
    return points.div(out_res - 1).add(-0.5).mul(2).mul((res - 1) / res)


def unnormalize(points, res, out_res):
    return points.div((res - 1) / res).div(2).add(0.5).mul(out_res - 1)


def _affine(points, matrix, invert):
    """[p, 1] @ ([M; 0 0 1] or its inverse)^T, homogeneous coordinate dropped (spatial_transformer.py:645-649, :693-696)."""
    n, p = points.shape[:2]
    hom = torch.cat([points, torch.ones(n, p, 1, dtype=points.dtype, device=points.device)], 2)
    last = torch.tensor([[[0, 0, 1]]], dtype=matrix.dtype, device=matrix.device).repeat(n, 1, 1)
    m3 = torch.cat([matrix, last], 1)
    return (hom @ (torch.inverse(m3) if invert else m3).permute(0, 2, 1))[..., [0, 1]]


def congeal_query_ref(points, matrix, size, composed):
    """Source key points (pixels) -> congealed-frame query: normalise, invert the similarity, and for a composed STN the
    un-normalise / normalise round trip between its two STNs (spatial_transformer.py:169-178, :641-651)."""
    q = _affine(normalize(points, size, size), matrix, invert=True)
    return normalize(unnormalize(q, size, size), size, size) if composed else q


def nn_distances_ref(grid, query):
    """The reference's expanded distance |p|^2 + |g|^2 - 2 g.p (spatial_transformer.py:659-663): (N, HW, P)."""
    n, h, w, _ = grid.shape
    g = grid.reshape(n, h, w, 1, 1, 2)
    pts = query.reshape(n, 1, 1, query.size(1), 2, 1)
    sim = (g @ pts)[..., 0, 0]
    dist = pts.pow(2).squeeze(-1).sum(dim=-1) + g.pow(2).sum(dim=-1).squeeze(-1) - 2 * sim
    return dist.reshape(n, h * w, query.size(1))


def unravel_index(indices, shape):
    coord = []
    for dim in reversed(shape):
        coord.append(indices % dim)
        indices = indices // dim
    return torch.stack(coord, dim=-1)


def pck_transfer_points_ref(points, gt, visible, thresh, alphas, matrix_src, size, delta_src=None, identity=None,
                            grid_dst=None, matrix_dst=None):
    """The op set's `pck_transfer_points` (gangealing_b200/evaluation/ops.py), restated with the reference's tensor
    operations.  -> (counts (A,) int64, est (B, P, 2), nn_index (B, P) int64 or None)."""
    composed = delta_src is not None
    q = congeal_query_ref(points, matrix_src, size, composed)
    nn_index = None
    if composed:
        g = delta_src + identity
        f = g.size(1)
        nn_index = nn_distances_ref(g, q).argmin(dim=1)
        idx = unravel_index(nn_index, (f, f)).to(points.dtype)
        qn = normalize(idx, size, f)
        est = F.grid_sample(grid_dst.permute(0, 3, 1, 2), qn.unsqueeze(2), padding_mode="border",
                            align_corners=False).squeeze(3).permute(0, 2, 1)
    else:
        est = _affine(q, matrix_dst, invert=False)
    est = unnormalize(est, size, size)
    err = (est - gt).norm(dim=-1).unsqueeze(-1)                                   # (B, P, 1)
    correct = err <= (alphas.view(1, -1) * thresh.view(-1, 1)).unsqueeze(1)      # (B, P, A), inclusive (pck.py:155)
    if visible is not None:
        correct = correct & (visible != 0).unsqueeze(-1)
    return correct.sum(dim=(0, 1)), est, nn_index


def match_flows_ref(t, imgA, imgB, pointsA, pointsB=None, permutation=None, **stn_forward_kwargs):
    """spatial_transformer.py:242-295 line by line (both quirks: the second relabelling permutes pointsA again, and
    pointsB is never relabelled), with tv_per_sample_ref for the smoothness."""
    imgA_flip, imgB_flip = imgA.flip(3,), imgB.flip(3,)
    _, flows = t(torch.cat([imgA, imgB, imgA_flip, imgB_flip], 0), return_flow=True, **stn_forward_kwargs)
    flowA, flowB, flowAf, flowBf = flows.chunk(4, dim=0)
    tvA, tvAf, tvB, tvBf = (tv_per_sample_ref(f) for f in (flowA, flowAf, flowB, flowBf))
    pick = torch.stack([tvA + tvB, tvAf + tvB, tvA + tvBf, tvAf + tvBf], 0).argmin(dim=0).view(imgA.size(0), 1, 1, 1)
    imgA = torch.where(pick % 2 == 0, imgA, imgA_flip)
    imgB = torch.where(pick <= 1, imgB, imgB_flip)
    pointsA = pointsA.clone()
    pointsA[:, :, 0] = torch.where((pick % 2 == 0).view(pick.size(0), 1), pointsA[:, :, 0], imgA.size(-1) - 1 - pointsA[:, :, 0])
    if permutation is not None:
        pointsA = torch.where((pick % 2 == 0).view(pick.size(0), 1, 1), pointsA, pointsA[:, permutation])
    if pointsB is not None:
        pointsB = pointsB.clone()
        pointsB[:, :, 0] = torch.where((pick <= 1).view(pick.size(0), 1), pointsB[:, :, 0], imgB.size(-1) - 1 - pointsB[:, :, 0])
        if permutation is not None:
            pointsA = torch.where((pick <= 1).view(pick.size(0), 1, 1), pointsA, pointsA[:, permutation])
        return imgA, imgB, pointsA, pointsB, pick
    return imgA, imgB, pointsA, pick


@torch.no_grad()
def pck_transfer_ref(t, loader, alpha=0.1, num_pairs=10000, device="cpu", transfer_both_ways=True, permutation=None,
                     match_flows=True, **stn_forward_kwargs):
    """applications/pck.py:103-175 on one process: match_flows_ref, then t.transfer_points per direction (8N STN
    forwards per batch).  -> (A,) float32."""
    num_alphas = len(alpha) if isinstance(alpha, (list, tuple)) else 1
    correct = torch.zeros(num_alphas, device=device)
    alpha = torch.tensor(alpha, device=device).view(1, num_alphas)
    pairs_seen, key_points_seen = 0, 0
    while pairs_seen < num_pairs:
        d = next(loader)
        if d["imgsA"].size(0) > num_pairs - pairs_seen:
            d = {key: val[:num_pairs - pairs_seen] for key, val in d.items()}
        imgsA, imgsB, kpsA, kpsB = d["imgsA"].to(device), d["imgsB"].to(device), d["kpsA"].to(device), d["kpsB"].to(device)
        if kpsA.size(-1) == 3:
            visible = kpsA[..., 2:3] * kpsB[..., 2:3]
            kpsA, kpsB = kpsA[..., :2].clone(), kpsB[..., :2].clone()
        else:
            visible = torch.ones(kpsA.size(0), kpsA.size(1), 1, device=device)
        if match_flows:
            imgsA, imgsB, kpsA, kpsB, _ = match_flows_ref(t, imgsA, imgsB, kpsA, kpsB, permutation, **stn_forward_kwargs)
        est = t.transfer_points(imgsA, imgsB, kpsA, **stn_forward_kwargs)
        thr = (torch.tensor(max(imgsB.size(-2), imgsB.size(-1)), device=device) if "threshB" not in d
               else (d["scaleB"] * d["threshB"]).to(device))
        correct += ((est - kpsB).norm(dim=-1).unsqueeze(-1) <= (alpha * thr.view(-1, 1)).unsqueeze(1)).mul(visible).sum(dim=(0, 1))
        if transfer_both_ways:
            est = t.transfer_points(imgsB, imgsA, kpsB, **stn_forward_kwargs)
            thr = (torch.tensor(max(imgsA.size(-2), imgsA.size(-1)), device=device) if "threshA" not in d
                   else (d["scaleA"] * d["threshA"]).to(device))
            correct += ((est - kpsA).norm(dim=-1).unsqueeze(-1) <= (alpha * thr.view(-1, 1)).unsqueeze(1)).mul(visible).sum(dim=(0, 1))
        pairs_seen += imgsA.size(0)
        key_points_seen += visible.sum() * (1 + transfer_both_ways)
    return correct.float() / key_points_seen


def determine_flips_ref(t, imgs, iters=1, padding_mode="border"):
    """applications/__init__.py:71-75 (no classifier, flip inference on): -> (images, flip indices (N, 1, 1, 1))."""
    _, flipped, idx = t.forward_with_flip(imgs, return_inputs=True, return_flip_indices=True, padding_mode=padding_mode,
                                          iters=iters)
    return flipped, idx


def flow_scores_ref(t, batch, iters=1, padding_mode="border"):
    """applications/flow_scores.py:33-38 for one batch: -> (N,) negated per-sample smoothness after the flip decision."""
    batch, _ = determine_flips_ref(t, batch, iters, padding_mode)
    _, flows = t(batch, return_flow=True, iters=iters, padding_mode=padding_mode)
    return -tv_per_sample_ref(flows)


def cpu_ops():
    """oracle.blend.cpu_ops() plus `tv_per_sample` and `pck_transfer_points`: the op set that runs match_flows and
    gangealing_b200.evaluation on the CPU restatement."""
    from . import blend
    return types.SimpleNamespace(**vars(blend.cpu_ops()), tv_per_sample=tv_per_sample_ref,
                                 pck_transfer_points=pck_transfer_points_ref)


# ------------------------------------------------------------------------------------------------ near-tie exemptions
def nn_near_ties(grid, query, band, perturbation=0.0):
    """(B, P) bool: the float64 second-best squared distance lies within `band` of the best (the NN index may go either
    way).  `perturbation` bounds how far the compared side's grid and query may lie from these (the two sides ran the
    network on different hardware): it widens the band by what such a shift can change the squared distances."""
    d = nn_distances_ref(grid.double(), query.double())
    two = d.topk(2, dim=1, largest=False).values
    return (two[:, 1] - two[:, 0]) <= band + 4 * perturbation * (two[:, 0].clamp_min(0).sqrt() + perturbation)


def pick_near_ties(tv, band):
    """(N,) bool: the two smallest of match_flows' four smoothness sums lie within `band` (relative) of each other."""
    tvA, tvB, tvAf, tvBf = tv.double().chunk(4, dim=0)
    sums = torch.stack([tvA + tvB, tvAf + tvB, tvA + tvBf, tvAf + tvBf], 0)
    two = sums.topk(2, dim=0, largest=False).values
    return (two[1] - two[0]) <= band * two[0].abs().clamp_min(1e-12)


def threshold_near_ties(est, gt, thresh, alphas, tol=1e-4):
    """(B, P) bool: the error of some alpha lies within `tol` pixels of its threshold."""
    err = (est.double() - gt.double()).norm(dim=-1).unsqueeze(-1)
    thr = (alphas.double().view(1, -1) * thresh.double().view(-1, 1)).unsqueeze(1)
    return ((err - thr).abs() <= tol).any(dim=-1)
