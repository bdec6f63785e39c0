"""PCK-Transfer (reference applications/pck.py:103-175) from ONE STN forward per batch.

The reference runs the STN on 4N images in `match_flows`, then on N + N in `transfer_points` for A -> B and N + N more for
B -> A.  Those 4N later images are exactly the ones `match_flows` already warped (the STN treats every sample on its own),
so `pck_transfer_batch` keeps, per sample, the similarity matrix, residual flow and sampling grid of the variant the
flip inference picked, and scores both directions in one `pck_transfer_points` call of 2N source -> destination pairs.
"""
import torch

from ..stn.transformer import ComposedSTN, flip_key_points, match_pick
from ..training.distributed import all_gather, get_rank, get_world_size, primary

_STN_KWARGS = ("iters", "padding_mode")


def _check(t, stn_forward_kwargs):
    unknown = sorted(set(stn_forward_kwargs) - set(_STN_KWARGS))
    if unknown:
        raise TypeError("pck_transfer: unsupported STN forward arguments %s (only iters and padding_mode)" % unknown)
    if getattr(t, "num_heads", 1) > 1:
        raise ValueError("pck_transfer: clustering STNs (num_heads > 1) are not supported; evaluate one head at a time")


def _stn_outputs(t, imgs, stn_forward_kwargs):
    """-> (matrix (M, 2, 3), residual flow or None, sampling grid or None) of one forward over imgs."""
    if isinstance(t, ComposedSTN):
        return t._matrix_flow_grid(imgs, **stn_forward_kwargs)
    if t.is_flow:
        raise ValueError("pck_transfer: a flow-only SpatialTransformer has no similarity to invert; use a ComposedSTN")
    _, matrix = t(imgs, return_flow=True, **stn_forward_kwargs)
    return matrix, None, None


def pck_transfer_batch(t, imgsA, imgsB, kpsA, kpsB, alphas, threshA=None, threshB=None, visible=None, permutation=None,
                       transfer_both_ways=True, match_flows=True, **stn_forward_kwargs):
    """One batch of pck_transfer: N pairs (imgsA, imgsB) (N, C, S, S) with key points kpsA / kpsB (N, P, 2) in pixels.
    alphas: (A,) tensor on the images' device; threshA / threshB: (N,) per-image thresholds (default max(H, W));
    visible: (N, P) 0/1 (default all); permutation: device int64 tensor (P,) or None.
    No host synchronisation: the call can be captured in a CUDA graph.
    -> (counts (A,) int64 of correct transfers, number of visible key points scored (float scalar))."""
    args, kwargs, _, n_vis = transfer_arguments(t, imgsA, imgsB, kpsA, kpsB, alphas, threshA, threshB, visible, permutation,
                                                transfer_both_ways, match_flows, **stn_forward_kwargs)
    counts, _, _ = t.ops.pck_transfer_points(*args, **kwargs)
    return counts, n_vis


def transfer_arguments(t, imgsA, imgsB, kpsA, kpsB, alphas, threshA=None, threshB=None, visible=None, permutation=None,
                       transfer_both_ways=True, match_flows=True, **stn_forward_kwargs):
    """pck_transfer_batch up to the scoring call: -> (args, kwargs of the op set's pck_transfer_points, pick (N, 1, 1, 1) or
    None, number of visible key points scored)."""
    _check(t, stn_forward_kwargs)
    n, size, dev = imgsA.size(0), imgsA.size(-1), imgsA.device
    if match_flows and not isinstance(t, ComposedSTN):
        raise ValueError("pck_transfer: match_flows needs a ComposedSTN (flip inference compares residual flows)")
    if visible is None:
        visible = torch.ones(n, kpsA.size(1), device=dev)
    full = float(max(imgsA.size(-2), imgsA.size(-1)))
    threshA = torch.full((n,), full, device=dev) if threshA is None else threshA
    threshB = torch.full((n,), full, device=dev) if threshB is None else threshB
    imgs = [imgsA, imgsB] + ([imgsA.flip(3,), imgsB.flip(3,)] if match_flows else [])
    matrix, delta, grid = _stn_outputs(t, torch.cat(imgs, 0), stn_forward_kwargs)
    rowA = torch.arange(n, device=dev)
    rowB = rowA + n
    pick = None
    if match_flows:
        pick = match_pick(t.ops.tv_per_sample(delta))
        rowA = rowA + 2 * n * (pick.view(n) % 2)               # the flipped variant sits 2N rows further down
        rowB = rowB + 2 * n * (pick.view(n) > 1).long()
        kpsA, kpsB = flip_key_points(pick, kpsA, kpsB, permutation, size)
    if transfer_both_ways:
        src, dst = torch.cat([rowA, rowB]), torch.cat([rowB, rowA])
        pts, gt, thresh = torch.cat([kpsA, kpsB]), torch.cat([kpsB, kpsA]), torch.cat([threshB, threshA])
        vis = torch.cat([visible, visible])
    else:
        src, dst, pts, gt, thresh, vis = rowA, rowB, kpsA, kpsB, threshB, visible
    if delta is not None:
        kwargs = dict(delta_src=delta[src], identity=t.identity_flow, grid_dst=grid[dst])
    else:
        kwargs = dict(matrix_dst=matrix[dst])
    return (pts, gt, vis, thresh, alphas, matrix[src], size), kwargs, pick, visible.sum() * (1 + bool(transfer_both_ways))


@torch.inference_mode()
def pck_transfer(t, loader, alpha=0.1, num_pairs=10000, device="cuda", quiet=True, transfer_both_ways=True,
                 permutation=None, match_flows=True, **stn_forward_kwargs):
    """PCK-Transfer of STN `t` over `num_pairs` pairs drawn from `loader` (an iterator of batch dicts with imgsA, imgsB,
    kpsA, kpsB (N, P, 2 or 3: x, y, visibility) and optionally threshA / scaleA, threshB / scaleB), split across ranks as
    the reference does.  alpha: float or list of up to 8 floats.  -> (A,) tensor: the fraction of visible key points
    transferred within alpha * threshold, over both directions if transfer_both_ways."""
    _check(t, stn_forward_kwargs)
    world = get_world_size()
    pairs_needed = num_pairs // world + (get_rank() < num_pairs % world)   # some ranks take one extra pair
    alphas = torch.tensor(alpha, dtype=torch.float32, device=device).view(-1)
    perm = None if permutation is None else torch.as_tensor(permutation, dtype=torch.long, device=device)
    correct = torch.zeros(alphas.numel(), dtype=torch.int64, device=device)
    seen = torch.zeros((), dtype=torch.float32, device=device)
    pbar = None
    if not quiet and primary():
        from tqdm import tqdm
        pbar = tqdm(total=pairs_needed)
    pairs_seen = 0
    while pairs_seen < pairs_needed:
        d = next(loader)
        still = pairs_needed - pairs_seen
        if d["imgsA"].size(0) > still:            # do not overshoot the number of pairs
            d = {key: val[:still] for key, val in d.items()}
        imgsA, imgsB, kpsA, kpsB = d["imgsA"].to(device), d["imgsB"].to(device), d["kpsA"].to(device), d["kpsB"].to(device)
        visible = None
        if kpsA.size(-1) == 3:                    # (x, y, visibility)
            visible = kpsA[..., 2] * kpsB[..., 2]
            kpsA, kpsB = kpsA[..., :2].contiguous(), kpsB[..., :2].contiguous()
        threshA = (d["scaleA"] * d["threshA"]).to(device) if "threshA" in d else None
        threshB = (d["scaleB"] * d["threshB"]).to(device) if "threshB" in d else None
        counts, n_vis = pck_transfer_batch(t, imgsA, imgsB, kpsA, kpsB, alphas, threshA, threshB, visible, perm,
                                           transfer_both_ways, match_flows, **stn_forward_kwargs)
        correct += counts
        seen += n_vis
        pairs_seen += imgsA.size(0)
        if pbar is not None:
            pbar.update(imgsA.size(0))
    total = all_gather(seen.view(1)).sum()
    return torch.stack(all_gather(correct, cat=False), 0).sum(dim=0).float() / total
