"""The two sm_90a ops of PCK-Transfer evaluation (csrc/pck.cu), registered in `cuda_ops()` as `tv_per_sample` and
`pck_transfer_points`; oracle/pck.py restates both on the CPU with the same signatures."""
import torch

from .. import _lib


def tv_per_sample(flow):
    """total_variation_loss(flow, reduce_batch=False) (reference models/losses/loss.py:4-12) of a (N, H, W, 2) flow: one
    launch, one CTA per sample, bitwise reproducible.  -> (N,) float32."""
    _lib.require_cuda(flow)
    if flow.dim() != 4 or flow.size(-1) != 2:
        raise RuntimeError("tv_per_sample: expected a (N, H, W, 2) flow, got %s" % (tuple(flow.shape),))
    f = flow.detach().float().contiguous()
    n, h, w, _ = f.shape
    out = torch.empty(n, dtype=torch.float32, device=f.device)
    _lib.check(_lib.load().gg_tv_per_sample(out.data_ptr(), f.data_ptr(), n, h, w, _lib.stream()), "gg_tv_per_sample")
    return out


def pck_transfer_points(points, gt, visible, thresh, alphas, matrix_src, size, delta_src=None, identity=None, grid_dst=None,
                        matrix_dst=None):
    """One transfer direction of PCK-Transfer for B (source, destination) pairs, in one C-ABI call (gg_pck_transfer).

    points / gt: (B, P, 2) key points in pixels of the size x size source / destination images; visible: (B, P) 0/1 or None;
    thresh: (B,) per-destination threshold; alphas: (A,) with 1 <= A <= 8; matrix_src: (B, 2, 3) the source's similarity.
    Composed STN: delta_src (B, F, F, 2) the source's residual flow, identity (1, F, F, 2) its identity flow and grid_dst
    (B, F, F, 2) the destination's sampling grid.  Similarity-only STN: matrix_dst (B, 2, 3) instead.
    -> (counts (A,) int64: visible points with |est - gt| <= alpha * thresh, est (B, P, 2), nn_index (B, P) int64 or None)."""
    flow = delta_src is not None
    _lib.require_cuda(points, gt, visible, thresh, alphas, matrix_src, delta_src, identity, grid_dst, matrix_dst)
    b, p = points.shape[0], points.shape[1]
    if points.dim() != 3 or points.size(2) != 2 or gt.shape != points.shape:
        raise RuntimeError("pck_transfer_points: points and gt must both be (B, P, 2)")
    if thresh.shape != (b,) or matrix_src.shape != (b, 2, 3) or alphas.dim() != 1:
        raise RuntimeError("pck_transfer_points: thresh (B,), matrix_src (B, 2, 3) and alphas (A,) expected")
    if visible is not None and visible.shape != (b, p):
        raise RuntimeError("pck_transfer_points: visible must be (B, P)")
    if flow:
        if identity is None or grid_dst is None:
            raise RuntimeError("pck_transfer_points: a composed STN needs delta_src, identity and grid_dst")
        f = delta_src.size(1)
        if delta_src.shape != (b, f, f, 2) or identity.numel() != f * f * 2 or grid_dst.dim() != 4 or grid_dst.size(0) != b:
            raise RuntimeError("pck_transfer_points: delta_src (B, F, F, 2), identity (1, F, F, 2), grid_dst (B, F, F, 2)")
    elif matrix_dst is None or matrix_dst.shape != (b, 2, 3):
        raise RuntimeError("pck_transfer_points: a similarity-only STN needs matrix_dst (B, 2, 3)")
    c = lambda t: None if t is None else t.detach().float().contiguous()
    points, gt, visible, thresh, alphas, matrix_src, delta_src, identity, grid_dst, matrix_dst = map(
        c, (points, gt, visible, thresh, alphas, matrix_src, delta_src, identity, grid_dst, matrix_dst))
    dev = points.device
    lib = _lib.load()
    f = delta_src.size(1) if flow else 0
    counts = torch.zeros(alphas.numel(), dtype=torch.int64, device=dev)
    est = torch.empty(b, p, 2, dtype=torch.float32, device=dev)
    nn_index = torch.empty(b, p, dtype=torch.int64, device=dev) if flow else None
    ws = torch.empty(max(1, lib.gg_pck_transfer_workspace(b, p, f)), dtype=torch.uint8, device=dev)
    gh, gw = (grid_dst.size(1), grid_dst.size(2)) if flow else (0, 0)
    _lib.check(lib.gg_pck_transfer(counts.data_ptr(), est.data_ptr(), _lib.ptr(nn_index), ws.data_ptr(), points.data_ptr(),
                                   gt.data_ptr(), _lib.ptr(visible), thresh.data_ptr(), alphas.data_ptr(),
                                   matrix_src.data_ptr(), _lib.ptr(matrix_dst), _lib.ptr(delta_src), _lib.ptr(identity),
                                   _lib.ptr(grid_dst), b, p, alphas.numel(), int(size), f, gh, gw, _lib.stream()),
               "gg_pck_transfer")
    return counts, est, nn_index
