"""uint8 grids and per-cluster sums of the training visuals (csrc/trainvis.cu): the colour-wheel flow grid, the grid of
images normalised by per-image ranges, and the routing of congealed images to clusters.  Grids are (Hg, Wg, 3) uint8 on
the device in torchvision make_grid's layout (a single image without padding)."""
import torch

from .. import _lib

__all__ = ["flow_image_grid", "image_grid", "cluster_accumulate", "grid_shape"]


def grid_shape(n, h, w, nrow, padding=2):
    """make_grid's (Hg, Wg) for n images of h x w."""
    xmaps = min(nrow, n)
    pad = 0 if n == 1 else padding
    return -(-n // xmaps) * (h + pad) + pad, xmaps * (w + pad) + pad


@torch.no_grad()
def flow_image_grid(flow, nrow, padding=2):
    """flow_to_image (reference utils/vis_tools/flow_vis.py:106-130) of flow (N, H, W, 2), the radius normalised by the
    batch's largest, laid out as make_grid(range=(0, 1)) + images2grid would lay out its result: floor(255 * colour)."""
    _lib.require_cuda(flow)
    if flow.dim() != 4 or flow.size(3) != 2 or flow.size(0) < 1:
        raise RuntimeError("flow_image_grid: flow must be (N, H, W, 2) with N >= 1")
    f = _lib.dense_f32(flow)
    n, h, w = f.shape[:3]
    hg, wg = grid_shape(n, h, w, nrow, padding)
    out = torch.empty((hg, wg, 3), dtype=torch.uint8, device=f.device)
    ws = torch.empty(2, dtype=torch.float32, device=f.device)
    _lib.check(_lib.load().gg_flow_image_grid(out.data_ptr(), ws.data_ptr(), f.data_ptr(), n, h, w, int(nrow), int(padding),
                                              _lib.stream()), "gg_flow_image_grid")
    return out


@torch.no_grad()
def image_grid(images, ranges, nrow, padding=2):
    """make_grid(normalize=True) with range ranges[i] = (lo, hi) for image i, then images2grid (reference
    utils/vis_tools/helpers.py:39-43).  images (N, 3, H, W); ranges (N, 2) fp32."""
    _lib.require_cuda(images, ranges)
    if images.dim() != 4 or images.size(1) != 3 or images.size(0) < 1:
        raise RuntimeError("image_grid: images must be (N, 3, H, W) with N >= 1")
    n, _, h, w = images.shape
    if tuple(ranges.shape) != (n, 2):
        raise RuntimeError("image_grid: ranges must be (N, 2) with N = %d" % n)
    x = images.float().contiguous()
    r = _lib.dense_f32(ranges)
    hg, wg = grid_shape(n, h, w, nrow, padding)
    out = torch.empty((hg, wg, 3), dtype=torch.uint8, device=x.device)
    _lib.check(_lib.load().gg_image_grid(out.data_ptr(), x.data_ptr(), r.data_ptr(), n, h, w, int(nrow), int(padding),
                                         _lib.stream()), "gg_image_grid")
    return out


@torch.no_grad()
def cluster_accumulate(sums, counts, keep, images, sel):
    """Route image n's slot sel[n] to cluster sel[n] % K, in place: sums[k] += it, counts[k] += 1, and it is copied to
    keep[k, counts[k]] while that is below n_keep.  images (F, N, K, C, H, W), any strides (slot s = flip s // K, head
    s % K: assign_fake_images_to_clusters' output as a view, or a batch expanded with zero strides); sel (N,) int64 in
    [0, F * K) (checked here, one host sync); sums (K, C, H, W) fp32, counts (K,) int64, keep (K, n_keep, C, H, W) fp32 or
    None.  Each sum adds its images in order: bitwise the sequential fp32 sum, across calls."""
    _lib.require_cuda(sums, counts, keep, images, sel)
    if images.dim() != 6:
        raise RuntimeError("cluster_accumulate: images must be (F, N, K, C, H, W)")
    f, n, k, c, h, w = images.shape
    if images.dtype != torch.float32 or sel.dtype != torch.int64 or tuple(sel.shape) != (n,):
        raise RuntimeError("cluster_accumulate: images fp32 and sel (N,) int64 with N = %d" % n)
    if sums.dtype != torch.float32 or not sums.is_contiguous() or tuple(sums.shape) != (k, c, h, w):
        raise RuntimeError("cluster_accumulate: sums must be contiguous fp32 (%d, %d, %d, %d)" % (k, c, h, w))
    if counts.dtype != torch.int64 or not counts.is_contiguous() or tuple(counts.shape) != (k,):
        raise RuntimeError("cluster_accumulate: counts must be contiguous int64 (%d,)" % k)
    n_keep = 0
    if keep is not None:
        if keep.dtype != torch.float32 or not keep.is_contiguous() or keep.dim() != 5 or keep.size(0) != k or \
                tuple(keep.shape[2:]) != (c, h, w):
            raise RuntimeError("cluster_accumulate: keep must be contiguous fp32 (%d, n_keep, %d, %d, %d)" % (k, c, h, w))
        n_keep = keep.size(1)
    sel = sel.contiguous()
    if n and bool(((sel < 0) | (sel >= f * k)).any()):
        raise RuntimeError("cluster_accumulate: selections must lie in [0, %d)" % (f * k))
    st = images.stride()
    _lib.check(_lib.load().gg_cluster_accumulate(sums.data_ptr(), counts.data_ptr(), _lib.ptr(keep), images.data_ptr(),
                                                 sel.data_ptr(), n, f * k, k, c, h, w, st[1], st[0], st[2], st[3], st[4],
                                                 st[5], n_keep, _lib.stream()), "gg_cluster_accumulate")
