"""splat2d -- drop-in for reference utils/splat2d_cuda/functional.py:31-64 on sm_90a.

`splat2d(input, coordinates, values, sigma, soft_normalize=False)`: same argument checks (as RuntimeError /
AssertionError messages), CUDA + float32 only, forward only (the reference's backward raises too).
"""
import torch
import torch.autograd as ag

from .. import _lib

__all__ = ["splat2d", "splat2d_lookup", "nn_argmin", "track_points_lerp", "splat_composite_grid",
           "splat_lookup_composite_grid"]


class Splat2DFunction(ag.Function):
    @staticmethod
    def forward(ctx, input, coordinates, values, sigma, soft_normalize=False):
        assert coordinates.dtype == torch.float32 and values.dtype == torch.float32, \
            "Splat2D only takes float coordinates and values, got {} and {} instead.".format(coordinates.type(), values.type())
        assert coordinates.size(0) == values.size(0) and coordinates.size(1) == values.size(1), \
            "coordinates should be size (N, num_points, 2) and values should be size (N, num_points, *), got {} and {} instead.".format(
                coordinates.shape, values.shape)
        assert input.size(0) == coordinates.size(0) and input.dim() == 4, \
            "input should be of size (N, *, H, W), got {} instead".format(input.shape)
        assert sigma.size(0) == input.size(0), "sigma should be a tensor of size (N,)"
        if not coordinates.is_cuda:
            raise NotImplementedError("Splat2D currently only has support for GPU (cuda).")
        _lib.require_cuda(input, values, sigma)
        if input.dtype != torch.float32 or sigma.dtype != torch.float32:
            raise RuntimeError("splat2d: input and sigma must be float32")
        n, c, h, w = input.shape
        if values.dim() != 3 or values.size(2) != c or coordinates.size(2) != 2:
            raise RuntimeError("splat2d: values must be (N, P, %d) and coordinates (N, P, 2)" % c)
        input, coordinates, values, sigma = [t.contiguous() for t in (input, coordinates, values, sigma)]
        lib = _lib.load()
        out = torch.empty_like(input)
        ws = torch.empty(max(1, lib.gg_splat2d_workspace(n, c, h, w) // 4), dtype=torch.float32, device=input.device)
        rc = lib.gg_splat2d_forward(out.data_ptr(), ws.data_ptr(), input.data_ptr(), coordinates.data_ptr(),
                                    values.data_ptr(), sigma.data_ptr(), n, coordinates.size(1), c, h, w,
                                    1 if soft_normalize else 0, _lib.stream())
        _lib.check(rc, "gg_splat2d_forward")
        return out

    @staticmethod
    def backward(ctx, grad_output):
        raise NotImplementedError


splat2d = Splat2DFunction.apply


def splat2d_lookup(input, grid, query, values, sigma, res, out_res, soft_normalize=False):
    """`uncongeal_points`' lookup fused into the splat (csrc/splat.cu LOOKUP; SURVEY.md 8(f) rank 4):
        points = unnormalize(F.grid_sample(grid as image, query, 'border'), res, out_res)      spatial_transformer.py:141-157,621-623
        out    = splat2d(input, points, values, sigma, soft_normalize)                         functional.py:31-64
    in ONE scatter pass: the sampling grid is read where the points are loaded.  grid: (N, Hg, Wg, 2) sampling grid of the STN;
    query: (N, P, 2) normalised congealed-frame coordinates; values: (N, P, C <= 3).  -> (out, points (N, P, 2) pixels)."""
    _lib.require_cuda(input, grid, query, values, sigma)
    if input.dim() != 4 or grid.dim() != 4 or grid.size(-1) != 2 or query.dim() != 3 or query.size(-1) != 2:
        raise RuntimeError("splat2d_lookup: expected input (N, C, H, W), grid (N, Hg, Wg, 2), query (N, P, 2)")
    n, c, h, w = input.shape
    if grid.size(0) != n or query.size(0) != n or values.shape[:2] != query.shape[:2] or values.size(2) != c or sigma.size(0) != n:
        raise RuntimeError("splat2d_lookup: batch / point / channel counts disagree")
    if c > 3:
        raise RuntimeError("splat2d_lookup: C <= 3 (RGB colours or a 1-channel mask)")
    input, grid, query, values, sigma = [t.float().contiguous() for t in (input, grid, query, values, sigma)]
    lib = _lib.load()
    out = torch.empty_like(input)
    points = torch.empty_like(query)
    ws = torch.empty(max(1, lib.gg_splat2d_workspace(n, c, h, w) // 4), dtype=torch.float32, device=input.device)
    rc = lib.gg_splat2d_lookup_forward(out.data_ptr(), points.data_ptr(), ws.data_ptr(), input.data_ptr(), grid.data_ptr(),
                                       query.data_ptr(), values.data_ptr(), sigma.data_ptr(), n, query.size(1), c, h, w,
                                       grid.size(1), grid.size(2), (res - 1) / res, float(out_res - 1),
                                       1 if soft_normalize else 0, _lib.stream())
    _lib.check(rc, "gg_splat2d_lookup_forward")
    return out, points


def nn_argmin(grid, points):
    """index[n, p] = argmin_{hw} |points[n, p]|^2 + |grid[n, hw]|^2 - 2 grid[n, hw] . points[n, p]  (first minimum), the
    brute-force search of `congeal_points` (spatial_transformer.py:655-668) without the (N, H, W, P) distance tensor.
    grid: (N, H, W, 2) or (N, HW, 2); points: (N, P, 2).  -> (N, P) int64."""
    _lib.require_cuda(grid, points)
    n = grid.size(0)
    g = grid.reshape(n, -1, 2).float().contiguous()
    pts = points.float().contiguous()
    if pts.dim() != 3 or pts.size(0) != n or pts.size(2) != 2:
        raise RuntimeError("nn_argmin: points must be (N, P, 2)")
    lib = _lib.load()
    p = pts.size(1)
    index = torch.empty((n, p), dtype=torch.int64, device=g.device)
    ws = torch.empty(max(1, lib.gg_nn_argmin_workspace(n, p) // 8), dtype=torch.int64, device=g.device)
    _lib.check(lib.gg_nn_argmin(index.data_ptr(), ws.data_ptr(), g.data_ptr(), pts.data_ptr(), n, p, g.size(1), _lib.stream()),
               "gg_nn_argmin")
    return index


@torch.no_grad()
def track_points_lerp(base, target, alphas, points, centers, patch_size):
    """Dense point tracking of the congealing animation (reference vis_correspondence.py:59-114, looped over the frames of
    smoothly_sample_image :183-205) in one launch: frame t searches the patch_size^2 window around each point's centre of
    pad_grid(base.lerp(target, alphas[t])) for the entry nearest to the point and carries it to frame t + 1.
    base / target (N, H, H, 2); alphas (T,); points (N, P, 2) normalised; centers (N, P, 2) integer pixel centres before
    frame 0, each in [-1, H] (checked here with one host sync).  Inference only.
    -> (track (T, N, P, 2) int64, the last frame's centres (N, P, 2) int64)."""
    _lib.require_cuda(base, target, alphas, points, centers)
    if target.dim() != 4 or target.size(-1) != 2 or base.shape != target.shape:
        raise RuntimeError("track_points_lerp: base and target must both be (N, H, W, 2)")
    n, h, w = target.shape[:3]
    if points.dim() != 3 or points.size(0) != n or points.size(2) != 2 or centers.shape != points.shape:
        raise RuntimeError("track_points_lerp: points and centers must be (N, P, 2) with N = %d" % n)
    if alphas.dim() != 1:
        raise RuntimeError("track_points_lerp: alphas must be (T,)")
    if centers.is_floating_point():
        raise RuntimeError("track_points_lerp: centers must be integer pixel coordinates")
    c = centers.to(torch.int64).clone(memory_format=torch.contiguous_format)
    if c.numel() and bool(((c < -1) | (c[..., 0:1] > w) | (c[..., 1:2] > h)).any()):
        raise RuntimeError("track_points_lerp: patch centres must lie in [-1, W] x [-1, H] (the padded grid)")
    b, tg = base.float().contiguous(), target.float().contiguous()
    al, pts = alphas.float().contiguous(), points.float().contiguous()
    t = al.numel()
    track = torch.empty((t, n, points.size(1), 2), dtype=torch.int64, device=base.device)
    _lib.check(_lib.load().gg_track_points_lerp(track.data_ptr(), c.data_ptr(), b.data_ptr(), tg.data_ptr(), al.data_ptr(),
                                                pts.data_ptr(), t, n, points.size(1), h, w, int(patch_size), _lib.stream()),
               "gg_track_points_lerp")
    return track, c


@torch.no_grad()
def splat_composite_grid(images, points, colors, alpha_channel, sigma, opacity, nrow, max_workspace_bytes=1 << 29,
                         padding=2):
    """The label-propagation animation's frames (reference vis_correspondence.py:133-158): for every frame t,
    splat_points(images[t], points[t], sigma, opacity, colors, alpha_channel) (utils/vis_tools/helpers.py:134-194, alpha
    blending) then images2grid(nrow=nrow, normalize=True, range=(-1, 1)) (helpers.py:39-43), in one scatter and one
    composite launch per chunk of frames (csrc/splat.cu).
    images (T, N, 3, R, R) fp32; points (T, N, P, 2) pixel (x, y) or None (then the frames' images2grid); colors
    (N or 1, P, 3) and alpha_channel (N or 1, P, 1) or None, broadcast over the frames.  The frames are splatted in chunks
    whose accumulators fit max_workspace_bytes (T_chunk * N * R^2 * 16 bytes, 32 with an alpha channel).
    -> (T, Hg, Wg, 3) uint8 on the device, make_grid's layout (a single image without padding)."""
    _lib.require_cuda(images, points, colors, alpha_channel)
    if images.dim() != 5 or images.size(2) != 3 or images.size(3) != images.size(4):
        raise RuntimeError("splat_composite_grid: images must be (T, N, 3, R, R)")
    t, n, _, r, _ = images.shape
    p = 0
    if points is not None:
        if points.dim() != 4 or tuple(points.shape[:2]) != (t, n) or points.size(3) != 2:
            raise RuntimeError("splat_composite_grid: points must be (T, N, P, 2) with (T, N) = (%d, %d)" % (t, n))
        p = points.size(2)
        if colors is None:
            raise ValueError("splat_composite_grid: colors is required (plotly colour scales are not supported)")
    counts = []
    for name, v, c in (("colors", colors, 3), ("alpha_channel", alpha_channel, 1)):
        if v is not None and (v.dim() != 3 or v.size(0) not in (1, n) or v.size(1) != p or v.size(2) != c):
            raise RuntimeError("splat_composite_grid: %s must be (N or 1, P, %d) with N = %d, P = %d" % (name, c, n, p))
        counts.append(v.size(0) if v is not None else 1)
    images = images.float().contiguous()
    points, colors, alpha_channel = [None if (v is None or p == 0) else v.float().contiguous()
                                     for v in (points, colors, alpha_channel)]
    lib = _lib.load()
    xmaps = min(nrow, n)
    pad = 0 if n == 1 else padding
    hg, wg = -(-n // xmaps) * (r + pad) + pad, xmaps * (r + pad) + pad
    out = torch.empty((t, hg, wg, 3), dtype=torch.uint8, device=images.device)
    ws, ws_bytes = None, 0
    if p > 0 and t > 0:
        frame = lib.gg_splat_composite_grid_workspace(1, n, r, int(alpha_channel is not None))
        ws_bytes = frame * max(1, min(t, max_workspace_bytes // frame))
        ws = torch.empty(ws_bytes // 4, dtype=torch.float32, device=images.device)
    rc = lib.gg_splat_composite_grid(out.data_ptr(), _lib.ptr(ws), ws_bytes, images.data_ptr(), _lib.ptr(points),
                                     _lib.ptr(colors), _lib.ptr(alpha_channel), float(sigma), float(opacity), t, n, p, 3, r,
                                     int(nrow), int(padding), counts[0], counts[1], _lib.stream())
    _lib.check(rc, "gg_splat_composite_grid")
    return out


@torch.no_grad()
def splat_lookup_composite_grid(images, grid, query, flip, colors, alpha_channel, sigma, opacity, nrow, padding=2):
    """A dense label put on real images (reference applications/propagate_to_images.py:62-73) as one grid:
    uncongeal_points' lookup of `query` in every image's sampling grid (unnormalised to the images' R), the x mirror
    (R - 1) - x where the image was flipped, splat_points (alpha blending) and images2grid(nrow, padding, range=(-1, 1)),
    in one scatter and one composite launch (csrc/splat.cu).
    images (N, 3, R, R) fp32; grid (N, Hg, Wg, 2) the STN's sampling grids; query (1 or N, P, 2) normalised congealed
    coordinates; flip (N,) bool or None; colors (N or 1, P, 3) (required) and alpha_channel (N or 1, P, 1) or None.
    -> ((Hg, Wg, 3) uint8 grid, (N, P, 2) fp32 pixel coordinates on the unflipped images), both on the device."""
    _lib.require_cuda(images, grid, query, flip, colors, alpha_channel)
    if images.dim() != 4 or images.size(1) != 3 or images.size(2) != images.size(3):
        raise RuntimeError("splat_lookup_composite_grid: images must be (N, 3, R, R)")
    n, _, r, _ = images.shape
    if grid.dim() != 4 or grid.size(0) != n or grid.size(3) != 2:
        raise RuntimeError("splat_lookup_composite_grid: grid must be (N, Hg, Wg, 2) with N = %d" % n)
    if query.dim() != 3 or query.size(0) not in (1, n) or query.size(2) != 2:
        raise RuntimeError("splat_lookup_composite_grid: query must be (N or 1, P, 2) with N = %d" % n)
    p = query.size(1)
    if colors is None:
        raise ValueError("splat_lookup_composite_grid: colors is required (plotly colour scales are not supported)")
    counts = []
    for name, v, c in (("colors", colors, 3), ("alpha_channel", alpha_channel, 1)):
        if v is not None and (v.dim() != 3 or v.size(0) not in (1, n) or v.size(1) != p or v.size(2) != c):
            raise RuntimeError("splat_lookup_composite_grid: %s must be (N or 1, P, %d) with N = %d, P = %d" % (name, c, n, p))
        counts.append(v.size(0) if v is not None else 1)
    if flip is not None and flip.numel() != n:
        raise RuntimeError("splat_lookup_composite_grid: flip must hold N = %d values" % n)
    images, grid, query, colors = [v.float().contiguous() for v in (images, grid, query, colors)]
    alpha_channel = None if alpha_channel is None else alpha_channel.float().contiguous()
    flip = None if flip is None else flip.reshape(n).to(torch.uint8).contiguous()
    lib = _lib.load()
    xmaps = min(nrow, n)
    pad = 0 if n == 1 else padding
    hg, wg = -(-n // xmaps) * (r + pad) + pad, xmaps * (r + pad) + pad
    out = torch.empty((hg, wg, 3), dtype=torch.uint8, device=images.device)
    points = torch.empty((n, p, 2), dtype=torch.float32, device=images.device)
    ws_bytes = lib.gg_splat_composite_grid_workspace(1, n, r, int(alpha_channel is not None))
    ws = torch.empty(max(1, ws_bytes // 4), dtype=torch.float32, device=images.device)
    rc = lib.gg_splat_lookup_composite_grid(out.data_ptr(), points.data_ptr(), ws.data_ptr(), ws_bytes, images.data_ptr(),
                                            grid.data_ptr(), query.data_ptr(), _lib.ptr(flip), colors.data_ptr(),
                                            _lib.ptr(alpha_channel), float(sigma), float(opacity), n, p, query.size(0), 3, r,
                                            grid.size(1), grid.size(2), int(nrow), int(padding), counts[0], counts[1],
                                            _lib.stream())
    _lib.check(rc, "gg_splat_lookup_composite_grid")
    return out, points
