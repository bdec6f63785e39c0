"""Laplacian pyramid blending on sm_90a -- drop-in for reference utils/laplacian_blending.py:13-107 (`LaplacianBlender`)
and the blend branches of splat_points (utils/vis_tools/helpers.py:134-194).

`laplacian_blend(img0, img1, mask, levels, kernel_size, sigma, level_size_adder=0, level_sigma_multiplier=2)` runs
csrc/blend.cu (one fused launch per level, separable blur, all three gradients).  CUDA fp32 only; no fallback.
"""
import math

import torch
import torch.autograd as ag
import torch.nn as nn

from .. import _lib
from .functional import splat2d

__all__ = ["laplacian_blend", "LaplacianBlender", "splat_points", "BLEND_PRESETS"]

MAX_WIDTH = 63   # taps per level accepted by csrc/blend.cu

# splat_points' presets (helpers.py:188-193), as LaplacianBlender keyword arguments
BLEND_PRESETS = {
    "laplacian": dict(levels=5, gaussian_kernel_size=45, gaussian_sigma=1),
    "laplacian_light": dict(levels=3, gaussian_kernel_size=11, gaussian_sigma=0.5),
}

_taps_cache = {}


def _gaussian_taps(width, sigma):
    """cv2.getGaussianKernel(width, sigma), sigma > 0: exp(-(i - (width-1)/2)^2 / (2 sigma^2)) normalised, in float64."""
    c = (width - 1) * 0.5
    g = [math.exp(-0.5 / (sigma * sigma) * (i - c) ** 2) for i in range(width)]
    s = math.fsum(g)
    return [v / s for v in g]


def _check_config(levels, kernel_size, sigma, level_size_adder, level_sigma_multiplier):
    assert kernel_size % 2 == 1, "gaussian_kernel_size needs to be odd for easier padding"
    assert level_size_adder % 2 == 0, "level_size_adder needs to be even for easier padding"
    if levels < 1:
        raise RuntimeError("laplacian_blend: levels must be >= 1 (got %d)" % levels)
    if levels > 1:
        width = kernel_size + level_size_adder
        if width < 1 or width > MAX_WIDTH:
            raise RuntimeError("laplacian_blend: level width %d is outside 1..%d" % (width, MAX_WIDTH))
        if sigma <= 0 or level_sigma_multiplier <= 0:
            raise RuntimeError("laplacian_blend: sigma and level_sigma_multiplier must be positive")


def level_taps(levels, kernel_size, sigma, level_size_adder=0, level_sigma_multiplier=2, device=None):
    """(levels - 1, width) fp32 taps on `device`, computed in float64 once per configuration and device (a cached device
    tensor: no host-to-device copy once warm, so a blend inside a CUDA-graph capture reuses it)."""
    key = (int(levels), int(kernel_size), float(sigma), int(level_size_adder), float(level_sigma_multiplier), str(device))
    t = _taps_cache.get(key)
    if t is None:
        width = kernel_size + level_size_adder
        rows = [_gaussian_taps(width, sigma * level_sigma_multiplier ** level) for level in range(levels - 1)]
        t = torch.tensor(rows, dtype=torch.float64).reshape(max(levels - 1, 0), width).float().to(device)
        _taps_cache[key] = t
    return t


def _check_tensors(img0, img1, mask):
    _lib.require_cuda(img0, img1, mask)
    for t in (img0, img1, mask):
        if t.dtype != torch.float32:
            raise RuntimeError("laplacian_blend: float32 tensors only (got %s)" % t.dtype)
    if img0.dim() != 4 or img1.shape != img0.shape or mask.dim() != 4:
        raise RuntimeError("laplacian_blend: img0 and img1 must be (N, C, H, W) of the same shape, mask (N, 1, H, W); got "
                           "%s, %s, %s" % (tuple(img0.shape), tuple(img1.shape), tuple(mask.shape)))
    if mask.size(1) != 1:
        raise RuntimeError("laplacian_blend: mask input should have num_channels==1, but got num_channels==%d" % mask.size(1))
    if mask.size(0) != img0.size(0) or mask.shape[2:] != img0.shape[2:]:
        raise RuntimeError("laplacian_blend: mask %s does not match the images %s" % (tuple(mask.shape), tuple(img0.shape)))
    if img0.numel() == 0:
        raise RuntimeError("laplacian_blend: empty tensors")


class LaplacianBlendFunction(ag.Function):
    @staticmethod
    def forward(ctx, img0, img1, mask, taps, levels, width):
        img0, img1, mask = img0.contiguous(), img1.contiguous(), mask.contiguous()
        n, c, h, w = img0.shape
        lib = _lib.load()
        out = torch.empty_like(img0)
        nbytes = lib.gg_laplacian_blend_workspace(n, c, h, w, levels, 0)
        ws = torch.empty(max(1, nbytes // 4), dtype=torch.float32, device=img0.device)
        _lib.check(lib.gg_laplacian_blend_forward(out.data_ptr(), ws.data_ptr(), img0.data_ptr(), img1.data_ptr(),
                                                  mask.data_ptr(), taps.data_ptr() if levels > 1 else None, n, c, h, w,
                                                  levels, width, _lib.stream()), "gg_laplacian_blend_forward")
        ctx.save_for_backward(img0, img1, mask, taps)
        ctx.levels, ctx.width = levels, width
        return out

    @staticmethod
    def backward(ctx, grad_out):
        img0, img1, mask, taps = ctx.saved_tensors
        g = grad_out.contiguous()
        _lib.require_cuda(g)
        if g.dtype != torch.float32:
            g = g.float()
        n, c, h, w = img0.shape
        lib = _lib.load()
        g0, g1, gm = torch.empty_like(img0), torch.empty_like(img1), torch.empty_like(mask)
        nbytes = lib.gg_laplacian_blend_workspace(n, c, h, w, ctx.levels, 1)
        ws = torch.empty(max(1, nbytes // 4), dtype=torch.float32, device=img0.device)
        _lib.check(lib.gg_laplacian_blend_backward(g0.data_ptr(), g1.data_ptr(), gm.data_ptr(), ws.data_ptr(), g.data_ptr(),
                                                   img0.data_ptr(), img1.data_ptr(), mask.data_ptr(),
                                                   taps.data_ptr() if ctx.levels > 1 else None, n, c, h, w, ctx.levels,
                                                   ctx.width, _lib.stream()), "gg_laplacian_blend_backward")
        need = ctx.needs_input_grad
        return (g0 if need[0] else None, g1 if need[1] else None, gm if need[2] else None, None, None, None)


def laplacian_blend(img0, img1, mask, levels, kernel_size, sigma, level_size_adder=0, level_sigma_multiplier=2):
    """LaplacianBlender(levels, kernel_size, sigma, level_size_adder, level_sigma_multiplier)(img0, img1, mask): img0 / img1
    (N, C, H, W), mask (N, 1, H, W), all CUDA float32.  Differentiable in all three inputs."""
    _check_config(levels, kernel_size, sigma, level_size_adder, level_sigma_multiplier)
    _check_tensors(img0, img1, mask)
    taps = level_taps(levels, kernel_size, sigma, level_size_adder, level_sigma_multiplier, img0.device)
    return LaplacianBlendFunction.apply(img0, img1, mask, taps, int(levels), int(kernel_size + level_size_adder))


class LaplacianBlender(nn.Module):
    """Drop-in for the reference's LaplacianBlender: same constructor and forward(img0, img1, mask).  The taps are
    computed without cv2 (float64 1-D Gaussians) and cached per device instead of registered as 2-D buffers."""

    def __init__(self, levels=5, gaussian_kernel_size=45, gaussian_sigma=1, level_size_adder=0, level_sigma_multiplier=2):
        super().__init__()
        _check_config(levels, gaussian_kernel_size, gaussian_sigma, level_size_adder, level_sigma_multiplier)
        self.levels = levels
        self.gaussian_kernel_size = gaussian_kernel_size
        self.gaussian_sigma = gaussian_sigma
        self.level_size_adder = level_size_adder
        self.level_sigma_multiplier = level_sigma_multiplier
        self.kernel_padding = [(gaussian_kernel_size + level_size_adder) // 2] * levels

    def forward(self, img0, img1, mask):
        return laplacian_blend(img0, img1, mask, self.levels, self.gaussian_kernel_size, self.gaussian_sigma,
                               self.level_size_adder, self.level_sigma_multiplier)


def blend(images, prop_obj, prop_mask, blend_alg):
    """splat_points' compositing step (helpers.py:186-193)."""
    if blend_alg == "alpha":
        return prop_mask * prop_obj + (1 - prop_mask) * images
    if blend_alg not in BLEND_PRESETS:
        raise ValueError("blend_alg must be 'alpha', 'laplacian' or 'laplacian_light' (got %r)" % (blend_alg,))
    kw = BLEND_PRESETS[blend_alg]
    return laplacian_blend(images, prop_obj, prop_mask, kw["levels"], kw["gaussian_kernel_size"], kw["gaussian_sigma"])


@torch.inference_mode()
def splat_points(images, points, sigma, opacity, colors, alpha_channel=None, blend_alg="alpha"):
    """Reference utils/vis_tools/helpers.py:134-194 with explicit colours: splat `colors` (N, P, 3) (or (N, K*P, 3)) at
    `points` (N, P, 2) or (N, K, P, 2) (pixels) onto `images` (N, C, H, W) and composite with `blend_alg`.
    `sigma`: float or (N,) tensor; `alpha_channel`: optional (N, P, 1) opacities.  Plotly colour scales are not
    supported: `colors` is required."""
    if colors is None:
        raise ValueError("splat_points: colors is required (plotly colour scales are not supported)")
    assert images.dim() == 4
    assert points.dim() == 3 or points.dim() == 4
    n = images.size(0)
    if points.dim() == 4:
        points = points.reshape(points.size(0), points.size(1) * points.size(2), 2)
    if alpha_channel is None:
        alpha_channel = torch.ones(n, points.size(1), 1, device=images.device)
    if isinstance(sigma, (float, int)):
        sigma = torch.full((n,), float(sigma), device=images.device)
    blank_img = torch.zeros(n, images.size(1), images.size(2), images.size(3), device=images.device)
    blank_mask = torch.zeros(n, 1, images.size(2), images.size(3), device=images.device)
    prop_obj = splat2d(blank_img, points, colors, sigma, False)
    prop_mask = splat2d(blank_mask, points, alpha_channel, sigma, True) * opacity
    return blend(images, prop_obj, prop_mask, blend_alg)
