"""Perceptual-loss front end in one pass (csrc/lpips.cu): unit-normalise two feature maps over channels, squared
difference, optional per-channel weights, spatial mean.

reference: models/losses/lpips.py:26-28 (`normalize_tensor`), :193-205 (difference, `lins` / channel sum), :226
(`spatial_average`).  `feature_distance(f0, f1, weight=None)` returns (N, 1, 1, 1) like the reference's per-layer `res`.
CUDA tensors only (like every op here: no CPU path in the product).  The fused kernels want channels-last fp32 or bf16 feature
maps (forward: one read of both maps; backward: one read + one write of both): other layouts / float dtypes are
converted to that form first (one copy), anything the kernel cannot take (trainable `lins` weights, odd channel counts)
raises -- there is no eager tensor-op route."""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import _lib


def _channels_ok(c):
    c4 = c // 4
    return c % 4 == 0 and c <= 1024 and ((c4 < 32 and c4 & (c4 - 1) == 0) or (c4 >= 32 and c4 % 32 == 0))


def _as_kernel_input(f):
    """channels-last fp32 / bf16 view or copy of a (N, C, H, W) feature map (autograd-tracked conversion when needed)."""
    if f.dtype not in (torch.float32, torch.bfloat16):
        f = f.float()
    if f.shape[1] > 1 and f.shape[2] * f.shape[3] > 1:
        f = f.contiguous(memory_format=torch.channels_last)
    else:   # degenerate shapes are both layouts at once: any dense buffer is (N, HW, C)
        f = f.contiguous()
    return f


class _FeatureDistance(Function):
    @staticmethod
    def forward(ctx, f0, f1, weight, eps):
        _lib.require_cuda(f0, f1, weight)
        n, c, h, w = f0.shape
        lib = _lib.load()
        wt = _lib.dense_f32(weight.detach().reshape(-1)) if weight is not None else None
        out = torch.empty(n, dtype=torch.float32, device=f0.device)
        ws = torch.empty(max(1, lib.gg_feature_distance_workspace(n, c, h * w) // 4), dtype=torch.float32, device=f0.device)
        rc = lib.gg_feature_distance_forward(out.data_ptr(), ws.data_ptr(), f0.data_ptr(), f1.data_ptr(), _lib.ptr(wt),
                                             _lib.dtype_code(f0), n, c, h * w, eps, _lib.stream())
        _lib.check(rc, "gg_feature_distance_forward")
        ctx.save_for_backward(f0, f1, wt)
        ctx.eps = eps
        return out.reshape(n, 1, 1, 1)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        f0, f1, wt = ctx.saved_tensors
        need0, need1 = ctx.needs_input_grad[:2]
        n, c, h, w = f0.shape
        g = g.reshape(n).float().contiguous()
        g0 = torch.empty_like(f0) if need0 else None
        g1 = torch.empty_like(f1) if need1 else None
        if need0 or need1:
            rc = _lib.load().gg_feature_distance_backward(_lib.ptr(g0), _lib.ptr(g1), g.data_ptr(), f0.data_ptr(),
                                                          f1.data_ptr(), _lib.ptr(wt), _lib.dtype_code(f0), n, c, h * w, ctx.eps,
                                                          _lib.stream())
            _lib.check(rc, "gg_feature_distance_backward")
        return g0, g1, None, None


def feature_distance(f0, f1, weight=None, eps=1e-10):
    """mean_hw sum_c w_c (f0/|f0| - f1/|f1|)^2 -> (N, 1, 1, 1).  `weight`: (C,) non-trainable `lins` weights or None."""
    _lib.require_cuda(f0, f1, weight)
    if f0.dim() != 4 or f0.shape != f1.shape:
        raise RuntimeError("feature_distance: expected two (N, C, H, W) maps of one shape, got %s and %s" %
                           (tuple(f0.shape), tuple(f1.shape)))
    if not _channels_ok(f0.shape[1]):
        raise RuntimeError("feature_distance: C=%d is not supported by the fused kernel (C %% 4 == 0, C <= 1024, C/4 a power "
                           "of two below 32 or a multiple of 32)" % f0.shape[1])
    if weight is not None and weight.requires_grad:
        raise RuntimeError("feature_distance: trainable `lins` weights are not supported (the reference trains with "
                           "frozen LPIPS weights, lpips.py:13-22)")
    a, b = _as_kernel_input(f0), _as_kernel_input(f1)
    if a.dtype != b.dtype:
        a, b = a.float(), b.float()
    return _FeatureDistance.apply(a, b, weight, float(eps))


class _FeatureDistanceStacked(Function):
    """feature_distance(f[:N], f[N:]) on ONE stacked (2N, C, H, W) channels-last map: the two halves are the two images'
    features of a single backbone pass; the gradient is written straight into the halves of one (2N, ...) tensor (slicing the
    halves out with autograd would zero-fill and copy each half's gradient into a full-size tensor again)."""

    @staticmethod
    def forward(ctx, f, weight, eps):
        _lib.require_cuda(f, weight)
        n2, c, h, w = f.shape
        n = n2 // 2
        lib = _lib.load()
        wt = _lib.dense_f32(weight.detach().reshape(-1)) if weight is not None else None
        out = torch.empty(n, dtype=torch.float32, device=f.device)
        ws = torch.empty(max(1, lib.gg_feature_distance_workspace(n, c, h * w) // 4), dtype=torch.float32, device=f.device)
        half = n * c * h * w * f.element_size()
        rc = lib.gg_feature_distance_forward(out.data_ptr(), ws.data_ptr(), f.data_ptr(), f.data_ptr() + half, _lib.ptr(wt),
                                             _lib.dtype_code(f), n, c, h * w, eps, _lib.stream())
        _lib.check(rc, "gg_feature_distance_forward")
        ctx.save_for_backward(f, wt)
        ctx.eps = eps
        return out.reshape(n, 1, 1, 1)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        f, wt = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None, None
        n2, c, h, w = f.shape
        n = n2 // 2
        g = g.reshape(n).float().contiguous()
        gf = torch.empty_like(f)
        half = n * c * h * w * f.element_size()
        rc = _lib.load().gg_feature_distance_backward(gf.data_ptr(), gf.data_ptr() + half, g.data_ptr(), f.data_ptr(),
                                                      f.data_ptr() + half, _lib.ptr(wt), _lib.dtype_code(f), n, c, h * w, ctx.eps,
                                                      _lib.stream())
        _lib.check(rc, "gg_feature_distance_backward")
        return gf, None, None


def feature_distance_stacked(f, weight=None, eps=1e-10):
    """feature_distance(f[:N], f[N:], weight) for a stacked (2N, C, H, W) map -> (N, 1, 1, 1)."""
    _lib.require_cuda(f, weight)
    if f.dim() != 4 or f.shape[0] % 2 != 0:
        raise RuntimeError("feature_distance_stacked: expected a (2N, C, H, W) map, got %s" % (tuple(f.shape),))
    if not _channels_ok(f.shape[1]):
        raise RuntimeError("feature_distance_stacked: C=%d is not supported by the fused kernel" % f.shape[1])
    if weight is not None and weight.requires_grad:
        raise RuntimeError("feature_distance_stacked: trainable `lins` weights are not supported")
    return _FeatureDistanceStacked.apply(_as_kernel_input(f), weight, float(eps))

