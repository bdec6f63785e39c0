"""upfirdn2d -- drop-in for reference models/stylegan2/op/upfirdn2d.py:145-156 on sm_90a.

`upfirdn2d(input, kernel, up=1, down=1, pad=(0, 0))` keeps the reference signature (the 2-tuple pad
is applied to both axes).  Forward and both backward orders call gg_upfirdn2d (include/gg_b200.h):
the gradient of an upfirdn2d is an upfirdn2d with the flipped filter, up<->down swapped and the
`g_pad` padding of upfirdn2d.py:111-116, so one kernel family serves all three.
"""
import torch
from torch.autograd import Function

from .. import _lib
from . import nhwc


def _out_size(in_h, in_w, kh, kw, up, down, pad):
    up_x, up_y = up
    down_x, down_y = down
    px0, px1, py0, py1 = pad
    out_h = (in_h * up_y + py0 + py1 - kh) // down_y + 1
    out_w = (in_w * up_x + px0 + px1 - kw) // down_x + 1
    return out_h, out_w


def _taps(kernel):
    """The C ABI takes fp32 taps in device memory, un-flipped."""
    if kernel.dtype != torch.float32 or not kernel.is_contiguous():
        kernel = kernel.float().contiguous()
    return kernel


def upfirdn2d_raw(x, kernel, up, down, pad):
    """(N, C, H, W) -> (N, C, H', W'); no autograd.  up/down are (x, y) pairs, pad = (x0, x1, y0, y1)."""
    _lib.require_cuda(x, kernel)
    if x.dim() != 4:
        raise RuntimeError("upfirdn2d expects a 4-D (N, C, H, W) input, got %s" % (tuple(x.shape),))
    taps = _taps(kernel)
    kh, kw = taps.shape
    n, c, in_h, in_w = x.shape
    out_h, out_w = _out_size(in_h, in_w, kh, kw, up, down, pad)
    if out_h < 1 or out_w < 1:
        raise RuntimeError("upfirdn2d: empty output (%d x %d)" % (out_h, out_w))
    if nhwc.blur_ok(x, kh, kw, up, down):
        # channels-last activations stay channels-last (TMA tensor-map kernel, csrc/nhwc.cu; fp32 or bf16 storage)
        return nhwc.blur(x, kernel, pad, mode=0)[0]
    x = x.contiguous()
    out = torch.empty((n, c, out_h, out_w), dtype=x.dtype, device=x.device)
    rc = _lib.load().gg_upfirdn2d(out.data_ptr(), x.data_ptr(), taps.data_ptr(), _lib.dtype_code(x), n * c,
                                  in_h, in_w, kh, kw, up[0], up[1], down[0], down[1], pad[0], pad[1], pad[2],
                                  pad[3], _lib.stream())
    _lib.check(rc, "gg_upfirdn2d")
    return out


def grad_pad(in_h, in_w, out_h, out_w, kh, kw, up, down, pad):
    """Padding of the adjoint resampling (reference upfirdn2d.py:111-116)."""
    up_x, up_y = up
    down_x, down_y = down
    px0, _, py0, _ = pad
    g_px0 = kw - px0 - 1
    g_py0 = kh - py0 - 1
    g_px1 = in_w * up_x - out_w * down_x + px0 - up_x + 1
    g_py1 = in_h * up_y - out_h * down_y + py0 - up_y + 1
    return (g_px0, g_px1, g_py0, g_py1)


class _UpFirDn2dGrad(Function):
    """grad_input = upfirdn2d(grad_output, flip(kernel), up<->down, g_pad); differentiable again."""

    @staticmethod
    def forward(ctx, grad_output, kernel, up, down, pad, g_pad, in_size):
        flipped = _lib.flipped_filter(kernel)
        grad_input = upfirdn2d_raw(grad_output, flipped, down, up, g_pad)
        if tuple(grad_input.shape[2:]) != tuple(in_size[2:]):
            raise RuntimeError("upfirdn2d backward: adjoint produced %s, expected %s" %
                               (tuple(grad_input.shape), tuple(in_size)))
        ctx.save_for_backward(kernel)
        ctx.cfg = (up, down, pad)
        return grad_input

    @staticmethod
    def backward(ctx, gradgrad_input):
        (kernel,) = ctx.saved_tensors
        up, down, pad = ctx.cfg
        return UpFirDn2d.apply(gradgrad_input, kernel, up, down, pad), None, None, None, None, None, None


class UpFirDn2d(Function):
    @staticmethod
    def forward(ctx, input, kernel, up, down, pad):
        out = upfirdn2d_raw(input, kernel, up, down, pad)
        ctx.save_for_backward(kernel)
        kh, kw = kernel.shape
        ctx.cfg = (up, down, pad, grad_pad(input.shape[2], input.shape[3], out.shape[2], out.shape[3], kh, kw,
                                            up, down, pad), tuple(input.shape))
        return out

    @staticmethod
    def backward(ctx, grad_output):
        (kernel,) = ctx.saved_tensors
        up, down, pad, g_pad, in_size = ctx.cfg
        return _UpFirDn2dGrad.apply(grad_output, kernel, up, down, pad, g_pad, in_size), None, None, None, None


def upfirdn2d(input, kernel, up=1, down=1, pad=(0, 0)):
    """FIR resample `input` (N, C, H, W) with the 2-D `kernel`: zero-insert x`up`, pad, filter, keep every
    `down`-th sample.  Same call signature as the reference; CUDA tensors only."""
    return UpFirDn2d.apply(input, kernel, (up, up), (down, down), (pad[0], pad[1], pad[0], pad[1]))
