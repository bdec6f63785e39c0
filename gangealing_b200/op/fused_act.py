"""fused_leaky_relu / FusedLeakyReLU -- drop-in for reference models/stylegan2/op/fused_act.py.

forward : gg_fused_bias_act(act=3, grad=0)            (fused_act.py:52-58)
backward: gg_bias_act_backward -- the act=3/grad=1 kernel call AND the grad_input.sum(dims) bias
          reduction of fused_act.py:29-38 in one pass over the gradient
2nd ord.: gg_fused_bias_act(gradgrad_input, gradgrad_bias, out, act=3, grad=1)  (fused_act.py:42-49)
"""
import torch
from torch import nn
from torch.autograd import Function

from .. import _lib
from . import nhwc


def fused_bias_act_raw(x, bias, ref, act, grad, alpha, scale):
    """Python face of the reference's native `fused.fused_bias_act(input, bias, refer, act, grad, alpha,
    scale)` (fused_bias_act.cpp:11-17); `None`/empty tensors mean "no bias"/"no ref"."""
    _lib.require_cuda(x, bias, ref)
    cl = _lib.is_nhwc(x) and (ref is None or (ref.shape == x.shape and ref.stride() == x.stride()))
    if not cl:
        x = x.contiguous()
    if bias is not None and bias.numel() == 0:
        bias = None
    if ref is not None and ref.numel() == 0:
        ref = None
    if bias is not None:
        bias = bias.to(x.dtype).contiguous()
    if ref is not None:
        if ref.shape != x.shape or ref.dtype != x.dtype:
            raise RuntimeError("fused_bias_act: ref must match the input's shape and dtype")
        if not cl:
            ref = ref.contiguous()
    step_b = 1
    if not cl:  # channels-last memory is (N*H*W, C): the bias index is simply i % C
        for s in x.shape[2:]:
            step_b *= s
    out = torch.empty_like(x)
    rc = _lib.load().gg_fused_bias_act(out.data_ptr(), x.data_ptr(), _lib.ptr(bias), _lib.ptr(ref),
                                       _lib.dtype_code(x), act, grad, alpha, scale, x.numel(), step_b,
                                       0 if bias is None else bias.numel(), _lib.stream())
    _lib.check(rc, "gg_fused_bias_act")
    return out


def bias_act_backward_raw(grad_output, out, alpha, scale, want_bias_grad):
    """gx = (out > 0 ? g : alpha*g)*scale and, optionally, grad_bias = gx.sum(all dims but 1) (fp32)."""
    _lib.require_cuda(grad_output, out)
    if nhwc.rowwise_ok(out) and grad_output.shape == out.shape:
        g = grad_output.contiguous(memory_format=torch.channels_last)
        if g.dtype != out.dtype:
            g = g.to(out.dtype)
        return nhwc.bias_act_backward(g, out, alpha, scale, want_bias_grad)
    g = grad_output.contiguous()
    out = out.contiguous()
    if g.shape != out.shape or g.dtype != out.dtype:
        raise RuntimeError("bias_act_backward: grad_output/out mismatch")
    n = g.shape[0] if g.dim() > 0 else 1
    c = g.shape[1] if g.dim() > 1 else 1
    hw = 1
    for s in g.shape[2:]:
        hw *= s
    gx = torch.empty_like(g)
    lib = _lib.load()
    grad_bias = ws = None
    if want_bias_grad:
        grad_bias = torch.empty(c, dtype=torch.float32, device=g.device)
        ws = torch.empty(max(1, lib.gg_bias_act_backward_workspace(n, c, hw) // 4), dtype=torch.float32,
                         device=g.device)
    rc = lib.gg_bias_act_backward(gx.data_ptr(), _lib.ptr(grad_bias), _lib.ptr(ws), g.data_ptr(), out.data_ptr(),
                                  _lib.dtype_code(g), alpha, scale, n, c, hw, _lib.stream())
    _lib.check(rc, "gg_bias_act_backward")
    return gx, grad_bias


class _FusedLeakyReLUGrad(Function):
    @staticmethod
    def forward(ctx, grad_output, out, negative_slope, scale, want_bias_grad, bias_dtype=None):
        gx, grad_bias = bias_act_backward_raw(grad_output, out, negative_slope, scale, want_bias_grad)
        ctx.save_for_backward(out)
        ctx.cfg = (negative_slope, scale)
        if grad_bias is None:
            grad_bias = gx.new_zeros(())  # placeholder, never used
        else:   # the reduction is fp32; it is handed back in the bias' own dtype (fp32 master parameters under bf16 activations)
            grad_bias = grad_bias.to(bias_dtype if bias_dtype is not None else gx.dtype)
        return gx, grad_bias

    @staticmethod
    def backward(ctx, gradgrad_input, gradgrad_bias):
        (out,) = ctx.saved_tensors
        negative_slope, scale = ctx.cfg
        bias = gradgrad_bias if (gradgrad_bias is not None and gradgrad_bias.dim() == 1) else None
        gradgrad_out = fused_bias_act_raw(gradgrad_input, bias, out, 3, 1, negative_slope, scale)
        return gradgrad_out, None, None, None, None, None


class FusedLeakyReLUFunction(Function):
    @staticmethod
    def forward(ctx, input, bias, negative_slope, scale):
        _lib.require_cuda(input, bias)
        if nhwc.elementwise_ok(input) and (bias is None or bias.numel() in (0, input.shape[1])):
            # channels-last: the 16-byte-vector streaming kernel of csrc/nhwc.cu (the flat kernel's per-element `i % C`
            # bias indexing is slower)
            b = bias if (bias is not None and bias.numel() > 0) else None
            out = nhwc.noise_bias_act(input, None, None, b, None, negative_slope, scale)
        else:
            out = fused_bias_act_raw(input, bias, None, 3, 0, negative_slope, scale)
        ctx.save_for_backward(out)
        ctx.cfg = (negative_slope, scale, bias.dtype if bias is not None else None)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        (out,) = ctx.saved_tensors
        negative_slope, scale, bias_dtype = ctx.cfg
        want_bias = ctx.needs_input_grad[1]
        grad_input, grad_bias = _FusedLeakyReLUGrad.apply(grad_output, out, negative_slope, scale, want_bias, bias_dtype)
        return grad_input, (grad_bias if want_bias else None), None, None


def fused_leaky_relu(input, bias, negative_slope=0.2, scale=2 ** 0.5):
    """leaky_relu(input + bias[channel dim 1], negative_slope) * scale.  Unlike the reference's CPU branch
    (fused_act.py:87-94, which hard-codes 0.2) `negative_slope` is always honoured, as in its CUDA kernel."""
    return FusedLeakyReLUFunction.apply(input, bias, negative_slope, scale)


class FusedLeakyReLU(nn.Module):
    """Same parameter name (`bias`) and defaults as reference fused_act.py:74-83 (state-dict compatible)."""

    def __init__(self, channel, negative_slope=0.2, scale=2 ** 0.5):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(channel))
        self.negative_slope = negative_slope
        self.scale = scale

    def forward(self, input):
        return fused_leaky_relu(input, self.bias.type(input.dtype), self.negative_slope, self.scale)
