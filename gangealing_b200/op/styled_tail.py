"""Fused StyledConv tails -- the ops the reference runs as 2-3 separate passes over the activation.

  noise_bias_act      : NoiseInjection -> FusedLeakyReLU                      (networks.py:346-348)
  blur_noise_bias_act : Blur -> NoiseInjection -> FusedLeakyReLU              (networks.py:266, 346-348)

Both are differentiable w.r.t. every tensor input.  Backward shares the fused bias-act backward
kernel; the blur adjoint goes through the differentiable `upfirdn2d`, so higher orders compose.
"""
import torch
from torch.autograd import Function

from .. import _lib
from . import nhwc
from .fused_act import bias_act_backward_raw
from .modconv import channel_scale_raw
from .nhwc import _f32
from .upfirdn2d import UpFirDn2d, _taps, grad_pad


# bench.py sets this to a list to time every fused-blur launch with CUDA events on the launching stream:
# entries are (start_event, end_event, algorithmic_bytes).  None (default): no instrumentation.
TIMING = None


def _noise_plane(noise, x, out_h, out_w):
    if noise is None:
        return None
    n = x.shape[0]
    if noise.numel() != n * out_h * out_w:
        noise = noise.expand(n, 1, out_h, out_w)
    return noise.to(x.dtype).contiguous()


class _StyledTail(Function):
    @staticmethod
    def forward(ctx, x, noise, noise_weight, bias, kernel, pad, row_scale, negative_slope, scale):
        _lib.require_cuda(x, noise, noise_weight, bias, kernel, row_scale)
        cl = nhwc.elementwise_ok(x) if kernel is None else nhwc.blur_ok(x, *kernel.shape)
        if not cl:
            x = x.contiguous()
        n, c, in_h, in_w = x.shape
        lib = _lib.load()
        nw = _f32(noise_weight.reshape(-1)) if noise_weight is not None else None
        b = _f32(bias.reshape(-1)) if bias is not None else None
        rs = _f32(row_scale.reshape(-1)) if row_scale is not None else None
        if cl:
            if kernel is None:
                out = nhwc.noise_bias_act(x, noise, nw, b, rs, negative_slope, scale)
            else:
                out = nhwc.blur(x, kernel, pad, mode=1, noise=noise, noise_weight=nw, bias=b, row_scale=rs,
                                negative_slope=negative_slope, gain=scale)[0]      # timed through op.nhwc.TIMING
        elif kernel is None:
            out = torch.empty_like(x)
            nz = _noise_plane(noise, x, in_h, in_w)
            rc = lib.gg_noise_bias_act(out.data_ptr(), x.data_ptr(), _lib.ptr(nz), _lib.ptr(nw), _lib.ptr(b),
                                       _lib.ptr(rs), _lib.dtype_code(x), negative_slope, scale, n, c, in_h * in_w,
                                       _lib.stream())
            _lib.check(rc, "gg_noise_bias_act")
        else:
            taps = _taps(kernel)
            kh, kw = taps.shape
            out_h = in_h + pad[2] + pad[3] - kh + 1
            out_w = in_w + pad[0] + pad[1] - kw + 1
            out = torch.empty((n, c, out_h, out_w), dtype=x.dtype, device=x.device)
            nz = _noise_plane(noise, x, out_h, out_w)
            if TIMING is not None:
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
            rc = lib.gg_blur_noise_bias_act(out.data_ptr(), x.data_ptr(), taps.data_ptr(), _lib.ptr(nz),
                                            _lib.ptr(nw), _lib.ptr(b), _lib.ptr(rs), _lib.dtype_code(x), n, c,
                                            in_h, in_w, kh, kw, pad[0], pad[1], pad[2], pad[3], 3,
                                            negative_slope, scale, _lib.stream())
            _lib.check(rc, "gg_blur_noise_bias_act")
            if TIMING is not None:
                ev1.record()
                es = x.element_size()
                nbytes = es * n * c * (in_h * in_w + out_h * out_w) + (es * n * out_h * out_w if nz is not None else 0) \
                    + 4 * (c + 1 + kh * kw)
                TIMING.append((ev0, ev1, nbytes))
        ctx.save_for_backward(out, noise, noise_weight, kernel, row_scale, x if row_scale is not None else None)
        ctx.cfg = (pad, negative_slope, scale, tuple(x.shape))
        return out

    @staticmethod
    def backward(ctx, grad_output):
        out, noise, noise_weight, kernel, row_scale, x_saved = ctx.saved_tensors
        pad, negative_slope, scale, in_size = ctx.cfg
        need_x, need_noise, need_nw, need_bias, _, _, need_rs = ctx.needs_input_grad[:7]
        # d(out)/d(pre-activation): shared with FusedLeakyReLU's backward kernel
        gx, gbias = bias_act_backward_raw(grad_output, out, negative_slope, scale, need_bias)
        g_noise = g_nw = g_rs = g_x = None
        if noise is not None and (need_noise or need_nw):
            per_plane = gx.sum(dim=1, keepdim=True)  # (N, 1, H, W)
            if need_nw:
                g_nw = (per_plane * noise.to(per_plane.dtype)).sum().reshape(noise_weight.shape).to(noise_weight.dtype)
            if need_noise:
                w = noise_weight.reshape(()) if noise_weight is not None else 1.0
                g_noise = (per_plane * w).to(noise.dtype)
                while g_noise.dim() > noise.dim():
                    g_noise = g_noise.squeeze(0)
                if g_noise.shape != noise.shape:
                    g_noise = g_noise.sum_to_size(noise.shape)
        if need_x or need_rs:
            if kernel is None:
                g_t = gx
            else:
                kh, kw = kernel.shape
                gp = grad_pad(in_size[2], in_size[3], out.shape[2], out.shape[3], kh, kw, (1, 1), (1, 1), pad)
                g_t = UpFirDn2d.apply(gx, _lib.flipped_filter(kernel), (1, 1), (1, 1), gp)  # adjoint blur
            if row_scale is not None:
                # one fused pass: g_x = g_t * rs  and  g_rs = sum_hw g_t * x   (<B(x), g> = <x, B^T g>)
                g_x, dot = channel_scale_raw(g_t, row_scale.detach().reshape(in_size[0], in_size[1]),
                                             y=x_saved if need_rs else None)
                if need_rs:
                    g_rs = dot.reshape(row_scale.shape).to(row_scale.dtype)
            else:
                g_x = g_t
        if gbias is not None:
            gbias = gbias.to(out.dtype)
        return (g_x if need_x else None), g_noise, g_nw, gbias, None, None, g_rs, None, None


def noise_bias_act(x, noise, noise_weight, bias, negative_slope=0.2, scale=2 ** 0.5, row_scale=None):
    """leaky_relu(row_scale*x + noise_weight*noise + bias[c]) * scale in one pass.
    x: (N, C, H, W); noise: (N, 1, H, W) (or broadcastable) or None; noise_weight: 1-element tensor; bias: (C,);
    row_scale: (N, C) or None (demodulation coefficients of a weight-shared modulated convolution)."""
    return _StyledTail.apply(x, noise, noise_weight, bias, None, None, row_scale, negative_slope, scale)


def blur_noise_bias_act(x, kernel, pad, noise, noise_weight, bias, negative_slope=0.2, scale=2 ** 0.5,
                        row_scale=None):
    """leaky_relu(row_scale*upfirdn2d(x, kernel, pad=pad) + noise_weight*noise + bias[c]) * scale in one pass
    over the activation (kernel <= 4x4, up = down = 1).  `pad` is the Blur module's 2-tuple."""
    pad4 = (pad[0], pad[1], pad[0], pad[1])
    return _StyledTail.apply(x, noise, noise_weight, bias, kernel, pad4, row_scale, negative_slope, scale)
