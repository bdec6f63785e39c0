"""Modulated-convolution weight path: modulate -> demodulate -> (transposed layout for the up-conv), fused.

reference: models/stylegan2/networks.py:233-253 (`weight = scale*W*style`, `demod = rsqrt(sum w^2 + 1e-8)`,
`weight *= demod`) and :255-262 (transpose + reshape for conv_transpose2d): ~6 ATen launches materialising three
(B, O, I, k, k) temporaries per layer.  Here (csrc/modconv.cu):
    demod[b,o] = rsqrt(scale^2 * sum_i Wsq[o,i] * style[b,i]^2 + eps)    one wgmma (tensor-core) GEMM
    out        = scale * W * style[b,i] * demod[b,o]                     one pass, written in the conv's layout
`Wsq = sum_k W^2` and the pre-transposed filter bank are cached per (storage, version) -- the generator is frozen.
Backward (w.r.t. the style only -- the generator's filters never need a gradient in GANgealing):
    T[b,o,i] = sum_k g[b,o,i,k] W[o,i,k];  gd = scale * sum_i T s;  gs = scale * sum_o T d - scale^2 s * ((gd d^3) @ Wsq)
"""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import _lib
from . import nhwc

def channel_scale_raw(x, s, y=None):
    """out = x * s[n, c]; with `y`: also row_dot[n, c] = sum_hw x*y (fp32).  x: (N, C, H, W); s: (N, C) fp32."""
    _lib.require_cuda(x, s, y)
    if nhwc.rowwise_ok(x):
        if y is not None:
            y = y.contiguous(memory_format=torch.channels_last)
            if y.dtype != x.dtype:
                y = y.to(x.dtype)
        return nhwc.channel_scale(x, s, y)
    x = x.contiguous()
    n, c = x.shape[0], x.shape[1]
    hw = x.numel() // max(n * c, 1)
    s = s.reshape(n * c)
    if s.dtype != torch.float32 or not s.is_contiguous():
        s = s.float().contiguous()
    lib = _lib.load()
    out = torch.empty_like(x)
    dot = ws = None
    if y is not None:
        y = y.contiguous()
        dot = torch.empty((n, c), dtype=torch.float32, device=x.device)
        ws = torch.empty(max(1, lib.gg_channel_scale_workspace(n * c, hw) // 4), dtype=torch.float32, device=x.device)
    rc = lib.gg_channel_scale(out.data_ptr(), _lib.ptr(dot), _lib.ptr(ws), x.data_ptr(), _lib.ptr(y), s.data_ptr(),
                              _lib.dtype_code(x), n * c, hw, _lib.stream())
    _lib.check(rc, "gg_channel_scale")
    return out, dot


class _ChannelScale(Function):
    @staticmethod
    def forward(ctx, x, s):
        out, _ = channel_scale_raw(x, s.detach())
        ctx.save_for_backward(x, s)
        return out

    @staticmethod
    def backward(ctx, g):
        x, s = ctx.saved_tensors
        need_x, need_s = ctx.needs_input_grad
        if need_s:   # one pass: g*s and sum_hw g*x
            gx, gs = channel_scale_raw(g, s.detach(), y=x)
            return (gx if need_x else None), gs.reshape(s.shape).to(s.dtype)
        return _ChannelScale.apply(g, s.detach()), None


def channel_scale(x, s):
    """x (N, C, H, W) * s (N, C)[:, :, None, None] in one fused pass (differentiable in both)."""
    return _ChannelScale.apply(x, s)


class _Demod(Function):
    """demod[b, o] = rsqrt(scale^2 * sum_i Wsq[o, i] style[b, i]^2 + eps) on the tensor cores (wgmma, TF32 hi/lo)."""

    @staticmethod
    def forward(ctx, weight, style, scale, eps):
        _, o, i, kh, kw = weight.shape
        s = style.detach()
        if s.dtype != torch.float32 or not s.is_contiguous():
            s = s.float().contiguous()
        _, wsq, _ = _derived(weight, False)
        b = s.shape[0]
        lib = _lib.load()
        demod = torch.empty((b, o), dtype=torch.float32, device=s.device)
        for b0 in range(0, b, 256):
            nb = min(256, b - b0)
            rc = lib.gg_modconv_demod(demod[b0:].data_ptr(), wsq.data_ptr(), s[b0:].data_ptr(), scale, eps, nb, o, i,
                                      _lib.stream())
            _lib.check(rc, "gg_modconv_demod")
        ctx.save_for_backward(s, demod, wsq)
        ctx.cfg = (scale, style.dtype)
        return demod

    @staticmethod
    @once_differentiable
    def backward(ctx, gd):
        s, demod, wsq = ctx.saved_tensors
        scale, style_dtype = ctx.cfg
        gs = -(scale * scale) * s * ((gd.float() * demod.pow(3)) @ wsq)
        return None, gs.to(style_dtype), None, None


def demod_coefficients(weight, style, scale, eps=1e-8):
    """(B, O) demodulation coefficients of ModulatedConv2d (reference networks.py:245-246), differentiable in `style`."""
    if weight.requires_grad:
        w = (scale * weight) * style.reshape(style.shape[0], 1, -1, 1, 1)
        return torch.rsqrt(w.pow(2).sum([2, 3, 4]) + eps)
    _lib.require_cuda(weight, style)
    return _Demod.apply(weight, style, float(scale), float(eps))


def shared_conv_weight(weight, scale, transposed, channels_last=False, dtype=None):
    """scale * W as the weight of a weight-SHARED convolution: (O, I, k, k), or (I, O, k, k) for conv_transpose2d, in
    `dtype` (default: the parameter's).  Memoised on the parameter object for frozen filter banks."""
    dtype = weight.dtype if dtype is None else dtype
    if weight.requires_grad:
        w = (weight[0] * scale).to(dtype)
        return w.transpose(0, 1) if transposed else w
    memo = _lib.tensor_cache(weight)
    key = ("shared", float(scale), bool(transposed), bool(channels_last), dtype)
    w = memo.get(key)
    if w is None:
        w = (weight.detach()[0] * scale).to(dtype)
        w = w.transpose(0, 1).contiguous() if transposed else w.contiguous()
        if channels_last and w.shape[2] * w.shape[3] > 1:
            w = w.contiguous(memory_format=torch.channels_last)
        memo[key] = w
    return w


class _ToRGB(Function):
    """out = wm (B, 3, C) applied to the channels-last activation + bias + skip, one pass (csrc/nhwc.cu)."""

    @staticmethod
    def forward(ctx, x, wm, bias, skip):
        _lib.require_cuda(x, wm, bias, skip)
        n, c, h, w = x.shape
        wmc = _lib.dense_f32(wm.detach())
        b = bias.detach().float().reshape(-1).contiguous() if bias is not None else None
        sk = _lib.dense_f32(skip.detach()) if skip is not None else None
        out = torch.empty((n, 3, h, w), dtype=torch.float32, device=x.device)
        rc = _lib.load().gg_to_rgb_nhwc_forward(out.data_ptr(), x.data_ptr(), wmc.data_ptr(), _lib.ptr(b), _lib.ptr(sk),
                                                n, c, h * w, _lib.stream())
        _lib.check(rc, "gg_to_rgb_nhwc_forward")
        ctx.save_for_backward(x, wmc)
        ctx.meta = (bias.shape if bias is not None else None, wm.dtype)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, wmc = ctx.saved_tensors
        bias_shape, wm_dtype = ctx.meta
        need_x, need_w, need_b, need_s = ctx.needs_input_grad
        n, c, h, w = x.shape
        g = g.float().contiguous()
        lib = _lib.load()
        gx = gw = ws = None
        if need_x:
            gx = torch.empty_like(x)
        if need_w:
            gw = torch.empty((n, 3, c), dtype=torch.float32, device=x.device)
            ws = torch.empty(max(1, lib.gg_to_rgb_nhwc_workspace(n, c, h * w) // 4), dtype=torch.float32, device=x.device)
        if need_x or need_w:
            rc = lib.gg_to_rgb_nhwc_backward(_lib.ptr(gx), _lib.ptr(gw), _lib.ptr(ws), g.data_ptr(), x.data_ptr(),
                                             wmc.data_ptr(), n, c, h * w, _lib.stream())
            _lib.check(rc, "gg_to_rgb_nhwc_backward")
        gb = g.sum(dim=(0, 2, 3)).reshape(bias_shape) if need_b and bias_shape is not None else None
        return gx, (gw.to(wm_dtype) if gw is not None else None), gb, (g if need_s else None)


def modulated_conv2d(x, weight, style, scale, demodulate=True, upsample=False, padding=1, eps=1e-8, bias=None, skip=None):
    """ModulatedConv2d's convolution, weight-shared: conv(scale*W*s, x) == conv(scale*W, x*s), so ONE weight-shared
    (dense, tensor-core friendly) cuDNN convolution replaces the reference's grouped convolution over B materialised
    filter banks (networks.py:255-280); tools/convbench.py times the two formulations.
    Returns (raw, demod): the caller applies `demod` (B, O) -- or None -- as the per-(sample, channel) row scale of its
    fused activation tail (it commutes with the blur).  `bias` (1, O, 1, 1) / `skip` (B, O, H, W) are added to `raw`
    (the to-RGB layer's epilogue, networks.py:400-405)."""
    from . import conv2d_gradfix
    _, o, i, kh, kw = weight.shape
    if kh == 1 and kw == 1 and not upsample and not demodulate:
        # to-RGB: a (3 x C) matrix per sample
        wm = (scale * weight[0, :, :, 0, 0]).unsqueeze(0) * style.unsqueeze(1)            # (B, O, I)
        b, _, h, w_ = x.shape
        if _lib.is_nhwc(x) and o == 3 and i % 32 == 0 and i <= 1024 and x.dtype == torch.float32 and _lib.aligned16(x):
            return _ToRGB.apply(x, wm, bias, skip), None      # one fused pass over the channels-last activation
        if _lib.is_nhwc(x):   # (B, HW, I) @ (B, I, O): reads the channels-last activation in place
            rgb = torch.bmm(x.permute(0, 2, 3, 1).reshape(b, h * w_, i), wm.type(x.dtype).transpose(1, 2))
            rgb = rgb.reshape(b, h, w_, o).permute(0, 3, 1, 2)
        else:                 # one batched GEMM reads the activation once, nothing is re-written
            rgb = torch.bmm(wm.type(x.dtype), x.reshape(b, i, h * w_)).reshape(b, o, h, w_)
        return _epilogue(rgb, bias, skip), None
    xs = channel_scale(x, style)
    w = shared_conv_weight(weight, scale, transposed=upsample, channels_last=_lib.is_nhwc(x), dtype=x.dtype)
    if upsample:
        raw = conv2d_gradfix.conv_transpose2d(xs, w, padding=0, stride=2)
    else:
        raw = conv2d_gradfix.conv2d(xs, w, padding=padding)
    d = demod_coefficients(weight, style, scale, eps) if demodulate else None
    return _epilogue(raw, bias, skip), d


def _epilogue(raw, bias, skip):
    if bias is not None:
        raw = raw + bias.type(raw.dtype)
    if skip is not None:
        raw = raw.float() + skip
    return raw


def _derived(weight, need_t):
    """(W as (O, I, kk) fp32, Wsq (O, I), W^T (I, O, kk) or None) of a filter bank, memoised on the parameter object
    (invalidated by in-place updates)."""
    memo = _lib.tensor_cache(weight)
    ent = memo.get("derived")
    if ent is None:
        _, o, i, kh, kw = weight.shape
        w3 = weight.detach().reshape(o, i, kh * kw)
        if w3.dtype != torch.float32 or not w3.is_contiguous():
            w3 = w3.float().contiguous()
        wsq = torch.empty((o, i), dtype=torch.float32, device=w3.device)
        _lib.check(_lib.load().gg_modconv_wsq(wsq.data_ptr(), w3.data_ptr(), o, i, kh * kw, _lib.stream()), "gg_modconv_wsq")
        ent = [w3, wsq, None]
        memo["derived"] = ent
    if need_t and ent[2] is None:
        ent[2] = ent[0].transpose(0, 1).contiguous()
    return ent[0], ent[1], ent[2]


def modulated_weight_composite(weight, style, scale, demodulate=True, transposed=False, eps=1e-8):
    """Plain tensor-op formulation, differentiable w.r.t. the filters too (not needed by GANgealing's frozen G)."""
    b = style.shape[0]
    _, o, i, kh, kw = weight.shape
    w = (scale * weight) * style.reshape(b, 1, i, 1, 1)
    if demodulate:
        w = w * torch.rsqrt(w.pow(2).sum([2, 3, 4]) + eps).reshape(b, o, 1, 1, 1)
    if transposed:
        return w.transpose(1, 2).reshape(b * i, o, kh, kw)
    return w.reshape(b * o, i, kh, kw)


class _ModulatedWeight(Function):
    @staticmethod
    def forward(ctx, weight, style, scale, demodulate, transposed, eps):
        _lib.require_cuda(weight, style)
        _, o, i, kh, kw = weight.shape
        kk = kh * kw
        b = style.shape[0]
        s = style.detach()
        if s.dtype != torch.float32 or not s.is_contiguous():
            s = s.float().contiguous()
        lib = _lib.load()
        st = _lib.stream()
        w3, wsq, wt = _derived(weight, transposed)
        demod = None
        if demodulate:
            demod = torch.empty((b, o), dtype=torch.float32, device=s.device)
            for b0 in range(0, b, 256):  # the tensor-core tile holds at most 256 batch columns
                nb = min(256, b - b0)
                rc = lib.gg_modconv_demod(demod[b0:].data_ptr(), wsq.data_ptr(), s[b0:].data_ptr(), scale, eps, nb, o, i, st)
                _lib.check(rc, "gg_modconv_demod")
        out = torch.empty((b * i, o, kh, kw) if transposed else (b * o, i, kh, kw), dtype=torch.float32, device=s.device)
        rc = lib.gg_modconv_modulate(out.data_ptr(), (wt if transposed else w3).data_ptr(), s.data_ptr(), _lib.ptr(demod),
                                     scale, b, o, i, kk, 1 if transposed else 0, st)
        _lib.check(rc, "gg_modconv_modulate")
        ctx.save_for_backward(w3, s, demod, wsq)
        ctx.cfg = (scale, transposed, (o, i, kh, kw), style.dtype)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        w3, s, demod, wsq = ctx.saved_tensors
        scale, transposed, (o, i, kh, kw), style_dtype = ctx.cfg
        b = s.shape[0]
        g = grad_out.reshape(b, i, o, kh * kw).transpose(1, 2) if transposed else grad_out.reshape(b, o, i, kh * kw)
        t = torch.einsum("boik,oik->boi", g.float(), w3)
        if demod is not None:
            gd = scale * torch.einsum("boi,bi->bo", t, s)
            gs = scale * torch.einsum("boi,bo->bi", t, demod) - (scale * scale) * s * ((gd * demod.pow(3)) @ wsq)
        else:
            gs = scale * t.sum(dim=1)
        return None, gs.to(style_dtype), None, None, None, None


def modulated_weight(weight, style, scale, demodulate=True, transposed=False, eps=1e-8):
    """weight (1, O, I, k, k), style (B, I) -> per-sample filters for the grouped convolution:
    (B*O, I, k, k), or (B*I, O, k, k) when `transposed` (the layout conv_transpose2d(groups=B) wants)."""
    _, o, i, kh, kw = weight.shape
    inner = (o if transposed else i) * kh * kw
    if weight.requires_grad or inner % 4 != 0:
        # filters that need a gradient (never in GANgealing) or odd tiny banks (to-RGB: O = 3, k = 1, I % 4 == 0 is fine)
        return modulated_weight_composite(weight, style, scale, demodulate, transposed, eps)
    return _ModulatedWeight.apply(weight, style, float(scale), bool(demodulate), bool(transposed), float(eps))
