"""The generator's synthesis path fused ACROSS layer boundaries (channels-last activations, fp32 or bf16 storage).

reference: models/stylegan2/networks.py:514-586 (Generator.forward), :344-350 (StyledConv), :233-282 (ModulatedConv2d),
:389-405 (ToRGB).  Per resolution the reference runs  modulate -> grouped conv -> [blur] -> noise -> bias+lrelu  twice and a
to-RGB 1x1 grouped convolution + bias + up-sampled skip.  Here, per layer:

    raw = conv(scale*W, xs)                     one weight-SHARED cuDNN convolution on the already modulated input
    xs', rgb = fused_tail(raw, ...)             ONE kernel: [blur +] demodulation + noise + bias + lrelu, emits the NEXT
                                                convolution's modulated input xs' = o * s_next and (conv layers) the
                                                to-RGB image rgb = wm . o + bias + skip -- the unscaled activation o is
                                                written only when a backward pass will reduce over it
and the backward of a fused tail is one pass (two for the blur layers), with the style / demodulation / to-RGB weight
gradients reduced inside it (csrc/styled.cu, csrc/nhwc.cu mode 2).  A layer whose styles are constants (every layer above
the latent learner's inject index) owes the backward pass only g_raw, and g_raw needs only the SIGN of o: such a tail writes
a sign mask (1 bit per element) instead of o and keeps neither o nor raw; its backward reads (g_xs, mask).  Round 1's separate `channel_scale` passes (15.7 % of
the step), the to-RGB kernels, the gradient add of the RGB branch and the demodulation row-dot pass are gone.

Only the frozen-generator case GANgealing needs is fused (gradients flow to the latents/styles, never to the generator's
own parameters); anything else takes the layer-by-layer ops of styled_tail.py / modconv.py.
"""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import _lib
from . import conv2d_gradfix, nhwc, style_path
from .modconv import channel_scale, shared_conv_weight
from .upfirdn2d import grad_pad, upfirdn2d

CL = torch.channels_last


class _FusedTail(Function):
    """(raw, demod, s_next, wm, skip) -> (xs, rgb).  noise / noise_weight / bias / rgb_bias are constants here."""

    @staticmethod
    def forward(ctx, raw, demod, s_next, wm, skip, noise, noise_weight, bias, rgb_bias, kernel, pad, negative_slope, gain):
        _lib.require_cuda(raw, demod, s_next, wm, skip, noise)
        needs = ctx.needs_input_grad
        reduces = needs[1] or needs[2] or needs[3]      # a sum over the activation is owed to demod, s_next or wm
        save = needs[0] or reduces
        # only g_raw is owed: the backward pass needs lrelu'(o), the sign mask, and neither o nor raw
        masked = needs[0] and not reduces and (kernel is None or s_next is not None)
        if kernel is None:
            out, xs, rgb = nhwc.styled_tail(raw, noise, noise_weight, bias, demod, s_next, wm, rgb_bias, skip,
                                            save and not masked, negative_slope, gain, want_mask=masked)
        else:
            if wm is not None:
                raise RuntimeError("fused tail: the blur (up-sampling) layers carry no to-RGB branch")
            pad4 = (pad[0], pad[1], pad[0], pad[1])
            out, xs, _ = nhwc.blur(raw, kernel, pad4, mode=1, noise=noise, noise_weight=noise_weight, bias=bias,
                                   row_scale=demod, scale2=s_next, want_out=(save and not masked) or s_next is None,
                                   want_out2=s_next is not None, negative_slope=negative_slope, gain=gain, want_mask=masked)
            rgb = None
        ctx.cfg = (kernel is not None, pad, negative_slope, gain, tuple(raw.shape), masked, raw.dtype)
        if save:
            ctx.save_for_backward(raw if (needs[1] and demod is not None) else None, out,      # masked: `out` is the mask
                                  demod.detach() if demod is not None else None,
                                  s_next.detach() if s_next is not None else None,
                                  wm.detach() if wm is not None else None, kernel)
        if skip is not None and rgb is None:
            raise RuntimeError("fused tail: skip without a to-RGB branch")
        return xs, rgb

    @staticmethod
    @once_differentiable
    def backward(ctx, g_xs, g_rgb):
        raw, out, demod, s_next, wm, kernel = ctx.saved_tensors
        is_blur, pad, negative_slope, gain, raw_shape, masked, dtype = ctx.cfg
        need_raw, need_d, need_s, need_w, need_skip = ctx.needs_input_grad[:5]
        if g_xs is not None:
            g_xs = g_xs.contiguous(memory_format=CL)
            if g_xs.dtype != dtype:
                g_xs = g_xs.to(dtype)
        if g_rgb is not None:
            g_rgb = g_rgb.float().contiguous()
        g_raw = d_s = d_d = d_w = None
        if g_xs is None and g_rgb is None:
            return (None,) * 13
        if masked and not is_blur:
            g_raw = nhwc.styled_tail_backward_mask(g_xs, g_rgb, out, s_next, demod, wm, negative_slope, gain, dtype)
        elif not is_blur:
            g_raw, d_s, d_d, d_w = nhwc.styled_tail_backward(
                g_xs, g_rgb, out, raw, s_next, demod, wm, need_s, need_d and demod is not None, need_w,
                negative_slope, gain)
        else:
            # pass 1: g_t = lrelu'(out)*gain*(g_xs*s_next)   (+ d_s_next)      pass 2: adjoint blur, *demod, <B^T g_t, raw>
            if masked:
                g_t = nhwc.styled_tail_backward_mask(g_xs, None, out, s_next, None, None, negative_slope, gain, dtype)
            else:
                g_t, d_s, _, _ = nhwc.styled_tail_backward(g_xs, None, out, None, s_next, None, None, need_s, False, False,
                                                           negative_slope, gain)
            kh, kw = kernel.shape
            pad4 = (pad[0], pad[1], pad[0], pad[1])
            gp = grad_pad(raw_shape[2], raw_shape[3], g_t.shape[2], g_t.shape[3], kh, kw, (1, 1), (1, 1), pad4)
            want_dot = need_d and demod is not None
            g_raw, _, d_d = nhwc.blur(g_t, _lib.flipped_filter(kernel), gp, mode=2, row_scale=demod, mul=raw if want_dot else None,
                                      want_dot=want_dot)
            if tuple(g_raw.shape) != raw_shape:
                raise RuntimeError("fused tail backward: adjoint produced %s, expected %s" % (tuple(g_raw.shape), raw_shape))
        return (g_raw if need_raw else None, d_d if need_d else None, d_s if need_s else None, d_w if need_w else None,
                g_rgb if need_skip else None, None, None, None, None, None, None, None, None)


def fused_tail(raw, demod, s_next, wm, skip, noise, noise_weight, bias, rgb_bias, kernel=None, pad=None, negative_slope=0.2,
               gain=2 ** 0.5):
    """-> (xs, rgb): see the module docstring.  raw: channels-last (N, C, H, W) conv output; demod (N, C) or None;
    s_next (N, C) or None (last layer); wm (N, 3, C) / rgb_bias (3,) / skip (N, 3, H, W) or None; kernel/pad: the
    up-sampling layer's Blur (then H, W shrink by the filter support) or None."""
    return _FusedTail.apply(raw, demod, s_next, wm, skip, noise, noise_weight, bias, rgb_bias, kernel, pad, negative_slope, gain)


def fusable(generator, latent, act_dtype):
    """The cross-layer fused synthesis serves the frozen, plain (no fp16-normalisation branch) generator on CUDA whose
    channel counts fit the 16-byte-vector kernels."""
    if not latent.is_cuda or getattr(generator, "num_fp16_res", 0) != 0 and not generator.run_fp32:
        return False
    vec = 8 if act_dtype == torch.bfloat16 else 4
    layers = [generator.conv1] + list(generator.convs)
    for layer in layers:
        conv = layer.conv
        if conv.normalize or conv.downsample or not conv.demodulate or conv.out_channel % (8 * vec) or conv.in_channel % vec:
            return False
        if conv.kernel_size != 3 or layer.activate.scale <= 0:
            return False
    for m in list(generator.to_rgbs) + [generator.to_rgb1]:
        if m.conv.normalize or m.conv.demodulate or m.conv.out_channel != 3:
            return False
    return not any(p.requires_grad for p in generator.parameters())


def synthesis(generator, latent, noise, act_dtype=torch.float32, row_needs_grad=None):
    """Generator.forward's synthesis network (reference networks.py:562-586) on the fused path.  latent: (B, n_latent, D);
    noise: list (one entry per StyledConv; None entries are sampled, in the reference's order); row_needs_grad: see
    style_path.all_styles.  -> image (B, 3, S, S) fp32."""
    layers = [generator.conv1] + list(generator.convs)
    rgbs = [generator.to_rgb1] + list(generator.to_rgbs)
    b = latent.shape[0]
    # the whole style path up front, batched over layers (op/style_path.py): 3 GEMMs + 1 wgmma launch instead of 33 chains
    styles, rgb_styles = style_path.all_styles(generator, latent, layers, rgbs, list(range(len(layers))),
                                               [2 * r + 1 for r in range(len(rgbs))], row_needs_grad)
    demods = style_path.all_demod([layer.conv.weight for layer in layers], styles, [layer.conv.scale for layer in layers],
                                  layers[0].conv.eps)
    x0 = generator.input(latent).to(act_dtype).contiguous(memory_format=CL)
    xs = channel_scale(x0, styles[0])
    rgb = None
    for i, layer in enumerate(layers):
        conv, act = layer.conv, layer.activate
        w = shared_conv_weight(conv.weight, conv.scale, transposed=conv.upsample, channels_last=True, dtype=act_dtype)
        if conv.upsample:
            raw = conv2d_gradfix.conv_transpose2d(xs, w, padding=0, stride=2)
            blur = conv.blur
            out_h = raw.shape[2] + blur.pad[0] + blur.pad[1] - blur.kernel.shape[0] + 1
            out_w = raw.shape[3] + blur.pad[0] + blur.pad[1] - blur.kernel.shape[1] + 1
        else:
            raw = conv2d_gradfix.conv2d(xs, w, padding=conv.padding)
            blur = None
            out_h, out_w = raw.shape[2], raw.shape[3]
        nz = noise[i]
        if nz is None:   # same draw (shape, order) as NoiseInjection.forward, networks.py:293-296; always fp32
            nz = type(layer.noise).sample(b, out_h, out_w, styles[0])
        demod = demods[i]
        s_next = styles[i + 1] if i + 1 < len(layers) else None
        wm = rgb_bias = skip = None
        if not conv.upsample:          # conv1 and the second StyledConv of every resolution feed a ToRGB
            to_rgb = rgbs[i // 2]
            rconv = to_rgb.conv
            s_rgb = rgb_styles[i // 2]
            wm = (rconv.scale * rconv.weight[0, :, :, 0, 0]).unsqueeze(0) * s_rgb.unsqueeze(1)      # (B, 3, C)
            rgb_bias = to_rgb.bias
            if rgb is not None:
                skip = upfirdn2d(rgb, to_rgb.upsample.kernel, up=to_rgb.upsample.up, down=1, pad=to_rgb.upsample.pad)
        xs, new_rgb = fused_tail(raw, demod, s_next, wm, skip, nz, layer.noise.weight, act.bias, rgb_bias,
                                 kernel=blur.kernel if blur is not None else None, pad=blur.pad if blur is not None else None,
                                 negative_slope=act.negative_slope, gain=act.scale)
        if new_rgb is not None:
            rgb = new_rgb
    return rgb
