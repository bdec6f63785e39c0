"""StyleGAN2 generator + the conv blocks shared with the STN trunk -- host-side mirror of reference
models/stylegan2/networks.py, state-dict compatible (same module tree and parameter names), written against
the fused sm_90a ops:

  * StyledConv = modulated conv (cuDNN) + ONE fused tail kernel:
        upsampling layers : blur + noise + bias + leaky-ReLU*sqrt(2)   (reference: 3 passes, networks.py:266,346-348)
        plain layers      : noise + bias + leaky-ReLU*sqrt(2)          (reference: 2 passes)
  * Blur / Upsample go through upfirdn2d's bulk-TMA band kernel.
Classes and constructor arguments follow the reference so checkpoints load unchanged; `ops=` lets test
infrastructure run the same host code on the CPU oracle (see gangealing_b200/opset.py).
"""
import math
import random

import torch
from torch import nn
from torch.nn import functional as F

from ..opset import cuda_ops


def make_kernel(k):
    k = torch.tensor(k, dtype=torch.float32)
    if k.ndim == 1:
        k = k[None, :] * k[:, None]
    return k / k.sum()


class PixelNorm(nn.Module):
    def forward(self, input):
        return input * torch.rsqrt(torch.mean(input ** 2, dim=1, keepdim=True) + 1e-8)


class _FirModule(nn.Module):
    """Common base of Blur / Upsample / Downsample: a registered `kernel` buffer + upfirdn2d parameters."""

    def __init__(self, kernel, up, down, pad, ops):
        super().__init__()
        self.register_buffer("kernel", kernel)
        self.up, self.down, self.pad = up, down, pad
        self.ops = ops if ops is not None else cuda_ops()

    def forward(self, input):
        # the registered fp32 buffer itself is passed (the C ABI takes fp32 taps for every activation dtype): a per-call
        # `.type(...)` copy would defeat the per-filter memo (separability test, flipped taps) and sync the host
        return self.ops.upfirdn2d(input, self.kernel, up=self.up, down=self.down, pad=self.pad)


class Upsample(_FirModule):
    def __init__(self, kernel, factor=2, ops=None):
        k = make_kernel(kernel) * (factor ** 2)
        p = k.shape[0] - factor
        super().__init__(k, factor, 1, ((p + 1) // 2 + factor - 1, p // 2), ops)
        self.factor = factor


class Downsample(_FirModule):
    def __init__(self, kernel, factor=2, ops=None):
        k = make_kernel(kernel)
        p = k.shape[0] - factor
        super().__init__(k, 1, factor, ((p + 1) // 2, p // 2), ops)
        self.factor = factor


class Blur(_FirModule):
    def __init__(self, kernel, pad, upsample_factor=1, ops=None):
        k = make_kernel(kernel)
        if upsample_factor > 1:
            k = k * (upsample_factor ** 2)
        super().__init__(k, 1, 1, pad, ops)


class EqualConv2d(nn.Module):
    def __init__(self, in_channel, out_channel, kernel_size, stride=1, padding=0, bias=True, ops=None):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_channel, in_channel, kernel_size, kernel_size))
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.stride, self.padding = stride, padding
        self.bias = nn.Parameter(torch.zeros(out_channel)) if bias else None
        self.ops = ops if ops is not None else cuda_ops()

    scaler = None     # op/scaled_weights.WeightScaler of the training step, or None (set per instance by the Trainer)

    def forward(self, input, gain=1.0):
        """`gain`: extra output scale folded into the equalised-lr weight scale (ResBlock folds its 1/sqrt(2) here)."""
        w = self.scaler.get(self, input.dtype, gain) if self.scaler is not None and input.is_cuda else None
        if w is None:
            w = self.weight * (self.scale * gain)
        b = self.bias
        if w.dtype != input.dtype:      # bf16 activations (BASELINE config 3): fp32 master weights, bf16 tensor-core conv
            w = w.to(input.dtype)
        if b is not None and b.dtype != input.dtype:
            b = b.to(input.dtype)
        return self.ops.conv2d(input, w, bias=b, stride=self.stride, padding=self.padding)

    def __repr__(self):
        return (f"{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]},"
                f" {self.weight.shape[2]}, stride={self.stride}, padding={self.padding})")


class EqualLinear(nn.Module):
    def __init__(self, in_dim, out_dim, bias=True, bias_init=0, lr_mul=1, activation=None, ops=None):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_dim, in_dim).div_(lr_mul))
        self.bias = nn.Parameter(torch.zeros(out_dim).fill_(bias_init)) if bias else None
        self.activation = activation
        self.scale = (1 / math.sqrt(in_dim)) * lr_mul
        self.lr_mul = lr_mul
        self.ops = ops if ops is not None else cuda_ops()

    scaler = None     # see EqualConv2d.scaler

    def forward(self, input):
        w = self.scaler.get(self, input.dtype) if self.scaler is not None and input.is_cuda else None
        if w is None:
            w = self.weight * self.scale
        if self.activation:
            out = F.linear(input, w)
            return self.ops.fused_leaky_relu(out, self.bias * self.lr_mul)
        return F.linear(input, w, bias=self.bias * self.lr_mul)

    def __repr__(self):
        return f"{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]})"


class ScaledLeakyReLU(nn.Module):
    def __init__(self, negative_slope=0.2):
        super().__init__()
        self.negative_slope = negative_slope

    def forward(self, input):
        return F.leaky_relu(input, negative_slope=self.negative_slope) * math.sqrt(2)


class FusedLeakyReLU(nn.Module):
    """Same parameter (`bias`) as the reference's op/fused_act.py:74-83, routed through the injected op set."""

    def __init__(self, channel, negative_slope=0.2, scale=2 ** 0.5, ops=None):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(channel))
        self.negative_slope, self.scale = negative_slope, scale
        self.ops = ops if ops is not None else cuda_ops()

    def forward(self, input):
        # bf16 activations keep the fp32 master bias (the channels-last kernel takes fp32 per-channel constants)
        bias = self.bias if input.dtype == torch.bfloat16 else self.bias.type(input.dtype)
        return self.ops.fused_leaky_relu(input, bias, self.negative_slope, self.scale)


class ModulatedConv2d(nn.Module):
    """Weight-modulated convolution (reference networks.py:171-282).  `forward(..., fuse_blur=False)` returns the
    raw up-convolution so the caller can fuse the blur into its activation tail."""

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, demodulate=True, upsample=False,
                 downsample=False, blur_kernel=[1, 3, 3, 1], normalize=False, ops=None):
        super().__init__()
        self.eps = 1e-8
        self.kernel_size, self.in_channel, self.out_channel = kernel_size, in_channel, out_channel
        self.upsample, self.downsample, self.normalize = upsample, downsample, normalize
        self.ops = ops if ops is not None else cuda_ops()
        if upsample:
            factor = 2
            p = (len(blur_kernel) - factor) - (kernel_size - 1)
            self.blur = Blur(blur_kernel, pad=((p + 1) // 2 + factor - 1, p // 2 + 1), upsample_factor=factor, ops=ops)
        if downsample:
            factor = 2
            p = (len(blur_kernel) - factor) + (kernel_size - 1)
            self.blur = Blur(blur_kernel, pad=((p + 1) // 2, p // 2), ops=ops)
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.padding = kernel_size // 2
        self.weight = nn.Parameter(torch.randn(1, out_channel, in_channel, kernel_size, kernel_size))
        self.modulation = EqualLinear(style_dim, in_channel, bias_init=1, ops=ops)
        self.demodulate = demodulate

    def __repr__(self):
        return (f"{self.__class__.__name__}({self.in_channel}, {self.out_channel}, {self.kernel_size}, "
                f"upsample={self.upsample}, downsample={self.downsample})")

    def conv_raw(self, input, style):
        """-> (raw, demod): the convolution WITHOUT blur and demodulation, plus the (B, O) demodulation coefficients
        (or None when they are already folded into the result).  The op set chooses the formulation: the sm_90a set
        runs ONE weight-shared convolution on modulated activations, the CPU oracle the reference's grouped one."""
        style = self.modulation(style)
        plain = not (self.normalize or (input.dtype == torch.float16 and self.demodulate)) and not self.downsample
        if plain:
            return self.ops.modulated_conv2d(input, self.weight, style, self.scale, self.demodulate, self.upsample,
                                             self.padding, self.eps)
        return self._reference_formulation(input, style), None

    def forward(self, input, style, fuse_blur=True):
        raw, demod = self.conv_raw(input, style)
        if demod is not None:
            raw = self.ops.channel_scale(raw, demod)
        if self.upsample and fuse_blur:
            return self.blur(raw)
        return raw

    def _reference_formulation(self, input, style):
        """Per-sample filter banks + grouped convolution (reference networks.py:236-280): kept for the fp16
        pre-scaling branch and the (unused) downsampling variant."""
        batch, in_channel, height, width = input.shape
        weight = self.weight
        scale = self.scale
        if self.normalize or (input.dtype == torch.float16 and self.demodulate):
            style = style / torch.max(torch.abs(style))
            fan = torch.tensor(in_channel * weight.size(3) * weight.size(4), dtype=torch.float32)
            weight = scale * weight * torch.sqrt(1.0 / fan) / torch.amax(torch.abs(scale * weight), dim=(2, 3, 4), keepdims=True)
            scale = 1.0
        w = self.ops.modulated_weight(weight, style, scale, self.demodulate, transposed=self.upsample, eps=self.eps)
        w = w.type(input.dtype)
        x = input.reshape(1, batch * in_channel, height, width)
        if self.upsample:
            out = self.ops.conv_transpose2d(x, w, padding=0, stride=2, groups=batch)
        elif self.downsample:
            xb = self.blur(input)
            out = self.ops.conv2d(xb.reshape(1, batch * in_channel, xb.shape[2], xb.shape[3]), w, padding=0, stride=2,
                                  groups=batch)
        else:
            out = self.ops.conv2d(x, w, padding=self.padding, groups=batch)
        return out.view(batch, self.out_channel, out.shape[2], out.shape[3])


class NoiseInjection(nn.Module):
    def __init__(self):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(1))

    @staticmethod
    def sample(batch, height, width, like):
        return like.new_empty(batch, 1, height, width).normal_()

    def forward(self, image, noise=None):
        if noise is None:
            noise = self.sample(image.shape[0], image.shape[2], image.shape[3], image)
        return image + self.weight.type(image.dtype) * noise.type(image.dtype)


class ConstantInput(nn.Module):
    def __init__(self, channel, size=4):
        super().__init__()
        self.input = nn.Parameter(torch.randn(1, channel, size, size))
        self.size = size

    def forward(self, input):
        return self.input.repeat(input.shape[0], 1, 1, 1)


class StyledConv(nn.Module):
    """conv -> noise -> bias -> leaky ReLU.  The three elementwise stages (and the blur of upsampling layers) run as
    ONE kernel: `blur_noise_bias_act` / `noise_bias_act` (reference networks.py:344-350 runs them separately)."""

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, upsample=False, blur_kernel=[1, 3, 3, 1],
                 demodulate=True, normalize=False, ops=None):
        super().__init__()
        self.conv = ModulatedConv2d(in_channel, out_channel, kernel_size, style_dim, upsample=upsample,
                                    blur_kernel=blur_kernel, demodulate=demodulate, normalize=normalize, ops=ops)
        self.noise = NoiseInjection()
        self.activate = FusedLeakyReLU(out_channel, ops=ops)
        self.ops = ops if ops is not None else cuda_ops()

    def forward(self, input, style, noise=None):
        act = self.activate
        raw, demod = self.conv.conv_raw(input, style)
        if self.conv.upsample:
            blur = self.conv.blur
            out_h = raw.shape[2] + blur.pad[0] + blur.pad[1] - blur.kernel.shape[0] + 1
            out_w = raw.shape[3] + blur.pad[0] + blur.pad[1] - blur.kernel.shape[1] + 1
            if noise is None:
                noise = NoiseInjection.sample(raw.shape[0], out_h, out_w, raw)
            return self.ops.blur_noise_bias_act(raw, blur.kernel, blur.pad, noise, self.noise.weight, act.bias,
                                                act.negative_slope, act.scale, row_scale=demod)
        if noise is None:
            noise = NoiseInjection.sample(raw.shape[0], raw.shape[2], raw.shape[3], raw)
        return self.ops.noise_bias_act(raw, noise, self.noise.weight, act.bias, act.negative_slope, act.scale,
                                       row_scale=demod)


class ToRGB(nn.Module):
    def __init__(self, in_channel, style_dim, upsample=True, blur_kernel=[1, 3, 3, 1], normalize=False, ops=None):
        super().__init__()
        if upsample:
            self.upsample = Upsample(blur_kernel, ops=ops)
        self.conv = ModulatedConv2d(in_channel, 3, 1, style_dim, demodulate=False, normalize=normalize, ops=ops)
        self.bias = nn.Parameter(torch.zeros(1, 3, 1, 1))

    def forward(self, input, style, skip=None):
        conv = self.conv
        up = self.upsample(skip) if skip is not None else None
        if not (conv.normalize or conv.downsample or conv.upsample or conv.demodulate):
            # bias and skip ride in the op set's to-RGB epilogue (one pass over the activation on sm_90a)
            out, _ = conv.ops.modulated_conv2d(input, conv.weight, conv.modulation(style), conv.scale, False, False,
                                               conv.padding, conv.eps, bias=self.bias, skip=up)
            return out
        out = conv(input, style) + self.bias.type(input.dtype)
        if up is not None:
            out = out.float() + up
        return out


class ConvLayer(nn.Sequential):
    """[Blur] -> EqualConv2d -> [FusedLeakyReLU | ScaledLeakyReLU]   (reference networks.py:589-635)."""

    def __init__(self, in_channel, out_channel, kernel_size, downsample=False, blur_kernel=[1, 3, 3, 1], bias=True,
                 activate=True, ops=None):
        layers = []
        if downsample:
            factor = 2
            p = (len(blur_kernel) - factor) + (kernel_size - 1)
            layers.append(Blur(blur_kernel, pad=((p + 1) // 2, p // 2), ops=ops))
            stride, self.padding = 2, 0
        else:
            stride, self.padding = 1, kernel_size // 2
        layers.append(EqualConv2d(in_channel, out_channel, kernel_size, padding=self.padding, stride=stride,
                                  bias=bias and not activate, ops=ops))
        if activate:
            layers.append(FusedLeakyReLU(out_channel, ops=ops) if bias else ScaledLeakyReLU(0.2))
        super().__init__(*layers)


class ResBlock(nn.Module):
    def __init__(self, in_channel, out_channel, blur_kernel=[1, 3, 3, 1], downsample=True, ops=None):
        super().__init__()
        self.conv1 = ConvLayer(in_channel, in_channel, 3, ops=ops)
        self.conv2 = ConvLayer(in_channel, out_channel, 3, downsample=downsample, ops=ops)
        self.skip = ConvLayer(in_channel, out_channel, 1, downsample=downsample, activate=False, bias=False, ops=ops)

    def forward(self, input):
        """(conv2(conv1(x)) + skip(x)) / sqrt(2)   (reference networks.py:638-657).  On the sm_90a op set the 1/sqrt(2) is
        folded into the two branches -- the gain of conv2's fused bias+lrelu pass and the skip convolution's weight scale --
        so the block ends in ONE add instead of add + divide (and its backward loses the matching multiply): two
        activation-sized passes less per block and direction."""
        act, skip_conv = self.conv2[-1], self.skip[-1]
        if (input.is_cuda and isinstance(act, FusedLeakyReLU) and getattr(act.ops, "name", None) == "sm_90a"
                and isinstance(skip_conv, EqualConv2d) and skip_conv.bias is None):
            inv = 1.0 / math.sqrt(2)
            main = self.conv1(input)
            for layer in list(self.conv2)[:-1]:
                main = layer(main)
            bias = act.bias if main.dtype == torch.bfloat16 else act.bias.type(main.dtype)   # as FusedLeakyReLU.forward
            main = act.ops.fused_leaky_relu(main, bias, act.negative_slope, act.scale * inv)
            side = input
            for layer in list(self.skip)[:-1]:
                side = layer(side)
            return main + skip_conv(side, gain=inv)
        return (self.conv2(self.conv1(input)) + self.skip(input)) / math.sqrt(2)


def channel_table(channel_multiplier):
    return {4: 512, 8: 512, 16: 512, 32: 512, 64: 256 * channel_multiplier, 128: 128 * channel_multiplier,
            256: 64 * channel_multiplier, 512: 32 * channel_multiplier, 1024: 16 * channel_multiplier}


class Generator(nn.Module):
    """StyleGAN2 synthesis + mapping network (reference networks.py:396-586); frozen during GANgealing training."""

    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, blur_kernel=[1, 3, 3, 1], lr_mlp=0.01,
                 num_fp16_res=0, run_fp32=True, ops=None):
        super().__init__()
        self.size, self.style_dim = size, style_dim
        self.style = nn.Sequential(PixelNorm(), *[EqualLinear(style_dim, style_dim, lr_mul=lr_mlp, activation="fused_lrelu", ops=ops)
                                                  for _ in range(n_mlp)])
        self.channels = channel_table(channel_multiplier)
        self.input = ConstantInput(self.channels[4])
        self.conv1 = StyledConv(self.channels[4], self.channels[4], 3, style_dim, blur_kernel=blur_kernel, ops=ops)
        self.to_rgb1 = ToRGB(self.channels[4], style_dim, upsample=False, ops=ops)
        self.log_size = int(math.log(size, 2))
        self.num_layers = (self.log_size - 2) * 2 + 1
        self.convs, self.upsamples, self.to_rgbs = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        self.noises = nn.Module()
        for layer_idx in range(self.num_layers):
            res = (layer_idx + 5) // 2
            self.noises.register_buffer(f"noise_{layer_idx}", torch.randn(1, 1, 2 ** res, 2 ** res))
        in_channel = self.channels[4]
        for i in range(3, self.log_size + 1):
            mixed = i > self.log_size - num_fp16_res
            out_channel = self.channels[2 ** i]
            self.convs.append(StyledConv(in_channel, out_channel, 3, style_dim, upsample=True, blur_kernel=blur_kernel,
                                         normalize=mixed, ops=ops))
            self.convs.append(StyledConv(out_channel, out_channel, 3, style_dim, blur_kernel=blur_kernel,
                                         normalize=mixed, ops=ops))
            self.to_rgbs.append(ToRGB(out_channel, style_dim, normalize=False, ops=ops))
            in_channel = out_channel
        self.n_latent = self.log_size * 2 - 2
        self.num_fp16_res, self.run_fp32 = num_fp16_res, run_fp32
        # keep the synthesis activations channels-last (NHWC) between cuDNN's NHWC-native convolutions; the fused
        # kernels of this package have native channels-last variants (csrc/nhwc.cu).  Set by the Trainer on CUDA.
        self.channels_last = False
        # storage type of the synthesis activations on the channels-last path: fp32 (BASELINE config 2) or bf16 (config 3:
        # bf16 activations, fp32 arithmetic inside the fused kernels, bf16 tensor-core convolutions, fp32 RGB image)
        self.act_dtype = torch.float32
        self.fuse_synthesis = True      # cross-layer fused tails (op/styled_fused.py) when the configuration allows

    def ops_are_native(self):
        return getattr(self.conv1.ops, "name", None) == "sm_90a"

    def make_noise(self, batch_size=1):
        device = self.input.input.device
        noises = [torch.randn(batch_size, 1, 4, 4, device=device)]
        for i in range(3, self.log_size + 1):
            noises += [torch.randn(batch_size, 1, 2 ** i, 2 ** i, device=device) for _ in range(2)]
        return noises

    def batch_latent(self, n_latent):
        return self.style(torch.randn(n_latent, self.style_dim, device=self.input.input.device))

    def mean_latent(self, n_latent):
        return self.batch_latent(n_latent).mean(dim=0, keepdim=True)

    def get_latent(self, input):
        return self.style(input)

    def forward(self, styles, mapping_only=False, return_latents=False, inject_index=None, truncation=1,
                truncation_latent=None, input_is_latent=False, noise=None, randomize_noise=True):
        if not input_is_latent:
            styles = [self.style(s) for s in styles]
            if mapping_only:
                return styles
        if noise is None:
            noise = [None] * self.num_layers if randomize_noise else \
                [getattr(self.noises, f"noise_{i}") for i in range(self.num_layers)]
        if truncation < 1:
            styles = [truncation_latent + truncation * (styles[0] - truncation_latent), styles[0]]
        row_needs_grad = None       # per latent row; None: whatever `latent` itself says
        if len(styles) < 2 or inject_index == self.n_latent:
            inject_index = self.n_latent
            latent = styles[0].unsqueeze(1).repeat(1, inject_index, 1) if styles[0].ndim < 3 else styles[0]
        else:
            if inject_index is None:
                inject_index = random.randint(1, self.n_latent - 1)
            latent = torch.cat([styles[0].unsqueeze(1).repeat(1, inject_index, 1),
                                styles[1].unsqueeze(1).repeat(1, self.n_latent - inject_index, 1)], 1)
            # the concatenation requires grad as soon as one part does; the fused synthesis is told which rows really do
            row_needs_grad = [styles[0].requires_grad] * inject_index + [styles[1].requires_grad] * (self.n_latent - inject_index)

        if self.channels_last and self.fuse_synthesis and self.ops_are_native():
            from ..op import styled_fused
            if styled_fused.fusable(self, latent, self.act_dtype):
                image = styled_fused.synthesis(self, latent, noise, self.act_dtype, row_needs_grad)
                return (image, latent) if return_latents else (image, None)
        x0 = self.input(latent)
        if self.channels_last:
            x0 = x0.contiguous(memory_format=torch.channels_last)
        out = self.conv1(x0, latent[:, 0], noise=noise[0])
        skip = self.to_rgb1(out, latent[:, 1])
        i = 1
        for j, (up, conv, n_up, n_conv, to_rgb) in enumerate(
                zip(self.convs[::2], self.convs[1::2], noise[1::2], noise[2::2], self.to_rgbs), 3):
            half = j > self.log_size - self.num_fp16_res and not self.run_fp32
            out = out.type(torch.float16 if half else torch.float32)
            out = up(out, latent[:, i], noise=n_up)
            out = conv(out, latent[:, i + 1], noise=n_conv)
            skip = to_rgb(out, latent[:, i + 2], skip)
            i += 2
        return (skip, latent) if return_latents else (skip, None)
