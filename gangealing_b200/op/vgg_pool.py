"""The VGG16 slice boundary of the perceptual loss in one pass per direction (csrc/lpips.cu).

reference: models/losses/lpips_backbones.py:106-121 -- torchvision's `features` run Conv2d -> ReLU -> MaxPool2d(2, 2) at the
end of slices 1-4, and the ReLU output is ALSO the feature map the distance taps (lpips.py:181-192).  ATen walks that map four
more times (max_pool forward + index map, max_pool backward, the add of the two gradients meeting at the tap, ReLU backward);
`bias_relu_pool(raw, bias)` returns `(y, pooled)` from one read of the convolution output, and its backward is one pass that
recomputes the window arg-max from `y` (first maximum, row-major: ATen's max_pool2d rule).  CUDA, channels-last, fp32 / bf16.
"""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import _lib


def supported(x):
    """Shapes the fused kernel takes: (N, C, H, W) channels-last, H and W even, C a multiple of one 16-byte vector."""
    if x.dim() != 4 or x.dtype not in (torch.float32, torch.bfloat16) or not x.is_cuda:
        return False
    n, c, h, w = x.shape
    return h % 2 == 0 and w % 2 == 0 and h > 0 and w > 0 and c % (16 // x.element_size()) == 0


class _BiasReluPool(Function):
    @staticmethod
    def forward(ctx, raw, bias):
        n, c, h, w = raw.shape
        y = torch.empty_like(raw)                                       # channels-last like raw
        pooled = torch.empty(n, c, h // 2, w // 2, dtype=raw.dtype, device=raw.device, memory_format=torch.channels_last)
        b = None if bias is None else _lib.dense_f32(bias.detach())
        with torch.cuda.device(raw.device):
            _lib.check(_lib.load().gg_bias_relu_pool_nhwc_forward(y.data_ptr(), pooled.data_ptr(), raw.data_ptr(), _lib.ptr(b),
                                                                  _lib.dtype_code(raw), n, c, h, w, _lib.stream()),
                       "gg_bias_relu_pool_nhwc_forward")
        ctx.save_for_backward(y)
        return y, pooled

    @staticmethod
    @once_differentiable
    def backward(ctx, g_y, g_pooled):
        (y,) = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None
        n, c, h, w = y.shape
        cl = torch.channels_last

        def prep(g):
            if g is None:
                return None
            return g.to(y.dtype).contiguous(memory_format=cl)
        g_y, g_pooled = prep(g_y), prep(g_pooled)
        g_raw = torch.empty_like(y)
        with torch.cuda.device(y.device):
            _lib.check(_lib.load().gg_bias_relu_pool_nhwc_backward(g_raw.data_ptr(), _lib.ptr(g_y), _lib.ptr(g_pooled), y.data_ptr(),
                                                                   _lib.dtype_code(y), n, c, h, w, _lib.stream()),
                       "gg_bias_relu_pool_nhwc_backward")
        return g_raw, None


def bias_relu_pool(raw, bias):
    """(relu(raw + bias[c]), max_pool2d of it with a 2x2 window and stride 2).  `bias`: (C,) frozen (no gradient) or None."""
    _lib.require_cuda(raw, bias)
    if bias is not None and bias.requires_grad:
        raise RuntimeError("bias_relu_pool: a trainable bias is not supported (the perceptual network is frozen, lpips.py:136-139)")
    if not supported(raw):
        raise RuntimeError("bias_relu_pool: expected a CUDA (N, C, H, W) fp32/bf16 map with even H, W and C a multiple of one "
                           "16-byte vector, got %s %s" % (tuple(raw.shape), raw.dtype))
    if not raw.is_contiguous(memory_format=torch.channels_last):
        raw = raw.contiguous(memory_format=torch.channels_last)
    return _BiasReluPool.apply(raw, bias)
