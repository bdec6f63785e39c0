"""Raw (no autograd) Python faces of the channels-last kernel family (csrc/nhwc.cu, csrc/styled.cu).

Everything here takes / returns channels-last (N, C, H, W) CUDA tensors whose storage type is fp32 or bf16 (the C ABI's
`dtype`); per-channel constants, noise planes and reductions are fp32.  The autograd wrappers live in styled_tail.py
(generic ops with the reference's call surfaces) and styled_fused.py (the generator's cross-layer fused path).
"""
import torch

from .. import _lib

CL = torch.channels_last

# bench.py sets this to a list to time every fused blur-tail launch (gg_blur_nhwc mode 1) with CUDA events on the launching
# stream: entries are (start_event, end_event, algorithmic_bytes).  None (default): no instrumentation.
TIMING = None


# Which tensors each kernel family takes.  Every kernel moves 16 bytes of channels at a time (V = 4 fp32 / 8 bf16 channels),
# so the activation must start on a 16-byte boundary (the blur's TMA descriptor needs that too).
def elementwise_ok(t):
    """noise_bias_act: a 16-byte-aligned channels-last activation whose C is a multiple of V."""
    return _lib.is_nhwc(t) and t.shape[1] % _lib.nhwc_vec(t) == 0 and _lib.aligned16(t)


def rowwise_ok(t):
    """channel_scale, bias_act_backward: as elementwise, and C / V <= 256 (a CTA's threads cover one pixel's channels)."""
    return elementwise_ok(t) and t.shape[1] // _lib.nhwc_vec(t) <= 256


def blur_ok(t, kh, kw, up=(1, 1), down=(1, 1)):
    """blur: C a multiple of 8 V (a CTA covers 8 threads x 16 bytes of channels), a filter of at most 4 x 4 taps and no
    up- or down-sampling."""
    return (_lib.is_nhwc(t) and t.shape[1] % (8 * _lib.nhwc_vec(t)) == 0 and kh <= 4 and kw <= 4
            and up == (1, 1) and down == (1, 1) and _lib.aligned16(t))


def _f32(t, numel=None):
    """`t` as dense, 16-byte-aligned fp32 (a copy when it is not).  Callers bind the result to a name until the launch: a
    temporary freed while the argument list is still being built lets the next one reuse its memory."""
    if t is None:
        return None
    t = _lib.dense_f32(t.detach())
    if numel is not None and t.numel() != numel:
        raise RuntimeError("channels-last op: expected %d fp32 values, got %d" % (numel, t.numel()))
    return t


def noise_plane(noise, n, h, w):
    """(N, 1, H, W) (or broadcastable) noise -> dense fp32 (N, H, W) plane, or None."""
    if noise is None:
        return None
    noise = noise.detach()
    if noise.numel() != n * h * w:
        noise = noise.expand(n, 1, h, w)
    return noise.float().contiguous()


def sign_mask_empty(n, c, h, w, device):
    """Storage of the sign mask of an (N, C, H, W) channels-last activation: (N, H, W, C/32) 32-bit words (csrc/common.cuh)."""
    if c % 32:
        raise RuntimeError("sign mask: C = %d is not a multiple of 32" % c)
    return torch.empty((n, h, w, c // 32), dtype=torch.int32, device=device)


def blur(x, kernel, pad, mode=0, noise=None, noise_weight=None, bias=None, row_scale=None, scale2=None, want_out=True,
         want_out2=False, mul=None, want_dot=False, negative_slope=0.2, gain=1.0, act=3, want_mask=False):
    """gg_blur_nhwc.  pad = (x0, x1, y0, y1).  -> (out, out2, row_dot).  want_mask (mode 1): gg_blur_nhwc_mask, `out` is the
    sign mask of the activation instead of the activation."""
    n, c, in_h, in_w = x.shape
    taps = kernel.detach()
    if taps.dtype != torch.float32 or not taps.is_contiguous():
        taps = taps.float().contiguous()
    kh, kw = taps.shape
    out_h = in_h + pad[2] + pad[3] - kh + 1
    out_w = in_w + pad[0] + pad[1] - kw + 1
    if out_h < 1 or out_w < 1:
        raise RuntimeError("blur: empty output (%d x %d)" % (out_h, out_w))
    lib = _lib.load()
    code = _lib.dtype_code(x)

    def empty():
        return torch.empty((n, c, out_h, out_w), dtype=x.dtype, device=x.device, memory_format=CL)
    if want_mask and mode != 1:
        raise RuntimeError("blur: the sign mask belongs to the fused tail (mode 1)")
    if want_mask:
        out = sign_mask_empty(n, c, out_h, out_w, x.device)
    else:
        out = empty() if (want_out or mode != 1) else None
    out2 = empty() if (mode == 1 and want_out2) else None
    nz = noise_plane(noise, n, out_h, out_w) if mode == 1 else None
    dot = ws = None
    if mode == 2 and want_dot:
        if (mul is None or mul.shape != (n, c, out_h, out_w) or mul.dtype != x.dtype or not mul.is_contiguous(memory_format=CL)
                or not _lib.aligned16(mul)):
            raise RuntimeError("blur (adjoint epilogue): `mul` must be a 16-byte-aligned channels-last tensor of the output's "
                               "shape and dtype")
        dot = torch.empty((n, c), dtype=torch.float32, device=x.device)
        nbytes = lib.gg_blur_nhwc_workspace(code, n, c, in_h, in_w, kh, kw, pad[0], pad[1], pad[2], pad[3])
        ws = torch.empty(max(1, nbytes // 4), dtype=torch.float32, device=x.device)
    timed = TIMING is not None and mode == 1
    if timed:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    nw, b, rs, s2 = _f32(noise_weight, 1), _f32(bias, c), _f32(row_scale, n * c), _f32(scale2, n * c)
    sep = 1 if _lib.filter_is_separable(kernel) else 0
    if want_mask:
        rc = lib.gg_blur_nhwc_mask(out.data_ptr(), _lib.ptr(out2), x.data_ptr(), taps.data_ptr(), _lib.ptr(nz), _lib.ptr(nw),
                                   _lib.ptr(b), _lib.ptr(rs), _lib.ptr(s2), code, n, c, in_h, in_w, kh, kw, sep, pad[0],
                                   pad[1], pad[2], pad[3], act, negative_slope, gain, _lib.stream())
    else:
        rc = lib.gg_blur_nhwc(_lib.ptr(out), _lib.ptr(out2), x.data_ptr(), taps.data_ptr(), _lib.ptr(nz),
                              _lib.ptr(nw), _lib.ptr(b), _lib.ptr(rs),
                              _lib.ptr(s2), _lib.ptr(mul if dot is not None else None), _lib.ptr(dot), _lib.ptr(ws),
                              code, n, c, in_h, in_w, kh, kw, sep, pad[0], pad[1],
                              pad[2], pad[3], mode, act, negative_slope, gain, _lib.stream())
    _lib.check(rc, "gg_blur_nhwc_mask" if want_mask else "gg_blur_nhwc")
    if timed:
        ev1.record()
        es = x.element_size()
        writes = (out is not None and not want_mask) + (out2 is not None)
        TIMING.append((ev0, ev1, es * n * c * (in_h * in_w + writes * out_h * out_w) + (4 * n * out_h * out_w if nz is not None else 0)
                       + (out.numel() * 4 if want_mask else 0)
                       + 4 * ((2 + (scale2 is not None)) * c + 1 + kh * kw)))
    return out, out2, dot


def noise_bias_act(x, noise, noise_weight, bias, row_scale, negative_slope, gain):
    n, c, h, w = x.shape
    out = torch.empty_like(x)
    nz, nw, b, rs = noise_plane(noise, n, h, w), _f32(noise_weight, 1), _f32(bias, c), _f32(row_scale, n * c)
    rc = _lib.load().gg_noise_bias_act_nhwc(out.data_ptr(), x.data_ptr(), _lib.ptr(nz), _lib.ptr(nw), _lib.ptr(b),
                                            _lib.ptr(rs), _lib.dtype_code(x), negative_slope, gain, n, c, h * w,
                                            _lib.stream())
    _lib.check(rc, "gg_noise_bias_act_nhwc")
    return out


def bias_act_backward(g, out_saved, negative_slope, gain, want_bias_grad):
    n, c, h, w = out_saved.shape
    lib = _lib.load()
    gx = torch.empty_like(out_saved)
    grad_bias = ws = None
    if want_bias_grad:
        grad_bias = torch.empty(c, dtype=torch.float32, device=g.device)
        ws = torch.empty(max(1, lib.gg_nhwc_rowwise_workspace(n, c, h * w) // 4), dtype=torch.float32, device=g.device)
    rc = lib.gg_bias_act_backward_nhwc(gx.data_ptr(), _lib.ptr(grad_bias), _lib.ptr(ws), g.data_ptr(), out_saved.data_ptr(),
                                       _lib.dtype_code(out_saved), negative_slope, gain, n, c, h * w, _lib.stream())
    _lib.check(rc, "gg_bias_act_backward_nhwc")
    return gx, grad_bias


def channel_scale(x, s, y=None):
    n, c, h, w = x.shape
    lib = _lib.load()
    out = torch.empty_like(x)
    dot = ws = None
    if y is not None:
        dot = torch.empty((n, c), dtype=torch.float32, device=x.device)
        ws = torch.empty(max(1, lib.gg_nhwc_rowwise_workspace(n, c, h * w) // 4), dtype=torch.float32, device=x.device)
    sc = _f32(s, n * c)
    rc = lib.gg_channel_scale_nhwc(out.data_ptr(), _lib.ptr(dot), _lib.ptr(ws), x.data_ptr(), _lib.ptr(y), sc.data_ptr(),
                                   _lib.dtype_code(x), n, c, h * w, _lib.stream())
    _lib.check(rc, "gg_channel_scale_nhwc")
    return out, dot


def _activation_like(t, like, who, name):
    """The styled tails read `t` 16 bytes at a time as a channels-last (N, C, H, W) tensor of `like`'s shape and dtype."""
    if t is not None and (t.shape != like.shape or t.dtype != like.dtype or not t.is_contiguous(memory_format=CL)
                          or not _lib.aligned16(t)):
        raise RuntimeError("%s: %s must be a 16-byte-aligned channels-last tensor of the activation's shape and dtype"
                           % (who, name))


def _rgb_grad_ok(g_rgb, n, h, w, who):
    """The styled tails' backward reads the to-RGB gradient as planar (N, 3, H*W) fp32."""
    if g_rgb is not None and (g_rgb.shape != (n, 3, h, w) or g_rgb.dtype != torch.float32 or not g_rgb.is_contiguous()):
        raise RuntimeError("%s: g_rgb must be a dense fp32 (N, 3, H, W) tensor" % who)


def styled_tail(raw, noise, noise_weight, bias, demod, s_next, wm, rgb_bias, skip, want_out, negative_slope, gain, act=3,
                want_mask=False):
    """gg_styled_tail_nhwc -> (out or None, xs or None, rgb or None).  want_mask: gg_styled_tail_mask_nhwc, the first
    result is the sign mask of the activation instead of the activation."""
    _activation_like(raw, raw, "styled_tail", "raw")
    n, c, h, w = raw.shape
    if want_mask:
        out = sign_mask_empty(n, c, h, w, raw.device)
    else:
        out = torch.empty_like(raw) if want_out else None
    xs = torch.empty_like(raw) if s_next is not None else None
    rgb = torch.empty((n, 3, h, w), dtype=torch.float32, device=raw.device) if wm is not None else None
    sk = None
    if skip is not None and rgb is not None:
        sk = skip.detach()
        if sk.dtype != torch.float32 or not sk.is_contiguous():
            sk = sk.float().contiguous()
        if sk.shape != rgb.shape:
            raise RuntimeError("styled_tail: skip must be (N, 3, H, W)")
    consts = [noise_plane(noise, n, h, w), _f32(noise_weight, 1), _f32(bias, c), _f32(demod, n * c), _f32(s_next, n * c),
              _f32(wm, n * 3 * c), _f32(rgb_bias, 3)]
    lib = _lib.load()
    entry = lib.gg_styled_tail_mask_nhwc if want_mask else lib.gg_styled_tail_nhwc
    rc = entry(_lib.ptr(out), _lib.ptr(xs), _lib.ptr(rgb), raw.data_ptr(), *[_lib.ptr(t) for t in consts], _lib.ptr(sk),
               _lib.dtype_code(raw), act, negative_slope, gain, n, c, h * w, _lib.stream())
    _lib.check(rc, "gg_styled_tail_mask_nhwc" if want_mask else "gg_styled_tail_nhwc")
    return out, xs, rgb


def styled_tail_backward(g_xs, g_rgb, out_saved, raw, s_next, demod, wm, want_ds, want_dd, want_dwm, negative_slope, gain):
    """gg_styled_tail_backward_nhwc -> (g_raw, d_s_next, d_demod, d_wm)."""
    n, c, h, w = out_saved.shape
    lib = _lib.load()
    dev = out_saved.device
    want_ds = want_ds and g_xs is not None
    want_dd = want_dd and raw is not None
    want_dwm = want_dwm and g_rgb is not None
    for name, t in (("out_saved", out_saved), ("g_xs", g_xs), ("raw", raw if want_dd else None)):
        _activation_like(t, out_saved, "styled_tail_backward", name)
    _rgb_grad_ok(g_rgb, n, h, w, "styled_tail_backward")
    g_raw = torch.empty_like(out_saved)
    # the requested sums are row slices of ONE (N, R, C) block: a single finish launch, views handed to autograd
    rows = int(want_ds) + int(want_dd) + 3 * int(want_dwm)
    block = torch.empty((n, rows, c), dtype=torch.float32, device=dev) if rows else None
    r = 0
    d_s = d_d = d_w = None
    if want_ds:
        d_s = block[:, r]; r += 1
    if want_dd:
        d_d = block[:, r]; r += 1
    if want_dwm:
        d_w = block[:, r:r + 3]
    code = _lib.dtype_code(out_saved)
    ws = None
    if rows:
        ws = torch.empty(max(1, lib.gg_styled_tail_backward_workspace(code, n, c, h * w) // 4), dtype=torch.float32, device=dev)
    consts = [_f32(s_next, n * c), _f32(demod, n * c), _f32(wm, n * 3 * c)]
    rc = lib.gg_styled_tail_backward_nhwc(g_raw.data_ptr(), _lib.ptr(d_s), _lib.ptr(d_d), _lib.ptr(d_w), _lib.ptr(ws),
                                          _lib.ptr(g_xs), _lib.ptr(g_rgb), out_saved.data_ptr(),
                                          _lib.ptr(raw if want_dd else None),
                                          *[_lib.ptr(t) for t in consts],
                                          code, negative_slope, gain, n, c, h * w, rows * c, _lib.stream())
    _lib.check(rc, "gg_styled_tail_backward_nhwc")
    return g_raw, d_s, d_d, d_w


def styled_tail_backward_mask(g_xs, g_rgb, mask, s_next, demod, wm, negative_slope, gain, dtype):
    """gg_styled_tail_backward_mask_nhwc -> g_raw (channels-last (N, C, H, W) of `dtype`): the data gradient of the tail
    from the forward pass's sign mask (N, H, W, C/32), when no style, demodulation or to-RGB weight gradient is wanted."""
    n, h, w, words = mask.shape
    c = 32 * words
    g_raw = torch.empty((n, c, h, w), dtype=dtype, device=mask.device, memory_format=CL)
    _activation_like(g_xs, g_raw, "styled_tail_backward_mask", "g_xs")
    _rgb_grad_ok(g_rgb, n, h, w, "styled_tail_backward_mask")
    consts = [_f32(s_next, n * c), _f32(demod, n * c), _f32(wm, n * 3 * c)]
    rc = _lib.load().gg_styled_tail_backward_mask_nhwc(g_raw.data_ptr(), _lib.ptr(g_xs), _lib.ptr(g_rgb), mask.data_ptr(),
                                                       *[_lib.ptr(t) for t in consts], _lib.dtype_code(g_raw),
                                                       negative_slope, gain, n, c, h * w, _lib.stream())
    _lib.check(rc, "gg_styled_tail_backward_mask_nhwc")
    return g_raw
