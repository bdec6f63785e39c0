"""Every half-precision storage path against float64: each stored value rounded once, each fp32 reduction at fp32 accuracy.

bf16 (and, on the NCHW path, fp16) is a storage format here: a kernel reads its half-precision operands, computes in fp32
and rounds every stored value once (DESIGN.md section 3.4).  Each launch below is called through its raw Python face and
compared with a float64 reference evaluated on the exact half-precision operands it reads, with the checks of
oracle/rounding.py:

  stored outputs   |y - ref| <= 1/2 ulp + k * 2^-24 * A      k = fp32 roundings on the way to the store (stated per test)
  fp32 outputs     |y - ref| <= c * 2^-24 * sum|terms|        c = the longest chain of fp32 roundings of the reduction,
                                                              derived from the launch geometry below

Every check prints its worst observed ratios (`[contract] ...` lines, visible with `pytest -s`).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from fp64_contract import (DEV, SQRT2, blur_k, blur_plan, ceil_div, check_once, check_sum, cl, distance64, distance_c_terms,
                           distance_forward_c, finish_depth, fir64, lrelu64, randn, rowwise_c, seeded, slope_gain)
from oracle import stylegan2_ops as so

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
CS = [64, 192, 512]                   # 192: a non-power-of-two multiple of the bf16 blur multiple (64)
SPATIAL = [(4, 4), (9, 9), (33, 29)]


# ------------------------------------------------------------------------------------------------ launch geometry -> c
def _sm():
    from gangealing_b200 import _lib
    return _lib.sm_count()


def filt(kind, gain=1.0):
    if kind == "sep":
        return (so.make_kernel([1, 3, 3, 1]) * gain).to(DEV)
    g = torch.Generator().manual_seed(11)
    k = torch.randn(4, 4, generator=g) * gain / 4
    return k.to(DEV)


# ================================================================================================ channels-last family
@pytest.mark.parametrize("c", CS)
@pytest.mark.parametrize("hw", SPATIAL)
@pytest.mark.parametrize("noise,row_scale", [(False, False), (True, False), (False, True), (True, True)])
def test_noise_bias_act_nhwc(c, hw, noise, row_scale):
    """o = lrelu(rs*x + b + nw*noise)*gain: nw*noise, the fma, + noise, *slope, *gain -> k = 5."""
    from gangealing_b200.op import nhwc
    g = seeded(c + hw[0])
    n = 3
    x = cl(randn((n, c, *hw), g, BF))
    nz = randn((n, 1, *hw), g) if noise else None
    nw = torch.tensor([0.7], device=DEV) if noise else None
    b = randn((c,), g)
    rs = torch.rand(n, c, generator=g, device=DEV) + 0.5 if row_scale else None
    y = nhwc.noise_bias_act(x, nz, nw, b, rs, 0.2, SQRT2)
    x64 = x.double()
    r64 = rs.double()[:, :, None, None] if rs is not None else 1.0
    pre = x64 * r64 + b.double()[:, None, None]
    a = (x64 * r64).abs() + b.double().abs()[:, None, None]
    if noise:
        pre = pre + nw.double() * nz.double()
        a = a + (nw.double() * nz.double()).abs()
    check_once(y, lrelu64(pre, 0.2, SQRT2), a * slope_gain(0.2, SQRT2), 5, "noise_bias_act C=%d %s" % (c, hw))


@pytest.mark.parametrize("c", CS)
@pytest.mark.parametrize("hw", SPATIAL + [(257, 257)])
def test_bias_act_backward_nhwc(c, hw):
    """gx = (out > 0 ? g : slope*g)*gain stored once (k = 2); grad_bias = sum of the UNROUNDED gx."""
    from gangealing_b200.op import nhwc
    if hw == (257, 257) and c != 192:
        pytest.skip("one channel count at the full-size plane")
    g = seeded(c * 7 + hw[0])
    n = 2
    gy = cl(randn((n, c, *hw), g, BF))
    out = randn((n, c, *hw), g)
    out = cl(torch.where(torch.rand(out.shape, generator=g, device=DEV) < 0.05, torch.zeros_like(out), out).to(BF))
    gx, gb = nhwc.bias_act_backward(gy, out, 0.2, SQRT2, True)
    slope = torch.where(out.double() > 0, 1.0, 0.2) * SQRT2
    ref = gy.double() * slope
    check_once(gx, ref, ref.abs(), 2, "bias_act_backward gx C=%d %s" % (c, hw))
    check_sum(gb, ref.sum((0, 2, 3)), ref.abs().sum((0, 2, 3)), rowwise_c(n, c, hw[0] * hw[1], 2, False, BF, _sm()),
              "bias_act_backward grad_bias C=%d %s" % (c, hw))


@pytest.mark.parametrize("c", CS)
@pytest.mark.parametrize("hw", SPATIAL)
def test_channel_scale_with_row_dot_nhwc(c, hw):
    """out = x*s (k = 1); row_dot = sum_p x*y (one fma per pixel on a thread's chain)."""
    from gangealing_b200.op import nhwc
    g = seeded(c * 3 + hw[1])
    n = 3
    x = cl(randn((n, c, *hw), g, BF))
    yv = cl(randn((n, c, *hw), g, BF))
    s = randn((n, c), g)
    out, dot = nhwc.channel_scale(x, s, yv)
    ref = x.double() * s.double()[:, :, None, None]
    check_once(out, ref, ref.abs(), 1, "channel_scale C=%d %s" % (c, hw))
    t = x.double() * yv.double()
    check_sum(dot, t.sum((2, 3)), t.abs().sum((2, 3)), rowwise_c(n, c, hw[0] * hw[1], 0, True, BF, _sm()),
              "channel_scale row_dot C=%d %s" % (c, hw))


@pytest.mark.parametrize("c", CS)
@pytest.mark.parametrize("hw", SPATIAL)
@pytest.mark.parametrize("pad", [1, 2])
@pytest.mark.parametrize("gain", [1.0, 4.0])
@pytest.mark.parametrize("kind", ["sep", "rand"])
def test_blur_mode0_nhwc(c, hw, pad, gain, kind):
    """Plain blur (the STN trunk's pads (1,1) / (2,2)): k = blur_k."""
    from gangealing_b200.op import nhwc
    g = seeded(c + hw[0] + pad)
    k = filt(kind, gain)
    x = cl(randn((2, c, *hw), g, BF))
    p4 = (pad, pad, pad, pad)
    y, _, _ = nhwc.blur(x, k, p4, mode=0)
    check_once(y, fir64(x.double(), k, p4), fir64(x.double().abs(), k.abs(), p4), blur_k(k),
               "blur mode 0 %s gain %g pad %d C=%d %s" % (kind, gain, pad, c, hw))


BLUR_TAIL_SHAPES = [(3, 64, 9, 9), (2, 192, 33, 29), (4, 512, 4, 4), (2, 128, 257, 257)]


@pytest.mark.parametrize("shape", BLUR_TAIL_SHAPES)
@pytest.mark.parametrize("slope", [0.2, 1.5])       # 0.2: the gain-folded FAST epilogue; 1.5: the general one
@pytest.mark.parametrize("kind", ["sep", "rand"])
def test_blur_mode1_fused_tail_nhwc(shape, slope, kind):
    """out = RN(o), out2 = RN(o*s_next) from the fp32 o, o = lrelu(rs*B(x) + b + nw*noise)*gain.
    k = blur_k + 5 (gain folded into rs / b / nw, nw*noise, b + noise, the fma, *slope [, *gain]); out2: + 1."""
    from gangealing_b200.op import nhwc
    if shape[2] == 257 and (kind != "sep" or slope != 0.2):
        pytest.skip("the benchmark layer in its own configuration")
    n, c, h, w = shape
    g = seeded(c + h + int(slope * 10))
    k = filt(kind, 4.0)
    p4 = (1, 1, 1, 1)
    x = cl(randn((n, c, h, w), g, BF))
    oh, ow = h - 1, w - 1
    nz = randn((n, 1, oh, ow), g)
    nw = torch.tensor([0.3], device=DEV)
    b = randn((c,), g) * 0.5
    rs = torch.rand(n, c, generator=g, device=DEV) + 0.5
    s2 = randn((n, c), g) + 1.0
    out, out2, _ = nhwc.blur(x, k, p4, mode=1, noise=nz, noise_weight=nw, bias=b, row_scale=rs, scale2=s2, want_out=True,
                             want_out2=True, negative_slope=slope, gain=SQRT2)
    r64, s64 = rs.double()[:, :, None, None], s2.double()[:, :, None, None]
    pre = r64 * fir64(x.double(), k, p4) + b.double()[:, None, None] + nw.double() * nz.double()
    a = (r64 * fir64(x.double().abs(), k.abs(), p4) + b.double().abs()[:, None, None] + (nw.double() * nz.double()).abs())
    a = a * slope_gain(slope, SQRT2)
    o = lrelu64(pre, slope, SQRT2)
    kk = blur_k(k) + 5
    what = "blur mode 1 %s slope %g %s" % (kind, slope, tuple(shape))
    check_once(out, o, a, kk, what + " out")
    check_once(out2, o * s64, a * s64.abs(), kk + 1, what + " out2")


@pytest.mark.parametrize("shape", [(3, 64, 9, 9), (2, 192, 33, 29), (4, 512, 4, 4), (2, 128, 256, 256)])
@pytest.mark.parametrize("kind", ["sep", "rand"])
def test_blur_mode2_adjoint_epilogue_nhwc(shape, kind):
    """g_raw = RN(B(g)*rs) (k = blur_k + 1); dot = sum_p B(g)*mul: blur_k + the fma, a thread's rows of its segment, the
    CTA's 32 column groups, the finish kernel."""
    from gangealing_b200.op import nhwc
    if shape[2] == 256 and kind != "sep":
        pytest.skip("the benchmark layer with its own filter")
    n, c, h, w = shape
    g = seeded(c + h + 5)
    k = torch.flip(filt(kind, 4.0), [0, 1]).contiguous()
    p4 = (2, 2, 2, 2)                                  # the adjoint of the (1, 1)-padded 4-tap blur
    x = cl(randn((n, c, h, w), g, BF))
    oh, ow = h + 1, w + 1
    rs = torch.rand(n, c, generator=g, device=DEV) + 0.5
    mul = cl(randn((n, c, oh, ow), g, BF))
    y, _, dot = nhwc.blur(x, k, p4, mode=2, row_scale=rs, mul=mul, want_dot=True)
    t, ta = fir64(x.double(), k, p4), fir64(x.double().abs(), k.abs(), p4)
    r64 = rs.double()[:, :, None, None]
    what = "blur mode 2 %s %s" % (kind, tuple(shape))
    check_once(y, t * r64, ta * r64, blur_k(k) + 1, what + " g_raw")
    p = blur_plan(BF, n, c, h, w, 4, 4, p4, _sm())
    check_sum(dot, (t * mul.double()).sum((2, 3)), (ta * mul.double().abs()).sum((2, 3)),
              blur_k(k) + 1 + p["seg_rows"] + 32 + finish_depth(p["xblocks"] * p["segs"]), what + " dot")


TAIL_SHAPES = [(3, 64, 4, 4), (2, 192, 9, 9), (2, 512, 33, 29), (2, 128, 256, 256)]


def tail_inputs(shape, seed):
    n, c, h, w = shape
    g = seeded(seed)
    t = {"raw": cl(randn((n, c, h, w), g, BF)), "noise": randn((n, 1, h, w), g), "nw": torch.tensor([0.3], device=DEV),
         "bias": randn((c,), g) * 0.5, "demod": torch.rand(n, c, generator=g, device=DEV) + 0.5,
         "s_next": randn((n, c), g) + 1.0, "wm": randn((n, 3, c), g) / c ** 0.5, "rgb_bias": randn((3,), g),
         "skip": randn((n, 3, h, w), g)}
    return t


@pytest.mark.parametrize("shape", TAIL_SHAPES)
@pytest.mark.parametrize("slope", [0.2, 1.5])
def test_styled_tail_forward_nhwc(shape, slope):
    """out = RN(o) (k = 6: gain folded into demod / bias / nw, nw*noise, b + noise, the fma, *slope [, *gain]),
    xs = RN(o*s_next) (k = 7), rgb = wm . o + rgb_bias + skip in fp32: a lane's C/8 fmas, 3 butterfly steps, 2 adds and
    the 6 roundings of o -> c = C/8 + 11."""
    from gangealing_b200.op import nhwc
    n, c, h, w = shape
    t = tail_inputs(shape, c + h + int(slope * 10))
    out, xs, rgb = nhwc.styled_tail(t["raw"], t["noise"], t["nw"], t["bias"], t["demod"], t["s_next"], t["wm"], t["rgb_bias"],
                                    t["skip"], True, slope, SQRT2)
    d64 = t["demod"].double()[:, :, None, None]
    noise = t["nw"].double() * t["noise"].double()
    pre = t["raw"].double() * d64 + t["bias"].double()[:, None, None] + noise
    a = ((t["raw"].double() * d64).abs() + t["bias"].double().abs()[:, None, None] + noise.abs()) * slope_gain(slope, SQRT2)
    o = lrelu64(pre, slope, SQRT2)
    s64 = t["s_next"].double()[:, :, None, None]
    what = "styled_tail slope %g %s" % (slope, tuple(shape))
    check_once(out, o, a, 6, what + " out")
    check_once(xs, o * s64, a * s64.abs(), 7, what + " xs")
    wm = t["wm"].double()
    ref = torch.einsum("noc,nchw->nohw", wm, o) + t["rgb_bias"].double().reshape(1, 3, 1, 1) + t["skip"].double()
    ab = torch.einsum("noc,nchw->nohw", wm.abs(), a) + t["rgb_bias"].double().abs().reshape(1, 3, 1, 1) + t["skip"].double().abs()
    check_sum(rgb, ref, ab, c // 8 + 11, what + " rgb")


@pytest.mark.parametrize("shape", TAIL_SHAPES)
@pytest.mark.parametrize("slope", [0.2, 1.5])
def test_styled_tail_backward_nhwc(shape, slope):
    """g_raw = RN(lrelu'(out)*gain*(g_xs*s_next + wm^T g_rgb)*demod): g_xs*s, 3 fmas, *slope, *gain, *demod -> k = 7.
    d_s_next = sum g_xs*out, d_wm = sum g_rgb*out (one fma per pixel), d_demod = sum g_t*raw (+ the 6 roundings of g_t):
    a thread's pixels, the CTA's pixel lanes, the finish kernel."""
    from gangealing_b200.op import nhwc
    n, c, h, w = shape
    t = tail_inputs(shape, c + h + 1)
    g = seeded(c + h + 2)
    gxs = cl(randn((n, c, h, w), g, BF))
    grgb = randn((n, 3, h, w), g)
    out = randn((n, c, h, w), g)
    out = cl(torch.where(torch.rand(out.shape, generator=g, device=DEV) < 0.05, torch.zeros_like(out), out).to(BF))
    g_raw, d_s, d_d, d_w = nhwc.styled_tail_backward(gxs, grgb, out, t["raw"], t["s_next"], t["demod"], t["wm"], True, True,
                                                     True, slope, SQRT2)
    s64 = t["s_next"].double()[:, :, None, None]
    d64 = t["demod"].double()[:, :, None, None]
    wm = t["wm"].double()
    go = gxs.double() * s64 + torch.einsum("noc,nohw->nchw", wm, grgb.double())
    goa = (gxs.double() * s64).abs() + torch.einsum("noc,nohw->nchw", wm.abs(), grgb.double().abs())
    sl = torch.where(out.double() > 0, 1.0, slope) * SQRT2
    gt, gta = go * sl, goa * sl.abs()
    what = "styled_tail_backward slope %g %s" % (slope, tuple(shape))
    check_once(g_raw, gt * d64, gta * d64.abs(), 7, what + " g_raw")
    c0 = rowwise_c(n, c, h * w, 0, True, BF, _sm())
    o64, r64 = out.double(), t["raw"].double()
    check_sum(d_s, (gxs.double() * o64).sum((2, 3)), (gxs.double() * o64).abs().sum((2, 3)), c0, what + " d_s_next")
    check_sum(d_d, (gt * r64).sum((2, 3)), (gta * r64.abs()).sum((2, 3)), c0 + 6, what + " d_demod")
    dw = torch.einsum("nohw,nchw->noc", grgb.double(), o64)
    dwa = torch.einsum("nohw,nchw->noc", grgb.double().abs(), o64.abs())
    check_sum(d_w, dw, dwa, c0, what + " d_wm")


# ================================================================================================ perceptual front end
def distance_backward_k(c):
    """g = gs*(t*ia - a*ka), t = w*(a*ia - b*ib), ka = (sum t*a)*ia*ia/ra: the sums S twice, the inverse norm four times
    over (e_ia each) and ~16 products, differences and the 2*g/HW scale."""
    s, e_ia, _, _ = distance_c_terms(c)
    return int(math.ceil(2 * s + 4 * e_ia + 16))


@pytest.mark.parametrize("c", [4, 8, 16, 32, 64, 128, 256, 384, 512, 768, 1024])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("stacked", [False, True])
def test_feature_distance_bf16_value_and_gradients(c, weighted, stacked):
    """Every <L, TRIPS> instantiation of launch_distance (L = 1..32, TRIPS = 1, 2, 3, 4, 6, 8), forward and backward."""
    from gangealing_b200.op.feature_distance import feature_distance, feature_distance_stacked
    g = seeded(c + 2 * int(weighted) + int(stacked))
    n, h, w = 2, 6, 5
    a = cl(torch.relu(randn((n, c, h, w), g)).to(BF))
    b = cl(torch.relu(randn((n, c, h, w), g) + 0.2).to(BF))
    wt = torch.rand(c, generator=g, device=DEV) + 0.1 if weighted else None
    gout = randn((n, 1, 1, 1), g)
    if stacked:
        f = cl(torch.cat([a, b])).requires_grad_(True)
        r = feature_distance_stacked(f, wt)
        (gf,) = torch.autograd.grad(r, [f], gout)
        g0, g1 = gf[:n], gf[n:]
    else:
        aa, bb = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        r = feature_distance(aa, bb, wt)
        g0, g1 = torch.autograd.grad(r, [aa, bb], gout)
    assert g0.dtype == BF and g1.dtype == BF
    d, da, r0, a0, r1, a1 = distance64(a.double(), b.double(), wt, gout)
    what = "feature_distance C=%d weight=%s stacked=%s" % (c, weighted, stacked)
    check_sum(r.reshape(n), d, da, distance_forward_c(n, c, h * w), what + " value")
    k = distance_backward_k(c)
    check_once(g0, r0, a0, k, what + " g0")
    check_once(g1, r1, a1, k, what + " g1")


@pytest.mark.parametrize("shape", [(2, 64, 32, 32), (2, 256, 8, 4), (3, 192, 10, 6)])
def test_bias_relu_pool_bf16_forward_and_backward(shape):
    """y = RN(relu(raw + b)) (k = 1), pooled = the max of the STORED y, g_raw = RN([y > 0]*(g_y + [first max]*g_pooled))
    (k = 1) with the arg-max decided on the stored y."""
    from gangealing_b200.op.vgg_pool import bias_relu_pool
    n, c, h, w = shape
    g = seeded(c + h)
    raw = cl(randn(shape, g, BF)).requires_grad_(True)
    bias = randn((c,), g)
    gy = cl(randn(shape, g, BF))
    gp = cl(randn((n, c, h // 2, w // 2), g, BF))
    y, p = bias_relu_pool(raw, bias)
    pre = raw.detach().double() + bias.double()[:, None, None]
    check_once(y, torch.relu(pre), raw.detach().double().abs() + bias.double().abs()[:, None, None], 1,
               "bias_relu_pool y %s" % (shape,))
    y64 = y.detach().double()
    win = y64.reshape(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)
    assert torch.equal(p.double(), win.max(-1).values)
    (gr,) = torch.autograd.grad([y, p], [raw], [gy, gp])
    first = F.one_hot(win.argmax(-1), 4).double()           # torch.argmax returns the first maximal index
    first = first.reshape(n, c, h // 2, w // 2, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h, w)
    gpu = gp.double().repeat_interleave(2, 2).repeat_interleave(2, 3)
    ref = torch.where(y64 > 0, gy.double() + first * gpu, torch.zeros_like(y64))
    absr = torch.where(y64 > 0, gy.double().abs() + first * gpu.abs(), torch.zeros_like(y64))
    check_once(gr, ref, absr, 1, "bias_relu_pool g_raw %s" % (shape,))


# ================================================================================================ weight cast
def test_weight_scaler_bf16_products_are_rounded_once():
    """scale_cast_multi_kernel: RN_bf16(w*scale) from the fp32 master weight; the scale (times the gain) reaches the kernel
    as one fp32 value -> k = 2.  Sizes cover several 32768-element chunks, a tail that is not a multiple of 4, and two
    tensors in one launch."""
    from gangealing_b200.op.scaled_weights import WeightScaler
    g = seeded(5)
    mods = [torch.nn.Linear(1, 1, bias=False).to(DEV) for _ in range(3)]
    sizes = [(512, 300), (3, 7, 5), (64, 3, 3, 3)]
    for m, sz in zip(mods, sizes):
        m.weight = torch.nn.Parameter(randn(sz, g))
    scales = [1 / math.sqrt(300), 1 / math.sqrt(35), 1 / math.sqrt(27)]
    gains = [1.0, SQRT2, 1.0]
    scaler = WeightScaler(list(zip(mods, scales)))
    with scaler.step():
        for m, gn in zip(mods, gains):
            assert scaler.get(m, BF, gn) is None          # first sighting: learns the dtype
        outs = [scaler.get(m, BF, gn) for m, gn in zip(mods, gains)]
    for o, m, s, gn in zip(outs, mods, scales, gains):
        assert o is not None and o.dtype == BF
        ref = m.weight.detach().double() * (s * gn)
        check_once(o, ref, ref.abs(), 2, "WeightScaler %s" % (tuple(m.weight.shape),))


# ================================================================================================ NCHW half precision
HALF = [torch.float16, torch.bfloat16]
# whole planes, several per item | several bands | several bands, tall and narrow | generic kernel (out_w < 24) | vec_io off
NCHW_SHAPES = [(2, 16, 33, 33), (1, 4, 257, 257), (1, 2, 1030, 70), (2, 3, 20, 20), (2, 4, 31, 31)]


def _nchw_filter(kind):
    if kind == "sep":
        return (so.make_kernel([1, 3, 3, 1]) * 4).to(DEV)
    return torch.randn(3, 3, generator=torch.Generator().manual_seed(4)).to(DEV) / 3


def nchw_k(kernel):
    """NCHW FIR (fir4_band_kernel<T, -1> lane_strip: separable 9, otherwise one fma per tap; the generic kernel takes every
    tap of the window as an fma): at most max(9, taps)."""
    return max(9, kernel.numel())


def nchw_sum_c(m):
    """An fp32 reduction of m terms on the NCHW kernels: a thread's serial chain (at most m/32 terms), warp and CTA sums
    (5 + 8), a finish chain over the partials (at most m/32 + 5): bounded by 2*ceil(m/32) + 20."""
    return 2 * ceil_div(m, 32) + 20


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("shape", NCHW_SHAPES)
@pytest.mark.parametrize("kind", ["sep", "rand"])
def test_upfirdn2d_nchw_half(dtype, shape, kind):
    from gangealing_b200 import op
    g = seeded(shape[2] + shape[3])
    k = _nchw_filter(kind)
    x = randn(shape, g, dtype)
    y = op.upfirdn2d(x, k, pad=(1, 1))
    p4 = (1, 1, 1, 1)
    check_once(y, fir64(x.double(), k, p4), fir64(x.double().abs(), k.abs(), p4), nchw_k(k),
               "upfirdn2d %s %s %s" % (dtype, kind, shape))


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("shape", NCHW_SHAPES)
def test_blur_noise_bias_act_nchw_half(dtype, shape):
    """lrelu(rs*B(x) + b + nw*noise)*gain; the noise plane is stored in the activation's dtype.
    k = blur_k + the fma with rs, the fma with the noise, slope*gain, the product -> blur_k + 4."""
    from gangealing_b200 import op
    n, c, h, w = shape
    g = seeded(h + w + 1)
    k = _nchw_filter("sep")
    x = randn(shape, g, dtype)
    nz = randn((n, 1, h - 1, w - 1), g, dtype)
    nw = torch.tensor([0.3], device=DEV)
    b = randn((c,), g) * 0.5
    rs = torch.rand(n, c, generator=g, device=DEV) + 0.5
    y = op.blur_noise_bias_act(x, k, (1, 1), nz, nw, b, row_scale=rs)
    p4 = (1, 1, 1, 1)
    r64 = rs.double()[:, :, None, None]
    noise = nw.double() * nz.double()
    pre = r64 * fir64(x.double(), k, p4) + b.double()[:, None, None] + noise
    a = (r64 * fir64(x.double().abs(), k.abs(), p4) + b.double().abs()[:, None, None] + noise.abs()) * slope_gain(0.2, SQRT2)
    check_once(y, lrelu64(pre, 0.2, SQRT2), a, nchw_k(k) + 4, "blur_noise_bias_act %s %s" % (dtype, shape))


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("shape", [(2, 16, 33, 33), (2, 3, 20, 19), (1, 8, 64, 64)])
def test_elementwise_nchw_half(dtype, shape):
    """fused_leaky_relu forward (the bias is cast to the activation's dtype; + b, *slope, *gain: k = 3) and backward (gx:
    k = 2; grad_bias sums the STORED gx, like the reference's grad_input.sum()), noise_bias_act (k = 5) and channel_scale
    (out k = 1, row_dot one fma per pixel)."""
    from gangealing_b200 import op
    from gangealing_b200.op.modconv import channel_scale_raw
    n, c, h, w = shape
    g = seeded(h * w + c)
    x = randn(shape, g, dtype)
    b = randn((c,), g)
    gy = randn(shape, g, dtype)
    what = "%s %s" % (dtype, shape)
    xl, bl = x.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y = op.fused_leaky_relu(xl, bl)
    bq = b.to(dtype).double()[:, None, None]
    pre = x.double() + bq
    check_once(y, lrelu64(pre, 0.2, SQRT2), (x.double().abs() + bq.abs()) * slope_gain(0.2, SQRT2), 3, "fused_leaky_relu " + what)
    gx, gb = torch.autograd.grad(y, [xl, bl], gy)
    sl = torch.where(y.double() > 0, 1.0, 0.2) * SQRT2
    ref = gy.double() * sl
    check_once(gx, ref, ref.abs(), 2, "fused_leaky_relu gx " + what)
    check_sum(gb, gx.double().sum((0, 2, 3)), gx.double().abs().sum((0, 2, 3)), nchw_sum_c(n * h * w),
              "fused_leaky_relu grad_bias " + what)
    # noise + bias + leaky-ReLU with a row scale
    nz = randn((n, 1, h, w), g, dtype)
    nw = torch.tensor([0.7], device=DEV)
    rs = torch.rand(n, c, generator=g, device=DEV) + 0.5
    y = op.noise_bias_act(x, nz, nw, b, row_scale=rs)
    r64 = rs.double()[:, :, None, None]
    noise = nw.double() * nz.double()
    pre = x.double() * r64 + b.double()[:, None, None] + noise
    a = ((x.double() * r64).abs() + b.double().abs()[:, None, None] + noise.abs()) * slope_gain(0.2, SQRT2)
    check_once(y, lrelu64(pre, 0.2, SQRT2), a, 5, "noise_bias_act " + what)
    # channel scale with its row dot
    s = randn((n, c), g)
    out, dot = channel_scale_raw(x, s, y=gy)
    ref = x.double() * s.double()[:, :, None, None]
    check_once(out, ref, ref.abs(), 1, "channel_scale " + what)
    t = x.double() * gy.double()
    check_sum(dot, t.sum((2, 3)), t.abs().sum((2, 3)), nchw_sum_c(h * w), "channel_scale row_dot " + what)
