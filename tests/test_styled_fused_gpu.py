"""GPU parity of the cross-layer fused StyledConv / ToRGB tails (csrc/styled.cu, csrc/nhwc.cu modes 1-2, op/styled_fused.py)
against the CPU oracle -- forward, every gradient, fp32 and bf16 storage, including the benchmark's 257^2 -> 256^2 layer."""
import pytest
import torch

from conftest import assert_close
from fp64_contract import BF16, check_once, check_sum, fir64, library, rowwise_c
from oracle import opset
from oracle import stylegan2_ops as so
from styled_reference import bf16_tail_contract, dekink, inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
CL = torch.channels_last


def _oracle_tail(raw, demod, s_next, wm, skip, noise, nw, bias, rgb_bias, kernel, pad, slope=0.2, gain=2 ** 0.5):
    """Reference formulation: [Blur] -> demodulate -> NoiseInjection -> FusedLeakyReLU (networks.py:266,291-298,346-348);
    next layer's modulation (networks.py:236,243); ToRGB 1x1 modulated conv + bias + skip (networks.py:389-405)."""
    if kernel is not None:
        o = so.blur_noise_bias_act_ref(raw, kernel, pad, noise, nw, bias, negative_slope=slope, scale=gain, row_scale=demod)
    else:
        o = so.noise_bias_act_ref(raw * demod[:, :, None, None], noise, nw, bias, negative_slope=slope, scale=gain)
    xs = o * s_next[:, :, None, None] if s_next is not None else None
    rgb = None
    if wm is not None:
        rgb = torch.einsum("noc,nchw->nohw", wm, o) + rgb_bias.reshape(1, 3, 1, 1)
        if skip is not None:
            rgb = rgb + skip
    return xs, rgb


def _run_both(t, blur, dtype, slope=0.2):
    from gangealing_b200.op.styled_fused import fused_tail
    k = so.make_kernel([1, 3, 3, 1]) * 4 if blur else None
    pad = (1, 1) if blur else None
    names = [nm for nm in ("raw", "demod", "s_next", "wm", "skip") if t[nm] is not None]
    # storage rounding is part of the input: the oracle sees the same (bf16-representable) activation values
    raw_q = t["raw"].to(dtype).float()
    lo = {nm: (raw_q if nm == "raw" else t[nm]).clone().requires_grad_(True) for nm in names}
    xs_o, rgb_o = _oracle_tail(lo["raw"], lo["demod"], lo.get("s_next"), lo.get("wm"), lo.get("skip"), t["noise"], t["nw"],
                               t["bias"], t["rgb_bias"], k, pad, slope)
    outs_o = [v for v in (xs_o, rgb_o) if v is not None]
    gouts = [v for v in (t["g_xs"].to(dtype).float() if t["g_xs"] is not None else None, t["g_rgb"]) if v is not None]
    grads_o = torch.autograd.grad(outs_o, [lo[nm] for nm in names], gouts)
    lg = {nm: (t[nm].to(DEV).to(dtype).contiguous(memory_format=CL) if nm == "raw" else t[nm].to(DEV)).requires_grad_(True)
          for nm in names}
    xs, rgb = fused_tail(lg["raw"], lg["demod"], lg.get("s_next"), lg.get("wm"), lg.get("skip"), t["noise"].to(DEV), t["nw"].to(DEV),
                         t["bias"].to(DEV), t["rgb_bias"].to(DEV) if t["rgb_bias"] is not None else None,
                         kernel=k.to(DEV) if blur else None, pad=pad, negative_slope=slope)
    outs = [v for v in (xs, rgb) if v is not None]
    gd = [(g.to(DEV).to(o.dtype).contiguous(memory_format=CL) if o.dim() == 4 and o.shape[1] != 3 else g.to(DEV))
          for g, o in zip(gouts, outs)]
    grads = torch.autograd.grad(outs, [lg[nm] for nm in names], gd)
    return (xs_o, rgb_o, dict(zip(names, grads_o))), (xs, rgb, dict(zip(names, grads)))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape,blur,with_rgb,with_next", [
    ((2, 64, 16, 16), False, True, True), ((3, 512, 4, 4), False, True, True), ((2, 128, 40, 24), False, True, False),
    ((2, 256, 9, 7), False, False, True), ((2, 64, 17, 17), True, False, True), ((2, 128, 33, 41), True, False, True),
    ((1, 512, 9, 9), True, False, True)])
def test_fused_tail_forward_and_all_gradients_vs_oracle(shape, blur, with_rgb, with_next, dtype):
    t = dekink(inputs(*shape, blur, with_rgb, with_next, seed=shape[1] + shape[2]), blur, dtype)
    (xs_o, rgb_o, go), (xs, rgb, gg) = _run_both(t, blur, dtype)
    if xs_o is not None:
        assert xs.dtype == dtype and xs.is_contiguous(memory_format=CL)
    if rgb_o is not None:
        assert rgb.dtype == torch.float32
    if dtype == torch.bfloat16:   # each stored value rounded once, each fp32 sum at fp32 accuracy (against float64)
        bf16_tail_contract(t, blur, xs, rgb, gg)
        return
    if xs_o is not None:
        assert_close(xs, xs_o, rtol=1e-5, what="xs (next conv input)")
    if rgb_o is not None:
        assert_close(rgb, rgb_o, rtol=1e-5, what="rgb")
    for nm in go:
        tol = {"raw": 1e-5, "demod": 2e-4, "s_next": 2e-4, "wm": 2e-4, "skip": 1e-6}[nm]
        assert_close(gg[nm], go[nm], rtol=tol, what="grad " + nm)


@pytest.mark.parametrize("blur", [False, True])
def test_fused_tail_at_the_benchmark_layer_vs_oracle(blur):
    """(2, 128, 257, 257) -> 256^2 (blur tail) and (2, 128, 256, 256) (conv tail + to-RGB, the last layer): the fused
    kernels against the CPU oracle directly.  Leaky-ReLU flips slope where the pre-activation is within rounding of zero,
    so the full-tensor comparison uses slope 1 (the linear pre-activation: every other term of the kernel is exercised) and
    the activated output is compared wherever |pre-activation| exceeds the rounding noise."""
    n, c, h = 2, 128, 257 if blur else 256
    t = inputs(n, c, h, h, blur, not blur, True, seed=99)
    (xs_o, rgb_o, go), (xs, rgb, gg) = _run_both(t, blur, torch.float32, slope=1.0)
    assert_close(xs, xs_o, rtol=1e-5, what="linear xs")
    if rgb_o is not None:
        assert_close(rgb, rgb_o, rtol=1e-5, what="linear rgb")
    for nm in go:
        assert_close(gg[nm], go[nm], rtol=3e-4 if nm != "raw" else 1e-5, what="linear grad " + nm)
    (xs_o, rgb_o, _), (xs, rgb, _) = _run_both(t, blur, torch.float32, slope=0.2)
    pre = xs_o / t["s_next"][:, :, None, None]
    safe = (pre.abs() > 1e-4).to(DEV)
    err = ((xs.float() - xs_o.to(DEV)).abs() * safe).max().item()
    assert err <= 1e-5 * xs_o.abs().max().item(), err
    assert safe.float().mean().item() > 0.999


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-3), (torch.bfloat16, 4e-2)])
def test_generator_fused_synthesis_matches_cpu_oracle(dtype, tol):
    """Whole synthesis network: cross-layer fused path (channels-last, fp32 / bf16 storage) vs the reference formulation
    (grouped per-sample filters) on the CPU oracle -- image and the gradient w.r.t. the latent."""
    from gangealing_b200.stylegan2 import Generator
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        torch.manual_seed(0)
        g_cpu = Generator(64, 64, 2, channel_multiplier=2, ops=opset.cpu_ops()).eval()
        opset.fill_parameters(g_cpu, 4)
        g_gpu = Generator(64, 64, 2, channel_multiplier=2).eval()
        g_gpu.load_state_dict(g_cpu.state_dict())
        g_gpu.to(DEV)
        for m in (g_cpu, g_gpu):
            for p in m.parameters():
                p.requires_grad = False
        g_gpu.channels_last, g_gpu.act_dtype = True, dtype
        noise = g_cpu.make_noise(2)
        w = torch.randn(2, g_cpu.n_latent, 64) * 0.7
        go = torch.randn(2, 3, 64, 64)
        wc = w.clone().requires_grad_(True)
        img_c, _ = g_cpu([wc], input_is_latent=True, noise=noise)
        (gw_c,) = torch.autograd.grad(img_c, wc, go)
        wg = w.to(DEV).requires_grad_(True)
        from gangealing_b200.op import styled_fused
        assert styled_fused.fusable(g_gpu, wg, dtype)
        img_g, _ = g_gpu([wg], input_is_latent=True, noise=[x.to(DEV) for x in noise])
        (gw_g,) = torch.autograd.grad(img_g, wg, go.to(DEV))
        assert img_g.dtype == torch.float32
        assert_close(img_g, img_c, rtol=tol, what="image")
        assert_close(gw_g, gw_c, rtol=tol * 2, what="latent gradient")
        # the layer-by-layer path (round 1's) computes the same thing
        g_gpu.fuse_synthesis = False
        if dtype == torch.float32:
            img_u, _ = g_gpu([wg], input_is_latent=True, noise=[x.to(DEV) for x in noise])
            assert_close(img_u, img_c, rtol=tol, what="unfused image")
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_channels_last_family_in_both_storage_types(dtype):
    """blur / fused_leaky_relu (forward + backward with bias gradient) / channel_scale on channels-last fp32 and bf16.
    bf16: the storage contract against float64 (tests/test_bf16_storage_gpu.py) -- k / c stated at each check."""
    from gangealing_b200 import op
    from gangealing_b200.op.modconv import channel_scale
    g = torch.Generator().manual_seed(7)
    lo = dtype == torch.bfloat16
    x = torch.randn(2, 128, 33, 29, generator=g)
    xq = x.to(dtype).float()
    b = torch.randn(128, generator=g)
    s = torch.randn(2, 128, generator=g)
    go = torch.randn(2, 128, 33, 29, generator=g).to(dtype).float()
    k = so.make_kernel([1, 3, 3, 1])
    xg = x.to(DEV).to(dtype).contiguous(memory_format=CL)
    x64, go64 = xq.double().to(DEV), go.double().to(DEV)
    n, c, hw = 2, 128, 33 * 29
    y = op.upfirdn2d(xg, k.to(DEV), pad=(2, 1))
    assert y.dtype == dtype and y.is_contiguous(memory_format=CL)
    if lo:   # separable blur: 9 roundings
        check_once(y, fir64(x64, k.to(DEV), (2, 1, 2, 1)), fir64(x64.abs(), k.to(DEV), (2, 1, 2, 1)), 9, "blur")
    else:
        assert_close(y, so.upfirdn2d_ref(xq, k, pad=(2, 1)), rtol=1e-5, what="blur")
    lo_ = [xq.clone().requires_grad_(True), b.clone().requires_grad_(True)]
    yo = so.fused_leaky_relu_ref(lo_[0], lo_[1])
    gxo, gbo = torch.autograd.grad(yo, lo_, go)
    lg = [xg.clone().requires_grad_(True), b.to(DEV).requires_grad_(True)]
    yg = op.fused_leaky_relu(lg[0], lg[1])
    assert yg.dtype == dtype and yg.is_contiguous(memory_format=CL)
    gx, gb = torch.autograd.grad(yg, lg, go.to(DEV).to(dtype).contiguous(memory_format=CL))
    if lo:
        pre = x64 + b.double().to(DEV)[:, None, None]
        sl = torch.where(pre > 0, 1.0, 0.2) * 2 ** 0.5
        check_once(yg, pre * sl, (x64.abs() + b.double().to(DEV).abs()[:, None, None]) * 2 ** 0.5, 5, "fused_leaky_relu")
        sl = torch.where(yg.double() > 0, 1.0, 0.2) * 2 ** 0.5   # the backward's slope: the sign of the stored output
        check_once(gx, go64 * sl, (go64 * sl).abs(), 2, "flr grad x")
        check_sum(gb, (go64 * sl).sum((0, 2, 3)), (go64 * sl).abs().sum((0, 2, 3)),
                  rowwise_c(n, c, hw, 2, False, BF16, library().sm_count()), "flr grad bias")
    else:
        assert_close(yg, yo, rtol=1e-6, what="fused_leaky_relu")
        assert_close(gx, gxo, rtol=1e-6, what="flr grad x")
        assert_close(gb, gbo, rtol=2e-4, what="flr grad bias")
    lo_ = [xq.clone().requires_grad_(True), s.clone().requires_grad_(True)]
    yo = lo_[0] * lo_[1][:, :, None, None]
    gxo, gso = torch.autograd.grad(yo, lo_, go)
    lg = [xg.clone().requires_grad_(True), s.to(DEV).requires_grad_(True)]
    yg = channel_scale(lg[0], lg[1])
    gx, gs = torch.autograd.grad(yg, lg, go.to(DEV).to(dtype).contiguous(memory_format=CL))
    if lo:
        s64 = s.double().to(DEV)[:, :, None, None]
        check_once(yg, x64 * s64, (x64 * s64).abs(), 1, "channel_scale")
        check_once(gx, go64 * s64, (go64 * s64).abs(), 1, "channel_scale grad x")
        check_sum(gs, (go64 * x64).sum((2, 3)), (go64 * x64).abs().sum((2, 3)),
                  rowwise_c(n, c, hw, 0, True, BF16, library().sm_count()), "channel_scale grad s")
    else:
        assert_close(yg, yo, rtol=1e-6, what="channel_scale")
        assert_close(gx, gxo, rtol=1e-6, what="channel_scale grad x")
        assert_close(gs, gso, rtol=2e-4, what="channel_scale grad s")
