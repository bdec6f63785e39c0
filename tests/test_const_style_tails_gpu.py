"""The fused tails of layers whose styles are constants (every layer above the latent learner's inject index): they write a
sign mask instead of the activation, and their backward computes g_raw from (g_xs, mask) alone.  The route is chosen from
`requires_grad` of the latent rows a layer reads; everything it computes must equal the general route bit for bit."""
import dataclasses

import pytest
import torch

from gangealing_b200 import _lib
from styled_reference import bf16_tail_contract, dekink, inputs

DEV = "cuda"
CL = torch.channels_last
gpu = pytest.mark.gpu

# the launch plans of tests/test_styled_fused_gpu.py plus the benchmark's channel counts at 32^2 .. 256^2
SHAPES = [((2, 64, 16, 16), False, True, True), ((3, 512, 4, 4), False, True, True), ((2, 128, 40, 24), False, True, False),
          ((2, 256, 9, 7), False, False, True), ((2, 64, 17, 17), True, False, True), ((2, 128, 33, 41), True, False, True),
          ((1, 512, 9, 9), True, False, True), ((2, 512, 32, 32), False, True, True), ((2, 512, 65, 65), True, False, True),
          ((2, 256, 128, 128), False, True, True), ((1, 128, 257, 257), True, False, True),
          ((1, 128, 256, 256), False, True, False)]


def _unpack(mask, c):
    """(N, H, W, C/32) int32 words -> (N, C, H, W) bool."""
    bits = (mask.unsqueeze(-1) >> torch.arange(32, device=mask.device, dtype=torch.int32)) & 1       # (N, H, W, C/32, 32)
    return bits.reshape(*mask.shape[:3], c).permute(0, 3, 1, 2).bool()


def _tail_inputs(shape, blur, with_rgb, with_next, dtype, exact_zero):
    n, c, h, w = shape
    t = inputs(n, c, h, w, blur, with_rgb, with_next, seed=c + h)
    if exact_zero:      # every 8th channel is exactly 0 after the activation: raw = bias = 0 and no noise
        t["raw"][:, ::8] = 0
        t["bias"][::8] = 0
        t["noise"] = None
    d = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in t.items()}
    d["raw"] = d["raw"].to(dtype).contiguous(memory_format=CL)
    if d["g_xs"] is not None:
        d["g_xs"] = d["g_xs"].to(dtype).contiguous(memory_format=CL)
    return t, d


def _forward(d, blur, want_mask):
    from gangealing_b200.op import nhwc
    from oracle import stylegan2_ops as so
    if blur:
        k = (so.make_kernel([1, 3, 3, 1]) * 4).to(DEV)
        out, xs, _ = nhwc.blur(d["raw"], k, (1, 1, 1, 1), mode=1, noise=d["noise"], noise_weight=d["nw"], bias=d["bias"],
                               row_scale=d["demod"], scale2=d["s_next"], want_out=True, want_out2=True, negative_slope=0.2,
                               gain=2 ** 0.5, want_mask=want_mask)
        return out, xs, None
    return nhwc.styled_tail(d["raw"], d["noise"], d["nw"], d["bias"], d["demod"], d["s_next"], d["wm"], d["rgb_bias"], d["skip"],
                            True, 0.2, 2 ** 0.5, want_mask=want_mask)


@gpu
@pytest.mark.parametrize("exact_zero", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape,blur,with_rgb,with_next", SHAPES)
def test_mask_forward_equals_the_sign_of_the_general_routes_activation(shape, blur, with_rgb, with_next, dtype, exact_zero):
    _, d = _tail_inputs(shape, blur, with_rgb, with_next, dtype, exact_zero)
    out, xs, rgb = _forward(d, blur, False)
    mask, xs_m, rgb_m = _forward(d, blur, True)
    assert mask.dtype == torch.int32 and tuple(mask.shape) == (out.shape[0], out.shape[2], out.shape[3], out.shape[1] // 32)
    for a, b in ((xs, xs_m), (rgb, rgb_m)):
        assert (a is None) == (b is None)
        if a is not None:
            assert torch.equal(a, b)
    assert torch.equal(_unpack(mask, out.shape[1]), out > 0)
    if exact_zero:
        assert (out[:, ::8] == 0).all() and not _unpack(mask, out.shape[1])[:, ::8].any()


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape,blur,with_rgb,with_next", SHAPES)
def test_mask_backward_equals_the_general_kernels_bitwise(shape, blur, with_rgb, with_next, dtype):
    """g_raw (non-blur) / g_t (pass 1 of the blur layers) from (g_xs, mask) against the general kernel reading the stored
    activation with every reduction off."""
    from gangealing_b200.op import nhwc
    _, d = _tail_inputs(shape, blur, with_rgb, with_next, dtype, True)
    out, _, _ = _forward(d, blur, False)
    mask, _, _ = _forward(d, blur, True)
    demod, wm, g_rgb = (None, None, None) if blur else (d["demod"], d["wm"], d["g_rgb"])
    ref = nhwc.styled_tail_backward(d["g_xs"], g_rgb, out, None, d["s_next"], demod, wm, False, False, False, 0.2, 2 ** 0.5)[0]
    got = nhwc.styled_tail_backward_mask(d["g_xs"], g_rgb, mask, d["s_next"], demod, wm, 0.2, 2 ** 0.5, dtype)
    assert got.dtype == ref.dtype and got.is_contiguous(memory_format=CL) and torch.equal(got, ref)


def _fused(t, d, blur, grad_names):
    """fused_tail with `grad_names` requiring grad -> (xs, rgb, g_raw)."""
    from gangealing_b200.op.styled_fused import fused_tail
    from oracle import stylegan2_ops as so
    k = (so.make_kernel([1, 3, 3, 1]) * 4).to(DEV) if blur else None
    a = {nm: (d[nm].clone().requires_grad_(nm in grad_names) if d[nm] is not None else None)
         for nm in ("raw", "demod", "s_next", "wm", "skip")}
    xs, rgb = fused_tail(a["raw"], a["demod"], a["s_next"], a["wm"], a["skip"], d["noise"], d["nw"], d["bias"], d["rgb_bias"],
                         kernel=k, pad=(1, 1) if blur else None)
    outs = [(o, g) for o, g in ((xs, d["g_xs"]), (rgb, d["g_rgb"])) if o is not None]
    g_raw, = torch.autograd.grad([o for o, _ in outs], [a["raw"]], [g for _, g in outs])
    return xs, rgb, g_raw


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape,blur,with_rgb,with_next", SHAPES)
def test_fused_tail_with_constant_styles_equals_the_general_route(shape, blur, with_rgb, with_next, dtype, monkeypatch):
    """Through autograd: only `raw` requires grad (sign-mask route) vs every input requiring grad (general route)."""
    from gangealing_b200.op import nhwc
    t, d = _tail_inputs(shape, blur, with_rgb, with_next, dtype, False)
    calls = []
    real = nhwc.styled_tail_backward_mask
    monkeypatch.setattr(nhwc, "styled_tail_backward_mask", lambda *a: calls.append(1) or real(*a))
    xs_m, rgb_m, g_m = _fused(t, d, blur, ("raw",))
    assert calls, "the sign-mask route was not taken"
    del calls[:]
    xs, rgb, g = _fused(t, d, blur, ("raw", "demod", "s_next", "wm"))
    assert not calls
    for a, b in ((xs, xs_m), (rgb, rgb_m), (g, g_m)):
        assert (a is None) == (b is None)
        if a is not None:
            assert a.dtype == b.dtype and torch.equal(a, b)


@gpu
@pytest.mark.parametrize("shape,blur,with_rgb,with_next", SHAPES[:7])
def test_sign_mask_route_meets_the_bf16_storage_contract(shape, blur, with_rgb, with_next):
    """The general route's float64 contract (bf16_tail_contract: each stored value rounded once) on the sign-mask route."""
    t = dekink(inputs(*shape, blur, with_rgb, with_next, seed=shape[1] + shape[2]), blur, torch.bfloat16)
    d = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in t.items()}
    d["raw"] = d["raw"].to(torch.bfloat16).contiguous(memory_format=CL)
    if d["g_xs"] is not None:
        d["g_xs"] = d["g_xs"].to(torch.bfloat16).contiguous(memory_format=CL)
    xs, rgb, g_raw = _fused(t, d, blur, ("raw",))
    bf16_tail_contract(t, blur, xs, rgb, {"raw": g_raw})


def test_argument_validation_of_the_sign_mask_entry_points():
    dll = _lib.load()
    one = 1     # any non-null pointer value: validation must reject these calls before dereferencing anything
    st = [None] * 8
    assert dll.gg_styled_tail_mask_nhwc(one, None, None, one, *st, 0, 3, 0.2, 1.0, 1, 20, 16, None) == -2     # C % 32
    assert dll.gg_styled_tail_mask_nhwc(one, None, None, one, *st, 2, 3, 0.2, 1.0, 1, 32, 16, None) == -2     # bf16: C % 64
    assert dll.gg_styled_tail_mask_nhwc(None, one, None, one, None, None, None, None, one, None, None, None,
                                        0, 3, 0.2, 1.0, 1, 32, 16, None) == -1                                # no mask
    assert b"mask" in dll.gg_last_error()
    assert dll.gg_styled_tail_mask_nhwc(one, one, None, one, *st, 0, 3, 0.2, 1.0, 1, 32, 16, None) == -1      # xs without s_next
    assert dll.gg_styled_tail_mask_nhwc(one, None, None, one, *st, 0, 2, 0.2, 1.0, 1, 32, 16, None) == -2     # act
    tail = [0, 0.2, 1.0, 1, 32, 16, None]       # dtype, alpha, scale, N, C, HW, stream
    assert dll.gg_styled_tail_backward_mask_nhwc(one, None, None, one, None, None, None, *tail) == -1         # no upstream gradient
    assert dll.gg_styled_tail_backward_mask_nhwc(one, one, None, one, None, None, None, *tail) == -1          # g_xs without s_next
    assert dll.gg_styled_tail_backward_mask_nhwc(one, None, one, one, None, None, None, *tail) == -1          # g_rgb without wm
    assert dll.gg_styled_tail_backward_mask_nhwc(one, one, None, None, one, None, None, *tail) == -1          # no mask
    assert dll.gg_styled_tail_backward_mask_nhwc(one, one, None, one, one, None, None, 0, 0.2, 1.0, 1, 48, 16, None) == -2   # C % 32
    assert dll.gg_styled_tail_backward_mask_nhwc(one, one, None, one, one, None, None, 1, 0.2, 1.0, 1, 32, 16, None) == -2   # fp16
    blur = [0, 1, 32, 8, 8, 4, 4, 1, 1, 1, 1, 1, 3, 0.2, 1.0, None]   # dtype, N, C, h, w, kh, kw, sep, pads, act, alpha, scale, stream
    ptrs = [one, None, one, one] + [None] * 5
    assert dll.gg_blur_nhwc_mask(*ptrs, 0, 1, 20, *blur[3:]) == -2                                           # C % 32
    assert dll.gg_blur_nhwc_mask(*ptrs, 2, 1, 32, *blur[3:]) == -2                                           # bf16: C % 64
    assert dll.gg_blur_nhwc_mask(*ptrs, 0, 1, 32, 8, 8, 5, 5, *blur[7:]) == -2                               # filter > 4x4
    assert dll.gg_blur_nhwc_mask(*ptrs, *blur[:12], 2, 0.2, 1.0, None) == -2                                 # act
    assert dll.gg_blur_nhwc_mask(None, None, one, one, *([None] * 5), *blur) == -1                           # no mask
    assert dll.gg_blur_nhwc_mask(one, one, one, one, *([None] * 5), *blur) == -1                             # out2 without scale2


def test_two_part_latent_marks_the_constant_styles_and_keeps_the_gradient():
    """CPU, oracle op set: the generator's two-latent call equals the one-tensor call (image and d loss / d coefficients),
    and the styles read from the constant part do not require grad."""
    from gangealing_b200.op import style_path
    from gangealing_b200.stylegan2 import Generator
    from gangealing_b200.training import DirectionInterpolator
    from oracle import opset
    g = opset.fill_parameters(Generator(64, 64, 2, channel_multiplier=1, ops=opset.cpu_ops()).eval(), 11)
    for prm in g.parameters():
        prm.requires_grad = False
    inject = 3
    ll = DirectionInterpolator(None, 2, inject, g.n_latent, num_heads=2, dim_latent=64)
    opset.fill_parameters(ll, 13, gain=0.5)
    w = torch.randn(3, 64, generator=torch.Generator().manual_seed(2))
    noise = [getattr(g.noises, "noise_%d" % i) for i in range(g.num_layers)]
    one = ll([w], psi=0.6)
    two = ll([w], psi=0.6, split=True)
    assert len(one) == 1 and tuple(one[0].shape) == (6, g.n_latent, 64)
    assert two[0].requires_grad and not two[1].requires_grad
    img1, lat1 = g(one, input_is_latent=True, noise=noise, return_latents=True)
    img2, lat2 = g(two, input_is_latent=True, inject_index=inject, noise=noise, return_latents=True)
    assert torch.equal(lat1, lat2) and torch.equal(img1, img2)
    g1, = torch.autograd.grad(img1.square().mean(), [ll.coefficients])
    g2, = torch.autograd.grad(img2.square().mean(), [ll.coefficients])
    assert torch.equal(g1, g2) and g1.abs().max() > 0
    layers, rgbs = [g.conv1] + list(g.convs), [g.to_rgb1] + list(g.to_rgbs)
    conv_idx, rgb_idx = list(range(len(layers))), [2 * r + 1 for r in range(len(rgbs))]
    rows = [True] * inject + [False] * (g.n_latent - inject)
    styles, rgb_styles = style_path.all_styles(g, lat2, layers, rgbs, conv_idx, rgb_idx, rows)
    plain, plain_rgb = style_path.all_styles(g, lat2, layers, rgbs, conv_idx, rgb_idx)
    for got, ref, idx in ((styles, plain, conv_idx), (rgb_styles, plain_rgb, rgb_idx)):
        for s, p, row in zip(got, ref, idx):
            assert torch.equal(s, p) and p.requires_grad and s.requires_grad == (row < inject)


def _one_tensor_pairs(generator, ll, resize_fake2stn, psi, batch, dim_latent, freeze_ll, device, z=None):
    """sample_gan_supervised_pairs with the reference-shaped one-tensor latent call: every style requires grad."""
    with torch.set_grad_enabled(not freeze_ll):
        unaligned_in, w_noise = generator([z], noise=None, return_latents=True)
        aligned_target, _ = generator(ll([w_noise[:, 0, :]], psi=psi), input_is_latent=True, noise=None)
    return unaligned_in, resize_fake2stn(aligned_target)


@gpu
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_training_step_equals_the_one_tensor_latent_step_bitwise(dtype, monkeypatch):
    """One Trainer step (batch 4) on the sign-mask route vs the same step with every style requiring grad: losses and every
    updated parameter bitwise equal; the step then replays from a CUDA graph."""
    from gangealing_b200.op import nhwc
    from gangealing_b200.training import losses
    from gangealing_b200.training.step import TrainConfig, Trainer
    old = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    try:
        cfg = TrainConfig(gen_size=128, flow_size=64, dim_latent=64, n_mlp=2, batch=4, inject=3, gen_channel_multiplier=1,
                          stn_channel_multiplier=0.5, dtype=dtype, seed=4)
        new, ref = Trainer(cfg, DEV), Trainer(dataclasses.replace(cfg), DEV)
        z = torch.randn(cfg.batch, cfg.dim_latent, generator=torch.Generator().manual_seed(11)).to(DEV)
        calls = []
        real = nhwc.styled_tail_backward_mask
        monkeypatch.setattr(nhwc, "styled_tail_backward_mask", lambda *a: calls.append(1) or real(*a))
        torch.manual_seed(100)
        out_new = new.step(z=z)
        n_layers = len(new.generator.convs) + 1
        assert len(calls) == n_layers - cfg.inject, "layers %d.. of %d should run on the sign-mask route" % (cfg.inject, n_layers)
        del calls[:]
        monkeypatch.setattr(losses, "sample_gan_supervised_pairs", _one_tensor_pairs)
        torch.manual_seed(100)
        out_ref = ref.step(z=z)
        assert not calls
        monkeypatch.undo()
        torch.cuda.synchronize()
        for k in out_ref:
            assert torch.equal(out_new[k], out_ref[k]), "loss %s differs" % k
        for name, ma, mb in (("stn", new.t_module, ref.t_module), ("stn_ema", new.t_ema, ref.t_ema),
                             ("latent_learner", new.ll_module, ref.ll_module)):
            for (k, pa), (_, pb) in zip(ma.named_parameters(), mb.named_parameters()):
                assert torch.equal(pa, pb), "%s.%s differs" % (name, k)
        new.capture(warmup=2)
        out = new.step()
        torch.cuda.synchronize()
        assert all(torch.isfinite(v) for v in out.values())
    finally:
        torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = old
