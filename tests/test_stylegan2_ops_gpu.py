"""GPU parity: the sm_90a ops (through the C ABI) vs the oracle and the reference-generated fixtures.
Tolerance: 1e-3 relative fp32 (BASELINE.json north_star); low-precision dtypes use their own epsilon."""
import pytest
import torch

from conftest import assert_close, golden_cases, load_golden
from demod_reference import DEMOD_CASES, DEMOD_RTOL, demod_inputs, demod_ref, max_rel_err
from oracle import stylegan2_ops as so

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops():
    from gangealing_b200 import op
    return op


# ------------------------------------------------------------------------------------------------ upfirdn2d
def test_upfirdn2d_golden_fixtures():
    op = _ops()
    blob = load_golden("upfirdn2d")
    for name in golden_cases(blob):
        up, down, p0, p1 = [int(v) for v in blob[name + ".cfg"]]
        y = op.upfirdn2d(blob[name + ".x"].to(DEV), blob[name + ".k"].to(DEV), up=up, down=down, pad=(p0, p1))
        assert_close(y, blob[name + ".y"], rtol=1e-4, what=name)


HOT_SHAPES = [  # (N, C, H_in, W_in), pad -- SURVEY.md Appendix A tuples
    ((2, 128, 257, 257), (1, 1)), ((2, 256, 129, 129), (1, 1)), ((2, 512, 65, 65), (1, 1)),
    ((2, 512, 33, 33), (1, 1)), ((2, 512, 17, 17), (1, 1)), ((3, 512, 9, 9), (1, 1)),
    ((2, 64, 128, 128), (2, 2)), ((2, 64, 128, 128), (1, 1)), ((2, 128, 64, 64), (2, 2)),
    ((2, 512, 32, 32), (1, 1)), ((2, 512, 16, 16), (2, 2)), ((2, 512, 8, 8), (1, 1)),
    ((2, 128, 256, 256), (2, 2)),  # backward of the 256^2 blur (g_pad = (2, 2))
    ((1, 3, 450, 450), (2, 1)), ((1, 2, 1030, 70), (2, 2)), ((1, 1, 40, 3000), (1, 1)),
]


@pytest.mark.parametrize("shape,pad", HOT_SHAPES)
def test_upfirdn2d_blur_hot_shapes(shape, pad):
    op = _ops()
    g = torch.Generator().manual_seed(hash((shape, pad)) % 1000)
    x = torch.randn(*shape, generator=g)
    k = so.make_kernel([1, 3, 3, 1]) * 4
    y = op.upfirdn2d(x.to(DEV), k.to(DEV), pad=pad)
    assert_close(y, so.upfirdn2d_ref(x, k, pad=pad), rtol=1e-4, what=str(shape))


@pytest.mark.parametrize("up,down,pad,shape", [(2, 1, (2, 1), (2, 3, 128, 128)), (1, 2, (1, 1), (2, 3, 256, 256)),
                                               (2, 1, (2, 1), (5, 3, 4, 4)), (1, 2, (1, 1), (2, 16, 64, 64)),
                                               (3, 2, (4, 3), (1, 2, 31, 17))])
def test_upfirdn2d_resampling_modes(up, down, pad, shape):
    op = _ops()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(*shape, generator=g)
    k = so.make_kernel([1, 3, 3, 1]) * (up ** 2)
    y = op.upfirdn2d(x.to(DEV), k.to(DEV), up=up, down=down, pad=pad)
    assert_close(y, so.upfirdn2d_ref(x, k, up=up, down=down, pad=pad), rtol=1e-4)


@pytest.mark.parametrize("dtype,tol", [(torch.float16, 2e-3), (torch.bfloat16, 1.6e-2)])
def test_upfirdn2d_low_precision(dtype, tol):
    op = _ops()
    g = torch.Generator().manual_seed(3)
    k = so.make_kernel([1, 3, 3, 1])
    for shape, pad in [((2, 8, 65, 65), (1, 1)), ((1, 4, 128, 128), (2, 2)), ((2, 3, 33, 31), (2, 1))]:
        x = torch.randn(*shape, generator=g).to(dtype)
        y = op.upfirdn2d(x.to(DEV), k.to(DEV), pad=pad)
        assert y.dtype == dtype
        assert_close(y, so.upfirdn2d_ref(x.float(), k, pad=pad), rtol=tol, what=str(dtype))
    x = torch.randn(2, 3, 16, 16, generator=g).to(dtype)
    y = op.upfirdn2d(x.to(DEV), (k * 4).to(DEV), up=2, pad=(2, 1))
    assert_close(y, so.upfirdn2d_ref(x.float(), k * 4, up=2, pad=(2, 1)), rtol=tol)


@pytest.mark.parametrize("up,down,pad,shape", [(1, 1, (1, 1), (2, 4, 33, 33)), (1, 1, (2, 2), (1, 3, 64, 64)),
                                               (2, 1, (2, 1), (2, 3, 16, 16)), (1, 2, (1, 1), (1, 2, 32, 32))])
def test_upfirdn2d_autograd_first_and_second_order(up, down, pad, shape):
    op = _ops()
    g = torch.Generator().manual_seed(11)
    k = so.make_kernel([1, 3, 3, 1]) * (up ** 2)
    x = torch.randn(*shape, generator=g)
    xo = x.clone().requires_grad_(True)
    yo = so.upfirdn2d_ref(xo, k, up=up, down=down, pad=pad)
    w = torch.randn(yo.shape, generator=g)
    (gxo,) = torch.autograd.grad((yo * w).sum(), xo, create_graph=True)
    v = torch.randn(x.shape, generator=g)
    (ggo,) = torch.autograd.grad((gxo * v).sum(), xo, allow_unused=True)
    # ours
    xg = x.to(DEV).requires_grad_(True)
    wg = w.to(DEV).requires_grad_(True)
    yg = op.upfirdn2d(xg, k.to(DEV), up=up, down=down, pad=pad)
    (gxg,) = torch.autograd.grad((yg * wg).sum(), xg, create_graph=True)
    assert_close(gxg, gxo, rtol=1e-4, what="grad")
    # second order: d/dw of <grad_x, v> = upfirdn2d(v) (the op is linear, so d/dx is zero)
    (gwg,) = torch.autograd.grad((gxg * v.to(DEV)).sum(), wg)
    assert_close(gwg, so.upfirdn2d_ref(v, k, up=up, down=down, pad=pad), rtol=1e-4, what="gradgrad")
    assert ggo is None or ggo.abs().max() == 0


def test_upfirdn2d_properties_full_size():
    """BASELINE config-2 size (per-GPU batch 5, 256^2 layer): linearity + unit DC gain, no oracle needed."""
    op = _ops()
    k = (so.make_kernel([1, 3, 3, 1]) * 4).to(DEV)
    a = torch.randn(5, 128, 257, 257, device=DEV)
    b = torch.randn(5, 128, 257, 257, device=DEV)
    ya, yb = op.upfirdn2d(a, k, pad=(1, 1)), op.upfirdn2d(b, k, pad=(1, 1))
    yc = op.upfirdn2d(0.5 * a - 2 * b, k, pad=(1, 1))
    assert_close(yc, 0.5 * ya - 2 * yb, rtol=1e-5, what="linearity")
    ones = torch.ones(5, 128, 257, 257, device=DEV)
    y1 = op.upfirdn2d(ones, k, pad=(1, 1))
    assert y1.shape == (5, 128, 256, 256)
    assert_close(y1[:, :, 2:-2, 2:-2], torch.full((5, 128, 252, 252), 4.0), rtol=1e-6, what="dc gain")
    # adjoint identity <Ax, y> == <x, A^T y>  (A^T = the op's own backward)
    x = a.requires_grad_(True)
    y = op.upfirdn2d(x, k, pad=(1, 1))
    w = torch.randn_like(y)
    (gx,) = torch.autograd.grad((y * w).sum(), x)
    lhs = (y.detach().double() * w.double()).sum()
    rhs = (x.detach().double() * gx.double()).sum()
    # fp32 outputs: the two sums differ by rounding noise ~ eps * sum|terms|, not eps * |sum| (the terms cancel)
    assert abs(lhs - rhs) <= 1e-6 * (y.detach().double() * w.double()).abs().sum()


def test_upfirdn2d_errors():
    op = _ops()
    k = so.make_kernel([1, 3, 3, 1]).to(DEV)
    with pytest.raises(RuntimeError):
        op.upfirdn2d(torch.zeros(1, 1, 2, 2, device=DEV), k, pad=(0, 0))  # filter larger than input
    with pytest.raises(RuntimeError):
        op.upfirdn2d(torch.zeros(4, 4, device=DEV), k)
    with pytest.raises(RuntimeError):
        op.upfirdn2d(torch.zeros(1, 1, 8, 8, device=DEV, dtype=torch.float64), k)
    y = op.upfirdn2d(torch.zeros(0, 3, 8, 8, device=DEV), k, pad=(2, 1))  # empty batch is fine
    assert y.shape == (0, 3, 8, 8)


# ------------------------------------------------------------------------------------------------ fused_bias_act
def test_fused_leaky_relu_golden_fixtures():
    op = _ops()
    blob = load_golden("fused_act")
    for name in golden_cases(blob):
        x = blob[name + ".x"].to(DEV).requires_grad_(True)
        b = blob[name + ".b"].to(DEV).requires_grad_(True)
        y = op.fused_leaky_relu(x, b)
        assert_close(y, blob[name + ".y"], rtol=1e-5, what=name + " fwd")
        gx, gb = torch.autograd.grad(y, [x, b], blob[name + ".g"].to(DEV))
        assert_close(gx, blob[name + ".gx"], rtol=1e-5, what=name + " gx")
        assert_close(gb, blob[name + ".gb"], rtol=1e-4, what=name + " gb")


@pytest.mark.parametrize("shape", [(5, 128, 64, 64), (2, 512, 4, 4), (3, 512), (2, 7, 33, 31), (1, 3, 1, 1),
                                   (2, 64, 128, 128), (2, 5, 100, 100)])
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-5), (torch.float16, 2e-3), (torch.bfloat16, 1.6e-2)])
def test_fused_leaky_relu_shapes_dtypes(shape, dtype, tol):
    op = _ops()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(*shape, generator=g).to(dtype)
    b = torch.randn(shape[1], generator=g).to(dtype)
    go = torch.randn(*shape, generator=g).to(dtype)
    xg, bg = x.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
    y = op.fused_leaky_relu(xg, bg, 0.1, 1.5)
    yo = so.fused_leaky_relu_ref(x.float(), b.float(), 0.1, 1.5)
    assert y.dtype == dtype
    assert_close(y, yo, rtol=tol, what="fwd")
    gx, gb = torch.autograd.grad(y, [xg, bg], go.to(DEV))
    # backward is defined on the STORED output (ref = out), like the reference
    gxo, gbo = so.fused_leaky_relu_backward_ref(go.float(), y.detach().float().cpu(), 0.1, 1.5)
    assert_close(gx, gxo, rtol=tol, what="gx")
    n_red = x.numel() // shape[1]
    assert_close(gb, gbo, rtol=max(tol, 1e-4) * (n_red ** 0.5 if dtype != torch.float32 else 1), what="gb")


def test_fused_bias_act_raw_table_and_double_backward():
    from gangealing_b200.op.fused_act import fused_bias_act_raw
    op = _ops()
    g = torch.Generator().manual_seed(9)
    x = torch.randn(3, 6, 5, 7, generator=g)
    b = torch.randn(6, generator=g)
    r = torch.randn(3, 6, 5, 7, generator=g)
    for act in (1, 3):
        for grad in (0, 1, 2):
            for bias in (None, b):
                ref = r if grad == 1 else None
                y = fused_bias_act_raw(x.to(DEV), None if bias is None else bias.to(DEV),
                                       None if ref is None else ref.to(DEV), act, grad, 0.3, 1.7)
                yo = so.fused_bias_act_ref(x, bias, ref, act, grad, 0.3, 1.7)
                assert_close(y, yo, rtol=1e-6, what="act%d grad%d" % (act, grad))
    # double backward through FusedLeakyReLU (fused_act.py:42-49)
    xg = x.to(DEV).requires_grad_(True)
    bg = b.to(DEV).requires_grad_(True)
    y = op.fused_leaky_relu(xg, bg)
    go = torch.randn(y.shape, generator=g).to(DEV).requires_grad_(True)
    gx, gb = torch.autograd.grad(y, [xg, bg], go, create_graph=True)
    v = torch.randn(x.shape, generator=g).to(DEV)
    u = torch.randn(b.shape, generator=g).to(DEV)
    (ggo,) = torch.autograd.grad((gx * v).sum() + (gb * u).sum(), go)
    expect = so.fused_bias_act_ref(v.cpu(), u.cpu(), y.detach().cpu(), 3, 1, 0.2, 2 ** 0.5)
    assert_close(ggo, expect, rtol=1e-5, what="double backward")


def test_fused_bias_act_backward_is_deterministic_and_exact_on_integers():
    from gangealing_b200.op.fused_act import bias_act_backward_raw
    g = torch.randint(-8, 9, (4, 16, 128, 128), device=DEV).float()
    out = torch.randn(4, 16, 128, 128, device=DEV)
    gx1, gb1 = bias_act_backward_raw(g, out, 0.5, 2.0, True)   # all values exactly representable
    gx2, gb2 = bias_act_backward_raw(g, out, 0.5, 2.0, True)
    assert torch.equal(gb1, gb2) and torch.equal(gx1, gx2)
    expect = torch.where(out > 0, g, g * 0.5) * 2.0
    assert torch.equal(gx1, expect)
    assert torch.equal(gb1, expect.sum(dim=(0, 2, 3)))  # integer-valued sums: bit-exact


# ------------------------------------------------------------------------------------------------ fused tails
@pytest.mark.parametrize("shape", [(2, 16, 64, 64), (3, 8, 4, 4), (2, 5, 33, 31), (1, 128, 256, 256)])
def test_noise_bias_act(shape):
    op = _ops()
    g = torch.Generator().manual_seed(21)
    n, c, h, w = shape
    x = torch.randn(*shape, generator=g)
    noise = torch.randn(n, 1, h, w, generator=g)
    nw = torch.randn(1, generator=g)
    b = torch.randn(c, generator=g)
    go = torch.randn(*shape, generator=g)
    xo, no, nwo, bo = [t.clone().requires_grad_(True) for t in (x, noise, nw, b)]
    yo = so.noise_bias_act_ref(xo, no, nwo, bo)
    grads_o = torch.autograd.grad(yo, [xo, no, nwo, bo], go)
    xg, ng, nwg, bg = [t.to(DEV).requires_grad_(True) for t in (x, noise, nw, b)]
    y = op.noise_bias_act(xg, ng, nwg, bg)
    assert_close(y, yo, rtol=1e-5, what="fwd")
    grads = torch.autograd.grad(y, [xg, ng, nwg, bg], go.to(DEV))
    for a, e, nm in zip(grads, grads_o, ("x", "noise", "noise_weight", "bias")):
        assert_close(a, e, rtol=2e-4, what="grad " + nm)
    y2 = op.noise_bias_act(xg, None, None, bg)  # noise=None path
    assert_close(y2, so.fused_leaky_relu_ref(x, b), rtol=1e-5)


@pytest.mark.parametrize("shape,pad", [((2, 16, 65, 65), (1, 1)), ((2, 4, 257, 257), (1, 1)), ((3, 8, 9, 9), (1, 1)),
                                       ((1, 6, 129, 129), (1, 1)), ((2, 3, 40, 50), (2, 2))])
def test_blur_noise_bias_act(shape, pad):
    op = _ops()
    g = torch.Generator().manual_seed(22)
    n, c, h, w = shape
    k = so.make_kernel([1, 3, 3, 1]) * 4
    oh, ow = h + pad[0] + pad[1] - 3, w + pad[0] + pad[1] - 3
    x = torch.randn(*shape, generator=g)
    noise = torch.randn(n, 1, oh, ow, generator=g)
    nw = torch.randn(1, generator=g)
    b = torch.randn(c, generator=g)
    rs = torch.rand(n, c, generator=g) + 0.5
    go = torch.randn(n, c, oh, ow, generator=g)
    for row_scale in (None, rs):
        leaves_o = [t.clone().requires_grad_(True) for t in (x, noise, nw, b)]
        rso = None if row_scale is None else row_scale.clone().requires_grad_(True)
        yo = so.blur_noise_bias_act_ref(leaves_o[0], k, pad, leaves_o[1], leaves_o[2], leaves_o[3], row_scale=rso)
        grads_o = torch.autograd.grad(yo, leaves_o + ([] if rso is None else [rso]), go)
        leaves = [t.to(DEV).requires_grad_(True) for t in (x, noise, nw, b)]
        rsg = None if row_scale is None else row_scale.to(DEV).requires_grad_(True)
        y = op.blur_noise_bias_act(leaves[0], k.to(DEV), pad, leaves[1], leaves[2], leaves[3], row_scale=rsg)
        assert_close(y, yo, rtol=1e-4, what="fwd")
        grads = torch.autograd.grad(y, leaves + ([] if rsg is None else [rsg]), go.to(DEV))
        for a, e, nm in zip(grads, grads_o, ("x", "noise", "noise_weight", "bias", "row_scale")):
            assert_close(a, e, rtol=3e-4, what="grad " + nm)


# ------------------------------------------------------------------------------------------------ modulated weights
@pytest.mark.parametrize("b,o,i,k,transposed,demod", [(5, 512, 512, 3, False, True), (3, 256, 512, 3, True, True),
                                                      (2, 128, 128, 3, False, True), (4, 3, 512, 1, False, False),
                                                      (32, 128, 256, 3, True, True), (2, 64, 32, 3, False, True),
                                                      (300, 128, 64, 3, False, True)])
def test_modulated_weight_tensor_core_demod(b, o, i, k, transposed, demod):
    from gangealing_b200.op.modconv import modulated_weight
    g = torch.Generator().manual_seed(b + o)
    w = torch.randn(1, o, i, k, k, generator=g)
    s = torch.randn(b, i, generator=g) + 1.0
    scale = 1.0 / (i * k * k) ** 0.5
    ref = so.modulated_weight_ref(w, s, scale, demod)
    ref = ref.transpose(1, 2).reshape(b * i, o, k, k) if transposed else ref.reshape(b * o, i, k, k)
    sg = s.to(DEV).requires_grad_(True)
    out = modulated_weight(w.to(DEV), sg, scale, demod, transposed)
    assert_close(out, ref, rtol=1e-4, what="modulated weight")   # hi/lo split TF32 GEMM: fp32-grade
    # gradient w.r.t. the style vs autograd through the restatement
    so_ = s.clone().requires_grad_(True)
    r2 = so.modulated_weight_ref(w, so_, scale, demod)
    r2 = r2.transpose(1, 2).reshape(b * i, o, k, k) if transposed else r2.reshape(b * o, i, k, k)
    go = torch.randn(ref.shape, generator=g)
    (gs_ref,) = torch.autograd.grad((r2 * go).sum(), so_)
    (gs,) = torch.autograd.grad((out * go.to(DEV)).sum(), sg)
    assert_close(gs, gs_ref, rtol=2e-3, what="style gradient")


@pytest.mark.parametrize("shape", [(3, 16, 64, 64), (2, 8, 4, 4), (2, 5, 33, 31), (1, 4, 256, 256)])
def test_channel_scale_forward_backward(shape):
    from gangealing_b200.op.modconv import channel_scale
    g = torch.Generator().manual_seed(1)
    x = torch.randn(*shape, generator=g)
    s = torch.randn(shape[0], shape[1], generator=g)
    go = torch.randn(*shape, generator=g)
    xo, so_ = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
    yo = xo * so_[:, :, None, None]
    gxo, gso = torch.autograd.grad(yo, [xo, so_], go)
    xg, sg = x.to(DEV).requires_grad_(True), s.to(DEV).requires_grad_(True)
    y = channel_scale(xg, sg)
    assert_close(y, yo, rtol=1e-6)
    gx, gs = torch.autograd.grad(y, [xg, sg], go.to(DEV))
    assert_close(gx, gxo, rtol=1e-6, what="gx")
    assert_close(gs, gso, rtol=1e-4, what="gs")


@pytest.mark.parametrize("b,cin,cout,h,upsample,k", [(3, 64, 32, 16, False, 3), (2, 32, 64, 8, True, 3), (2, 64, 3, 16, False, 1),
                                                     (4, 128, 128, 32, False, 3)])
def test_modulated_conv2d_dense_formulation_matches_the_grouped_reference(b, cin, cout, h, upsample, k):
    """conv(W*s*d, x) (reference, grouped) == d * conv(W, x*s) (this repo, weight-shared), values and gradients."""
    from gangealing_b200.op.modconv import channel_scale, modulated_conv2d
    from oracle import opset
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        g = torch.Generator().manual_seed(b * cin)
        w = torch.randn(1, cout, cin, k, k, generator=g)
        x = torch.randn(b, cin, h, h, generator=g)
        s = torch.randn(b, cin, generator=g) + 1.0
        scale = 1.0 / (cin * k * k) ** 0.5
        demod = k == 3
        xo, so_ = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
        ref, none = opset.cpu_ops().modulated_conv2d(xo, w, so_, scale, demod, upsample, k // 2)
        assert none is None
        go = torch.randn(ref.shape, generator=g)
        gxo, gso = torch.autograd.grad(ref, [xo, so_], go)
        xg, sg = x.to(DEV).requires_grad_(True), s.to(DEV).requires_grad_(True)
        raw, d = modulated_conv2d(xg, w.to(DEV), sg, scale, demod, upsample, k // 2)
        out = channel_scale(raw, d) if d is not None else raw
        assert_close(out, ref, rtol=1e-4, what="modulated conv")
        gx, gs = torch.autograd.grad(out, [xg, sg], go.to(DEV))
        assert_close(gx, gxo, rtol=2e-4, what="gx")
        assert_close(gs, gso, rtol=2e-3, what="gstyle")
    finally:
        torch.backends.cudnn.allow_tf32 = old


def test_noise_bias_act_with_row_scale():
    op = _ops()
    g = torch.Generator().manual_seed(31)
    x = torch.randn(2, 6, 16, 16, generator=g)
    noise = torch.randn(2, 1, 16, 16, generator=g)
    nw, b, rs = torch.randn(1, generator=g), torch.randn(6, generator=g), torch.rand(2, 6, generator=g) + 0.5
    go = torch.randn(2, 6, 16, 16, generator=g)
    leaves_o = [t.clone().requires_grad_(True) for t in (x, rs)]
    yo = so.noise_bias_act_ref(leaves_o[0] * leaves_o[1][:, :, None, None], noise, nw, b)
    go_x, go_rs = torch.autograd.grad(yo, leaves_o, go)
    xg, rsg = x.to(DEV).requires_grad_(True), rs.to(DEV).requires_grad_(True)
    y = op.noise_bias_act(xg, noise.to(DEV), nw.to(DEV), b.to(DEV), row_scale=rsg)
    assert_close(y, yo, rtol=1e-5)
    gx, grs = torch.autograd.grad(y, [xg, rsg], go.to(DEV))
    assert_close(gx, go_x, rtol=1e-5, what="gx")
    assert_close(grs, go_rs, rtol=1e-4, what="g row_scale")


# ------------------------------------------------------------------------------------------------ demodulation coefficients
# the 13 demodulated convolutions of the 256^2 generator (channel multiplier 2) as (O, I): conv1 at 4^2, then an up-sampling
# and a plain convolution per resolution 8^2 .. 256^2
GEN256_DEMOD_LAYERS = [(512, 512)] * 9 + [(256, 512), (256, 256), (128, 256), (128, 128)]


def _demod_style_grad_ref(w, s, scale, gd, eps=1e-8):
    """float64 autograd of demod_ref w.r.t. the style, and the same contraction over |terms| (the scale of its rounding)."""
    sd = s.double().requires_grad_(True)
    (gs,) = torch.autograd.grad(demod_ref(w, sd, scale, eps), sd, gd.double())
    d = demod_ref(w, s, scale, eps)
    wsq = w.double()[0].pow(2).sum(dim=(2, 3))
    mag = scale ** 2 * s.double().abs() * ((gd.double().abs() * d.pow(3)) @ wsq)
    return gs, mag


@pytest.mark.parametrize("b,o,i", DEMOD_CASES)
def test_demod_coefficients_vs_float64(b, o, i):
    """modconv.demod_coefficients (wgmma TF32 hi/lo GEMM) vs float64 rsqrt(scale^2 * sum_i Wsq s^2 + eps), per element
    relative error <= DEMOD_RTOL (derived in tests/test_demod_precision.py, which also shows a TF32-only kernel misses it).
    The cases reach every <NA, NS> instance of demod_wgmma_kernel.  Observed on an H100 80GB HBM3 (700 W power limit):
    max 5.4e-6 (B=17, O=127, I=513), the split itself ~5e-7 (emulated): the tensor core's fp32 accumulation over the k-steps
    dominates, growing with I -- so the bound stays at 8e-6 rather than 4x the observed value.
    Style gradient (_Demod.backward) vs float64 autograd, relative to the sum of |terms| of its contraction."""
    from gangealing_b200.op.modconv import demod_coefficients
    w, s, scale = demod_inputs(b, o, i)
    sg = s.to(DEV).requires_grad_(True)
    d = demod_coefficients(w.to(DEV), sg, scale)
    assert d.shape == (b, o) and d.dtype == torch.float32
    err = max_rel_err(d, demod_ref(w, s, scale))
    assert err <= DEMOD_RTOL, "max relative error %.2e > %.1e" % (err, DEMOD_RTOL)
    gd = torch.randn(b, o, generator=torch.Generator().manual_seed(o))
    (gs,) = torch.autograd.grad(d, sg, gd.to(DEV))
    gs_ref, mag = _demod_style_grad_ref(w, s, scale, gd)
    excess = ((gs.double().cpu() - gs_ref).abs() - 1e-5 * mag).max().item()
    assert excess <= 0, "style gradient error exceeds 1e-5 of |terms| by %.3e" % excess


def test_batched_demod_matches_the_single_layer_kernel_bitwise():
    """style_path.all_demod (one launch for every layer, csrc/modconv.cu DemodBatch) with the 256^2 generator's 13 layer
    shapes plus an I=32 layer that forces NA=1 for the whole batch: each layer within DEMOD_RTOL of float64 and BITWISE
    equal to demod_coefficients of that layer alone -- the same MMAs in the same k order -- and the _DemodAll.backward
    gradients vs float64 autograd."""
    from gangealing_b200.op import style_path
    from gangealing_b200.op.modconv import demod_coefficients
    b = 8
    layers = GEN256_DEMOD_LAYERS + [(64, 32)]
    ws, ss, scales = [], [], []
    for j, (o, i) in enumerate(layers):
        w, s, scale = demod_inputs(b, o, i, seed=j)
        ws.append(w), ss.append(s), scales.append(scale)
    sg = [s.to(DEV).requires_grad_(True) for s in ss]
    wd = [w.to(DEV) for w in ws]
    dm = style_path.all_demod(wd, sg, scales)
    gds = [torch.randn(d.shape, generator=torch.Generator().manual_seed(j)) for j, d in enumerate(dm)]
    grads = torch.autograd.grad(dm, sg, [g.to(DEV) for g in gds])
    for j, (w, s, scale) in enumerate(zip(ws, ss, scales)):
        err = max_rel_err(dm[j], demod_ref(w, s, scale))
        assert err <= DEMOD_RTOL, "layer %d: max relative error %.2e" % (j, err)
        single = demod_coefficients(wd[j], s.to(DEV), scale)
        assert torch.equal(dm[j], single), "layer %d differs from the single-layer launch" % j
        gs_ref, mag = _demod_style_grad_ref(w, s, scale, gds[j])
        excess = ((grads[j].double().cpu() - gs_ref).abs() - 1e-5 * mag).max().item()
        assert excess <= 0, "layer %d: style gradient error exceeds 1e-5 of |terms| by %.3e" % (j, excess)
