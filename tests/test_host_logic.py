"""Host-side plumbing that needs no GPU: per-tensor memoisation, filter classification, layout predicates,
output-size arithmetic of the resamplers."""
import torch

from gangealing_b200 import _lib
from gangealing_b200.op.upfirdn2d import _out_size, grad_pad


def test_tensor_cache_is_per_object_and_invalidated_by_in_place_updates():
    a = torch.zeros(4, 4)
    memo = _lib.tensor_cache(a)
    memo["x"] = 1
    assert _lib.tensor_cache(a).get("x") == 1
    b = torch.zeros(4, 4)                       # a different object, even at a recycled address, starts empty
    assert _lib.tensor_cache(b).get("x") is None
    a.add_(1.0)                                 # in-place update bumps the version -> stale entries are dropped
    assert _lib.tensor_cache(a).get("x") is None


def test_filter_separability_is_decided_per_filter_not_per_address():
    k = torch.tensor([1., 3., 3., 1.])
    sep = k[:, None] * k[None, :]
    assert _lib.filter_is_separable(sep)
    for _ in range(8):                          # temporaries of the same shape recycle storage: must not alias the memo
        r = torch.randn(4, 4)
        assert not _lib.filter_is_separable(r)
        del r
        t = sep.clone()
        assert _lib.filter_is_separable(t)
        del t
    assert _lib.filter_is_separable(torch.zeros(3, 3))
    assert _lib.filter_is_separable(torch.tensor([[2.0]]))
    assert not _lib.filter_is_separable(torch.eye(3))


def test_flipped_filter_is_memoised_and_inherits_separability():
    k = torch.arange(12.0).reshape(3, 4)
    f = _lib.flipped_filter(k)
    assert torch.equal(f, torch.flip(k, [0, 1]))
    assert _lib.flipped_filter(k) is f
    assert torch.equal(_lib.flipped_filter(f), k)
    sep = torch.outer(torch.tensor([1., 2., 1.]), torch.tensor([1., 3., 3., 1.]))
    assert _lib.filter_is_separable(sep)
    assert _lib.tensor_cache(_lib.flipped_filter(sep)).get("separable") is True


def test_layout_predicate():
    x = torch.zeros(2, 8, 4, 4)
    assert not _lib.is_nhwc(x)
    assert _lib.is_nhwc(x.contiguous(memory_format=torch.channels_last))
    assert not _lib.is_nhwc(torch.zeros(2, 8, 1, 1).contiguous(memory_format=torch.channels_last))  # ambiguous: NCHW path
    assert not _lib.is_nhwc(torch.zeros(2, 8))
    # which channels-last kernels take a tensor: 16-byte channel vectors (4 fp32 / 8 bf16), <= 256 of them per pixel for the
    # row-wise kernels, 8 of them per CTA for the blur (<= 4x4 taps, no resampling)
    from gangealing_b200.op import nhwc

    def cl(c, dtype=torch.float32):
        return torch.zeros(1, c, 2, 2, dtype=dtype).contiguous(memory_format=torch.channels_last)
    assert nhwc.elementwise_ok(cl(4)) and not nhwc.elementwise_ok(cl(6)) and not nhwc.elementwise_ok(cl(4, torch.bfloat16))
    assert not nhwc.elementwise_ok(cl(8, torch.float16)) and not nhwc.elementwise_ok(x)
    assert nhwc.rowwise_ok(cl(1024)) and not nhwc.rowwise_ok(cl(1028)) and nhwc.elementwise_ok(cl(1028))
    assert nhwc.rowwise_ok(cl(2048, torch.bfloat16)) and not nhwc.rowwise_ok(cl(2056, torch.bfloat16))
    assert nhwc.blur_ok(cl(32), 4, 4) and not nhwc.blur_ok(cl(16), 4, 4) and not nhwc.blur_ok(cl(32, torch.bfloat16), 4, 4)
    assert nhwc.blur_ok(cl(64, torch.bfloat16), 3, 4) and not nhwc.blur_ok(cl(32), 5, 4) and not nhwc.blur_ok(cl(32), 4, 5)
    assert not nhwc.blur_ok(cl(32), 4, 4, (2, 2), (1, 1)) and not nhwc.blur_ok(cl(32), 4, 4, (1, 1), (1, 2))
    # the activation itself is read 16 bytes at a time: a view one element past a 16-byte boundary takes the NCHW route,
    # one a whole 16 bytes past keeps the channels-last one
    def at(c, off, dtype=torch.float32):
        buf = torch.zeros(off + 4 * c, dtype=dtype)
        return buf[off:].as_strided((1, c, 2, 2), (4 * c, 1, 2 * c, c))
    for c, dtype in ((32, torch.float32), (64, torch.bfloat16)):
        step = 16 // torch.tensor([], dtype=dtype).element_size()
        aligned = at(c, 0, dtype)
        assert aligned.data_ptr() % 16 == 0 and _lib.is_nhwc(aligned)
        assert nhwc.elementwise_ok(aligned) and nhwc.rowwise_ok(aligned) and nhwc.blur_ok(aligned, 4, 4)
        assert nhwc.elementwise_ok(at(c, step, dtype)) and nhwc.blur_ok(at(c, step, dtype), 4, 4)
        off = at(c, 1, dtype)
        assert _lib.is_nhwc(off) and off.data_ptr() % 16 != 0
        assert not nhwc.elementwise_ok(off) and not nhwc.rowwise_ok(off) and not nhwc.blur_ok(off, 4, 4)
    # per-channel constants reach the kernels as 16-byte-aligned fp32: a slice is copied, a whole tensor is not
    b = torch.arange(9, dtype=torch.float32)
    assert nhwc._f32(b) is not None and nhwc._f32(b).data_ptr() == b.data_ptr()
    s = nhwc._f32(b[1:], 8)
    assert s.data_ptr() % 16 == 0 and s.data_ptr() != b[1:].data_ptr() and torch.equal(s, b[1:])
    assert _lib.dense_f32(b[4:]).data_ptr() == b[4:].data_ptr()
    assert _lib.dense_f32(b[1:].double()).dtype == torch.float32


def test_upfirdn2d_size_arithmetic_matches_the_reference_formulae():
    # reference upfirdn2d.py:103-104 (output size) and :111-116 (g_pad)
    for (h, w, k, up, down, pad) in [(9, 9, 4, 1, 1, (1, 1)), (4, 4, 4, 2, 1, (2, 1)), (16, 12, 4, 1, 2, (1, 1)), (7, 5, 3, 2, 2, (0, 1))]:
        p4 = (pad[0], pad[1], pad[0], pad[1])
        oh, ow = _out_size(h, w, k, k, (up, up), (down, down), p4)
        assert oh == (h * up + pad[0] + pad[1] - k) // down + 1
        assert ow == (w * up + pad[0] + pad[1] - k) // down + 1
        gp = grad_pad(h, w, oh, ow, k, k, (up, up), (down, down), p4)
        # the adjoint maps (oh, ow) back to (h, w): sizes must round-trip
        bh, bw = _out_size(oh, ow, k, k, (down, down), (up, up), gp)
        assert (bh, bw) == (h, w)


def test_ops_refuse_cpu_tensors():
    import pytest
    from gangealing_b200 import op
    from gangealing_b200.op.modconv import channel_scale
    with pytest.raises(RuntimeError):
        op.upfirdn2d(torch.zeros(1, 1, 8, 8), torch.ones(4, 4), pad=(1, 1))
    with pytest.raises(RuntimeError):
        op.fused_leaky_relu(torch.zeros(1, 4, 2, 2), torch.zeros(4))
    with pytest.raises(RuntimeError):
        channel_scale(torch.zeros(1, 4, 2, 2), torch.ones(1, 4))


def test_weight_scaler_group_plan_and_layer_discovery():
    """op/scaled_weights: groups are consecutive runs of layers in forward order, bounded by a byte budget (an oversized layer
    stands alone), and the layer discovery finds exactly the trainable EqualConv2d / EqualLinear of a network."""
    from gangealing_b200.op.scaled_weights import equalized_layers, plan_groups
    from gangealing_b200.stn import get_stn
    from oracle import opset
    assert plan_groups([], 100) == []
    assert plan_groups([10, 20, 30], 100) == [[0, 1, 2]]
    assert plan_groups([60, 50, 10, 200, 5, 5], 100) == [[0], [1, 2], [3], [4, 5]]
    groups = plan_groups([7] * 25, 20)
    assert [i for g in groups for i in g] == list(range(25)) and all(len(g) <= 2 for g in groups)
    stn = get_stn(["similarity", "flow"], flow_size=64, supersize=64, channel_multiplier=0.25, num_heads=1, ops=opset.cpu_ops())
    layers = equalized_layers(stn)
    names = {id(m): n for n, m in stn.named_modules()}
    found = [names[id(m)] for m, _ in layers]
    assert len(found) == len(set(found)) >= 30
    assert any(n.endswith("final_linear") for n in found) and any("flow_out" in n for n in found) and any(".skip." in n for n in found)
    assert all(isinstance(s, float) and s > 0 for _, s in layers)
    # module registration order is the order the layers run in (groups must be runs of consecutively executed layers)
    assert found.index("stns.0.convs.0.0") < found.index("stns.0.final_conv.0") < found.index("stns.1.convs.0.0")
    for prm in stn.stns[0].parameters():
        prm.requires_grad = False
    assert all(names[id(m)].startswith("stns.1.") for m, _ in equalized_layers(stn))
