"""CPU: libgg_b200.so loads without a GPU and exports exactly the symbols include/gg_b200.h declares."""
import os
import re

from conftest import ROOT
from gangealing_b200 import _lib


def _declared():
    text = open(os.path.join(ROOT, "include", "gg_b200.h")).read()
    return sorted(set(re.findall(r"GG_API\s+[\w\s\*]+?\b(gg_\w+)\s*\(", text)))


def test_header_symbols_are_bound_and_exported():
    declared = _declared()
    assert "gg_upfirdn2d" in declared and "gg_fused_bias_act" in declared
    dll = _lib.load()
    for name in declared:
        assert hasattr(dll, name), "libgg_b200.so does not export %s" % name
    assert sorted(_lib.SIGNATURES) == declared, "ctypes table and header disagree"


def test_version_and_error_string():
    dll = _lib.load()
    assert dll.gg_version() >= 1
    assert isinstance(dll.gg_last_error(), bytes)


def test_bad_arguments_are_reported_not_fatal():
    dll = _lib.load()
    # no device work is reached: argument validation happens first
    rc = dll.gg_fused_bias_act(None, None, None, None, 0, 3, 0, 0.2, 1.0, 16, 1, 0, None)
    assert rc == -1 and b"null" in dll.gg_last_error()
    rc = dll.gg_fused_bias_act(None, None, None, None, 0, 7, 0, 0.2, 1.0, 16, 1, 0, None)
    assert rc < 0
    rc = dll.gg_upfirdn2d(None, None, None, 3, 1, 4, 4, 4, 4, 1, 1, 1, 1, 0, 0, 0, 0, None)
    assert rc < 0  # filter larger than input / unsupported dtype
    assert dll.gg_bias_act_backward_workspace(2, 3, 4096) == 2 * 3 * 4


def test_ops_refuse_cpu_tensors():
    import pytest
    import torch
    from gangealing_b200.op import fused_leaky_relu, upfirdn2d
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        upfirdn2d(torch.zeros(1, 1, 8, 8), torch.ones(4, 4))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        fused_leaky_relu(torch.zeros(1, 2, 4, 4), torch.zeros(2))


def test_argument_validation_of_the_channels_last_and_loss_entry_points():
    """Host-side validation runs before any device work: unsupported shapes come back as status codes + messages."""
    dll = _lib.load()
    one = 1  # any non-null pointer value: validation must reject these calls before dereferencing anything
    # perceptual front end: C must be a power of two below 128 or a multiple of 128
    assert dll.gg_feature_distance_forward(one, one, one, one, None, 0, 2, 24, 16, 1e-10, None) == -2
    assert b"feature_distance" in dll.gg_last_error()
    assert dll.gg_feature_distance_forward(one, one, one, one, None, 0, 2, 192, 16, 1e-10, None) == -2
    assert dll.gg_feature_distance_backward(one, one, one, one, one, None, 0, -1, 64, 16, 1e-10, None) == -1
    assert dll.gg_feature_distance_workspace(0, 64, 16) == 0
    # BilinearDownsample: stride range, reflection needs a plane larger than stride/2
    assert dll.gg_tent_downsample_forward(one, one, one, one, 1, 3, 8, 8, 0, None) == -2
    assert dll.gg_tent_downsample_forward(one, one, one, one, 1, 3, 8, 8, 17, None) == -2
    assert dll.gg_tent_downsample_forward(one, one, one, one, 1, 3, 2, 8, 4, None) == -1
    assert dll.gg_tent_downsample_backward(one, one, one, one, 1, 3, 8, 8, 0, None) == -2
    assert dll.gg_tent_downsample_forward(None, None, None, None, 0, 3, 8, 8, 2, None) == 0      # empty batch: nothing to do
    # to-RGB and the NHWC family: channel-count contracts
    assert dll.gg_to_rgb_nhwc_forward(one, one, one, None, None, 1, 20, 16, None) == -2
    assert dll.gg_to_rgb_nhwc_backward(one, one, one, one, one, one, 1, 6, 16, None) == -2
    assert dll.gg_channel_scale_nhwc(one, None, None, one, None, one, 0, 1, 6, 16, None) == -2
    assert dll.gg_channel_scale_nhwc(one, None, None, one, None, one, 2, 1, 12, 16, None) == -2      # bf16: C % 8
    assert dll.gg_channel_scale_nhwc(one, None, None, one, None, one, 1, 1, 8, 16, None) == -2       # fp16: unsupported
    assert dll.gg_channel_scale_nhwc(one, None, None, one, None, None, 0, 1, 8, 16, None) == -1      # null scale
    assert dll.gg_bias_act_backward_nhwc(one, None, None, one, None, 0, 0.2, 1.0, 1, 8, 16, None) == -1  # null saved output
    assert dll.gg_noise_bias_act_nhwc(one, one, None, None, None, None, 0, 0.2, 1.0, 1, 6, 16, None) == -2
    blur_tail = [0, 1, 20, 8, 8, 4, 4, 1, 1, 1, 1, 1, 0, 1, 0.0, 1.0, None]   # dtype, N, C, h, w, kh, kw, sep, pads, mode, act, alpha, scale, stream
    ptrs = [one, None, one, one] + [None] * 8
    assert dll.gg_blur_nhwc(*ptrs, *blur_tail) == -2                                               # C % 32
    assert dll.gg_blur_nhwc(*ptrs, 2, 1, 32, *blur_tail[3:]) == -2                                 # bf16: C % 64
    assert dll.gg_blur_nhwc(*ptrs, 0, 1, 32, 8, 8, 5, 5, *blur_tail[7:]) == -2                     # filter > 4x4
    assert dll.gg_blur_nhwc(*ptrs, 0, 1, 32, 8, 8, 4, 4, 1, 1, 1, 1, 1, 0, 2, 0.0, 1.0, None) == -2  # act
    assert dll.gg_blur_nhwc(*ptrs, 0, 1, 32, 8, 8, 4, 4, 1, 1, 1, 1, 1, 3, 1, 0.0, 1.0, None) == -1  # mode
    assert dll.gg_blur_nhwc(one, one, one, one, *([None] * 8), 0, 1, 32, 8, 8, 4, 4, 1, 1, 1, 1, 1, 0, 1, 0.0, 1.0, None) == -1  # out2 is mode 1's
    assert dll.gg_blur_nhwc_workspace(0, 2, 64, 17, 17, 4, 4, 1, 1, 1, 1) > 0
    # cross-layer fused tails
    st = [None] * 8
    assert dll.gg_styled_tail_nhwc(one, None, None, one, *st, 0, 3, 0.2, 1.0, 1, 20, 16, None) == -2     # C % 32
    assert dll.gg_styled_tail_nhwc(one, None, None, one, *st, 2, 3, 0.2, 1.0, 1, 32, 16, None) == -2     # bf16: C % 64
    assert dll.gg_styled_tail_nhwc(None, None, None, one, *st, 0, 3, 0.2, 1.0, 1, 32, 16, None) == -1    # nothing to write
    assert dll.gg_styled_tail_nhwc(None, one, None, one, *st, 0, 3, 0.2, 1.0, 1, 32, 16, None) == -1     # xs without s_next
    assert dll.gg_styled_tail_nhwc(one, None, None, one, *st, 0, 2, 0.2, 1.0, 1, 32, 16, None) == -2     # act
    assert dll.gg_styled_tail_backward_nhwc(one, None, None, None, None, None, None, one, None, None, None, None,
                                            0, 0.2, 1.0, 1, 32, 16, 32, None) == -1                      # no upstream gradient
    assert dll.gg_styled_tail_backward_nhwc(one, None, None, None, None, one, None, one, None, None, None, None,
                                            0, 0.2, 1.0, 1, 32, 16, 32, None) == -1                      # g_xs without s_next
    assert dll.gg_styled_tail_backward_workspace(0, 2, 64, 256) > 0


def test_misaligned_vector_operands_are_refused():
    """Kernels that read a per-channel constant as float4 refuse a pointer off a 16-byte boundary (a slice such as b[1:])
    with a status code, before any device work, instead of faulting on the device."""
    dll = _lib.load()
    a, m = 16, 4     # an aligned and a misaligned non-null pointer value; validation must not dereference either

    def refused(rc):
        return rc == -1 and b"aligned" in dll.gg_last_error()
    assert refused(dll.gg_noise_bias_act_nhwc(a, a, None, None, m, None, 0, 0.2, 1.0, 1, 8, 16, None))          # bias
    assert refused(dll.gg_noise_bias_act_nhwc(a, a, None, None, None, m, 2, 0.2, 1.0, 1, 8, 16, None))          # row_scale
    assert refused(dll.gg_to_rgb_nhwc_forward(a, a, m, None, None, 1, 32, 16, None))                            # wm
    assert refused(dll.gg_to_rgb_nhwc_forward(a, a, a, None, m, 1, 32, 16, None))                               # skip, HW % 4 == 0
    assert refused(dll.gg_to_rgb_nhwc_backward(a, None, None, a, a, m, 1, 32, 16, None))                        # wm
    assert refused(dll.gg_bias_relu_pool_nhwc_forward(a, a, a, m, 0, 1, 8, 4, 4, None))                         # bias
    assert refused(dll.gg_feature_distance_forward(a, a, a, a, m, 0, 2, 64, 16, 1e-10, None))                   # weight
    assert refused(dll.gg_feature_distance_backward(a, a, a, a, a, m, 2, 2, 64, 16, 1e-10, None))               # weight
    # the shape contracts are still checked first
    assert dll.gg_to_rgb_nhwc_forward(a, a, m, None, None, 1, 20, 16, None) == -2


def test_misaligned_float2_operands_are_refused():
    """Entries whose kernels read or write flows and sampling grids as float2 refuse a pointer off an 8-byte boundary (a
    view such as buf[1:].view(n, h, w, 2)) with a status code, before any device work."""
    dll = _lib.load()
    a, m = 16, 4

    def refused(rc):
        return rc == -1 and b"aligned" in dll.gg_last_error()
    fwd = [a, a, a, a, a, None, None]        # delta, flow, low, mask, identity, base, alpha
    for i in (0, 1, 2, 4):
        args = list(fwd)
        args[i] = m
        assert refused(dll.gg_flow_compose_forward(*args, 2, 3, 3, 2, None)), i
    bwd = [a, a, a, a, a, a, a, a, a, a]     # g_mask, g_low, g_base, g_delta, g_flow, low, mask, identity, base, alpha
    for i in (1, 3, 4, 5, 7):
        args = list(bwd)
        args[i] = m
        assert refused(dll.gg_flow_compose_backward(*args, 2, 3, 3, 2, None)), i
    assert refused(dll.gg_warp_sample_indices(a, m, 1, 8, 8, 4, 4, 0.0, 0.0, 1, None))
    assert refused(dll.gg_mipmap_warp_forward(a, None, a, None, m, 0, 1, 1, 8, 8, 4, 4, 0, 0.0, 0.0, 1, None))
    flow_mode = [a, a, a, None, a, None, None, a, a, a, None]    # out, grid_out, delta_out, levels, src, pyr, theta, low, mask, identity, alpha
    for i in (1, 2, 7, 9):
        args = list(flow_mode)
        args[i] = m
        assert refused(dll.gg_stn_sample_forward(*args, 2, 0, 1, 1, 8, 8, 8, 8, 4, 4, 2, 0, 0.0, 0.0, 1, None)), i
    assert refused(dll.gg_stn_sample_forward(a, m, None, None, a, None, a, None, None, None, None, 1, 0, 1, 1, 8, 8, 8, 8,
                                             0, 0, 1, 0, 0.0, 0.0, 1, None))               # affine mode: grid_out
    lerp = [a, a, a, None, a, 32, a, a]      # out, grid_out, src, pyr, base, base_stride, target, alphas
    for i in (1, 4, 6):
        args = list(lerp)
        args[i] = m
        assert refused(dll.gg_mipmap_warp_lerp_forward(*args, 1, 0, 1, 1, 8, 8, 4, 4, 0, 0.0, 0.0, 1, None)), i
    for i in (3, 5):                        # acc, src, pyr, base, base_stride, target, alphas
        args = [a, a, None, a, 32, a, a]
        args[i] = m
        assert refused(dll.gg_mipmap_warp_lerp_mean(*args, 1, 0, 1, 1, 8, 8, 4, 4, 0, 0.0, 0.0, 1, 0, None)), i
    assert refused(dll.gg_mipmap_warp_backward(None, None, a, a, a, None, m, 0, 1, 1, 8, 8, 4, 4, 0, 0.0, 0.0, 1, None))
    assert refused(dll.gg_mipmap_warp_backward(None, None, m, a, a, None, a, 0, 1, 1, 8, 8, 4, 4, 0, 0.0, 0.0, 1, None))


def test_flow_backward_validates_before_its_first_launch():
    """gg_flow_compose_backward checks every argument, the sample count of the g_base grid included, before it launches
    the g_mask and g_low kernels (the pointers below are never dereferenced)."""
    dll = _lib.load()
    a = 16
    rc = dll.gg_flow_compose_backward(a, a, a, a, a, a, a, a, a, a, 1 << 31, 1, 1, 1, None)
    assert rc == -1 and b"too many samples" in dll.gg_last_error()
    # identity is required when g_flow meets a base warp, whichever outputs are requested
    assert dll.gg_flow_compose_backward(a, a, None, None, a, a, a, None, a, None, 2, 2, 2, 2, None) == -1
    assert dll.gg_flow_compose_backward(a, a, a, a, a, None, a, a, a, a, 2, 2, 2, 2, None) == -1      # null low
