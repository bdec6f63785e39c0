"""Flow composition of the flow STN head -- one fused kernel per direction (csrc/flow.cu).

`flow_compose(low_res_flow, mask, identity_flow, base_warp, alpha, downsample)` returns
(delta_flow, flow) exactly as reference FlowHead.forward computes them (warping_heads.py:239-244):
RAFT convex upsampling (upsample_flow :180-193), identity + delta, apply_affine (:268-277), alpha lerp.
`apply_affine(matrix, grid)` and `upsample_flow(flow, mask, downsample)` keep the reference call surfaces.
"""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import _lib


def _f32c(t):
    if t is None:
        return None
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.float().contiguous()
    return t


def flow_meta(low, mask, base):
    """(dtype, shape) of the caller's low, mask and base warp (None when absent): what flow_grads casts back to."""
    return tuple(None if t is None else (t.dtype, tuple(t.shape)) for t in (low, mask, base))


def flow_inputs(who, low, mask, identity, base, alpha, s):
    """Validate the flow head's raw outputs and return them as contiguous fp32 (low, mask, identity, base, alpha), with
    a 1-element alpha expanded to the batch: the kernels read alpha[n] for every n."""
    if low.dim() != 4 or low.shape[-1] != 2:
        raise RuntimeError("%s: low-res flow must be (N, H, W, 2), got %s" % (who, tuple(low.shape)))
    n, h, w, _ = low.shape
    if mask.shape[0] != n or mask.numel() != n * 9 * s * s * h * w:
        raise RuntimeError("%s: mask must be (N, 9*%d*%d, H, W), got %s" % (who, s, s, tuple(mask.shape)))
    low_c, mask_c, ident_c, base_c, alpha_c = _f32c(low), _f32c(mask), _f32c(identity), _f32c(base), _f32c(alpha)
    if ident_c is not None and ident_c.numel() != s * h * s * w * 2:
        raise RuntimeError("%s: identity_flow must be (1, %d, %d, 2)" % (who, s * h, s * w))
    if base_c is not None and base_c.numel() != n * 6:
        raise RuntimeError("%s: base_warp must be (N, 2, 3)" % who)
    if alpha_c is not None:
        # the reference broadcasts `identity_flow.lerp(flow, alpha[:, None, None, None])` (warping_heads.py:243-244)
        alpha_c = alpha_c.reshape(-1)
        if alpha_c.numel() == 1:
            alpha_c = alpha_c.expand(n).contiguous()
        elif alpha_c.numel() != n:
            raise RuntimeError("%s: alpha must have 1 or N=%d elements, got %d" % (who, n, alpha_c.numel()))
    return low_c, mask_c, ident_c, base_c, alpha_c


def flow_grads(flow_in, like, s, g_delta, g_flow, need_low, need_mask, need_base):
    """gg_flow_compose_backward for the fp32 inputs `flow_in` of flow_inputs and the fp32 gradients arriving at delta and
    at the composed grid (either may be None) -> (g_low, g_mask, g_base) in the dtypes and shapes `like` (flow_meta) of
    the caller's tensors; None where not needed."""
    low, mask, ident, base, alpha = flow_in
    n, h, w, _ = low.shape
    g_mask = torch.empty_like(mask) if need_mask else None
    g_low = torch.zeros_like(low) if need_low else None
    g_base = torch.zeros((n, 2, 3), dtype=torch.float32, device=low.device) if (need_base and base is not None) else None
    rc = _lib.load().gg_flow_compose_backward(_lib.ptr(g_mask), _lib.ptr(g_low), _lib.ptr(g_base), _lib.ptr(g_delta),
                                              _lib.ptr(g_flow), low.data_ptr(), mask.data_ptr(), _lib.ptr(ident),
                                              _lib.ptr(base), _lib.ptr(alpha), n, h, w, s, _lib.stream())
    _lib.check(rc, "gg_flow_compose_backward")
    (low_dt, _), (mask_dt, mask_shape), base_like = like
    if g_mask is not None:
        g_mask = g_mask.reshape(mask_shape).to(mask_dt)
    if g_low is not None:
        g_low = g_low.to(low_dt)
    if g_base is not None:
        g_base = g_base.reshape(base_like[1]).to(base_like[0])
    return g_low, g_mask, g_base


class _FlowCompose(Function):
    @staticmethod
    def forward(ctx, low, mask, identity, base, alpha, s, want_flow):
        _lib.require_cuda(low, mask, identity, base, alpha)
        flow_in = flow_inputs("flow_compose", low, mask, identity, base, alpha, s)
        low_c, mask_c, ident_c, base_c, alpha_c = flow_in
        n, h, w, _ = low.shape
        delta = torch.empty((n, s * h, s * w, 2), dtype=torch.float32, device=low.device)
        flow = torch.empty_like(delta) if want_flow else None
        rc = _lib.load().gg_flow_compose_forward(delta.data_ptr(), _lib.ptr(flow), low_c.data_ptr(), mask_c.data_ptr(),
                                                 _lib.ptr(ident_c), _lib.ptr(base_c), _lib.ptr(alpha_c), n, h, w, s,
                                                 _lib.stream())
        _lib.check(rc, "gg_flow_compose_forward")
        ctx.save_for_backward(*flow_in)
        ctx.cfg = (s, flow_meta(low, mask, base))
        if flow is None:
            flow = delta.new_zeros(())
            ctx.mark_non_differentiable(flow)
        return delta, flow

    @staticmethod
    @once_differentiable
    def backward(ctx, g_delta, g_flow):
        s, like = ctx.cfg
        need_low, need_mask, _, need_base = ctx.needs_input_grad[:4]
        g_delta = _f32c(g_delta) if g_delta is not None else None
        g_flow = _f32c(g_flow) if (g_flow is not None and g_flow.dim() == 4) else None
        g_low, g_mask, g_base = flow_grads(ctx.saved_tensors, like, s, g_delta, g_flow, need_low, need_mask, need_base)
        return g_low, g_mask, None, g_base, None, None, None


def flow_compose(low_res_flow, mask, identity_flow, base_warp=None, alpha=None, downsample=8):
    """-> (delta_flow (N, sH, sW, 2), flow (N, sH, sW, 2)); fp32."""
    return _FlowCompose.apply(low_res_flow, mask, identity_flow, base_warp, alpha, downsample, True)


def upsample_flow(flow, mask, downsample=8):
    """RAFT convex upsampling [H/s, W/s, 2] -> [H, W, 2] (reference FlowHead.upsample_flow)."""
    return _FlowCompose.apply(flow, mask, None, None, None, downsample, False)[0]


def apply_affine(matrix, grid):
    """[gx, gy, 1] @ matrix^T at every grid point (reference warping_heads.py:268-277); plain tensor ops --
    inside the flow head this step is fused into flow_compose."""
    n = grid.size(0)
    flat = grid.reshape(n, -1, 2)
    out = flat @ matrix[:, :, :2].transpose(1, 2) + matrix[:, None, :, 2]
    return out.reshape(grid.size())
