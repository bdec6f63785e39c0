"""The generator's STYLE path batched over layers (frozen generator).

reference: every ModulatedConv2d runs its own `modulation` EqualLinear (networks.py:146-149, :236) and its own
demodulation reduction (:245-246) -- 20 small GEMMs + 13 demodulation chains per generator pass, each a few
microseconds of work behind a launch.  All of them depend only on the latent, so they are computed up front:

    styles   one batched GEMM per distinct in-channel count (3 for the 256^2 generator) over the stacked, pre-scaled
             modulation weights:  s[l] = latent[:, idx[l]] @ (W_l * scale_l)^T + bias_l * lr_mul
    demod    ONE launch of the wgmma demodulation GEMM for all modulated convolutions (csrc/modconv.cu DemodBatch);
             backward: one batched GEMM per distinct (O, I) filter shape
"""
import ctypes

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import _lib
from .modconv import _derived


class _Plan:
    """Stacked, pre-scaled modulation weights of a frozen generator, grouped by in-channel count."""

    def __init__(self, convs, rgbs, conv_idx, rgb_idx):
        mods = [(("conv", i), m.conv.modulation, conv_idx[i]) for i, m in enumerate(convs)] + \
               [(("rgb", i), m.conv.modulation, rgb_idx[i]) for i, m in enumerate(rgbs)]
        groups = {}
        for key, lin, li in mods:
            groups.setdefault(lin.weight.shape[0], []).append((key, lin, li))
        self.groups = []
        for c, members in sorted(groups.items(), reverse=True):
            w = torch.stack([(lin.weight.detach() * lin.scale).t().contiguous() for _, lin, _ in members])     # (L, D, C)
            b = torch.stack([(lin.bias.detach() * lin.lr_mul) for _, lin, _ in members]).unsqueeze(1)          # (L, 1, C)
            idx = torch.tensor([li for _, _, li in members], device=w.device)
            self.groups.append((w, b, idx, [key for key, _, _ in members], [li for _, _, li in members]))
        self.stamp = tuple((lin.weight._version, lin.weight.data_ptr(), lin.bias._version) for _, lin, _ in mods)

    def valid(self, convs, rgbs):
        mods = [m.conv.modulation for m in convs] + [m.conv.modulation for m in rgbs]
        return self.stamp == tuple((lin.weight._version, lin.weight.data_ptr(), lin.bias._version) for lin in mods)


def all_styles(generator, latent, convs, rgbs, conv_idx, rgb_idx, row_needs_grad=None):
    """-> (styles of the StyledConvs, styles of the ToRGBs): lists of (B, C_in) fp32 tensors, differentiable in `latent`.
    row_needs_grad: per latent row, whether what the caller built that row from requires grad (None: as `latent` does).  A
    style read from a constant row is returned detached: the values are those of the same batched GEMM, but its consumers
    (demodulation, the fused tails) then see that nothing is owed to it and skip that part of their backward."""
    plan = getattr(generator, "_gg_style_plan", None)
    if plan is None or not plan.valid(convs, rgbs):
        plan = _Plan(convs, rgbs, conv_idx, rgb_idx)
        generator._gg_style_plan = plan
    out = {}
    for w, b, idx, keys, rows in plan.groups:
        lat = latent.index_select(1, idx).transpose(0, 1)          # (L, B, D)
        s = torch.baddbmm(b, lat, w)                               # (L, B, C)
        for j, key in enumerate(keys):
            out[key] = s[j] if row_needs_grad is None or row_needs_grad[rows[j]] else s[j].detach()
    return [out[("conv", i)] for i in range(len(convs))], [out[("rgb", i)] for i in range(len(rgbs))]


class _DemodAll(Function):
    """demod_l[b, o] = rsqrt(scale_l^2 * sum_i Wsq_l[o, i] * style_l[b, i]^2 + eps) for every layer, one launch."""

    @staticmethod
    def forward(ctx, meta, *styles):
        weights, scales, eps = meta
        lib = _lib.load()
        n = len(styles)
        b = styles[0].shape[0]
        if b > 256:
            raise RuntimeError("batched demodulation: batch %d > 256" % b)
        ss, wsqs, outs = [], [], []
        for w, s in zip(weights, styles):
            s = s.detach()
            if s.dtype != torch.float32 or not s.is_contiguous():
                s = s.float().contiguous()
            ss.append(s)
            wsqs.append(_derived(w, False)[1])
            outs.append(torch.empty((b, w.shape[1]), dtype=torch.float32, device=s.device))
        P, F, I = ctypes.c_void_p * n, ctypes.c_float * n, ctypes.c_int * n
        rc = lib.gg_modconv_demod_batched(n, P(*[o.data_ptr() for o in outs]), P(*[w.data_ptr() for w in wsqs]),
                                          P(*[s.data_ptr() for s in ss]), F(*[float(x) for x in scales]),
                                          I(*[w.shape[1] for w in weights]), I(*[w.shape[2] for w in weights]), float(eps), b,
                                          _lib.stream())
        _lib.check(rc, "gg_modconv_demod_batched")
        # a coefficient whose style is constant is constant: its consumers owe it no gradient
        ctx.mark_non_differentiable(*[o for l, o in enumerate(outs) if not ctx.needs_input_grad[1 + l]])
        ctx.save_for_backward(*ss, *outs, *wsqs)
        ctx.cfg = (n, tuple(float(x) for x in scales), tuple(s.dtype for s in styles))
        return tuple(outs)

    @staticmethod
    @once_differentiable
    def backward(ctx, *gds):
        n, scales, dtypes = ctx.cfg
        saved = ctx.saved_tensors
        ss, ds, wsqs = saved[:n], saved[n:2 * n], saved[2 * n:]
        grads = [None] * n
        groups = {}
        for l in range(n):
            if gds[l] is not None and ctx.needs_input_grad[1 + l]:
                groups.setdefault(tuple(wsqs[l].shape), []).append(l)
        for _, members in groups.items():     # gs = -(scale^2) * s * ((gd * demod^3) @ Wsq): one batched GEMM per filter shape
            t = torch.stack([gds[l].float() * ds[l].pow(3) * (-(scales[l] ** 2)) for l in members])      # (L, B, O)
            w = torch.stack([wsqs[l] for l in members])                                                  # (L, O, I)
            gs = torch.bmm(t, w)
            for j, l in enumerate(members):
                grads[l] = (gs[j] * ss[l]).to(dtypes[l])
        return (None,) + tuple(grads)


def all_demod(weights, styles, scales, eps=1e-8):
    """weights: list of (1, O, I, k, k) frozen filter banks; styles: list of (B, I); -> list of (B, O) coefficients."""
    for w in weights:
        if w.requires_grad:
            raise RuntimeError("batched demodulation serves frozen filter banks only")
    _lib.require_cuda(*weights, *styles)
    return list(_DemodAll.apply((tuple(weights), tuple(scales), eps), *styles))
