"""The STN side of the training step (csrc/flow.cu, csrc/optim.cu, csrc/pck.cu) against float64, over their launch plans.

  flow_compose_fwd_kernel     delta = sum_k softmax(mask)_k * s*low[nbr k] (RAFT convex up-sampling), flow = identity + delta
                              [-> base warp] [-> alpha lerp]; one thread per full-resolution pixel, grid-stride
  flow_compose_bwd_kernel     g_mask = p_k (t_k - sum_j p_j t_j), t_k = <g, s*low[nbr k]>
  flow_low_bwd_kernel         g_low: one warp per low-resolution entry, lanes stride over its 9*s*s pixels, butterfly sum
  flow_base_bwd_kernel        g_base: one CTA per sample, per-thread trips, 8 warp partials summed in order
  tv_fwd_kernel + tv_finish   the batch-reduced Huber total variation: per-CTA partials, then one 256-thread finish
  tv_bwd_kernel               its gather-form gradient, 4 * tv_blocks CTAs
  tv_per_sample_kernel        the per-sample smoothness match_flows decides flips with: one 512-thread CTA per sample
  adam_tick_kernel            state = (t, 1 - b1^t, sqrt(1 - b2^t)) formed in double
  adam_ema_kernel             Adam + EMA for a table of tensors, CTA -> (tensor, chunk), float4 path behind a gate
  scale_cast_multi_kernel     dst = (dst type)(src * scale) for a table of tensors, the same CTA map and gate

This file

  * restates the host-side planning in Python (grid_for, tv_blocks, the CTA -> (tensor, chunk) maps and the vector gate) and
    labels every case with its route; a CPU test asserts that the cases reach every label, planned for 132 SMs (H100 SXM),
    and a GPU test checks the launched kernels of each flow-backward output subset, of the TV forward and of a tick-only
    Adam step under torch.profiler;
  * checks every output against float64 evaluated on the exact operands the launch reads (oracle/rounding.py):
        stored value   |y - ref| <= k * 2^-24 * A                   (assert_fp32_sum with c = k)
        fp32 sum       |y - ref| <= c * 2^-24 * sum|terms|
    with k and c derived from each kernel's operation order next to each check.  The softmax weights carry an error that
    grows with the logit spread (l_k - max is rounded before expf), so the flow checks add 2^-24 * sum A_k (|d_k| + S) per
    element on top of the constant, d_k = l_k - max and S = sum_j p_j |d_j|;
  * pins the flow backward's g_base to exact zeros when no gradient reaches it through a base warp, and the flow / sampler
    faces to the same values on contiguous views that start off a 16-byte boundary as on aligned copies.

Every check prints its worst observed k / c (`[contract] ...` lines with `pytest -s`), and the module prints the worst per
path when it finishes.
"""
import math
import re
import struct

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fp64_contract import (BF16, CODE, DEV, F32, H100_SMS, Worst, assert_routes_reached, ceil_div, f32, grid_for, launched,
                           library, run_fresh, seeded)
from oracle.rounding import U32, assert_fp32_sum

THREADS = 256
ADAM_CHUNK = 65536                # gangealing_b200.training.fused_optim._CHUNK
SCALE_CHUNK = 32768               # gangealing_b200.op.scaled_weights._CHUNK
BETAS, EPS = (0.9, 0.999), 1e-8
DECAY = 0.5 ** (32 / 10000)
SHORT = {F32: "f32", BF16: "bf16"}
ESIZE = {F32: 4, BF16: 2}


# ======================================================================================== planner restatement (no GPU)
def tv_blocks(total, sms=H100_SMS):
    """optim.cu tv_blocks: at most 4 CTAs per SM."""
    return min(max(ceil_div(total, THREADS), 1), 4 * sms)


def _trip_label(tag, total, per_trip):
    if total < per_trip:
        return "%s: one partial trip" % tag
    if total == per_trip:
        return "%s: exactly one full trip" % tag
    return "%s: a second, partial trip" % tag if total < 2 * per_trip else "%s: several trips" % tag


FWD_CONFIGS = ("delta only", "flow", "flow+base", "flow+alpha", "flow+alpha broadcast", "flow+base+alpha")
LOGITS = ("narrow", "wide", "ties")


def flow_fwd_route(case, sms=H100_SMS):
    n, lh, lw, s, cfg, logits = case
    total = n * s * s * lh * lw
    blocks = grid_for(total, sms=sms)
    labels = {_trip_label("flow fwd", total, blocks * THREADS), "fwd: %s" % cfg, "logits: %s" % logits,
              "flow fwd: s = %d" % s}
    if lh == 1 or lw == 1:
        labels.add("flow fwd: a 1-wide low-resolution side (every neighbour but one padded)")
    if lh != lw:
        labels.add("flow fwd: non-square")
    return dict(blocks=blocks, labels=labels)


BWD_OUTPUTS = ("g_mask", "g_low", "g_base")
UPSTREAM = ("delta", "flow", "both")


def flow_bwd_route(case, sms=H100_SMS):
    """gg_flow_compose_backward -> dict(names: kernels launched in order, labels)."""
    n, lh, lw, s, outs, up, base, logits = case
    total = n * s * s * lh * lw
    entries = n * lh * lw
    per = s * s * lh * lw
    g_flow = up in ("flow", "both")
    names, labels = [], {"bwd: %s from %s" % ("+".join(outs), up), "logits: %s" % logits}
    if "g_mask" in outs:
        names.append("flow_compose_bwd_kernel")
        labels.add(_trip_label("g_mask", total, grid_for(total, sms=sms) * THREADS))
    if "g_low" in outs:
        names.append("flow_low_bwd_kernel")
        warps = grid_for(entries * 32, sms=sms) * THREADS // 32
        labels.add(_trip_label("g_low entries", entries, warps))
        terms = 9 * s * s
        labels.add("g_low lanes: %d terms, %s" % (terms, "idle lanes" if terms < 32 else "%d strides" % ceil_div(terms, 32)))
    if "g_base" in outs:
        if g_flow and base:
            names.append("flow_base_bwd_kernel")
            labels.add("g_base: %s" % ("fewer pixels than threads" if per < THREADS else "pixels = threads" if per == THREADS
                                       else "several trips per thread"))
        else:
            labels.add("g_base: zeroed by the entry (%s)" % ("no g_flow" if not g_flow else "no base warp"))
    return dict(names=names, labels=labels, lanes_chain=ceil_div(9 * s * s, 32), base_trips=ceil_div(per, THREADS))


def tv_route(case, sms=H100_SMS):
    n, h, w, data = case
    total = n * h * w * 2
    blocks = tv_blocks(total, sms)
    trips = ceil_div(total, blocks * THREADS)
    bwd_trips = ceil_div(total, 4 * blocks * THREADS)
    labels = {_trip_label("tv fwd", total, blocks * THREADS), "tv data: %s" % data,
              "tv finish: %s" % ("fewer than 256 partials" if blocks < 256 else "exactly 256 partials" if blocks == 256
                                 else "two trips (more than 256 partials)"),
              "tv bwd: %s" % ("one trip" if bwd_trips == 1 else "several trips")}
    if h == 2 and w == 2:
        labels.add("tv: H = W = 2")
    if h != w:
        labels.add("tv: non-square")
    return dict(blocks=blocks, trips=trips, finish_trips=ceil_div(blocks, 256), bwd_trips=bwd_trips, labels=labels)


def tvps_route(case):
    n, h, w, data = case
    per = h * w * 2
    trips = ceil_div(per, 512)
    lab = "tv_per_sample: %s" % ("fewer elements than threads" if per < 512 else "elements = threads" if per == 512
                                 else "several trips per thread")
    return dict(trips=trips, labels={lab, "tv data: %s" % data})


OPERANDS = ("p", "g", "m", "v", "ema")


def cta_map(numels, chunk):
    """fused_optim / scaled_weights: CTA -> (tensor, chunk) in table order."""
    return [(ti, c) for ti, nm in enumerate(numels) for c in range(ceil_div(nm, chunk))]


def adam_route(case):
    """gg_adam_ema_step for a hand-built table.  case: (name, rows, chunk); a row is (numel, {operand: element offset}, ema,
    lr group).  Allocations are 256-byte aligned, so an operand is 16-byte aligned iff its offset is a multiple of 4."""
    name, rows, chunk = case
    labels = set()
    blocks = cta_map([r[0] for r in rows], chunk)
    if not blocks:
        labels.add("adam: blocks == 0 (tick only)")
    for ti, c in blocks:
        numel, offs, ema, _ = rows[ti]
        e0, e1 = c * chunk, min(c * chunk + chunk, numel)
        bad = [op for op in OPERANDS if offs.get(op, 0) % 4 and (op != "ema" or ema)]
        vec = not bad and e0 % 4 == 0
        if vec:
            labels.add("adam: vector path")
            labels.add("adam: vector path, %s" % ("a scalar tail" if (e1 - e0) % 4 else "no tail"))
            if (e1 - e0) < 4:
                labels.add("adam: vector path with no float4 (fewer than 4 elements)")
        elif len(bad) == 1:
            labels.add("adam: scalar path, only %s misaligned" % bad[0])
        elif not bad:
            labels.add("adam: scalar path, e0 % 4 != 0")
        labels.add("adam: %s, %s" % ("with EMA" if ema else "no EMA twin", "vector" if vec else "scalar"))
        if c > 0:
            labels.add("adam: several chunks per tensor")
        if e1 - e0 < chunk:
            labels.add("adam: a partial last chunk")
    if len({r[3] for r in rows}) > 1:
        labels.add("adam: two learning-rate groups")
    return dict(blocks=blocks, labels=labels)


def scale_route(case):
    """gg_scale_cast_multi.  case: (name, rows); a row is (src dtype, dst dtype, numel, src offset, dst offset) in
    elements; an operand is 16-byte aligned iff offset * element size is a multiple of 16."""
    name, rows = case
    labels = set()
    for ti, c in cta_map([r[2] for r in rows], SCALE_CHUNK):
        sd, dd, numel, so, do = rows[ti]
        e0, e1 = c * SCALE_CHUNK, min(c * SCALE_CHUNK + SCALE_CHUNK, numel)
        vec = (so * ESIZE[sd]) % 16 == 0 and (do * ESIZE[dd]) % 16 == 0 and e0 % 4 == 0
        pair = "%s->%s" % (SHORT[sd], SHORT[dd])
        labels.add("scale-cast %s: %s" % (pair, "vector" if vec else "scalar"))
        if vec and (e1 - e0) % 4:
            labels.add("scale-cast %s: vector path's scalar tail" % pair)
        if not vec:
            labels.add("scale-cast: %s misaligned" % ("src" if (so * ESIZE[sd]) % 16 else "dst"))
        if c > 0:
            labels.add("scale-cast: several chunks per tensor")
    return dict(labels=labels)


# ------------------------------------------------------------------------------------------------------------- cases
FLOW_FWD_CASES = []
for _shape in [(2, 1, 1, 1), (2, 1, 1, 8), (3, 2, 2, 3), (2, 16, 16, 8), (1, 5, 7, 3), (2, 2, 16, 1), (1, 16, 3, 8)]:
    for _i, _cfg in enumerate(FWD_CONFIGS):
        FLOW_FWD_CASES.append(_shape + (_cfg, LOGITS[_i % 3]))
        FLOW_FWD_CASES.append(_shape + (_cfg, LOGITS[(_i + 1) % 3]))
FLOW_FWD_CASES += [(33, 16, 16, 8, "flow+base+alpha", "wide"), (34, 16, 16, 8, "flow+base+alpha", "narrow"),
                   (34, 16, 16, 8, "delta only", "ties")]

FLOW_BWD_CASES = []
_subsets = [tuple(o for o, b in zip(BWD_OUTPUTS, bits) if b) for bits in
            [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)]]
for _j, _shape in enumerate([(2, 1, 1, 1), (2, 2, 2, 3), (2, 16, 16, 8), (1, 5, 7, 3), (3, 2, 3, 2), (1, 4, 4, 4)]):
    for _i, _outs in enumerate(_subsets):
        for _up in UPSTREAM:
            FLOW_BWD_CASES.append(_shape + (_outs, _up, True, LOGITS[(_i + _j) % 3]))
FLOW_BWD_CASES += [(2, 3, 5, 2, ("g_mask", "g_low", "g_base"), "both", False, "wide"),
                   (66, 16, 16, 1, ("g_mask", "g_low", "g_base"), "both", True, "narrow"),
                   (67, 16, 16, 1, ("g_mask", "g_low", "g_base"), "both", True, "wide"),
                   (34, 16, 16, 8, ("g_mask", "g_low", "g_base"), "both", True, "narrow")]

TV_CASES = [(1, 2, 2, "exact knee"), (3, 2, 2, "random"), (2, 5, 7, "exact knee"), (1, 3, 64, "random"),
            (2, 16, 16, "random"), (2, 128, 128, "exact knee"), (2, 128, 128, "random"), (1, 160, 240, "random"),
            (1, 264, 256, "exact knee"), (1, 264, 257, "random"), (2, 400, 400, "random"), (2, 400, 400, "exact knee")]
TVPS_CASES = [(3, 2, 2, "exact knee"), (2, 5, 7, "random"), (2, 16, 16, "exact knee"), (1, 13, 20, "random"),
              (4, 128, 128, "random"), (2, 33, 17, "exact knee")]

_A = dict(p=0, g=0, m=0, v=0, ema=0)
ADAM_CASES = [
    ("aligned", [(2 * ADAM_CHUNK + 5, {}, True, 0), (1000, {}, True, 1), (7, {}, False, 0), (3, {}, True, 1),
                 (ADAM_CHUNK, {}, False, 1)], ADAM_CHUNK),
] + [("%s misaligned" % op, [(ADAM_CHUNK + 9, {op: 1}, True, 0), (70, {op: 3}, True, 1), (6, {}, False, 0)], ADAM_CHUNK)
     for op in OPERANDS] + [
    ("chunk 1026", [(5000, {}, True, 0), (1030, {}, False, 1)], 1026),
    ("no tensors", [], ADAM_CHUNK),
]

SCALE_CASES = []
for _sd in (F32, BF16):
    for _dd in (F32, BF16):
        SCALE_CASES.append(("%s->%s aligned" % (SHORT[_sd], SHORT[_dd]),
                            [(_sd, _dd, 2 * SCALE_CHUNK + 3, 0, 0), (_sd, _dd, 100, 0, 0), (_sd, _dd, 5, 0, 0),
                             (_sd, _dd, 3, 0, 0)]))
        SCALE_CASES.append(("%s->%s src misaligned" % (SHORT[_sd], SHORT[_dd]),
                            [(_sd, _dd, SCALE_CHUNK + 7, 1, 0), (_sd, _dd, 33, 3, 0), (_sd, _dd, 8, 0, 0)]))
        SCALE_CASES.append(("%s->%s dst misaligned" % (SHORT[_sd], SHORT[_dd]),
                            [(_sd, _dd, SCALE_CHUNK + 7, 0, 1), (_sd, _dd, 33, 0, 2)]))

REQUIRED = (
    ["flow fwd: one partial trip", "flow fwd: exactly one full trip", "flow fwd: a second, partial trip"]
    + ["fwd: %s" % c for c in FWD_CONFIGS] + ["logits: %s" % lg for lg in LOGITS]
    + ["flow fwd: s = %d" % s for s in (1, 3, 8)]
    + ["flow fwd: a 1-wide low-resolution side (every neighbour but one padded)", "flow fwd: non-square"]
    + ["bwd: %s from %s" % ("+".join(o), u) for o in _subsets for u in UPSTREAM]
    + ["g_mask: one partial trip", "g_mask: exactly one full trip", "g_mask: a second, partial trip",
       "g_low entries: one partial trip", "g_low entries: exactly one full trip", "g_low entries: a second, partial trip",
       "g_low lanes: 9 terms, idle lanes", "g_low lanes: 36 terms, 2 strides", "g_low lanes: 81 terms, 3 strides",
       "g_low lanes: 576 terms, 18 strides",
       "g_base: fewer pixels than threads", "g_base: pixels = threads", "g_base: several trips per thread",
       "g_base: zeroed by the entry (no g_flow)", "g_base: zeroed by the entry (no base warp)"]
    + ["tv fwd: one partial trip", "tv fwd: exactly one full trip", "tv fwd: a second, partial trip", "tv fwd: several trips",
       "tv finish: fewer than 256 partials", "tv finish: exactly 256 partials", "tv finish: two trips (more than 256 partials)",
       "tv bwd: one trip", "tv bwd: several trips", "tv: H = W = 2", "tv: non-square", "tv data: exact knee",
       "tv data: random", "tv_per_sample: fewer elements than threads", "tv_per_sample: elements = threads",
       "tv_per_sample: several trips per thread"]
    + ["adam: vector path", "adam: vector path, a scalar tail", "adam: vector path, no tail",
       "adam: vector path with no float4 (fewer than 4 elements)", "adam: scalar path, e0 % 4 != 0",
       "adam: with EMA, vector", "adam: with EMA, scalar", "adam: no EMA twin, vector", "adam: no EMA twin, scalar",
       "adam: several chunks per tensor", "adam: a partial last chunk", "adam: blocks == 0 (tick only)",
       "adam: two learning-rate groups"]
    + ["adam: scalar path, only %s misaligned" % op for op in OPERANDS]
    + ["scale-cast %s->%s: %s" % (SHORT[a], SHORT[b], r) for a in (F32, BF16) for b in (F32, BF16) for r in ("vector", "scalar")]
    + ["scale-cast %s->%s: vector path's scalar tail" % (SHORT[a], SHORT[b]) for a in (F32, BF16) for b in (F32, BF16)]
    + ["scale-cast: src misaligned", "scale-cast: dst misaligned", "scale-cast: several chunks per tensor"]
)


def all_labels(sms=H100_SMS):
    reached = set()
    for cs in FLOW_FWD_CASES:
        reached |= flow_fwd_route(cs, sms)["labels"]
    for cs in FLOW_BWD_CASES:
        reached |= flow_bwd_route(cs, sms)["labels"]
    for cs in TV_CASES:
        reached |= tv_route(cs, sms)["labels"]
    for cs in TVPS_CASES:
        reached |= tvps_route(cs)["labels"]
    for cs in ADAM_CASES:
        reached |= adam_route(cs)["labels"]
    for cs in SCALE_CASES:
        reached |= scale_route(cs)["labels"]
    return reached


def test_cases_reach_every_route():
    """Coverage of the cases below, by the restatement planned for 132 SMs: the grid-stride trips of the flow forward and
    g_mask (N = 33 at 128^2 is exactly one full trip, N = 34 a second, partial one), g_low's entry trips (N = 66 / 67 at
    16^2) and lane strides (s = 1, 2, 3, 8), g_base's per-thread trips, every backward output subset from each upstream
    gradient, both sides of each TV trip and finish threshold, every Adam / scale-cast gate outcome (each operand
    misaligned on its own, e0 % 4 != 0, tails, rows without an EMA twin, all four dtype pairs) and a tick-only Adam step."""
    from gangealing_b200.op import scaled_weights
    from gangealing_b200.training import fused_optim
    assert fused_optim._CHUNK == ADAM_CHUNK and scaled_weights._CHUNK == SCALE_CHUNK
    reached = all_labels()
    assert_routes_reached(REQUIRED, reached)


def test_restated_tv_blocks_match_the_workspace_query():
    """tv_route's CTA count agrees with gg_tv_loss_workspace (one fp32 partial per CTA), planned for the SM count the
    library sees (132 without a device)."""
    from gangealing_b200 import _lib
    lib = _lib.load()
    sms = _lib.sm_count()
    for cs in TV_CASES:
        n, h, w, _ = cs
        assert lib.gg_tv_loss_workspace(n, h, w) == tv_route(cs, sms)["blocks"] * 4, cs


# ======================================================================================================== GPU checks
WORST = Worst("k (stored values) / c (sums) per path", "%-48s %.2f")
_report_worst = WORST.fixture()


def check(y, ref, a, c, path, what, extra=None):
    obs = assert_fp32_sum(y, ref, a, c, "%s: %s" % (path, what), extra64=extra)
    WORST.note(path, obs)
    print("[contract] %s: %s: obs=%.2f (bound %g)" % (path, what, obs, c))


def nan_like(shape):
    return torch.full(shape, float("nan"), dtype=F32, device=DEV)


# ------------------------------------------------------------------------------------------------ flow composition
def flow_inputs(n, lh, lw, s, logits, seed):
    g = seeded(seed)
    low = torch.randn(n, lh, lw, 2, generator=g, device=DEV) * 0.3
    if logits == "narrow":
        mask = torch.randn(n, 9 * s * s, lh, lw, generator=g, device=DEV) * 0.5
    elif logits == "wide":
        mask = (torch.rand(n, 9 * s * s, lh, lw, generator=g, device=DEV) * 2 - 1) * 20
    else:                      # exact ties: a few integer levels, so several logits share the maximum
        mask = torch.randint(-1, 2, (n, 9 * s * s, lh, lw), generator=g, device=DEV).float()
    hf, wf = lh * s, lw * s
    ys = (2 * torch.arange(hf, device=DEV, dtype=torch.float64) + 1) / hf - 1
    xs = (2 * torch.arange(wf, device=DEV, dtype=torch.float64) + 1) / wf - 1
    ident = torch.stack(torch.meshgrid(xs, ys, indexing="xy"), -1).float().reshape(1, hf, wf, 2).contiguous()
    base = (torch.eye(2, 3, device=DEV) + torch.randn(n, 2, 3, generator=g, device=DEV) * 0.3).contiguous()
    alpha = torch.rand(n, generator=g, device=DEV)
    return low, mask, ident, base, alpha


def to_mask_order(t, s):
    """(N, lh*s, lw*s) full-resolution plane -> (N, s, s, lh, lw), the order of the mask's pixel axes."""
    n, hf, wf = t.shape
    return t.view(n, hf // s, s, wf // s, s).permute(0, 2, 4, 1, 3)


def to_full(t):
    """(N, s, s, lh, lw) -> (N, lh*s, lw*s)."""
    n, s, _, lh, lw = t.shape
    return t.permute(0, 3, 1, 4, 2).reshape(n, lh * s, lw * s)


def convex64(low, mask, s):
    """float64 convex up-sampling on the kernel's operands: softmax weights p (N, 9, s, s, lh, lw), the scaled neighbours
    fx, fy (N, 9, 1, 1, lh, lw) and the per-weight spread |d_k| + sum_j p_j |d_j|, d = logit - max."""
    n, lh, lw, _ = low.shape
    L = mask.double().view(n, 9, s, s, lh, lw)
    d = L - L.amax(1, keepdim=True)
    p = torch.softmax(L, 1)
    pad = F.pad(low.double().permute(0, 3, 1, 2), (1, 1, 1, 1))
    nb = torch.stack([pad[:, :, ky:ky + lh, kx:kx + lw] for ky in range(3) for kx in range(3)], 1) * s
    fx, fy = nb[:, :, 0][:, :, None, None], nb[:, :, 1][:, :, None, None]
    spread = d.abs() + (p * d.abs()).sum(1, keepdim=True)
    return p, fx, fy, spread


# delta = fmaf chain over 9 terms p_k * (s*f_k).  Per term: expf 2 ulp (4u) and the rounded l_k - max (|d_k| u) in the
# weight, the 8 additions of the softmax denominator (8u, plus the weighted average of the weights' errors, S + 4), the
# reciprocal and the product (2u), s*f (1u) and the 9-step chain (9u): 28 + |d_k| + S.
K_DELTA = 28
# A stored composed grid, from the stored delta: id + delta (1 rounding); the base warp M0 gx + M1 gy + M2 (3 more on the
# terms, the first one propagated: 4); the alpha lerp id + a (g - id) (3 more).
K_ID, K_BASE, K_ALPHA = 1, 4, 3


def compose64(delta, ident, base, alpha):
    d = delta.double()
    idn = ident.double()
    gx, gy = idn[..., 0] + d[..., 0], idn[..., 1] + d[..., 1]
    ax, ay = idn[..., 0].abs() + d[..., 0].abs(), idn[..., 1].abs() + d[..., 1].abs()
    k = K_ID
    if base is not None:
        M = base.double().view(-1, 1, 1, 6)
        M = [M[..., i] for i in range(6)]
        gx, gy = M[0] * gx + M[1] * gy + M[2], M[3] * gx + M[4] * gy + M[5]
        ax, ay = (M[0].abs() * ax + M[1].abs() * ay + M[2].abs(), M[3].abs() * ax + M[4].abs() * ay + M[5].abs())
        k = K_BASE
    if alpha is not None:
        a = alpha.double().view(-1, 1, 1)
        ix, iy = idn[..., 0], idn[..., 1]
        gx, gy = ix + a * (gx - ix), iy + a * (gy - iy)
        ax, ay = ix.abs() + a.abs() * (ax + ix.abs()), iy.abs() + a.abs() * (ay + iy.abs())
        k += K_ALPHA
    return torch.stack([gx, gy], -1), torch.stack([ax, ay], -1), k


def _fwd_id(cs):
    return "N%d-%dx%d-s%d-%s-%s" % (cs[0], cs[1], cs[2], cs[3], cs[4].replace(" ", "_").replace("+", "_"), cs[5])


@pytest.mark.gpu
@pytest.mark.parametrize("case", FLOW_FWD_CASES, ids=_fwd_id)
def test_flow_compose_forward(case):
    n, lh, lw, s, cfg, logits = case
    low, mask, ident, base, alpha = flow_inputs(n, lh, lw, s, logits, seed=n * 1000 + lh * 31 + s)
    want_flow = cfg != "delta only"
    base_a = base if "base" in cfg else None
    alpha_a = None
    if "alpha" in cfg:
        alpha_a = alpha if "broadcast" not in cfg else alpha[:1].contiguous()
    delta = nan_like((n, lh * s, lw * s, 2))
    flow = nan_like((n, lh * s, lw * s, 2)) if want_flow else None
    alpha_n = None if alpha_a is None else alpha_a.expand(n).contiguous()
    lib = library()
    rc = lib.load().gg_flow_compose_forward(delta.data_ptr(), lib.ptr(flow), low.data_ptr(), mask.data_ptr(),
                                            lib.ptr(ident if want_flow else None), lib.ptr(base_a), lib.ptr(alpha_n),
                                            n, lh, lw, s, lib.stream())
    lib.check(rc, "gg_flow_compose_forward")
    p, fx, fy, spread = convex64(low, mask, s)
    for c, fc in ((0, fx), (1, fy)):
        terms = p * fc
        ref = to_full(terms.sum(1))
        a = to_full(terms.abs().sum(1))
        extra = U32 * to_full((terms.abs() * spread).sum(1))
        check(delta[..., c], ref, a, K_DELTA, "flow fwd delta", "%s %s" % (_fwd_id(case), "xy"[c]), extra)
    if want_flow:
        ref, a, k = compose64(delta, ident, base_a, alpha_n)
        check(flow, ref, a, k, "flow fwd flow", _fwd_id(case))
    # the Python faces run the same launch
    from gangealing_b200.stn.flow import flow_compose, upsample_flow
    if want_flow:
        d2, f2 = flow_compose(low, mask, ident, base_a, alpha_a, s)
        assert torch.equal(d2, delta) and torch.equal(f2, flow)
    else:
        assert torch.equal(upsample_flow(low, mask, s), delta)


def bwd64(low, mask, ident, base, alpha, s, g_delta, g_flow):
    """float64 backward on the kernel's operands, in mask order -> dict of per-pixel gradients and their abs bounds."""
    n, lh, lw, _ = low.shape
    p, fx, fy, spread = convex64(low, mask, s)
    cx, cy = (p * fx), (p * fy)
    z = torch.zeros(n, s, s, lh, lw, dtype=torch.float64, device=DEV)
    gdx, gdy, agx, agy = z.clone(), z.clone(), z.clone(), z.clone()
    k_gd = 0
    out = dict(p=p, fx=fx, fy=fy, spread=spread)
    if g_delta is not None:
        gd = g_delta.double()
        gdx, gdy = to_mask_order(gd[..., 0], s), to_mask_order(gd[..., 1], s)
        agx, agy = gdx.abs(), gdy.abs()
    if g_flow is not None:
        gf = g_flow.double()
        gfx, gfy = to_mask_order(gf[..., 0], s), to_mask_order(gf[..., 1], s)
        if alpha is not None:
            a = alpha.double().view(n, 1, 1, 1, 1)
            gfx, gfy = gfx * a, gfy * a
        if base is not None:
            M = [base.double().view(n, 6)[:, i].view(n, 1, 1, 1, 1) for i in range(6)]
            idx = to_mask_order(ident.double()[..., 0].expand(n, -1, -1), s)
            idy = to_mask_order(ident.double()[..., 1].expand(n, -1, -1), s)
            gx, gy = idx + cx.sum(1), idy + cy.sum(1)
            Gx, Gy = idx.abs() + cx.abs().sum(1), idy.abs() + cy.abs().sum(1)
            sx, sy = (cx.abs() * spread).sum(1), (cy.abs() * spread).sum(1)
            ax, ay = gfx.abs(), gfy.abs()
            out["v"] = [gfx * gx, gfx * gy, gfx, gfy * gx, gfy * gy, gfy]
            out["v_abs"] = [ax * Gx, ax * Gy, ax, ay * Gx, ay * Gy, ay]
            out["v_spread"] = [ax * sx, ax * sy, 0 * ax, ay * sx, ay * sy, 0 * ay]
            px, py = M[0] * gfx + M[3] * gfy, M[1] * gfx + M[4] * gfy
            apx, apy = M[0].abs() * ax + M[3].abs() * ay, M[1].abs() * ax + M[4].abs() * ay
            k_gd = 4          # alpha product, the two roundings of M^T g, the add to g_delta
        else:
            px, py, apx, apy = gfx, gfy, gfx.abs(), gfy.abs()
            k_gd = 2
        gdx, gdy, agx, agy = gdx + px, gdy + py, agx + apx, agy + apy
    out.update(gdx=gdx, gdy=gdy, agx=agx, agy=agy, k_gd=k_gd)
    return out


def gather_low(q):
    """(N, 9, lh, lw) terms of pixel block (h, w) for neighbour k -> (N, lh, lw) sums at the entries (h + ky - 1, w + kx - 1)."""
    _, _, lh, lw = q.shape
    qp = F.pad(q, (1, 1, 1, 1))
    return sum(qp[:, 3 * ky + kx, 2 - ky:2 - ky + lh, 2 - kx:2 - kx + lw] for ky in range(3) for kx in range(3))


def _bwd_id(cs):
    return "N%d-%dx%d-s%d-%s-from_%s%s-%s" % (cs[0], cs[1], cs[2], cs[3], "+".join(cs[4]), cs[5], "" if cs[6] else "-nobase", cs[7])


def flow_bwd_run(case, seed):
    n, lh, lw, s, outs, up, with_base, logits = case
    low, mask, ident, base, alpha = flow_inputs(n, lh, lw, s, logits, seed)
    base = base if with_base else None
    g = seeded(seed + 1)
    g_delta = torch.randn(n, lh * s, lw * s, 2, generator=g, device=DEV) if up in ("delta", "both") else None
    g_flow = torch.randn(n, lh * s, lw * s, 2, generator=g, device=DEV) if up in ("flow", "both") else None
    o = dict(g_mask=nan_like(mask.shape) if "g_mask" in outs else None,
             g_low=nan_like(low.shape) if "g_low" in outs else None,
             g_base=nan_like((n, 2, 3)) if "g_base" in outs else None)
    lib = library()
    rc = lib.load().gg_flow_compose_backward(lib.ptr(o["g_mask"]), lib.ptr(o["g_low"]), lib.ptr(o["g_base"]), lib.ptr(g_delta),
                                             lib.ptr(g_flow), low.data_ptr(), mask.data_ptr(), ident.data_ptr(), lib.ptr(base),
                                             alpha.data_ptr(), n, lh, lw, s, lib.stream())
    lib.check(rc, "gg_flow_compose_backward")
    return (low, mask, ident, base, alpha, g_delta, g_flow), o


@pytest.mark.gpu
@pytest.mark.parametrize("case", FLOW_BWD_CASES, ids=_bwd_id)
def test_flow_compose_backward(case):
    n, lh, lw, s, outs, up, with_base, logits = case
    route = flow_bwd_route(case)
    (low, mask, ident, base, alpha, g_delta, g_flow), o = flow_bwd_run(case, seed=7 * n + lh + 100 * s)
    r = bwd64(low, mask, ident, base, alpha, s, g_delta, g_flow)
    p, fx, fy, spread, k_gd = r["p"], r["fx"], r["fy"], r["spread"], r["k_gd"]
    gdx, gdy, agx, agy = (r[k][:, None] for k in ("gdx", "gdy", "agx", "agy"))
    cid = _bwd_id(case)
    if o["g_mask"] is not None:
        # t_k = <g, s f_k> (k_gd + 1 + 2), t_bar = 9-step chain over p_j t_j, (t_k - t_bar) and the product with p_k, each
        # weight carrying 18 + |d| + S: c = k_gd + 50 against A = p_k (T_k + sum_j p_j T_j), T_k = |g| . |s f_k|
        t = gdx * fx + gdy * fy
        T = agx * fx.abs() + agy * fy.abs()
        pT = (p * T).sum(1, keepdim=True)
        ref = p * (t - (p * t).sum(1, keepdim=True))
        a = p * (T + pT)
        extra = U32 * p * ((p * T * spread).sum(1, keepdim=True) + spread * (T + pT))
        check(o["g_mask"], ref.reshape(mask.shape), a.reshape(mask.shape), k_gd + 50, "flow bwd g_mask", cid,
              extra.reshape(mask.shape))
    if o["g_low"] is not None:
        # terms s p_k gd: the weight (18 + |d| + S) and s*p (1), gd (k_gd), the lane's fma chain (ceil(9 s^2 / 32)) and the
        # 5-step butterfly
        c = k_gd + route["lanes_chain"] + 24
        for ci, (gd, ag) in enumerate(((gdx, agx), (gdy, agy))):
            terms = s * p * gd
            ab = s * p * ag
            ref = gather_low(terms.sum((2, 3)))
            a = gather_low(ab.sum((2, 3)))
            extra = U32 * gather_low((ab * spread).sum((2, 3)))
            check(o["g_low"][..., ci], ref, a, c, "flow bwd g_low", "%s %s" % (cid, "xy"[ci]), extra)
    if o["g_base"] is not None:
        if g_flow is None or base is None:
            assert bool((o["g_base"] == 0).all()), "%s: g_base must be written as exact zeros" % cid
        else:
            # v = g' (id + delta): the alpha product (1), id + delta (1 + the delta's 28), the product (1); then the
            # per-thread trips, the 5-step butterfly and the 8 warp partials
            c = 31 + route["base_trips"] + 5 + 8
            ref = torch.stack([v.sum((1, 2, 3, 4)) for v in r["v"]], 1)
            a = torch.stack([v.sum((1, 2, 3, 4)) for v in r["v_abs"]], 1)
            extra = U32 * torch.stack([v.sum((1, 2, 3, 4)) for v in r["v_spread"]], 1)
            check(o["g_base"].view(n, 6), ref, a, c, "flow bwd g_base", cid, extra)


@pytest.mark.gpu
def test_flow_backward_faces_match_the_entry():
    """The autograd face hands the kernel the same operands: its gradients equal a direct call bitwise."""
    from gangealing_b200.stn.flow import flow_compose
    n, lh, lw, s = 2, 4, 5, 3
    low, mask, ident, base, alpha = flow_inputs(n, lh, lw, s, "narrow", 11)
    args = [t.clone().requires_grad_(True) for t in (low, mask, base)]
    d, f = flow_compose(args[0], args[1], ident, args[2], alpha, s)
    g = seeded(12)
    gd, gf = torch.randn(d.shape, generator=g, device=DEV), torch.randn(f.shape, generator=g, device=DEV)
    got = torch.autograd.grad([d, f], args, [gd, gf])
    o = dict(g_mask=torch.empty_like(mask), g_low=torch.empty_like(low), g_base=torch.empty(n, 2, 3, device=DEV))
    lib = library()
    lib.check(lib.load().gg_flow_compose_backward(o["g_mask"].data_ptr(), o["g_low"].data_ptr(), o["g_base"].data_ptr(),
                                                  gd.data_ptr(), gf.data_ptr(), low.data_ptr(), mask.data_ptr(),
                                                  ident.data_ptr(), base.data_ptr(), alpha.data_ptr(), n, lh, lw, s,
                                                  lib.stream()), "gg_flow_compose_backward")
    assert torch.equal(got[0], o["g_low"]) and torch.equal(got[1], o["g_mask"]) and torch.equal(got[2], o["g_base"])


# ------------------------------------------------------------------------------------------------ misaligned views
def offset_copy(t, off=1):
    """A contiguous view of `t`'s values that starts `off` elements into a fresh buffer: off a 16-byte boundary."""
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=t.device)
    v = buf[off:].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 != 0
    return v


@pytest.mark.gpu
def test_flow_faces_on_offset_views_match_aligned_copies():
    """flow_compose / upsample_flow / stn_sample_flow on contiguous views that start 4 bytes off (low, identity, the
    upstream gradients) give the values of the aligned copies bitwise: the faces hand the kernels aligned copies."""
    from gangealing_b200.stn.flow import flow_compose, upsample_flow
    from gangealing_b200.stn.sampling import stn_sample_flow
    n, lh, lw, s = 2, 4, 4, 8
    low, mask, ident, base, alpha = flow_inputs(n, lh, lw, s, "narrow", 21)
    g = seeded(22)
    gd, gf = torch.randn(n, lh * s, lw * s, 2, generator=g, device=DEV), torch.randn(n, lh * s, lw * s, 2, generator=g, device=DEV)

    def run(lo, mk, idn, gdd, gff):
        lo = lo.detach().requires_grad_(True)
        mk = mk.detach().requires_grad_(True)
        bs = base.clone().requires_grad_(True)
        d, f = flow_compose(lo, mk, idn, bs, alpha, s)
        grads = torch.autograd.grad([d, f], [lo, mk, bs], [gdd, gff])
        return (d, f, upsample_flow(lo, mk, s)) + grads
    want = run(low, mask, ident, gd, gf)
    got = run(offset_copy(low), offset_copy(mask), offset_copy(ident), offset_copy(gd), offset_copy(gf))
    for w, y in zip(want, got):
        assert torch.equal(w, y)
    img = torch.randn(n, 3, lh * s, lw * s, generator=g, device=DEV)
    for levels in (None, 3):
        w = stn_sample_flow(img, low, mask, ident, base, alpha, s, max_num_levels=levels)
        y = stn_sample_flow(img, offset_copy(low), mask, offset_copy(ident), base, alpha, s, max_num_levels=levels)
        for a, b in zip(w, y):
            assert (a is None and b is None) or torch.equal(a, b)


@pytest.mark.gpu
def test_sampler_faces_on_offset_views_match_aligned_copies():
    """mipmap_warp (and its grid gradient), sample_indices, mipmap_warp_lerp and mipmap_warp_lerp_mean on grids that
    start 4 bytes off give the values of the aligned copies bitwise."""
    from gangealing_b200.stn.sampling import mipmap_warp, mipmap_warp_lerp, mipmap_warp_lerp_mean, sample_indices
    g = seeded(31)
    n, ho, wo = 2, 12, 20
    img = torch.randn(n, 3, 32, 32, generator=g, device=DEV)
    grid = (torch.rand(n, ho, wo, 2, generator=g, device=DEV) * 2 - 1) * 1.1
    target = (torch.rand(n, ho, wo, 2, generator=g, device=DEV) * 2 - 1)
    alphas = torch.tensor([0.0, 0.3, 1.0], device=DEV)
    go = torch.randn(n, 3, ho, wo, generator=g, device=DEV)

    def warp(gr):
        gr = gr.detach().requires_grad_(True)
        out, lev = mipmap_warp(img, gr, max_num_levels=3)
        (gg,) = torch.autograd.grad(out, gr, go)
        return out, lev, gg
    for w, y in zip(warp(grid), warp(offset_copy(grid))):
        assert torch.equal(w, y)
    assert torch.equal(sample_indices(grid, (32, 32)), sample_indices(offset_copy(grid), (32, 32)))
    for w, y in zip(mipmap_warp_lerp(img, grid, target, alphas), mipmap_warp_lerp(img, offset_copy(grid), offset_copy(target), alphas)):
        assert torch.equal(w, y)
    assert torch.equal(mipmap_warp_lerp_mean(img, grid[:1], target, alphas),
                       mipmap_warp_lerp_mean(img, offset_copy(grid[:1]), offset_copy(target), alphas))


# ------------------------------------------------------------------------------------------------ total variation
def tv_flow(n, h, w, data, seed):
    g = torch.Generator().manual_seed(seed)
    if data == "random":
        f = torch.randn(n, h, w, 2, generator=g) * 1.5            # differences on both sides of the knee
    else:
        # values on the 2^-23 grid below 1.25 + 2^-23: every difference is exact in fp32, and many are exactly +-1 and
        # +-(1 +- 2^-23), so the kernel's branch at the knee is decided without rounding
        base = torch.randint(0, 2, (n, h, w, 2), generator=g).double() * 0.25
        off = torch.tensor([0.0, 1.0, 1 - 2.0 ** -23, 1 + 2.0 ** -23], dtype=torch.float64)
        f = (base + off[torch.randint(0, 4, (n, h, w, 2), generator=g)]).float()
    return f.to(DEV).contiguous()


def _diffs(f):
    f = f.double()
    return f[:, :-1] - f[:, 1:], f[:, :, :-1] - f[:, :, 1:]


def huber64(d):
    a = d.abs()
    return torch.where(a <= 1, 0.5 * a * a, a - 0.5)


def hgrad64(d):
    return torch.where(d.abs() <= 1, d, torch.sign(d))


def tv_invs(n, h, w):
    """The kernel's fp32 weights 1 / (N (H-1) W 2) and 1 / (N H (W-1) 2), in its operation order."""
    one, two = np.float32(1), np.float32(2)
    inv_y = one / (np.float32(n) * np.float32(h - 1) * np.float32(w) * two)
    inv_x = one / (np.float32(n) * np.float32(h) * np.float32(w - 1) * two)
    return float(inv_y), float(inv_x)


def _tv_id(cs):
    return "N%d-%dx%d-%s" % (cs[0], cs[1], cs[2], cs[3].replace(" ", "_"))


@pytest.mark.gpu
@pytest.mark.parametrize("case", TV_CASES, ids=_tv_id)
def test_tv_loss(case):
    n, h, w, data = case
    route = tv_route(case)
    f = tv_flow(n, h, w, data, seed=n * h + w)
    dy, dx = _diffs(f)
    if data == "exact knee":
        assert torch.equal(dx.float().double(), dx) and torch.equal(dy.float().double(), dy)
        if dx.numel() >= 64:
            assert all(bool((dx.abs() == v).any()) for v in (1.0, 1 + 2.0 ** -23, 1 - 2.0 ** -23))
    inv_y, inv_x = tv_invs(n, h, w)
    lib = library()
    dll = lib.load()
    out = nan_like((1,))
    ws = nan_like((dll.gg_tv_loss_workspace(n, h, w) // 4,))
    lib.check(dll.gg_tv_loss_forward(out.data_ptr(), ws.data_ptr(), f.data_ptr(), n, h, w, lib.stream()), "gg_tv_loss_forward")
    ref = huber64(dy).sum() * inv_y + huber64(dx).sum() * inv_x
    a = (huber64(dy) + dy.abs()).sum() * inv_y + (huber64(dx) + dx.abs()).sum() * inv_x
    # a term: the rounded difference and the Huber branch (3); two fmas per element per trip; 5-step butterfly, 8 warp
    # partials; the finish's trips over the partials, its butterfly and its 8 warp partials
    c = 3 + 2 * route["trips"] + 5 + 8 + route["finish_trips"] + 5 + 8
    check(out.view(()), ref, a, c, "tv fwd", _tv_id(case))
    go = torch.tensor([2.5], device=DEV)
    grad = nan_like(f.shape)
    lib.check(dll.gg_tv_loss_backward(grad.data_ptr(), go.data_ptr(), f.data_ptr(), n, h, w, lib.stream()), "gg_tv_loss_backward")
    hy, hx = hgrad64(dy) * inv_y, hgrad64(dx) * inv_x
    G = torch.zeros(f.shape, dtype=torch.float64, device=DEV)
    A = torch.zeros_like(G)
    G[:, :-1] += hy
    G[:, 1:] -= hy
    G[:, :, :-1] += hx
    G[:, :, 1:] -= hx
    A[:, :-1] += hy.abs()
    A[:, 1:] += hy.abs()
    A[:, :, :-1] += hx.abs()
    A[:, :, 1:] += hx.abs()
    # huber'(d) is d or +-1 (the rounded difference: 1), a chain of up to 4 fmas (4), the product with the upstream (1)
    check(grad, 2.5 * G, 2.5 * A, 6, "tv bwd", _tv_id(case))


@pytest.mark.gpu
@pytest.mark.parametrize("case", TVPS_CASES, ids=_tv_id)
def test_tv_per_sample(case):
    from gangealing_b200.evaluation.ops import tv_per_sample
    n, h, w, data = case
    f = tv_flow(n, h, w, data, seed=3 * n + h * w)
    dy, dx = _diffs(f)
    got = tv_per_sample(f)
    cy, cx = (h - 1) * w * 2, h * (w - 1) * 2
    ref = huber64(dy).sum((1, 2, 3)) / cy + huber64(dx).sum((1, 2, 3)) / cx
    a = (huber64(dy) + dy.abs()).sum((1, 2, 3)) / cy + (huber64(dx) + dx.abs()).sum((1, 2, 3)) / cx
    # the term (3), the per-thread trips, the 5-step butterfly, 16 warp partials, the two divisions and the final add
    c = 3 + tvps_route(case)["trips"] + 5 + 16 + 2
    check(got, ref, a, c, "tv per sample", _tv_id(case))


# ------------------------------------------------------------------------------------------------ Adam + EMA
def _hyper():
    """The kernel's fp32 hyper-parameters: 1 - b1, b2, 1 - b2, eps, decay, 1 - decay (the differences formed in double)."""
    b1, b2 = BETAS
    return tuple(f32(x) for x in (1.0 - b1, b2, 1.0 - b2, EPS, DECAY, 1.0 - DECAY))


def adam_expect(before, after, lr, state, ema):
    """Check one step's stored outputs against float64 on that step's stored inputs.  before / after: (p, g, m, v, ema)."""
    omb1, b2, omb2, eps, decay, omd = _hyper()
    p, g, m, v, e = (None if t is None else t.double() for t in before)
    p1, m1, v1, e1 = (None if t is None else t.double() for t in (after[0], after[2], after[3], after[4]))
    res = {}
    # m' = fmaf(1-b1, g - m, m): the difference and the fma (2, and 1 for the second-order terms of a bound this tight)
    res["m"] = (m + omb1 * (g - m), m.abs() + omb1 * (g.abs() + m.abs()), 3)
    # v' = fmaf((1-b2) g, g, b2 v): (1-b2) g, b2 v and the fma (2, and 1 as above)
    res["v"] = (omb2 * g * g + b2 * v, omb2 * g * g + b2 * v, 3)
    # p' from the stored m', v': sqrt, 1/state[2], the product, + eps (4), the quotient (1), lr / state[1] (1), the
    # product with it (1) and the subtraction (1): 8 against |p| + |update|
    s1, s2 = float(state[1]), float(state[2])
    upd = (float(lr) / s1) * m1 / (v1.sqrt() / s2 + eps)
    res["p"] = (p - upd, p.abs() + upd.abs(), 8)
    if e is not None:
        # ema' = fmaf(decay, e, (1-decay) p'): on the stored p' (2, and 1 as above)
        res["ema"] = (decay * e + omd * p1, decay * e.abs() + omd * p1.abs(), 3)
    return res


def _adam_table(rows):
    return torch.tensor([[p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), 0 if e is None else e.data_ptr(),
                          p.numel(), lr.data_ptr()] for p, g, m, v, e, lr in rows], dtype=torch.int64).to(DEV)


def _operand(numel, off, gen, scale=1.0, positive=False):
    buf = torch.empty(numel + off, device=DEV)
    t = buf[off:]
    t.copy_((torch.rand(numel, generator=gen, device=DEV) if positive else torch.randn(numel, generator=gen, device=DEV)) * scale)
    return t


def _grad_values(numel, gen):
    """Gradients spanning 1e-6 .. 1e3, every 17th one exactly zero."""
    g = torch.randn(numel, generator=gen, device=DEV) * 10.0 ** (torch.rand(numel, generator=gen, device=DEV) * 9 - 6)
    g[::17] = 0
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("case", ADAM_CASES, ids=lambda cs: cs[0].replace(" ", "_"))
def test_adam_ema_step(case):
    name, spec, chunk = case
    gen = seeded(sum(map(ord, name)))
    lrs = [torch.tensor(1e-3, device=DEV), torch.tensor(3e-2, device=DEV)]
    rows = []
    for numel, offs, ema, grp in spec:
        o = {op: offs.get(op, 0) for op in OPERANDS}
        p = _operand(numel, o["p"], gen)
        gr = _operand(numel, o["g"], gen)
        m = _operand(numel, o["m"], gen, 1e-2)
        v = _operand(numel, o["v"], gen, 1e-3, positive=True)
        e = _operand(numel, o["ema"], gen) if ema else None
        rows.append([p, gr, m, v, e, lrs[grp]])
    table = _adam_table(rows) if rows else None
    cmap = cta_map([r[0] for r in spec], chunk)
    bt = torch.tensor([t for t, _ in cmap] or [0], dtype=torch.int32, device=DEV)
    bc = torch.tensor([c for _, c in cmap] or [0], dtype=torch.int32, device=DEV)
    state = torch.tensor([0.0, float("nan"), float("nan")], device=DEV)
    lib = library()
    for step, t0 in enumerate((0.0, 1.0, 998.0, 2.0 ** 24 - 2)):
        state[0] = t0
        for r in rows:
            r[1].copy_(_grad_values(r[0].numel(), gen))
        before = [[None if t is None else t.clone() for t in r[:5]] for r in rows]
        lib.check(lib.load().gg_adam_ema_step(lib.ptr(table), bt.data_ptr(), bc.data_ptr(), len(cmap), chunk, state.data_ptr(),
                                              BETAS[0], BETAS[1], EPS, DECAY, lib.stream()), "gg_adam_ema_step")
        st = state.cpu()
        t = t0 + 1
        assert float(st[0]) == t
        # the tick forms both in double and rounds once
        b1c, b2c = 1.0 - BETAS[0] ** t, math.sqrt(1.0 - BETAS[1] ** t)
        assert abs(float(st[1]) - b1c) <= U32 * b1c * (1 + 1e-9) and abs(float(st[2]) - b2c) <= U32 * b2c * (1 + 1e-9), (t, st)
        for i, (r, b) in enumerate(zip(rows, before)):
            if not cmap:
                assert all(torch.equal(x, y) for x, y in zip(r[:5], b) if x is not None)
                continue
            res = adam_expect(b, r[:5], r[5].item(), st, r[4])
            for op, (ref, a, k) in res.items():
                y = r[OPERANDS.index(op)]
                check(y, ref, a, k, "adam %s" % op, "%s row %d step %d" % (name, i, step))


@pytest.mark.gpu
def test_fused_adam_ema_with_bucket_view_gradients():
    """FusedAdamEMA with gradients that are views into one flat bucket at odd element offsets (DDP's
    gradient_as_bucket_view): the kernel takes its scalar path; every step's outputs against float64 on that step's inputs,
    with two parameter groups at different learning rates."""
    from gangealing_b200.training.fused_optim import FusedAdamEMA
    gen = seeded(41)
    shapes = [(64, 3, 3, 3), (130,), (7, 5), (ADAM_CHUNK + 3,)]
    params = [torch.randn(s, generator=gen, device=DEV).requires_grad_(True) for s in shapes]
    emas = [p.detach().clone() for p in params[:2]]
    opt = FusedAdamEMA([{"params": params[:2], "lr": 1e-3}, {"params": params[2:], "lr": 2e-2}],
                       ema_pairs=dict(zip(params[:2], emas)), ema_decay=DECAY)
    total = sum(p.numel() for p in params)
    bucket = torch.empty(total + 3 * len(params) + 1, device=DEV)
    off, views = 1, []
    for p in params:
        assert off % 2 == 1                      # every view starts at an odd element offset: off a 16-byte boundary
        views.append(bucket[off:off + p.numel()].view(p.shape))
        off += p.numel() + 1
        off += 1 - off % 2
    for step in range(3):
        for p, vw in zip(params, views):
            vw.copy_(_grad_values(p.numel(), gen).view(p.shape))
            p.grad = vw
        before = [(p.detach().clone(), p.grad.clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone(),
                   None if i >= 2 else emas[i].clone()) for i, p in enumerate(params)]
        opt.step()
        assert all(p.grad.data_ptr() == vw.data_ptr() for p, vw in zip(params, views))
        st = opt._state3.cpu()
        for i, (p, b) in enumerate(zip(params, before)):
            after = (p.detach(), p.grad, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"], None if i >= 2 else emas[i])
            lr = opt.lr_tensor(0 if i < 2 else 1).item()
            for op, (ref, a, k) in adam_expect(b, after, lr, st, after[4]).items():
                check(after[OPERANDS.index(op)], ref, a, k, "adam %s" % op, "bucket views, tensor %d step %d" % (i, step))


# ------------------------------------------------------------------------------------------------ equalised-lr scaling
def _scale_id(cs):
    return cs[0].replace(" ", "_").replace(">", "")


@pytest.mark.gpu
@pytest.mark.parametrize("case", SCALE_CASES, ids=_scale_id)
def test_scale_cast_multi(case):
    """dst == (src.float() * scale).to(dst dtype) bitwise: one correctly rounded fp32 product and one rounding to bf16."""
    name, spec = case
    gen = seeded(sum(map(ord, name)))
    rows, pads = [], []
    for i, (sd, dd, numel, so, do) in enumerate(spec):
        # each operand sits inside a buffer twice its size: the NaN guard bands around dst must stay NaN
        sbuf = torch.randn(2 * numel + so + 8, generator=gen, device=DEV).to(sd)
        src = sbuf[so:so + numel]
        dbuf = torch.full((2 * numel + do + 8,), float("nan"), dtype=dd, device=DEV)
        dst = dbuf[do:do + numel]
        scale = f32(1 / math.sqrt(9 * (i + 3)))
        rows.append((src, dst, scale))
        pads.append((dbuf, do, numel))
    lib = library()
    blob = b"".join(struct.pack("<QQqfi", s.data_ptr(), d.data_ptr(), s.numel(), sc, CODE[s.dtype] | (CODE[d.dtype] << 8))
                    for s, d, sc in rows)
    table = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(DEV)
    cmap = cta_map([r[2] for r in spec], SCALE_CHUNK)
    bt = torch.tensor([t for t, _ in cmap], dtype=torch.int32, device=DEV)
    bc = torch.tensor([c for _, c in cmap], dtype=torch.int32, device=DEV)
    lib.check(lib.load().gg_scale_cast_multi(table.data_ptr(), bt.data_ptr(), bc.data_ptr(), len(cmap), SCALE_CHUNK,
                                             lib.stream()), "gg_scale_cast_multi")
    for i, (src, dst, sc) in enumerate(rows):
        want = (src.cpu().float() * torch.tensor(sc, dtype=F32)).to(dst.dtype)
        got = dst.cpu()
        bad = (got.view(torch.int16 if dst.dtype == BF16 else torch.int32) !=
               want.view(torch.int16 if dst.dtype == BF16 else torch.int32))
        assert not bool(bad.any()), "%s row %d: %d of %d elements differ, first at %d" % (
            name, i, int(bad.sum()), bad.numel(), int(bad.nonzero()[0]))
    for dbuf, do, numel in pads:
        assert bool(dbuf[:do].isnan().all()) and bool(dbuf[do + numel:].isnan().all()), "%s: a write outside dst" % name
    print("[contract] scale-cast %s: bitwise" % name)


# ------------------------------------------------------------------------------------------------ entry behaviour
@pytest.mark.gpu
def test_flow_backward_zeroes_g_base_without_a_base_path():
    """g_base requested without g_flow, or without a base warp, is written as exact zeros by the entry itself."""
    n, lh, lw, s = 3, 2, 3, 2
    low, mask, ident, base, alpha = flow_inputs(n, lh, lw, s, "narrow", 51)
    gd = torch.randn(n, lh * s, lw * s, 2, generator=seeded(52), device=DEV)
    lib = library()
    for g_flow, b in ((None, base), (gd, None)):
        gb = nan_like((n, 2, 3))
        lib.check(lib.load().gg_flow_compose_backward(None, None, gb.data_ptr(), gd.data_ptr(), lib.ptr(g_flow), low.data_ptr(),
                                                      mask.data_ptr(), ident.data_ptr(), lib.ptr(b), alpha.data_ptr(), n, lh, lw,
                                                      s, lib.stream()), "gg_flow_compose_backward")
        assert bool((gb == 0).all())


# ------------------------------------------------------------------------------------------------ launch sets
KERNELS = re.compile(r"(flow_compose_fwd_kernel|flow_compose_bwd_kernel|flow_low_bwd_kernel|flow_base_bwd_kernel|"
                     r"tv_fwd_kernel|tv_finish_kernel|tv_bwd_kernel|adam_tick_kernel|adam_ema_kernel)")


@pytest.mark.gpu
def test_launch_sets_match_the_restatement():
    """Each flow-backward output subset launches exactly the restated kernels, the TV forward launches tv_fwd then
    tv_finish, and an Adam step with no CTAs launches only the tick."""
    run_fresh("test_stn_step_family_gpu", "check_launch_sets")


def check_launch_sets():
    """The body of test_launch_sets_match_the_restatement (raises AssertionError on a mismatch)."""
    seen = []

    def expect(label, names, fn):
        got = launched(fn, KERNELS)
        seen.append("%-56s -> %s" % (label, got))
        assert got == names, "%s: launched %s, the restatement predicts %s" % (label, got, names)
    done = set()
    for cs in FLOW_BWD_CASES:
        r = flow_bwd_route(cs)
        key = (cs[4], cs[5], cs[6])
        if key in done:
            continue
        done.add(key)
        expect("flow bwd %s from %s%s" % ("+".join(cs[4]), cs[5], "" if cs[6] else " (no base)"), r["names"],
               lambda: flow_bwd_run(cs, 3))
    lib = library()
    dll = lib.load()
    f = tv_flow(2, 16, 16, "random", 1)
    out = torch.empty(1, device=DEV)
    ws = torch.empty(dll.gg_tv_loss_workspace(2, 16, 16) // 4, device=DEV)
    expect("tv forward", ["tv_fwd_kernel", "tv_finish_kernel"],
           lambda: lib.check(dll.gg_tv_loss_forward(out.data_ptr(), ws.data_ptr(), f.data_ptr(), 2, 16, 16, lib.stream()), "tv"))
    state = torch.zeros(3, device=DEV)
    expect("adam, blocks == 0", ["adam_tick_kernel"],
           lambda: lib.check(dll.gg_adam_ema_step(None, None, None, 0, ADAM_CHUNK, state.data_ptr(), BETAS[0], BETAS[1], EPS,
                                                  DECAY, lib.stream()), "adam"))
    for line in seen:
        print("[route] " + line)
    print("[route] %d launch sets" % len(seen))
