"""The fp32 FIR kernels against float64, over the code paths their host-side planners choose.

Four kernels run every Blur of the generator and the STN trunk in fp32 storage: fir4_band_kernel (NCHW, csrc/upfirdn2d.cu;
its separable fast path StripF32<IW4, S0, FUSED, VEC> is 64 straight-line variants), the polyphase x2 resamplers
up2_k4_kernel / down2_k4_kernel, upfirdn2d_generic_kernel, and blur_nhwc_kernel (channels-last, csrc/nhwc.cu).  Each picks
its path on the host from the shapes, pads, filter and pointer alignment.  This file

  * restates those planners in Python (plan_band, item_geom and the warp-task walk of the band kernel, the polyphase gates
    of gg_upfirdn2d, blur_plan of the NHWC kernel) and uses the restatement to label every case below; a CPU test asserts
    that the cases reach every variant and every side of every threshold, and a GPU test asserts, by the launched
    kernel's name under torch.profiler, that the restatement routes like the C++;
  * checks every output element against upfirdn2d_ref evaluated in float64 on the exact fp32 operands:
        |y - ref| <= c * 2^-24 * sum|terms|   (oracle.rounding.assert_fp32_sum)
    with c the longest chain of fp32 roundings of the path (stated per path below) and, for a rank-1 filter the band /
    NHWC kernels factorise in fp32, the factorisation error sum|x| * |ku (x) kv - k| added as an explicit allowance;
  * pins the band kernel's zero-weight reads to zeroed memory (DESIGN.md deviation (5)): pads whose stored outputs would
    weight columns outside -3 .. in_w + 2 take the generic kernel.

Every check prints its worst observed c (`[contract] ...` lines with `pytest -s`), and the module prints the worst c per
path when it finishes.
"""
import math
import re

import numpy as np
import pytest
import torch

from fp64_contract import (DEV, F32, H100_SMS, SQRT2, Worst, assert_routes_reached, at_offset, blur_plan, ceil_div,
                           launched, seeded)
from oracle import stylegan2_ops as so

GG_F32 = 0                        # gangealing_b200._lib.GG_F32

# ======================================================================================== planner restatement (no GPU)
K_RS, K_CO, K_WARPS, K_GUARD, K_MAX_PPI = 8, 4, 8, 16, 32   # csrc/upfirdn2d.cu band-kernel constants
STAGE_BUDGET, RING_LIMIT = 36 * 1024, 64 * 1024


def out_size(h, w, kh, kw, up, down, pad):
    """pad = (x0, x1, y0, y1); up / down = (x, y)."""
    return (h * up[1] + pad[2] + pad[3] - kh) // down[1] + 1, (w * up[0] + pad[0] + pad[1] - kw) // down[0] + 1


def band_plan(planes, in_h, in_w, out_h, out_w, pad_x0, es=4):
    """plan_band: -> (plan dict, None) or (None, reason the generic kernel runs)."""
    if out_w < 24 or out_h < 8:
        return None, "tiny"
    if pad_x0 > 3 or out_w - pad_x0 > in_w:
        return None, "wide pad"
    per16 = 16 // es
    lx_log2 = 5
    while lx_log2 > 0 and (1 << (lx_log2 - 1)) * K_CO >= out_w:
        lx_log2 -= 1
    lx, ly = 1 << lx_log2, 32 >> lx_log2
    strip_w, strip_h = lx * K_CO, ly * K_RS
    strips_x = out_w // strip_w if out_w // strip_w > 0 else 1

    def slot(rows):
        rows8 = ceil_div(rows, K_RS) * K_RS
        return ceil_div(K_GUARD // es + (rows8 + 3) * in_w + 2 * per16 + 4, per16) * per16

    ppi = 1
    if slot(out_h) * es <= STAGE_BUDGET:
        r, bands = out_h, 1
        tasks = strips_x * ceil_div(out_h, strip_h)
        ppi = min(ceil_div(K_WARPS, tasks), STAGE_BUDGET // (slot(out_h) * es))
        ppi = min(max(ppi, 1), planes, K_MAX_PPI)
    else:
        r = strip_h * ceil_div(K_WARPS, strips_x)
        while r > strip_h and slot(r) * es > STAGE_BUDGET:
            r -= strip_h
        if slot(r) * es > RING_LIMIT:
            return None, "ring"
        if r >= out_h:
            return None, "one band"
        bands = ceil_div(out_h, r)
    if slot(r) * ppi * es * 3 > 200 * 1024:
        return None, "smem"
    return dict(planes=planes, in_h=in_h, in_w=in_w, out_h=out_h, out_w=out_w, pad_x0=pad_x0, lx_log2=lx_log2, r=r,
                bands=bands, ppi=ppi, slot=slot(r), slot_of=slot, es=es,
                n_items=ceil_div(planes, ppi) if bands == 1 else planes * bands), None


def band_walk(p, pad_y0, in_off):
    """item_geom + the warp-task loop of fir4_band_kernel (fp32): yields (item geometry, S0 = pos0 & 3) per warp task that
    stores outputs.  in_off: element offset of the input from a 16-byte boundary."""
    in_h, in_w, out_h, out_w = p["in_h"], p["in_w"], p["out_h"], p["out_w"]
    lx_main = 1 << p["lx_log2"]
    full_x = out_w // (lx_main * K_CO)
    tail_w = out_w - full_x * lx_main * K_CO
    lt = 0
    while (1 << lt) * K_CO < tail_w:
        lt += 1
    for item in range(p["n_items"]):
        if p["bands"] == 1:
            m0, n_planes, oy0, rows = item * p["ppi"], min(p["ppi"], p["planes"] - item * p["ppi"]), 0, out_h
        else:
            m0, n_planes = item // p["bands"], 1
            oy0 = (item % p["bands"]) * p["r"]
            rows = min(p["r"], out_h - oy0)
        vy0, vrows = oy0 - pad_y0, rows + 3
        lo = max(vy0, 0)
        nreal = min(vy0 + vrows - 1, in_h - 1) - lo + 1
        n_top = (lo if nreal > 0 else vy0 + vrows) - vy0
        d0 = ceil_div(K_GUARD // 4 + n_top * in_w, 4) * 4
        geom = dict(m0=m0, n_planes=n_planes, oy0=oy0, rows=rows, nreal=nreal)
        main_tasks = full_x * ceil_div(rows, (32 >> p["lx_log2"]) * K_RS)
        tail_tasks = ceil_div(rows, (32 >> lt) * K_RS) if tail_w > 0 else 0
        for pl in range(n_planes):
            if nreal <= 0:
                v0 = d0 - vrows * in_w
            else:
                shift = (in_off + ((m0 + pl) * in_h + lo) * in_w) % 4
                v0 = d0 + shift - (lo - vy0) * in_w
            for rem in range(main_tasks + tail_tasks):
                if rem < main_tasks:
                    sy, xs, lg = rem // full_x, (rem % full_x) * lx_main * K_CO, p["lx_log2"]
                else:
                    sy, xs, lg = rem - main_tasks, full_x * lx_main * K_CO, lt
                oys = oy0 + sy * (32 >> lg) * K_RS          # lane 0: the smallest row and column of the warp
                if min(K_RS, oy0 + rows - oys) <= 0 or xs >= out_w:
                    continue
                yield geom, (v0 + (oys - oy0) * in_w + (xs - p["pad_x0"])) & 3


def band_factor(k):
    """fir4_band_kernel's (and blur_nhwc_kernel's) rank-1 factorisation of the flipped 4x4 taps in fp32, restated:
    -> (separable, float64 filter E such that upfirdn2d_ref(|x|, E) = sum |x| * |ku (x) kv - k| over the window)."""
    kh, kw = k.shape
    kf = np.zeros((4, 4), np.float32)
    kf[:kh, :kw] = np.flip(k.detach().cpu().numpy().astype(np.float32), (0, 1))
    big, a0, b0 = np.float32(0), 0, 0
    for a in range(4):
        for b in range(4):
            if abs(kf[a, b]) > big:
                big, a0, b0 = abs(kf[a, b]), a, b
    inv = np.float32(1) / kf[a0, b0] if big > 0 else np.float32(0)
    ku = (kf[:, b0] * inv).astype(np.float32)
    kv = kf[a0, :].copy()
    err = np.outer(ku.astype(np.float64), kv.astype(np.float64)) - kf.astype(np.float64)
    dev, lim = float(np.abs(err).max()), 1e-6 * float(big)
    assert not (0.5 * lim < dev < 2 * lim), "test filter too close to the rank-1 threshold: %g vs %g" % (dev, lim)
    e = np.flip(np.abs(err[:kh, :kw]), (0, 1)).copy()
    return dev <= lim, torch.from_numpy(e)


def fir_route(shape, k, up=(1, 1), down=(1, 1), pad=(0, 0, 0, 0), in_off=0, out_off=0, fused=False, noise_off=None):
    """gg_upfirdn2d / gg_blur_noise_bias_act (fp32) -> dict(kind, kernel name, c, factorisation allowance, labels)."""
    n, c, in_h, in_w = shape
    kh, kw = k.shape
    out_h, out_w = out_size(in_h, in_w, kh, kw, up, down, pad)
    planes = n * c
    labels = set()
    plan, why = None, None
    if fused or (up == (1, 1) and down == (1, 1) and kh <= 4 and kw <= 4):
        plan, why = band_plan(planes, in_h, in_w, out_h, out_w, pad[0])
        labels.add("band: %s" % ("planned" if plan else "generic (%s)" % why))
        labels |= _threshold_labels(plan, why, out_h, out_w, in_w)
    if plan is not None:
        sep, e = band_factor(k)
        vec = out_w % 4 == 0 and out_off % 4 == 0 and (noise_off is None or noise_off % 4 == 0)
        iw4 = in_w & 3
        if sep:
            for geom, s0 in band_walk(plan, pad[2], in_off):
                labels.add("StripF32<%d, %d, %s, %s>" % (iw4, s0, str(fused).lower(), str(vec).lower()))
        else:
            labels.add("band fp32 16-tap lane_strip")
        for geom, _ in band_walk(plan, pad[2], in_off):
            if geom["nreal"] <= 0:
                labels.add("band: padding-only band")
        if plan["bands"] > 1:
            labels.add("band: several bands per plane")
        if plan["bands"] == 1 and plan["ppi"] > 1 and planes % plan["ppi"]:
            labels.add("band: items of several planes, partial last item")
        return dict(kind="band", name="fir4_band_kernel<float, %d, %s>" % (iw4, str(fused).lower()),
                    c=9 if sep else 16, extra=e if sep else None, labels=labels, plan=plan)
    if not fused and kh == 4 and kw == 4:
        aligned = in_off % 4 == 0 and out_off % 4 == 0
        if up == (2, 2) and down == (1, 1):
            ok_pad, ok_shape = pad == (2, 1, 2, 1), in_w % 2 == 0
            if aligned and ok_pad and ok_shape:
                return dict(kind="up2", name="up2_k4_kernel", c=4, extra=None, labels=labels | {"polyphase: up2"})
            labels.add("polyphase: up2 fallback (%s)" % ("odd width" if not ok_shape else "misaligned" if not aligned
                                                         else "other pads"))
        if up == (1, 1) and down == (2, 2):
            ok_pad, ok_shape = pad == (1, 1, 1, 1), in_w % 4 == 0 and in_h % 2 == 0
            if aligned and ok_pad and ok_shape:
                return dict(kind="down2", name="down2_k4_kernel", c=16, extra=None, labels=labels | {"polyphase: down2"})
            labels.add("polyphase: down2 fallback (%s)" % ("in_w % 4" if in_w % 4 else "odd height" if in_h % 2 else
                                                           "misaligned" if not aligned else "other pads"))
    if fused:
        tmpl = "true, 0, 0"
    elif up == (2, 2) and down == (1, 1):
        tmpl = "false, 2, 1"
    elif up == (1, 1) and down == (2, 2):
        tmpl = "false, 1, 2"
    else:
        tmpl = "false, 0, 0"
    return dict(kind="generic", name="upfirdn2d_generic_kernel<float, %s>" % tmpl, c=kh * kw, extra=None,
                labels=labels | {"generic <%s>" % tmpl}, plan=None)


def _threshold_labels(plan, why, out_h, out_w, in_w):
    lab = set()
    if why == "tiny":
        lab.add("threshold: out_w 23 -> generic" if out_w == 23 else "threshold: out_h 7 -> generic" if out_h == 7 else "")
    if plan is not None:
        if out_w == 24:
            lab.add("threshold: out_w 24 -> band")
        if out_h == 8:
            lab.add("threshold: out_h 8 -> band")
        step = K_RS * in_w * plan["es"]            # one more strip of rows
        whole = plan["slot_of"](out_h) * plan["es"]
        if plan["bands"] == 1 and whole + step > STAGE_BUDGET:
            lab.add("threshold: whole plane just inside the 36 KB stage")
        if plan["bands"] > 1 and whole - step <= STAGE_BUDGET:
            lab.add("threshold: plane just over the 36 KB stage -> bands")
        if plan["bands"] > 1 and plan["slot"] * plan["es"] > STAGE_BUDGET:
            lab.add("threshold: 8-row band over the stage budget, inside the 64 KB ring")
    if why == "ring":
        lab.add("threshold: 8-row band over the 64 KB ring -> generic")
    lab.discard("")
    return lab


def nhwc_route(shape, k, pad, mode, slope, gain, sms):
    n, c, h, w = shape
    sep, e = band_factor(k)
    p = blur_plan(F32, n, c, h, w, k.shape[0], k.shape[1], pad, sms)
    fast = mode == 1 and gain > 0 and 0 <= slope <= 1
    name = "blur_nhwc_kernel<float, %d, %s, %s>" % (mode, str(sep).lower(), str(fast).lower())
    labels = {name}
    if p["chunks"] > 1:
        labels.add("nhwc: several channel chunks")
    if p["out_w"] % 64:
        labels.add("nhwc: x-tail block")
    if p["segs"] > 1:
        labels.add("nhwc: several row segments")
    if p["out_h"] < 16:
        labels.add("nhwc: out_h < 16")
    return dict(name=name, c=9 if sep else 16, extra=e if sep else None, plan=p, labels=labels)


# ============================================================================================================ cases
def filt(kind, kh=4, kw=4, seed=0):
    """fp32 filters: binom ([1,3,3,1] outer product, exact), rank1 (random, rounded to fp32: not exactly rank 1), full."""
    g = torch.Generator().manual_seed(1000 + 17 * kh + kw + seed)
    if kind == "binom":
        return so.make_kernel([1, 3, 3, 1]) * 4
    if kind == "rank1":
        return (torch.outer(torch.rand(kh, generator=g) + 0.25, torch.randn(kw, generator=g))).float()
    return torch.randn(kh, kw, generator=g).float() / math.sqrt(kh * kw)


# 1) the StripF32 sweep: in_w mod 4 = 0..3 x pad_x0 = 0..3 (pad_x1 keeps out_w % 4 == 0) x plain / fused x vector / scalar
#    I/O (scalar: output at a 1-element offset).  10 planes of 13 rows: a 6-plane item plus a partial one, and plane
#    alignments that rotate with the plane index.
STRIP_CASES = [(w, px0, fused, vec) for w in (36, 37, 38, 39) for px0 in range(4) for fused in (False, True)
               for vec in (True, False)]


def strip_case(w, px0, fused, vec):
    px1 = (3 - w - px0) % 4
    kind = "binom" if (w + px0) % 2 == 0 else "rank1"
    return dict(shape=(2, 5, 13, w), k=filt(kind, seed=w + px0), pad=(px0, px1, 2, 1), in_off=1 + 2 * int(fused),
                out_off=0 if vec else 1, fused=fused)


# 2) filters x pads through autograd (forward and the adjoint in backward): 1x1 .. 4x4, non-square, >4x4
FILTERS = [(1, 1, "full"), (1, 4, "binom1d"), (2, 3, "full"), (3, 3, "rank1"), (4, 2, "rank1"), (4, 4, "binom"),
           (4, 4, "rank1"), (4, 4, "full"), (3, 5, "rank1"), (5, 5, "full")]
PADS = [(-2, 1, 0, 3), (-1, 2, 1, -1), (0, 0, 2, 1), (1, 1, 1, 1), (2, 1, 3, -2), (3, 3, 0, 0), (3, -2, -1, 2),
        (4, 0, 1, 1), (0, 4, 2, 2), (5, 6, 4, -1), (6, 5, -2, 6), (-1, 2, -1, 2)]
SWEEP_SHAPES = [(2, 5, 21, 40), (3, 3, 19, 41), (1, 7, 23, 42), (2, 4, 17, 43), (1, 3, 9, 13)]


def sweep_filter(kh, kw, kind):
    if kind == "binom1d":
        return (torch.tensor([[1.0, 3.0, 3.0, 1.0]]) / 8).expand(kh, kw).contiguous()
    return filt(kind, kh, kw)


def sweep_case(fi, pi):
    kh, kw, kind = FILTERS[fi]
    return dict(shape=SWEEP_SHAPES[(fi + pi) % len(SWEEP_SHAPES)], k=sweep_filter(kh, kw, kind), pad=PADS[pi])


# 3) planner thresholds and band geometry (raw calls with independent x / y pads)
GEOMETRY_CASES = [
    ((1, 3, 12, 25), (1, 0, 1, 1)),       # out_w 23 -> generic
    ((1, 3, 12, 26), (1, 0, 1, 1)),       # out_w 24 -> band
    ((1, 3, 9, 30), (1, 1, 1, 0)),        # out_h 7 -> generic
    ((1, 3, 10, 30), (1, 1, 1, 0)),       # out_h 8 -> band
    ((1, 2, 136, 64), (1, 2, 1, 2)),      # whole 136-row plane: just inside the 36 KB stage
    ((1, 2, 137, 64), (1, 2, 1, 2)),      # 137 rows: just over -> two bands
    ((1, 2, 40, 64), (1, 2, 1, 200)),     # 200 rows of bottom padding: a band that sees only zeros
    ((2, 1, 60, 1000), (1, 2, 2, 1)),     # 8-row bands of 1000 columns: over the stage budget, inside the ring
    ((1, 1, 20, 1480), (1, 2, 1, 2)),     # the widest rows the ring takes
    ((1, 1, 20, 1500), (1, 2, 1, 2)),     # 8 rows over 64 KB -> generic
    ((1, 1, 10, 1000), (1, 2, 1, 0)),     # 8 rows over the stage budget in one 8-row band -> generic
    ((3, 4, 257, 257), (1, 1, 1, 1)),     # the largest hot-path plane: several bands per plane
]

# 4) polyphase resamplers and each of their fallbacks: (shape, up, down, pad, in_off, out_off)
POLY_CASES = [
    ((2, 3, 16, 24), 2, 1, (2, 1, 2, 1), 0, 0),
    ((2, 3, 16, 25), 2, 1, (2, 1, 2, 1), 0, 0),     # odd width
    ((2, 3, 16, 24), 2, 1, (2, 1, 2, 1), 1, 0),     # input 4 bytes past a 16-byte boundary
    ((2, 3, 16, 24), 2, 1, (2, 1, 2, 1), 0, 2),     # output 8 bytes past
    ((2, 3, 16, 24), 2, 1, (2, 2, 2, 2), 0, 0),     # other pads
    ((2, 3, 32, 48), 1, 2, (1, 1, 1, 1), 0, 0),
    ((2, 3, 32, 50), 1, 2, (1, 1, 1, 1), 0, 0),     # in_w % 4 == 2
    ((2, 3, 31, 48), 1, 2, (1, 1, 1, 1), 0, 0),     # odd height
    ((2, 3, 32, 48), 1, 2, (1, 1, 1, 1), 3, 0),     # misaligned input
    ((2, 3, 32, 48), 1, 2, (2, 1, 2, 1), 0, 0),     # other pads
]

# 5) the fused NCHW tail: (noise, bias, row_scale) present or absent x (act, slope, gain); half the noise planes misaligned
EPILOGUES = [(3, 0.2, SQRT2), (3, 1.5, 1.0), (1, 0.2, -1.0), (3, 0.2, -1.0)]
TAIL_CASES = [(nz, b, rs, e) for nz in (False, True) for b in (False, True) for rs in (False, True) for e in range(4)]
TAIL_SHAPES = [(2, 5, 33, 33), (1, 3, 130, 130), (2, 3, 9, 9), (2, 4, 31, 30)]    # plane items | bands | generic | scalar I/O


def tail_case(nz, b, rs, e):
    i = (4 * nz + 2 * b + rs + e) % len(TAIL_SHAPES)
    kind = ("binom", "rank1", "full")[(e + i) % 3]
    pad = ((1, 1, 1, 1), (2, 1, 2, 1), (2, 2, 1, 3))[(nz + e) % 3]
    return dict(shape=TAIL_SHAPES[i], k=filt(kind, seed=e), pad=pad, noise=nz, noise_off=(1 + e % 3) if nz and e % 2 else 0,
                bias=b, rs=rs, epi=EPILOGUES[e])


# 6) channels-last: (shape, pad, mode, kind, slope, gain)
NHWC_SHAPES = [(2, 96, 20, 70), (1, 32, 9, 30), (2, 32, 40, 64)]     # 3 channel chunks + x-tail | out_h < 16 | row segments
NHWC_CASES = [(s, mode, kind, ep) for s in range(3) for mode in (0, 1, 2) for kind in ("binom", "rank1", "full")
              for ep in ((0.2, SQRT2), (1.5, SQRT2)) if mode == 1 or ep[0] == 0.2]
NHWC_PADS = [(1, 1, 1, 1), (2, 2, 2, 2), (2, 1, 0, 3)]

# 7) the cases a zero-weight read outside the zeroed guards would have turned NaN (now on the generic kernel):
#    (shape, filter shape, pad) and the backward of a (-1, 2) crop
WIDE_PAD_CASES = [((2, 3, 20, 40), (4, 4), (1, 4, 1, 1)), ((2, 3, 20, 40), (1, 1), (1, 1, 1, 1)),
                  ((2, 3, 20, 40), (4, 4), (4, 0, 2, 2)), ((2, 3, 20, 40), (4, 4), (6, 5, 4, 6))]


# ======================================================================================================== CPU check
def all_routes(sms=H100_SMS):
    out = []
    for w, px0, fused, vec in STRIP_CASES:
        cs = strip_case(w, px0, fused, vec)
        out.append(fir_route(cs["shape"], cs["k"], pad=cs["pad"], in_off=cs["in_off"], out_off=cs["out_off"],
                             fused=fused, noise_off=0 if fused else None))
    for fi in range(len(FILTERS)):
        for pi in range(len(PADS)):
            cs = sweep_case(fi, pi)
            out.append(fir_route(cs["shape"], cs["k"], pad=cs["pad"]))
            out.append(backward_route(cs))
    for shape, pad in GEOMETRY_CASES:
        out.append(fir_route(shape, filt("binom"), pad=pad))
    for shape, up, down, pad, io, oo in POLY_CASES:
        out.append(fir_route(shape, filt("binom"), (up, up), (down, down), pad, io, oo))
    for case in TAIL_CASES:
        cs = tail_case(*case)
        out.append(fir_route(cs["shape"], cs["k"], pad=cs["pad"], fused=True, noise_off=cs["noise_off"] if cs["noise"] else None))
    for si, mode, kind, (slope, gain) in NHWC_CASES:
        out.append(nhwc_route(NHWC_SHAPES[si], filt(kind, seed=si), NHWC_PADS[si], mode, slope, gain, sms))
    for shape, (kh, kw), pad in WIDE_PAD_CASES:
        out.append(fir_route(shape, filt("binom" if kh == 4 else "full", kh, kw), pad=pad))
    return out


def backward_route(cs):
    n, c, h, w = cs["shape"]
    kh, kw = cs["k"].shape
    oh, ow = out_size(h, w, kh, kw, (1, 1), (1, 1), cs["pad"])
    gp = grad_pad(h, w, oh, ow, kh, kw, cs["pad"])
    return fir_route((n, c, oh, ow), torch.flip(cs["k"], [0, 1]), pad=gp)


def grad_pad(h, w, oh, ow, kh, kw, pad):
    """op/upfirdn2d.py grad_pad for up = down = 1."""
    return (kw - pad[0] - 1, w - ow + pad[0], kh - pad[2] - 1, h - oh + pad[2])


REQUIRED = (["StripF32<%d, %d, %s, %s>" % (i, s, f, v) for i in range(4) for s in range(4) for f in ("false", "true")
             for v in ("false", "true")]
            + ["band fp32 16-tap lane_strip", "band: items of several planes, partial last item",
               "band: several bands per plane", "band: padding-only band",
               "threshold: out_w 23 -> generic", "threshold: out_w 24 -> band", "threshold: out_h 7 -> generic",
               "threshold: out_h 8 -> band", "threshold: whole plane just inside the 36 KB stage",
               "threshold: plane just over the 36 KB stage -> bands",
               "threshold: 8-row band over the stage budget, inside the 64 KB ring",
               "threshold: 8-row band over the 64 KB ring -> generic", "band: generic (one band)",
               "band: generic (wide pad)",
               "polyphase: up2", "polyphase: up2 fallback (odd width)", "polyphase: up2 fallback (misaligned)",
               "polyphase: up2 fallback (other pads)", "polyphase: down2", "polyphase: down2 fallback (in_w % 4)",
               "polyphase: down2 fallback (odd height)", "polyphase: down2 fallback (misaligned)",
               "polyphase: down2 fallback (other pads)",
               "generic <true, 0, 0>", "generic <false, 0, 0>", "generic <false, 2, 1>", "generic <false, 1, 2>",
               "nhwc: several channel chunks", "nhwc: x-tail block", "nhwc: several row segments", "nhwc: out_h < 16"]
            + ["blur_nhwc_kernel<float, %d, %s, %s>" % (m, s, f) for m in (0, 1, 2) for s in ("true", "false")
               for f in (("true", "false") if m == 1 else ("false",))])


def test_cases_reach_every_fp32_fir_path():
    """Coverage of the sweep below, by the planner restatement: every StripF32 variant, the 16-tap lane, every band
    geometry class, both sides of every planner threshold, each polyphase kernel and each of its fallbacks, and every
    NHWC variant and geometry class."""
    reached = set()
    for r in all_routes():
        reached |= r["labels"]
    assert_routes_reached(REQUIRED, reached, noun="fp32 FIR classes")


def test_wide_pads_leave_the_band_kernel_and_hot_pads_stay():
    """The zero-weight columns of the band kernel's fp32 separable path must lie in -3 .. in_w + 2: wider pads plan the
    generic kernel, the generator's pads (1,1), (2,2), (2,1) and their adjoints keep the band kernel."""
    k = filt("binom")
    for shape, (kh, kw), pad in WIDE_PAD_CASES:
        assert fir_route(shape, torch.ones(kh, kw), pad=pad)["kind"] == "generic", (shape, pad)
    crop = grad_pad(40, 40, 38, 38, 4, 4, (-1, 2, -1, 2))
    assert crop == (4, 1, 4, 1) and fir_route((2, 3, 38, 38), k, pad=crop)["kind"] == "generic"
    for p in ((1, 1), (2, 2), (2, 1), (1, 2)):
        for shape in ((4, 512, 33, 33), (4, 128, 257, 257), (4, 64, 129, 129)):
            assert fir_route(shape, k, pad=(p[0], p[1], p[0], p[1]))["kind"] == "band", (shape, p)


# ======================================================================================================== GPU checks
WORST = Worst("c per fp32 FIR path", "%-46s c_obs = %.2f", kind_suffix=False)
_report_worst = WORST.fixture()
check_sum = WORST.check_sum


def ref64(x, k, up=(1, 1), down=(1, 1), pad=(0, 0, 0, 0)):
    return so.upfirdn2d_ref_full(x.double(), k.to(x.device).double(), up[0], up[1], down[0], down[1], *pad)


def fir_raw(x, k, up=(1, 1), down=(1, 1), pad=(0, 0, 0, 0), out_off=0):
    """gg_upfirdn2d with 4 independent pads, the output `out_off` elements past a 16-byte boundary."""
    from gangealing_b200 import _lib
    n, c, h, w = x.shape
    kh, kw = k.shape
    oh, ow = out_size(h, w, kh, kw, up, down, pad)
    out = torch.empty(out_off + n * c * oh * ow, device=x.device)[out_off:].view(n, c, oh, ow)
    rc = _lib.load().gg_upfirdn2d(out.data_ptr(), x.data_ptr(), k.data_ptr(), GG_F32, n * c, h, w, kh, kw, up[0], up[1],
                                  down[0], down[1], *pad, _lib.stream())
    _lib.check(rc, "gg_upfirdn2d")
    return out


def fused_raw(x, k, pad, noise, nw, bias, rs, act, alpha, scale, out_off=0):
    from gangealing_b200 import _lib
    n, c, h, w = x.shape
    kh, kw = k.shape
    oh, ow = out_size(h, w, kh, kw, (1, 1), (1, 1), pad)
    out = torch.empty(out_off + n * c * oh * ow, device=x.device)[out_off:].view(n, c, oh, ow)
    rc = _lib.load().gg_blur_noise_bias_act(out.data_ptr(), x.data_ptr(), k.data_ptr(), _lib.ptr(noise), _lib.ptr(nw),
                                            _lib.ptr(bias), _lib.ptr(rs), GG_F32, n, c, h, w, kh, kw, *pad, act, alpha,
                                            scale, _lib.stream())
    _lib.check(rc, "gg_blur_noise_bias_act")
    return out


def check_fir(y, x, k, route, what, up=(1, 1), down=(1, 1), pad=(0, 0, 0, 0)):
    """y = upfirdn2d(x, k): every element within c * 2^-24 * sum|x*k| of the float64 value (+ the factorisation error)."""
    kd = k.to(DEV)
    extra = ref64(x.abs(), route["extra"], up, down, pad) if route["extra"] is not None else None
    check_sum(y, ref64(x, kd, up, down, pad), ref64(x.abs(), kd.abs(), up, down, pad), route["c"], route["name"], what, extra)


@pytest.mark.gpu
@pytest.mark.parametrize("w,px0,fused,vec", STRIP_CASES)
def test_band_strip_variant(w, px0, fused, vec):
    """One launch per StripF32<IW4, *, FUSED, VEC> x pad_x0: the item's plane alignments supply every S0."""
    cs = strip_case(w, px0, fused, vec)
    g = seeded(w * 8 + px0)
    x = at_offset(torch.randn(cs["shape"], generator=g, device=DEV), cs["in_off"])
    k = cs["k"].to(DEV)
    pad = cs["pad"]
    route = fir_route(cs["shape"], cs["k"], pad=pad, in_off=cs["in_off"], out_off=cs["out_off"], fused=fused,
                      noise_off=0 if fused else None)
    assert route["kind"] == "band"
    what = "in_w %d pad %s in_off %d out_off %d" % (w, pad, cs["in_off"], cs["out_off"])
    if not fused:
        check_fir(fir_raw(x, k, pad=pad, out_off=cs["out_off"]), x, k, route, what, pad=pad)
        return
    n, c = cs["shape"][:2]
    oh, ow = out_size(cs["shape"][2], w, 4, 4, (1, 1), (1, 1), pad)
    nz = torch.randn(n, oh, ow, generator=g, device=DEV)
    nw = torch.tensor([0.7], device=DEV)
    b = torch.randn(c, generator=g, device=DEV)
    rs = torch.rand(n * c, generator=g, device=DEV) + 0.5
    y = fused_raw(x, k, pad, nz, nw, b, rs, 3, 0.2, SQRT2, cs["out_off"])
    check_tail(y, x, k, route, pad, nz, nw, b, rs, 0.2, SQRT2, what)


def check_tail(y, x, k, route, pad, nz, nw, b, rs, alpha, gain, what):
    """out = lrelu(rs*B(x) + b + nw*noise)*gain: the blur's c plus the epilogue's 5 roundings (the rs fma, the noise fma,
    alpha*gain - gain, gain*t, the final fma; the generic kernel: rs*t + b, the noise fma, alpha*gain, the product)."""
    n, c = x.shape[:2]
    alpha, gain = float(np.float32(alpha)), float(np.float32(gain))
    kd = k.to(DEV)
    t, ta = ref64(x, kd, pad=pad), ref64(x.abs(), kd.abs(), pad=pad)
    r64 = rs.double().reshape(n, c, 1, 1) if rs is not None else torch.ones(1, dtype=torch.float64, device=DEV)
    pre, a = r64 * t, r64.abs() * ta
    if b is not None:
        pre, a = pre + b.double()[:, None, None], a + b.double().abs()[:, None, None]
    if nz is not None:
        nn_ = nw.double() * nz.double().reshape(n, 1, *t.shape[2:])
        pre, a = pre + nn_, a + nn_.abs()
    sg = abs(gain) * max(1.0, abs(alpha))
    out = torch.where(pre > 0, pre, pre * alpha) * gain
    extra = None
    if route["extra"] is not None:
        extra = r64.abs() * ref64(x.abs(), route["extra"], pad=pad) * sg
    check_sum(y, out, a * sg, route["c"] + 5, route["name"] + " fused", what, extra)


@pytest.mark.gpu
@pytest.mark.parametrize("fi", range(len(FILTERS)))
@pytest.mark.parametrize("pi", range(len(PADS)))
def test_filters_and_pads_forward_and_backward(fi, pi):
    """Autograd through UpFirDn2d with independent x / y pads: the forward, then the gradient (the adjoint resampling:
    flipped filter, grad_pad) against the float64 adjoint."""
    from gangealing_b200.op.upfirdn2d import UpFirDn2d
    cs = sweep_case(fi, pi)
    g = seeded(100 * fi + pi)
    k = cs["k"].to(DEV)
    x = torch.randn(cs["shape"], generator=g, device=DEV).requires_grad_(True)
    y = UpFirDn2d.apply(x, k, (1, 1), (1, 1), cs["pad"])
    what = "%s %dx%d pad %s" % (FILTERS[fi][2], k.shape[0], k.shape[1], cs["pad"])
    check_fir(y, x.detach(), k, fir_route(cs["shape"], cs["k"], pad=cs["pad"]), what + " forward", pad=cs["pad"])
    gy = torch.randn(y.shape, generator=g, device=DEV)
    (gx,) = torch.autograd.grad(y, x, gy)
    n, c, h, w = cs["shape"]
    gp = grad_pad(h, w, y.shape[2], y.shape[3], k.shape[0], k.shape[1], cs["pad"])
    check_fir(gx, gy, torch.flip(k, [0, 1]), backward_route(cs), what + " backward, adjoint pad %s" % (gp,), pad=gp)


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(GEOMETRY_CASES)))
def test_band_geometry_and_thresholds(case):
    shape, pad = GEOMETRY_CASES[case]
    g = seeded(7 + case)
    k = filt("binom") if case % 2 == 0 else filt("full")
    x = torch.randn(shape, generator=g, device=DEV)
    route = fir_route(shape, k, pad=pad)
    check_fir(fir_raw(x, k.to(DEV), pad=pad), x, k, route, "%s pad %s" % (shape, pad), pad=pad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(POLY_CASES)))
def test_polyphase_resamplers_and_fallbacks(case):
    """x2 up-sampler: 4 fmas per output (c = 4); x2 decimator: 16 (c = 16); the generic fallback: kh*kw."""
    shape, up, down, pad, io, oo = POLY_CASES[case]
    g = seeded(50 + case)
    k = filt("binom") if case % 2 == 0 else filt("full")
    x = at_offset(torch.randn(shape, generator=g, device=DEV), io)
    route = fir_route(shape, k, (up, up), (down, down), pad, io, oo)
    y = fir_raw(x, k.to(DEV), (up, up), (down, down), pad, oo)
    check_fir(y, x, k, route, "%s up %d down %d pad %s offsets %d/%d" % (shape, up, down, pad, io, oo), (up, up), (down, down), pad)


@pytest.mark.gpu
@pytest.mark.parametrize("up", [2, 1])
def test_polyphase_autograd(up):
    """The to-RGB skip's Upsample and its backward (each resampler is the other's adjoint), through autograd."""
    from gangealing_b200 import op
    g = seeded(up)
    k = filt("binom").to(DEV)
    down = 3 - up
    pad = (2, 1) if up == 2 else (1, 1)
    x = torch.randn(2, 3, 16, 32, generator=g, device=DEV).requires_grad_(True)
    y = op.upfirdn2d(x, k, up=up, down=down, pad=pad)
    p4 = (pad[0], pad[1], pad[0], pad[1])
    check_fir(y, x.detach(), k, fir_route(tuple(x.shape), k, (up, up), (down, down), p4), "autograd forward",
              (up, up), (down, down), p4)
    gy = torch.randn(y.shape, generator=g, device=DEV)
    (gx,) = torch.autograd.grad(y, x, gy)
    gp = (1, 1, 1, 1) if up == 2 else (2, 1, 2, 1)
    check_fir(gx, gy, torch.flip(k, [0, 1]), fir_route(tuple(gy.shape), k, (down, down), (up, up), gp), "autograd backward",
              (down, down), (up, up), gp)


@pytest.mark.gpu
@pytest.mark.parametrize("nz,b,rs,e", TAIL_CASES)
def test_blur_noise_bias_act_epilogue(nz, b, rs, e):
    cs = tail_case(nz, b, rs, e)
    act, slope, gain = cs["epi"]
    n, c, h, w = cs["shape"]
    g = seeded(1000 + 16 * nz + 8 * b + 4 * rs + e)
    x = torch.randn(cs["shape"], generator=g, device=DEV)
    k = cs["k"].to(DEV)
    oh, ow = out_size(h, w, 4, 4, (1, 1), (1, 1), cs["pad"])
    noise = at_offset(torch.randn(n, oh, ow, generator=g, device=DEV), cs["noise_off"]) if nz else None
    nw = torch.tensor([0.6], device=DEV) if nz else None
    bias = torch.randn(c, generator=g, device=DEV) if b else None
    rsv = torch.rand(n * c, generator=g, device=DEV) + 0.5 if rs else None
    route = fir_route(cs["shape"], cs["k"], pad=cs["pad"], fused=True, noise_off=cs["noise_off"] if nz else None)
    y = fused_raw(x, k, cs["pad"], noise, nw, bias, rsv, act, slope, gain)
    what = "%s pad %s noise %s (offset %d) bias %s rs %s act %d slope %g gain %g" % (
        cs["shape"], cs["pad"], nz, cs["noise_off"], b, rs, act, slope, gain)
    check_tail(y, x, k, route, cs["pad"], noise, nw, bias, rsv, slope if act == 3 else 1.0, gain, what)


def nhwc_dot_c(route):
    p = route["plan"]
    # mode 2's dot: a thread's fmas over its 2 columns x segment rows, the CTA's 32 column groups, the finish kernel
    return route["c"] + 1 + 2 * p["seg_rows"] + 32 + (ceil_div(p["xblocks"] * p["segs"], 32) + 2 + 32)


@pytest.mark.gpu
@pytest.mark.parametrize("si,mode,kind,ep", NHWC_CASES)
def test_blur_nhwc_f32(si, mode, kind, ep):
    """Channels-last fp32: mode 0 (c = 9 / 16), mode 1 (+5, out2 +6: see the bf16 storage tests), mode 2 (g_raw: +1;
    row_dot: + a thread's fmas, 32 column groups, the finish kernel)."""
    from gangealing_b200 import _lib
    from gangealing_b200.op import nhwc
    slope, gain = ep
    shape, pad = NHWC_SHAPES[si], NHWC_PADS[si]
    n, c, h, w = shape
    g = seeded(300 + 10 * si + mode)
    k = filt(kind, seed=si)
    kd = k.to(DEV)
    route = nhwc_route(shape, k, pad, mode, slope, gain, _lib.sm_count())
    x = torch.randn(shape, generator=g, device=DEV).contiguous(memory_format=torch.channels_last)
    oh, ow = route["plan"]["out_h"], route["plan"]["out_w"]
    t, ta = ref64(x, kd, pad=pad), ref64(x.abs(), kd.abs(), pad=pad)
    fx = ref64(x.abs(), route["extra"], pad=pad) if route["extra"] is not None else None
    path, what = route["name"], "%s pad %s %s" % (shape, pad, kind)
    if mode == 0:
        y, _, _ = nhwc.blur(x, kd, pad, mode=0)
        check_sum(y, t, ta, route["c"], path, what, fx)
    elif mode == 1:
        nz = torch.randn(n, 1, oh, ow, generator=g, device=DEV)
        nw = torch.tensor([0.3], device=DEV)
        b = torch.randn(c, generator=g, device=DEV) * 0.5
        rs = torch.rand(n, c, generator=g, device=DEV) + 0.5
        s2 = torch.randn(n, c, generator=g, device=DEV) + 1.0
        out, out2, _ = nhwc.blur(x, kd, pad, mode=1, noise=nz, noise_weight=nw, bias=b, row_scale=rs, scale2=s2,
                                 want_out=True, want_out2=True, negative_slope=slope, gain=gain)
        r64, s64 = rs.double()[:, :, None, None], s2.double()[:, :, None, None]
        pre = r64 * t + b.double()[:, None, None] + nw.double() * nz.double()
        sg = abs(gain) * max(1.0, slope)
        a = (r64 * ta + b.double().abs()[:, None, None] + (nw.double() * nz.double()).abs()) * sg
        gf, sf = float(np.float32(gain)), float(np.float32(slope))
        o = torch.where(pre > 0, pre, pre * sf) * gf
        e1 = r64 * fx * sg if fx is not None else None
        check_sum(out, o, a, route["c"] + 5, path, what + " out", e1)
        check_sum(out2, o * s64, a * s64.abs(), route["c"] + 6, path, what + " out2", e1 * s64.abs() if e1 is not None else None)
    else:
        rs = torch.rand(n, c, generator=g, device=DEV) + 0.5
        mul = torch.randn(n, c, oh, ow, generator=g, device=DEV).contiguous(memory_format=torch.channels_last)
        y, _, dot = nhwc.blur(x, kd, pad, mode=2, row_scale=rs, mul=mul, want_dot=True)
        r64 = rs.double()[:, :, None, None]
        check_sum(y, t * r64, ta * r64, route["c"] + 1, path, what + " g_raw", fx * r64 if fx is not None else None)
        m64 = mul.double()
        check_sum(dot, (t * m64).sum((2, 3)), (ta * m64.abs()).sum((2, 3)), nhwc_dot_c(route), path,
                  what + " row_dot", (fx * m64.abs()).sum((2, 3)) if fx is not None else None)


KERNELS = re.compile(r"(fir4_band_kernel|upfirdn2d_generic_kernel|up2_k4_kernel|down2_k4_kernel|blur_nhwc_kernel)(<[^>]*>)?")


def routing_cases():
    """One case per class: (label, route, launcher)."""
    k4, k1 = filt("binom"), filt("full", 1, 1)
    out = []
    for w, px0, fused, vec in STRIP_CASES[::9]:
        cs = strip_case(w, px0, fused, vec)
        out.append(("strip w %d fused %s" % (w, fused), cs["shape"], cs["k"], dict(pad=cs["pad"], fused=fused,
                                                                                  out_off=cs["out_off"])))
    out.append(("16-tap", (2, 5, 21, 40), filt("full"), dict(pad=(1, 1, 1, 1))))
    for shape, pad in GEOMETRY_CASES:
        out.append(("geometry %s pad %s" % (shape, pad), shape, k4, dict(pad=pad)))
    for shape, up, down, pad, io, oo in POLY_CASES:
        out.append(("poly %s up %d down %d pad %s off %d/%d" % (shape, up, down, pad, io, oo), shape, k4,
                    dict(up=(up, up), down=(down, down), pad=pad, in_off=io, out_off=oo)))
    for shape, (kh, kw), pad in WIDE_PAD_CASES:
        out.append(("wide pad %s %dx%d" % (pad, kh, kw), shape, k4 if kh == 4 else k1, dict(pad=pad)))
        out.append(("wide pad %s %dx%d fused" % (pad, kh, kw), shape, k4 if kh == 4 else k1, dict(pad=pad, fused=True)))
    out.append(("crop backward (4, 1, 4, 1)", (2, 3, 38, 38), k4, dict(pad=(4, 1, 4, 1))))
    for p in ((1, 1), (2, 2), (2, 1), (1, 2)):
        out.append(("hot pad %s" % (p,), (4, 64, 129, 129), k4, dict(pad=(p[0], p[1], p[0], p[1]))))
        out.append(("hot pad %s fused" % (p,), (4, 64, 129, 129), k4, dict(pad=(p[0], p[1], p[0], p[1]), fused=True)))
    return out


@pytest.mark.gpu
def test_routing_matches_the_restatement():
    """The kernel each case launches (name and template arguments) is the one the Python planner predicts."""
    from gangealing_b200 import _lib
    from gangealing_b200.op import nhwc
    seen = []
    for label, shape, k, kw_ in routing_cases():
        fused = kw_.get("fused", False)
        up, down, pad = kw_.get("up", (1, 1)), kw_.get("down", (1, 1)), kw_["pad"]
        io, oo = kw_.get("in_off", 0), kw_.get("out_off", 0)
        route = fir_route(shape, k, up, down, pad, io, oo, fused, 0 if fused else None)
        x = at_offset(torch.randn(shape, device=DEV), io)
        kd = k.to(DEV)
        if fused:
            n, c = shape[:2]
            oh, ow = out_size(shape[2], shape[3], *k.shape, up, down, pad)
            nz, nw = torch.randn(n, oh, ow, device=DEV), torch.ones(1, device=DEV)
            b, rs = torch.zeros(c, device=DEV), torch.ones(n * c, device=DEV)
            names = launched(lambda: fused_raw(x, kd, pad, nz, nw, b, rs, 3, 0.2, SQRT2, oo), KERNELS)
        else:
            names = launched(lambda: fir_raw(x, kd, up, down, pad, oo), KERNELS)
        seen.append("%-48s -> %s" % (label, names))
        assert names == [route["name"]], "%s: launched %s, the restatement predicts %s" % (label, names, route["name"])
    for si, mode, kind, (slope, gain) in NHWC_CASES:
        shape, pad = NHWC_SHAPES[si], NHWC_PADS[si]
        k = filt(kind, seed=si)
        route = nhwc_route(shape, k, pad, mode, slope, gain, _lib.sm_count())
        x = torch.randn(shape, device=DEV).contiguous(memory_format=torch.channels_last)
        kd = k.to(DEV)
        p = route["plan"]
        kwargs = {}
        if mode == 1:
            kwargs = dict(bias=torch.zeros(shape[1], device=DEV), negative_slope=slope, gain=gain)
        if mode == 2:
            kwargs = dict(row_scale=torch.ones(shape[0], shape[1], device=DEV), want_dot=True,
                          mul=torch.ones(shape[0], shape[1], p["out_h"], p["out_w"], device=DEV).contiguous(
                              memory_format=torch.channels_last))
        names = [nm for nm in launched(lambda: nhwc.blur(x, kd, pad, mode=mode, **kwargs), KERNELS)]
        seen.append("%-48s -> %s" % ("nhwc %s mode %d %s slope %g" % (shape, mode, kind, slope), names))
        assert names == [route["name"]], (shape, mode, kind, names, route["name"])
    for line in seen:
        print("[route] " + line)


@pytest.mark.gpu
def test_zero_weight_columns_stay_finite_after_nan_in_shared_memory():
    """First a band launch whose bulk copies fill every stage slot of every CTA with NaN; then the cases whose stored
    outputs would weight columns outside -3 .. in_w + 2 (pad_x1 = 4, a 1x1 filter with pad 1, wider pads, the gradient of
    a (-1, 2) crop) must be finite and within their bound.  Shared memory need not keep its contents between launches, so
    this can miss a regression; the routing test is what proves the planner keeps these cases off the band kernel."""
    from gangealing_b200.op.upfirdn2d import UpFirDn2d
    k4 = filt("binom")
    poison_shape = (2, 64, 256, 256)
    route = fir_route(poison_shape, k4, pad=(1, 1, 1, 1))
    assert route["kind"] == "band" and route["plan"]["bands"] > 1 and route["plan"]["slot"] * 4 > STAGE_BUDGET - 2048
    assert route["plan"]["n_items"] >= 3 * 2 * H100_SMS               # every stage of every CTA is filled at least once
    nan_x = torch.full(poison_shape, float("nan"), device=DEV)

    def poison():
        assert bool(torch.isnan(fir_raw(nan_x, k4.to(DEV), pad=(1, 1, 1, 1))).all())

    g = seeded(77)
    for shape, (kh, kw), pad in WIDE_PAD_CASES:
        k = k4 if kh == 4 else filt("full", kh, kw)
        x = torch.randn(shape, generator=g, device=DEV)
        r = fir_route(shape, k, pad=pad)
        poison()
        check_fir(fir_raw(x, k.to(DEV), pad=pad), x, k, r, "after NaN shared memory: pad %s" % (pad,), pad=pad)
        n, c, h, w = shape
        oh, ow = out_size(h, w, kh, kw, (1, 1), (1, 1), pad)
        nz, nw = torch.randn(n, oh, ow, generator=g, device=DEV), torch.tensor([0.5], device=DEV)
        b, rs = torch.randn(c, generator=g, device=DEV), torch.rand(n * c, generator=g, device=DEV) + 0.5
        poison()
        y = fused_raw(x, k.to(DEV), pad, nz, nw, b, rs, 3, 0.2, SQRT2)
        check_tail(y, x, k, fir_route(shape, k, pad=pad, fused=True, noise_off=0), pad, nz, nw, b, rs, 0.2, SQRT2,
                   "after NaN shared memory: fused pad %s" % (pad,))
    x = torch.randn(2, 3, 40, 40, generator=g, device=DEV).requires_grad_(True)
    y = UpFirDn2d.apply(x, k4.to(DEV), (1, 1), (1, 1), (-1, 2, -1, 2))
    gy = torch.randn(y.shape, generator=g, device=DEV)
    poison()
    (gx,) = torch.autograd.grad(y, x, gy)
    gp = grad_pad(40, 40, y.shape[2], y.shape[3], 4, 4, (-1, 2, -1, 2))
    kf = torch.flip(k4, [0, 1])
    check_fir(gx, gy, kf, fir_route(tuple(gy.shape), kf, pad=gp), "after NaN shared memory: crop gradient, pad %s" % (gp,),
              pad=gp)
