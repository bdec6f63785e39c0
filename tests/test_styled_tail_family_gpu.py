"""The generator's fused StyledConv / ToRGB tails (csrc/styled.cu) against float64, over the code paths their launchers choose.

  styled_tail_nhwc_kernel<T, FAST, MASK>      demod + noise + bias + lrelu; out = o (MASK: its sign mask), xs = o*s_next,
                                              rgb = wm . o + rgb_bias + skip
  styled_tail_bwd_nhwc_kernel<T, MASK>        g_raw = lrelu'(out)*gain*(g_xs*s_next + wm^T g_rgb)*demod, and (general route)
                                              the per-CTA partial sums of d_s_next, d_demod and d_wm, finished by
                                              nhwc_finish_kernel: one launch for a packed (N, r, C) block, else one per sum

This file

  * restates the host-side planning in Python (fwd_route: the FAST gate, fwd_chunk and the trip structure; bwd_route:
    bwd_chunk, the pixel lanes, the U-pixel unrolled loop and its remainder, the reduction rows and the finish launches)
    and labels every case with its route; a CPU test asserts that the cases reach every label, planned for 132 SMs
    (H100 SXM), and a GPU test asserts, by the launched kernels' names under torch.profiler, that the restatement routes
    like the C++;
  * checks every output against float64 evaluated on the exact operands the launch reads (oracle/rounding.py):
        stored fp32 (out, xs, g_raw)   |y - ref| <= k * 2^-24 * A                 (assert_fp32_sum with c = k)
        stored bf16                    |y - ref| <= 1/2 ulp + k * 2^-24 * A        (assert_rounded_once)
        fp32 sums (rgb, d_*)           |y - ref| <= c * 2^-24 * sum|terms|
    with k and c derived from the kernels' operation order next to each check (fwd_k, bwd_k, the reduction geometry);
  * pins the sums over empty planes to exact zeros, a bad reduce_pitch to a refusal before any device work, and the
    Python faces' refusal of activations that are not 16-byte-aligned channels-last tensors of the right shape and dtype.

Every check prints its worst observed k / c (`[contract] ...` lines with `pytest -s`), and the module prints the worst per
route when it finishes.
"""
import re

import pytest
import torch

from fp64_contract import (BF16, CODE, DEV, F32, H100_SMS, SHORT, SQRT2, TNAME, VEC, Worst, assert_routes_reached,
                           ceil_div, f32, launched, library, nan_at, rowwise_c, rowwise_geometry, run_fresh, saved_output,
                           seeded)
from oracle.rounding import U32

UNROLL = {F32: 4, BF16: 2}        # pixels in flight per thread in the backward's unrolled loop
TRIP = 128                        # pixels one forward trip covers: 32 groups of 8 lanes x 4 pixels
ABSENT = ("noise", "noise_weight", "bias", "demod", "rgb_bias", "skip")


def _b(v):
    return "true" if v else "false"


def subsets_label(ds, dd, dwm):
    names = [nm for nm, on in (("d_s_next", ds), ("d_demod", dd), ("d_wm", dwm)) if on]
    return "+".join(names) if names else "none"


# ======================================================================================== planner restatement (no GPU)
def fast_gate(act, slope, gain):
    """launch_tail_fwd: the gain-folded epilogue max(T, T*slope), T = gain*t, equals lrelu(t)*gain."""
    a, g = f32(slope), f32(gain)
    return g > 0 and ((act == 3 and 0 <= a <= 1) or act == 1)


def fwd_route(dtype, n, c, hw, outputs, act=3, slope=0.2, gain=SQRT2, mask=False, sms=H100_SMS, absent=()):
    """launch_tail_fwd / fwd_chunk of csrc/styled.cu -> dict(name, chunk, k, j, partial, clamped, labels).
    outputs: a subset of {"out", "xs", "rgb"} ("out" is the sign mask when `mask`)."""
    v = VEC[dtype]
    fast = fast_gate(act, slope, gain)
    name = "styled_tail_nhwc_kernel<%s, %s, %s>" % (TNAME[dtype], _b(fast), _b(mask))
    k = max(1, min(ceil_div(8 * sms, n), ceil_div(hw, TRIP)))
    chunk = ceil_div(ceil_div(hw, k), TRIP) * TRIP
    kk = ceil_div(hw, chunk)
    j = c // (8 * v)
    last = hw - (kk - 1) * chunk                     # pixels of a sample's last CTA
    partial = last % TRIP != 0
    clamped = last % 4 != 0                          # a group's tail pixels are clamped, recomputed and not stored
    tag = "fwd %s" % SHORT[dtype]
    labels = {name, "fwd: %s" % ("FAST (gain folded)" if fast else "general epilogue"),
              "%s: K %s" % (tag, "= 1" if kk == 1 else "> 1"), "%s: J %s" % (tag, "= 1" if j == 1 else "> 1")}
    a, g = f32(slope), f32(gain)
    if act == 1:
        labels.add("fwd: linear, %s" % ("FAST" if fast else "gain <= 0 (general)"))
    elif not fast:
        labels.add("fwd general: slope > 1" if a > 1 else "fwd general: slope < 0" if a < 0 else "fwd general: gain <= 0")
    elif a in (0.0, 1.0):
        labels.add("fwd FAST: slope = %g" % a)
    if c == 2048:
        labels.add("%s: C = 2048" % tag)
    if hw < 4:
        labels.add("%s: HW < 4 (fewer pixels than one group)" % tag)
    if hw < TRIP:
        labels.add("%s: HW < 128 (fewer pixels than one trip)" % tag)
    if partial:
        labels.add("%s: a partial last trip" % tag)
        if 1 <= (last % TRIP) % 16 <= 12:
            labels.add("%s: a warp's groups leave the loop at different trips" % tag)
    if clamped:
        labels.add("%s: clamped tail pixels (HW %% 4 != 0)" % tag)
    if hw % chunk:
        labels.add("%s: a shorter last CTA (HW %% chunk != 0)" % tag)
    if chunk > TRIP:
        labels.add("%s: chunk of several trips" % tag)
    labels.add("fwd: outputs %s" % "+".join("mask" if (o == "out" and mask) else o for o in sorted(outputs)))
    for op in absent:
        if op in ("rgb_bias", "skip") and "rgb" not in outputs:
            continue
        labels.add("fwd: no %s" % op)
    return dict(name=name, chunk=chunk, k=kk, j=j, partial=partial, clamped=clamped, fast=fast, labels=labels)


def bwd_route(dtype, n, c, hw, g_xs, g_rgb, ds, dd, dwm, mask=False, layout="packed", sms=H100_SMS):
    """gg_styled_tail_backward_nhwc / _mask_nhwc of csrc/styled.cu -> dict(name, names launched in order, lanes, chunk, k,
    u, unrolled, remainder, r, finish, labels).  layout: "packed" (one (N, r, C) block, reduce_pitch r*C, as the Python
    face allocates), "dense" (separate dense outputs, reduce_pitch C) or "pitch0" (separate, reduce_pitch 0)."""
    v, u = VEC[dtype], UNROLL[dtype]
    cv = c // v
    lanes, chunk, kk = rowwise_geometry(n, cv, hw, sms)
    lens = {chunk, hw - (kk - 1) * chunk}
    unrolled = max(lens) > (u - 1) * lanes           # pp + (U-1)*lanes_p < p1 for the first pixel lane
    remainder = any(ceil_div(m - pl, lanes) % u for m in lens for pl in range(min(lanes, m)))
    name = "styled_tail_bwd_nhwc_kernel<%s, %s>" % (TNAME[dtype], _b(mask))
    r = ds + dd + 3 * dwm
    if r == 0:
        finish, nfin = "none", 0
    elif layout == "packed" or (layout == "dense" and r == 1):    # a lone dense sum with pitch C is a packed block of 1
        finish, nfin = "one packed launch", 1
    else:
        finish, nfin = "per sum (pitch %s)" % ("C" if layout == "dense" else "0"), ds + dd + dwm
    tag = "bwd %s" % SHORT[dtype]
    labels = {name, "%s: C/V = %d" % (tag, cv), "%s: K %s" % (tag, "= 1" if kk == 1 else "> 1"),
              "bwd %s: %s" % ("mask" if mask else "general",
                              "g_xs + g_rgb" if g_xs and g_rgb else "g_xs only" if g_xs else "g_rgb only")}
    if lanes == 1:
        labels.add("%s: lanes_p = 1 (C/V = 256)" % tag)
    if 256 % cv:
        labels.add("%s: 256 %% C/V != 0 (idle threads)" % tag)
    if unrolled:
        labels.add("%s: unrolled loop" % tag)
    if remainder:
        labels.add("%s: remainder loop" % tag)
    if remainder and not unrolled:
        labels.add("%s: remainder loop only" % tag)
    if unrolled and not remainder:
        labels.add("%s: unrolled loop only" % tag)
    if chunk % (u * lanes):
        labels.add("%s: chunk not a multiple of U x lanes_p" % tag)
    if not mask:
        labels.add("bwd sums: %s" % subsets_label(ds, dd, dwm))
        labels.add("bwd finish: %s" % finish)
    names = [name] + ["nhwc_finish_kernel"] * nfin
    return dict(name=name, names=names, lanes=lanes, chunk=chunk, k=kk, u=u, unrolled=unrolled, remainder=remainder,
                r=r, finish=finish, labels=labels)


# ============================================================================================================ cases
# forward: (dtype, n, c, hw, outputs, absent, act, slope, gain, mask)
ALL_OUT = ("out", "xs", "rgb")
FWD_GEOMETRY = {
    F32: [(1, 32, 1), (2, 64, 3), (3, 96, 16), (32, 192, 81), (1, 512, 128), (2, 2048, 129), (3, 32, 957),
          (2, 64, 65536), (32, 32, 16383), (1, 2048, 957), (2, 96, 4099)],
    BF16: [(1, 64, 1), (2, 192, 3), (3, 512, 16), (32, 64, 81), (1, 2048, 129), (2, 64, 128), (3, 192, 957),
           (2, 64, 65536), (32, 64, 16383), (2, 2048, 957), (2, 192, 4099)],
}
EPILOGUES = [(3, 0.2, SQRT2), (3, 1.5, SQRT2), (3, -0.3, 1.0), (3, 0.2, -0.7), (3, 0.2, 0.0), (3, 0.0, 2.0), (3, 1.0, 1.0),
             (1, 0.2, SQRT2), (1, 0.2, -1.3)]
ABSENT_SETS = [("noise",), ("noise_weight",), ("bias",), ("demod",), ("rgb_bias", "skip"),
               ("noise", "bias", "demod", "rgb_bias", "skip")]
OUTPUT_SETS = [("out",), ("xs",), ("rgb",), ("out", "xs"), ("xs", "rgb"), ("out", "rgb")]
MASK_OUTPUTS = [("out",), ("out", "xs"), ("out", "rgb"), ALL_OUT]


def fwd_cases():
    out = []
    for dt in (F32, BF16):
        for n, c, hw in FWD_GEOMETRY[dt]:
            out.append((dt, n, c, hw, ALL_OUT, (), 3, 0.2, SQRT2, False))
        for act, slope, gain in EPILOGUES:
            out.append((dt, 2, 128, 129, ALL_OUT, (), act, slope, gain, False))
        for i, ab in enumerate(ABSENT_SETS):
            act, slope, gain = EPILOGUES[i % 2]          # FAST and general alternate
            out.append((dt, 3, 192, 81, ALL_OUT, ab, act, slope, gain, False))
        for i, outs in enumerate(OUTPUT_SETS):
            act, slope, gain = EPILOGUES[(i + 1) % 2]
            out.append((dt, 2, 64 * (1 + i % 2), 957, outs, (), act, slope, gain, False))
        for i, outs in enumerate(MASK_OUTPUTS):
            for act, slope, gain in (EPILOGUES[0], EPILOGUES[1]):
                n, c, hw = ((1, 64, 3), (2, 128, 129), (3, 192, 957), (2, 64, 4099))[i]
                out.append((dt, n, c, hw, outs, (), act, slope, gain, True))
    return out


FWD_CASES = fwd_cases()

# backward: (dtype, n, c, hw, g_xs, g_rgb, ds, dd, dwm, mask, layout, slope, gain, demod)
BWD_CVS = [8, 24, 128, 256]           # 32 / 10 / 2 / 1 pixel lanes; 24 leaves 16 threads idle


def bwd_geometry(dt, cv, sms=H100_SMS):
    """Per C/V: K = 1 with a chunk just under 4 lane trips (fp32: unrolled and remainder; bf16: both); K > 1 with a chunk
    that is not a multiple of U x lanes_p; a chunk shorter than U lane trips (remainder only); many CTAs."""
    lanes = max(256 // cv, 1)
    c = cv * VEC[dt]
    u = UNROLL[dt]
    k5 = ceil_div(8 * sms, 5)
    return [(1, c, 4 * lanes - 1), (5, c, 7 * u * lanes + 3), (3, c, (u - 1) * lanes), (2, c, k5 * 2 * u * lanes + 5)]


def bwd_cases():
    out = []
    for dt in (F32, BF16):
        geo = [g for cv in BWD_CVS for g in bwd_geometry(dt, cv)]
        subsets = [(ds, dd, dwm) for ds in (0, 1) for dd in (0, 1) for dwm in (0, 1)]
        for i, (n, c, hw) in enumerate(geo):            # every geometry with every sum, the packed block
            slope, gain = ((0.2, SQRT2), (1.5, SQRT2), (0.2, -0.7), (-0.3, 1.0))[i % 4]
            out.append((dt, n, c, hw, True, True, 1, 1, 1, False, "packed", slope, gain, True))
        for i, (ds, dd, dwm) in enumerate(subsets):     # the 8 sum subsets
            n, c, hw = geo[(3 * i + 1) % len(geo)]
            out.append((dt, n, c, hw, True, True, ds, dd, dwm, False, "packed", 0.2, SQRT2, i % 3 != 2))
        for layout in ("dense", "pitch0"):               # per-sum finish launches through the C ABI
            for n, c, hw, s in ((5, 32 * VEC[dt] // 4, 1000, (1, 1, 1)), (2, 96 * VEC[dt] // 4, 3000, (1, 0, 1)),
                                (3, 64 * VEC[dt] // 4, 777, (0, 1, 0))):
                out.append((dt, n, c, hw, True, True, *s, False, layout, 0.2, SQRT2, True))
        for n, c, hw in (geo[1], geo[6]):                # one upstream gradient
            out.append((dt, n, c, hw, True, False, 1, 1, 0, False, "packed", 0.2, SQRT2, True))
            out.append((dt, n, c, hw, False, True, 0, 1, 1, False, "packed", 1.5, SQRT2, True))
            out.append((dt, n, c, hw, False, True, 0, 0, 0, False, "packed", 0.2, SQRT2, False))
        for i, (n, c, hw) in enumerate(geo):             # the sign-mask route (C % 32 == 0 for every geometry here)
            gx, gr = ((True, True), (True, False), (False, True))[i % 3]
            out.append((dt, n, c, hw, gx, gr, 0, 0, 0, True, "packed", (0.2, 1.5)[i % 2], SQRT2, i % 4 != 3))
    return out


BWD_CASES = bwd_cases()


def fwd_route_of(case, sms=H100_SMS):
    dt, n, c, hw, outs, ab, act, slope, gain, mask = case
    return fwd_route(dt, n, c, hw, outs, act, slope, gain, mask, sms, ab)


def bwd_route_of(case, sms=H100_SMS):
    dt, n, c, hw, gx, gr, ds, dd, dwm, mask, layout = case[:11]
    return bwd_route(dt, n, c, hw, gx, gr, ds, dd, dwm, mask, layout, sms)


# ======================================================================================================== CPU checks
def _required():
    req = []
    for dt in (F32, BF16):
        tn = TNAME[dt]
        req += ["styled_tail_nhwc_kernel<%s, %s, %s>" % (tn, f, m) for f in ("true", "false") for m in ("true", "false")]
        req += ["styled_tail_bwd_nhwc_kernel<%s, %s>" % (tn, m) for m in ("true", "false")]
        tag = "fwd %s" % SHORT[dt]
        req += ["%s: %s" % (tag, s) for s in (
            "K = 1", "K > 1", "J = 1", "J > 1", "C = 2048", "HW < 4 (fewer pixels than one group)",
            "HW < 128 (fewer pixels than one trip)", "a partial last trip", "a warp's groups leave the loop at different trips",
            "clamped tail pixels (HW % 4 != 0)", "a shorter last CTA (HW % chunk != 0)", "chunk of several trips")]
        tag = "bwd %s" % SHORT[dt]
        req += ["%s: C/V = %d" % (tag, cv) for cv in BWD_CVS]
        req += ["%s: %s" % (tag, s) for s in (
            "K = 1", "K > 1", "lanes_p = 1 (C/V = 256)", "256 % C/V != 0 (idle threads)", "unrolled loop", "remainder loop",
            "remainder loop only", "unrolled loop only", "chunk not a multiple of U x lanes_p")]
    req += ["fwd: FAST (gain folded)", "fwd: general epilogue", "fwd: linear, FAST", "fwd: linear, gain <= 0 (general)",
            "fwd general: slope > 1", "fwd general: slope < 0", "fwd general: gain <= 0", "fwd FAST: slope = 0",
            "fwd FAST: slope = 1"]
    req += ["fwd: no %s" % op for op in ABSENT]
    req += ["fwd: outputs %s" % s for s in ("out", "xs", "rgb", "out+xs", "rgb+xs", "out+rgb", "out+rgb+xs", "mask",
                                            "mask+xs", "mask+rgb", "mask+rgb+xs")]
    req += ["bwd sums: %s" % subsets_label(ds, dd, dwm) for ds in (0, 1) for dd in (0, 1) for dwm in (0, 1)]
    req += ["bwd finish: %s" % s for s in ("none", "one packed launch", "per sum (pitch C)", "per sum (pitch 0)")]
    req += ["bwd %s: %s" % (m, s) for m in ("general", "mask") for s in ("g_xs only", "g_rgb only", "g_xs + g_rgb")]
    req += ["nhwc_finish_kernel"]
    return req


REQUIRED = _required()


def all_routes(sms=H100_SMS):
    out = [fwd_route_of(cs, sms) for cs in FWD_CASES]
    for cs in BWD_CASES:
        r = bwd_route_of(cs, sms)
        r["labels"] |= set(r["names"][1:])
        out.append(r)
    return out


def test_cases_reach_every_route():
    """Coverage of the cases below, by the restatement planned for 132 SMs: each of the 8 forward and 4 backward
    instantiations, both sides of the FAST gate, every output subset and absent operand, K = 1 and K > 1 on both kernels,
    the forward's trip edges (HW < 4, < 128, % 128, % chunk, J = 1 and > 1), the backward's lane geometry (lanes_p = 1,
    idle threads, unrolled / remainder loop), all 8 sum subsets with each finish layout, and one or both upstream
    gradients on both backward routes."""
    reached = set()
    for r in all_routes():
        reached |= r["labels"]
    assert_routes_reached(REQUIRED, reached)


def test_restated_geometry_matches_the_workspace_query():
    """bwd_route's K agrees with gg_styled_tail_backward_workspace (5 fp32 partial rows per CTA and channel), planned for
    the SM count the library sees (132 without a device)."""
    from gangealing_b200 import _lib
    lib = _lib.load()
    sms = _lib.sm_count()
    for cs in BWD_CASES:
        dt, n, c, hw = cs[:4]
        assert lib.gg_styled_tail_backward_workspace(CODE[dt], n, c, hw) == n * bwd_route_of(cs, sms)["k"] * 5 * c * 4


def test_bad_reduce_pitch_is_refused_before_any_device_work():
    """A reduce_pitch other than 0, C or r*C is an argument error, returned before anything is launched (the pointers
    below are never dereferenced)."""
    from gangealing_b200 import _lib
    dll = _lib.load()
    one = 16
    for pitch in (7, 2 * 32, -32):      # r = 5: r*C = 160
        rc = dll.gg_styled_tail_backward_nhwc(one, one, one, one, one, one, one, one, one, one, one, one, 0, 0.2, 1.0,
                                              1, 32, 16, pitch, None)
        assert rc == -1 and b"reduce_pitch" in dll.gg_last_error(), (pitch, rc)
    # only d_s_next requested (r = 1): 0 and C are the valid pitches
    assert dll.gg_styled_tail_backward_nhwc(one, one, None, None, one, one, None, one, None, one, None, None, 0, 0.2, 1.0,
                                            1, 32, 16, 64, None) == -1
    # an empty plane is validated the same way before its sums are zeroed
    assert dll.gg_styled_tail_backward_nhwc(None, one, None, None, None, None, None, None, None, None, None, None, 0, 0.2,
                                            1.0, 2, 32, 0, 5, None) == -1


# ======================================================================================================== GPU checks
WORST = Worst("k (stored values) / c (sums) per route")
_report_worst = WORST.fixture()
check_stored, check_sum = WORST.check_stored, WORST.check_sum


def unpack_mask(words, c):
    """(N, HW, C/32) int32 words -> (N, HW, C) bool: bit b of word w is channel 32 w + b."""
    bits = (words.unsqueeze(-1) >> torch.arange(32, device=words.device, dtype=torch.int32)) & 1
    return bits.reshape(*words.shape[:-1], c).bool()


# ---------------------------------------------------------------------------------------------- forward
def fwd_k(case, fast):
    """fp32 roundings between the operands and o, on the longest chain (the noise term):
    FAST     d' = d*gain, b' = b*gain, nw' = nw*gain (1), nw'*noise (1), b' + nz (1), fma(x, d', .) (1), max(T, T*slope) (1
             if act 3)                                                               -> 5 (act 1: 4; no noise: 3 / 2)
    general  nw*noise (1), b + nz (1), fma (1), t*slope (1 if act 3), *gain (1)     -> 5 (act 1: 4; no noise: 3 / 2)
    The folds of the FAST route replace the general route's final *gain: same count, different places."""
    act, noise = case[6], "noise" not in case[5]
    neg = 1 if act == 3 else 0
    if fast:
        return (1 + 1 + 1 + 1 + neg) if noise else (1 + 1 + neg)
    return (1 + 1 + 1 + neg + 1) if noise else (1 + neg + 1)


def fwd_inputs(case, seed):
    dt, n, c, hw, outs, ab, act, slope, gain, mask = case
    g = seeded(seed)
    t = dict(raw=torch.randn(n, hw, c, generator=g, device=DEV).to(dt),
             noise=None if "noise" in ab else torch.randn(n, hw, generator=g, device=DEV),
             nw=None if "noise_weight" in ab else torch.tensor([0.3], device=DEV),   # kept without noise: ignored then
             bias=None if "bias" in ab else torch.randn(c, generator=g, device=DEV) * 0.5,
             demod=None if "demod" in ab else torch.rand(n, c, generator=g, device=DEV) + 0.5,
             s_next=torch.randn(n, c, generator=g, device=DEV) + 1.0 if "xs" in outs else None,
             wm=torch.randn(n, 3, c, generator=g, device=DEV) / c ** 0.5 if "rgb" in outs else None)
    rgb = "rgb" in outs
    t["rgb_bias"] = torch.randn(3, generator=g, device=DEV) if rgb and "rgb_bias" not in ab else None
    t["skip"] = torch.randn(n, 3, hw, generator=g, device=DEV) if rgb and "skip" not in ab else None
    if act == 3 and f32(gain) != 0:
        _dekink(t, dt)
    return t


def fwd_pre64(t):
    """-> (pre-activation, the same on absolute values) in float64 on the exact operands, (N, HW, C)."""
    x = t["raw"].double()
    if t["demod"] is not None:
        x = x * t["demod"].double()[:, None, :]
    pre, a = x, x.abs()
    if t["bias"] is not None:
        b = t["bias"].double()
        pre, a = pre + b, a + b.abs()
    if t["noise"] is not None:
        nz = (t["nw"].double() if t["nw"] is not None else 1.0) * t["noise"].double()[:, :, None]
        pre, a = pre + nz, a + nz.abs()
    return pre, a


def _dekink(t, dt):
    """Leaky-ReLU takes a different branch for a pre-activation within rounding of 0 in the kernel and in float64, and the
    branches differ by (1 - slope)*|pre|: move `raw` wherever |pre| < 2^-12 A, far beyond any bound checked here."""
    for _ in range(8):
        pre, a = fwd_pre64(t)
        bad = pre.abs() < a * 2.0 ** -12
        if not bool(bad.any()):
            return
        t["raw"] = torch.where(bad, t["raw"].float() + 0.375, t["raw"].float()).to(dt)
    raise AssertionError("could not move the inputs away from the activation kink")


def fwd_run(case, t):
    """One FWD_CASES entry through the C ABI into NaN-filled outputs -> (out or mask, xs, rgb)."""
    dt, n, c, hw, outs, ab, act, slope, gain, mask = case
    L = library()
    lib = L.load()
    out = None
    if "out" in outs:
        out = torch.full((n, hw, c // 32), 0x5A5A5A5A, dtype=torch.int32, device=DEV) if mask else nan_at((n, hw, c), dt)
    xs = nan_at((n, hw, c), dt) if "xs" in outs else None
    rgb = nan_at((n, 3, hw), F32) if "rgb" in outs else None
    entry = lib.gg_styled_tail_mask_nhwc if mask else lib.gg_styled_tail_nhwc
    L.check(entry(L.ptr(out), L.ptr(xs), L.ptr(rgb), t["raw"].data_ptr(), L.ptr(t["noise"]), L.ptr(t["nw"]), L.ptr(t["bias"]),
                  L.ptr(t["demod"]), L.ptr(t["s_next"]), L.ptr(t["wm"]), L.ptr(t["rgb_bias"]), L.ptr(t["skip"]), CODE[dt],
                  act, slope, gain, n, c, hw, L.stream()), "gg_styled_tail%s_nhwc" % ("_mask" if mask else ""))
    return out, xs, rgb


def _fwd_id(cs):
    dt, n, c, hw, outs, ab, act, slope, gain, mask = cs
    return "%s-n%d-c%d-hw%d-%s%s-act%d-s%g-g%.3g%s" % (SHORT[dt], n, c, hw, "+".join(outs), "-no_" + "_".join(ab) if ab else "",
                                                      act, slope, gain, "-mask" if mask else "")


@pytest.mark.gpu
@pytest.mark.parametrize("case", FWD_CASES, ids=_fwd_id)
def test_styled_tail_forward(case):
    """out = o (k = fwd_k), xs = RN(o*s_next) (k = fwd_k + 1), rgb = wm . o + rgb_bias + skip: a lane's C/8 fmas over its
    channel vectors, 3 butterfly steps, + rgb_bias, + skip, on o's fwd_k roundings -> c = C/8 + 5 + fwd_k.  The sign mask:
    each bit equals the sign of the float64 o wherever |o| exceeds o's rounding bound."""
    dt, n, c, hw, outs, ab, act, slope, gain, mask = case
    sms = library().sm_count()
    route = fwd_route_of(case, sms)
    path = route["name"]
    t = fwd_inputs(case, c + hw + 7 * n + int(100 * slope) + 13 * act)
    out, xs, rgb = fwd_run(case, t)
    pre, a = fwd_pre64(t)
    sl, gn = f32(slope), f32(gain)
    if act == 3:
        o, ao = torch.where(pre > 0, pre, pre * sl) * gn, a * abs(gn) * max(1.0, abs(sl))
    else:
        o, ao = pre * gn, a * abs(gn)
    k = fwd_k(case, route["fast"])
    what = "C=%d HW=%d N=%d (chunk %d, K %d, J %d) act %d slope %g gain %g" % (c, hw, n, route["chunk"], route["k"],
                                                                                route["j"], act, slope, gain)
    if out is not None and not mask:
        check_stored(out, o, ao, k, path, what + " out")
    if out is not None and mask:
        bits = unpack_mask(out, c)
        det = o.abs() > k * U32 * ao + 2.0 ** -120
        assert torch.equal(bits[det], (o > 0)[det]), "%s: %s: %d mask bits differ from the sign of o" % (
            path, what, int((bits[det] != (o > 0)[det]).sum()))
        if gn != 0:
            assert float(det.double().mean()) > 0.99, "the dekinked o should be determinate almost everywhere"
    if xs is not None:
        s = t["s_next"].double()[:, None, :]
        check_stored(xs, o * s, ao * s.abs(), k + 1, path, what + " xs")
    if rgb is not None:
        w = t["wm"].double()
        ref, ra = torch.einsum("noc,npc->nop", w, o), torch.einsum("noc,npc->nop", w.abs(), ao)
        if t["rgb_bias"] is not None:
            ref, ra = ref + t["rgb_bias"].double()[:, None], ra + t["rgb_bias"].double().abs()[:, None]
        if t["skip"] is not None:
            ref, ra = ref + t["skip"].double(), ra + t["skip"].double().abs()
        check_sum(rgb, ref, ra, c // 8 + 5 + k, path, what + " rgb")


# ---------------------------------------------------------------------------------------------- backward
def bwd_k(gx, gr):
    """fp32 roundings of g_t = lrelu'(out)*gain*g_o on its longest chain: g_xs*s_next (1), the three to-RGB fmas (3),
    *slope (1), *gain (1) -> 6 with both upstream gradients, 3 with g_xs only, 5 with g_rgb only (the first fma's
    addend g_xs*s_next is 0).  g_raw = g_t*demod adds one more when demod is given."""
    return (1 if gx else 0) + (3 if gr else 0) + 2


def sum_outputs(n, c, ds, dd, dwm, layout):
    """NaN-filled destinations: one (N, r, C) block (packed) or separate dense tensors carved from one buffer with gaps
    between them, so that they can never be mistaken for a packed block -> (d_s, d_d, d_w, reduce_pitch)."""
    r = ds + dd + 3 * dwm
    if r == 0:
        return None, None, None, 0
    if layout == "packed":
        block = nan_at((n, r, c), F32)
        i = 0
        d_s = d_d = d_w = None
        if ds:
            d_s, i = block[:, i], i + 1
        if dd:
            d_d, i = block[:, i], i + 1
        if dwm:
            d_w = block[:, i:i + 3]
        return d_s, d_d, d_w, r * c
    gap = 64
    buf = nan_at((gap + 5 * (n * c + gap),), F32)
    views, pos = [], gap
    for on, rows in ((ds, 1), (dd, 1), (dwm, 3)):
        if on:
            views.append(buf[pos:pos + rows * n * c].view((n, c) if rows == 1 else (n, 3, c)))
            pos += rows * n * c + gap
        else:
            views.append(None)
    return views[0], views[1], views[2], c if layout == "dense" else 0


def bwd_run(case, seed):
    dt, n, c, hw, gx, gr, ds, dd, dwm, mask, layout, slope, gain, has_demod = case
    L = library()
    lib = L.load()
    g = seeded(seed)
    t = dict(g_xs=torch.randn(n, hw, c, generator=g, device=DEV).to(dt) if gx else None,
             g_rgb=torch.randn(n, 3, hw, generator=g, device=DEV) if gr else None,
             s_next=torch.randn(n, c, generator=g, device=DEV) + 1.0 if gx else None,
             demod=torch.rand(n, c, generator=g, device=DEV) + 0.5 if has_demod else None,
             wm=torch.randn(n, 3, c, generator=g, device=DEV) / c ** 0.5 if gr else None,
             raw=torch.randn(n, hw, c, generator=g, device=DEV).to(dt) if dd else None)
    if mask:
        t["mask"] = torch.randint(-2 ** 31, 2 ** 31, (n, hw, c // 32), generator=g, device=DEV, dtype=torch.int32)
        t["pos"] = unpack_mask(t["mask"], c)
    else:
        t["out"] = saved_output((n, hw, c), g, dt)
        t["pos"] = t["out"] > 0
    g_raw = nan_at((n, hw, c), dt)
    d_s, d_d, d_w, pitch = sum_outputs(n, c, ds, dd, dwm, layout)
    if mask:
        L.check(lib.gg_styled_tail_backward_mask_nhwc(g_raw.data_ptr(), L.ptr(t["g_xs"]), L.ptr(t["g_rgb"]),
                                                      t["mask"].data_ptr(), L.ptr(t["s_next"]), L.ptr(t["demod"]),
                                                      L.ptr(t["wm"]), CODE[dt], slope, gain, n, c, hw, L.stream()),
                "gg_styled_tail_backward_mask_nhwc")
    else:
        r = ds + dd + 3 * dwm
        ws = torch.empty(max(1, lib.gg_styled_tail_backward_workspace(CODE[dt], n, c, hw) // 4), device=DEV) if r else None
        L.check(lib.gg_styled_tail_backward_nhwc(g_raw.data_ptr(), L.ptr(d_s), L.ptr(d_d), L.ptr(d_w), L.ptr(ws),
                                                 L.ptr(t["g_xs"]), L.ptr(t["g_rgb"]), t["out"].data_ptr(), L.ptr(t["raw"]),
                                                 L.ptr(t["s_next"]), L.ptr(t["demod"]), L.ptr(t["wm"]), CODE[dt], slope,
                                                 gain, n, c, hw, pitch, L.stream()), "gg_styled_tail_backward_nhwc")
    return t, g_raw, d_s, d_d, d_w


def _bwd_id(cs):
    dt, n, c, hw, gx, gr, ds, dd, dwm, mask, layout, slope, gain, has_demod = cs
    return "%s-n%d-c%d-hw%d-%s-%s%s-s%g-g%.3g%s" % (
        SHORT[dt], n, c, hw, "mask" if mask else "sums_" + subsets_label(ds, dd, dwm), "+".join(
            nm for nm, on in (("gxs", gx), ("grgb", gr)) if on), "" if mask or not (ds or dd or dwm) else "-" + layout,
        slope, gain, "" if has_demod else "-nodemod")


@pytest.mark.gpu
@pytest.mark.parametrize("case", BWD_CASES, ids=_bwd_id)
def test_styled_tail_backward(case):
    """g_raw = RN(g_t*demod) (k = bwd_k [+ 1 with demod]); d_s_next = sum g_xs*out and d_wm = sum g_rgb*out (c = a
    thread's fmas over its pixels + the CTA's pixel lanes + nhwc_finish_kernel's depth over K, as rowwise_c); d_demod =
    sum g_t*raw (that c + bwd_k, the roundings of g_t).  lrelu' comes from the saved activation (general route: ~5 % exact
    zeros take the slope) or from the sign mask (MASK route: random bits)."""
    dt, n, c, hw, gx, gr, ds, dd, dwm, mask, layout, slope, gain, has_demod = case
    sms = library().sm_count()
    route = bwd_route_of(case, sms)
    path = route["name"]
    t, g_raw, d_s, d_d, d_w = bwd_run(case, c + hw + 3 * n + 5 * ds + 7 * dd + 11 * dwm)
    go = torch.zeros(n, hw, c, dtype=torch.float64, device=DEV)
    goa = torch.zeros_like(go)
    if gx:
        x = t["g_xs"].double() * t["s_next"].double()[:, None, :]
        go, goa = go + x, goa + x.abs()
    if gr:
        w, gy = t["wm"].double(), t["g_rgb"].double()
        go, goa = go + torch.einsum("noc,nop->npc", w, gy), goa + torch.einsum("noc,nop->npc", w.abs(), gy.abs())
    sl = torch.where(t["pos"], torch.ones_like(go), torch.full_like(go, f32(slope))) * f32(gain)
    gt, gta = go * sl, goa * sl.abs()
    k = bwd_k(gx, gr)
    what = "C=%d HW=%d N=%d (lanes %d, chunk %d, K %d, U %d) slope %g gain %g" % (
        c, hw, n, route["lanes"], route["chunk"], route["k"], route["u"], slope, gain)
    if has_demod:
        d64 = t["demod"].double()[:, None, :]
        check_stored(g_raw, gt * d64, gta * d64.abs(), k + 1, path, what + " g_raw")
    else:
        check_stored(g_raw, gt, gta, k, path, what + " g_raw (no demod)")
    if mask:
        return
    # a thread's fma chain over its pixels, the CTA's pixel lanes in order, nhwc_finish_kernel over a sample's K CTAs
    cc = rowwise_c(n, c, hw, 0, True, dt, sms)
    o64 = t["out"].double()
    fin = route["finish"]
    if ds:
        y = t["g_xs"].double() * o64
        check_sum(d_s, y.sum(1), y.abs().sum(1), cc, path, what + " d_s_next, finish %s" % fin)
    if dd:
        r64 = t["raw"].double()
        check_sum(d_d, (gt * r64).sum(1), (gta * r64.abs()).sum(1), cc + k, path, what + " d_demod, finish %s" % fin)
    if dwm:
        gy = t["g_rgb"].double()
        check_sum(d_w, torch.einsum("nop,npc->noc", gy, o64), torch.einsum("nop,npc->noc", gy.abs(), o64.abs()), cc, path,
                  what + " d_wm, finish %s" % fin)


# ---------------------------------------------------------------------------------------------- empty planes, bad pitch
def _poison_allocator():
    """Leave NaN in the caching allocator's free small blocks, so that a small `torch.empty` result no launch writes is
    most likely NaN (the raw calls below check with explicit NaN buffers)."""
    ts = [torch.full((128,), float("nan"), device=DEV) for _ in range(256)]
    torch.cuda.synchronize()
    del ts


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, BF16])
def test_empty_planes_give_zero_sums(dt):
    """d_s_next, d_demod and d_wm over zero pixels (HW = 0, N*C > 0) are 0: through the Python face, and through the C ABI
    into a packed block and into separate outputs (reduce_pitch C and 0).  N = 0 writes nothing."""
    from gangealing_b200.op import nhwc
    L = library()
    lib = L.load()
    n, c = 2, 8 * VEC[dt]
    empty = torch.empty(n, c, 0, 5, dtype=dt, device=DEV).contiguous(memory_format=torch.channels_last)
    s = torch.ones(n, c, device=DEV)
    wm = torch.ones(n, 3, c, device=DEV)
    _poison_allocator()
    g_raw, d_s, d_d, d_w = nhwc.styled_tail_backward(empty, torch.empty(n, 3, 0, 5, device=DEV), empty, empty, s, s, wm,
                                                     True, True, True, 0.2, SQRT2)
    assert tuple(g_raw.shape) == (n, c, 0, 5)
    for got in (d_s, d_d, d_w):
        assert torch.equal(got, torch.zeros_like(got)), got
    for layout in ("packed", "dense", "pitch0"):
        for ds, dd, dwm in ((1, 1, 1), (1, 0, 0), (0, 1, 1)):
            d_s, d_d, d_w, pitch = sum_outputs(n, c, ds, dd, dwm, layout)
            L.check(lib.gg_styled_tail_backward_nhwc(None, L.ptr(d_s), L.ptr(d_d), L.ptr(d_w), None, None, None, None, None,
                                                     None, None, None, CODE[dt], 0.2, SQRT2, n, c, 0, pitch, L.stream()),
                    "gg_styled_tail_backward_nhwc")
            for got in (d_s, d_d, d_w):
                if got is not None:
                    assert torch.equal(got, torch.zeros_like(got)), (layout, ds, dd, dwm, got)
    block = nan_at((4, 5, c), F32)
    L.check(lib.gg_styled_tail_backward_nhwc(None, block[:, 0].data_ptr(), block[:, 1].data_ptr(), block[:, 2].data_ptr(),
                                             None, None, None, None, None, None, None, None, CODE[dt], 0.2, SQRT2, 0, c, 16,
                                             5 * c, L.stream()), "gg_styled_tail_backward_nhwc")
    assert bool(block.isnan().all()), "N = 0 has no sums to write"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, BF16])
def test_bad_reduce_pitch_leaves_every_output_untouched(dt):
    """A reduce_pitch other than 0, C or r*C returns -1 before the main kernel is launched: g_raw and the sums keep their
    NaN fill."""
    L = library()
    lib = L.load()
    n, c, hw = 2, 8 * VEC[dt], 300
    case = (dt, n, c, hw, True, True, 1, 1, 1, False, "dense", 0.2, SQRT2, True)
    t, _, _, _, _ = bwd_run(case, 3)
    for ds, dd, dwm, pitch in ((1, 1, 1, 2 * c), (1, 1, 1, c + 1), (1, 0, 0, 5 * c), (0, 1, 1, -c)):
        g_raw = nan_at((n, hw, c), dt)
        d_s, d_d, d_w, _ = sum_outputs(n, c, ds, dd, dwm, "dense")
        ws = torch.empty(lib.gg_styled_tail_backward_workspace(CODE[dt], n, c, hw) // 4, device=DEV)
        rc = lib.gg_styled_tail_backward_nhwc(g_raw.data_ptr(), L.ptr(d_s), L.ptr(d_d), L.ptr(d_w), ws.data_ptr(),
                                              t["g_xs"].data_ptr(), t["g_rgb"].data_ptr(), t["out"].data_ptr(),
                                              t["raw"].data_ptr(), t["s_next"].data_ptr(), t["demod"].data_ptr(),
                                              t["wm"].data_ptr(), CODE[dt], 0.2, SQRT2, n, c, hw, pitch, L.stream())
        assert rc == -1 and b"reduce_pitch" in lib.gg_last_error(), (pitch, rc)
        torch.cuda.synchronize()
        assert bool(g_raw.float().isnan().all()), "g_raw was written before the pitch was refused"
        for got in (d_s, d_d, d_w):
            assert got is None or bool(got.isnan().all())


# ---------------------------------------------------------------------------------------------- Python faces
def _misaligned_cl(t):
    """A copy of the channels-last tensor `t` one element past a 16-byte boundary."""
    n, c, h, w = t.shape
    m = torch.empty(1 + t.numel(), dtype=t.dtype, device=t.device)[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    m.copy_(t)
    assert m.is_contiguous(memory_format=torch.channels_last) and m.data_ptr() % 16
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, BF16])
def test_faces_refuse_activations_the_kernels_cannot_read(dt):
    """styled_tail and styled_tail_backward raise before any launch when raw, out_saved or g_xs is not a 16-byte-aligned
    channels-last tensor of the activation's shape and dtype (or g_rgb not dense fp32 (N, 3, H, W))."""
    from gangealing_b200.op import nhwc
    L = library()
    n, c, h, w = 2, 8 * VEC[dt], 5, 6
    g = seeded(5)
    cl = torch.channels_last
    raw = torch.randn(n, c, h, w, generator=g, device=DEV).to(dt).contiguous(memory_format=cl)
    out = raw.clone(memory_format=cl)
    s = torch.randn(n, c, generator=g, device=DEV)
    wm = torch.randn(n, 3, c, generator=g, device=DEV)
    g_rgb = torch.randn(n, 3, h, w, generator=g, device=DEV)
    other = F32 if dt == BF16 else BF16
    bad = {"NCHW": raw.contiguous(), "misaligned": _misaligned_cl(raw),
           "dtype": raw.to(other).contiguous(memory_format=cl),
           "shape": torch.randn(n, c, h, w + 1, device=DEV).to(dt).contiguous(memory_format=cl)}
    calls = L.CALLS
    for why, x in bad.items():
        if why not in ("dtype", "shape"):        # raw defines the activation: only its layout can be wrong
            with pytest.raises(RuntimeError, match="raw must be a 16-byte-aligned channels-last"):
                nhwc.styled_tail(x, None, None, None, None, s, wm, None, None, True, 0.2, SQRT2)
            with pytest.raises(RuntimeError, match="out_saved must be a 16-byte-aligned channels-last"):
                nhwc.styled_tail_backward(out.clone(memory_format=cl), None, x, None, s, s, None, True, False, False, 0.2,
                                          SQRT2)
        with pytest.raises(RuntimeError, match="g_xs must be a 16-byte-aligned channels-last tensor of the activation"):
            nhwc.styled_tail_backward(x, None, out, None, s, s, None, True, False, False, 0.2, SQRT2)
        with pytest.raises(RuntimeError, match="raw must be a 16-byte-aligned channels-last tensor of the activation"):
            nhwc.styled_tail_backward(out, g_rgb, out, x, None, s, wm, False, True, True, 0.2, SQRT2)
    with pytest.raises(RuntimeError, match="g_rgb must be a dense fp32"):
        nhwc.styled_tail_backward(None, g_rgb.transpose(2, 3), out, None, None, s, wm, False, False, True, 0.2, SQRT2)
    assert L.CALLS == calls, "a refused call reached the library"
    # the conforming tensors pass
    nhwc.styled_tail(raw, None, None, None, None, s, wm, None, None, True, 0.2, SQRT2)
    nhwc.styled_tail_backward(out, g_rgb, out, raw, s, s, wm, True, True, True, 0.2, SQRT2)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- routing
KERNELS = re.compile(r"(styled_tail_nhwc_kernel|styled_tail_bwd_nhwc_kernel|nhwc_finish_kernel)(<[^>]*>)?")


@pytest.mark.gpu
def test_routing_matches_the_restatement():
    """Every distinct route of the cases above launches the kernels (names, template arguments, number of finish
    launches) the restatement names."""
    run_fresh("test_styled_tail_family_gpu", "check_routing")


def check_routing():
    """The body of test_routing_matches_the_restatement (raises AssertionError on a mismatch)."""
    sms = library().sm_count()
    seen, done = [], set()

    def expect(label, key, names, fn):
        if key in done:
            return
        done.add(key)
        got = launched(fn, KERNELS)
        seen.append("%-72s -> %s" % (label, got))
        assert got == names, "%s: launched %s, the restatement predicts %s" % (label, got, names)

    for case in FWD_CASES:
        r = fwd_route_of(case, sms)
        t = fwd_inputs(case, 1)
        expect("fwd " + _fwd_id(case), (r["name"],), [r["name"]], lambda: fwd_run(case, t))
    for case in BWD_CASES:
        r = bwd_route_of(case, sms)
        expect("bwd " + _bwd_id(case), (tuple(r["names"]), r["finish"]), r["names"], lambda: bwd_run(case, 2))
    for line in seen:
        print("[route] " + line)
    print("[route] %d distinct routes" % len(seen))
