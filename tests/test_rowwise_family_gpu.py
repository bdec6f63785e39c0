"""The bias-activation, channel-scale and to-RGB kernels against float64, over the code paths their launchers choose.

These kernels run on every generator and STN layer of the step, forward and backward:

  csrc/bias_act.cu  rowwise_nchw_rows_kernel<T, MODE> (one warp per row, HW < 1024) and rowwise_nchw_kernel<T, VEC, MODE>
                    (a CTA per chunk of a row, 16-byte vectors or scalar), MODE 0 = channel scale (+ row_dot),
                    MODE 1 = bias-act backward (+ grad_bias), finished by row_finish_kernel / bias_grad_finish_kernel;
                    bias_act_flat_kernel<T, VEC, Index>; noise_bias_act_kernel<T, V> / noise_bias_act_scalar_kernel<T>
  csrc/nhwc.cu      noise_bias_act_nhwc_kernel<T>, rowwise_nhwc_kernel<T, MODE> + nhwc_finish_kernel,
                    to_rgb_nhwc_fwd_kernel, to_rgb_nhwc_bwd_kernel

Each launcher picks its kernel on the host from the shapes and the pointer alignment.  This file

  * restates those choices in Python (row_geom / launch_rowwise, launch_flat, launch_noise, rowwise_chunk, the to-RGB
    forward chunking) and labels every case with its route; a CPU test asserts that the cases reach every route and both
    sides of every threshold, planned for 132 SMs (H100 SXM), and a GPU test asserts, by the launched kernels' names under
    torch.profiler, that the restatement routes like the C++;
  * checks every output against float64 evaluated on the exact operands the launch reads (oracle/rounding.py):
        stored fp32      |y - ref| <= k * 2^-24 * A                   (assert_fp32_sum with c = k)
        stored fp16/bf16 |y - ref| <= 1/2 ulp + k * 2^-24 * A          (assert_rounded_once)
        fp32 sums        |y - ref| <= c * 2^-24 * sum|terms|           c from the launch geometry, stated per route
  * pins the empty-plane sums (row_dot, grad_bias, the channel scale's gradient, gwm) to exact zeros and the Python faces'
    handling of misaligned per-channel constants and activations.

Every check prints its worst observed k / c (`[contract] ...` lines with `pytest -s`), and the module prints the worst per
route when it finishes.  Not reached here: the 64-bit-index instantiations (bias_act_flat_kernel<T, *, long> at >= 2^31
elements and the NHWC 64-bit index path at more than 2^32 vectors), which need 8-16 GB tensors.
"""
import math
import re

import pytest
import torch

from fp64_contract import (BF16, CODE, DEV, F16, F32, H100_SMS, SHORT, SQRT2, TNAME, VEC, Worst, assert_routes_reached,
                           at_offset, ceil_div, cl, f32, finish_depth, launched, library, lrelu64, nan_at, randn, rowwise_c,
                           rowwise_geometry, run_fresh, saved_output, seeded, slope_gain)


# ======================================================================================== planner restatement (no GPU)
def row_geom(mode, hw):
    """row_geom of csrc/bias_act.cu -> (one warp per row, elements per CTA, K chunks per row)."""
    if hw < 1024:
        return True, hw, 1
    chunk = 16384 if mode == 0 else 8192
    return False, chunk, ceil_div(hw, chunk)


def nchw_rowwise_route(dtype, mode, n, c, hw, want_sum=True, x_off=0, y_off=0, out_off=0):
    """launch_rowwise of csrc/bias_act.cu -> dict(names launched in order, c of the sum, labels).  Offsets in elements
    from a 16-byte boundary."""
    v, tn = VEC[dtype], TNAME[dtype]
    small, chunk, k = row_geom(mode, hw)
    rows = n * c
    has_y = mode == 1 or want_sum
    tag = "nchw %s mode %d" % (SHORT[dtype], mode)
    labels = set()
    if small:
        names = ["rowwise_nchw_rows_kernel<%s, %d>" % (tn, mode)]
        chain, cta = ceil_div(hw, 32), 0
        labels.add("%s: rows, N*C %s" % (tag, "a multiple of 8" if rows % 8 == 0 else "not a multiple of 8"))
    else:
        shape_ok = hw % v == 0
        aligned = x_off % v == 0 and out_off % v == 0 and (not has_y or y_off % v == 0)
        vec = shape_ok and aligned
        names = ["rowwise_nchw_kernel<%s, %d, %d>" % (tn, v if vec else 1, mode)]
        m = min(chunk, hw)
        chain, cta = (ceil_div(m, 256 * v) * v if vec else ceil_div(m, 256)), 8
        labels.add("%s: %s" % (tag, "vector" if vec else "scalar (shape)" if not shape_ok else
                               "scalar (x misaligned)" if x_off % v else "scalar (y misaligned)" if y_off % v else
                               "scalar (out misaligned)"))
        labels.add("%s: K = %d" % (tag, k) if k <= 2 else "%s: K > 2" % tag)
        if hw == chunk:
            labels.add("%s: HW = chunk (K = 1)" % tag)
        if hw == chunk + 1:
            labels.add("%s: HW = chunk + 1 (K = 2)" % tag)
        if n > 1 and c > 1 and k > 1:
            labels.add("%s: N > 1, C > 1, K > 1" % tag)
    if hw == 1023:
        labels.add("%s: HW 1023 -> rows" % tag)
    if hw == 1024:
        labels.add("%s: HW 1024 -> chunked" % tag)
    finish = 0
    if want_sum:
        if mode == 1:
            names.append("bias_grad_finish_kernel")
            finish = ceil_div(n * k, 32) + 5
        elif not small:
            names.append("row_finish_kernel")
            finish = k
        labels.add("%s: with its sum" % tag)
    else:
        labels.add("%s: without a sum" % tag)
    labels |= set(names)
    return dict(names=names, c=chain + (1 if mode == 0 else 0) + 5 + cta + finish, labels=labels, k=k)


def flat_route(dtype, size, step_b, bias, ref, x_off=0, ref_off=0, out_off=0):
    """launch_flat of csrc/bias_act.cu (< 2^31 elements: 32-bit indices)."""
    v = VEC[dtype]
    aligned = x_off % v == 0 and out_off % v == 0 and (not ref or ref_off % v == 0)
    vec = (step_b % v == 0 or not bias) and size % v == 0 and aligned
    name = "bias_act_flat_kernel<%s, %d, unsigned int>" % (TNAME[dtype], v if vec else 1)
    why = ("vector" if vec else "scalar (misaligned)" if not aligned else "scalar (step_b %% %d)" % v
           if bias and step_b % v else "scalar (size %% %d)" % v)
    return dict(names=[name], labels={name, "flat: " + why})


def noise_route(dtype, n, c, hw, noise, x_off=0, noise_off=0, sms=H100_SMS):
    """launch_noise of csrc/bias_act.cu: the vector kernel, or the grid-stride scalar kernel capped at 16 CTAs per SM."""
    v = VEC[dtype]
    aligned = x_off % v == 0 and (not noise or noise_off % v == 0)
    vec = hw % v == 0 and aligned
    if vec:
        name = "noise_bias_act_kernel<%s, %d>" % (TNAME[dtype], v)
        labels = {name, "noise nchw: vector"}
    else:
        name = "noise_bias_act_scalar_kernel<%s>" % TNAME[dtype]
        labels = {name, "noise nchw: scalar (%s)" % ("shape" if hw % v else "x misaligned" if x_off % v else
                                                      "noise misaligned")}
        if n * c * hw > 16 * sms * 256:
            labels.add("noise nchw: scalar, a second grid-stride trip")
    return dict(names=[name], labels=labels)


def nhwc_rowwise_route(dtype, n, c, hw, sms=H100_SMS):
    """rowwise_chunk / launch_rowwise of csrc/nhwc.cu (and the elementwise noise_bias_act_nhwc_kernel)."""
    cv = c // VEC[dtype]
    lanes, chunk, k = rowwise_geometry(n, cv, hw, sms)
    tn = TNAME[dtype]
    tag = "nhwc %s" % SHORT[dtype]
    labels = {"%s: C/V = %d" % (tag, cv), "%s: N = %d" % (tag, n), "%s: K %s" % (tag, "= 1" if k == 1 else "> 1")}
    if chunk < 4 * lanes:
        labels.add("%s: chunk < 4 x lanes (tail loop only)" % tag)
    else:
        labels.add("%s: chunk >= 4 x lanes (4-pixel trips)" % tag)
    if chunk % lanes:
        labels.add("%s: chunk not a multiple of the lanes" % tag)
    if 256 % cv:
        labels.add("%s: lanes x C/V < 256 (idle threads)" % tag)
    names = {m: ["rowwise_nhwc_kernel<%s, %d>" % (tn, m), "nhwc_finish_kernel"] for m in (0, 1)}
    labels |= {names[0][0], names[1][0], "nhwc_finish_kernel", "noise_bias_act_nhwc_kernel<%s>" % tn}
    return dict(names=names, noise_name="noise_bias_act_nhwc_kernel<%s>" % tn, labels=labels, lanes=lanes, chunk=chunk,
                k=k)


def to_rgb_route(n, c, hw, sms=H100_SMS):
    """gg_to_rgb_nhwc_forward's chunking (a multiple of the 128 pixels one trip covers) and the backward's rowwise_chunk."""
    k = max(1, min(ceil_div(8 * sms, n), ceil_div(hw, 128)))
    chunk = ceil_div(ceil_div(hw, k), 128) * 128
    kf = ceil_div(hw, chunk)
    labels = {"to_rgb_nhwc_fwd_kernel", "to_rgb_nhwc_bwd_kernel", "to-RGB fwd: K %s" % ("= 1" if kf == 1 else "> 1"),
              "to-RGB fwd: %s" % ("float4 stores (HW % 4 == 0)" if hw % 4 == 0 else "scalar stores (HW % 4 != 0)")}
    if hw % 128:
        labels.add("to-RGB fwd: a partial last trip (HW % 128 != 0)")
    lanes, bchunk, kb = rowwise_geometry(n, c // 4, hw, sms)
    labels.add("to-RGB bwd: C/4 = %d (%d lanes)" % (c // 4, lanes))
    labels.add("to-RGB bwd: K %s" % ("= 1" if kb == 1 else "> 1"))
    if bchunk < 4 * lanes:
        labels.add("to-RGB bwd: chunk < 4 x lanes (tail loop only)")
    else:
        labels.add("to-RGB bwd: chunk >= 4 x lanes (4-pixel trips)")
    return dict(fwd_k=kf, lanes=lanes, bchunk=bchunk, kb=kb, labels=labels)


# ============================================================================================================ cases
HALF_ALL = [F32, F16, BF16]
NCHW_SMALL_HW = [1, 31, 32, 33, 1023]
NCHW_BIG_HW = [1024, 1025, 8192, 8193, 16384, 16385, 65536]


def nchw_cases():
    """(dtype, mode, n, c, hw, want_sum, x_off, y_off, out_off)"""
    out = []
    for dt in HALF_ALL:
        for mode in (0, 1):
            for i, hw in enumerate(NCHW_SMALL_HW):
                n, c = (2, 4) if i % 2 == 0 else (3, 5)          # N*C = 8 | 15 rows: full and partial 8-row CTAs
                out.append((dt, mode, n, c, hw, True, 0, 0, 0))
            for hw in NCHW_BIG_HW:
                out.append((dt, mode, 2, 3, hw, True, 0, 0, 0))
            out.append((dt, mode, 2, 3, 33, False, 0, 0, 0))
            out.append((dt, mode, 2, 3, 8192, False, 0, 0, 0))
            out.append((dt, mode, 2, 3, 8192, True, 1, 0, 0))     # x one element off a 16-byte boundary
            out.append((dt, mode, 2, 3, 8192, True, 0, 1, 0))     # y one element off
    return out


NCHW_CASES = nchw_cases()


def flat_cases():
    """(dtype, shape, layout, act, grad, bias, x_off, ref_off): layout 'nchw' | '2d' | 'cl'."""
    out = []
    i = 0
    for act in (1, 3):
        for grad in (0, 1, 2):
            for b in (True, False):
                out.append((HALF_ALL[i % 3], (2, 3, 8, 8), "nchw", act, grad, b, 0, 0))
                i += 1
    for dt in HALF_ALL:
        out.append((dt, (2, 3, 5, 5), "nchw", 3, 0, True, 0, 0))      # HW % V != 0 with a bias -> scalar
        out.append((dt, (2, 3, 5, 5), "nchw", 3, 1, False, 0, 0))     # no bias, size % V != 0 -> scalar
        out.append((dt, (4, 16), "2d", 3, 0, True, 0, 0))             # (N, C): step_b = 1
        out.append((dt, (2, 3, 8, 8), "nchw", 3, 1, True, 1, 0))      # x misaligned
        out.append((dt, (2, 3, 8, 8), "nchw", 3, 1, False, 0, 1))     # ref misaligned
    out.append((F32, (2, 12, 5, 6), "cl", 3, 0, True, 0, 0))          # channels-last through fused_bias_act_raw
    out.append((BF16, (2, 16, 5, 6), "cl", 3, 0, True, 0, 0))
    return out


FLAT_CASES = flat_cases()


def flat_step(shape, layout):
    if layout == "nchw":
        return shape[2] * shape[3]
    return 1


def noise_cases():
    """(dtype, shape, noise, noise_weight, bias, row_scale, x_off, noise_off)"""
    out = []
    i = 0
    for nz in (True, False):
        for nw in (True, False):
            for b in (True, False):
                for rs in (True, False):
                    for shape in ((2, 3, 8, 8), (2, 3, 5, 7)):         # vector | scalar by shape
                        out.append((HALF_ALL[i % 3], shape, nz, nw, b, rs, 0, 0))
                        i += 1
    for dt in HALF_ALL:
        out.append((dt, (2, 3, 8, 8), True, True, True, True, 1, 0))  # scalar: x misaligned
        out.append((dt, (2, 3, 8, 8), True, True, True, True, 0, 1))  # scalar: noise misaligned
    return out


NOISE_CASES = noise_cases()


def big_scalar_shape(sms):
    """A scalar (odd HW) plane larger than the scalar kernel's 16 CTAs x 256 threads per SM: a second grid-stride trip."""
    n, c = 2, 3
    return n, c, (16 * sms * 256 // (n * c)) * 5 // 4 | 1


NHWC_CVS = [1, 3, 12, 48, 255, 256]


def nhwc_cases(sms=H100_SMS):
    """(dtype, n, c, hw): per C/V, K = 1 with a chunk shorter than 4 lane trips; K = 2 with the tail loop only; and many
    CTAs with 4-pixel trips and a chunk that is not a multiple of the lanes."""
    out = []
    for dt in (F32, BF16):
        for cv in NHWC_CVS:
            lanes = max(256 // cv, 1)
            c = cv * VEC[dt]
            k5 = ceil_div(8 * sms, 5)
            out += [(dt, 1, c, 4 * lanes - 1), (dt, 5, c, 4 * lanes + 1), (dt, 5, c, k5 * 5 * lanes + 3)]
    return out


NHWC_CASES = nhwc_cases()
TO_RGB_CS = [32, 96, 512, 1024]
TO_RGB_HWS = [3, 4, 127, 128, 129, 4099, 65536]


def to_rgb_cases():
    """(n, c, hw, bias, skip, want_gx, want_gwm)"""
    out = []
    i = 0
    for c in TO_RGB_CS:
        for hw in TO_RGB_HWS:
            n = 1 if hw == 65536 else 2
            out.append((n, c, hw, i % 2 == 0, i % 4 < 2, i % 3 != 1, i % 3 != 0))   # gx only | both | gwm only
            i += 1
    return out


TO_RGB_CASES = to_rgb_cases()


# ======================================================================================================== CPU check
def all_routes(sms=H100_SMS):
    out = []
    for dt, mode, n, c, hw, ws, xo, yo, oo in NCHW_CASES:
        out.append(nchw_rowwise_route(dt, mode, n, c, hw, ws, xo, yo, oo))
    for dt, shape, layout, act, grad, b, xo, ro in FLAT_CASES:
        numel = math.prod(shape)
        out.append(flat_route(dt, numel, flat_step(shape, layout), b, grad == 1, xo, ro))
    for dt, shape, nz, nw, b, rs, xo, no in NOISE_CASES:
        out.append(noise_route(dt, shape[0], shape[1], shape[2] * shape[3], nz, xo, no, sms))
    n, c, hw = big_scalar_shape(sms)
    out.append(noise_route(F32, n, c, hw, True, sms=sms))
    for dt, n, c, hw in NHWC_CASES:
        out.append(nhwc_rowwise_route(dt, n, c, hw, sms))
    for n, c, hw, *_ in TO_RGB_CASES:
        out.append(to_rgb_route(n, c, hw, sms))
    return out


def _required():
    req = []
    for dt in HALF_ALL:
        tn, v = TNAME[dt], VEC[dt]
        for mode in (0, 1):
            tag = "nchw %s mode %d" % (SHORT[dt], mode)
            req += ["rowwise_nchw_rows_kernel<%s, %d>" % (tn, mode), "rowwise_nchw_kernel<%s, %d, %d>" % (tn, v, mode),
                    "rowwise_nchw_kernel<%s, 1, %d>" % (tn, mode)]
            req += ["%s: %s" % (tag, s) for s in (
                "rows, N*C a multiple of 8", "rows, N*C not a multiple of 8", "vector", "scalar (shape)",
                "scalar (x misaligned)", "scalar (y misaligned)", "K = 1", "K = 2", "K > 2", "HW = chunk (K = 1)",
                "HW = chunk + 1 (K = 2)", "N > 1, C > 1, K > 1", "HW 1023 -> rows", "HW 1024 -> chunked", "with its sum",
                "without a sum")]
        req += ["bias_act_flat_kernel<%s, %d, unsigned int>" % (tn, v), "bias_act_flat_kernel<%s, 1, unsigned int>" % tn,
                "noise_bias_act_kernel<%s, %d>" % (tn, v), "noise_bias_act_scalar_kernel<%s>" % tn]
    req += ["row_finish_kernel", "bias_grad_finish_kernel", "flat: vector", "flat: scalar (misaligned)",
            "flat: scalar (step_b % 4)", "flat: scalar (step_b % 8)", "flat: scalar (size % 4)", "flat: scalar (size % 8)",
            "noise nchw: vector", "noise nchw: scalar (shape)", "noise nchw: scalar (x misaligned)",
            "noise nchw: scalar (noise misaligned)", "noise nchw: scalar, a second grid-stride trip"]
    for dt in (F32, BF16):
        tn, tag = TNAME[dt], "nhwc %s" % SHORT[dt]
        req += ["rowwise_nhwc_kernel<%s, 0>" % tn, "rowwise_nhwc_kernel<%s, 1>" % tn, "noise_bias_act_nhwc_kernel<%s>" % tn]
        req += ["%s: C/V = %d" % (tag, cv) for cv in NHWC_CVS]
        req += ["%s: %s" % (tag, s) for s in ("N = 1", "N = 5", "K = 1", "K > 1", "chunk < 4 x lanes (tail loop only)",
                                               "chunk >= 4 x lanes (4-pixel trips)", "chunk not a multiple of the lanes",
                                               "lanes x C/V < 256 (idle threads)")]
    req += ["nhwc_finish_kernel", "to_rgb_nhwc_fwd_kernel", "to_rgb_nhwc_bwd_kernel", "to-RGB fwd: K = 1",
            "to-RGB fwd: K > 1", "to-RGB fwd: float4 stores (HW % 4 == 0)", "to-RGB fwd: scalar stores (HW % 4 != 0)",
            "to-RGB fwd: a partial last trip (HW % 128 != 0)", "to-RGB bwd: K = 1", "to-RGB bwd: K > 1",
            "to-RGB bwd: chunk < 4 x lanes (tail loop only)", "to-RGB bwd: chunk >= 4 x lanes (4-pixel trips)"]
    req += ["to-RGB bwd: C/4 = %d (%d lanes)" % (c // 4, max(256 // (c // 4), 1)) for c in TO_RGB_CS]
    return req


REQUIRED = _required()
UNREACHED = ["bias_act_flat_kernel<T, *, long> (>= 2^31 elements)", "NHWC 64-bit index path (> 2^32 vectors)"]


def test_cases_reach_every_route():
    """Coverage of the cases below, by the restatement planned for 132 SMs: every kernel instantiation the launchers pick
    below 2^31 elements, the vector and scalar routes with each reason for scalar, both sides of the 1024-element rows
    threshold and of a chunk boundary, K = 1, 2, > 2, and the channels-last and to-RGB geometry classes."""
    reached = set()
    for r in all_routes():
        reached |= r["labels"]
    assert_routes_reached(REQUIRED, reached, ["(8-16 GB tensors) " + lab for lab in UNREACHED])


def test_restated_geometry_matches_the_workspace_queries():
    """The restated K agrees with the library's workspace sizes (one fp32 partial per row and chunk / per CTA and channel)."""
    from gangealing_b200 import _lib
    lib = _lib.load()
    for hw in NCHW_SMALL_HW + NCHW_BIG_HW:
        assert lib.gg_channel_scale_workspace(6, hw) == 6 * row_geom(0, hw)[2] * 4
        assert lib.gg_bias_act_backward_workspace(2, 3, hw) == 6 * row_geom(1, hw)[2] * 4
    if torch.cuda.is_available():    # the channels-last plan depends on the device's SM count
        sms = _lib.sm_count()
        for dt, n, c, hw in NHWC_CASES:
            assert lib.gg_nhwc_rowwise_workspace(n, c, hw) >= n * nhwc_rowwise_route(dt, n, c, hw, sms)["k"] * c * 4


# ======================================================================================================== GPU checks
WORST = Worst("k (stored values) / c (sums) per route")
_report_worst = WORST.fixture()
check_stored, check_sum = WORST.check_stored, WORST.check_sum
A32, G32 = f32(0.2), f32(SQRT2)       # the slope and gain as the launches receive them


def act_grad64(gate):
    """(gate > 0 ? 1 : slope) * gain of the backward, with the fp32 slope and gain, in float64 (torch.where of two Python
    scalars would make a float32 tensor)."""
    return torch.where(gate > 0, torch.ones_like(gate), torch.full_like(gate, A32)) * G32


# ---------------------------------------------------------------------------------------------- NCHW row-wise
def nchw_rowwise(case, g):
    """Runs one NCHW_CASES entry through the C ABI -> (out, sum or None, x, y, s)."""
    dt, mode, n, c, hw, want_sum, xo, yo, oo = case
    L = library()
    lib = L.load()
    x = randn((n, c, hw), g, dt, xo)
    out = nan_at((n, c, hw), dt, oo)
    if mode == 0:
        y = randn((n, c, hw), g, dt, yo) if want_sum else None
        s = torch.randn(n * c, generator=g, device=DEV) + 0.25
        dot = torch.full((n * c,), float("nan"), device=DEV) if want_sum else None
        ws = torch.empty(max(1, lib.gg_channel_scale_workspace(n * c, hw) // 4), device=DEV) if want_sum else None
        L.check(lib.gg_channel_scale(out.data_ptr(), L.ptr(dot), L.ptr(ws), x.data_ptr(), L.ptr(y), s.data_ptr(), CODE[dt],
                                     n * c, hw, L.stream()), "gg_channel_scale")
        return out, dot, x, y, s
    y = saved_output((n, c, hw), g, dt, yo)
    gb = torch.full((c,), float("nan"), device=DEV) if want_sum else None
    ws = torch.empty(max(1, lib.gg_bias_act_backward_workspace(n, c, hw) // 4), device=DEV) if want_sum else None
    L.check(lib.gg_bias_act_backward(out.data_ptr(), L.ptr(gb), L.ptr(ws), x.data_ptr(), y.data_ptr(), CODE[dt], 0.2, SQRT2,
                                     n, c, hw, L.stream()), "gg_bias_act_backward")
    return out, gb, x, y, None


@pytest.mark.gpu
@pytest.mark.parametrize("case", NCHW_CASES, ids=lambda cs: "%s-m%d-%dx%dx%d-%s-off%d%d%d" % (
    SHORT[cs[0]], cs[1], cs[2], cs[3], cs[4], "sum" if cs[5] else "nosum", cs[6], cs[7], cs[8]))
def test_rowwise_nchw(case):
    """MODE 0: out = RN(x*s) (k = 1); row_dot = sum x*y (c = a thread's chain + 1 for the fma + 5 warp steps [+ 8 CTA
    warps] [+ K for row_finish_kernel]).  MODE 1: gx = RN((y > 0 ? g : 0.2 g)*gain) (k = 2); grad_bias = the sum of the
    STORED gx (c = a thread's chain + 5 [+ 8] + ceil(N*K/32) + 5 for bias_grad_finish_kernel)."""
    dt, mode, n, c, hw, want_sum, xo, yo, oo = case
    route = nchw_rowwise_route(dt, mode, n, c, hw, want_sum, xo, yo, oo)
    path = route["names"][0]
    out, sm, x, y, s = nchw_rowwise(case, seeded(hw + 31 * mode + 7 * xo + 3 * yo))
    x64 = x.double()
    if mode == 0:
        ref = x64 * s.double().reshape(n, c, 1)
        check_stored(out, ref, ref.abs(), 1, path, "out")
        if want_sum:
            t = x64 * y.double()
            check_sum(sm, t.sum(2).reshape(-1), t.abs().sum(2).reshape(-1), route["c"], path, "row_dot")
        return
    sl = act_grad64(y.double())
    ref = x64 * sl
    check_stored(out, ref, ref.abs(), 2, path, "gx")
    if want_sum:
        gx = out.double()
        check_sum(sm, gx.sum((0, 2)), gx.abs().sum((0, 2)), route["c"], path, "grad_bias")


# ---------------------------------------------------------------------------------------------- flat kernel
def flat_run(case, g):
    dt, shape, layout, act, grad, b, xo, ro = case
    L = library()
    c = shape[1]
    x = randn(shape, g, dt, xo)
    bias = torch.randn(c, generator=g, device=DEV) if b else None
    ref = saved_output(shape, g, dt, ro) if grad == 1 else None
    if layout == "cl":
        from gangealing_b200.op.fused_act import fused_bias_act_raw
        x = x.contiguous(memory_format=torch.channels_last)
        assert L.is_nhwc(x)
        out = fused_bias_act_raw(x, bias, ref, act, grad, 0.2, SQRT2)
    else:
        out = nan_at(shape, dt)
        bt = bias.to(dt) if bias is not None else None
        L.check(L.load().gg_fused_bias_act(out.data_ptr(), x.data_ptr(), L.ptr(bt), L.ptr(ref), CODE[dt], act, grad, 0.2,
                                           SQRT2, x.numel(), flat_step(shape, layout), c if b else 0, L.stream()),
                "gg_fused_bias_act")
    return out, x, bias, ref


@pytest.mark.gpu
@pytest.mark.parametrize("case", FLAT_CASES, ids=lambda cs: "%s-%s-%s-act%d-grad%d-%s-off%d%d" % (
    SHORT[cs[0]], "x".join(map(str, cs[1])), cs[2], cs[3], cs[4], "bias" if cs[5] else "nobias", cs[6], cs[7]))
def test_flat_bias_act(case):
    """out = RN(act(x + RN_T(b), ref)*gain): + b, *slope, *gain -> k = 3 (the bias is cast to the activation's type first,
    as fused_bias_act_raw does); grad = 2 stores exact zeros."""
    dt, shape, layout, act, grad, b, xo, ro = case
    route = flat_route(dt, math.prod(shape), flat_step(shape, layout), b, grad == 1, xo, ro)
    out, x, bias, ref = flat_run(case, seeded(act * 10 + grad + 100 * xo + 1000 * ro + len(shape)))
    path = route["names"][0]
    if grad == 2:
        assert bool((out == 0).all()), "%s: grad = 2 must store zeros" % path
        return
    bshape = (1, -1) + (1,) * (len(shape) - 2)
    b64 = bias.to(dt).double().reshape(bshape) if bias is not None else torch.zeros((), dtype=torch.float64, device=DEV)
    pre = x.double() + b64
    a = (x.double().abs() + b64.abs()) * slope_gain(0.2, SQRT2)
    if act == 1:
        r64 = pre * G32
    else:
        gate = pre if grad == 0 else ref.double()
        r64 = lrelu64(pre, A32, G32) if grad == 0 else torch.where(gate > 0, pre, pre * A32) * G32
    check_stored(out, r64, a, 3, path, "act %d grad %d %s %s" % (act, grad, layout, tuple(shape)))


# ---------------------------------------------------------------------------------------------- noise_bias_act NCHW
def noise_run(dt, shape, nz, nw, b, rs, xo, no, g):
    L = library()
    n, c, h, w = shape
    hw = h * w
    x = randn((n, c, hw), g, dt, xo)
    noise = randn((n, hw), g, dt, no) if nz else None
    nwt = torch.tensor([0.7], device=DEV) if nw else None
    bias = torch.randn(c, generator=g, device=DEV) if b else None
    rsv = torch.rand(n * c, generator=g, device=DEV) + 0.5 if rs else None
    out = nan_at((n, c, hw), dt)
    L.check(L.load().gg_noise_bias_act(out.data_ptr(), x.data_ptr(), L.ptr(noise), L.ptr(nwt), L.ptr(bias), L.ptr(rsv),
                                       CODE[dt], 0.2, SQRT2, n, c, hw, L.stream()), "gg_noise_bias_act")
    x64 = x.double()
    pre = x64 * (rsv.double().reshape(n, c, 1) if rs else 1.0)
    a = pre.abs()
    if b:
        pre, a = pre + bias.double()[:, None], a + bias.double().abs()[:, None]
    if nz:
        t = (0.7 if nw else 1.0) * noise.double()[:, None, :]
        pre, a = pre + t, a + t.abs()
    return out, lrelu64(pre, A32, G32), a * slope_gain(0.2, SQRT2)


@pytest.mark.gpu
@pytest.mark.parametrize("case", NOISE_CASES, ids=lambda cs: "%s-%s-nz%d-nw%d-b%d-rs%d-off%d%d" % (
    SHORT[cs[0]], "x".join(map(str, cs[1])), *map(int, cs[2:6]), cs[6], cs[7]))
def test_noise_bias_act_nchw(case):
    """out = RN(lrelu(rs*x + b + nw*noise)*gain): the fma with rs, the noise fma, *slope, *gain and one more for the scalar
    kernel's separate product -> k = 5.  noise_weight = None means 1."""
    dt, shape, nz, nw, b, rs, xo, no = case
    route = noise_route(dt, shape[0], shape[1], shape[2] * shape[3], nz, xo, no, library().sm_count())
    out, ref, a = noise_run(dt, shape, nz, nw, b, rs, xo, no, seeded(sum(shape) + 2 * nz + 4 * nw + 8 * b + 16 * rs))
    check_stored(out, ref, a, 5, route["names"][0], "%s noise %s nw %s bias %s rs %s" % (shape, nz, nw, b, rs))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", HALF_ALL)
def test_noise_bias_act_scalar_grid_stride(dt):
    """A scalar-route tensor larger than 16 CTAs x 256 threads per SM: threads take a second grid-stride trip."""
    sms = library().sm_count()
    n, c, hw = big_scalar_shape(sms)
    route = noise_route(dt, n, c, hw, True, sms=sms)
    assert "noise nchw: scalar, a second grid-stride trip" in route["labels"]
    out, ref, a = noise_run(dt, (n, c, hw, 1), True, False, True, True, 0, 0, seeded(5))
    check_stored(out, ref, a, 5, route["names"][0], "grid-stride (%d, %d, %d)" % (n, c, hw))


# ---------------------------------------------------------------------------------------------- channels-last family
def nhwc_shape(n, c, hw):
    """(N, C, H, W) with H * W = hw and H, W > 1 where possible (so the tensor is unambiguously channels-last)."""
    h = next((d for d in range(2, int(hw ** 0.5) + 1) if hw % d == 0), 1)
    return n, c, h, hw // h


@pytest.mark.gpu
@pytest.mark.parametrize("case", NHWC_CASES, ids=lambda cs: "%s-n%d-c%d-hw%d" % (SHORT[cs[0]], *cs[1:]))
def test_rowwise_nhwc(case):
    """channel_scale: out = RN(x*s) (k = 1), row_dot = sum x*y; bias_act_backward: gx = RN((out > 0 ? g : 0.2 g)*gain)
    (k = 2), grad_bias = the sum of the unrounded gx (+2); noise_bias_act_nhwc (k = 5).  Sums: a thread's pixels, the CTA's
    pixel lanes in order, nhwc_finish_kernel over the CTAs (per sample for row_dot, over N*K for grad_bias)."""
    from gangealing_b200.op import nhwc
    dt, n, c, hw = case
    sms = library().sm_count()
    route = nhwc_rowwise_route(dt, n, c, hw, sms)
    shape = nhwc_shape(n, c, hw)
    g = seeded(c + hw + n)
    what = "C=%d HW=%d N=%d (lanes %d, chunk %d, K %d)" % (c, hw, n, route["lanes"], route["chunk"], route["k"])
    x, y = cl(randn(shape, g, dt)), cl(randn(shape, g, dt))
    s = torch.randn(n, c, generator=g, device=DEV)
    out, dot = nhwc.channel_scale(x, s, y)
    ref = x.double() * s.double()[:, :, None, None]
    check_stored(out, ref, ref.abs(), 1, route["names"][0][0], what + " out")
    t = x.double() * y.double()
    check_sum(dot, t.sum((2, 3)), t.abs().sum((2, 3)), rowwise_c(n, c, hw, 0, True, dt, sms), route["names"][0][0],
              what + " row_dot")
    saved = cl(saved_output(shape, g, dt))
    gx, gb = nhwc.bias_act_backward(x, saved, 0.2, SQRT2, True)
    ref = x.double() * act_grad64(saved.double())
    check_stored(gx, ref, ref.abs(), 2, route["names"][1][0], what + " gx")
    check_sum(gb, ref.sum((0, 2, 3)), ref.abs().sum((0, 2, 3)), rowwise_c(n, c, hw, 2, False, dt, sms),
              route["names"][1][0], what + " grad_bias")
    noise = torch.randn(n, 1, shape[2], shape[3], generator=g, device=DEV)
    nw = torch.tensor([0.7], device=DEV)
    b = torch.randn(c, generator=g, device=DEV)
    rs = torch.rand(n, c, generator=g, device=DEV) + 0.5
    o = nhwc.noise_bias_act(x, noise, nw, b, rs, 0.2, SQRT2)
    pre = x.double() * rs.double()[:, :, None, None]
    a = pre.abs() + b.double().abs()[:, None, None] + (0.7 * noise.double()).abs()
    pre = pre + b.double()[:, None, None] + 0.7 * noise.double()
    check_stored(o, lrelu64(pre, A32, G32), a * slope_gain(0.2, SQRT2), 5, route["noise_name"], what + " noise_bias_act")


def to_rgb_run(case, g):
    """Raw to-RGB forward / backward on an NHWC activation held as (N, HW, C)."""
    L = library()
    lib = L.load()
    n, c, hw, b, sk, want_gx, want_gwm = case
    x = torch.randn(n, hw, c, generator=g, device=DEV)
    wm = torch.randn(n, 3, c, generator=g, device=DEV) / c ** 0.5
    bias = torch.randn(3, generator=g, device=DEV) if b else None
    skip = torch.randn(n, 3, hw, generator=g, device=DEV) if sk else None
    out = nan_at((n, 3, hw), F32)
    L.check(lib.gg_to_rgb_nhwc_forward(out.data_ptr(), x.data_ptr(), wm.data_ptr(), L.ptr(bias), L.ptr(skip), n, c, hw,
                                       L.stream()), "gg_to_rgb_nhwc_forward")
    gy = torch.randn(n, 3, hw, generator=g, device=DEV)
    gx = nan_at((n, hw, c), F32) if want_gx else None
    gwm = nan_at((n, 3, c), F32) if want_gwm else None
    ws = torch.empty(max(1, lib.gg_to_rgb_nhwc_workspace(n, c, hw) // 4), device=DEV) if want_gwm else None
    L.check(lib.gg_to_rgb_nhwc_backward(L.ptr(gx), L.ptr(gwm), L.ptr(ws), gy.data_ptr(), x.data_ptr(), wm.data_ptr(), n, c,
                                        hw, L.stream()), "gg_to_rgb_nhwc_backward")
    return x, wm, bias, skip, out, gy, gx, gwm


@pytest.mark.gpu
@pytest.mark.parametrize("case", TO_RGB_CASES, ids=lambda cs: "n%d-c%d-hw%d-b%d-skip%d-gx%d-gwm%d" % (
    cs[0], cs[1], cs[2], *map(int, cs[3:])))
def test_to_rgb_nhwc(case):
    """Forward: out = wm . x + bias + skip: a lane's C/8 fmas, 3 butterfly steps, + bias, + skip -> c = C/8 + 5.
    Backward: gx = sum_o wm*g (3 roundings, k = 3); gwm = sum_p g*x: a thread's pixels, the CTA's pixel lanes, the finish
    kernel over the K CTAs of a sample."""
    n, c, hw, b, sk, want_gx, want_gwm = case
    sms = library().sm_count()
    route = to_rgb_route(n, c, hw, sms)
    x, wm, bias, skip, out, gy, gx, gwm = to_rgb_run(case, seeded(c + hw))
    x64, w64, g64 = x.double(), wm.double(), gy.double()
    ref = torch.einsum("noc,npc->nop", w64, x64)
    a = torch.einsum("noc,npc->nop", w64.abs(), x64.abs())
    if b:
        ref, a = ref + bias.double()[:, None], a + bias.double().abs()[:, None]
    if sk:
        ref, a = ref + skip.double(), a + skip.double().abs()
    what = "C=%d HW=%d N=%d" % (c, hw, n)
    check_sum(out, ref, a, c // 8 + 5, "to_rgb_nhwc_fwd_kernel", what + " out (fwd K %d)" % route["fwd_k"])
    if want_gx:
        r = torch.einsum("noc,nop->npc", w64, g64)
        check_stored(gx, r, torch.einsum("noc,nop->npc", w64.abs(), g64.abs()), 3, "to_rgb_nhwc_bwd_kernel", what + " gx")
    if want_gwm:
        r = torch.einsum("nop,npc->noc", g64, x64)
        ra = torch.einsum("nop,npc->noc", g64.abs(), x64.abs())
        cc = ceil_div(route["bchunk"], route["lanes"]) + route["lanes"] + finish_depth(route["kb"])
        check_sum(gwm, r, ra, cc, "to_rgb_nhwc_bwd_kernel", what + " gwm (lanes %d, K %d)" % (route["lanes"], route["kb"]))


# ---------------------------------------------------------------------------------------------- empty planes
def _poison_allocator():
    """Leave NaN in the caching allocator's free small blocks, so that a small `torch.empty` result no launch writes is
    most likely NaN (the raw calls below check with explicit NaN buffers)."""
    ts = [torch.full((128,), float("nan"), device=DEV) for _ in range(256)]
    torch.cuda.synchronize()
    del ts


@pytest.mark.gpu
@pytest.mark.parametrize("dt", HALF_ALL)
def test_empty_planes_give_zero_sums_nchw(dt):
    """A sum over an empty plane is 0: row_dot of gg_channel_scale with HW = 0, grad_bias of gg_bias_act_backward with
    N*HW = 0, and the gradient of channel_scale(x, s) w.r.t. s for an (N, C, 0, W) input."""
    L = library()
    lib = L.load()
    for rows, hw in ((6, 0), (1, 0)):
        dot = torch.full((rows,), float("nan"), device=DEV)
        L.check(lib.gg_channel_scale(None, dot.data_ptr(), None, None, None, None, CODE[dt], rows, hw, L.stream()),
                "gg_channel_scale")
        assert torch.equal(dot, torch.zeros_like(dot)), dot
    for n, c, hw in ((2, 3, 0), (0, 3, 16)):
        gb = torch.full((c,), float("nan"), device=DEV)
        L.check(lib.gg_bias_act_backward(None, gb.data_ptr(), None, None, None, CODE[dt], 0.2, SQRT2, n, c, hw, L.stream()),
                "gg_bias_act_backward")
        assert torch.equal(gb, torch.zeros_like(gb)), gb
    from gangealing_b200.op.modconv import channel_scale
    x = torch.randn(2, 3, 0, 5, device=DEV, dtype=dt)
    s = torch.randn(2, 3, device=DEV, requires_grad=True)
    y = channel_scale(x, s)
    _poison_allocator()
    (gs,) = torch.autograd.grad(y, s, torch.randn_like(y))
    assert torch.equal(gs, torch.zeros_like(gs)), gs


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, BF16])
def test_empty_planes_give_zero_sums_nhwc(dt):
    """The channels-last row_dot (per sample and channel), grad_bias and the to-RGB gwm over zero pixels are 0."""
    L = library()
    lib = L.load()
    c = 4 * VEC[dt]
    dot = torch.full((2, c), float("nan"), device=DEV)
    s = torch.ones(2, c, device=DEV)
    # y and the saved output must be non-null; an empty plane reads nothing through them
    L.check(lib.gg_channel_scale_nhwc(None, dot.data_ptr(), None, None, s.data_ptr(), s.data_ptr(), CODE[dt], 2, c, 0,
                                      L.stream()), "gg_channel_scale_nhwc")
    assert torch.equal(dot, torch.zeros_like(dot)), dot
    for n, hw in ((2, 0), (0, 16)):
        gb = torch.full((c,), float("nan"), device=DEV)
        L.check(lib.gg_bias_act_backward_nhwc(None, gb.data_ptr(), None, None, s.data_ptr(), CODE[dt], 0.2, SQRT2, n, c, hw,
                                              L.stream()), "gg_bias_act_backward_nhwc")
        assert torch.equal(gb, torch.zeros_like(gb)), gb
    gwm = torch.full((2, 3, 32), float("nan"), device=DEV)
    L.check(lib.gg_to_rgb_nhwc_backward(None, gwm.data_ptr(), None, s.data_ptr(), s.data_ptr(), s.data_ptr(), 2, 32, 0,
                                        L.stream()), "gg_to_rgb_nhwc_backward")
    assert torch.equal(gwm, torch.zeros_like(gwm)), gwm


# ---------------------------------------------------------------------------------------------- misaligned operands
@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, BF16])
def test_faces_take_misaligned_constants_and_activations(dt):
    """Per-channel constants that are slices 4 bytes off a 16-byte boundary reach the float4 reads as aligned copies, and a
    channels-last activation one element off takes the NCHW route; every result is the float64 one."""
    from gangealing_b200 import op
    from gangealing_b200.op import nhwc
    from gangealing_b200.op.feature_distance import feature_distance
    from gangealing_b200.op.modconv import _ToRGB
    from gangealing_b200.op.vgg_pool import bias_relu_pool
    g = seeded(17)
    n, c, h, w = 2, 64, 6, 4
    x = cl(randn((n, c, h, w), g, dt))
    b_all = torch.randn(c + 1, generator=g, device=DEV)
    b = b_all[1:]
    assert b.is_contiguous() and b.data_ptr() % 16 == 4
    rs_all = torch.rand(n * c + 1, generator=g, device=DEV) + 0.5
    rs = rs_all[1:].view(n, c)
    y = nhwc.noise_bias_act(x, None, None, b, rs, 0.2, SQRT2)
    pre = x.double() * rs.double()[:, :, None, None] + b.double()[:, None, None]
    a = (x.double() * rs.double()[:, :, None, None]).abs() + b.double().abs()[:, None, None]
    check_stored(y, lrelu64(pre, A32, G32), a * slope_gain(0.2, SQRT2), 5, "noise_bias_act_nhwc (face)", "offset constants")
    y = op.fused_leaky_relu(x, b)
    bq = b.to(dt).double()[:, None, None] if dt != F32 else b.double()[:, None, None]
    check_stored(y, lrelu64(x.double() + b.double()[:, None, None], A32, G32),
                 (x.double().abs() + b.double().abs()[:, None, None]) * slope_gain(0.2, SQRT2), 5,
                 "fused_leaky_relu (face)", "offset bias")
    # a channels-last activation one element off a 16-byte boundary: the flat kernel's scalar route forward; the backward
    # gates on the (freshly allocated, aligned) output
    xl = torch.empty(1 + x.numel(), dtype=dt, device=DEV)[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    xl.copy_(x)
    assert xl.data_ptr() % 16 != 0 and library().is_nhwc(xl) and not nhwc.elementwise_ok(xl) and not nhwc.rowwise_ok(xl)
    xl.requires_grad_(True)
    bl = b.clone().requires_grad_(True)
    y = op.fused_leaky_relu(xl, bl)
    pre = x.double() + bq
    check_stored(y, lrelu64(pre, A32, G32), (x.double().abs() + bq.abs()) * slope_gain(0.2, SQRT2), 3,
                 "fused_leaky_relu (misaligned activation)", "forward")
    gy = cl(randn(y.shape, g, dt))
    gx, gb = torch.autograd.grad(y, [xl, bl], gy)
    ref = gy.double() * act_grad64(y.double())
    check_stored(gx, ref, ref.abs(), 2, "fused_leaky_relu (misaligned activation)", "gx")
    check_sum(gb.float(), ref.sum((0, 2, 3)), ref.abs().sum((0, 2, 3)),
              rowwise_c(n, c, h * w, 2, False, dt, library().sm_count()), "fused_leaky_relu (misaligned activation)",
              "grad_bias")
    if dt != F32:
        return
    # to-RGB with a wm and a skip off their boundaries, the VGG bias and the LPIPS weights likewise
    wm = at_offset(torch.randn(n, 3, c, generator=g, device=DEV) / 8, 1)
    skip = at_offset(torch.randn(n, 3, h, w, generator=g, device=DEV), 3)
    out = _ToRGB.apply(x, wm, None, skip)
    ref = torch.einsum("noc,nchw->nohw", wm.double(), x.double()) + skip.double()
    a = torch.einsum("noc,nchw->nohw", wm.double().abs(), x.double().abs()) + skip.double().abs()
    check_sum(out, ref, a, c // 8 + 5, "to_rgb_nhwc_fwd_kernel (face)", "offset wm, skip")
    yp, _ = bias_relu_pool(x, b)
    check_stored(yp, torch.relu(x.double() + b.double()[:, None, None]), x.double().abs() + b.double().abs()[:, None, None],
                 1, "bias_relu_pool (face)", "offset bias")
    f1 = cl(randn((n, c, h, w), g, dt))
    wt = (torch.rand(c + 1, generator=g, device=DEV) + 0.1)[1:]
    d_off = feature_distance(x, f1, wt)
    d_ref = feature_distance(x, f1, wt.clone())
    assert torch.equal(d_off, d_ref)


# ---------------------------------------------------------------------------------------------- routing
KERNELS = re.compile(r"(rowwise_nchw_rows_kernel|rowwise_nchw_kernel|row_finish_kernel|bias_grad_finish_kernel|"
                     r"bias_act_flat_kernel|noise_bias_act_scalar_kernel|noise_bias_act_nhwc_kernel|noise_bias_act_kernel|"
                     r"rowwise_nhwc_kernel|nhwc_finish_kernel|to_rgb_nhwc_fwd_kernel|to_rgb_nhwc_bwd_kernel)(<[^>]*>)?")


@pytest.mark.gpu
def test_routing_matches_the_restatement():
    """Every distinct route of the cases above launches the kernels (names, template arguments, order) the restatement
    names."""
    run_fresh("test_rowwise_family_gpu", "check_routing")


def check_routing():
    """The body of test_routing_matches_the_restatement (raises AssertionError on a mismatch)."""
    sms = library().sm_count()
    seen, done = [], set()

    def expect(label, names, fn, labels=()):
        # one launch per distinct kernel sequence and reason for it (vector / scalar and why)
        key = (tuple(names), frozenset(lab for lab in labels if "vector" in lab or "scalar" in lab))
        if key in done:
            return
        done.add(key)
        got = launched(fn, KERNELS)
        seen.append("%-56s -> %s" % (label, got))
        assert got == names, "%s: launched %s, the restatement predicts %s" % (label, got, names)

    for i, case in enumerate(NCHW_CASES):
        r = nchw_rowwise_route(*case)
        expect("nchw %s %s" % (SHORT[case[0]], case[1:]), r["names"], lambda: nchw_rowwise(case, seeded(i)), r["labels"])
    for case in FLAT_CASES:
        dt, shape, layout, act, grad, b, xo, ro = case
        r = flat_route(dt, math.prod(shape), flat_step(shape, layout), b, grad == 1, xo, ro)
        expect("flat %s %s %s off %d/%d" % (SHORT[dt], shape, layout, xo, ro), r["names"], lambda: flat_run(case, seeded(1)),
               r["labels"])
    for dt, shape, nz, nw, b, rs, xo, no in NOISE_CASES:
        r = noise_route(dt, shape[0], shape[1], shape[2] * shape[3], nz, xo, no, sms)
        expect("noise %s %s off %d/%d" % (SHORT[dt], shape, xo, no), r["names"],
               lambda: noise_run(dt, shape, nz, nw, b, rs, xo, no, seeded(2)), r["labels"])
    n, c, hw = big_scalar_shape(sms)
    r = noise_route(F32, n, c, hw, True, sms=sms)
    expect("noise grid-stride", r["names"], lambda: noise_run(F32, (n, c, hw, 1), True, True, True, True, 0, 0, seeded(3)),
           r["labels"])
    from gangealing_b200.op import nhwc
    for dt, n, c, hw in NHWC_CASES:
        r = nhwc_rowwise_route(dt, n, c, hw, sms)
        shape = nhwc_shape(n, c, hw)
        x = cl(torch.randn(shape, device=DEV).to(dt))
        s = torch.ones(n, c, device=DEV)
        lab = "nhwc %s C=%d HW=%d N=%d" % (SHORT[dt], c, hw, n)
        expect(lab + " channel_scale", r["names"][0], lambda: nhwc.channel_scale(x, s, x))
        expect(lab + " bias_act_backward", r["names"][1], lambda: nhwc.bias_act_backward(x, x, 0.2, 1.0, True))
        expect(lab + " noise_bias_act", [r["noise_name"]], lambda: nhwc.noise_bias_act(x, None, None, None, None, 0.2, 1.0))
    for case in TO_RGB_CASES:
        n, c, hw, b, sk, want_gx, want_gwm = case
        names = ["to_rgb_nhwc_fwd_kernel", "to_rgb_nhwc_bwd_kernel"] + (["nhwc_finish_kernel"] if want_gwm else [])
        expect("to-RGB %s" % (case,), names, lambda: to_rgb_run(case, seeded(4)))
    for line in seen:
        print("[route] " + line)
