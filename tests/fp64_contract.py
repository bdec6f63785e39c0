"""What the float64 contract tests of the kernel families share (not collected: the name does not match test_*.py).

Each family module restates in Python how the library plans its launches, labels its cases with the routes they take, and
checks every output against float64 with a bound derived from the kernel's operation order (oracle/rounding.py).  This
module holds the pieces they have in common:

  the dtype tables and small input helpers (randn, at_offset, nan_at, cl, ...)
  the checks: the registry of the worst observed k / c that a module prints when it finishes (Worst), the unregistered
    checks that print each ratio (check_once, check_sum), the coverage assertion
  the kernel-name probe (launched) and the fresh interpreter a module's launch check runs in (run_fresh)
  the float64 references and bounds more than one module checks with: fir64 and blur_k (blurs), distance64 and
    distance_forward_c (the perceptual feature distance)
  the one restatement of each C launch planner that more than one module plans with:

  blur_plan          csrc/nhwc.cu blur_plan
  rowwise_geometry   csrc/nhwc.cu rowwise_chunk and csrc/styled.cu bwd_chunk (rowwise_c, finish_depth: their sums)
  grid_for           csrc/flow_compose.cuh grid_for (grid_stride_batch: a batch that takes two of its trips)
"""
import math
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.rounding import assert_fp32_sum, assert_rounded_once

DEV = "cuda"
SQRT2 = 2 ** 0.5
H100_SMS = 132                    # SM count the CPU coverage checks plan with (H100 SXM)
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
VEC = {F32: 4, F16: 8, BF16: 8}   # elements per 16-byte access
TNAME = {F32: "float", F16: "__half", BF16: "__nv_bfloat16"}
CODE = {F32: 0, F16: 1, BF16: 2}  # gangealing_b200._lib.GG_F32 / GG_F16 / GG_BF16
SHORT = {F32: "fp32", F16: "fp16", BF16: "bf16"}


# ============================================================================================================ helpers
def ceil_div(a, b):
    return -(-a // b)


def f32(v):
    """A Python float as the fp32 value a kernel argument holds."""
    return float(np.float32(v))


def seeded(seed):
    """A CUDA generator with the given seed."""
    return torch.Generator(device=DEV).manual_seed(seed)


def library():
    from gangealing_b200 import _lib as lib
    return lib


def at_offset(t, off):
    """A copy of `t` whose data starts `off` elements past a 16-byte boundary (torch allocations are 512-byte aligned)."""
    buf = torch.empty(off + t.numel(), dtype=t.dtype, device=t.device)
    v = buf[off:].view(t.shape)
    v.copy_(t)
    return v


def cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def randn(shape, g, dtype=F32, off=0):
    t = torch.randn(shape, generator=g, device=DEV).to(dtype)
    return at_offset(t, off) if off else t


def saved_output(shape, g, dtype, off=0):
    """A forward output to gate on: mixed signs and ~5 % exact zeros (zero takes the negative slope)."""
    t = torch.randn(shape, generator=g, device=DEV)
    t = torch.where(torch.rand(shape, generator=g, device=DEV) < 0.05, torch.zeros_like(t), t).to(dtype)
    return at_offset(t, off) if off else t


def nan_at(shape, dtype, off=0):
    """An output buffer `off` elements past a 16-byte boundary, filled with NaN: an element no launch writes stays NaN."""
    buf = torch.full((off + math.prod(shape),), float("nan"), dtype=dtype, device=DEV)
    return buf[off:].view(shape)


def lrelu64(t, slope, gain):
    """Leaky-ReLU times the gain, with the slope and gain as given (pass them through f32 for a launch's fp32 values)."""
    return torch.where(t > 0, t, t * slope) * gain


def slope_gain(slope, gain):
    """Leaky-ReLU and gain scale |pre-activation| by at most this."""
    return abs(gain) * max(1.0, abs(slope))


# ======================================================================================================== the checks
def check_once(y, ref, a, k, what, extra=None):
    ulps, k_obs = assert_rounded_once(y, ref, a, k, what, extra)
    print("[contract] %s: %.4f ulp, k_obs=%.2f (k=%g)" % (what, ulps, k_obs, k))


def check_sum(y, ref, a, c, what, extra=None):
    r = assert_fp32_sum(y, ref, a, c, what, extra)
    print("[contract] %s: c_obs=%.2f (c=%d)" % (what, r, c))


class Worst:
    """The worst observed k (stored values) / c (sums) per path of one test module.  The module registers the report
    that prints them when its tests finish with `_report_worst = WORST.fixture()` (a fixture has to live in the module).

    header: what the report's title line names after "worst observed"; row: the format of one (path, worst) line;
    kind_suffix: whether a path's key carries " (k)" / " (c)" for the kind of check."""

    def __init__(self, header, row="%-64s %.2f", kind_suffix=True):
        self.header, self.row, self.kind_suffix = header, row, kind_suffix
        self.obs = defaultdict(float)

    def note(self, key, obs):
        self.obs[key] = max(self.obs[key], obs)

    def fixture(self):
        @pytest.fixture(scope="module", autouse=True)
        def report():
            yield
            if self.obs:
                print("\n[contract] worst observed %s:" % self.header)
                for key in sorted(self.obs):
                    print("[contract]   " + self.row % (key, self.obs[key]))
        return report

    def check_stored(self, y, ref, a, k, path, what):
        """A stored value: fp32 within k * 2^-24 * A; fp16 / bf16 within 1/2 ulp + k * 2^-24 * A."""
        if y.dtype == F32:
            obs = assert_fp32_sum(y, ref, a, k, "%s: %s" % (path, what))
        else:
            _, obs = assert_rounded_once(y, ref, a, k, "%s: %s" % (path, what))
        self.note(path + " (k)", obs)
        print("[contract] %s: %s: k_obs=%.2f (k=%d)" % (path, what, obs, k))

    def check_sum(self, y, ref, a, c, path, what, extra=None):
        """An fp32 sum within c * 2^-24 * sum|terms| (+ `extra`, an explicit float64 allowance)."""
        obs = assert_fp32_sum(y, ref, a, c, "%s: %s" % (path, what), extra)
        self.note(path + " (c)" if self.kind_suffix else path, obs)
        print("[contract] %s: %s: c_obs=%.2f (c=%d)" % (path, what, obs, c))


def launched(fn, kernels, sessions=3):
    """Names matching the compiled regex `kernels` of the kernels `fn` launches, in launch order, from torch.profiler's
    CUDA activity.  torch.profiler at times records a session's runtime calls without any device activity at all; such a
    session says nothing about the kernels, so it is repeated, up to `sessions` in all (`fn` launches the same kernels
    each time it runs).  A session with device activity is never repeated: its names are the answer."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(sessions):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        evs = prof.events()
        if any(e.device_type == torch.autograd.DeviceType.CUDA for e in evs):
            break
    else:
        raise RuntimeError("torch.profiler recorded no device activity in %d sessions (only %d runtime calls in the last): "
                           "the kernel names are unknown" % (sessions, len(evs)))
    names = [(e.time_range.start, m.group(0)) for e in evs for m in [kernels.search(e.name)] if m]
    return [nm for _, nm in sorted(names, key=lambda t: t[0])]


def run_fresh(module, function, timeout=900):
    """Run `function` of the test module `module` in a fresh interpreter, print its output and fail if it fails.  The
    launch checks that read kernel names run there: in a process that has already run other GPU tests, torch.profiler
    can record the runtime calls (cudaLaunchKernel) without any kernel activity, so the names could not be read."""
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([here, root] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    flags = ["-s"] if sys.flags.no_user_site else []
    proc = subprocess.run([sys.executable] + flags + ["-c", "import %s as t; t.%s()" % (module, function)],
                          cwd=root, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    print(proc.stdout)
    assert proc.returncode == 0, "%s.%s failed:\n%s" % (module, function, proc.stdout[-6000:])


def assert_routes_reached(required, reached, unreached=(), noun="routes"):
    """Print which of the `required` route labels the cases reach ([coverage] lines, with `pytest -s`) and those known
    to stay unreached, then assert that none is missing."""
    missing = [lab for lab in required if lab not in reached]
    print("[coverage] %d of %d %s reached" % (len(required) - len(missing), len(required), noun))
    for lab in required:
        print("[coverage]   %s %s" % ("ok     " if lab in reached else "MISSING", lab))
    for lab in unreached:
        print("[coverage]   unreached %s" % lab)
    assert not missing, "%s no case reaches: %s" % (noun, missing)


# ============================================================================================ float64 references, bounds
def fir64(x, k, pad):
    """upfirdn2d(up = down = 1) in float64: TRUE convolution with `k` (upfirdn2d.py:185-187), pad = (x0, x1, y0, y1)."""
    xp = F.pad(x, list(pad))
    kh, kw = k.shape
    oh, ow = xp.shape[2] - kh + 1, xp.shape[3] - kw + 1
    kf = torch.flip(k.double(), [0, 1]).tolist()
    out = torch.zeros(x.shape[0], x.shape[1], oh, ow, dtype=torch.float64, device=x.device)
    for a in range(kh):
        for b in range(kw):
            out += kf[a][b] * xp[:, :, a:a + oh, b:b + ow]
    return out


def blur_k(kernel):
    """fp32 roundings of one blurred value: separable = 4 horizontal + 4 vertical products/sums + the factorised column
    taps (col / pivot); otherwise 16 fused multiply-adds."""
    from gangealing_b200 import _lib
    return 9 if _lib.filter_is_separable(kernel) else 16


def distance_c_terms(c):
    """(S, e_ia, TRIPS, L): S = roundings of a pixel's sum of squares (a lane's 4*TRIPS fmas + log2(L) butterfly steps),
    e_ia = roundings in 1/(sqrt(S) + eps) (S/2 through the square root, sqrt, + eps, the division)."""
    c4 = c // 4
    L = min(32, c4)
    trips = c4 // L
    s = 4 * trips + int(math.log2(L))
    return s, s / 2 + 3, trips, L


def distance_forward_c(n, c, hw):
    """distance value: 2*(e_ia + 2) for the squared normalised difference, a lane's fmas and its pixels (chunk / groups),
    the warp sum (5), the CTA's 8 warps, *1/HW (2), the finish kernel's K partials."""
    s, e_ia, trips, L = distance_c_terms(c)
    groups = 256 // L
    k = max(1, min(ceil_div(8 * library().sm_count(), n), ceil_div(hw, 2 * groups), 64))
    chunk = ceil_div(hw, k)
    return int(math.ceil(2 * (e_ia + 2) + 4 * trips + ceil_div(chunk, groups) + 5 + 8 + 2 + ceil_div(hw, chunk)))


def distance64(a, b, w, gout, eps=1e-10):
    """float64 feature distance of the stored maps a, b (N, C, H, W), its value on absolute values, and the gradients with
    their absolute-value counterparts.  A pixel whose map is all zero gets gradient 0 (csrc/lpips.cu)."""
    hw = a.shape[2] * a.shape[3]
    wv = w.double().reshape(1, -1, 1, 1) if w is not None else torch.ones(1, a.shape[1], 1, 1, dtype=torch.float64, device=a.device)
    ra = a.square().sum(1, keepdim=True).sqrt()
    rb = b.square().sum(1, keepdim=True).sqrt()
    ia, ib = 1 / (ra + eps), 1 / (rb + eps)
    diff = a * ia - b * ib
    dabs = a.abs() * ia + b.abs() * ib
    d = (wv * diff * diff).sum(1).mean((1, 2))
    da = (wv.abs() * dabs * dabs).sum(1).mean((1, 2))
    gs = 2 * gout.double().reshape(-1, 1, 1, 1) / hw
    t, ta = wv * diff, wv.abs() * dabs
    res = [d, da]
    for f, r, i, sign in ((a, ra, ia, 1.0), (b, rb, ib, -1.0)):
        live = r > 0
        rr = torch.where(live, r, torch.ones_like(r))
        kf = (t * f).sum(1, keepdim=True) * i * i / rr
        ka = (ta * f.abs()).sum(1, keepdim=True) * i * i / rr
        res.append(torch.where(live, sign * gs * (t * i - f * kf), torch.zeros_like(f)))
        res.append(torch.where(live, gs.abs() * (ta * i + f.abs() * ka), torch.zeros_like(f)))
    return res


# ======================================================================================== planner restatements (no GPU)
def blur_plan(dtype, n, c, in_h, in_w, kh, kw, pad, sms):
    """blur_plan of csrc/nhwc.cu (fp32: 64 output columns and 32 channels per CTA; bf16: 32 columns and 64 channels),
    planned for `sms` SMs; pad = (x0, x1, y0, y1)."""
    v = VEC[dtype]
    cb, bx = 8 * v, 64 if v == 4 else 32
    out_h, out_w = in_h + pad[2] + pad[3] - kh + 1, in_w + pad[0] + pad[1] - kw + 1
    xblocks, chunks = ceil_div(out_w, bx), c // cb
    segs = ceil_div(4 * sms, xblocks * chunks * n)
    seg_rows = ceil_div(out_h, segs)
    if seg_rows < 16:
        seg_rows = out_h if out_h < 16 else 16
    seg_rows = ceil_div(seg_rows, 4) * 4
    return dict(out_h=out_h, out_w=out_w, xblocks=xblocks, chunks=chunks, seg_rows=seg_rows,
                segs=ceil_div(out_h, seg_rows))


def finish_depth(k):
    """nhwc_finish_kernel: a lane's serial chain over every 32nd of the K partial rows, (a0 + a1) + (a2 + a3), then the 32
    lane sums in order."""
    return ceil_div(k, 32) + 2 + 32


def rowwise_geometry(n, cv, hw, sms):
    """rowwise_chunk / bwd_chunk of csrc/nhwc.cu, csrc/styled.cu for C/V = cv channel vectors, planned for `sms` SMs:
    (pixel lanes, pixels per CTA, CTAs per sample)."""
    lanes = max(256 // cv, 1)
    k = max(1, min(ceil_div(8 * sms, n), ceil_div(hw, 4 * lanes)))
    chunk = ceil_div(hw, k)
    return lanes, chunk, ceil_div(hw, chunk)


def rowwise_c(n, c, hw, per_term, per_sample, dtype, sms):
    """A thread's serial sum over its pixels, the CTA's pixel lanes in order, then the finish kernel over the CTAs (per
    sample, or over all N*K partial rows)."""
    lanes, chunk, k = rowwise_geometry(n, c // VEC[dtype], hw, sms)
    return per_term + ceil_div(chunk, lanes) + lanes + finish_depth(k if per_sample else n * k)


def grid_for(total, sms, threads=256):
    """flow_compose.cuh grid_for: enough CTAs for `total` items, at most 16 per SM (grid-stride beyond that)."""
    return min(max(ceil_div(total, threads), 1), 16 * sms)


def grid_stride_batch(ho, wo):
    """A batch whose N * Ho * Wo output pixels exceed one trip of the sampler's grid-stride loops (grid_for's largest
    grid of 256 threads on this device), so that every thread makes a second trip."""
    return grid_for(1 << 62, library().sm_count()) * 256 // (ho * wo) + 2
