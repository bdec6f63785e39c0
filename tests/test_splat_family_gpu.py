"""splat2d's scatter and normalise kernels (csrc/splat.cu) against float64, over their launch plans.

  splat_direct_kernel<G, LOOKUP>   one thread per point, 64-thread CTAs; one 16-byte vector reduction per footprint pixel
                                   and group of 4 accumulator slots: G = 1 for C <= 3, G = 2 for C = 4..7; LOOKUP reads the
                                   point from the sampling grid first (gg_splat2d_lookup_forward, C <= 3 only)
  splat_scatter_generic_kernel     C >= 8, or H * W * slots >= 2^31: scalar atomics, grid-stride over at most 8 CTAs / SM
  splat_normalize_kernel           out = (input + S) / (alpha' + 1e-8), alpha' = max(alpha, 1) when soft, grid-stride
                                   over at most 8 CTAs / SM

The accumulators are interleaved per pixel: slot 0 sums the Gaussian weights a, slots 1..C sum a * value, padded to a
multiple of 4 slots.  This file restates splat_impl's routing and splat_grid in Python (planned for 132 SMs), labels
every case with the routes it takes and asserts on a machine without a GPU that the cases reach every label.  The GPU
half calls the entries through the C ABI with NaN-filled outputs and a NaN guard past the workspace, and checks:

  the touched pixels      exactly the windows of the accepted points (fp32 window bounds restated bitwise)
  the accumulators        |y - ref| <= c * 2^-24 * sum|terms| + extra, c = (the pixel fan-in: the atomics' order is
                          arbitrary) + the term's roundings; `extra` is the explicit float64 allowance for the fp32
                          exponent argument z = norm * (dx^2 + dy^2): a * |z| * k_z * 2^-24 per term (k_z = 5: the two
                          rounded differences count twice through their squares, the squares, their sum, the product)
  the output              first-order propagation of the sums' bounds through (input + S) / (alpha' + 1e-8) plus the
                          sum's, the denominator's and the division's roundings
  the looked-up points    against float64 grid_sample + unnormalise, and the splat against the float64 reference
                          evaluated on the points the kernel wrote

The float64 reference is a vectorised index_add_ over every (point, window pixel) pair on the GPU.
"""

import pytest
import torch

from fp64_contract import DEV, H100_SMS, Worst, assert_routes_reached, ceil_div, f32, library, nan_at
from oracle.rounding import U32

INT_MAX = 0x7FFFFFFF
GUARD = 1024
K_Z = 5                     # roundings of the exponent argument, relative to |z|
C_EXP = 4                   # expf's 2 ulp, in units of 2^-24 * a
TINY = 2.0 ** -126          # per term and slot: expf and the float reductions (red / atom .add.f32) flush results
                            # below the normal range to zero, and the reductions their inputs too (2 TINY)


# ======================================================================================== planner restatement (no GPU)
def slots_of(c):
    return ceil_div(c + 1, 4) * 4


def splat_grid(total, sms):
    return min(max(ceil_div(total, 256), 1), 8 * sms)


def route(n, p, c, h, w, lookup=False):
    """splat_impl: the scatter kernel a call launches ('none' without points), or the refusal."""
    slots = slots_of(c)
    if lookup and (slots != 4 or h * w * slots >= INT_MAX):
        return "refused"
    if n * c * h * w == 0:
        return "early return"
    if n * p == 0:
        return "none"
    if slots <= 8 and h * w * slots < INT_MAX:
        return "direct<1, true>" if lookup else "direct<1>" if slots == 4 else "direct<2>"
    return "generic"


def trips(total, sms=H100_SMS):
    return ceil_div(total, splat_grid(total, sms) * 256)


# ------------------------------------------------------------------------------------------------------------- cases
# (name, N, P, C, H, W, sigmas, soft, points)  points: "uniform" (some beyond the border), "edges" (the special x
# values), "dup" (one point repeated), "corners" (windows clamped at every border), "lookup"
CASES = [
    ("c1", 2, 300, 1, 48, 48, (0.3, 0.9), True, "uniform"),
    ("c2", 1, 500, 2, 32, 40, (0.7,), False, "uniform"),
    ("c3", 2, 500, 3, 32, 40, (0.7, 1.6), False, "edges"),
    ("c3-large", 1, 2000, 3, 64, 64, (1.3,), False, "uniform"),
    ("c3-tiny", 3, 1, 3, 8, 8, (0.5, 0.6, 0.7), False, "uniform"),
    ("c4", 1, 100, 4, 16, 16, (1.0,), False, "corners"),
    ("c5", 2, 200, 5, 20, 24, (0.8, 0.4), True, "uniform"),
    ("c7", 1, 300, 7, 24, 20, (1.1,), False, "edges"),
    ("c8", 1, 300, 8, 24, 20, (0.6,), False, "corners"),
    ("c9", 1, 64, 9, 16, 16, (0.6,), True, "uniform"),
    ("c16", 2, 200, 16, 12, 14, (0.9, 0.5), False, "edges"),
    ("c8-trips", 1, 300000, 8, 64, 64, (0.5,), False, "uniform"),                # N*P > 8 * 132 * 256
    ("c3-normalise-trips", 2, 400, 3, 256, 256, (1.0, 0.4), True, "uniform"),   # N*C*H*W > 8 * 132 * 256
    ("wide", 2, 20, 3, 9, 7, (6.0, 3.0), False, "uniform"),                     # footprint wider than the image
    ("underflow", 1, 200, 3, 40, 40, (0.12,), False, "uniform"),               # expf underflows at window corners
    ("p0", 2, 0, 3, 16, 16, (1.0, 1.0), True, "uniform"),
    ("c0", 2, 50, 0, 16, 16, (1.0, 1.0), False, "uniform"),

]


def _disc(res=128, rad=40):
    """A rasterised disc of res^2 points at half-pixel spacing (dense mask splats, up-sampled 2x)."""
    ys, xs = torch.meshgrid(torch.arange(float(res)), torch.arange(float(res)), indexing="ij")
    inside = ((ys - res / 2) ** 2 + (xs - res / 2) ** 2) < rad ** 2
    return torch.stack([xs[inside] / 2 + 0.13, ys[inside] / 2 + 0.21], dim=1)[None]


DISC_POINTS = _disc()
# contention: thousands of atomics on the same pixels
CONTENTION_CASES = [
    ("dup", 1, 4096, 3, 64, 64, (1.0,), False, "dup"),
    ("disc", 1, DISC_POINTS.shape[1], 3, 64, 64, (0.6,), False, "disc"),
]
LOOKUP_CASES = [
    ("lookup-c3", 2, 5000, 3, 64, 64, (0.3, 1.3), False, "lookup"),
    ("lookup-c1", 1, 3000, 1, 48, 40, (0.8,), True, "lookup"),
]
GRID_HW = (32, 24)


def points_for(case):
    """The case's (N, P, 2) points, values, input and sigma, on the CPU (deterministic)."""
    name, n, p, c, h, w, sig, soft, kind = case
    g = torch.Generator().manual_seed(sum(map(ord, name)) + p)
    if kind == "lookup":
        q = torch.randint(-5000, 5001, (n, p, 2), generator=g).float() / 4096      # dyadic, some beyond the border
        pts = q
    elif kind == "dup":
        pts = torch.tensor([10.3, 20.7]).repeat(n, p, 1)
    elif kind == "disc":
        pts = DISC_POINTS.clone()
    else:
        pts = torch.rand(n, p, 2, generator=g) * torch.tensor([w * 1.2, h * 1.2]) - torch.tensor([w * 0.1, h * 0.1])
        if kind == "corners" and p >= 8:
            pts[:, :8] = torch.tensor([[0.2, 0.3], [w - 0.4, 0.1], [0.0, h - 0.2], [w - 0.01, h - 0.01],
                                       [w / 2, 0.0], [w / 2, h - 0.5], [0.1, h / 2], [w - 0.6, h / 2]])
        if kind == "edges" and p >= 8:
            wf = torch.tensor(float(w))
            pts[:, :8, 1] = h / 2
            pts[:, 0, 0] = wf                                                  # x = W: rejected
            pts[:, 1, 0] = torch.nextafter(wf, torch.tensor(0.0))              # accepted
            pts[:, 2, 0] = -0.0                                                # accepted
            pts[:, 3, 0] = -1e-30                                              # rejected
            pts[:, 4, 0] = float("nan")                                        # rejected
            pts[:, 5, 1] = float(h)                                            # y = H: rejected
            pts[:, 6, 1] = torch.nextafter(torch.tensor(float(h)), torch.tensor(0.0))
    vals = torch.randn(n, p, c, generator=g)
    inp = torch.randn(n, c, h, w, generator=g)
    return pts.contiguous(), vals, inp, torch.tensor(sig, dtype=torch.float32)


def _accepted(x, h, w):
    y = x[..., 1]
    x = x[..., 0]
    return (x >= 0) & (x < float(w)) & (y >= 0) & (y < float(h))


def case_labels(case, pts=None):
    name, n, p, c, h, w, sig, soft, kind = case
    r = route(n, p, c, h, w, lookup=kind == "lookup")
    labels = set()
    if r in ("direct<1>", "direct<2>", "generic"):
        labels.add("%s C=%d" % (r, c))
    if r == "direct<1, true>":
        labels.add("lookup route with points_out")
    if r == "early return":
        labels.add("C = 0: early return")
    if r == "none":
        labels.add("P = 0: normaliser only")
    if r == "generic" and trips(n * p) > 1:
        labels.add("generic scatter: second grid-stride trip")
    if n * c * h * w and trips(n * c * h * w) > 1:
        labels.add("normaliser: second grid-stride trip")
    if n * c * h * w:
        labels.add("soft on" if soft else "soft off")
    if len(set(sig)) > 1:
        labels.add("per-sample sigma differs across n")
    if any(4 * s > max(h, w) for s in sig):
        labels.add("footprint wider than the image")
    if kind == "dup" and p >= 1000:
        labels.add("fan-in of thousands of duplicate points")
    if kind == "disc":
        labels.add("dense rasterised disc (every pixel of it under many footprints)")
    if any(s < 0.15 for s in sig):
        labels.add("expf underflows at a window corner")
    if pts is None:
        pts = points_for(case)[0]
    if kind != "lookup" and p:
        x, y = pts[..., 0], pts[..., 1]
        ok = _accepted(pts, h, w)
        ln = torch.tensor(sig).view(-1, 1) * 2
        if bool((ok & (x - ln < 0)).any()):
            labels.add("window clamped at the left border")
        if bool((ok & (torch.ceil(x + ln) > w - 1)).any()):
            labels.add("window clamped at the right border")
        if bool((ok & (y - ln < 0)).any()):
            labels.add("window clamped at the top border")
        if bool((ok & (torch.ceil(y + ln) > h - 1)).any()):
            labels.add("window clamped at the bottom border")
        if kind == "edges":
            labels |= {"x = W rejected", "x = nextafter(W, 0) accepted", "x = -0.0 accepted", "tiny negative x rejected",
                       "NaN rejected"}
            assert not bool(ok[:, 0].any() or ok[:, 3].any() or ok[:, 4].any() or ok[:, 5].any())
            assert bool(ok[:, 1].all() and ok[:, 2].all() and ok[:, 6].all())
    return labels


REQUIRED = (["direct<1> C=%d" % c for c in (1, 2, 3)] + ["direct<2> C=%d" % c for c in (4, 5, 7)]
            + ["generic C=%d" % c for c in (8, 9, 16)]
            + ["generic scatter: second grid-stride trip", "normaliser: second grid-stride trip", "soft on", "soft off",
               "P = 0: normaliser only", "C = 0: early return", "lookup route with points_out",
               "window clamped at the left border", "window clamped at the right border",
               "window clamped at the top border", "window clamped at the bottom border",
               "footprint wider than the image", "per-sample sigma differs across n", "x = W rejected",
               "x = nextafter(W, 0) accepted", "x = -0.0 accepted", "tiny negative x rejected", "NaN rejected",
               "fan-in of thousands of duplicate points", "expf underflows at a window corner",
               "dense rasterised disc (every pixel of it under many footprints)"])
UNREACHED = ["generic because H * W * slots >= 2^31 (about 9 GB of accumulators at one sample: not run)"]


def test_cases_reach_every_route():
    reached = set()
    for case in CASES + CONTENTION_CASES + LOOKUP_CASES:
        reached |= case_labels(case)
    assert_routes_reached(REQUIRED, reached, UNREACHED)


def test_routing_restatement():
    """The direct / generic split, the lookup guard and the early return, at the boundaries."""
    assert route(1, 10, 3, 64, 64) == "direct<1>" and route(1, 10, 7, 64, 64) == "direct<2>"
    assert route(1, 10, 8, 64, 64) == "generic"
    assert route(1, 10, 3, 16384, 32767) == "direct<1>"            # H * W * 4 = 2^31 - 2^16 * 4 < 2^31 - 1
    assert route(1, 10, 3, 16384, 32768) == "generic"               # H * W * 4 = 2^31
    assert route(1, 10, 3, 16384, 32768, lookup=True) == "refused"
    assert route(1, 10, 4, 8, 8, lookup=True) == "refused"
    assert route(0, 10, 3, 8, 8) == route(1, 10, 0, 8, 8) == "early return"
    assert splat_grid(1, H100_SMS) == 1 and splat_grid(1 << 40, H100_SMS) == 8 * H100_SMS
    lib = library().load()
    for c in (0, 1, 3, 4, 7, 8, 9, 16):
        assert lib.gg_splat2d_workspace(2, c, 5, 7) == 2 * 5 * 7 * slots_of(c) * 4


# ======================================================================================================== GPU checks
WORST = Worst("c per path", "%-48s %.2f")
_report_worst = WORST.fixture()


def reference(pts, vals, inp, sig, soft):
    """float64 accumulators (N, H, W, C + 1), their sums of |terms|, the z allowance, the fan-in, the touched set, and the
    output with its magnitude, from the fp32 window bounds of splat_gpu_impl / splat.cu restated bitwise."""
    n, p, _ = pts.shape
    c, h, w = inp.shape[1], inp.shape[2], inp.shape[3]
    acc = torch.zeros(n * h * w, c + 1, dtype=torch.float64, device=DEV)
    acc_abs = torch.zeros_like(acc)
    zx = torch.zeros(n * h * w, c + 1, dtype=torch.float64, device=DEV)
    fan = torch.zeros(n * h * w, dtype=torch.float64, device=DEV)
    if p:
        x, y = pts[..., 0], pts[..., 1]
        ok = _accepted(pts, h, w)
        sd = sig.view(n, 1).expand(n, p)
        ln = 2 * sd
        norm = -1.0 / ((2 * sd) * sd)                                       # fp32, as the kernel rounds it
        t = torch.clamp(torch.floor(y - ln), min=0)
        b = torch.clamp(torch.ceil(y + ln), max=float(h - 1))
        l = torch.clamp(torch.floor(x - ln), min=0)
        r = torch.clamp(torch.ceil(x + ln), max=float(w - 1))
        idx = torch.nonzero(ok)
        ni, pi = idx[:, 0], idx[:, 1]
        t, b, l, r = (v[ni, pi].long() for v in (t, b, l, r))
        span_y, span_x = int((b - t).max()) + 1 if len(ni) else 0, int((r - l).max()) + 1 if len(ni) else 0
        xs, ys, nrm = x[ni, pi].double(), y[ni, pi].double(), norm[ni, pi].double()
        v = torch.cat([torch.ones(len(ni), 1, device=DEV), vals[ni, pi]], 1).double()
        for dy in range(span_y):
            py = t + dy
            for dx0 in range(0, span_x, 64):
                dx = torch.arange(dx0, min(span_x, dx0 + 64), device=DEV)
                px = l[:, None] + dx[None]
                live = (py[:, None] <= b[:, None]) & (px <= r[:, None])
                k, j = torch.nonzero(live, as_tuple=True)
                pxk, pyk = px[k, j], py[k]
                z = nrm[k] * ((pxk.double() - xs[k]) ** 2 + (pyk.double() - ys[k]) ** 2)
                a = torch.exp(z)
                dest = (ni[k] * h + pyk) * w + pxk
                term = a[:, None] * v[k]
                acc.index_add_(0, dest, term)
                acc_abs.index_add_(0, dest, term.abs())
                zx.index_add_(0, dest, term.abs() * (z.abs() * K_Z * U32)[:, None] + 2 * TINY)
                fan.index_add_(0, dest, torch.ones_like(a))
    shape = (n, h, w, c + 1)
    return acc.view(shape), acc_abs.view(shape), zx.view(shape), fan.view(n, h, w)


def output_reference(inp, acc, acc_abs, zx, c_acc, soft):
    """out, its magnitude and the explicit allowance: (input + S) / den with den = alpha' + 1e-8 (fp32 constant)."""
    i64 = inp.double()
    s = acc[..., 1:].permute(0, 3, 1, 2)
    s_abs = acc_abs[..., 1:].permute(0, 3, 1, 2)
    x_s = zx[..., 1:].permute(0, 3, 1, 2)
    alpha = acc[..., 0].unsqueeze(1)
    x_a = zx[..., 0].unsqueeze(1)
    den = (torch.clamp(alpha, min=1.0) if soft else alpha) + f32(1e-8)
    out = (i64 + s) / den
    num_abs = i64.abs() + s_abs
    # first order: dS / den + num * dalpha / den^2, with dS <= c u S_abs + x_s, dalpha <= c u alpha + x_a; the sum, the
    # denominator and the division add one rounding each (c + 3 in units of u * mag)
    mag = num_abs / den * (1 + alpha / den)
    extra = x_s / den + num_abs * x_a / den ** 2
    return out, mag, extra


def run_splat(pts, vals, inp, sig, soft, lookup=None):
    lib = library()
    n, c, h, w = inp.shape
    p = pts.shape[1]
    out = nan_at((n, c, h, w), torch.float32)
    nbytes = lib.load().gg_splat2d_workspace(n, c, h, w)
    ws = torch.full((nbytes // 4 + GUARD,), float("nan"), device=DEV)
    if lookup is None:
        rc = lib.load().gg_splat2d_forward(out.data_ptr(), ws.data_ptr(), inp.data_ptr(), pts.data_ptr(), vals.data_ptr(),
                                           sig.data_ptr(), n, p, c, h, w, int(soft), lib.stream())
        lib.check(rc, "gg_splat2d_forward")
        pts_out = None
    else:
        grid, res, out_res = lookup
        pts_out = nan_at((n, p, 2), torch.float32)
        rc = lib.load().gg_splat2d_lookup_forward(out.data_ptr(), pts_out.data_ptr(), ws.data_ptr(), inp.data_ptr(),
                                                  grid.data_ptr(), pts.data_ptr(), vals.data_ptr(), sig.data_ptr(), n, p,
                                                  c, h, w, grid.shape[1], grid.shape[2], (res - 1) / res,
                                                  float(out_res - 1), int(soft), lib.stream())
        lib.check(rc, "gg_splat2d_lookup_forward")
    torch.cuda.synchronize()
    assert bool(ws[nbytes // 4:].isnan().all()), "the launches wrote past the workspace"
    acc = ws[:nbytes // 4].view(n, h, w, slots_of(c)) if nbytes else None
    return out, acc, pts_out


def check_splat(case, pts, vals, inp, sig, soft, out, acc):
    name = case[0]
    n, c, h, w = inp.shape
    path = route(n, pts.shape[1], c, h, w, lookup=case[-1] == "lookup")
    ref, ref_abs, zx, fan = reference(pts, vals, inp, sig, soft)
    touched = fan > 0
    got = acc[..., :c + 1].double()
    # the touched set: untouched pixels hold exact zeros in every slot; touched ones a positive weight sum wherever the
    # float64 sum stays clear of expf's underflow allowance
    assert bool((acc[~touched] == 0).all()), "%s: a pixel outside every window was written" % name
    clear = ref[..., 0] > 2 * zx[..., 0] + 1e-30
    assert bool((acc[..., 0][touched & clear] > 0).all()), "%s: a touched pixel holds no weight" % name
    assert bool((acc[..., c + 1:] == 0).all()), "%s: a padding slot was written" % name
    fan_max = int(fan.max()) if fan.numel() else 0
    c_alpha = fan_max + C_EXP                                  # the additions (the first onto 0 is exact) + expf
    c_val = fan_max + C_EXP + 1                                # + the product a * value
    WORST.check_sum(got[..., 0], ref[..., 0], ref_abs[..., 0], c_alpha, "alpha, %s" % path, name, zx[..., 0])
    if c:
        WORST.check_sum(got[..., 1:], ref[..., 1:], ref_abs[..., 1:], c_val, "sums, %s" % path, name, zx[..., 1:])
    o64, mag, extra = output_reference(inp, ref, ref_abs, zx, c_val, soft)
    WORST.check_sum(out, o64, mag, c_val + 3, "normalised, %s" % path, "%s (fan-in %d)" % (name, fan_max), extra)


def _to_dev(case):
    pts, vals, inp, sig = points_for(case)
    return pts.to(DEV), vals.to(DEV), inp.to(DEV), sig.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda cs: cs[0])
def test_splat2d(case):
    name, n, p, c, h, w, sig, soft, kind = case
    pts, vals, inp, sg = _to_dev(case)
    out, acc, _ = run_splat(pts, vals, inp, sg, soft)
    if n * c * h * w == 0:
        assert out.numel() == 0
        assert acc is None or bool(acc.isnan().all()), "an empty output still touched the workspace"
        return
    check_splat(case, pts, vals, inp, sg, soft, out, acc)


@pytest.mark.gpu
def test_splat2d_duplicate_points_and_dense_mask():
    """Contention: 4096 copies of one point (fan-in 4096 on each pixel of its window), and a dense rasterised disc at
    half-pixel spacing, every pixel under dozens of footprints; each element within its fan-in's bound."""
    for case in CONTENTION_CASES:
        pts, vals, inp, sg = _to_dev(case)
        out, acc, _ = run_splat(pts, vals, inp, sg, case[7])
        check_splat(case, pts, vals, inp, sg, case[7], out, acc)


def lookup64(grid, q, res, out_res):
    """float64 F.grid_sample(grid as an image, q, 'border', align_corners=False) + unnormalise, with k and m as the fp32
    values the entry receives; and the same on |grid| for the magnitude."""
    import torch.nn.functional as F
    k, m = f32((res - 1) / res), f32(out_res - 1)
    res_ = []
    for gv in (grid.double(), grid.double().abs()):
        s = F.grid_sample(gv.permute(0, 3, 1, 2), q.double().unsqueeze(2), padding_mode="border", align_corners=False)
        res_.append(s.squeeze(3).permute(0, 2, 1))
    ox, oa = res_
    return ((ox / k) / 2 + 0.5) * m, (oa / abs(k) / 2 + 0.5) * abs(m)


@pytest.mark.gpu
@pytest.mark.parametrize("case", LOOKUP_CASES, ids=lambda cs: cs[0])
def test_splat2d_lookup(case):
    """The looked-up points: dyadic queries make the grid coordinate ((q + 1) gw - 1) / 2 and the bilinear fractions
    exact, so a point carries the 4-term fma chain with its rounded weight products (5), then / k, + 0.5 and * m (3):
    c = 8 against float64 grid_sample + unnormalise.  Then the splat against float64 on the points the kernel wrote."""
    name, n, p, c, h, w, sig, soft, kind = case
    q, vals, inp, sg = _to_dev(case)
    gh, gw = GRID_HW
    gen = torch.Generator().manual_seed(12)
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, gh), torch.linspace(-1, 1, gw), indexing="ij")
    grid = (torch.stack([xs, ys], -1)[None].repeat(n, 1, 1, 1) * 0.9 + 0.03 * torch.randn(n, gh, gw, 2, generator=gen)).to(DEV)
    res = out_res = w
    out, acc, pts_out = run_splat(q, vals, inp, sg, soft, (grid, res, out_res))
    ref_p, mag_p = lookup64(grid, q, res, out_res)
    WORST.check_sum(pts_out, ref_p, mag_p, 8, "looked-up points", name)
    check_splat(case, pts_out, vals, inp, sg, soft, out, acc)


@pytest.mark.gpu
def test_lookup_is_refused_where_the_direct_kernel_cannot_serve_it():
    """Only the direct kernel performs the lookup, and it needs H * W * 4 slots < 2^31.  At H * W = 2^29 (16384 x 32768,
    one sample, one channel) the entry returns GG_ERR_UNSUPPORTED before any device work, on real buffers: points_out
    stays NaN."""
    free, _ = torch.cuda.mem_get_info()
    if free < 16 * 2 ** 30:
        pytest.skip("needs 16 GB of free device memory (2 GB input, 2 GB output, 8.6 GB workspace): %.1f GB free"
                    % (free / 2 ** 30))
    lib = library()
    n, c, h, w, p = 1, 1, 16384, 32768, 4
    assert route(n, p, c, h, w, lookup=True) == "refused"
    inp = torch.empty(n, c, h, w, device=DEV)
    out = torch.empty(n, c, h, w, device=DEV)
    ws = torch.empty(lib.load().gg_splat2d_workspace(n, c, h, w) // 4, device=DEV)
    grid = torch.zeros(n, 8, 8, 2, device=DEV)
    q = torch.zeros(n, p, 2, device=DEV)
    vals = torch.ones(n, p, c, device=DEV)
    sig = torch.ones(n, device=DEV)
    pts_out = nan_at((n, p, 2), torch.float32)
    try:
        rc = lib.load().gg_splat2d_lookup_forward(out.data_ptr(), pts_out.data_ptr(), ws.data_ptr(), inp.data_ptr(),
                                                  grid.data_ptr(), q.data_ptr(), vals.data_ptr(), sig.data_ptr(), n, p, c,
                                                  h, w, 8, 8, f32((w - 1) / w), float(w - 1), 0, lib.stream())
        torch.cuda.synchronize()
        assert rc == -2, "rc %d: %s" % (rc, lib.load().gg_last_error())
        assert bool(pts_out.isnan().all()), "points_out was written"
    finally:
        del inp, out, ws
        torch.cuda.empty_cache()
