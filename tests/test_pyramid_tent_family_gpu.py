"""The STN's input path (csrc/warp.cu's mip pyramid, csrc/resample.cu's tent) against float64, over their launch plans.

  mip_build_all_kernel      levels 1..E of one plane per 512-thread CTA, each level from the previous one in shared memory;
                            launched when levels 1..E of a plane fit in 48 KB of static shared memory, or in 200 KB after
                            the opt-in
  mip_down_kernel           otherwise one launch per level (level 1 from the source dtype through the power-of-two reflect
                            padding lp / rp, levels >= 2 from fp32), grid-stride
  mip_down_bwd_kernel       the adjoint, coarse to fine, atomics over the reflected taps (and the lp fold on level 1)
  warp_compose_fwd_kernel   read at one level: the bilinear sample of level L upsampled to full resolution (level_value)
  tent_down_fwd_kernel      reflect-pad s/2 + separable per-channel taps with stride s, one gather per output
  tent_down_bwd_kernel      its adjoint in gather form

Every index here depends on shapes only, never on data, so every bound below is derived, none tuned.  This file

  * restates the host-side planning in Python (make_pyramid: lp / rp, the padded size, the feasibility rules and the level
    offsets; build_t's route; the tent's output size and smallest legal plane), checks the restatement against the
    library's own answers on a machine without a GPU, labels every case with its route and asserts that the cases reach
    every label;
  * checks every output against float64 evaluated on the exact operands the launch reads (oracle/rounding.py):
        fp32 sum       |y - ref| <= c * 2^-24 * sum|terms|              (assert_fp32_sum)
        stored half    |y - ref| <= 1/2 ulp + c * 2^-24 * sum|terms|    (assert_rounded_once with k = c)
    with c derived next to each check, and the adjoints also by the inner-product identity <A x, g> = <x, A^T g>.

Single-level reads use separable grids whose entries are multiples of 2^-12, so every sampling coordinate is exact in
fp32.  The level of detail measures neighbour distances with a (size - 1) / 2 scale: where size - 1 is a power of two
on an axis, the grid step places neighbours exactly 2^L px apart and the level of detail alone yields level L.  For
other sizes no dyadic step can do that, so the same grid keeps the distance just under 2^L and min_level = L pins the
level; either way w = 0 and l0 = l1 = L, asserted through the returned levels.  How the level of detail is chosen, and
the sampler between levels, is checked against float64 by test_warp_family_gpu.py.

Every check prints its worst observed c (`[contract] ...` lines with `pytest -s`), and the module prints the worst per
path when it finishes.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fp64_contract import BF16, DEV, F16, F32, H100_SMS, Worst, assert_routes_reached, grid_for, library, seeded
from oracle.rounding import U32, assert_fp32_sum, assert_rounded_once
from oracle.sampling import create_stack, downsample_2x, grid_sample_bilinear

THREADS = 256
MAX_LEVELS = 8                                  # warp.cu kMaxLevels
STATIC_SMEM, OPTIN_SMEM = 48 * 1024, 200 * 1024
SHORT = {F32: "f32", F16: "f16", BF16: "bf16"}
PAD_MODES = ("zeros", "border", "reflection")


# ======================================================================================== planner restatement (no GPU)
def reflect(j, n):
    """ReflectionPad semantics (no edge repeat), one reflection: warp.cu reflect_idx, resample.cu reflect_index."""
    if j < 0:
        j = -j
    if j >= n:
        j = 2 * (n - 1) - j
    return j


def make_pyramid(hs, ws, planes, extra):
    """warp.cu make_pyramid -> dict(lp, rp, hp, wp, offsets) or None where the library refuses the shape.  The width alone
    decides the reflect padding to a power of two, and both axes take it; offsets[i] is level i's first float (1-based),
    offsets[0] the total."""
    lp = rp = 0
    if ws & (ws - 1):
        target = 1
        while target < ws:
            target <<= 1
        lp = (target - ws) // 2
        rp = target - ws - lp
    hp, wp = hs + lp + rp, ws + lp + rp
    if lp >= hs or rp >= hs or lp >= ws or rp >= ws:
        return None                                          # ReflectionPad2d needs padding < size
    if extra < 0 or extra > MAX_LEVELS:
        return None
    offsets, off = [0] * (extra + 1), 0
    for i in range(1, extra + 1):
        if (hp >> (i - 1)) < 2 or (wp >> (i - 1)) < 2 or hp % (1 << i) or wp % (1 << i):
            return None                                      # level i needs an even level i - 1 of at least 2 x 2
        offsets[i] = off
        off += planes * (hp >> i) * (wp >> i)
    offsets[0] = off
    return dict(lp=lp, rp=rp, hp=hp, wp=wp, offsets=offsets)


def pyramid_elems(planes, hs, ws, extra):
    """gg_mipmap_pyramid_elems: floats of levels 1..E, -1 for a refused shape."""
    if planes < 0 or hs < 1 or ws < 1:
        return -1
    py = make_pyramid(hs, ws, planes, extra)
    return -1 if py is None else py["offsets"][0]


def level_shape(py, i):
    return py["hp"] >> i, py["wp"] >> i


def _trips(tag, total, sms):
    return "%s: %s" % (tag, "one trip" if total <= grid_for(total, sms=sms) * THREADS else "several trips")


def build_route(planes, hs, ws, extra, sms=H100_SMS):
    """warp.cu build_t: one fused launch when levels 1..E of a plane fit in shared memory (static up to 48 KB, after the
    opt-in up to 200 KB), else one mip_down launch per level; nothing for planes == 0 or E == 0."""
    py = make_pyramid(hs, ws, planes, extra)
    smem = 4 * sum(h * w for h, w in (level_shape(py, i) for i in range(1, extra + 1)))
    if planes == 0 or extra == 0:
        return "no launch"
    if smem <= OPTIN_SMEM and planes <= 0x7fffffff:
        return "fused, static shared memory" if smem <= STATIC_SMEM else "fused, 200 KB opt-in"
    return "one launch per level"


def pyramid_labels(case, sms=H100_SMS):
    planes, hs, ws, extra, dtype = case
    py = make_pyramid(hs, ws, planes, extra)
    route = build_route(planes, hs, ws, extra, sms)
    labels = {"build: %s" % route, "build: %s, %s" % (route, SHORT[dtype]), "extra = %d" % extra,
              "one plane" if planes == 1 else "many planes"}
    total1 = planes * (py["hp"] >> 1) * (py["wp"] >> 1)
    if route == "one launch per level":
        labels.add(_trips("per-level build, level 1", total1, sms))
    labels.add(_trips("adjoint, level 1", total1, sms))
    pad = py["lp"] + py["rp"]
    labels.add("power-of-two source" if pad == 0 else "%s total padding" % ("even" if pad % 2 == 0 else "odd"))
    if pad and py["lp"] == 0:
        labels.add("padding on the right / bottom only (lp = 0)")
    if hs != ws and pad:
        labels.add("non-square, the height takes the width's padding")
    return labels


def tent_out(n, s):
    """resample.cu check_tent: output size of one axis."""
    p = s // 2
    return (n + 2 * p - 2 * s) // s + 1


def tent_min_plane(s):
    """The smallest legal plane of one axis: larger than the padding s // 2, and the padded axis holds one 2s window."""
    p = s // 2
    return max(p + 1, 2 * s - 2 * p)


def tent_legal(h, w, s):
    if not 1 <= s <= 16:
        return False
    return min(h, w) >= tent_min_plane(s)


def tent_sources(n, s):
    """Padded positions u (0 <= u < n + 2p) of each input index, by reflecting every padded position (independent of
    resample.cu padded_positions, which lists them per input index)."""
    p = s // 2
    src = [[] for _ in range(n)]
    for u in range(n + 2 * p):
        src[reflect(u - p, n)].append(u)
    return src


def tent_window_counts(n, s):
    """Per input index: the (padded position, output window) pairs that read it -- the gather-form backward's terms."""
    oh = tent_out(n, s)
    return np.array([sum(sum(1 for o in range(oh) if o * s <= u < o * s + 2 * s) for u in us)
                     for us in tent_sources(n, s)])


def tent_labels(case):
    n, c, h, w, s = case
    hm = tent_min_plane(s)
    labels = {"tent: stride %d" % s}
    if (h, w) == (hm, hm):
        labels.add("tent: the smallest legal plane")
    if (h, w) == (hm + 1, hm):
        labels.add("tent: the smallest legal plane + one row")
    if (h, w) == (hm, hm + 1):
        labels.add("tent: the smallest legal plane + one column")
    if h != w:
        labels.add("tent: non-square")
    if h % 2 and w % 2:
        labels.add("tent: odd sizes")
    if n > 1 and c > 1:
        labels.add("tent: N, C > 1")
    if (h, w, s) == (256, 256, 2):
        labels.add("tent: 256^2 at s = 2")
    for size in (h, w):
        if any(len({0 if u < s // 2 else 2 if u >= size + s // 2 else 1 for u in us}) == 3 for us in tent_sources(size, s)):
            labels.add("tent: an input index reached from the left reflection, the interior and the right reflection")
    return labels


# ------------------------------------------------------------------------------------------------------------- cases
PYR_CASES = [
    # (planes, hs, ws, E, dtype)
    (1, 128, 128, 7, F32), (6, 128, 128, 1, F16), (5, 2, 2, 1, F32), (4, 3, 3, 2, BF16), (3, 5, 5, 3, F32),
    (2, 32, 32, 5, BF16), (1, 64, 64, 6, F16),                                         # static shared memory
    (3, 256, 256, 8, F32), (3, 256, 256, 8, F16), (2, 256, 256, 4, BF16), (3, 129, 129, 8, F32),
    (3, 129, 129, 8, BF16), (2, 194, 450, 8, F32), (1, 194, 450, 8, F16), (3, 65, 129, 6, F32),    # 200 KB opt-in
    (3, 512, 512, 3, F32), (12, 512, 512, 8, F32), (3, 512, 512, 8, F16), (3, 512, 512, 2, BF16),
    (3, 450, 450, 8, F32), (2, 450, 450, 5, BF16), (2, 257, 257, 8, F32),             # one launch per level
]
ADJ_CASES = sorted({c[:4] for c in PYR_CASES})
SINGLE_CASES = [
    # (N, C, hs, ws, E, dtype)
    (1, 3, 128, 128, 7, F32), (2, 2, 3, 3, 2, F32), (1, 3, 5, 5, 3, F32), (1, 3, 256, 256, 8, F16),
    (1, 3, 129, 129, 8, BF16), (1, 2, 194, 450, 8, F32), (1, 3, 65, 129, 6, F32), (1, 2, 450, 450, 5, BF16),
    (1, 3, 512, 512, 8, F32), (2, 1, 2, 2, 1, F32),
]
TENT_CASES = []
for _s in range(1, 17):
    _m = tent_min_plane(_s)
    TENT_CASES += [(2, 3, _m, _m, _s), (2, 3, _m + 1, _m, _s), (1, 3, _m, _m + 1, _s), (2, 3, 3 * _s + 5, 2 * _s + 7, _s)]
TENT_CASES.append((4, 3, 256, 256, 2))

REQUIRED = (
    ["build: %s, %s" % (r, SHORT[d]) for r in ("fused, static shared memory", "fused, 200 KB opt-in", "one launch per level")
     for d in (F32, F16, BF16)]
    + ["extra = %d" % e for e in range(1, 9)]
    + ["one plane", "many planes", "power-of-two source", "even total padding", "odd total padding",
       "padding on the right / bottom only (lp = 0)", "non-square, the height takes the width's padding",
       "per-level build, level 1: one trip", "per-level build, level 1: several trips",
       "adjoint, level 1: one trip", "adjoint, level 1: several trips"]
    + ["single level: L = %d" % L for L in range(9)]
    + ["single level: from the level of detail", "single level: pinned by min_level"]
    + ["tent: stride %d" % s for s in range(1, 17)]
    + ["tent: the smallest legal plane", "tent: the smallest legal plane + one row",
       "tent: the smallest legal plane + one column", "tent: non-square", "tent: odd sizes", "tent: N, C > 1",
       "tent: 256^2 at s = 2",
       "tent: an input index reached from the left reflection, the interior and the right reflection"]
)


def lod_exact(size):
    """The level of detail scales an axis by (size - 1) / 2: a dyadic grid step lands exactly on 2^L px iff size - 1 is a
    power of two."""
    return size >= 2 and (size - 1) & (size - 2) == 0


def single_labels(case):
    n, c, hs, ws, extra, dtype = case
    labels = {"single level: L = %d" % L for L in range(extra + 1)}
    labels.add("single level: from the level of detail" if (lod_exact(hs) or lod_exact(ws))
               else "single level: pinned by min_level")
    return labels


def all_labels(sms=H100_SMS):
    reached = set()
    for cs in PYR_CASES:
        reached |= pyramid_labels(cs, sms)
    for cs in SINGLE_CASES:
        reached |= single_labels(cs)
    for cs in TENT_CASES:
        reached |= tent_labels(cs)
    return reached


def test_cases_reach_every_route():
    """Coverage of the cases below, by the restatement planned for 132 SMs: each build route in each source dtype, every
    E = 1..8, power-of-two sources and sources with even, odd and right-only padding, a non-square source that takes the
    width's padding, one and several grid-stride trips of the level-1 launches, single-level reads at every L = 0..8 by
    both mechanisms, and for the tent every stride 1..16 at its smallest legal plane and one row / column more."""
    reached = all_labels()
    assert_routes_reached(REQUIRED, reached)


def test_every_case_is_feasible_and_routed_as_labelled():
    for planes, hs, ws, extra, _ in PYR_CASES:
        assert make_pyramid(hs, ws, planes, extra) is not None, (hs, ws, extra)
    for n, c, hs, ws, extra, _ in SINGLE_CASES:
        assert make_pyramid(hs, ws, n * c, extra) is not None, (hs, ws, extra)
    for n, c, h, w, s in TENT_CASES:
        assert tent_legal(h, w, s), (h, w, s)
    # the sizes the route boundaries fall between
    assert build_route(1, 128, 256, 7) == "fused, static shared memory"
    assert build_route(1, 65, 129, 6) == "fused, 200 KB opt-in"          # level 1 alone is exactly 48 KB
    assert build_route(1, 194, 450, 8) == "fused, 200 KB opt-in"
    assert build_route(1, 450, 450, 1) == "one launch per level"


_SWEEP = sorted(set(range(1, 21)) | {31, 32, 33, 63, 64, 65, 96, 127, 128, 129, 130, 192, 194, 200, 255, 256, 257, 384,
                                      450, 511, 512, 513, 700, 1024})


def test_restated_pyramid_matches_the_library():
    """pyramid_elems agrees with gg_mipmap_pyramid_elems (a host-only query) over a sweep of shapes, refused ones (-1)
    included: sources too small for their padding, E = 0 and E > 8, levels that are not even, bad plane counts."""
    from gangealing_b200 import _lib
    lib = _lib.load()
    checked = refused = 0
    for hs in _SWEEP:
        for ws in _SWEEP:
            for extra in (0, 1, 2, 3, 5, 8, 9):
                for planes in (1, 3):
                    want = pyramid_elems(planes, hs, ws, extra)
                    got = lib.gg_mipmap_pyramid_elems(planes, hs, ws, extra)
                    assert got == want, (planes, hs, ws, extra, got, want)
                    checked += 1
                    refused += want < 0
    for args in [(-1, 8, 8, 1), (0, 8, 8, 1), (1, 0, 8, 1), (1, 8, 0, 1), (1, 8, 8, -1), (0, 450, 450, 8)]:
        assert lib.gg_mipmap_pyramid_elems(*args) == pyramid_elems(*args), args
    assert refused > 0 and refused < checked
    print("[plan] %d shapes checked, %d refused" % (checked, refused))


def test_restated_tent_legality_matches_the_entry():
    """tent_legal agrees with gg_tent_downsample_forward / _backward's shape checks (made before any pointer is used, so
    a legal shape with null pointers fails on the pointers instead): stride 0, stride 17, planes <= s // 2 and planes
    whose padded size is shorter than one 2s window are refused, on either axis."""
    from gangealing_b200 import _lib
    lib = _lib.load()
    for s in range(0, 18):
        for n in range(0, 40):
            for h, w in ((n, 40), (40, n)):
                want = tent_legal(h, w, s)
                for entry in (lib.gg_tent_downsample_forward, lib.gg_tent_downsample_backward):
                    rc = entry(None, None, None, None, 1, 1, h, w, s, None)
                    assert rc != 0
                    msg = lib.gg_last_error().decode()
                    assert ("null tensor" in msg) == want, (s, h, w, msg)
                    if want and s >= 1:
                        assert tent_out(h, s) >= 1 and tent_out(w, s) >= 1
    # nothing to do: an empty batch is legal whatever the plane size, but never the stride
    assert lib.gg_tent_downsample_forward(None, None, None, None, 0, 3, 1, 1, 4, None) == 0
    assert lib.gg_tent_downsample_forward(None, None, None, None, 0, 3, 8, 8, 17, None) != 0


# ======================================================================================================== GPU checks
WORST = Worst("c per path", "%-48s %.2f")
_report_worst = WORST.fixture()


def check(y, ref, a, c, path, what):
    y = y.detach().cpu()
    if y.dtype in (F16, BF16):
        _, obs = assert_rounded_once(y, ref, a, c, "%s: %s" % (path, what))
    else:
        obs = assert_fp32_sum(y, ref, a, c, "%s: %s" % (path, what))
    WORST.note(path, obs)
    print("[contract] %s: %s: obs=%.2f (bound %g)" % (path, what, obs, c))


def pyramid64(x64, py, extra):
    """float64 levels 1..E of x64 (planes, hs, ws): reflect-pad to the power of two with the width's padding, then
    ReflectionPad2d(1) + [1,3,3,1]^2/64 stride 2 per level (oracle/sampling.py downsample_2x)."""
    cur = x64[None]
    if py["lp"] or py["rp"]:
        cur = F.pad(cur, (py["lp"], py["rp"], py["lp"], py["rp"]), mode="reflect")
    out = []
    for _ in range(extra):
        cur = downsample_2x(cur)
        out.append(cur[0])
    return out


def pyramid_levels(flat, py, planes, extra):
    """Level i (planes, h, w) of the library's flat pyramid, at the restated offsets."""
    levels = [None]
    for i in range(1, extra + 1):
        h, w = level_shape(py, i)
        off = py["offsets"][i]
        levels.append(flat[off:off + planes * h * w].view(planes, h, w))
    return levels


def _pyr_id(cs):
    planes, hs, ws, extra, dtype = cs
    return "P%d-%dx%d-E%d-%s" % (planes, hs, ws, extra, SHORT[dtype])


# A level-i value is a 16-term fmaf chain with exact dyadic weights f[a] f[b] / 64 (16 roundings), over level i-1 values
# that carry their own error; the weights are positive and sum to 1, so that error reaches level i at most as large as
# it was, relative to the float64 pyramid of |x|: c_i = 16 + c_{i-1} = 16 i.
def c_level(i):
    return 16 * i


@pytest.mark.gpu
@pytest.mark.parametrize("case", PYR_CASES, ids=_pyr_id)
def test_pyramid_levels(case):
    from gangealing_b200.stn.sampling import _pyramid
    planes, hs, ws, extra, dtype = case
    py = make_pyramid(hs, ws, planes, extra)
    route = build_route(planes, hs, ws, extra)
    x = torch.randn(1, planes, hs, ws, generator=seeded(hs * 7 + ws + extra), device=DEV).to(dtype)
    flat = _pyramid(x, extra)
    assert flat.numel() == py["offsets"][0]
    x64 = x[0].double().cpu()
    ref, ref_abs = pyramid64(x64, py, extra), pyramid64(x64.abs(), py, extra)
    got = pyramid_levels(flat, py, planes, extra)
    for i in range(1, extra + 1):
        check(got[i], ref[i - 1], ref_abs[i - 1], c_level(i), "pyramid, %s" % route, "%s level %d" % (_pyr_id(case), i))


def down_t(g, shape, pad=None):
    """float64 transpose of one pyramid step into a (planes, h, w) level -- the vjp of downsample_2x [after the
    power-of-two reflect padding]."""
    z = torch.zeros(shape, dtype=torch.float64, requires_grad=True)
    zz = z[None]
    if pad is not None:
        zz = F.pad(zz, pad, mode="reflect")
    y = downsample_2x(zz)[0]
    return torch.autograd.grad(y, z, g)[0]


def tap_fanin(n_in, dest, lp=None):
    """Per destination index of one axis: how many (output, tap) pairs of a pyramid step from an n_in-long level read it,
    through ReflectionPad2d(1) and, on level 1 (lp given), the reflect padding to the power of two (warp.cu down_tap)."""
    cnt = np.zeros(dest, dtype=np.int64)
    for o in range(n_in // 2):
        for a in range(4):
            j = reflect(2 * o + a - 1, n_in)
            if lp is not None:
                j = reflect(j - lp, dest)
            cnt[j] += 1
    return cnt


def adjoint_cs(hs, ws, py, extra):
    """c of every level of the adjoint's result (index 0: grad_src).  Level E is only read.  An element of level i - 1
    receives `fan-in` atomicAdds of products g * w (w exact, the product rounded once) onto its initial value: fan-in + 1
    roundings of terms bounded by the float64 transpose of |G|; its share of level i's error arrives through positive
    weights, at most c_i relative to the same bound: c_{i-1} = c_i + max fan-in + 1."""
    cs = [0] * (extra + 1)
    for i in range(extra, 0, -1):
        h_in, w_in = level_shape(py, i - 1)
        if i == 1:
            fy, fx = tap_fanin(h_in, hs, py["lp"]), tap_fanin(w_in, ws, py["lp"])
        else:
            fy, fx = tap_fanin(h_in, h_in), tap_fanin(w_in, w_in)
        cs[i - 1] = cs[i] + int(fy.max() * fx.max()) + 1
    return cs


@pytest.mark.gpu
@pytest.mark.parametrize("case", ADJ_CASES, ids=lambda cs: "P%d-%dx%d-E%d" % cs)
def test_pyramid_adjoint(case):
    """gg_mipmap_build_backward adds build^T(G) to grad_src and leaves every intermediate level holding its own total
    gradient; compared per level with the float64 transpose, and by <build(x), G> = <x, build^T(G)> in float64."""
    from gangealing_b200.stn.sampling import _pyramid
    lib = library()
    planes, hs, ws, extra = case
    py = make_pyramid(hs, ws, planes, extra)
    gen = seeded(hs * 13 + ws + extra)
    G = [torch.randn(planes, hs, ws, generator=gen, device=DEV)]
    G += [torch.randn(planes, *level_shape(py, i), generator=gen, device=DEV) for i in range(1, extra + 1)]
    grad_pyr = torch.cat([g.reshape(-1) for g in G[1:]])
    grad_src = G[0].clone()
    rc = lib.load().gg_mipmap_build_backward(grad_src.data_ptr(), grad_pyr.data_ptr(), planes, hs, ws, extra, lib.stream())
    lib.check(rc, "gg_mipmap_build_backward")
    got = [grad_src] + pyramid_levels(grad_pyr, py, planes, extra)[1:]

    G64 = [g.double().cpu() for g in G]
    ref, ref_abs = [None] * (extra + 1), [None] * (extra + 1)
    ref[extra], ref_abs[extra] = G64[extra], G64[extra].abs()
    pad = (py["lp"], py["rp"], py["lp"], py["rp"]) if (py["lp"] or py["rp"]) else None
    for i in range(extra, 0, -1):
        shape = G64[i - 1].shape
        p = pad if i == 1 else None
        ref[i - 1] = G64[i - 1] + down_t(ref[i], shape, p)
        ref_abs[i - 1] = G64[i - 1].abs() + down_t(ref_abs[i], shape, p)
    cs = adjoint_cs(hs, ws, py, extra)
    assert torch.equal(got[extra].cpu(), G[extra].cpu()), "level E is only read"
    for i in range(extra - 1, -1, -1):
        check(got[i], ref[i], ref_abs[i], cs[i], "adjoint, level" if i else "adjoint, grad_src",
              "P%d-%dx%d-E%d %s" % (planes, hs, ws, extra, "level %d" % i if i else "grad_src"))

    # the inner-product identity on the library's own forward and adjoint, in float64
    x = torch.randn(1, planes, hs, ws, generator=gen, device=DEV)
    fwd = pyramid_levels(_pyramid(x, extra), py, planes, extra)
    x64 = x[0].double().cpu()
    fwd_abs = pyramid64(x64.abs(), py, extra)
    lhs = sum(float((fwd[i].double().cpu() * G64[i]).sum()) for i in range(1, extra + 1))
    rhs = float((x64 * (got[0].double().cpu() - G64[0])).sum())
    bound = sum(c_level(i) * U32 * float((fwd_abs[i - 1] * G64[i].abs()).sum()) for i in range(1, extra + 1))
    bound += cs[0] * U32 * float((x64.abs() * ref_abs[0]).sum())
    # ... which the float64 reference itself meets to float64 accuracy
    ref_fwd = pyramid64(x64, py, extra)
    lhs64 = sum(float((ref_fwd[i - 1] * G64[i]).sum()) for i in range(1, extra + 1))
    rhs64 = float((x64 * (ref[0] - G64[0])).sum())
    assert abs(lhs64 - rhs64) <= 1e-12 * bound / U32, (lhs64, rhs64)
    obs = abs(lhs - rhs) / (bound / cs[0]) if bound else 0.0
    assert abs(lhs - rhs) <= bound, "inner-product identity: |%.9g - %.9g| > %.3g" % (lhs, rhs, bound)
    print("[contract] adjoint identity: P%d-%dx%d-E%d: |<Px, G> - <x, P^T G>| = %.3g <= %.3g" %
          (planes, hs, ws, extra, abs(lhs - rhs), bound))
    WORST.note("adjoint identity (in units of the grad_src c)", obs)


@pytest.mark.gpu
def test_pyramid_adjoint_without_work_leaves_grad_src_untouched():
    lib = library()
    gen = seeded(5)
    grad_src = torch.randn(3, 64, 64, generator=gen, device=DEV)
    grad_pyr = torch.randn(3 * 32 * 32, generator=gen, device=DEV)
    keep_src, keep_pyr = grad_src.clone(), grad_pyr.clone()
    for planes, extra in ((0, 1), (3, 0), (0, 0)):
        rc = lib.load().gg_mipmap_build_backward(grad_src.data_ptr(), grad_pyr.data_ptr(), planes, 64, 64, extra, lib.stream())
        lib.check(rc, "gg_mipmap_build_backward")
        torch.cuda.synchronize()
        assert torch.equal(grad_src, keep_src) and torch.equal(grad_pyr, keep_pyr), (planes, extra)


def axis_points(size, L):
    """Grid entries along one axis for a read at level L: multiples of 2^-12 from -1.25, step 2^(L+1-k) with
    2^k >= size - 1, so neighbours sit (size - 1) 2^(L-k) <= 2^L px apart in level-of-detail coordinates (equal iff
    size - 1 = 2^k), and ((g + 1) size - 1) / 2 is exact in fp32."""
    k = max(0, math.ceil(math.log2(size - 1))) if size > 1 else 0
    step = 2.0 ** (L + 1 - k)
    count = max(2, int(math.floor(2.5 / step)) + 1)
    return -1.25 + 3 * 2.0 ** -12 + step * torch.arange(count, dtype=torch.float64)


def _single_id(cs):
    n, c, hs, ws, extra, dtype = cs
    return "N%d-C%d-%dx%d-E%d-%s" % (n, c, hs, ws, extra, SHORT[dtype])


# The read at level L: level_value is a bilinear up-sampling (weights exact: inv_scale = 2^-L and the coordinates are
# exact) of 4 level values, uy.l0 * (ux.l0 v00 + ux.l1 v01) + ...: a product, an addition, a product, an addition -- 4
# roundings per term; the sampler's bilinear sum v * (wx * wy) over 4 corners: 2 products and 3 additions -- 5.  The
# level values carry c_level(L) relative to the |x| pyramid and reach the output through positive weights.
def c_single(L):
    return 5 + (c_level(L) + 4 if L > 0 else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SINGLE_CASES, ids=_single_id)
def test_single_level_reads(case):
    """The sampler read at exactly level L (w = 0, l0 = l1 = L) equals the bilinear sample of the float64 Gaussian stack
    level L (oracle/sampling.py create_stack: the level upsampled to the padded size, cropped by lp), for every L = 0..E
    and every padding mode, with no pixel exempt."""
    from gangealing_b200.stn.sampling import _pyramid
    lib = library()
    n, c, hs, ws, extra, dtype = case
    x = torch.randn(n, c, hs, ws, generator=seeded(hs * 3 + ws), device=DEV).to(dtype)
    pyr = _pyramid(x, extra)
    x64 = x.double().cpu()
    stack, stack_abs = create_stack(x64, extra + 1), create_stack(x64.abs(), extra + 1)
    exact = lod_exact(hs) or lod_exact(ws)
    for L in range(extra + 1):
        xs, ys = axis_points(ws, L), axis_points(hs, L)
        g64 = torch.stack(torch.broadcast_tensors(xs[None, :], ys[:, None]), -1)[None].expand(n, -1, -1, -1).contiguous()
        grid = g64.float().to(DEV)
        assert torch.equal(grid.double().cpu(), g64)
        ho, wo = g64.shape[1], g64.shape[2]
        min_level = 0.0 if exact else float(L)
        for mode in PAD_MODES:
            out = torch.empty(n, c, ho, wo, dtype=dtype, device=DEV)
            levels = torch.empty(n, ho, wo, dtype=torch.float32, device=DEV)
            rc = lib.load().gg_mipmap_warp_forward(out.data_ptr(), levels.data_ptr(), x.data_ptr(), lib.ptr(pyr),
                                                   grid.data_ptr(), lib.dtype_code(x), n, c, hs, ws, ho, wo, extra,
                                                   float(extra), min_level, lib.PAD_MODES[mode], lib.stream())
            lib.check(rc, "gg_mipmap_warp_forward")
            assert bool((levels == L).all()), "levels %s, want %d" % (levels.unique().tolist()[:8], L)
            ref = grid_sample_bilinear(stack[:, :, L].contiguous(), g64, mode)[0]
            ref_abs = grid_sample_bilinear(stack_abs[:, :, L].contiguous(), g64, mode)[0]
            check(out, ref, ref_abs, c_single(L), "single level, %s" % ("level of detail" if exact else "min_level"),
                  "%s L=%d %s" % (_single_id(case), L, mode))


def tent64(x, kh, kv, s):
    """float64 reflect-pad s // 2 + per-channel taps kh along x then kv along y, stride s (index arithmetic of its own)."""
    p = s // 2
    n, c, h, w = x.shape
    oh, ow = tent_out(h, s), tent_out(w, s)
    xp = F.pad(x, [p] * 4, mode="reflect") if p else x
    hz = sum(kh[None, :, None, None, j] * xp[:, :, :, j:j + s * (ow - 1) + 1:s] for j in range(2 * s))
    return sum(kv[None, :, i, None, None] * hz[:, :, i:i + s * (oh - 1) + 1:s, :] for i in range(2 * s))


def _tent_id(cs):
    return "N%d-C%d-%dx%d-s%d" % cs


@pytest.mark.gpu
@pytest.mark.parametrize("case", TENT_CASES, ids=_tent_id)
def test_tent_forward_and_adjoint(case):
    """bilinear_downsample with distinct random taps per channel and per axis (taps_h != taps_v), forward and gather-form
    backward against float64, and <T x, g> = <x, T^T g>."""
    from gangealing_b200.stn.sampling import bilinear_downsample
    n, c, h, w, s = case
    gen = seeded(h * 100 + w + s)
    x = torch.randn(n, c, h, w, generator=gen, device=DEV)
    kh = torch.randn(c, 2 * s, generator=gen, device=DEV)
    kv = torch.randn(c, 2 * s, generator=gen, device=DEV)
    xg = x.clone().requires_grad_(True)
    y = bilinear_downsample(xg, s, kh.reshape(c, 1, 1, 2 * s), kv.reshape(c, 1, 2 * s, 1))
    assert y.shape == (n, c, tent_out(h, s), tent_out(w, s))
    gout = torch.randn(y.shape, generator=gen, device=DEV)
    y.backward(gout)
    x64, kh64, kv64, g64 = (t.double().cpu() for t in (x, kh, kv, gout))
    # forward: per output, the horizontal fmaf chain over 2s taps then the vertical one over 2s: 4s roundings
    ref, ref_abs = tent64(x64, kh64, kv64, s), tent64(x64.abs(), kh64.abs(), kv64.abs(), s)
    check(y, ref, ref_abs, 4 * s, "tent forward", _tent_id(case))
    # backward: an input element sums count_y * count_x terms (restated window counts) in one fmaf chain, each term's
    # weight wv * kh rounded once first: c = max count + 1
    x64r = x64.clone().requires_grad_(True)
    ref_g = torch.autograd.grad(tent64(x64r, kh64, kv64, s), x64r, g64)[0]
    xa = torch.zeros_like(x64).requires_grad_(True)
    ref_g_abs = torch.autograd.grad(tent64(xa, kh64.abs(), kv64.abs(), s), xa, g64.abs())[0]
    c_bwd = int(tent_window_counts(h, s).max() * tent_window_counts(w, s).max()) + 1
    check(xg.grad, ref_g, ref_g_abs, c_bwd, "tent backward", _tent_id(case))
    lhs = float((y.detach().double().cpu() * g64).sum())
    rhs = float((x64 * xg.grad.double().cpu()).sum())
    bound = U32 * (4 * s * float((ref_abs * g64.abs()).sum()) + c_bwd * float((x64.abs() * ref_g_abs).sum()))
    assert abs(lhs - rhs) <= bound, "inner-product identity: |%.9g - %.9g| > %.3g" % (lhs, rhs, bound)
    print("[contract] tent identity: %s: %.3g <= %.3g" % (_tent_id(case), abs(lhs - rhs), bound))


@pytest.mark.gpu
def test_tent_entries_refuse_bad_strides_and_planes():
    """The Python face raises on a stride outside 1..16 and on a plane not larger than s // 2, and the entries refuse
    them on real tensors, leaving the output as it was."""
    from gangealing_b200.stn.sampling import bilinear_downsample
    lib = library()
    x = torch.randn(1, 3, 8, 8, device=DEV)
    for s in (0, 17):
        with pytest.raises(RuntimeError):
            bilinear_downsample(x, s, torch.ones(3, 1, 1, max(2 * s, 1), device=DEV),
                                torch.ones(3, 1, max(2 * s, 1), 1, device=DEV))
    with pytest.raises(RuntimeError):
        bilinear_downsample(torch.randn(1, 3, 2, 9, device=DEV), 4, torch.ones(3, 1, 1, 8, device=DEV),
                            torch.ones(3, 1, 8, 1, device=DEV))
    taps = torch.ones(3, 32, device=DEV)
    out = torch.full((64,), float("nan"), device=DEV)
    for h, w, s in ((8, 8, 0), (8, 8, 17), (2, 9, 4), (9, 2, 4), (3, 8, 3)):
        for entry in (lib.load().gg_tent_downsample_forward, lib.load().gg_tent_downsample_backward):
            assert entry(out.data_ptr(), x.data_ptr(), taps.data_ptr(), taps.data_ptr(), 1, 3, h, w, s, lib.stream()) != 0
    torch.cuda.synchronize()
    assert bool(out.isnan().all())
