"""Rounding contract of the half-precision storage paths -- TEST INFRASTRUCTURE (see oracle/__init__.py).

bf16 / fp16 are storage formats in this project: every kernel reads its half-precision operands, computes in fp32 and
rounds each stored value once, to nearest (DESIGN.md section 3.4).  The two checks below state that contract against a
float64 reference evaluated on the exact operands a launch reads:

  assert_rounded_once   a stored half-precision output y:
                            |y - ref| <= 1/2 ulp(max(|ref|, |y|)) + k * 2^-24 * A
                        ulp is the bf16 / fp16 spacing of that binade (floored at the subnormal spacing), A is the same
                        reference evaluated on absolute values and k counts the fp32 roundings on the way to the store.
                        Any fp32 evaluation order plus ONE round-to-nearest store passes; a truncating store, a double
                        rounding (an intermediate stored and re-read) or half-precision arithmetic does not.
  assert_fp32_sum       an fp32 output computed from half-precision operands (a reduction, a dot product):
                            |y - ref| <= c * 2^-24 * sum|terms|
                        c follows from the kernel's reduction structure (the longest chain of fp32 additions an element
                        of the sum goes through, plus the roundings of the term itself).

Both take an optional `extra64`: a further absolute allowance per element, for an intermediate rounding a kernel is
documented to make (DESIGN.md's list of deviations), stated by the caller next to the check.

For reporting, assert_rounded_once returns (worst |y - ref| in ulps of the element's binade, the smallest k that would
pass) and assert_fp32_sum the worst |y - ref| / (2^-24 * sum|terms|), i.e. the smallest c that would pass.
"""
import torch

U32 = 2.0 ** -24                     # unit roundoff of fp32 (round to nearest)

# (explicit mantissa bits, smallest normal exponent) of the storage types
_FORMATS = {torch.bfloat16: (7, -126), torch.float16: (10, -14)}


def ulp(v, dtype):
    """Spacing of `dtype` in the binade of |v| (float64 tensor); below the normal range the subnormal spacing."""
    bits, emin = _FORMATS[dtype]
    _, e = torch.frexp(v.abs())      # |v| = m * 2^e, m in [0.5, 1)  ->  binade exponent e - 1 (0 for v == 0)
    e = torch.where(v == 0, torch.full_like(e, emin + 1), e)
    return torch.ldexp(torch.ones_like(v), (torch.clamp(e - 1, min=emin) - bits).to(v.dtype))


def _flat64(t, device):
    return t.detach().to(device=device, dtype=torch.float64).reshape(-1)


def _report(what, bad, worst, detail):
    return "%s: %d of %d elements outside the bound; worst at index %s: %s" % (what, int(bad.sum()), bad.numel(), worst, detail)


def assert_rounded_once(y, ref64, abs64, k, what="", extra64=None):
    """y: the stored bf16 / fp16 tensor; ref64 / abs64: float64 reference and the reference on absolute values, same
    shape (any layout, any device).  k: fp32 roundings between the operands and the store.
    -> (worst error in ulps, smallest k that passes)."""
    if y.dtype not in _FORMATS:
        raise TypeError("%s: assert_rounded_once checks a bf16 / fp16 tensor, got %s" % (what, y.dtype))
    assert tuple(y.shape) == tuple(ref64.shape) == tuple(abs64.shape), \
        "%s: shapes %s / %s / %s" % (what, tuple(y.shape), tuple(ref64.shape), tuple(abs64.shape))
    if y.numel() == 0:
        return 0.0
    dev = y.device
    yv, r, a = _flat64(y, dev), _flat64(ref64, dev), _flat64(abs64, dev)
    assert bool(torch.isfinite(r).all()) and bool(torch.isfinite(a).all()), "%s: non-finite reference" % what
    assert bool(torch.isfinite(yv).all()), "%s: %d non-finite outputs" % (what, int((~torch.isfinite(yv)).sum()))
    u = ulp(torch.maximum(r.abs(), yv.abs()), y.dtype)
    err = (yv - r).abs()
    slack = 0.5 * u + (_flat64(extra64, dev) if extra64 is not None else 0.0)
    bound = slack + k * U32 * a
    bad = err > bound
    ratio = err / u
    over = (err - slack).clamp(min=0)
    k_obs = float(torch.where(a > 0, over / (U32 * torch.where(a > 0, a, torch.ones_like(a))),
                              torch.where(over > 0, torch.full_like(over, float("inf")), torch.zeros_like(over))).max())
    if bool(bad.any()):
        i = int(torch.argmax(torch.where(bad, err / bound, torch.zeros_like(err))))
        idx = tuple(int(j) for j in torch.unravel_index(torch.tensor(i), tuple(y.shape)))
        raise AssertionError(_report(what, bad, idx, "value %.9g, reference %.9g, error %.4f ulp, bound %.4f ulp "
                                     "(1/2 ulp + k=%g x 2^-24 x A, A = %.6g)" % (
                                         float(yv[i]), float(r[i]), float(ratio[i]), float(bound[i] / u[i]), k, float(a[i]))))
    return float(ratio.max()), k_obs


def assert_fp32_sum(y, ref64, abs64, c, what="", extra64=None):
    """y: fp32 output; ref64: float64 reference (exact terms); abs64: float64 sum of |terms| per element.
    -> worst |y - ref| / (2^-24 * sum|terms|)."""
    assert tuple(y.shape) == tuple(ref64.shape) == tuple(abs64.shape), \
        "%s: shapes %s / %s / %s" % (what, tuple(y.shape), tuple(ref64.shape), tuple(abs64.shape))
    if y.numel() == 0:
        return 0.0
    dev = y.device
    yv, r, a = _flat64(y, dev), _flat64(ref64, dev), _flat64(abs64, dev)
    assert bool(torch.isfinite(yv).all()), "%s: %d non-finite outputs" % (what, int((~torch.isfinite(yv)).sum()))
    err = (yv - r).abs()
    scale = U32 * a
    if extra64 is not None:
        err = (err - _flat64(extra64, dev)).clamp(min=0)
    bound = c * scale
    bad = err > bound
    ratio = torch.where(scale > 0, err / torch.where(scale > 0, scale, torch.ones_like(scale)),
                        torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    if bool(bad.any()):
        i = int(torch.argmax(torch.where(bad, ratio, torch.zeros_like(ratio))))
        idx = tuple(int(j) for j in torch.unravel_index(torch.tensor(i), tuple(y.shape)))
        raise AssertionError(_report(what, bad, idx, "value %.9g, reference %.9g, error %.4g x 2^-24 x sum|terms| "
                                     "> c = %g (sum|terms| = %.6g)" % (float(yv[i]), float(r[i]), float(ratio[i]), c, float(a[i]))))
    return float(ratio.max())
