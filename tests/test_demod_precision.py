"""The error bound of the tensor-core demodulation GEMM (csrc/modconv.cu demod_wgmma_kernel), proved on the CPU.

demod[b, o] = rsqrt(scale^2 * sum_i Wsq[o, i] * s[b, i]^2 + eps).  The kernel feeds TF32 MMAs, which read 10 explicit
mantissa bits of each operand.  It splits both operands, v = hi + lo with hi = v truncated to 10 bits, and issues three
MMAs per k-step (hi.hi + hi.lo + lo.hi): only lo.lo (~2^-20 relative, itself under the truncation of lo) is dropped, so
the result is fp32-grade.  Every term is nonnegative (no cancellation), so the per-element relative error against float64
is the right measure, and DEMOD_RTOL (demod_reference.py) bounds it.  Here two emulations of the kernel's arithmetic
run in float64 on the inputs the GPU test uses (tests/test_stylegan2_ops_gpu.py): one product per k-step with both
operands truncated to TF32 -- a kernel that dropped its lo products -- must VIOLATE the bound, the hi/lo split must MEET it.  So the bound sits
between what a TF32-only kernel and the split kernel can reach.
"""
import torch

from demod_reference import DEMOD_CASES, DEMOD_RTOL, EPS, demod_inputs, demod_ref, max_rel_err


def _tf32(v):
    """What a TF32 MMA reads of an fp32 value: its top 19 bits (10 explicit mantissa bits), the rest truncated."""
    return (v.float().view(torch.int32) & -8192).view(torch.float32)


def demod_emulated(w, s, scale, split, eps=EPS):
    """The kernel's arithmetic in float64: fp32 Wsq and fp32 squared styles as the operands, then either one TF32 product
    per k-step (`split` False) or the hi/lo split with three products (`split` True)."""
    a = w[0].float().pow(2).sum(dim=(2, 3))               # (O, I) fp32
    bq = s.float() * s.float()                            # (B, I) fp32
    a_hi, b_hi = _tf32(a), _tf32(bq)
    if split:
        a_lo, b_lo = _tf32(a - a_hi), _tf32(bq - b_hi)
        acc = b_hi.double() @ a_hi.double().t() + b_lo.double() @ a_hi.double().t() + b_hi.double() @ a_lo.double().t()
    else:
        acc = b_hi.double() @ a_hi.double().t()
    return torch.rsqrt(float(torch.tensor(scale, dtype=torch.float32)) ** 2 * acc + eps)


def test_demod_bound_separates_tf32_only_from_the_hi_lo_split():
    for b, o, i in DEMOD_CASES:
        w, s, scale = demod_inputs(b, o, i)
        want = demod_ref(w, s, scale)
        tf32_only = max_rel_err(demod_emulated(w, s, scale, split=False), want)
        hi_lo = max_rel_err(demod_emulated(w, s, scale, split=True), want)
        assert tf32_only > DEMOD_RTOL, "B=%d O=%d I=%d: a TF32-only kernel (%.2e) would pass the bound" % (b, o, i, tf32_only)
        assert hi_lo <= DEMOD_RTOL, "B=%d O=%d I=%d: the hi/lo split (%.2e) misses the bound" % (b, o, i, hi_lo)
