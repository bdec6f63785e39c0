"""The error bound of the tensor-core demodulation GEMM (csrc/modconv.cu demod_wgmma_kernel), proved on the CPU.

demod[b, o] = rsqrt(scale^2 * sum_i Wsq[o, i] * s[b, i]^2 + eps).  The kernel feeds TF32 MMAs, which read 10 explicit
mantissa bits of each operand.  It splits both operands, v = hi + lo with hi = v truncated to 10 bits, and issues three
MMAs per k-step (hi.hi + hi.lo + lo.hi): only lo.lo (~2^-20 relative, itself under the truncation of lo) is dropped, so
the result is fp32-grade.  Every term is nonnegative (no cancellation), so the per-element relative error against float64
is the right measure, and DEMOD_RTOL below bounds it.  Here two emulations of the kernel's arithmetic run in float64 on
the inputs the GPU test uses (tests/test_stylegan2_ops_gpu.py): one product per k-step with both operands truncated to
TF32 -- a kernel that dropped its lo products -- must VIOLATE the bound, the hi/lo split must MEET it.  So the bound sits
between what a TF32-only kernel and the split kernel can reach.
"""
import torch

# per-element relative error bound of the demodulation coefficients against float64.  Budget: the dropped lo.lo products
# (2^-20 worst case, biased low by the truncation), fp32 accumulation of the MMA partial sums, the fp32 Wsq, rsqrtf.
# The accumulation dominates on the GPU: up to 5.4e-6 at I = 513 on an H100, where this emulation (exact sums) gives 2e-7.
DEMOD_RTOL = 8e-6
EPS = 1e-8

# (B, O, I): every template instance <NA, NS> launch_demod can pick (NS = 16-column slices of the padded batch, NA = 32-wide
# k-blocks staged per pipeline step: 4 needs a padded batch <= 32 and I >= 128, 2 a padded batch <= 64 and I > 32);
# B = 300 is split by the host into 256 + 44.  O spreads 1, 127, 128, 129, 200 and 512 over the 128-row tiles.
DEMOD_CASES = [
    (1, 1, 128),      # <4,1>
    (17, 127, 513),   # <4,2>
    (16, 128, 33),    # <2,1>
    (32, 129, 127),   # <2,2>
    (33, 200, 100),   # <2,4>
    (5, 512, 32),     # <1,1>
    (20, 129, 3),     # <1,2>  I % 4 != 0: scalar loads
    (64, 127, 32),    # <1,4>
    (65, 200, 257),   # <1,8>
    (256, 128, 130),  # <1,16>
    (300, 512, 130),  # <1,16> twice: 256 + 44
]


def demod_inputs(b, o, i, k=3, seed=0):
    """-> weight (1, O, I, k, k) fp32, style (B, I) fp32, scale.  Styles over a wide range (|s| = exp(U(-4, 4)), both
    signs) with some exact zeros; a few all-zero filter rows (their coefficient is rsqrt(eps))."""
    g = torch.Generator().manual_seed(seed + 7 * b + 13 * o + i)
    w = torch.randn(1, o, i, k, k, generator=g)
    if o > 2:
        w[0, torch.randperm(o, generator=g)[: max(1, o // 50)]] = 0.0
    s = torch.exp(torch.rand(b, i, generator=g) * 8.0 - 4.0) * torch.sign(torch.randn(b, i, generator=g))
    s[torch.rand(b, i, generator=g) < 0.05] = 0.0
    return w, s, 1.0 / (i * k * k) ** 0.5


def demod_ref(w, s, scale, eps=EPS):
    """float64 rsqrt(scale^2 * sum_i Wsq[o, i] s[b, i]^2 + eps), Wsq from the fp32 filters in float64 -> (B, O)."""
    wsq = w.double()[0].pow(2).sum(dim=(2, 3))
    return torch.rsqrt(scale ** 2 * (s.double().pow(2) @ wsq.t()) + eps)


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


def max_rel_err(got, want):
    return ((got.double().cpu() - want) / want).abs().max().item()


def test_demod_bound_separates_tf32_only_from_the_hi_lo_split():
    for b, o, i in DEMOD_CASES:
        w, s, scale = demod_inputs(b, o, i)
        want = demod_ref(w, s, scale)
        tf32_only = max_rel_err(demod_emulated(w, s, scale, split=False), want)
        hi_lo = max_rel_err(demod_emulated(w, s, scale, split=True), want)
        assert tf32_only > DEMOD_RTOL, "B=%d O=%d I=%d: a TF32-only kernel (%.2e) would pass the bound" % (b, o, i, tf32_only)
        assert hi_lo <= DEMOD_RTOL, "B=%d O=%d I=%d: the hi/lo split (%.2e) misses the bound" % (b, o, i, hi_lo)
