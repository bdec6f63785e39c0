"""The demodulation coefficients' float64 reference, error bound and cases (not collected: the name does not match
test_*.py).  test_demod_precision.py shows on the CPU that the bound separates a TF32-only kernel from the hi/lo split the
kernel runs; the GPU tests hold csrc/modconv.cu demod_wgmma_kernel to it and use the same inputs."""
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


def max_rel_err(got, want):
    return ((got.double().cpu() - want) / want).abs().max().item()
