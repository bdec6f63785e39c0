"""The half-precision rounding checks of oracle/rounding.py accept exactly what the storage contract allows (one
round-to-nearest store after fp32 arithmetic) and reject the ways a kernel gets it subtly wrong."""
import pytest
import torch

from oracle.rounding import U32, assert_fp32_sum, assert_rounded_once, ulp


def _ref(n=100_000, seed=0):
    g = torch.Generator().manual_seed(seed)
    mag = torch.pow(10.0, torch.rand(n, generator=g, dtype=torch.float64) * 6 - 3)
    return torch.randn(n, generator=g, dtype=torch.float64) * mag


def _truncate(x32):
    """fp32 -> bf16 by dropping the low 16 bits (round toward zero)."""
    return (x32.view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)


def test_ulp_of_the_storage_types():
    v = torch.tensor([1.0, 1.5, 2.0, -3.0, 0.0, 2.0 ** -20, 65504.0], dtype=torch.float64)
    assert ulp(v, torch.bfloat16).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -6, 2.0 ** -133, 2.0 ** -27, 2.0 ** 8]
    # fp16: floored at the subnormal spacing 2^-24
    assert ulp(v, torch.float16).tolist() == [2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 2.0 ** -9, 2.0 ** -24, 2.0 ** -24, 2.0 ** 5]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_accepts_one_rounding_from_float64_and_from_fp32(dtype):
    ref = _ref()
    if dtype == torch.float16:
        ref = ref.clamp(-6e4, 6e4)
    # torch converts float64 -> fp16 through fp32: k = 1 covers that intermediate rounding as well
    assert assert_rounded_once(ref.to(dtype), ref, ref.abs(), 1, "RN(ref)")[0] <= 0.5 + 1e-4
    # through fp32 first: one fp32 rounding (k = 1) and one store
    assert_rounded_once(ref.float().to(dtype), ref, ref.abs(), 1, "RN(fl32(ref))")


def test_rejects_a_truncating_store():
    ref = _ref()
    with pytest.raises(AssertionError, match="outside the bound"):
        assert_rounded_once(_truncate(ref.float()), ref, ref.abs(), 4, "truncated")


def test_rejects_double_rounding():
    """RN(RN(t) * g): the intermediate stored in bf16 and re-read before the last product."""
    t = _ref(seed=1).float()
    gain = 2 ** 0.5
    ref = t.double() * gain
    assert_rounded_once((t * gain).to(torch.bfloat16), ref, ref.abs(), 2, "single rounding")
    with pytest.raises(AssertionError, match="outside the bound"):
        assert_rounded_once((t.to(torch.bfloat16).float() * gain).to(torch.bfloat16), ref, ref.abs(), 2, "double rounding")


@pytest.mark.parametrize("step", [1, -1])
def test_rejects_a_single_element_one_ulp_off(step):
    ref = _ref(seed=2)
    ref[12345] = 1.3                 # RN_bf16(1.3) = 1.296875: 0.4 ulp below, mid-binade
    y = ref.to(torch.bfloat16)
    assert_rounded_once(y, ref, ref.abs(), 1, "exact")
    bits = y.view(torch.int16).clone()
    bits[12345] += step
    with pytest.raises(AssertionError, match=r"1 of 100000 elements .* index \(12345,\)"):
        assert_rounded_once(bits.view(torch.bfloat16), ref, ref.abs(), 1, "one ulp off")


def test_fp32_sum_accepts_fp32_summation_and_rejects_summing_rounded_terms():
    g = torch.Generator().manual_seed(3)
    terms = torch.randn(64, 4096, generator=g).float()
    ref = terms.double().sum(1)
    a = terms.double().abs().sum(1)
    # a serial fp32 sum of 4096 terms: at most 4095 roundings on the longest chain
    c = assert_fp32_sum(terms.cumsum(1)[:, -1], ref, a, 4095, "serial fp32 sum")
    assert c < 4095
    with pytest.raises(AssertionError, match="outside the bound"):
        assert_fp32_sum(terms.to(torch.bfloat16).float().double().sum(1).float(), ref, a, 64, "sum of bf16-rounded terms")
    assert U32 == 2.0 ** -24
