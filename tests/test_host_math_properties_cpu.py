"""Property tests (hypothesis) of the library's host-side integer helpers against exact big-integer / Decimal restatements of
the reference's definitions: batch_frexp (quant_utils.py:188-213, Decimal ROUND_HALF_UP of mantissa * 2^31) and the dyadic
requantisation round(v * m / 2^e) with torch.round = round-half-to-even (quant_utils.py:406-408).  No kernels are launched."""
import math
from decimal import ROUND_HALF_UP, Decimal
from fractions import Fraction

import pytest
from hypothesis import given, settings, strategies as st

from hawq_b200 import _lib
from hawq_b200.build import build_library
from oracle import int_ref as ir


@pytest.fixture(scope="module", autouse=True)
def lib():
    build_library()
    return _lib.load()


def frexp_reference(r):
    """the reference's arithmetic, literally: np.frexp + Decimal(mant * 2**31).quantize(1, ROUND_HALF_UP), e = 31 - exp."""
    mant, ex = math.frexp(r)
    m = int(Decimal(mant * (2 ** 31)).quantize(Decimal("1"), rounding=ROUND_HALF_UP))
    return m, 31 - ex


def rhe_exact(v, m, e):
    q = Fraction(v * m, 2 ** e)
    fl = math.floor(q)
    rem = q - fl
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
        fl += 1
    return max(-2 ** 31, min(2 ** 31 - 1, fl))


ratios = st.one_of(
    st.floats(min_value=1e-12, max_value=1e6, allow_nan=False, allow_infinity=False),
    # mantissas whose scaled value sits exactly on .5 (ties of ROUND_HALF_UP) or on the 2^31 roll-over
    st.builds(lambda k, ex: math.ldexp((k + 0.5) / 2 ** 31, ex), st.integers(2 ** 30, 2 ** 31 - 1), st.integers(-30, 20)),
    st.builds(lambda ex: math.ldexp(1.0 - 2.0 ** -40, ex), st.integers(-30, 20)),
)


@settings(max_examples=400, deadline=None)
@given(ratios)
def test_dyadic_equals_reference_definition(r):
    m, e = frexp_reference(r)
    assert ir.dyadic(r) == (m, e)                       # the oracle restates it with floor(x + 0.5)
    if 1 <= e <= 62:
        assert _lib.dyadic(r) == (m, e)
        assert m <= 2 ** 31                             # 2^31 itself is allowed (no renormalisation in the reference)
    elif e > 62:
        assert _lib.dyadic(r) == (0, 1)                 # ratio < 2^-31 * 2^-31: every product rounds to 0
    else:
        with pytest.raises(_lib.HawqError):
            _lib.dyadic(r)


values = st.one_of(st.integers(-2 ** 31, 2 ** 31 - 1), st.integers(-70000, 70000))


@settings(max_examples=600, deadline=None)
@given(values, st.integers(0, 2 ** 31), st.integers(1, 62))
def test_host_requant_is_exact_round_half_even(lib, v, m, e):
    assert lib.hawq_rhe_requant_host(v, m, e) == rhe_exact(v, m, e)


@settings(max_examples=300, deadline=None)
@given(st.integers(-2 ** 20, 2 ** 20), st.integers(1, 40), st.integers(0, 11))
def test_host_requant_exact_ties(lib, q, k, odd_shift):
    """v * m = (2q + 1) * 2^(e-1): exactly half way -> the even neighbour."""
    e = k + 1
    m = 2 ** k if k <= 31 else 2 ** 31
    v = 2 * q + 1
    if v * m % 2 ** (e - 1) != 0 or (v * m // 2 ** (e - 1)) % 2 == 0:
        return                                           # not a tie for this (m, e): covered by the generic property
    got = lib.hawq_rhe_requant_host(v, m, e)
    assert got == rhe_exact(v, m, e) and got % 2 == 0


# ------------------------------------------------------------------------------------------------------------------------------
# The arithmetic of the fused epilogues (hawq_b200/csrc/common.cuh, conv_igemm.cuh), modelled with exact rationals: one FP64 FMA
# with the 1.5 * 2^52 constant rounds (v + bias) * m / 2^e once, to nearest-even, and the low mantissa word is the integer result.
# float(Fraction) is correctly rounded, so this checks the ALGORITHM (not the CUDA code, which the -m gpu tests cover).
import struct  # noqa: E402

from hypothesis import example  # noqa: E402

MAGIC = 3 * 2 ** 51            # 1.5 * 2^52
OFF_S = 2 ** 52 + 2 ** 31      # double({0x43300000, v ^ 0x80000000}) = 2^52 + 2^31 + v
OFF_U = 2 ** 52                # double({0x43300000, u})              = 2^52 + u
K_DEEP = 3 * 3 * 512           # deepest ResNet convolution (72 k-tiles)
ACC_BOUND = {8: K_DEEP * 128 * 128, 4: K_DEEP * 15 * 128}   # |acc| for int8 / unsigned 4-bit activations, int8 weights


def _lo_word(y):
    bits = struct.unpack("<Q", struct.pack("<d", y))[0]
    lo = bits & 0xFFFFFFFF
    return lo - 2 ** 32 if lo >= 2 ** 31 else lo, bits >> 32


def sat32(v):
    return max(-2 ** 31, min(2 ** 31 - 1, v))


def bias_window(acc_bound):
    """set_bias_window (api.cu): the biases for which acc + bias stays inside int32 for every |acc| <= acc_bound."""
    b = min(acc_bound, 2 ** 31)
    return b - 2 ** 31, 2 ** 31 - 1 - b


def fast_signed(v, bias, m, e, acc_bound=ACC_BOUND[8]):
    """RqFp64 (conv_igemm.cuh): d = v + bias through the folded int -> double conversion (sCb), clamped to int32 in a CTA with a
    bias outside the window, then one FMA"""
    d = float(OFF_S + v)                                   # exact: < 2^53
    cb = float(OFF_S - bias)                               # exact
    dv = d - cb                                            # exact: v + bias
    assert Fraction(dv) == v + bias
    lo, hi = bias_window(acc_bound)
    if not lo <= bias <= hi:                               # a clamped CTA
        dv = min(max(dv, -2.0 ** 31), 2.0 ** 31 - 1)
    y = float(Fraction(dv) * Fraction(m, 2 ** e) + MAGIC)  # the FMA: one rounding
    return _lo_word(y)


def fast_unsigned_folded(u, m, e):
    big_m = Fraction(m, 2 ** e)
    c = float(Fraction(MAGIC) - OFF_U * big_m)
    assert Fraction(c) == Fraction(MAGIC) - OFF_U * big_m  # the folded constant is exact for e <= 51
    y = float(Fraction(OFF_U + u) * big_m + Fraction(c))
    return _lo_word(y)[0]


M_5E8, E_5E8 = ir.dyadic(5e-8)   # a near-dead channel: tiny ratio, bias at the int32 limit


@settings(max_examples=1000, deadline=None)
@given(st.sampled_from([8, 4]), st.integers(-ACC_BOUND[8], ACC_BOUND[8]), st.integers(-2 ** 31, 2 ** 31 - 1), st.integers(0, 2 ** 31),
       st.integers(31, 62))
@example(8, ACC_BOUND[8], 2 ** 31 - 1, 2 ** 31, 31)
@example(8, -ACC_BOUND[8], -2 ** 31, 2 ** 31, 31)
@example(4, ACC_BOUND[8], 2 ** 31 - 1, 2 ** 31, 31)
@example(8, 5_000_000, 2 ** 31 - 1, M_5E8, E_5E8)
@example(8, -5_000_000, -2 ** 31, M_5E8, E_5E8)
@example(8, 75_000_000, 2 ** 31 - 1000, 2 ** 31, 31)
def test_fma_requant_is_exact_for_ratios_up_to_one(a_bits, v, bias, m, e):
    """acc up to the K = 4608 bound of either activation width, any int32 bias: the epilogue equals RHE(sat32(acc + bias) * ratio)."""
    if a_bits == 4:
        v = v * 15 // 128                                  # |acc| <= K * 15 * 128
    q, _ = fast_signed(v, bias, m, e, ACC_BOUND[a_bits])
    assert q == rhe_exact(sat32(v + bias), m, e)


@settings(max_examples=600, deadline=None)
@given(st.integers(-2 ** 30, 2 ** 30), st.integers(-2 ** 31, 2 ** 31 - 1), st.integers(2 ** 30, 2 ** 31), st.integers(11, 40))
@example(2 ** 30, 2 ** 31 - 1, 2 ** 31, 11)
@example(-2 ** 30, -2 ** 31, 2 ** 31, 11)
@example(-2 ** 30, -2 ** 31, 2 ** 30, 40)
@example(2 ** 30, 2 ** 30, 2 ** 31, 40)
def test_fma_requant_wide_ratios_with_overflow_check(v, bias, m, e):
    """ratios up to 2^20, |acc| <= 2^30 and any int32 bias: the result is RHE(sat32(acc + bias) * ratio) whenever the kernel's
    validity check passes, and the check fails exactly when that rounded value leaves int32 (then HAWQ_FLAG_REQUANT_OVERFLOW is
    raised and the saturating kernels are used)."""
    q, hi = fast_signed(v, bias, m, e, acc_bound=2 ** 30)
    exact = Fraction(sat32(v + bias) * m, 2 ** e)
    fl = math.floor(exact)
    rem = exact - fl
    r = fl + (1 if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1) else 0)   # unsaturated RHE
    valid = ((hi + ((q >> 31) & 1)) ^ 0x43380000) == 0          # bit-pattern form of the checked FP64 term in conv_igemm.cuh (t - 1.5 * 2^52 in int32)
    assert valid == (-2 ** 31 <= r < 2 ** 31)
    if valid:
        assert q == r


@settings(max_examples=600, deadline=None)
@given(st.integers(0, 2 ** 31 - 1), st.integers(0, 2 ** 31), st.integers(31, 51))
def test_folded_unsigned_fma_is_exact(u, m, e):
    assert fast_unsigned_folded(u, m, e) == rhe_exact(u, m, e)
