"""CPU: the Python restatement of the MSM's signed-digit recoding (tests/msm_digits.py), which the GPU shape tests use to
assert their own preconditions.  For every window width the library accepts (8 ... 23): the signed digits reconstruct
the scalar; the carry out of the top window — which the kernel drops — is 0 for every scalar below r, because the top
window of a 254-bit scalar holds t = 254 - c (W - 1) <= c - 1 bits; and scalars of 2^254 and more can carry out, which
is why that holds only for canonical scalars."""
import random

import numpy as np
import pytest

import msm_digits as md

R = md.R
WIDTHS = range(8, 24)
edge_scalars = md.edge_scalars


def test_constants_read_from_the_kernel():
    assert md.SEG_LEN == 32 and md.COMBINE_SEQ == 64 and md.HEAVY_MIN == 2049 and md.SCAN_TILE == 4096


@pytest.mark.parametrize("c", WIDTHS)
def test_digits_reconstruct_and_never_carry_out_below_r(c):
    W, half = md.num_windows(c), 1 << (c - 1)
    assert W <= 32  # the plan's table index has 5 bits
    t = 254 - c * (W - 1)
    assert 1 <= t <= c - 1, "the top window of a canonical scalar must stay below half a window"
    rng = random.Random(0xD161 + c)
    scalars = edge_scalars(c) + [rng.randrange(R) for _ in range(400)]
    raws = set()
    for s in scalars:
        digits, carry = md.signed_digits(s, c)
        assert carry == 0, hex(s)
        assert md.reconstruct(digits, c, carry) == s, hex(s)
        assert all(0 <= m <= half for _, _, m, _ in digits)
        raws |= {raw for _, raw, _, _ in digits}
    # the edge digits occur: the last bucket (positive half), half + 1 (negative, carry), 2^c (magnitude 0, carry only)
    assert {half, half + 1, 1 << c} <= raws
    # a carry chain reaches the top window
    digits, _ = md.signed_digits((1 << 253) - 1, c)
    assert all(raw in ((1 << c) - 1, 1 << c) for _, raw, _, _ in digits[:-1]) and digits[-1][1] >= 1


def test_carry_out_above_2_254():
    """Where the W windows span 255 or 256 bits the top window is a full c bits wide, and s = 2^(cW) - 1 (>= 2^254)
    carries out of it: the sum of the digits alone is then wrong.  At the other widths the top window is narrower than
    half a window for every 256-bit input."""
    carrying = []
    for c in WIDTHS:
        W = md.num_windows(c)
        if c * W <= 256:
            s = (1 << (c * W)) - 1
            assert s >= 1 << 254
            digits, carry = md.signed_digits(s, c)
            assert carry == 1 and md.reconstruct(digits, c, 0) != s
            carrying.append(c)
        else:
            digits, carry = md.signed_digits((1 << 256) - 1, c)
            assert carry == 0 and md.reconstruct(digits, c, 0) == (1 << 256) - 1
    assert carrying == [8, 15, 16, 17]


@pytest.mark.parametrize("c", [8, 11, 16, 23])
def test_vectorised_digits_match(c):
    import oracle_c
    rng = random.Random(c)
    scalars = edge_scalars(c) + [rng.randrange(R) for _ in range(200)]
    arr = oracle_c.ints_to_array(scalars)
    mag, neg, carry = md.digit_arrays(arr, c)
    for i, s in enumerate(scalars):
        digits, cy = md.signed_digits(s, c)
        assert [m for _, _, m, _ in digits] == list(mag[i]) and [x for _, _, _, x in digits] == list(neg[i])
        assert cy == carry[i]
    counts = md.bucket_counts(scalars, c, n_phys=3)
    dense = md.bucket_counts_np(arr, c, n_phys=3)
    assert {b: int(v) for b, v in enumerate(dense) if v} == dict(counts)
    assert np.count_nonzero(dense) > 0
