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
    assert md.IDX_BITS == 26 and (md.ENTRIES_LOG, md.BUCKETS_LOG, md.SEGMENTS_LOG) == (32, 31, 30)


def test_guard_shapes_land_on_their_guard():
    """Each shape of GUARD_SHAPES trips the guard it is named for, with one MSM fewer in the batch inside that limit: the
    GPU test that runs them checks each guard at its boundary.  The entries and segments shapes trip nothing else and
    one MSM fewer is not refused at all."""
    limit = {"entries": 1 << md.ENTRIES_LOG, "buckets": 1 << md.BUCKETS_LOG, "segments": 1 << md.SEGMENTS_LOG}
    for name, (n, c, n_phys, batch) in md.GUARD_SHAPES.items():
        assert 1 <= n_phys <= md.num_windows(c) and batch <= 64, name
        at = md.index_space(n, c, n_phys, batch)
        below = md.index_space(n, c, n_phys, batch - 1)
        assert at["refused"] and at[name] >= limit[name] > below[name], name
        assert name == "buckets" or not below["refused"], name
        assert [k for k in limit if at[k] >= limit[k]] == (["buckets", "segments"] if name == "buckets" else [name])
    assert md.index_space(*md.GUARD_SHAPES["entries"])["entries"] == 1 << 32
    # the buckets guard cannot trip alone: every bucket is at least one worst-case segment
    for c in range(8, 24):
        for n_phys in (1, md.num_windows(c)):
            batch = -(-(1 << md.BUCKETS_LOG) // (n_phys << (c - 1)))
            assert md.index_space(1, c, n_phys, batch)["segments"] >= 1 << md.SEGMENTS_LOG


def test_large_launches_inside_the_index_space():
    """The GPU runs of 2^22 points at c = 16: 40 MSMs put the worst-case entry offsets past 2^31 (bit 31 set in real
    offsets, as at most one digit in 2^15 is zero), 63 just below 2^32; 64 would be refused.  One MSM of 2^26 points
    at any automatic window stays inside every limit."""
    big = md.index_space(1 << 22, 16, 1, 40)
    assert big["entries"] >= (1 << 31) + (1 << 28) and not big["refused"]
    top = md.index_space(1 << 22, 16, 1, 63)
    assert (1 << 32) - top["entries"] == 1 << 26 and not top["refused"]
    assert md.index_space(1 << 22, 16, 1, 64)["refused"]
    for wb in (0, 1):
        c = md.choose_window(1 << 26, wb)
        assert not md.index_space(1 << 26, c, md.num_windows(c), 1)["refused"]


def test_physical_windows_restatement():
    """The budget split of msm_choose_plan: 2^26 points at c = 20 (13 windows) need 52 GiB unsplit, so half of an
    idle 80 GB GPU's memory takes two physical windows (7 tables); a forced split is a floor, not a ceiling."""
    assert md.choose_window(1 << 26, 0) == 20 and md.num_windows(20) == 13
    gib = 1 << 30
    assert md.physical_windows(1 << 26, 13, 52 * gib) == 1
    assert md.physical_windows(1 << 26, 13, 52 * gib - 1) == 2
    assert md.physical_windows(1 << 26, 13, 39 * gib) == 2
    assert md.physical_windows(1 << 26, 13, 0) == 13
    assert md.physical_windows(1 << 26, 13, 39 * gib, forced=13) == 13
    assert md.physical_windows(1 << 26, 13, 39 * gib, forced=14) == 2  # out of range: ignored
    assert md.expected_plan(1 << 26, 0, 2) == {"window_bits": 20, "digits": 13, "physical_windows": 2, "tables": 7}


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
