"""Test infrastructure: the MSM's signed-digit recoding restated with Python integers.

`for_each_digit` (renegade_b200/csrc/msm.cu) cuts a canonical scalar into W = ceil(255 / c) windows of c bits and
recodes every window into a signed digit of magnitude <= 2^(c-1): a raw value above 2^(c-1) becomes raw - 2^c and
carries one into the next window; a raw value of exactly 2^c (a carry into an all-ones window) leaves magnitude 0 and
carries on.  The carry out of the top window is dropped.  A digit of magnitude m in window w goes to bucket
(w mod n_phys) * 2^(c-1) + m - 1 of its MSM, where n_phys is the number of physical windows of the plan (1 when
every window multiple is precomputed).

A bucket of k entries is folded in ceil(k / SEG_LEN) near-equal segments, and a bucket with more than COMBINE_SEQ
segments ("heavy") is combined by a block tree instead of one thread.  These constants, and the buckets per tile of
the histogram scan, are read from msm.cu, so the shape tests built on them follow the kernel if it changes."""
from __future__ import annotations

import os
import random
import re
from collections import Counter

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _msm_source() -> str:
    with open(os.path.join(ROOT, "renegade_b200", "csrc", "msm.cu")) as f:
        return f.read()


def _constant(pattern: str) -> int:
    m = re.search(pattern, _msm_source())
    assert m, f"msm.cu no longer matches {pattern!r}"
    return int(m.group(1))


SEG_LEN = _constant(r"#define B200_SEG_LEN (\d+)")
COMBINE_SEQ = _constant(r"constexpr int kCombineSeq = (\d+);")
HEAVY_MIN = SEG_LEN * COMBINE_SEQ + 1  # fewest entries of a heavy bucket
SCAN_TILE = _constant(r"constexpr int kScanThreads = (\d+);") * _constant(r"constexpr int kScanItems = (\d+);")  # buckets per scan tile
IDX_BITS = _constant(r"constexpr uint32_t kIdxBits = (\d+);")  # bits of the point index in a bucket entry
# msm_launch_batch refuses a launch whose worst-case entries, buckets or segments reach these powers of two
_GUARD = re.search(r"max_entries >= \(\(size_t\)1 << (\d+)\) \|\| n_buckets >= \(\(size_t\)1 << (\d+)\) \|\| "
                   r"max_segs >= \(\(size_t\)1 << (\d+)\)", _msm_source())
assert _GUARD, "msm.cu no longer states the launch guard of msm_launch_batch"
ENTRIES_LOG, BUCKETS_LOG, SEGMENTS_LOG = (int(g) for g in _GUARD.groups())

R = 0x30644E72E131A029B85045B68181585D2833E84879B97091_43E1F593F0000001  # the scalar field


def num_windows(c: int) -> int:
    """W of msm_choose_plan: enough c-bit windows for 255 bits."""
    return (255 + c - 1) // c


def choose_window(n: int, window_bits: int) -> int:
    """The window c of msm_choose_plan (msm.cu) restated: a fixed window as given, else the c in 6 … 23 with at most 32
    windows that minimises the throughput model (window_bits 0) or the latency model (1).  Where the two models pick
    different windows (31 and 4099 points: 8 / 10 and 13 / 15; 110 000 points: 17 / 16) the plan's window shows which
    model ran."""
    if window_bits > 1:
        return window_bits
    best, best_cost = 0, 1e300
    for c in range(6, 24):
        W = num_windows(c)
        if W > 32:
            continue
        t = 254 - c * (W - 1)
        nw = float(n) * W
        shrt = 0 if t >= c - 6 else c - 6 - t
        if window_bits == 0:
            buckets = float(1 << (c - 1))
            extra = max(0.0, nw / 32.0 - 0.55 * buckets)
            cost = (nw * (9.5 + 1.6 * (1.0 + 0.3 * shrt)) + buckets * 25.0 + extra * 12.5) / 66.7e6
        else:
            load = nw / float(1 << (c - 1))
            acc = max(nw / 6.6e6, 0.055 + 0.006 * min(load, 32.0) + 0.004 * min(load / 32.0, 64.0))
            top = float(n) / float(1 << t) / 32.0 if t < c - 1 else 0.0
            cost = (0.042 + nw * (1.0 + 0.1 * shrt) / 54e6 + acc + 0.13 + 0.0075 * c + float(1 << c) / 4.9e6
                    + 0.008 * min(top, 64.0))
        if cost < best_cost:
            best, best_cost = c, cost
    return best


def physical_windows(n: int, W: int, budget_bytes: int, forced: int = 1) -> int:
    """n_phys of msm_choose_plan: from the forced split (B200_MSM_PHYS_WINDOWS, ignored outside 1 … W), one more physical
    window at a time until the ceil(W / n_phys) tables of n 64-byte points fit the budget, or every window is physical."""
    phys = forced if 1 <= forced <= W else 1
    while -(-W // phys) * n * 64 > budget_bytes and phys < W:
        phys += 1
    return phys


def expected_plan(n: int, window_bits: int, phys: int = 1) -> dict:
    c = choose_window(n, window_bits)
    W = num_windows(c)
    return {"window_bits": c, "digits": W, "physical_windows": phys, "tables": -(-W // phys)}


def index_space(n: int, c: int, n_phys: int, batch: int) -> dict:
    """What msm_launch_batch sizes a launch of `batch` MSMs of n points by, before it allocates anything: the worst-case
    bucket entries (every digit non-zero), the buckets, and the worst-case segments (full ones plus one partial per
    bucket); and whether the launch is refused because one of them leaves its index space (32-bit entry offsets, bucket
    indices below 2^31, 30-bit segment counts in the scan's status word)."""
    entries = n * num_windows(c) * batch
    buckets = n_phys * (1 << (c - 1)) * batch
    segments = entries // SEG_LEN + buckets
    refused = entries >= 1 << ENTRIES_LOG or buckets >= 1 << BUCKETS_LOG or segments >= 1 << SEGMENTS_LOG
    return {"entries": entries, "buckets": buckets, "segments": segments, "refused": refused}


# One launch shape (n, c, n_phys, batch) per guard of msm_launch_batch, each the first batch past its limit (the
# b200_msm_batch_device cap of 64 for the entries): worst-case entries exactly 2^32; buckets past 2^31; segments past 2^30
# with entries and buckets inside theirs.  The guards run before anything is allocated, so the last two cost a
# one-point base set; the first needs 2^21 points at c = 8, split into one table.
GUARD_SHAPES = {
    "entries": (1 << 21, 8, 32, 64),
    "buckets": (1, 23, 12, 43),
    "segments": (1, 23, 12, 22),
}


def edge_scalars(c: int) -> list[int]:
    """Canonical scalars that hit the recoding's edges at window width c: per-window raw digits 0, 1, half - 1, half,
    half + 1, 2^c - 1 (each in every window, and mixed, so that carries run through every window); 2^m - 1, 2^m and
    2^m + 1 around every window boundary and at 252 / 253; r - 1, r - 2, (r - 1) / 2."""
    half = 1 << (c - 1)
    full = 252 // c  # windows wholly below bit 252: any digits there stay below r
    pats = [0, 1, half - 1, half, half + 1, (1 << c) - 1]
    out = [sum(v << (c * w) for w in range(full)) for v in pats]
    rng = random.Random(c)
    out += [sum(rng.choice(pats) << (c * w) for w in range(full)) for _ in range(24)]
    ms = {252, 253} | {k * c + d for k in range(1, num_windows(c)) for d in (-1, 0, 1)}
    for m in sorted(x for x in ms if 0 < x <= 253):
        out += [(1 << m) - 1, 1 << m, (1 << m) + 1]
    out += [R - 1, R - 2, (R - 1) // 2]
    return [s for s in out if s < R]


def signed_digits(s: int, c: int) -> tuple[list[tuple[int, int, int, bool]], int]:
    """([(window, raw, magnitude, negative)] for every window, carry out of the top window) as for_each_digit
    computes them for the 256-bit scalar s.  Windows of magnitude 0 are listed too (they add no entry)."""
    assert 0 <= s < 1 << 256
    half = 1 << (c - 1)
    out = []
    carry = 0
    for w in range(num_windows(c)):
        pos = w * c
        raw = ((s >> pos) & ((1 << c) - 1) if pos < 256 else 0) + carry
        if raw > half:
            out.append((w, raw, (1 << c) - raw, True))
            carry = 1
        else:
            out.append((w, raw, raw, False))
            carry = 0
    return out, carry


def reconstruct(digits, c: int, carry: int) -> int:
    """sum of the signed digits at their weights, plus the carry out of the top window."""
    v = sum((-m if neg else m) << (w * c) for w, _, m, neg in digits)
    return v + (carry << (len(digits) * c))


def bucket_counts(scalars, c: int, n_phys: int = 1) -> Counter:
    """{bucket: entries} of one MSM over canonical scalars (Python ints)."""
    half = 1 << (c - 1)
    cnt: Counter = Counter()
    for s in scalars:
        for w, _, m, _ in signed_digits(s, c)[0]:
            if m:
                cnt[(w % n_phys) * half + m - 1] += 1
    return cnt


def digit_arrays(scalars: np.ndarray, c: int):
    """Vectorised signed_digits over an (n, 4) uint64 array of canonical scalars: (magnitude[n, W], negative[n, W],
    carry_out[n]).  For the large shape tests; tests/test_msm_digits_cpu.py holds it equal to signed_digits."""
    s = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, 4)
    bits = np.unpackbits(s.view(np.uint8).reshape(-1, 32), axis=1, bitorder="little").astype(np.int64)
    n, W, half = s.shape[0], num_windows(c), 1 << (c - 1)
    weights = 1 << np.arange(c, dtype=np.int64)
    mag = np.zeros((n, W), dtype=np.int64)
    neg = np.zeros((n, W), dtype=bool)
    carry = np.zeros(n, dtype=np.int64)
    for w in range(W):
        lo, hi = w * c, min(w * c + c, 256)
        raw = (bits[:, lo:hi] * weights[:hi - lo]).sum(axis=1) + carry if lo < 256 else carry.copy()
        over = raw > half
        mag[:, w] = np.where(over, (1 << c) - raw, raw)
        neg[:, w] = over
        carry = over.astype(np.int64)
    return mag, neg, carry


def bucket_counts_np(scalars: np.ndarray, c: int, n_phys: int = 1) -> np.ndarray:
    """Entries per bucket (length n_phys * 2^(c-1)) of one MSM, from digit_arrays."""
    mag, _, _ = digit_arrays(scalars, c)
    half = 1 << (c - 1)
    phys = (np.arange(mag.shape[1]) % n_phys)[None, :].repeat(mag.shape[0], axis=0)
    live = mag > 0
    return np.bincount((phys * half + mag - 1)[live], minlength=n_phys * half)


def segments(count: int) -> int:
    return -(-count // SEG_LEN)


def is_heavy(count: int) -> bool:
    return segments(count) > COMBINE_SEQ
