"""Test infrastructure: satisfied circuits at the largest domains the prover runs on one GPU (2^18 … 2^22), built with
numpy instead of one gate at a time, and the device memory a key and its proofs take.

The prover's chunked scans (CH = 16 elements per thread and level) change their level structure only above the sizes the
rest of the suite proves: the grand product over n rows has 5 levels from 2^17 to 2^20 and 6 from 2^21, the opening
Horner scans over n + 3 coefficients reach 6 levels at 2^20.  `big_circuit` gives every gate kind of the synthetic mix
on rows at the start, on both sides of n/2 and at the end of the domain, all-zero selectors elsewhere, and copy cycles
across the chunk boundaries of every level.

`footprint_bytes` estimates the device memory of one context that holds its keys and has made k proofs in one call,
from the allocations in plonk.cu and msm.cu; NS, NW, CH, the coset rule, the workspace's constants and the MSM's
segment constants are read from the sources.  Measured on an idle H100 80GB HBM3 (free memory before and after), a
key and one proof used 3.71, 15.45, 28.91 and 55.82 GiB at 2^18, 2^20, 2^21 and 2^22, and with a second key 4.94,
20.35, 38.70 and 75.40 GiB; the estimates are at or above each, and estimate × 1.15 above every figure measured
(tests/README.md).  The SRS's window tables are counted
as one per window, what an idle GPU gets; the plan takes fewer when memory is short."""
from __future__ import annotations

import os
import random
import re
from dataclasses import dataclass, field

import numpy as np

import msm_digits as md
from renegade_b200 import synth
from test_prove_witness_cpu import wiring_permutation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = synth.R
RINV = pow(1 << 256, -1, R)
NUM_INPUTS = 17
GATE_KINDS = ("hash", "lc", "mul", "ecc", "const")


def plonk_source() -> str:
    with open(os.path.join(ROOT, "renegade_b200", "csrc", "plonk.cu")) as f:
        return f.read()


def _int(src: str, pattern: str) -> tuple:
    m = re.search(pattern, src)
    assert m, f"plonk.cu no longer matches {pattern!r}"
    return tuple(int(g) for g in m.groups())


def constants(src: str = None) -> dict:
    """The constants of plonk.cu the estimate depends on.  `workspace_elems` is restated in `workspace_elems` below; the
    source must still have the shape restated there."""
    src = plonk_source() if src is None else src
    c = {}
    c["NW"], = _int(src, r"constexpr int NW = (\d+);")
    c["NS"], = _int(src, r"constexpr int NS = (\d+);")
    c["CH"], = _int(src, r"constexpr int CH = (\d+);")
    c["kMaxEval"], = _int(src, r"constexpr int kMaxEval = (\d+);")
    c["kEvalSlots"], = _int(src, r"constexpr size_t kEvalSlots = (\d+);")
    # nc = log_n >= COSET_SWITCH ? COSETS_LARGE : COSETS_SMALL
    c["COSET_SWITCH"], c["COSETS_LARGE"], c["COSETS_SMALL"] = _int(src, r"const int nc = log_n >= (\d+) \? (\d+) : (\d+);")
    c["STAGE_PER_M"], = _int(src, r"std::max\((\d+) \* m, from_witness \? pk->num_vars : 0\)")
    c["NSCR2_PER_M"], = _int(src, r"bf\.nscr2->reserve\(\(size_t\)k \* (\d+) \* m \* sizeof\(fe\)\)")
    assert re.search(r"ntt_scratch\.reserve\(\(size_t\)NS \* m \* sizeof\(fe\)\)", src), \
        "preprocess no longer reserves NS * m elements of NTT scratch"
    assert re.search(r"const size_t S = n \+ 4, m = 8 \* n;\s*return k \* \(NW \* n \+ NW \* S \+ S \+ S \+ 3 \* n \+ "
                     r"\(2 \* \(n / CH\) \+ 4 \* CH \+ 64\) \+ 7 \* m \+ m \+ NW \* S \+ S \+ 2 \* \(S \+ 8\) \+\s*"
                     r"4 \* \(S / CH \+ 4 \* CH \+ 64\) \+ kMaxEval \* \(S / CH \+ S / CH / CH \+ 2 \* CH \+ 16\) \+ "
                     r"kEvalSlots\) \+\s*\(k \+ 7\) / 8 \+ 8;", src), "workspace_elems changed: restate it here"
    return c


def cosets(log_n: int, c: dict) -> int:
    return c["COSETS_LARGE"] if log_n >= c["COSET_SWITCH"] else c["COSETS_SMALL"]


def workspace_elems(n: int, k: int, c: dict) -> int:
    """plonk.cu's workspace_elems (m = 8n there, whatever the coset count)."""
    NW, CH = c["NW"], c["CH"]
    S, m = n + 4, 8 * n
    return k * (NW * n + NW * S + S + S + 3 * n + (2 * (n // CH) + 4 * CH + 64) + 7 * m + m + NW * S + S + 2 * (S + 8)
                + 4 * (S // CH + 4 * CH + 64) + c["kMaxEval"] * (S // CH + S // CH // CH + 2 * CH + 16)
                + c["kEvalSlots"]) + (k + 7) // 8 + 8


def msm_scratch_bytes(points: int, batch: int, c: int, W: int, n_phys: int = 1) -> int:
    """The MsmScratch one msm_launch_batch of `batch` MSMs of `points` points grows to (msm.cu): the histogram, bucket
    offsets and cursor, one 4-byte entry per digit, one XYZZ bucket (128 bytes) per bucket, the segment index, sums and
    order, the heavy-bucket list, the reduction tree (serial level of fan-in >= 4 plus the row and column sums) and the
    window sums."""
    src = md._msm_source()
    for buf in ("buckets.reserve(n_buckets * sizeof(g1_xyzz))", "seg_sums.reserve(max_segs * sizeof(g1_xyzz))",
                "entries.reserve(max_entries * 4)"):
        assert buf in src, f"msm.cu no longer reserves {buf}: restate msm_scratch_bytes"
    n_buckets = n_phys * (1 << (c - 1)) * batch
    n_windows = n_phys * batch
    entries = points * W * batch
    segs = entries // md.SEG_LEN + n_buckets
    heavy = segs // (md.COMBINE_SEQ + 1) + 2
    l_log = c // 2
    tree = (n_buckets >> 1) + n_windows * ((1 << l_log) + (1 << (c - 1 - l_log))) + 1
    return 4 * (5 * n_buckets + 2) + 4 * entries + 136 * segs + 4 * segs + 4 * heavy + 128 * (tree + 65 * n_windows) + 4096


def footprint_parts(log_n: int, k: int = 1, src: str = None, batch: bool = None, keys: int = 1) -> dict:
    """Bytes per allocation of one context that loaded the SRS (n + 3 powers), preprocessed `keys` keys and made k
    proofs in one prover call: `prove` (batch False, k = 1) or `prove_batch` (batch True; the default for k > 1), whose
    buffers are the context's batch set (`batch_*`: workspace, both NTT scratches and an MSM scratch of its own) beside
    the single prover's.  Elements are 32 bytes.  The MSM scratch is sized by the largest batched commitment: the NS
    selector commitments of preprocess, or the NW wire commitments of each proof."""
    batch = k > 1 if batch is None else batch
    c = constants(src)
    n = 1 << log_n
    m = cosets(log_n, c) * n
    NS, NW = c["NS"], c["NW"]
    fe = 32
    win = md.choose_window(n + 3, 0)
    W = md.num_windows(win)
    p = {
        # sel_coeffs, sig_coeffs, sig_evals, dom; ce_sel, ce_sig, coset_pts, l1_inv, cscale, cscale_inv; the wiring
        "key": keys * (((NS + 2 * NW + 1) * n + (NS + NW + 4) * m) * fe + NW * n * 4),
        "ntt_scratch": NS * m * fe,                                 # reserved by preprocess
        "domain": 3 * n * fe,                                       # twiddles both ways and the two coset tables
        "srs": W * (n + 3) * 64,                                    # one window table per window on an idle GPU
        "msm_scratch": max(msm_scratch_bytes(n, NS, win, W), msm_scratch_bytes(n + 3, NW, win, W)),
        # not an allocation of the library's: what a context measured beyond the allocations above (≈ 0.5 GiB at 2^20 …
        # 2^22 on an H100 80GB HBM3: the library's modules and the CUDA runtime's own reservations), rounded up
        "runtime": 1 << 30,
    }
    if batch:
        p["batch_workspace"] = workspace_elems(n, k, c) * fe
        p["batch_ntt_scratch"] = k * c["STAGE_PER_M"] * m * fe
        p["batch_ntt_scratch2"] = k * c["NSCR2_PER_M"] * m * fe
        p["batch_msm_scratch"] = msm_scratch_bytes(n + 3, k * NW, win, W)
    else:
        p["workspace"] = workspace_elems(n, 1, c) * fe
        p["ntt_scratch2"] = c["NSCR2_PER_M"] * m * fe
    return p


def footprint_bytes(log_n: int, k: int = 1, src: str = None, batch: bool = None, keys: int = 1) -> int:
    return sum(footprint_parts(log_n, k, src, batch, keys).values())


# ---- the circuit ------------------------------------------------------------------------------------------------------
@dataclass
class BigCircuit(synth.SynthCircuit):
    gate_rows: dict = field(default_factory=dict)    # row -> gate kind (GATE_KINDS) of every row with a gate
    boundary: dict = field(default_factory=dict)     # name -> (variable, sorted positions i * n + j) of the cycles placed
    stride_rows: np.ndarray = None                   # rows j whose five positions form one cycle (j, n + j, ..., 4n + j)


def scan_boundaries(log_n: int, ch: int = 16) -> list:
    """Rows 16^k (k >= 1) inside the domain: the chunk boundaries every level of the grand-product scan crosses."""
    out, b = [], ch
    while b < (1 << log_n):
        out.append(b)
        b *= ch
    return out


def gate_layout(log_n: int) -> dict:
    """row -> kind: 12 rows after the public inputs, 6 on each side of n/2 (rows n/2 - 7 … n/2 - 2, n/2 + 2 … n/2 + 7),
    the 7 rows n - 8 … n - 2; the kinds in turn, so that every group holds every kind."""
    n = 1 << log_n
    assert log_n >= 8
    rows = list(range(NUM_INPUTS, NUM_INPUTS + 12)) + list(range(n // 2 - 7, n // 2 - 1)) + \
        list(range(n // 2 + 2, n // 2 + 8)) + list(range(n - 8, n - 1))
    return {r: GATE_KINDS[i % len(GATE_KINDS)] for i, r in enumerate(rows)}


def random_fr(rng, count: int) -> np.ndarray:
    """(count, 4) canonical field elements, read as the Montgomery form of random values: top limb below r's."""
    out = rng.integers(0, 1 << 64, size=(count, 4), dtype=np.uint64)
    out[:, 3] %= np.uint64(R >> 192)
    return out


def to_int(limbs) -> int:
    return int.from_bytes(np.ascontiguousarray(limbs, dtype=np.uint64).tobytes(), "little") * RINV % R


def big_circuit(log_n: int, seed: int = 0) -> BigCircuit:
    """A satisfied circuit of domain 2^log_n with NUM_INPUTS public inputs, as wiring + witness vector and as table +
    permutation.  Variable 0 is the constant zero and 1 + p the variable first placed on position p = i * n + j; the
    copy cycles then move positions onto shared variables (later steps overwrite earlier ones):

    - random short cycles: a quarter of all positions in groups of 2 … 6;
    - stride-n cycles: a random eighth of the rows without gates, all five wires on one variable;
    - `bound_<b>`: all five wires of rows b - 1 and b for every b = 16^k in the domain;
    - `ends`: all five wires of rows 0, n/2 and n - 1 (where n/2 = 16^k the bound variable is this one);
    - each gate's output: w4 of its row, w0 of the next gate's row (the chain runs through every group of gate rows)
      and two random positions of rows without gates.

    Gate outputs are computed with Python integers; every other value is random."""
    n = 1 << log_n
    NW, P = synth.N_WIRES, synth.N_WIRES << log_n
    rng = np.random.default_rng(seed)
    rnd = random.Random(seed)
    gates = gate_layout(log_n)
    grows = sorted(gates)
    wv = np.arange(1, P + 1, dtype=np.uint32)   # flattened: position i * n + j
    num_vars = 1 + P

    def new_vars(count):
        nonlocal num_vars
        num_vars += count
        return np.arange(num_vars - count, num_vars, dtype=np.uint32)

    # the rows of the boundary cycles: ends on 0, n/2, n - 1; bound_b on b - 1 and b (ends itself where they meet)
    ends = int(new_vars(1)[0])
    special_rows = {0: ends, n // 2: ends, n - 1: ends}
    boundary = {}
    for b in scan_boundaries(log_n):
        v = ends if (b in special_rows or b - 1 in special_rows) else int(new_vars(1)[0])
        special_rows[b - 1] = special_rows[b] = v
        boundary[f"bound_{b}"] = v
    boundary["ends"] = ends
    taken = np.zeros(n, dtype=bool)
    taken[grows] = True
    taken[list(special_rows)] = True
    # random short cycles over a quarter of the positions
    pick = rng.choice(P, size=P // 4, replace=False)
    lens = rng.integers(2, 7, size=P // 8)
    starts = np.r_[0, np.cumsum(lens)]
    starts = starts[starts < len(pick)]
    group = np.searchsorted(starts, np.arange(len(pick)), side="right") - 1
    wv[pick] = wv[pick[starts]][group]
    # stride-n cycles on an eighth of the rows without gates or boundary cycles, a fresh variable each
    stride_rows = np.sort(rng.choice(np.flatnonzero(~taken), size=n // 8, replace=False))
    sv = new_vars(len(stride_rows))
    for i in range(NW):
        wv[i * n + stride_rows] = sv
    taken[stride_rows] = True
    for row, v in special_rows.items():
        wv[np.arange(NW) * n + row] = v
    # gate outputs: fresh variables, chained, each also on two positions of rows of none of the cycles above
    spare = np.flatnonzero(~taken)
    spots = rng.choice(NW * len(spare), size=2 * len(grows), replace=False)
    spots = (spots // len(spare)) * n + spare[spots % len(spare)]
    outs = {}
    for t, row in enumerate(grows):
        v = int(new_vars(1)[0])
        outs[row] = v
        wv[4 * n + row] = v
        wv[spots[2 * t: 2 * t + 2]] = v
        if t + 1 < len(grows):
            wv[grows[t + 1]] = v                # w0 of the next gate row
    witness = np.zeros((num_vars, 4), dtype=np.uint64)
    witness[1:] = random_fr(rng, num_vars - 1)
    # the gates, in row order (each gate's w0 is the previous gate's output)
    sel_int = {}
    wv2 = wv.reshape(NW, n)
    for row in grows:
        kind = gates[row]
        w = [to_int(witness[wv2[i, row]]) for i in range(4)]
        q = [0] * synth.N_SELECTORS
        q[synth.Q_O] = 1
        q[synth.Q_C] = rnd.randrange(R)
        if kind == "hash":
            for j in range(4):
                q[synth.Q_HASH + j] = rnd.randrange(R)
            res = q[synth.Q_C] + sum(q[synth.Q_HASH + j] * pow(w[j], 5, R) for j in range(4))
        elif kind == "lc":
            for j in range(4):
                q[synth.Q_LC + j] = rnd.randrange(R)
            res = q[synth.Q_C] + sum(q[synth.Q_LC + j] * w[j] for j in range(4))
        elif kind == "mul":
            q[synth.Q_MUL], q[synth.Q_MUL + 1] = rnd.randrange(R), rnd.randrange(R)
            res = q[synth.Q_C] + q[synth.Q_MUL] * w[0] * w[1] + q[synth.Q_MUL + 1] * w[2] * w[3]
        elif kind == "ecc":
            q[synth.Q_ECC], q[synth.Q_LC] = rnd.randrange(1, R), rnd.randrange(R)
            den = (q[synth.Q_O] - q[synth.Q_ECC] * w[0] * w[1] * w[2] * w[3]) % R
            assert den
            res = (q[synth.Q_C] + q[synth.Q_LC] * w[0]) * pow(den, -1, R)
        else:  # const: w4 = q_c
            res = q[synth.Q_C]
        sel_int[row] = q
        witness[outs[row]] = synth.to_mont_array([res % R])[0]
    selectors = np.zeros((synth.N_SELECTORS, n, 4), dtype=np.uint64)
    one = synth.to_mont_array([1])[0]
    selectors[synth.Q_O, :NUM_INPUTS] = one
    rows = np.array(grows)
    sel_mont = synth.to_mont_array([sel_int[r][s] for s in range(synth.N_SELECTORS) for r in grows])
    selectors[:, rows] = sel_mont.reshape(synth.N_SELECTORS, len(grows), 4)
    perm = wiring_permutation(wv)
    for name, v in boundary.items():
        boundary[name] = (v, np.flatnonzero(wv == v))
    return BigCircuit(
        log_n=log_n, num_inputs=NUM_INPUTS, k=synth.to_mont_array([pow(5, i, R) for i in range(NW)]), selectors=selectors,
        perm=perm, wires=witness[wv2], pub_inputs=witness[wv2[4, :NUM_INPUTS]], n_gates=n, selectors_int=None,
        wires_int=None, pub_inputs_int=None, wire_vars=wv2, witness=witness, gate_rows=gates, boundary=boundary,
        stride_rows=stride_rows)


def cycle_labels(perm: np.ndarray, max_len: int = 1 << 8) -> np.ndarray:
    """For every position, the smallest position of its cycle under perm (pointer doubling; cycles of at most max_len)."""
    lab = np.arange(len(perm), dtype=np.int64)
    step = np.asarray(perm, dtype=np.int64)
    reach = 1
    while reach < max_len:
        lab = np.minimum(lab, lab[step])
        step = step[step]
        reach *= 2
    assert (np.minimum(lab, lab[perm.astype(np.int64)]) == lab).all(), "a cycle longer than max_len"
    return lab


def variable_labels(wire_vars: np.ndarray) -> np.ndarray:
    """For every position, the smallest position that holds the same variable."""
    v = np.asarray(wire_vars).reshape(-1).astype(np.int64)
    first = np.full(int(v.max()) + 1, len(v), dtype=np.int64)
    np.minimum.at(first, v, np.arange(len(v)))
    return first[v]
