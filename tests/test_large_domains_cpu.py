"""The circuits of tests/large_domains.py on the host alone, before tests/test_gpu_large_domains.py proves them: every
gate holds, the copy permutation's cycles are exactly the variables' position sets, the boundary cycles sit on the
rows the generator names, the public inputs are the output wires of the first rows; at 2^10 the oracle proves and
verifies the circuit.  The memory estimate reads its constants from plonk.cu and msm.cu."""
import functools

import numpy as np
import pytest

import large_domains as ld
import msm_digits as md
from renegade_b200 import synth
from test_prove_witness_cpu import cycles
from test_witness_shapes_cpu import assert_gates_and_public_inputs, position_sets, to_int

SIZES = [10, 16, 20]


@functools.lru_cache(maxsize=1)
def circuit(log_n):
    return ld.big_circuit(log_n, seed=log_n)


@pytest.mark.parametrize("log_n", SIZES)
def test_gates_hold(log_n):
    circ = circuit(log_n)
    n, ni = circ.n, circ.num_inputs
    assert ni == 17 and circ.pub_inputs.shape == (ni, 4)
    assert (circ.wires == circ.witness[circ.wire_vars]).all()
    # gates on exactly the generator's rows and the public-input rows; everywhere else every selector is zero
    live = set(np.flatnonzero(circ.selectors.any(axis=(0, 2))).tolist())
    assert live == set(circ.gate_rows) | set(range(ni))
    assert_gates_and_public_inputs(circ)
    if log_n == 10:  # and the gate value on every row, the zero-selector rows included
        for j in range(n):
            q = [to_int(circ.selectors[s, j]) for s in range(synth.N_SELECTORS)]
            w = [to_int(circ.wires[i, j]) for i in range(synth.N_WIRES)]
            assert synth.gate_value(q, w, to_int(circ.pub_inputs[j]) if j < ni else 0) == 0, j
    # every kind in each group: after the public inputs, below n/2, above n/2, at the end
    groups = [range(ni, ni + 12), range(n // 2 - 7, n // 2 - 1), range(n // 2 + 2, n // 2 + 8), range(n - 8, n - 1)]
    for g in groups:
        assert {circ.gate_rows[r] for r in g} == set(ld.GATE_KINDS), g
    kinds = {"hash": synth.Q_HASH, "lc": synth.Q_LC, "mul": synth.Q_MUL, "ecc": synth.Q_ECC}
    for r, kind in circ.gate_rows.items():
        if kind in kinds:
            assert circ.selectors[kinds[kind], r].any(), (r, kind)
        assert circ.selectors[synth.Q_O, r].any() and circ.selectors[synth.Q_C, r].any()


@pytest.mark.parametrize("log_n", SIZES)
def test_cycles_are_the_variables(log_n):
    circ = circuit(log_n)
    n, wv = circ.n, circ.wire_vars
    perm = circ.perm.astype(np.int64)
    assert (np.sort(perm) == np.arange(5 * n)).all()
    assert (ld.cycle_labels(circ.perm) == ld.variable_labels(wv)).all()
    if log_n <= 16:  # the same by the set-based restatement
        assert cycles(circ.perm) == position_sets(wv)
    flat = wv.reshape(-1)
    counts = np.bincount(flat)
    # random short cycles and the gate outputs' cycles exist, and no cycle is longer than the boundary cycles
    assert (counts >= 2).sum() > n // 4 and counts.max() <= 20
    # stride-n: each chosen row's five positions are one variable that sits nowhere else
    sr = circ.stride_rows
    assert len(sr) == n // 8 and not set(sr.tolist()) & set(circ.gate_rows)
    for i in range(1, 5):
        assert (wv[i, sr] == wv[0, sr]).all()
    assert (counts[wv[0, sr]] == 5).all()


@pytest.mark.parametrize("log_n", SIZES)
def test_boundary_cycles(log_n):
    circ = circuit(log_n)
    n, flat = circ.n, circ.wire_vars.reshape(-1)
    rows = lambda *rr: sorted(i * n + r for i in range(5) for r in rr)  # noqa: E731
    bounds = ld.scan_boundaries(log_n)
    assert bounds == [16 ** k for k in range(1, (log_n - 1) // 4 + 1)]
    ends_rows = {0, n // 2, n - 1}
    for b in bounds:
        if b in ends_rows or b - 1 in ends_rows:
            ends_rows |= {b - 1, b}
    var, pos = circ.boundary["ends"]
    assert pos.tolist() == rows(*ends_rows) and (flat[pos] == var).all() and (flat == var).sum() == len(pos)
    for b in bounds:
        v, p = circ.boundary[f"bound_{b}"]
        assert (flat[rows(b - 1, b)] == v).all()  # rows 16^k - 1 and 16^k: one variable on all ten positions
        if v != var:
            assert p.tolist() == rows(b - 1, b) and (flat == v).sum() == 10
    # the public inputs: output wires of the first rows; row 0's is the ends variable, rows 15 and 16 share bound_16
    assert (circ.pub_inputs == circ.witness[circ.wire_vars[4, :circ.num_inputs]]).all()
    assert circ.wire_vars[4, 0] == var and circ.wire_vars[4, 15] == circ.wire_vars[4, 16]
    # the chain: each gate's output is w0 of the next gate row
    g = sorted(circ.gate_rows)
    assert all(circ.wire_vars[4, a] == circ.wire_vars[0, b] for a, b in zip(g, g[1:]))


def test_oracle_proves_2_10(oracle, pyoracle):
    py = pyoracle
    circ = circuit(10)
    tau = oracle.int_to_limbs(py.to_mont(0xB200B210 % py.R, py.R))
    srs = oracle.srs_from_tau(tau, circ.n + 3)
    opk = oracle.plonk_preprocess(10, circ.selectors, circ.perm, circ.k, srs)
    rc, proof, _, _ = oracle.plonk_prove(10, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs,
                                         synth.splitmix_blinders(0x210), srs)
    assert rc == 0
    assert oracle.plonk_verify_known_tau(10, circ.num_inputs, circ.k, opk, circ.pub_inputs, proof, tau)
    bad = circ.wires.copy()
    bad[1, circ.n - 1] = circ.wires[1, 0] + np.array([1, 0, 0, 0], dtype=np.uint64)  # the ends cycle broken at the wrap
    rc, _, _, _ = oracle.plonk_prove(10, circ.num_inputs, circ.k, opk, bad, circ.pub_inputs, synth.splitmix_blinders(1), srs)
    assert rc == 2


def test_footprint_reads_the_sources():
    src = ld.plonk_source()
    c = ld.constants(src)
    assert (c["NW"], c["NS"], c["CH"], c["COSET_SWITCH"], c["COSETS_LARGE"], c["COSETS_SMALL"]) == (5, 13, 16, 4, 6, 8)
    n = 1 << 20
    m = 6 * n
    base = ld.footprint_parts(20, src=src)
    # one more selector column: n + m more key elements (coefficients, coset evaluations), m more NTT scratch, and a
    # batched selector commitment of 14 MSMs
    more_ns = ld.footprint_parts(20, src=src.replace("constexpr int NS = 13;", "constexpr int NS = 14;"))
    assert more_ns["key"] - base["key"] == 32 * (n + m) and more_ns["ntt_scratch"] - base["ntt_scratch"] == 32 * m
    win = md.choose_window(n + 3, 0)
    assert more_ns["msm_scratch"] == ld.msm_scratch_bytes(n, 14, win, md.num_windows(win)) > base["msm_scratch"]
    # one more quotient coset: every m-sized allocation grows by n
    more_cosets = ld.footprint_parts(20, src=src.replace("const int nc = log_n >= 4 ? 6 : 8;", "const int nc = log_n >= 4 ? 7 : 8;"))
    per_m = {"key": c["NS"] + c["NW"] + 4, "ntt_scratch": c["NS"], "ntt_scratch2": c["NSCR2_PER_M"]}
    for part, count in per_m.items():
        assert more_cosets[part] - base[part] == 32 * count * n, part
    with pytest.raises(AssertionError):
        ld.constants(src.replace("ntt_scratch.reserve((size_t)NS * m", "ntt_scratch.reserve((size_t)NW * m"))
    # the MSM scratch follows the digit count: 2^20 points at c = 20 (13 windows) in 13 MSMs, entries and segments
    entries = n * 13 * 13
    assert ld.msm_scratch_bytes(n, 13, 20, 13) >= 4 * entries + 136 * (entries // md.SEG_LEN) + 128 * 13 * (1 << 19)
    # a batch adds its own buffers: k workspaces, both NTT scratches and the MSM scratch of k NW commitments
    b2 = ld.footprint_parts(20, 2, src=src)
    assert b2["batch_ntt_scratch"] == 2 * c["STAGE_PER_M"] * m * 32 and b2["batch_ntt_scratch2"] == 2 * c["NSCR2_PER_M"] * m * 32
    assert "workspace" not in b2 and b2["batch_workspace"] == 32 * ld.workspace_elems(n, 2, c)
    # ≈ 14 KB per row: 2^22 fits an 80 GB H100 with 15 % to spare, 2^23 does not fit at all
    assert ld.footprint_bytes(22) * 1.15 < 80e9 < ld.footprint_bytes(23)
