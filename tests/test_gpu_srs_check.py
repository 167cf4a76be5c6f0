"""b200_srs_check on the device: the reference's 512-point head and the seeded 2^16 + 3 SRS pass; every way of
replacing one power (doubled, negated, its neighbour, a power of another tau) at the first, a middle and the last index
fails the combined check and is located at exactly the pairs that contain it; a wrong tau H or a swapped pair fails
every pair; G2 points outside the subgroup, G2 records off the twist and G1 records off the curve are reported; the
report depends neither on the seed nor on the window plan; the edges of n; and proofs made on a context before and
after a check are byte-identical, with the prover's rounds replayed as graphs.  Every ptau file is built here: the
reference's header and section 1, section 2 declared at the size of its records, and section 3 holding the G2 pair."""
import ctypes as C
import struct

import numpy as np
import pytest

import bn254_pairing_py as pr
import bn254_py as py
import renegade_b200 as rb
from renegade_b200 import _lib
from renegade_b200 import circuit_types as ct
from test_srs_check_cpu import random_twist_point

pytestmark = pytest.mark.gpu

OTHER_TAU = 0x2E1F0D3C4B5A69788796A5B4C3D2E1F00F1E2D3C4B5A6978


def ptau(header80: bytes, points: np.ndarray, h, beta_h) -> bytes:
    recs = np.ascontiguousarray(points, dtype=np.uint64).tobytes()
    g2 = np.ascontiguousarray(h, dtype=np.uint64).tobytes() + np.ascontiguousarray(beta_h, dtype=np.uint64).tobytes()
    return header80[:68] + struct.pack("<IQ", 2, len(recs)) + recs + struct.pack("<IQ", 3, len(g2)) + g2


def head_points(srs_head) -> np.ndarray:
    return np.frombuffer(srs_head[80:80 + 512 * 64], dtype=np.uint64).reshape(512, 8).copy()


def seeded_points(srs_2_16) -> np.ndarray:
    return np.frombuffer(srs_2_16[80:], dtype=np.uint64).reshape(-1, 8).copy()


def check(ctx, pts, h, beta_h, n=None, seed=b"\x01" * 32, locate=True, window_bits=0, check_on_curve=True):
    bases = ctx.load_bases(pts, window_bits=window_bits, check_on_curve=check_on_curve)
    try:
        return rb.check_srs(ctx, bases, h, beta_h, n=n, seed=seed, locate=locate)
    finally:
        bases.free()


def g1_neg(p):
    y = sum(int(p[4 + i]) << (64 * i) for i in range(4))
    ny = (py.Q - y) % py.Q
    return np.concatenate([p[:4], np.array([(ny >> (64 * i)) & (2**64 - 1) for i in range(4)], dtype=np.uint64)])


def g1_dbl(oracle, p):
    out, inf = oracle.g1_add(p, 0, p, 0)
    assert not inf
    return out


def g2_rec(pt) -> np.ndarray:
    return np.frombuffer(pr.encode_g2_mont(pt), dtype=np.uint64).copy()


def expected_pairs(j, n):
    return [i for i in (j - 1, j) if 0 <= i <= n - 2]


# ---- 1. valid SRSs, through the ptau file -------------------------------------------------------------------------------
def test_reference_head_and_seeded_srs_are_valid(ctx, srs_head, g2_raw, srs_2_16, srs_2_16_g2):
    for pts, (h, bh) in ((head_points(srs_head), g2_raw), (seeded_points(srs_2_16), srs_2_16_g2)):
        data = ptau(srs_head, pts, h, bh)
        params = rb.parse_ptau_file(ctx, data, count=pts.shape[0])
        assert (params.h == h).all() and (params.beta_h == bh).all()
        rep = rb.check_srs(ctx, params.powers_of_g, params.h, params.beta_h)
        assert rep == rb.SrsReport(True, True, True, 0, []) and rep.valid
        params.powers_of_g.free()


def test_system_srs_from_ptau(ctx, srs_head, g2_raw, srs_2_16, srs_2_16_g2):
    saved = ct._SYSTEM_SRS
    try:
        pts = seeded_points(srs_2_16)
        s = ct.SystemSrs.from_ptau(ctx, ptau(srs_head, pts, *srs_2_16_g2), count=pts.shape[0])
        assert ct.system_srs() is s and len(s.powers_of_g) == pts.shape[0]
        assert (s.g2_h == srs_2_16_g2[0]).all() and (s.g2_tau_h == srs_2_16_g2[1]).all()
        # the head's powers with the seeded SRS's G2 pair: refused, and the installed SRS stays
        with pytest.raises(ct.ProverError) as e:
            ct.SystemSrs.from_ptau(ctx, ptau(srs_head, head_points(srs_head), *srs_2_16_g2), count=512)
        assert e.value.kind == "Srs" and not e.value.detail.consistent and e.value.detail.n_bad == 511
        assert ct.system_srs() is s
        # check=False installs whatever the file holds
        s2 = ct.SystemSrs.from_ptau(ctx, ptau(srs_head, head_points(srs_head), *srs_2_16_g2), count=512, check=False)
        assert ct.system_srs() is s2
    finally:
        ct._SYSTEM_SRS = saved


# ---- 2. one power replaced ----------------------------------------------------------------------------------------------
def test_one_replaced_power_is_located(ctx, oracle, srs_2_16, srs_2_16_g2):
    pts = seeded_points(srs_2_16)
    n = pts.shape[0]
    h, bh = srs_2_16_g2
    other = oracle.srs_from_tau(oracle.int_to_limbs(py.to_mont(OTHER_TAU % py.R, py.R)), n)
    for j in (0, n // 2, n - 1):
        variants = {"double": g1_dbl(oracle, pts[j]), "negate": g1_neg(pts[j]),
                    "neighbour": pts[j + 1] if j < n - 1 else pts[j - 1]}
        if j >= 1:
            variants["other_tau"] = other[j]
        for name, p in variants.items():
            bad = pts.copy()
            bad[j] = p
            rep = check(ctx, bad, h, bh)
            want = expected_pairs(j, n)
            assert not rep.consistent and rep.n_bad == len(want) and rep.bad == want, (j, name, rep)
            assert rep.g1_generator == (j != 0) and rep.g2_subgroup, (j, name)
            assert not rep.valid


# ---- 3. the wrong G2 pair -----------------------------------------------------------------------------------------------
def test_wrong_tau_h_or_swapped_pair_fails_every_pair(ctx, srs_head, g2_raw):
    pts = head_points(srs_head)
    h, bh = g2_raw
    wrong = g2_rec(pr.g2_mul(pr.decode_g2_mont(h.tobytes(), 0), OTHER_TAU % pr.R))
    for hh, bb in ((h, wrong), (bh, h)):
        rep = check(ctx, pts, hh, bb)
        assert not rep.consistent and rep.n_bad == 511 and rep.bad == list(range(8)), rep
        assert rep.g1_generator and rep.g2_subgroup
    # without locate the failed check is reported alone
    rep = check(ctx, pts, h, wrong, locate=False)
    assert not rep.consistent and rep.n_bad == 0 and rep.bad == []


# ---- 4. points outside the groups -----------------------------------------------------------------------------------------
def test_points_outside_the_groups(ctx, srs_head, g2_raw):
    import random
    pts = head_points(srs_head)
    h, bh = g2_raw
    full_order = g2_rec(random_twist_point(random.Random(0x7157)))
    assert not rb.backend.g2_in_subgroup(full_order)
    rep = check(ctx, pts, h, full_order)
    assert not rep.g2_subgroup and not rep.consistent and not rep.valid
    rep = check(ctx, pts, h, full_order, n=1)
    assert not rep.g2_subgroup and rep.consistent and rep.g1_generator
    # a G2 record off the twist
    off = bh.copy()
    off[0] ^= 1
    bases = ctx.load_bases(pts)
    for a, b in ((h, off), (off, bh)):
        with pytest.raises(_lib.B200Error) as e:
            rb.check_srs(ctx, bases, a, b)
        assert e.value.code == _lib.B200_ERR_NOT_ON_CURVE
    bases.free()
    # a G1 record off the curve, loaded unchecked: the pairs that contain it
    for j in (0, 200, 511):
        bad = pts.copy()
        bad[j, 4] ^= 1
        rep = check(ctx, bad, h, bh, check_on_curve=False)
        assert not rep.consistent and rep.bad == expected_pairs(j, 512) and rep.n_bad == len(rep.bad), (j, rep)


# ---- 5. seed and window plan --------------------------------------------------------------------------------------------
def test_report_does_not_depend_on_seed_or_window_plan(ctx, oracle, srs_head, g2_raw):
    pts = head_points(srs_head)
    h, bh = g2_raw
    bad = pts.copy()
    bad[100] = g1_dbl(oracle, pts[100])
    bad[300] = g1_neg(pts[300])
    for p, want in ((pts, rb.SrsReport(True, True, True, 0, [])),
                    (bad, rb.SrsReport(False, True, True, 4, [99, 100, 299, 300]))):
        for seed in (bytes(32), b"\xff" * 32, bytes(range(32))):
            for wb in (0, 1, 13):
                assert check(ctx, p, h, bh, seed=seed, window_bits=wb) == want, (seed, wb)
        assert check(ctx, p, h, bh, seed=None) == want  # a fresh random seed


# ---- 6. edges of n ------------------------------------------------------------------------------------------------------
def test_edges_of_n(ctx, oracle, srs_head, g2_raw):
    pts = head_points(srs_head)
    h, bh = g2_raw
    bases = ctx.load_bases(pts)
    for n in (1, 2, 3, 511, 512):
        assert rb.check_srs(ctx, bases, h, bh, n=n) == rb.SrsReport(True, True, True, 0, []), n
    for n in (0, 513):
        with pytest.raises(_lib.B200Error) as e:
            rb.check_srs(ctx, bases, h, bh, n=n)
        assert e.value.code == _lib.B200_ERR_INVALID
    lib, rep = ctx._lib, _lib.STRUCTS["b200_srs_report"]()
    hp, bp = h.ctypes.data, bh.ctypes.data
    seed = bytes(32)
    assert lib.b200_srs_check(None, bases._h, 4, hp, bp, seed, 1, C.byref(rep)) == _lib.B200_ERR_INVALID
    assert lib.b200_srs_check(ctx._h, None, 4, hp, bp, seed, 1, C.byref(rep)) == _lib.B200_ERR_INVALID
    assert lib.b200_srs_check(ctx._h, bases._h, 4, None, bp, seed, 1, C.byref(rep)) == _lib.B200_ERR_INVALID
    assert lib.b200_srs_check(ctx._h, bases._h, 4, hp, None, seed, 1, C.byref(rep)) == _lib.B200_ERR_INVALID
    assert lib.b200_srs_check(ctx._h, bases._h, 4, hp, bp, None, 1, C.byref(rep)) == _lib.B200_ERR_INVALID
    assert lib.b200_srs_check(ctx._h, bases._h, 4, hp, bp, seed, 1, None) == _lib.B200_ERR_INVALID
    bases.free()
    # a wrong P_0: n = 1 sees the generator only; a bad power past n is not looked at
    bad = pts.copy()
    bad[0] = g1_dbl(oracle, pts[0])
    assert check(ctx, bad, h, bh, n=1) == rb.SrsReport(True, False, True, 0, [])
    bad = pts.copy()
    bad[400] = g1_neg(pts[400])
    assert check(ctx, bad, h, bh, n=400) == rb.SrsReport(True, True, True, 0, [])
    assert check(ctx, bad, h, bh, n=401) == rb.SrsReport(False, True, True, 1, [399])


# ---- 7. proving around a check ------------------------------------------------------------------------------------------
def test_proofs_around_a_check_are_identical(srs_2_16, srs_2_16_g2):
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark
    c = rb.Context(0)
    try:
        pts = seeded_points(srs_2_16)
        h, bh = srs_2_16_g2
        bases = c.load_bases(pts)
        log_n = 10
        circ = synth.synth_circuit(log_n, num_inputs=3, seed=5, check=True)
        pk = PlonkKzgSnark.preprocess(c, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        bl = synth.splitmix_blinders(3)

        def prove():
            proof, _ = PlonkKzgSnark.prove_with_link_hint(c, pk, circ.wires, circ.pub_inputs, bl)
            return bytes(proof)

        g0 = c.graph_launches()
        before = [prove(), prove(), prove()]  # eager, captured, replayed
        c.msm_timing(True)
        c.msm_timing_totals(reset=True)
        rep = rb.check_srs(c, bases, h, bh)
        totals = c.msm_timing_totals()
        c.msm_timing(False)
        assert rep.valid
        assert totals["launches"] == 1 and totals["pairs"] == 2 * pts.shape[0]  # one batch-2 MSM over all the powers
        g1 = c.graph_launches()
        after = [prove(), prove(), prove()]
        assert c.graph_launches() > g1 > g0  # the rounds ran as graphs on both sides of the check
        assert all(p == before[0] for p in before + after)
        # a failing check with its locate pass in between, too
        rep = rb.check_srs(c, bases, bh, h)
        assert rep.n_bad == pts.shape[0] - 1
        assert prove() == before[0]
        pk.free()
        bases.free()
    finally:
        c.close()


# ---- 8. the prover service's --check-srs ----------------------------------------------------------------------------------
def _service(tmp_path, data: bytes, g2=None):
    """Starts the example prover service with --check-srs on `data` (and --g2 when given); -> the running process."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    srs = tmp_path / "srs.ptau"
    srs.write_bytes(data)
    cmd = [sys.executable, "-m", "host_circuits.service_routes", "--port", "0", "--password", "pw", "--srs", str(srs),
           "--workers", "1", "--check-srs"]
    if g2 is not None:
        (tmp_path / "g2.bin").write_bytes(np.concatenate(g2).astype(np.uint64).tobytes())
        cmd += ["--g2", str(tmp_path / "g2.bin")]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "examples")]))
    return subprocess.Popen(cmd, cwd=root, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)


def _first_lines(proc, want: str, limit_s: float = 300):
    """stdout lines up to the first that contains `want` (all of them if the process ends first); the process is
    killed after `limit_s` seconds."""
    import threading
    watchdog = threading.Timer(limit_s, proc.kill)
    watchdog.start()
    lines = []
    try:
        for line in proc.stdout:
            lines.append(line)
            if want in line:
                break
    finally:
        watchdog.cancel()
    return lines


def test_service_check_srs_flag(tmp_path, srs_head, g2_raw, srs_2_16, srs_2_16_g2):
    pts = seeded_points(srs_2_16)
    # the seeded powers with the reference's G2 pair in section 3: refused before serving
    proc = _service(tmp_path, ptau(srs_head, pts, *g2_raw))
    try:
        _, err = proc.communicate(timeout=300)
    finally:
        proc.kill()
        proc.wait()
    assert proc.returncode != 0 and "--check-srs" in err and "consistent=False" in err, err[-2000:]
    # the right pair in section 3, a wrong one in --g2: --g2 is the pair checked
    proc = _service(tmp_path, ptau(srs_head, pts, *srs_2_16_g2), g2=g2_raw)
    try:
        _, err = proc.communicate(timeout=300)
    finally:
        proc.kill()
        proc.wait()
    assert proc.returncode != 0 and "--check-srs" in err, err[-2000:]
    # a consistent SRS, its pair from section 3: the check passes and the service goes on to its keys
    proc = _service(tmp_path, ptau(srs_head, pts, *srs_2_16_g2))
    try:
        lines = _first_lines(proc, "SRS checked")
    finally:
        proc.kill()
        proc.communicate()
    assert lines and "SRS checked: 16387 powers" in lines[-1], "".join(lines)
