"""The SRS check, the parts that need no GPU: `b200_srs_parse_ptau_g2` on synthetic ptau files (every way the file can
fail), `b200_g2_in_subgroup` against a [r]Q == O restated here over the oracle's twist arithmetic, Python's
parse_ptau_file on the truncated files it has always accepted, and the header, the binding and the Rust shim agreeing
on the three new entry points and `b200_srs_report`."""
import ctypes as C
import os
import random
import re
import struct

import numpy as np
import pytest

import bn254_pairing_py as pr
from renegade_b200 import _lib, backend

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the reference's SRS file, where a checkout of it is at hand (never on a machine without one)
REFERENCE_SRS = os.environ.get("B200_REFERENCE_SRS", "/root/reference/srs/srs00")
FORMAT, NOT_ON_CURVE, INVALID = _lib.B200_ERR_FORMAT, _lib.B200_ERR_NOT_ON_CURVE, _lib.B200_ERR_INVALID


def golden(name):
    with open(os.path.join(ROOT, "tests", "golden", name), "rb") as f:
        return f.read()


def ptau(records: bytes, g2: bytes | None, sec2_size=None, sec3_id=3, sec3_size=None) -> bytes:
    """header and section 1 of the reference's file, section 2 (declared size: the records'), then section 3 holding
    `g2` (None: the file ends after section 2)."""
    head = golden("srs_head.bin")[:68]
    out = head + struct.pack("<IQ", 2, len(records) if sec2_size is None else sec2_size) + records
    if g2 is not None:
        out += struct.pack("<IQ", sec3_id, len(g2) if sec3_size is None else sec3_size) + g2
    return out


def head_records(k=512) -> bytes:
    return golden("srs_head.bin")[80:80 + 64 * k]


def parse_g2(data: bytes):
    lib = _lib.load()
    h, bh = np.zeros(16, dtype=np.uint64), np.zeros(16, dtype=np.uint64)
    rc = lib.b200_srs_parse_ptau_g2(data, len(data), h.ctypes.data_as(C.c_void_p), bh.ctypes.data_as(C.c_void_p))
    return rc, h, bh


def in_subgroup_lib(rec: bytes):
    out = C.c_int(-1)
    r = np.frombuffer(rec, dtype=np.uint64).copy()
    rc = _lib.load().b200_g2_in_subgroup(r.ctypes.data_as(C.c_void_p), C.byref(out))
    return rc, out.value


# ---- the twist over the oracle's Fq2 arithmetic, with the identity (None) ---------------------------------------------
def g2_add(p, q):
    if p is None:
        return q
    if q is None:
        return p
    if p[0] == q[0]:
        if p[1] != q[1] or p[1] == (0, 0):
            return None
        m = pr._fq2_div(pr._fq2_mul((3, 0), pr._fq2_mul(p[0], p[0])), pr._fq2_mul((2, 0), p[1]))
    else:
        m = pr._fq2_div(pr._fq2_sub(q[1], p[1]), pr._fq2_sub(q[0], p[0]))
    x = pr._fq2_sub(pr._fq2_sub(pr._fq2_mul(m, m), p[0]), q[0])
    return x, pr._fq2_sub(pr._fq2_mul(m, pr._fq2_sub(p[0], x)), p[1])


def g2_mul(p, k):
    acc = None
    for bit in bin(k)[2:]:
        acc = g2_add(acc, acc)
        if bit == "1":
            acc = g2_add(acc, p)
    return acc


def oracle_in_subgroup(p) -> bool:
    return p is not None and g2_mul(p, pr.R) is None


def fq_sqrt(a):
    """sqrt in Fq (q = 3 mod 4), or None"""
    s = pow(a, (pr.Q + 1) // 4, pr.Q)
    return s if s * s % pr.Q == a % pr.Q else None


def fq2_sqrt(a):
    """sqrt of a0 + a1 u in Fq2 = Fq[u]/(u^2 + 1), or None: with n = sqrt(a0^2 + a1^2), x0^2 = (a0 +- n) / 2 and
    x1 = a1 / (2 x0)"""
    a0, a1 = a
    n = fq_sqrt((a0 * a0 + a1 * a1) % pr.Q)
    if n is None:
        return None
    inv2 = pow(2, -1, pr.Q)
    for cand in ((a0 + n) * inv2 % pr.Q, (a0 - n) * inv2 % pr.Q):
        x0 = fq_sqrt(cand)
        if x0:
            x = (x0, a1 * pow(2 * x0, -1, pr.Q) % pr.Q)
            if pr._fq2_mul(x, x) == (a0 % pr.Q, a1 % pr.Q):
                return x
    return None


TWIST_B = (27 * pow(82, -1, pr.Q) % pr.Q, -3 * pow(82, -1, pr.Q) % pr.Q)  # 3 / (9 + u)


def random_twist_point(rng):
    while True:
        x = (rng.randrange(pr.Q), rng.randrange(pr.Q))
        rhs = pr._fq2_mul(pr._fq2_mul(x, x), x)
        rhs = ((rhs[0] + TWIST_B[0]) % pr.Q, (rhs[1] + TWIST_B[1]) % pr.Q)
        y = fq2_sqrt(rhs)
        if y is not None:
            assert pr.g2_is_on_curve((x, y))
            return x, y


# ---- b200_srs_parse_ptau_g2 -------------------------------------------------------------------------------------------
def test_parse_g2_returns_section_3():
    g2 = golden("srs_g2.bin")
    rc, h, bh = parse_g2(ptau(head_records(), g2))
    assert rc == _lib.B200_OK, _lib.load().b200_last_error()
    assert h.tobytes() == g2[:128] and bh.tobytes() == g2[128:]
    # section 3 longer than its first two records (the reference's holds 2^17 G2 powers): the first two are read
    rc, h, bh = parse_g2(ptau(head_records(3), g2 + bytes(128), sec3_size=1 << 24))
    assert rc == _lib.B200_OK and h.tobytes() == g2[:128] and bh.tobytes() == g2[128:]
    # an empty section 2
    rc, h, _ = parse_g2(ptau(b"", g2))
    assert rc == _lib.B200_OK and h.tobytes() == g2[:128]
    # Python
    h, bh = backend.read_ptau_g2(ptau(head_records(), g2))
    assert h.tobytes() == g2[:128] and bh.tobytes() == g2[128:]


@pytest.mark.parametrize("case", ["no_section_3", "header_cut", "records_cut", "one_record", "wrong_section",
                                  "section_3_short", "section_2_leaves", "section_2_huge", "section_2_one_past"])
def test_parse_g2_format_errors(case):
    g2 = golden("srs_g2.bin")
    recs = head_records(16)
    data = {
        "no_section_3": ptau(recs, None),
        "header_cut": ptau(recs, g2)[:68 + 12 + len(recs) + 7],
        "records_cut": ptau(recs, g2)[:-1],
        "one_record": ptau(recs, g2[:128]),
        "wrong_section": ptau(recs, g2, sec3_id=4),
        "section_3_short": ptau(recs, g2, sec3_size=255),
        "section_2_leaves": ptau(recs, g2, sec2_size=len(recs) + 12 + 256 + 64),
        "section_2_huge": ptau(recs, g2, sec2_size=(1 << 64) - 1),
        "section_2_one_past": ptau(recs, None, sec2_size=len(recs) + 1),
    }[case]
    rc, _, _ = parse_g2(data)
    assert rc == FORMAT, case
    with pytest.raises(_lib.B200Error) as e:
        backend.read_ptau_g2(data)
    assert e.value.code == FORMAT


def test_parse_g2_header_checks_and_curve():
    g2 = golden("srs_g2.bin")
    good = ptau(head_records(4), g2)
    assert parse_g2(b"PTAU" + good[4:])[0] == FORMAT
    assert parse_g2(good[:4] + struct.pack("<I", 2) + good[8:])[0] == FORMAT  # version
    assert parse_g2(good[:30])[0] == FORMAT
    # beta_h off the twist, and h with a coordinate >= q (x0 + q: the same residue, not a canonical encoding)
    bad = bytearray(g2)
    bad[128] ^= 1
    assert parse_g2(ptau(head_records(4), bytes(bad)))[0] == NOT_ON_CURVE
    x0 = int.from_bytes(g2[:32], "little") + pr.Q
    if x0 < 1 << 256:
        assert parse_g2(ptau(head_records(4), x0.to_bytes(32, "little") + g2[32:]))[0] == NOT_ON_CURVE
    lib = _lib.load()
    assert lib.b200_srs_parse_ptau_g2(None, 0, None, None) == INVALID


# ---- b200_g2_in_subgroup ----------------------------------------------------------------------------------------------
def test_g2_subgroup_agrees_with_the_oracle():
    rng = random.Random(0x5B5)
    g2 = golden("srs_g2.bin")
    h = pr.decode_g2_mont(g2, 0)
    points = [h, pr.decode_g2_mont(g2, 1)]
    points += [pr.g2_mul(h, rng.randrange(1, pr.R)) for _ in range(3)]
    outside = [random_twist_point(rng) for _ in range(3)]
    points += outside
    cofactor = 2 * pr.Q - pr.R  # #E'(Fq2) = r (2q - r): clearing it lands in the subgroup
    points += [g2_mul(outside[0], cofactor)]
    want = [True] * 5 + [False] * 3 + [True]
    for p, w in zip(points, want):
        assert oracle_in_subgroup(p) == w
        rc, got = in_subgroup_lib(pr.encode_g2_mont(p))
        assert rc == _lib.B200_OK and got == int(w)
        assert backend.g2_in_subgroup(np.frombuffer(pr.encode_g2_mont(p), dtype=np.uint64)) == w
    # the identity (all zero) is not in the subgroup; a record off the twist is an error
    assert in_subgroup_lib(bytes(128)) == (_lib.B200_OK, 0)
    bad = bytearray(g2[:128])
    bad[0] ^= 1
    assert in_subgroup_lib(bytes(bad))[0] == NOT_ON_CURVE
    assert _lib.load().b200_g2_in_subgroup(None, None) == INVALID


# ---- parse_ptau_file on the files it already accepts ------------------------------------------------------------------
class _Ctx:
    """Stands in for a Context: records what parse_ptau_file would load on the device."""

    def load_bases(self, points, window_bits=0, check_on_curve=False):
        self.loaded = np.array(points)
        return "bases"


def test_parse_ptau_file_keeps_truncated_files():
    head = golden("srs_head.bin")  # the reference's header and 512 powers, section 2 declared at full size
    ctx = _Ctx()
    params = backend.parse_ptau_file(ctx, head, count=512)
    assert params.h is None and params.beta_h is None and params.powers_of_g == "bases"
    assert ctx.loaded.tobytes() == head[80:80 + 512 * 64]
    g2 = golden("srs_g2.bin")
    params = backend.parse_ptau_file(ctx, ptau(head_records(), g2), count=512)
    assert params.h.tobytes() == g2[:128] and params.beta_h.tobytes() == g2[128:]
    # bytes after section 2 that are not section 3 were accepted before and still are, without a G2 pair
    params = backend.parse_ptau_file(ctx, ptau(head_records(), g2, sec3_id=4), count=512)
    assert params.h is None


# ---- the boundary -----------------------------------------------------------------------------------------------------
NEW = {
    "b200_srs_parse_ptau_g2": ["bytes", "len", "g2_h", "g2_tau_h"],
    "b200_g2_in_subgroup": ["rec", "in_subgroup"],
    "b200_srs_check": ["ctx", "srs", "n", "g2_h", "g2_tau_h", "seed", "locate", "out"],
}


def test_header_binding_and_shim_agree():
    _, structs, funcs, _ = _lib.parse_header()
    sig = {name: (ret, args) for name, ret, args in funcs}
    for name, args in NEW.items():
        assert name in _lib.EXPORTS
        assert sig[name][0] == "int" and [a for a, _ in sig[name][1]] == args, name
    assert dict(sig["b200_srs_check"][1])["out"] == "b200_srs_report *"
    assert dict(sig["b200_srs_check"][1])["seed"] == "const uint8_t *"
    assert structs["b200_srs_report"] == [("consistent", "uint64_t", ()), ("g1_generator", "uint64_t", ()),
                                          ("g2_subgroup", "uint64_t", ()), ("n_bad", "uint64_t", ()),
                                          ("bad", "uint64_t", (8,))]
    assert C.sizeof(_lib.STRUCTS["b200_srs_report"]) == 12 * 8
    assert len(_lib.EXPORTS) == 110
    lib = _lib.load()
    assert lib.b200_srs_check.argtypes == [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                           C.c_void_p]
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi.rs")).read()
    for name in NEW:
        assert re.search(rf"pub fn {name}\(", ffi), name
    assert re.search(r"pub struct b200_srs_report \{\s*pub consistent: u64,", ffi)
    shim = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()
    assert "pub fn parse_ptau_g2" in shim and "ffi::b200_srs_parse_ptau_g2(" in shim
    assert "pub fn check_srs" in shim and "ffi::b200_srs_check(" in shim


def test_srs_check_refuses_null_arguments_without_a_device():
    lib = _lib.load()
    rep = _lib.STRUCTS["b200_srs_report"]()
    z = np.zeros(16, dtype=np.uint64)
    p = z.ctypes.data_as(C.c_void_p)
    assert lib.b200_srs_check(None, None, 1, p, p, bytes(32), 1, C.byref(rep)) == INVALID
    assert lib.b200_srs_check(None, None, 1, None, None, None, 1, None) == INVALID


@pytest.mark.skipif(not os.path.exists(REFERENCE_SRS), reason="the reference's SRS file is not at hand")
def test_reference_section_3_is_the_golden_g2_pair():
    with open(REFERENCE_SRS, "rb") as f:
        data = f.read()
    rc, h, bh = parse_g2(data)
    assert rc == _lib.B200_OK
    assert h.tobytes() + bh.tobytes() == golden("srs_g2.bin")
    assert in_subgroup_lib(h.tobytes()) == (_lib.B200_OK, 1) and in_subgroup_lib(bh.tobytes()) == (_lib.B200_OK, 1)
