"""The 16-lane pairing arithmetic without a GPU: the fold of the high half of an Fq12 product that
`renegade_b200/csrc/pairing_warp.cuh` states as one linear map (lane j < 6: c_j = t_j - 82 h_j - 1476 h_(j+6); lane
j >= 6: c_j = t_j + 242 h_j + 18 h_(j-6), h_k = t_(12+k)) equals the sequential fold of `fq12_mul` on the Python pairing
oracle's field arithmetic; `b200_selftest_pairing` agrees across its header, the binding, a C compiler and the Rust
shim; and without a device it reports the missing device."""
import ctypes as C
import os
import random
import re
import subprocess
import sys

import pytest

import bn254_pairing_py as bp
from renegade_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q = bp.Q


def fold_constants():
    """(low own, low other, high own, high other) as the kernel header states them"""
    src = open(os.path.join(ROOT, "renegade_b200", "csrc", "pairing_warp.cuh")).read()
    m = re.search(r"constexpr int kFoldLowOwn = (-?\d+), kFoldLowOther = (-?\d+), kFoldHighOwn = (-?\d+), "
                  r"kFoldHighOther = (-?\d+);", src)
    assert m, "the fold constants are not in pairing_warp.cuh"
    return tuple(int(x) for x in m.groups())


def lane_fold(t):
    """The map of pairing_warp.cuh: lane j's output from its own t_j, h_j and its partner's h_(j +- 6)."""
    lo_own, lo_other, hi_own, hi_other = fold_constants()
    h = [t[12 + k] if 12 + k < len(t) else 0 for k in range(12)]  # h_11 = t_23 = 0
    return [(t[j] + lo_own * h[j] + lo_other * h[j + 6]) % Q if j < 6 else (t[j] + hi_own * h[j] + hi_other * h[j - 6]) % Q
            for j in range(12)]


def sequential_fold(t):
    """fq12_mul's fold: k = 22 down to 12, w^k = 18 w^(k-6) - 82 w^(k-12)"""
    t = list(t) + [0] * (23 - len(t))
    for k in range(22, 11, -1):
        t[k - 6] += 18 * t[k]
        t[k - 12] -= 82 * t[k]
    return [v % Q for v in t[:12]]


def lane_product(a, b):
    """The product as the lanes form it: lane j sums a_s b_((j - s) mod 12) over s = 0 .. 11 into t_j (s <= j) or
    t_(j+12) (s > j), 12 products on every lane, then the fold."""
    t = [0] * 24
    for j in range(12):
        for s in range(12):
            t[j if s <= j else j + 12] += a[s] * b[(j - s) % 12]
    return lane_fold(t[:23])


def _edges():
    yield [0] * 23
    yield [Q - 1] * 23
    for k in range(23):  # one term at a time: every column of the map
        yield [1 if i == k else 0 for i in range(23)]
        yield [Q - 1 if i == k else 0 for i in range(23)]


def test_fold_map_equals_the_sequential_fold():
    rng = random.Random(0xF01D)
    cases = list(_edges()) + [[rng.randrange(Q) for _ in range(23)] for _ in range(300)]
    cases += [[rng.choice((0, 1, Q - 1, rng.randrange(Q))) for _ in range(23)] for _ in range(300)]
    for t in cases:
        assert lane_fold(t) == sequential_fold(t), t


def test_lane_products_equal_the_oracle_product():
    """The split of the convolution and the fold together give the oracle's Fq12 product (its own sequential fold)."""
    rng = random.Random(0xA11CE)
    vals = [lambda: rng.randrange(Q), lambda: 0, lambda: 1, lambda: Q - 1]
    for it in range(200):
        a = [rng.choice(vals)() if it % 2 else rng.randrange(Q) for _ in range(12)]
        b = [rng.choice(vals)() for _ in range(12)]
        assert lane_product(a, b) == (bp.Fq12(a) * bp.Fq12(b)).c
    one = [1] + [0] * 11
    a = [rng.randrange(Q) for _ in range(12)]
    assert lane_product(a, one) == a and lane_product(one, one) == one and lane_product(a, [0] * 12) == [0] * 12


def test_lane_inverse_by_norms():
    """The inversion of pairing_warp.cuh: g = f conj(f) in Fq6, z = g g^(q^2) g^(q^4) in Fq + Fq w^6, and
    1 / (z0 + z6 w^6) = (z0 + 18 z6 - z6 w^6) / (z0^2 + 18 z0 z6 + 82 z6^2); checked against the oracle's inverse with the
    q^2-power map taken as exponentiation."""
    rng = random.Random(0x1417)
    conj = lambda x: bp.Fq12([(-v if k % 2 else v) for k, v in enumerate(x.c)])
    for _ in range(2):
        f = bp.Fq12([rng.randrange(Q) for _ in range(12)])
        g = f * conj(f)
        assert all(v == 0 for v in g.c[1::2])
        g2 = g ** (Q * Q)
        g24 = g2 * g2 ** (Q * Q)
        z = g * g24
        assert all(v == 0 for k, v in enumerate(z.c) if k % 6)
        z0, z6 = z.c[0], z.c[6]
        n = (z0 * z0 + 18 * z0 * z6 + 82 * z6 * z6) % Q
        ni = pow(n, Q - 2, Q)
        zi = bp.Fq12([(z0 + 18 * z6) * ni] + [0] * 5 + [-z6 * ni] + [0] * 5)
        assert conj(f) * g24 * zi == f.inv()


SELFTEST = ["ctx", "seed", "iters", "mismatches"]


def test_header_binding_compiler_and_shim_agree(tmp_path):
    _, structs, funcs, macros = _lib.parse_header(_lib.SELFTEST_HEADER)
    assert [name for name, _, _ in funcs] == _lib.SELFTEST_EXPORTS == ["b200_selftest_pairing"]
    assert not structs and not macros  # the core header's context type and error codes
    assert not set(_lib.SELFTEST_EXPORTS) & set(_lib.EXPORTS + _lib.SETTLEMENT_EXPORTS + _lib.VERIFY_JOB_EXPORTS +
                                                  _lib.EXPRESS_EXPORTS + _lib.RESERVED_EXPORTS)
    ret, args = funcs[0][1], funcs[0][2]
    assert ret == "int" and args == [("ctx", "b200_ctx *"), ("seed", "uint64_t"), ("iters", "size_t"),
                                     ("mismatches", "uint64_t *")]
    # the same signature as b200_selftest_field
    core = {name: a for name, _, a in _lib.parse_header()[2]}
    assert [t for _, t in core["b200_selftest_field"]] == [t for _, t in args]
    decls = [f"static {r} (*const p_{name})({', '.join(t for _, t in a)}) = {name};" for name, r, a in funcs]
    for includes in (['"b200selftest.h"'], ['"b200prover.h"', '"b200selftest.h"', '"b200verifyjobs.h"']):
        src = "".join(f"#include {h}\n" for h in includes) + "\n".join(decls) + "\n"
        (tmp_path / "t.c").write_text(src)
        r = subprocess.run(["gcc", "-std=c11", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c", str(tmp_path / "t.c"),
                            "-o", str(tmp_path / "t.o")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    lib = _lib.load()
    assert lib.b200_selftest_pairing.argtypes == [C.c_void_p, C.c_uint64, C.c_size_t, C.c_void_p]
    assert lib.b200_selftest_pairing.restype is C.c_int
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_rust_ffi as gen
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi_selftest.rs")).read()
    assert ffi == gen.generate(_lib.SELFTEST_HEADER), "ffi_selftest.rs is stale: run python tools/gen_rust_ffi.py"
    assert "pub fn b200_selftest_pairing(ctx: *mut b200_ctx, seed: u64, iters: usize, mismatches: *mut u64) -> c_int;" in ffi
    assert "pub mod ffi_selftest;" in open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()
    from renegade_b200.backend import Context
    assert callable(Context.selftest_pairing)


def test_reports_the_missing_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the missing-device path is the CPU container's")
    lib = _lib.load()
    bad = C.c_uint64(7)
    assert lib.b200_selftest_pairing(None, 1, 16, C.byref(bad)) == _lib.B200_ERR_NO_DEVICE
    assert bad.value == 7
    assert "no CUDA device" in lib.b200_last_error().decode()
