"""CPU: the host-side field arithmetic of the library (the host branches of renegade_b200/csrc/ff.cuh), built with g++
from the header's host path.
  * the division-step inversion (`fe_inv_safegcd` — Bernstein-Yang division steps, 62 at a time; on the prover's critical
    path in the affine normalisation of every commitment batch, and ~130 times per pairing) against the Fermat ladder and
    the binary Euclid, for Fq and Fr (tests/host_inverse_check.cpp);
  * the 64-bit CIOS product, add, sub, square and the fused a*b +- c*d against Python integers on the edge operands of
    tests/field_edges.py (tests/host_field_check.cpp)."""
import os
import subprocess

import numpy as np
import pytest

import field_edges as fx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _compile(src: str, exe) -> None:
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "renegade_b200", "csrc"),
                           "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", src), "-o", str(exe)])


def test_safegcd_inverse_matches_fermat_and_euclid(tmp_path):
    exe = tmp_path / "host_inverse_check"
    _compile("host_inverse_check.cpp", exe)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "Fq: mismatches 0" in out.stdout and "Fr: mismatches 0" in out.stdout


@pytest.mark.parametrize("field", [0, 1], ids=["fr", "fq"])
def test_host_field_ops_vs_integers(tmp_path, field):
    p = fx.R_FR if field == 0 else fx.Q
    exe = tmp_path / "host_field_check"
    _compile("host_field_check.cpp", exe)
    a, b = fx.pairs(p, cross=240)
    n = len(a)
    assert n > 50000
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    src.write_bytes(np.array([n], dtype=np.uint64).tobytes() + fx.to_array(a).tobytes() + fx.to_array(b).tobytes())
    subprocess.check_call([str(exe), str(field), str(src), str(dst)], timeout=300)
    got = np.fromfile(dst, dtype=np.uint64).reshape(6, n, 4)
    for k, op in enumerate((fx.OP_MUL, fx.OP_ADD, fx.OP_SUB, fx.OP_SQR, fx.OP_MUL_ADD2, fx.OP_MUL_SUB2)):
        exp = fx.expected(op, a, b, p)
        res = fx.from_array(got[k])
        bad = [i for i in range(n) if res[i] != exp[i]]
        assert not bad, (op, len(bad), [(hex(a[i]), hex(b[i])) for i in bad[:3]])
