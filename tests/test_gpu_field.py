"""GPU parity: device field arithmetic (IMAD.WIDE Montgomery multiplier, squarer, fused two-product forms,
carry-chain add/sub, Fermat inverse) vs the oracle and Python integers, bit-exact, through the C ABI."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_selftest_wide_vs_wordserial(ctx):
    # production multiplier vs the word-serial reference multiplier, on the device
    assert ctx.selftest_field(0xC0FFEE, 1 << 20) == 0


@pytest.mark.parametrize("field", [0, 1])
def test_field_ops_vs_oracle(ctx, oracle, pyoracle, field):
    py = pyoracle
    mod = py.R if field == 0 else py.Q
    n = 4096
    a = oracle.splitmix_fr(0xA11CE + field, n, False)  # < r < q: valid residues for both fields
    b = oracle.splitmix_fr(0xB0B + field, n, False)
    # edge operands: 0, 1, p-1
    a[0] = 0
    a[1] = oracle.int_to_limbs(1)
    a[2] = oracle.int_to_limbs(mod - 1)
    b[2] = oracle.int_to_limbs(mod - 1)
    b[3] = 0
    for op, name in ((0, "orc_fp_mul"), (1, "orc_fp_add"), (2, "orc_fp_sub")):
        got = ctx.field_op(field, op, a, b)
        exp = np.stack([oracle.fp_binop(name, field, a[i], b[i]) for i in range(n)])
        assert (got == exp).all(), name
    got = ctx.field_op(field, 3, a[:64], b[:64])
    exp = np.stack([oracle.fp_unop("orc_fp_inv", field, a[i]) for i in range(64)])
    assert (got == exp).all()


@pytest.mark.parametrize("field", [0, 1], ids=["fr", "fq"])
def test_field_ops_on_edge_operands(ctx, field):
    """All seven device ops of b200_field_op — product, add, sub, inverse, the dedicated squarer and the fused
    a*b +- c*d of the curve additions — against Python integers on the edge operands of tests/field_edges.py: the whole
    residue range (for Fq the operands in [r, q) included), powers of two and their neighbours, limb patterns, and
    products that land exactly on 1 and p - 1."""
    import field_edges as fx
    p = fx.R_FR if field == 0 else fx.Q
    a, b = fx.pairs(p)
    assert len(a) > 10000 and any(x >= fx.R_FR for x in a) == (field == 1)
    da, db = fx.to_array(a), fx.to_array(b)
    for op in range(7):
        got = fx.from_array(ctx.field_op(field, op, da, db))
        exp = fx.expected(op, a, b, p)
        bad = [i for i in range(len(a)) if got[i] != exp[i]]
        assert not bad, (op, len(bad), [(hex(a[i]), hex(b[i])) for i in bad[:3]])


@pytest.mark.parametrize("n", [1, 15, 16, 17, 4095, 4096, 4097, 3 * 4096 + 5])
def test_batch_inverse_device(ctx, oracle, pyoracle, n):
    """b200_fr_batch_inverse_device (one binary-Euclid inversion per block of 4096, Montgomery's trick on two levels):
    every element against the oracle's inverse, around the chunk and block boundaries; zeros stay zero and leave their
    neighbours alone."""
    import ctypes as C
    import torch
    from renegade_b200 import _lib
    a = oracle.splitmix_fr(0x1AB + n, n, True)  # Montgomery residues
    for z in {0, n // 2, n - 1} if n > 2 else set():
        a[z] = 0
    d = torch.from_numpy(a.view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    _lib.check(ctx._lib.b200_fr_batch_inverse_device(ctx._h, C.c_void_p(d.data_ptr()), n))
    got = d.cpu().numpy().view(np.uint64)
    idx = sorted(set(list(range(min(n, 40))) + list(range(max(0, n - 40), n)) + [n // 2] + list(range(max(0, 4096 - 20), min(n, 4096 + 20)))))
    # the oracle's inverse works on Montgomery residues like the device's: inv(aR) = a^-1 R
    for i in idx:
        exp = oracle.fp_unop("orc_fp_inv", 0, a[i])
        assert (got[i] == exp).all(), i
    # the rest through the defining property: x * x^-1 = 1 (device multiplier, already pinned above)
    prod = ctx.field_op(0, 0, a, got)
    mont_one = np.array(oracle.int_to_limbs(pyoracle.to_mont(1, pyoracle.R)), dtype=np.uint64)
    nz = np.array([a[i].any() for i in range(n)])
    assert (prod[nz] == mont_one).all()
    assert (got[~nz] == 0).all()
