"""Witness-vector bundles, pool witness batches and box witness jobs, the parts that need no GPU: the header, the Python
binding and the Rust shim agree on `b200_bundle_witness` and the five entry points; the C entry points refuse NULL
arguments before touching a device; and the Python wrappers check blinder lengths, keys without wiring, witness lengths
and link indices before any library call."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

from renegade_b200 import _lib, synth
from renegade_b200.backend import GroupLayout, ProverBox, ProverPool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = {
    "b200_pool_submit_bundle_witness": ["pool", "srs", "proofs", "n_proofs", "links", "n_links", "ticket"],
    "b200_pool_submit_prove_witness_batch": ["pool", "pk", "items", "k", "statuses", "ticket"],
    "b200_box_preprocess_wiring": ["box", "srs", "log_n", "num_inputs", "selectors_evals", "wire_vars", "num_vars", "k", "out"],
    "b200_box_submit_prove_witness": ["box", "pk", "witness", "blinders", "proof", "link_poly", "pub_inputs_out", "ticket"],
    "b200_box_submit_bundle_witness": ["box", "srs", "pks", "proofs", "n_proofs", "links", "n_links", "ticket"],
}
INVALID = _lib.B200_ERR_INVALID


def test_header_binding_and_shim_agree():
    _, structs, funcs, _ = _lib.parse_header()
    sig = {name: (ret, args) for name, ret, args in funcs}
    for name, args in NEW.items():
        assert name in _lib.EXPORTS
        assert sig[name][0] == "int" and [a for a, _ in sig[name][1]] == args, name
    assert dict(sig["b200_box_preprocess_wiring"][1])["wire_vars"] == "const unsigned *"
    assert dict(sig["b200_pool_submit_bundle_witness"][1])["proofs"] == "const b200_bundle_witness *"
    assert dict(sig["b200_box_submit_bundle_witness"][1])["pks"] == "const b200_box_pk * const *"
    assert [f for f, _, _ in structs["b200_bundle_witness"]] == ["pk", "witness", "blinders", "proof", "link_poly",
                                                                "pub_inputs_out"]
    assert C.sizeof(_lib.STRUCTS["b200_bundle_witness"]) == 6 * C.sizeof(C.c_void_p)
    lib = _lib.load()  # every declared symbol is exported, with the header's signature
    assert lib.b200_pool_submit_bundle_witness.argtypes == [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                                            C.c_size_t, C.c_void_p]
    assert lib.b200_box_preprocess_wiring.argtypes[2:4] == [C.c_uint, C.c_size_t]
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi.rs")).read()
    for name in NEW:
        assert re.search(rf"pub fn {name}\(", ffi), name
    assert re.search(r"pub struct b200_bundle_witness \{\s*pub pk: \*const b200_pk,\s*pub witness: \*const u64,", ffi)
    shim = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()
    assert "pub fn prove_from_witness_batch" in shim and "ffi::b200_pool_submit_prove_witness_batch(" in shim


def test_null_arguments_are_refused_without_a_device():
    lib = _lib.load()
    t = C.c_uint64()
    assert lib.b200_pool_submit_bundle_witness(None, None, None, 1, None, 0, C.byref(t)) == INVALID
    assert lib.b200_pool_submit_prove_witness_batch(None, None, None, 0, None, C.byref(t)) == INVALID
    h = C.c_void_p()
    assert lib.b200_box_preprocess_wiring(None, None, 4, 0, None, None, 1, None, C.byref(h)) == INVALID
    assert lib.b200_box_submit_prove_witness(None, None, None, None, None, None, None, C.byref(t)) == INVALID
    assert lib.b200_box_submit_bundle_witness(None, None, None, None, 1, None, 0, C.byref(t)) == INVALID


class _NoLibrary:
    """Stands in for the loaded library: any call means a check did not run first."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called before the arguments were checked")


def _pool():
    pool = ProverPool.__new__(ProverPool)
    pool._lib, pool._h, pool._keep, pool._borrowed = _NoLibrary(), None, {}, []
    return pool


def _box(shapes):
    box = ProverBox.__new__(ProverBox)
    box._lib, box._h, box._keep, box.devices = _NoLibrary(), None, {}, [0]
    box._shapes = shapes
    return box


def _key(num_vars=20, log_n=4, num_inputs=2):
    return SimpleNamespace(_h=C.c_void_p(0x1000), domain_size=1 << log_n, num_inputs=num_inputs, num_vars=num_vars)


@pytest.fixture
def parts():
    wit = np.zeros((20, 4), dtype=np.uint64)
    return wit, synth.splitmix_blinders(1), GroupLayout(alignment=4, offset=2, size=3)


def _refused(fn, *args, match):
    with pytest.raises(_lib.B200Error) as err:
        fn(*args)
    assert err.value.code == INVALID and re.search(match, str(err.value)), str(err.value)


def test_pool_bundle_checks_run_before_the_library(parts):
    wit, bl, lay = parts
    pool, pk = _pool(), _key()
    _refused(pool.submit_bundle_witness, None, [(pk, wit, bl[:16])], [], match="proof 0 has 16 blinders")
    _refused(pool.submit_bundle_witness, None, [(pk, wit, bl), (_key(num_vars=0), wit, bl)], [], match="proof 1 holds no wiring")
    _refused(pool.submit_bundle_witness, None, [(pk, wit[:-1], bl)], [], match="19 elements, the key takes 20")
    _refused(pool.submit_bundle_witness, None, [(pk, wit, bl), (pk, wit, bl)], [(0, 1, lay), (1, 2, lay)],
             match=r"link 1 names proof \(1, 2\) of a bundle of 2")
    _refused(pool.submit_bundle_witness, None, [(pk, wit, bl)], [(-1, 0, lay)], match="link 0")


def test_pool_witness_batch_checks_run_before_the_library(parts):
    wit, bl, _ = parts
    pool, pk = _pool(), _key()
    _refused(pool.submit_prove_witness_batch, _key(num_vars=0), [wit], [bl], match="holds no wiring")
    _refused(pool.submit_prove_witness_batch, pk, [wit, wit], [bl, bl[:3]], match="item 1 has 3 blinders")
    _refused(pool.submit_prove_witness_batch, pk, [wit, wit], [bl], match="2 witness vectors and 1 blinder vectors")
    _refused(pool.submit_prove_witness_batch, pk, [wit[:5]], [bl], match="item 0: the witness has 5 elements")


def test_box_checks_run_before_the_library(parts):
    wit, bl, lay = parts
    wired, tables = C.c_void_p(0x10), C.c_void_p(0x20)
    box = _box({0x10: _key(), 0x20: _key(num_vars=0)})
    stranger = C.c_void_p(0x30)  # a key another box made
    _refused(box.submit_prove_witness, stranger, wit, bl, match="not made by this box")
    _refused(box.submit_prove_witness, wired, wit, bl[:1], match="17 Fr elements")
    _refused(box.submit_prove_witness, wired, wit[:2], bl, match="2 elements, the key takes 20")
    _refused(box.submit_bundle_witness, None, [(wired, wit, bl), (tables, wit, bl)], [], match="proof 1 holds no wiring")
    _refused(box.submit_bundle_witness, None, [(wired, wit, bl)], [(0, 1, lay)], match="link 0 names proof")
    _refused(box.submit_bundle_witness, None, [(stranger, wit, bl)], [], match="not made by this box")
    _refused(box.submit_bundle, None, [(wired, 0, np.zeros((1, 4), dtype=np.uint64), bl)], [],
             match="public inputs / blinders do not match")
