"""Verification jobs, the parts that need no GPU: include/b200verifyjobs.h, the Python binding, a C compiler and the Rust
shim agree on the two entry points; the C entry points refuse NULL handles before touching a device; and the Python
wrappers refuse what `PlonkKzgSnark.verify_each` refuses before any library call."""
import ctypes as C
import os
import re
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from renegade_b200 import _lib
from renegade_b200.backend import ProverBox, ProverPool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = _lib.B200_ERR_INVALID
ARGS = ["mode", "vks", "n_vks", "proofs", "n_proofs", "links", "n_links", "g2_h", "g2_tau_h", "all_accepted", "verdicts",
        "ticket"]
NEW = {"b200_pool_submit_verify": ["pool"] + ARGS, "b200_box_submit_verify": ["box"] + ARGS}


def test_header_binding_and_shim_agree():
    _, structs, funcs, macros = _lib.parse_header(_lib.VERIFY_JOB_HEADER)
    sig = {name: (ret, args) for name, ret, args in funcs}
    assert [name for name, _, _ in funcs] == _lib.VERIFY_JOB_EXPORTS == list(NEW)
    assert not structs and not macros  # the job layer reuses the core header's structs and error codes
    assert not set(NEW) & set(_lib.EXPORTS + _lib.SETTLEMENT_EXPORTS) and len(_lib.EXPORTS) == 110
    for name, args in NEW.items():
        ret, a = sig[name]
        assert ret == "int" and [x for x, _ in a] == args, name
        d = dict(a)
        assert d["vks"] == "const b200_verifying_key *" and d["proofs"] == "const b200_batch_proof *", name
        assert d["links"] == "const b200_batch_link *" and d["g2_h"] == d["g2_tau_h"] == "const uint64_t *", name
        assert d["all_accepted"] == "int *" and d["verdicts"] == "uint8_t *" and d["ticket"] == "uint64_t *", name
    assert dict(sig["b200_pool_submit_verify"][1])["pool"] == "b200_pool *"
    assert dict(sig["b200_box_submit_verify"][1])["box"] == "b200_box *"
    lib = _lib.load()  # every declared symbol is exported, with the header's signature
    want = [C.c_void_p, C.c_int] + [C.c_void_p, C.c_size_t] * 3 + [C.c_void_p] * 5
    assert lib.b200_pool_submit_verify.argtypes == want and lib.b200_box_submit_verify.argtypes == want
    assert lib.b200_pool_submit_verify.restype == C.c_int
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_rust_ffi as gen
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi_verifyjobs.rs")).read()
    assert ffi == gen.generate(_lib.VERIFY_JOB_HEADER), "ffi_verifyjobs.rs is stale: run python tools/gen_rust_ffi.py"
    for name in NEW:
        assert re.search(rf"pub fn {name}\(", ffi), name
    assert "use super::ffi::*;" in ffi
    shim = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()
    assert "pub mod ffi_verifyjobs;" in shim
    assert "pub fn submit_verify(" in shim and "pub fn submit_verify_combined(" in shim
    assert "ffi_verifyjobs::b200_pool_submit_verify(" in shim


def test_header_compiles_to_the_binding(tmp_path):
    """What a C compiler makes of include/b200verifyjobs.h is the binding: every parsed signature initialises a pointer to
    the declared function (so the parameter types are exactly the header's), alone and beside the other job header."""
    _, _, funcs, _ = _lib.parse_header(_lib.VERIFY_JOB_HEADER)
    decls = [f"static {ret} (*const p_{name})({', '.join(t for _, t in args)}) = {name};" for name, ret, args in funcs]
    for includes in (['"b200verifyjobs.h"'], ['"b200settlement.h"', '"b200verifyjobs.h"', '"b200prover.h"']):
        src = "".join(f"#include {h}\n" for h in includes) + "\n".join(decls) + "\n"
        (tmp_path / "v.c").write_text(src)
        r = subprocess.run(["gcc", "-std=c11", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c",
                            str(tmp_path / "v.c"), "-o", str(tmp_path / "v.o")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr


def test_null_handles_are_refused_without_a_device():
    lib = _lib.load()
    t = C.c_uint64(77)
    v = (C.c_uint8 * 1)(9)
    h = np.zeros(16, dtype=np.uint64)
    hp = h.ctypes.data_as(C.c_void_p)
    for fn, who in ((lib.b200_pool_submit_verify, b"pool_submit_verify"), (lib.b200_box_submit_verify, b"box_submit_verify")):
        assert fn(None, 0, None, 0, None, 0, None, 0, hp, hp, None, v, C.byref(t)) == INVALID
        assert who in lib.b200_last_error()
        assert fn(None, 1, None, 0, None, 0, None, 0, hp, hp, None, v, None) == INVALID
    assert t.value == 77 and v[0] == 9  # nothing written


class _NoLibrary:
    """Stands in for the loaded library: any call means a check did not run first."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called before the arguments were checked")


def _vk(h, tau_h, num_inputs=1):
    return SimpleNamespace(log_n=4, num_inputs=num_inputs, k=np.zeros((5, 4), dtype=np.uint64),
                           selector_comms=np.zeros((13, 8), dtype=np.uint64), sigma_comms=np.zeros((5, 8), dtype=np.uint64),
                           g2_h=h, g2_tau_h=tau_h)


def _checks(submit):
    h, tau_h = np.zeros(16, dtype=np.uint64), np.ones(16, dtype=np.uint64)
    proof = _lib.STRUCTS["b200_proof"]()
    pi = np.zeros((1, 4), dtype=np.uint64)
    with pytest.raises(ValueError, match="one verifying key and one public-input vector per proof"):
        submit([_vk(h, tau_h)], [pi, pi], [proof])
    with pytest.raises(ValueError, match="must share the G2 pair"):
        submit([_vk(h, tau_h), _vk(tau_h, h)], [pi, pi], [proof, proof])
    with pytest.raises(ValueError, match="links without proofs need g2"):
        submit([], [], [], [(np.zeros(8), np.zeros(8), _lib.STRUCTS["b200_link_proof"](), None)])
    with pytest.raises(ValueError, match="without items needs g2"):
        submit([], [], [], combined=True)


def test_pool_and_box_checks_run_before_the_library():
    pool = ProverPool.__new__(ProverPool)
    pool._lib, pool._h, pool._keep, pool._borrowed = _NoLibrary(), None, {}, []
    box = ProverBox.__new__(ProverBox)
    box._lib, box._h, box._keep, box.devices, box._shapes = _NoLibrary(), None, {}, [0], {}
    for jobs in (pool, box):
        _checks(jobs.submit_verify)
        assert jobs._keep == {}
