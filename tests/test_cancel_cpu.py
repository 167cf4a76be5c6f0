"""Cancellation of pool and box jobs, the parts that need no GPU: include/b200cancel.h, the Python binding, a C compiler and
the Rust shim agree on the four entry points and on B200_ERR_CANCELLED; every refusal is B200_ERR_INVALID before any
device is touched; the Python calls check the ticket before any library call."""
import ctypes as C
import os
import subprocess
import sys

import pytest

from renegade_b200 import _lib
from renegade_b200.backend import ProverBox, ProverPool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = _lib.B200_ERR_INVALID
NEW = {
    "b200_pool_cancel": ("int", [("pool", "b200_pool *"), ("ticket", "uint64_t"), ("dropped", "size_t *")]),
    "b200_pool_cancel_all": ("int", [("pool", "b200_pool *"), ("dropped", "size_t *")]),
    "b200_box_cancel": ("int", [("box", "b200_box *"), ("ticket", "uint64_t"), ("dropped", "size_t *")]),
    "b200_box_cancel_all": ("int", [("box", "b200_box *"), ("dropped", "size_t *")]),
}


def test_header_binding_and_shim_agree():
    _, structs, funcs, macros = _lib.parse_header(_lib.CANCEL_HEADER)
    assert [name for name, _, _ in funcs] == _lib.CANCEL_EXPORTS == list(NEW)
    assert not structs and macros == {"B200_ERR_CANCELLED": -8}  # the core header's types, one new error code
    assert not set(NEW) & set(_lib.EXPORTS + _lib.SETTLEMENT_EXPORTS + _lib.VERIFY_JOB_EXPORTS + _lib.EXPRESS_EXPORTS +
                              _lib.RESERVED_EXPORTS + _lib.SELFTEST_EXPORTS)
    assert {name: (ret, args) for name, ret, args in funcs} == NEW
    lib = _lib.load()  # every declared symbol is exported, with the header's signature
    assert lib.b200_pool_cancel.argtypes == [C.c_void_p, C.c_uint64, C.c_void_p]
    assert lib.b200_pool_cancel_all.argtypes == [C.c_void_p, C.c_void_p]
    assert lib.b200_box_cancel.argtypes == [C.c_void_p, C.c_uint64, C.c_void_p]
    assert lib.b200_box_cancel_all.argtypes == [C.c_void_p, C.c_void_p]
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_rust_ffi as gen
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi_cancel.rs")).read()
    assert ffi == gen.generate(_lib.CANCEL_HEADER), "ffi_cancel.rs is stale: run python tools/gen_rust_ffi.py"
    assert "use super::ffi::*;" in ffi and all(f"pub fn {name}(" in ffi for name in NEW)
    assert "pub const B200_ERR_CANCELLED: c_int = -8;" in ffi
    shim = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()
    assert "pub mod ffi_cancel;" in shim
    for fn in ("pub fn cancel(&self, ticket: u64)", "pub fn cancel_all(&self)", "pub fn shutdown_now(self)"):
        assert fn in shim


def test_error_code_is_in_the_code_table():
    assert _lib.B200_ERR_CANCELLED == -8
    codes = {v for k, v in vars(_lib).items() if k == "B200_OK" or k.startswith("B200_ERR_")}
    assert len(codes) == len([k for k in vars(_lib) if k == "B200_OK" or k.startswith("B200_ERR_")])  # all distinct
    assert _lib.B200_ERR_CANCELLED in codes and _lib.B200_ERR_UNSATISFIED in codes
    _, _, _, core = _lib.parse_header(_lib.HEADER)
    assert "B200_ERR_CANCELLED" not in core  # the core header and its pinned counts stay as they were


def test_header_compiles_to_the_binding(tmp_path):
    """Every parsed signature initialises a pointer to the declared function, alone and beside the other headers."""
    _, _, funcs, _ = _lib.parse_header(_lib.CANCEL_HEADER)
    decls = [f"static {ret} (*const p_{name})({', '.join(t for _, t in args)}) = {name};" for name, ret, args in funcs]
    decls.append("_Static_assert(B200_ERR_CANCELLED == -8, \"code\");")
    for includes in (['"b200cancel.h"'],
                     ['"b200express.h"', '"b200cancel.h"', '"b200reserved.h"', '"b200verifyjobs.h"', '"b200settlement.h"',
                      '"b200prover.h"']):
        src = "".join(f"#include {h}\n" for h in includes) + "\n".join(decls) + "\n"
        (tmp_path / "c.c").write_text(src)
        r = subprocess.run(["gcc", "-std=c11", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c",
                            str(tmp_path / "c.c"), "-o", str(tmp_path / "c.o")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr


def test_null_handles_and_outputs_are_refused():
    lib = _lib.load()
    dropped = C.c_size_t(77)
    for fn, who in ((lib.b200_pool_cancel, b"pool_cancel"), (lib.b200_box_cancel, b"box_cancel")):
        assert fn(None, 1, C.byref(dropped)) == INVALID and who in lib.b200_last_error()
        assert fn(None, 1, None) == INVALID
    for fn, who in ((lib.b200_pool_cancel_all, b"pool_cancel_all"), (lib.b200_box_cancel_all, b"box_cancel_all")):
        assert fn(None, C.byref(dropped)) == INVALID and who in lib.b200_last_error()
        assert fn(None, None) == INVALID
    assert dropped.value == 77  # nothing written


class _NoLibrary:
    """Stands in for the library object: any call means a check did not run first."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called before the arguments were checked")


@pytest.mark.parametrize("ticket", [0, -1, 1 << 64, 1.0, True, "3", None])
@pytest.mark.parametrize("cls", [ProverPool, ProverBox])
def test_python_cancel_checks_the_ticket_first(cls, ticket):
    jobs = cls.__new__(cls)
    jobs._lib, jobs._h, jobs._jobs = _NoLibrary(), C.c_void_p(0xdead), {}
    with pytest.raises(ValueError, match="a ticket is an int"):
        jobs.cancel(ticket)
