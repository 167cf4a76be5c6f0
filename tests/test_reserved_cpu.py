"""Reserved SMs for the express lane, the parts that need no GPU: include/b200reserved.h, the Python binding, a C compiler
and the Rust shim agree on the four entry points; every refusal of the create calls is reported before any device is
touched, and the device's absence after them; the Python constructors refuse a bad `express_sms` before any library
call."""
import ctypes as C
import os
import subprocess
import sys

import pytest

from renegade_b200 import _lib
from renegade_b200.backend import ProverBox, ProverPool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, NO_DEVICE = _lib.B200_ERR_INVALID, _lib.B200_ERR_NO_DEVICE
NEW = {
    "b200_pool_create_reserved": ("int", [("device", "int"), ("n_workers", "unsigned"), ("n_express", "unsigned"),
                                          ("express_sms", "unsigned"), ("out", "b200_pool * *")]),
    "b200_pool_partition": ("int", [("pool", "const b200_pool *"), ("out", "unsigned *")]),
    "b200_pool_probe_sms": ("int", [("pool", "b200_pool *"), ("worker", "unsigned"), ("mask", "uint64_t *")]),
    "b200_box_create_reserved": ("int", [("devices", "const int *"), ("n_dev", "int"), ("workers_per_device", "unsigned"),
                                         ("express_per_device", "unsigned"), ("express_sms", "unsigned"),
                                         ("out", "b200_box * *")]),
}


def test_header_binding_and_shim_agree():
    _, structs, funcs, macros = _lib.parse_header(_lib.RESERVED_HEADER)
    assert [name for name, _, _ in funcs] == _lib.RESERVED_EXPORTS == list(NEW)
    assert not structs and not macros  # the reserved layer reuses the core header's types and error codes
    assert not set(NEW) & set(_lib.EXPORTS + _lib.SETTLEMENT_EXPORTS + _lib.VERIFY_JOB_EXPORTS + _lib.EXPRESS_EXPORTS)
    assert {name: (ret, args) for name, ret, args in funcs} == NEW
    lib = _lib.load()  # every declared symbol is exported, with the header's signature
    assert lib.b200_pool_create_reserved.argtypes == [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_void_p]
    assert lib.b200_pool_partition.argtypes == [C.c_void_p, C.c_void_p]
    assert lib.b200_pool_probe_sms.argtypes == [C.c_void_p, C.c_uint, C.c_void_p]
    assert lib.b200_box_create_reserved.argtypes == [C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_void_p]
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_rust_ffi as gen
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi_reserved.rs")).read()
    assert ffi == gen.generate(_lib.RESERVED_HEADER), "ffi_reserved.rs is stale: run python tools/gen_rust_ffi.py"
    assert "use super::ffi::*;" in ffi and all(f"pub fn {name}(" in ffi for name in NEW)
    assert "pub mod ffi_reserved;" in open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()


def test_header_compiles_to_the_binding(tmp_path):
    """Every parsed signature initialises a pointer to the declared function, alone and beside the other headers."""
    _, _, funcs, _ = _lib.parse_header(_lib.RESERVED_HEADER)
    decls = [f"static {ret} (*const p_{name})({', '.join(t for _, t in args)}) = {name};" for name, ret, args in funcs]
    for includes in (['"b200reserved.h"'],
                     ['"b200express.h"', '"b200reserved.h"', '"b200verifyjobs.h"', '"b200settlement.h"', '"b200prover.h"']):
        src = "".join(f"#include {h}\n" for h in includes) + "\n".join(decls) + "\n"
        (tmp_path / "r.c").write_text(src)
        r = subprocess.run(["gcc", "-std=c11", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c",
                            str(tmp_path / "r.c"), "-o", str(tmp_path / "r.o")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("n_workers,n_express,express_sms,rule", [
    (1, 1, 0, b"express_sms must be a positive multiple of 8"),
    (1, 1, 4, b"express_sms must be a positive multiple of 8"),
    (1, 1, 12, b"express_sms must be a positive multiple of 8"),
    (1, 1, 256, b"at least 8 SMs for the normal group"),
    (0, 1, 16, b"n_workers must be in [1, 64]"),  # a normal group of no workers
    (65, 1, 16, b"n_workers must be in [1, 64]"),
    (1, 0, 16, b"n_express must be in [1, 64]"),
    (1, 65, 16, b"n_express must be in [1, 64]"),
])
def test_pool_refusals_name_the_rule(n_workers, n_express, express_sms, rule):
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.b200_pool_create_reserved(0, n_workers, n_express, express_sms, C.byref(h)) == INVALID and not h.value
    assert rule in lib.b200_last_error()
    devs = (C.c_int * 2)(0, 0)
    assert lib.b200_box_create_reserved(devs, 2, n_workers, n_express, express_sms, C.byref(h)) == INVALID and not h.value
    assert rule in lib.b200_last_error()


def test_null_outputs_and_handles_are_refused():
    lib = _lib.load()
    assert lib.b200_pool_create_reserved(0, 1, 1, 16, None) == INVALID and b"null out" in lib.b200_last_error()
    devs = (C.c_int * 1)(0)
    assert lib.b200_box_create_reserved(devs, 1, 1, 1, 16, None) == INVALID
    assert lib.b200_box_create_reserved(None, 1, 1, 1, 16, C.byref(C.c_void_p())) == INVALID
    out = (C.c_uint * 2)(5, 6)
    assert lib.b200_pool_partition(None, out) == INVALID and list(out) == [5, 6]
    mask = (C.c_uint64 * 4)(1, 2, 3, 4)
    assert lib.b200_pool_probe_sms(None, 0, mask) == INVALID and list(mask) == [1, 2, 3, 4]


def test_create_reports_the_missing_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.b200_pool_create_reserved(0, 2, 1, 16, C.byref(h)) == NO_DEVICE and not h.value
    assert b"no CPU fallback" in lib.b200_last_error()
    devs = (C.c_int * 2)(0, 0)
    assert lib.b200_box_create_reserved(devs, 2, 1, 1, 8, C.byref(h)) == NO_DEVICE and not h.value


class _NoLibrary:
    """Stands in for the library: any load means a check did not run first."""

    def __call__(self):
        raise AssertionError("the library was loaded before the arguments were checked")


@pytest.mark.parametrize("express,express_sms,match", [
    (1, -8, "express_sms must be an int"), (1, 8.0, "express_sms must be an int"), (1, True, "express_sms must be an int"),
    (1, 4, "multiple of 8"), (1, 12, "multiple of 8"), (1, 256, "multiple of 8 in"), (0, 16, "needs express >= 1"),
])
def test_python_constructors_refuse_a_bad_reservation(monkeypatch, express, express_sms, match):
    monkeypatch.setattr(_lib, "load", _NoLibrary())
    with pytest.raises(ValueError, match=match):
        ProverPool(0, workers=2, express=express, express_sms=express_sms)
    with pytest.raises(ValueError, match=match):
        ProverBox([0, 0], workers_per_device=2, express_per_device=express, express_sms=express_sms)
