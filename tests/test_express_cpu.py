"""The express lane, the parts that need no GPU: include/b200express.h, the Python binding, a C compiler and the Rust shim
agree on the six entry points; the create calls report the missing device, and expedite / wait_info refuse NULL handles
before touching one; the Python constructors refuse a negative express count before any library call."""
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
    "b200_pool_create_express": ("int", [("device", "int"), ("n_workers", "unsigned"), ("n_express", "unsigned"),
                                         ("out", "b200_pool * *")]),
    "b200_pool_expedite": ("int", [("pool", "b200_pool *"), ("ticket", "uint64_t"), ("moved", "size_t *")]),
    "b200_pool_wait_info": ("int", [("pool", "b200_pool *"), ("ticket", "uint64_t"), ("info", "uint64_t *")]),
    "b200_box_create_express": ("int", [("devices", "const int *"), ("n_dev", "int"), ("workers_per_device", "unsigned"),
                                        ("express_per_device", "unsigned"), ("out", "b200_box * *")]),
    "b200_box_expedite": ("int", [("box", "b200_box *"), ("ticket", "uint64_t"), ("moved", "size_t *")]),
    "b200_box_wait_info": ("int", [("box", "b200_box *"), ("ticket", "uint64_t"), ("info", "uint64_t *")]),
}


def test_header_binding_and_shim_agree():
    _, structs, funcs, macros = _lib.parse_header(_lib.EXPRESS_HEADER)
    assert [name for name, _, _ in funcs] == _lib.EXPRESS_EXPORTS == list(NEW)
    assert not structs and not macros  # the express layer reuses the core header's types and error codes
    assert not set(NEW) & set(_lib.EXPORTS + _lib.SETTLEMENT_EXPORTS + _lib.VERIFY_JOB_EXPORTS)
    assert {name: (ret, args) for name, ret, args in funcs} == NEW
    lib = _lib.load()  # every declared symbol is exported, with the header's signature
    assert lib.b200_pool_expedite.argtypes == [C.c_void_p, C.c_uint64, C.c_void_p]
    assert lib.b200_pool_create_express.argtypes == [C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    assert lib.b200_box_create_express.argtypes == [C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_void_p]
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_rust_ffi as gen
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi_express.rs")).read()
    assert ffi == gen.generate(_lib.EXPRESS_HEADER), "ffi_express.rs is stale: run python tools/gen_rust_ffi.py"
    assert "use super::ffi::*;" in ffi and all(f"pub fn {name}(" in ffi for name in NEW)
    assert "pub mod ffi_express;" in open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()


def test_header_compiles_to_the_binding(tmp_path):
    """Every parsed signature initialises a pointer to the declared function, alone and beside the other headers."""
    _, _, funcs, _ = _lib.parse_header(_lib.EXPRESS_HEADER)
    decls = [f"static {ret} (*const p_{name})({', '.join(t for _, t in args)}) = {name};" for name, ret, args in funcs]
    for includes in (['"b200express.h"'], ['"b200verifyjobs.h"', '"b200express.h"', '"b200settlement.h"', '"b200prover.h"']):
        src = "".join(f"#include {h}\n" for h in includes) + "\n".join(decls) + "\n"
        (tmp_path / "e.c").write_text(src)
        r = subprocess.run(["gcc", "-std=c11", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c",
                            str(tmp_path / "e.c"), "-o", str(tmp_path / "e.o")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr


def test_create_reports_the_missing_device():
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.b200_pool_create_express(0, 2, 1, C.byref(h)) == NO_DEVICE and not h.value
    devs = (C.c_int * 2)(0, 0)
    assert lib.b200_box_create_express(devs, 2, 1, 1, C.byref(h)) == NO_DEVICE and not h.value
    # counts are checked before the device
    assert lib.b200_pool_create_express(0, 0, 1, C.byref(h)) == INVALID
    assert lib.b200_pool_create_express(0, 65, 0, C.byref(h)) == INVALID
    assert lib.b200_pool_create_express(0, 1, 65, C.byref(h)) == INVALID
    assert lib.b200_pool_create_express(0, 1, 1, None) == INVALID
    assert not h.value


def test_null_handles_are_refused():
    lib = _lib.load()
    moved = C.c_size_t(77)
    info = (C.c_uint64 * 2)(5, 6)
    for fn, who in ((lib.b200_pool_expedite, b"pool_expedite"), (lib.b200_box_expedite, b"box_expedite")):
        assert fn(None, 1, C.byref(moved)) == INVALID and who in lib.b200_last_error()
    for fn, who in ((lib.b200_pool_wait_info, b"pool_wait_info"), (lib.b200_box_wait_info, b"box_wait_info")):
        assert fn(None, 1, info) == INVALID and who in lib.b200_last_error()
    assert lib.b200_pool_wait_info(None, 1, None) == INVALID
    assert moved.value == 77 and list(info) == [5, 6]  # nothing written


class _NoLibrary:
    """Stands in for the library: any load means a check did not run first."""

    def __call__(self):
        raise AssertionError("the library was loaded before the arguments were checked")


@pytest.mark.parametrize("express", [-1, -64, 1.5, True, "1"])
def test_python_constructors_refuse_a_bad_express_count(monkeypatch, express):
    monkeypatch.setattr(_lib, "load", _NoLibrary())
    with pytest.raises(ValueError, match="express worker count"):
        ProverPool(0, workers=2, express=express)
    with pytest.raises(ValueError, match="express worker count"):
        ProverBox([0, 0], workers_per_device=2, express_per_device=express)
