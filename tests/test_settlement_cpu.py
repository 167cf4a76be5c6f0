"""Settlement jobs, the parts that need no GPU: include/b200settlement.h, the Python binding, a C compiler and the Rust
shim agree on `b200_settlement_link` and the six entry points; the C entry points refuse NULL arguments before touching a device; and
the Python wrappers check blinders, public inputs, wire tables, witness lengths, hint arrays, layouts and keys without
wiring before any library call."""
import ctypes as C
import os
import re
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from renegade_b200 import _lib, synth
from renegade_b200.backend import GroupLayout, LinkingHint, PlonkKzgSnark, ProverBox, ProverPool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = _lib.B200_ERR_INVALID
TAIL = ["links", "n_links", "statuses"]
NEW = {
    "b200_plonk_prove_settlement": ["ctx", "srs", "pk", "wires", "pub_inputs", "blinders", "proof", "link_poly"] + TAIL,
    "b200_plonk_prove_settlement_witness": ["ctx", "srs", "pk", "witness", "blinders", "proof", "link_poly",
                                            "pub_inputs_out"] + TAIL,
    "b200_pool_submit_settlement": ["pool", "srs", "proof"] + TAIL + ["ticket"],
    "b200_pool_submit_settlement_witness": ["pool", "srs", "proof"] + TAIL + ["ticket"],
    "b200_box_submit_settlement": ["box", "srs", "pk", "proof"] + TAIL + ["ticket"],
    "b200_box_submit_settlement_witness": ["box", "srs", "pk", "proof"] + TAIL + ["ticket"],
}


def test_header_binding_and_shim_agree():
    _, structs, funcs, macros = _lib.parse_header(_lib.SETTLEMENT_HEADER)
    sig = {name: (ret, args) for name, ret, args in funcs}
    assert [name for name, _, _ in funcs] == _lib.SETTLEMENT_EXPORTS == list(NEW)
    assert not set(NEW) & set(_lib.EXPORTS) and not macros  # the core header and its error codes stay as they are
    for name, args in NEW.items():
        assert sig[name][0] == "int" and [a for a, _ in sig[name][1]] == args, name
        assert dict(sig[name][1])["links"] == "const b200_settlement_link *", name
    assert dict(sig["b200_pool_submit_settlement"][1])["proof"] == "const b200_bundle_proof *"
    assert dict(sig["b200_box_submit_settlement_witness"][1])["proof"] == "const b200_bundle_witness *"
    assert dict(sig["b200_box_submit_settlement"][1])["pk"] == "const b200_box_pk *"
    assert [f for f, _, _ in structs["b200_settlement_link"]] == ["hint_poly", "hint_len", "hint_comm", "alignment", "offset",
                                                                 "size", "proof", "eta"]
    assert C.sizeof(_lib.STRUCTS["b200_settlement_link"]) == 8 * 8
    lib = _lib.load()  # every declared symbol is exported, with the header's signature
    assert lib.b200_plonk_prove_settlement.argtypes == [C.c_void_p] * 9 + [C.c_size_t, C.c_void_p]
    assert lib.b200_pool_submit_settlement.argtypes == [C.c_void_p] * 4 + [C.c_size_t, C.c_void_p, C.c_void_p]
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_rust_ffi as gen
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi_settlement.rs")).read()
    assert ffi == gen.generate(_lib.SETTLEMENT_HEADER), "ffi_settlement.rs is stale: run python tools/gen_rust_ffi.py"
    for name in NEW:
        assert re.search(rf"pub fn {name}\(", ffi), name
    assert re.search(r"pub struct b200_settlement_link \{\s*pub hint_poly: \*const u64,\s*pub hint_len: usize,", ffi)
    shim = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()
    assert "pub mod ffi_settlement;" in shim
    assert "pub fn prove_settlement<" in shim and "ffi_settlement::b200_pool_submit_settlement(" in shim
    assert "pub fn prove_settlement_from_witness<" in shim and "ffi_settlement::b200_pool_submit_settlement_witness(" in shim


def test_header_compiles_to_the_binding(tmp_path):
    """What a C compiler makes of include/b200settlement.h is the binding: every parsed signature initialises a pointer
    to the declared function, and `b200_settlement_link` has the ctypes class's size and field offsets."""
    _, structs, funcs, _ = _lib.parse_header(_lib.SETTLEMENT_HEADER)
    decls = [f"static {ret} (*const p_{name})({', '.join(t for _, t in args)}) = {name};" for name, ret, args in funcs]
    lines = [f'printf("{s} %zu\\n", sizeof({s}));' for s in structs]
    lines += [f'printf("{s}.{f} %zu %zu\\n", offsetof({s}, {f}), sizeof((({s}*)0)->{f}));'
              for s, fields in structs.items() for f, _, _ in fields]
    def gcc(src, out, *flags):
        (tmp_path / "s.c").write_text(src)
        r = subprocess.run(["gcc", "-std=c11", "-Werror", "-I" + os.path.join(ROOT, "include"), *flags, str(tmp_path / "s.c"),
                            "-o", str(tmp_path / out)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr

    gcc('#include "b200settlement.h"\n' + "\n".join(decls) + "\n", "s.o", "-c")
    gcc('#include <stdio.h>\n#include <stddef.h>\n#include "b200settlement.h"\nint main(void) {\n' + "\n".join(lines) +
        "\nreturn 0;\n}\n", "s")
    got = subprocess.run([str(tmp_path / "s")], capture_output=True, text=True, check=True).stdout.splitlines()
    want = []
    for s_ in structs:
        want.append(f"{s_} {C.sizeof(_lib.STRUCTS[s_])}")
    for s_, fields in structs.items():
        cls = _lib.STRUCTS[s_]
        want += [f"{s_}.{f} {getattr(cls, f).offset} {getattr(cls, f).size}" for f, _, _ in fields]
    assert got == want


def test_null_arguments_are_refused_without_a_device():
    lib = _lib.load()
    t = C.c_uint64()
    st = (C.c_int * 2)()
    assert lib.b200_plonk_prove_settlement(None, None, None, None, None, None, None, None, None, 0, st) == INVALID
    assert lib.b200_plonk_prove_settlement_witness(None, None, None, None, None, None, None, None, None, 1, st) == INVALID
    assert lib.b200_pool_submit_settlement(None, None, None, None, 0, None, C.byref(t)) == INVALID
    assert lib.b200_pool_submit_settlement_witness(None, None, None, None, 0, None, C.byref(t)) == INVALID
    assert lib.b200_box_submit_settlement(None, None, None, None, None, 0, None, C.byref(t)) == INVALID
    assert lib.b200_box_submit_settlement_witness(None, None, None, None, None, 0, None, C.byref(t)) == INVALID
    assert list(st) == [0, 0]  # nothing written


class _NoLibrary:
    """Stands in for the loaded library: any call means a check did not run first."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called before the arguments were checked")


class _Srs:
    """Stands in for Bases: 40 powers."""
    _h = None

    def __len__(self):
        return 40


def _key(num_vars=20, log_n=4, num_inputs=2):
    return SimpleNamespace(_h=C.c_void_p(0x1000), domain_size=1 << log_n, num_inputs=num_inputs, num_vars=num_vars)


def _refused(fn, *args, match):
    with pytest.raises(_lib.B200Error) as err:
        fn(*args)
    assert err.value.code == INVALID and re.search(match, str(err.value)), str(err.value)


@pytest.fixture
def parts():
    wit = np.zeros((20, 4), dtype=np.uint64)
    wires = np.zeros((5, 16, 4), dtype=np.uint64)
    pub = np.zeros((2, 4), dtype=np.uint64)
    hint = LinkingHint(np.zeros((18, 4), dtype=np.uint64), np.zeros(8, dtype=np.uint64))
    return wit, wires, pub, synth.splitmix_blinders(1), hint, GroupLayout(alignment=4, offset=2, size=3)


def _checks(prove, prove_witness, srs, pk, parts):
    """The refusals every settlement wrapper shares: prove(wires, pub, bl, links), prove_witness(pk, wit, bl, links)"""
    wit, wires, pub, bl, hint, lay = parts
    ok = [(hint, lay)]
    _refused(prove, wires, pub, bl[:16], ok, match="16 blinders, the prover draws 17")
    _refused(prove, wires, pub[:1], bl, ok, match="1 public inputs for a key with 2")
    _refused(prove, wires[:4], pub, bl, ok, match="the wire table has 64 elements")
    _refused(prove, wires, pub, bl, [(hint, lay), (hint,)], match="link 1 is not a \\(hint, layout\\) pair")
    _refused(prove, wires, pub, bl, [(LinkingHint(np.zeros(7, dtype=np.uint64), hint.linking_wire_comm), lay)],
             match="link 0's hint is not a vector of field elements")
    _refused(prove, wires, pub, bl, [(LinkingHint(hint.linking_wire_poly, np.zeros(4, dtype=np.uint64)), lay)],
             match="link 0's hint commitment must be 8 limbs")
    _refused(prove, wires, pub, bl, [(hint, GroupLayout(4, 2, 0))], match="link 0's group of 0 roots")
    _refused(prove, wires, pub, bl, [(hint, lay), (hint, GroupLayout(4, 2, 18))], match="link 1's group of 18 roots")
    _refused(prove, wires, pub, bl, [(hint, GroupLayout(29, 2, 3))], match="link 0 has alignment 29")
    _refused(prove_witness, _key(num_vars=0), wit, bl, ok, match="holds no wiring")
    _refused(prove_witness, pk, wit[:19], bl, ok, match="19 elements, the key takes 20")
    _refused(prove_witness, pk, wit, bl[:2], ok, match="2 blinders")


def test_context_checks_run_before_the_library(parts):
    ctx, srs, pk = SimpleNamespace(_lib=_NoLibrary(), _h=None), _Srs(), _key()
    _checks(lambda *a: PlonkKzgSnark.prove_settlement(ctx, srs, pk, *a),
            lambda k, *a: PlonkKzgSnark.prove_settlement_witness(ctx, srs, k, *a), srs, pk, parts)
    wit, wires, pub, bl, hint, lay = parts
    long_hint = LinkingHint(np.zeros((41, 4), dtype=np.uint64), hint.linking_wire_comm)
    _refused(PlonkKzgSnark.prove_settlement, ctx, srs, pk, wires, pub, bl, [(long_hint, lay)],
             match="link 0 has 41 coefficients, the SRS 40 powers")


def test_pool_checks_run_before_the_library(parts):
    pool = ProverPool.__new__(ProverPool)
    pool._lib, pool._h, pool._keep, pool._borrowed = _NoLibrary(), None, {}, []
    srs, pk = _Srs(), _key()
    _checks(lambda *a: pool.submit_settlement(srs, pk, *a), lambda k, *a: pool.submit_settlement_witness(srs, k, *a), srs, pk,
            parts)
    assert pool._keep == {}


def test_box_checks_run_before_the_library(parts):
    box = ProverBox.__new__(ProverBox)
    box._lib, box._h, box._keep, box.devices = _NoLibrary(), None, {}, [0]
    wired, tables, stranger = C.c_void_p(0x10), C.c_void_p(0x20), C.c_void_p(0x30)
    box._shapes = {0x10: _key(), 0x20: _key(num_vars=0)}
    _checks(lambda *a: box.submit_settlement(None, wired, *a),
            lambda k, *a: box.submit_settlement_witness(None, tables if k.num_vars == 0 else wired, *a), None, _key(), parts)
    wit, wires, pub, bl, hint, lay = parts
    _refused(box.submit_settlement, None, stranger, wires, pub, bl, [(hint, lay)], match="not made by this box")
    _refused(box.submit_settlement_witness, None, stranger, wit, bl, [(hint, lay)], match="not made by this box")
    assert box._keep == {}
