"""Compact proving keys, the parts that need no GPU: include/b200compact.h, the Python binding, a C compiler and the Rust
shim agree on the four entry points; NULL handles are refused before any device is touched; b200_plonk_footprint equals
the estimate restated here from plonk.cu and msm.cu, part by part, for every domain 2^2 … 2^25 in both modes (the default
mode against `large_domains.footprint_parts`), and puts a compact key and one proof of 2^23 under 80 GB with 15 % slack."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

import large_domains as ld
import msm_digits as md
from renegade_b200 import _lib
from renegade_b200.backend import PlonkKzgSnark

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = _lib.B200_ERR_INVALID
CTX_PK = [("ctx", "b200_ctx *"), ("srs", "const b200_bases *"), ("log_n", "unsigned"), ("num_inputs", "size_t"),
          ("selectors_evals", "const uint64_t *")]
NEW = {
    "b200_plonk_preprocess_compact": ("int", CTX_PK + [("perm", "const uint64_t *"), ("k", "const uint64_t *"),
                                                       ("out", "b200_pk * *")]),
    "b200_plonk_preprocess_wiring_compact": ("int", CTX_PK + [("wire_vars", "const unsigned *"), ("num_vars", "size_t"),
                                                              ("k", "const uint64_t *"), ("out", "b200_pk * *")]),
    "b200_pk_is_compact": ("int", [("pk", "const b200_pk *")]),
    "b200_plonk_footprint": ("int", [("log_n", "unsigned"), ("k", "size_t"), ("compact", "int"), ("out", "uint64_t *")]),
}
GB80 = 80 * 10**9
SLACK = 1.15


def test_header_binding_and_shim_agree():
    _, structs, funcs, macros = _lib.parse_header(_lib.COMPACT_HEADER)
    assert [name for name, _, _ in funcs] == _lib.COMPACT_EXPORTS == list(NEW)
    assert not structs and macros == {"B200_FOOTPRINT_PARTS": 12} == {"B200_FOOTPRINT_PARTS": _lib.FOOTPRINT_PARTS}
    assert len(PlonkKzgSnark.FOOTPRINT_PARTS) == _lib.FOOTPRINT_PARTS
    assert not set(NEW) & set(_lib.EXPORTS + _lib.SETTLEMENT_EXPORTS + _lib.VERIFY_JOB_EXPORTS + _lib.EXPRESS_EXPORTS +
                              _lib.RESERVED_EXPORTS + _lib.SELFTEST_EXPORTS + _lib.CANCEL_EXPORTS)
    assert {name: (ret, args) for name, ret, args in funcs} == NEW
    # the two preprocess calls take exactly the arguments of the default ones
    core = {name: args for name, _, args in _lib.parse_header(_lib.HEADER)[2]}
    assert NEW["b200_plonk_preprocess_compact"][1] == core["b200_plonk_preprocess"]
    assert NEW["b200_plonk_preprocess_wiring_compact"][1] == core["b200_plonk_preprocess_wiring"]
    lib = _lib.load()
    assert lib.b200_plonk_footprint.argtypes == [C.c_uint, C.c_size_t, C.c_int, C.c_void_p]
    assert lib.b200_pk_is_compact.argtypes == [C.c_void_p] and lib.b200_pk_is_compact.restype == C.c_int
    # the header's list of parts is the binding's
    text = open(_lib.COMPACT_HEADER).read()
    listed = re.findall(r"^ \*\s+(\d+) (\w+)", text, flags=re.M)
    assert [(int(i), p) for i, p in listed] == list(enumerate(PlonkKzgSnark.FOOTPRINT_PARTS))
    assert "b200_box_preprocess" in text  # box keys are named out of scope
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_rust_ffi as gen
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi_compact.rs")).read()
    assert ffi == gen.generate(_lib.COMPACT_HEADER), "ffi_compact.rs is stale: run python tools/gen_rust_ffi.py"
    assert "use super::ffi::*;" in ffi and all(f"pub fn {name}(" in ffi for name in NEW)
    assert "pub const B200_FOOTPRINT_PARTS: c_int = 12;" in ffi
    shim = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()
    assert "pub mod ffi_compact;" in shim and "pub fn preprocess_wiring_compact(&self, cs: &PlonkCircuit<Fr>)" in shim
    assert "ffi_compact::b200_plonk_preprocess_wiring_compact(" in shim


def test_header_compiles_to_the_binding(tmp_path):
    """Every parsed signature initialises a pointer to the declared function, alone and beside the other headers."""
    _, _, funcs, _ = _lib.parse_header(_lib.COMPACT_HEADER)
    decls = [f"static {ret} (*const p_{name})({', '.join(t for _, t in args)}) = {name};" for name, ret, args in funcs]
    decls.append("_Static_assert(B200_FOOTPRINT_PARTS == 12, \"parts\");")
    for includes in (['"b200compact.h"'],
                     ['"b200cancel.h"', '"b200compact.h"', '"b200express.h"', '"b200settlement.h"', '"b200prover.h"']):
        src = "".join(f"#include {h}\n" for h in includes) + "\n".join(decls) + "\n"
        (tmp_path / "c.c").write_text(src)
        r = subprocess.run(["gcc", "-std=c11", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c",
                            str(tmp_path / "c.c"), "-o", str(tmp_path / "c.o")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr


def test_null_handles_and_bad_arguments_are_refused():
    lib = _lib.load()
    out = C.c_void_p(0x1234)
    buf = (C.c_uint64 * 4)()
    wv = (C.c_uint * 4)()
    assert lib.b200_plonk_preprocess_compact(None, None, 4, 0, buf, buf, buf, C.byref(out)) == INVALID
    assert lib.b200_plonk_preprocess_wiring_compact(None, None, 4, 0, buf, wv, 4, buf, C.byref(out)) == INVALID
    assert out.value == 0x1234  # nothing written
    assert lib.b200_pk_is_compact(None) == 0
    parts = (C.c_uint64 * 12)(*([7] * 12))
    assert lib.b200_plonk_footprint(20, 1, 1, None) == INVALID
    for log_n, k in ((1, 1), (26, 1), (20, 0), (20, 65)):
        assert lib.b200_plonk_footprint(log_n, k, 1, parts) == INVALID, (log_n, k)
        assert b"plonk_footprint" in lib.b200_last_error()
    assert list(parts) == [7] * 12


# ---- the compact estimate, restated ----------------------------------------------------------------------------------
def compact_constants(src: str = None) -> dict:
    """ld.constants() plus the compact rules of plonk.cu, which must still read as restated in compact_footprint_parts."""
    src = ld.plonk_source() if src is None else src
    c = ld.constants(src)
    for rule in (r"static size_t coset_batch\(unsigned k\) \{ return NS \+ NW \+ \(size_t\)\(NW \+ 2\) \* k; \}",
                 r"return workspace_elems\(n, k\) - \(size_t\)k \* 7 \* 8 \* n \+ coset_batch\(k\) \* n;",
                 r"return std::max\(\{coset_batch\(k\) \* n, \(size_t\)k \* \(NW \+ 1\) \* \(n \+ 4\), \(size_t\)k \* num_vars\}\);",
                 r"c->ntt_scratch\.reserve\(\(size_t\)NS \* n \* sizeof\(fe\)\)",
                 r"for \(unsigned s0 = 0; s0 < \(unsigned\)NS; s0 \+= NW\)",
                 r"\(!compact && \(rc = alloc_fe\(&pk->ce_sel, NS \* m\)\)\)",
                 r"\(!compact && \(rc = alloc_fe\(&pk->ce_sig, NW \* m\)\)\)"):
        assert re.search(rule, src), f"plonk.cu's compact rule changed: restate it here ({rule})"
    return c


def compact_footprint_parts(log_n: int, k: int = 1) -> dict:
    """What one context holds with one compact key and a call of k proofs: the key keeps coefficients, sigma
    evaluations, the domain's points and the four per-coset point tables (4 m), no coset tables of the 18 polynomials;
    the NTT scratch holds preprocessing's NS n and a proof's per-coset batch; the MSM scratch is a proof's NW wire
    commitments (the selectors are committed NW at a time); the workspace holds one coset of each polynomial instead of
    all of them, except the quotient."""
    c = compact_constants()
    NS, NW = c["NS"], c["NW"]
    n = 1 << log_n
    m = ld.cosets(log_n, c) * n
    fe = 32
    win = md.choose_window(n + 3, 0)
    W = md.num_windows(win)

    def batch(q):
        return NS + NW + (NW + 2) * q

    def workspace(q):
        return ld.workspace_elems(n, q, c) - q * 7 * 8 * n + batch(q) * n

    def nscr(q):
        return max(batch(q) * n, q * (NW + 1) * (n + 4))

    p = {
        "key": ((NS + 2 * NW + 1) * n + 4 * m) * fe + NW * n * 4,
        "ntt_scratch": max(NS * n, nscr(1) if k == 1 else 0) * fe,
        "domain": 3 * n * fe,
        "srs": W * (n + 3) * 64,
        "msm_scratch": max(ld.msm_scratch_bytes(n, NW, win, W), ld.msm_scratch_bytes(n + 3, NW, win, W)),
        "runtime": 1 << 30,
    }
    if k == 1:
        p.update(workspace=workspace(1) * fe, ntt_scratch2=0)
    else:
        p.update(batch_workspace=workspace(k) * fe, batch_ntt_scratch=nscr(k) * fe, batch_ntt_scratch2=0,
                 batch_msm_scratch=ld.msm_scratch_bytes(n + 3, k * NW, win, W))
    return p


def _full(parts: dict) -> dict:
    return {name: parts.get(name, 0) for name in PlonkKzgSnark.FOOTPRINT_PARTS}


@pytest.mark.parametrize("k", [1, 3, 17, 64])
def test_footprint_equals_the_restated_estimate(k):
    for log_n in range(2, 26):
        assert PlonkKzgSnark.footprint(log_n, k, compact=False) == _full(ld.footprint_parts(log_n, k)), (log_n, k)
        assert PlonkKzgSnark.footprint(log_n, k, compact=True) == _full(compact_footprint_parts(log_n, k)), (log_n, k)


def test_compact_rules_are_read_from_the_source():
    src = ld.plonk_source()
    with pytest.raises(AssertionError):
        compact_constants(src.replace("return NS + NW + (size_t)(NW + 2) * k;", "return NS + NW + (size_t)(NW + 1) * k;"))
    with pytest.raises(AssertionError):
        compact_constants(src.replace("s0 += NW)", "s0 += NS)"))


def test_compact_keys_fit_2_23_on_one_80gb_gpu():
    """A compact key and one proof of 2^23 need ≈ 45.7 GiB (≈ 52.6 GiB with the 15 % slack), a default one ≈ 110 GiB; at 2^24
    a compact key needs ≈ 89.9 GiB, over 80 GB before any slack."""
    est = {log_n: sum(compact_footprint_parts(log_n).values()) for log_n in (22, 23, 24)}
    default = {log_n: ld.footprint_bytes(log_n) for log_n in (22, 23, 24)}
    print({log_n: f"compact {v / 2**30:.2f} GiB, default {default[log_n] / 2**30:.2f} GiB" for log_n, v in est.items()})
    assert est[23] * SLACK < GB80 < default[23]
    assert est[24] > GB80
    for log_n in (22, 23, 24):
        assert est[log_n] < 0.45 * default[log_n]
    # the key alone: no 18 x 6n coset tables
    parts = compact_footprint_parts(23)
    assert parts["key"] < ld.footprint_parts(23)["key"] / 3 and parts["ntt_scratch2"] == 0
