"""CPU tests of the drop-in boundary: the C-ABI library loads, exports exactly what
include/b200prover.h declares, fails loudly without a GPU (no CPU fallback), and its host-only
entry points (ptau parsing, partial-sum combination) behave like the reference's."""
import ctypes as C
import os
import subprocess
import sys
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "b200prover.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", src)))


def _gcc(src: str, path, *flags) -> None:
    path.with_suffix(".c").write_text(src)
    out = subprocess.run(["gcc", "-std=c11", "-Werror", "-I" + os.path.join(ROOT, "include"), *flags,
                          str(path.with_suffix(".c")), "-o", str(path)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def test_binding_matches_the_compiler(tmp_path):
    """The binding _lib derives from include/b200prover.h is what a C compiler makes of the header.  Every parsed
    signature initialises a pointer to the declared function, so a parse that differs from the declaration does not
    compile; every ctypes struct has the compiler's size and field offsets and sizes; every scalar type of the mapping
    has the compiler's size and signedness."""
    from renegade_b200 import _lib
    _, structs, funcs, _ = _lib.parse_header()
    assert header_symbols() == sorted(_lib.EXPORTS) and len(funcs) == len(_lib.EXPORTS)
    decls = [f"static {ret} (*const p_{name})({', '.join(t for _, t in args) or 'void'}) = {name};"
             for name, ret, args in funcs]
    _gcc('#include "b200prover.h"\n' + "\n".join(decls) + "\n", tmp_path / "signatures.o", "-c")

    lines = [f'printf("{t} %zu %d\\n", sizeof({t}), ({t})-1 < 0);' for t in _lib.SCALARS]
    lines.append('printf("void* %zu 0\\n", sizeof(void*));')
    for s, fields in structs.items():
        lines.append(f'printf("{s} %zu 0\\n", sizeof({s}));')
        lines += [f'printf("{s}.{f} %zu %zu\\n", offsetof({s}, {f}), sizeof((({s}*)0)->{f}));' for f, _, _ in fields]
    _gcc('#include <stdio.h>\n#include <stddef.h>\n#include "b200prover.h"\nint main(void) {\n' + "\n".join(lines) +
         "\nreturn 0;\n}\n", tmp_path / "layout")
    got = subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True, check=True).stdout.splitlines()

    want = [f"{t} {C.sizeof(ct)} {int(ct(-1).value < 0)}" for t, ct in _lib.SCALARS.items()]
    want.append(f"void* {C.sizeof(C.c_void_p)} 0")
    for s, fields in structs.items():
        cls = _lib.STRUCTS[s]
        assert [f for f, _ in cls._fields_] == [f for f, _, _ in fields]
        want.append(f"{s} {C.sizeof(cls)} 0")
        want += [f"{s}.{f} {getattr(cls, f).offset} {getattr(cls, f).size}" for f, _, _ in fields]
    assert got == want


def test_library_exports_every_declared_symbol():
    from renegade_b200 import _lib
    lib = _lib.load()
    for name in header_symbols():
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.b200_version()


def test_no_cpu_fallback():
    """Without a CUDA device the product path must fail loudly, not compute on the host."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the loud-failure path is the CPU container's")
    import renegade_b200 as rb
    from renegade_b200._lib import B200Error
    with pytest.raises(B200Error) as ei:
        rb.Context(0)
    assert ei.value.code == -6 and "no CPU fallback" in str(ei.value)


def test_product_does_not_import_oracle():
    """Nothing under renegade_b200/ may import, link or call anything under oracle/."""
    pkg = os.path.join(ROOT, "renegade_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", "Makefile")):
                txt = open(os.path.join(dirpath, f), errors="replace").read()
                for bad in ("oracle_c", "bn254_py", "bn254_oracle", "liboracle", "orc_"):
                    assert bad not in txt, (f, bad)


def test_srs_parse_ptau_host(srs_head):
    from renegade_b200 import _lib
    lib = _lib.load()
    buf = (C.c_char * len(srs_head)).from_buffer_copy(srs_head)
    rec, n = C.c_void_p(), C.c_size_t()
    rc = lib.b200_srs_parse_ptau(C.cast(buf, C.c_void_p), len(srs_head), C.byref(rec), C.byref(n))
    assert rc == 0 and n.value == 512
    assert rec.value - C.addressof(buf) == 80  # SURVEY.md §5.9: section 2 starts at byte 80
    # error behaviour mirrors srs.rs:74-118 (assertions there, error codes here)
    for mutate, msg in ((lambda b: b"xtau" + b[4:], "magic"),
                        (lambda b: b[:4] + (2).to_bytes(4, "little") + b[8:], "version"),
                        (lambda b: b[:8] + (10).to_bytes(4, "little") + b[12:], "sections"),
                        (lambda b: b[:28] + b"\x01" + b[29:], "modulus")):
        bad = mutate(srs_head)
        bbuf = (C.c_char * len(bad)).from_buffer_copy(bad)
        rc = lib.b200_srs_parse_ptau(C.cast(bbuf, C.c_void_p), len(bad), C.byref(rec), C.byref(n))
        assert rc == -4, msg
        assert msg in lib.b200_last_error().decode().lower()


def test_g1_sum_affine_host(oracle, pyoracle):
    """Host-side combination of per-GPU partial sums vs the oracle."""
    from renegade_b200.sharded import combine_partials
    py = pyoracle
    pts = oracle.known_dlog_bases(0xABCD, 5)
    rec = np.zeros((6, 9), dtype=np.uint64)
    rec[:5, :8] = pts
    rec[5, 8] = 1  # an identity partial
    out, inf = combine_partials(rec)
    a = py.splitmix_fr(0xABCD, 5)
    assert not inf and py.decode_g1_mont(out.tobytes(), 0) == py.g1_mul(py.G1_GEN, sum(a) % py.R)
    # P + (-P) = identity; P + P = 2P
    neg = pts[0].copy()
    neg[4:] = oracle.fp_binop("orc_fp_sub", oracle.FQ, np.zeros(4, dtype=np.uint64), pts[0, 4:])
    rec2 = np.zeros((2, 9), dtype=np.uint64)
    rec2[0, :8], rec2[1, :8] = pts[0], neg
    out, inf = combine_partials(rec2)
    assert inf and not out.any()
    rec2[1, :8] = pts[0]
    out, inf = combine_partials(rec2)
    assert py.decode_g1_mont(out.tobytes(), 0) == py.g1_mul(py.G1_GEN, 2 * a[0] % py.R)


def test_shard_range():
    from renegade_b200.sharded import shard_range
    for n in (0, 1, 7, 8, 1000, (1 << 17) + 3):
        for world in (1, 2, 3, 8):
            spans = [shard_range(n, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(spans[i][1] == spans[i + 1][0] for i in range(world - 1))
            sizes = [e - b for b, e in spans]
            assert max(sizes) - min(sizes) <= 1


def test_keccak256_known_answers(oracle):
    """Transcript hash of the product (C++) pinned by the Keccak-256 known answers, and equal to
    the oracle's independent C implementation on random lengths (block boundaries 135/136/137)."""
    from renegade_b200.backend import keccak256
    assert keccak256(b"").hex() == "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"
    assert keccak256(b"abc").hex() == "4e03657aea45a94fc7d47ba826c8d667c0d1e6e33a64a036ec44f58fa12d6c45"
    import random
    rnd = random.Random(7)
    for ln in (1, 55, 135, 136, 137, 271, 272, 273, 1000):
        msg = bytes(rnd.randrange(256) for _ in range(ln))
        assert keccak256(msg) == oracle.keccak256(msg), ln


def test_bad_arguments_return_error_codes():
    """The boundary never aborts or throws: NULL handles / pointers come back as B200_ERR_INVALID
    (SURVEY.md §5.3: a prover failure must surface as an error value)."""
    from renegade_b200 import _lib
    lib = _lib.load()
    out = (C.c_uint64 * 8)()
    inf = C.c_int(0)
    assert lib.b200_msm(None, None, 0, None, 0, 0, out, C.byref(inf)) == -1
    assert lib.b200_ntt(None, None, 10, 0, 0) == -1
    assert lib.b200_plonk_prove(None, None, None, None, None, None, None, None) == -1
    assert lib.b200_plonk_link(None, None, None, 0, None, 0, None, None, 8, 0, 4, None, None) == -1
    assert lib.b200_poseidon2_hash_batch(None, None, 1, 2, None) == -1
    assert lib.b200_init(0, None) == -1
    h = C.c_void_p()
    assert lib.b200_init(-3, C.byref(h)) in (-1, -6)   # bad ordinal (or no device at all on the CPU box)
    lib.b200_shutdown(None)           # tolerated
    lib.b200_bases_free(None, None)   # tolerated
    lib.b200_pk_free(None, None)


def test_pool_boundary_without_a_device():
    """The prover pool follows the same conventions: error values for NULL handles, NO_DEVICE (never a host
    fallback) when its contexts cannot be created."""
    import torch
    from renegade_b200 import _lib
    lib = _lib.load()
    t = C.c_uint64(0)
    assert lib.b200_pool_create(0, 0, C.byref(C.c_void_p())) == -1       # zero workers
    assert lib.b200_pool_create(0, 4, None) == -1
    assert lib.b200_pool_submit_prove(None, None, None, None, 0, None, None, None, C.byref(t)) == -1
    assert lib.b200_pool_submit_link(None, None, None, 0, None, 0, None, None, 8, 0, 4, None, C.byref(t)) == -1
    assert lib.b200_pool_wait(None, 1) == -1
    assert lib.b200_pool_wait_all(None) == -1
    assert lib.b200_pool_stats(None, None) == -1
    assert lib.b200_pool_workers(None) == 0
    assert not lib.b200_pool_ctx(None, 0)
    lib.b200_pool_destroy(None)  # tolerated
    if not torch.cuda.is_available():
        h = C.c_void_p()
        assert lib.b200_pool_create(0, 2, C.byref(h)) == -6 and not h.value
        assert b"no CPU fallback" in lib.b200_last_error()


def test_rust_shim_ffi_matches_the_header():
    """shim/gpu-prover/src/ffi.rs (what the Rust host links against) declares exactly the header's entry points with
    ABI-equivalent signatures.  The Rust file is parsed here independently of the generator and every type is mapped back
    to its C spelling."""
    from renegade_b200 import _lib
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_rust_ffi as gen
    opaque, structs, funcs, macros = gen.parse_header()
    src = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi.rs")).read()
    assert src == gen.generate(), "ffi.rs is stale: run python tools/gen_rust_ffi.py"
    block = src[src.index('extern "C" {'):]
    rust = {m.group(1): (m.group(2), m.group(3)) for m in
            re.finditer(r"pub fn (b200_\w+)\((.*?)\)(?: -> ([^;]+))?;", block)}
    assert sorted(rust) == sorted(f[0] for f in funcs) == sorted(_lib.EXPORTS)
    back = {"c_int": "int", "c_uint": "unsigned", "usize": "size_t", "u64": "uint64_t", "u8": "uint8_t", "f32": "float",
            "f64": "double", "c_char": "char", "c_void": "void"}

    def to_c(t):
        t = t.strip()
        ptrs = []
        while t.startswith("*"):
            kind, t = t.split(" ", 1)
            ptrs.append(kind)
        base = back.get(t, t)
        # innermost pointer's constness belongs to the pointee
        const = ptrs and ptrs[-1] == "*const"
        return ("const " if const else "") + base + "*" * len(ptrs)

    def canon(c):  # header spelling -> comparable form (arrays decay, outer `* const *` dropped)
        c = c.replace("unsigned int", "unsigned").replace(" * const *", "**").replace("* const *", "**")
        return c.replace(" *", "*").replace("* ", "*").strip()

    for name, ret, args in funcs:
        rargs, rret = rust[name]
        got = [to_c(a.split(":", 1)[1]) for a in rargs.split(", ") if a]
        want = [canon(t) for _, t in args]
        assert got == want, (name, got, want)
        assert (to_c(rret) if rret else "void") == canon(ret), (name, rret, ret)
    for k, v in macros.items():
        assert re.search(rf"pub const {k}: c_int = {v};", src)
    for sname, fields in structs.items():
        body = re.search(rf"pub struct {sname} \{{(.*?)\}}", src, flags=re.S).group(1)
        assert [f.strip() for f in body.strip().split(",\n") if f.strip()] == [f"pub {f}: {t}" for f, t in fields] or \
               [x.strip().rstrip(",") for x in body.strip().splitlines()] == [f"pub {f}: {t}" for f, t in fields]
