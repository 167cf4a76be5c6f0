"""ctypes binding of libb200prover.so, derived from its C ABI, include/b200prover.h, include/b200settlement.h,
include/b200verifyjobs.h, include/b200express.h, include/b200reserved.h, include/b200selftest.h, include/b200cancel.h and
include/b200compact.h.

The headers are parsed once, at import, and are the only description of the ABI here: `EXPORTS` lists the core
header's entry points in header order, `SETTLEMENT_EXPORTS` those of the settlement header, `VERIFY_JOB_EXPORTS` those of
the verification-job header, `EXPRESS_EXPORTS` those of the express-lane header, `RESERVED_EXPORTS` those of the reserved-SM header, `SELFTEST_EXPORTS` those of the self-test header, `CANCEL_EXPORTS` those of the cancellation header, `COMPACT_EXPORTS` those of the compact-key header (and `FOOTPRINT_PARTS` its one macro), `B200_OK` / `B200_ERR_*` are the `#define`s of the core header and of the cancellation header (B200_ERR_CANCELLED), `STRUCTS` holds one ctypes
class per struct of any header (by C name), and `load()` gives every entry point the argtypes / restype of its
declaration.  tools/gen_rust_ffi.py writes the Rust shim's ffi*.rs modules from the same parse, and tests/test_abi_cpu.py checks the parse, the struct layouts and the scalar types
against a C compiler.

The library is built in-tree by `__graft_entry__.build()` / `make -C renegade_b200/csrc`.
There is no CPU fallback: if the shared library is missing, or no CUDA device is visible, the
calls below raise — they never route to the oracle or to any host implementation.
"""
from __future__ import annotations

import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), "include", "b200prover.h")
SETTLEMENT_HEADER = os.path.join(os.path.dirname(_HERE), "include", "b200settlement.h")
VERIFY_JOB_HEADER = os.path.join(os.path.dirname(_HERE), "include", "b200verifyjobs.h")
EXPRESS_HEADER = os.path.join(os.path.dirname(_HERE), "include", "b200express.h")
RESERVED_HEADER = os.path.join(os.path.dirname(_HERE), "include", "b200reserved.h")
SELFTEST_HEADER = os.path.join(os.path.dirname(_HERE), "include", "b200selftest.h")
CANCEL_HEADER = os.path.join(os.path.dirname(_HERE), "include", "b200cancel.h")
COMPACT_HEADER = os.path.join(os.path.dirname(_HERE), "include", "b200compact.h")
# B200_LIB_PATH: developer knob to load an alternative build of the same library (tuning experiments)
LIB_PATH = os.environ.get("B200_LIB_PATH") or os.path.join(_HERE, "libb200prover.so")


def strip_comments(src: str) -> str:
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def _spell(ctype: str) -> str:
    """One spelling per C type: words and stars separated by single spaces ("const uint64_t * const *")."""
    return " ".join(ctype.replace("*", " * ").split())


def parse_header(path=HEADER):
    """-> (opaque struct names, {struct name: [(field, C type, array dims)]}, [(name, ret C type, [(arg name, arg C
    type)])], {macro: int}).  A parameter `T x[k]` is spelled `T *`; a field `T f[a][b]` is (f, T, (a, b))."""
    src = strip_comments(open(path).read())
    macros = {m.group(1): int(m.group(2).strip("()")) for m in re.finditer(r"#define\s+(B200_\w+)\s+(\(?-?\d+\)?)", src)}
    opaque = re.findall(r"typedef\s+struct\s+(\w+)\s+\1\s*;", src)
    structs = {}
    for body, name in re.findall(r"typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;", src, flags=re.S):
        fields = []
        for decl in body.split(";"):
            decl = " ".join(decl.split())
            if not decl:
                continue
            m = re.match(r"(.*?)(\w+)((?:\[\d+\])*)$", decl)
            dims = tuple(int(x) for x in re.findall(r"\[(\d+)\]", m.group(3)))
            fields.append((m.group(2), _spell(m.group(1)), dims))
        structs[name] = fields
    body = src[src.index('extern "C" {'):]
    funcs = []
    for ret, name, args in re.findall(r"\n\s*((?:const\s+)?[\w ]+?[\s\*]+)(b200_\w+)\s*\(([^;{}]*?)\)\s*;", body, flags=re.S):
        arglist = []
        args = " ".join(args.split())
        if args and args != "void":
            for a in args.split(","):
                a = a.strip()
                m = re.match(r"(.*?)(\w+)((?:\[\d*\])*)$", a)
                ctype, aname, arr = m.group(1).strip(), m.group(2), m.group(3)
                if arr:  # T name[k]  ==  T* name
                    ctype += "*" * arr.count("[")
                arglist.append((aname, _spell(ctype)))
        funcs.append((name, _spell(ret), arglist))
    return opaque, structs, funcs, macros


# C scalar type -> ctypes type.  Pointers are c_void_p (a `const char*` return is c_char_p); any other type is refused.
SCALARS = {"int": C.c_int, "unsigned": C.c_uint, "unsigned int": C.c_uint, "size_t": C.c_size_t, "uint64_t": C.c_uint64,
           "uint8_t": C.c_uint8, "float": C.c_float, "double": C.c_double}


def _ctype(ctype: str, ret: bool = False):
    if "*" in ctype:
        return C.c_char_p if ret and ctype == "const char *" else C.c_void_p
    if ret and ctype == "void":
        return None
    if ctype not in SCALARS:
        raise TypeError(f"{HEADER}: no ctypes type for the C type `{ctype}`")
    return SCALARS[ctype]


def _struct(name: str, fields) -> type:
    members = []
    for fname, ftype, dims in fields:
        t = _ctype(ftype)
        for k in reversed(dims):  # T f[a][b] -> (T * b) * a
            t = t * k
        members.append((fname, t))
    return type(name, (C.Structure,), {"_fields_": members})


for _h in (HEADER, SETTLEMENT_HEADER, VERIFY_JOB_HEADER, EXPRESS_HEADER, RESERVED_HEADER, SELFTEST_HEADER, CANCEL_HEADER,
           COMPACT_HEADER):
    if not os.path.exists(_h):
        raise ImportError(f"{_h} is missing: the binding of libb200prover is derived from it")
_, _structs, _funcs, _codes = parse_header()
_, _s_structs, _s_funcs, _ = parse_header(SETTLEMENT_HEADER)
_, _v_structs, _v_funcs, _ = parse_header(VERIFY_JOB_HEADER)
_, _e_structs, _e_funcs, _ = parse_header(EXPRESS_HEADER)
_, _r_structs, _r_funcs, _ = parse_header(RESERVED_HEADER)
_, _t_structs, _t_funcs, _ = parse_header(SELFTEST_HEADER)
_, _c_structs, _c_funcs, _c_codes = parse_header(CANCEL_HEADER)
_, _k_structs, _k_funcs, _k_macros = parse_header(COMPACT_HEADER)
FOOTPRINT_PARTS = _k_macros["B200_FOOTPRINT_PARTS"]  # entries of b200_plonk_footprint's out[]
_codes = {**_codes, **_c_codes}  # the code table: the core header's, then B200_ERR_CANCELLED
globals().update(_codes)  # B200_OK, B200_ERR_INVALID, ..., B200_ERR_UNSATISFIED, B200_ERR_CANCELLED
EXPORTS = [name for name, _, _ in _funcs]
SETTLEMENT_EXPORTS = [name for name, _, _ in _s_funcs]
VERIFY_JOB_EXPORTS = [name for name, _, _ in _v_funcs]
EXPRESS_EXPORTS = [name for name, _, _ in _e_funcs]
RESERVED_EXPORTS = [name for name, _, _ in _r_funcs]
SELFTEST_EXPORTS = [name for name, _, _ in _t_funcs]
CANCEL_EXPORTS = [name for name, _, _ in _c_funcs]
COMPACT_EXPORTS = [name for name, _, _ in _k_funcs]
STRUCTS = {name: _struct(name, fields) for name, fields in {**_structs, **_s_structs, **_v_structs, **_e_structs,
                                                        **_r_structs, **_t_structs, **_c_structs, **_k_structs}.items()}
_SIGNATURES = {name: ([_ctype(t) for _, t in args], _ctype(ret, ret=True))
               for name, ret, args in _funcs + _s_funcs + _v_funcs + _e_funcs + _r_funcs + _t_funcs + _c_funcs + _k_funcs}


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libb200prover error {code}: {msg}")
        self.code = code


_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the proving path)")
    lib = C.CDLL(LIB_PATH)
    for name, (argtypes, restype) in _SIGNATURES.items():
        fn = getattr(lib, name)  # raises AttributeError if a declared symbol is not exported
        fn.argtypes, fn.restype = argtypes, restype
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != B200_OK:
        raise B200Error(rc, (load().b200_last_error() or b"").decode(errors="replace"))
