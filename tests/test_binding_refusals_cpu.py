"""The Python binding's proof and link inputs, without a device: every entry point that takes a proof or a link refuses
each malformed input before any library call, with its own exception class and a message that names the entry point,
the item, proof or link, and the counts; and valid input reaches the library as the committed record of its arguments
(`golden/binding_calls.json`: every scalar, and every input array the pointers name)."""
import ctypes as C
import json
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

from renegade_b200 import _lib
from renegade_b200.backend import (B200LinkProof, B200Proof, Context, GroupLayout, LinkingHint, PlonkKzgSnark, ProverBox,
                                   ProverPool, link_proofs, link_proofs_batch, prove_raw)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "binding_calls.json")
INVALID = _lib.B200_ERR_INVALID
N, NUM_INPUTS, NUM_VARS = 16, 2, 20  # the key every case proves against: 2^4 rows, 2 public inputs, 20 variables
WIRED, TABLES = 0x10, 0x20  # box key handles: with wiring, and made by preprocess


class _NoLibrary:
    """Stands in for the loaded library: any call means a check did not run first."""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called before the arguments were checked")


class _Srs:
    """Stands in for Bases: 40 powers."""
    _h = C.c_void_p(0x5)

    def __len__(self):
        return 40


def _key(num_vars=NUM_VARS):
    return SimpleNamespace(_h=C.c_void_p(0x1000), log_n=4, domain_size=N, num_inputs=NUM_INPUTS, num_vars=num_vars)


def _objects(lib):
    """(context, pool, box) over the stand-in library `lib`, made without a device."""
    ctx = Context.__new__(Context)
    ctx._lib, ctx._h, ctx.device = lib, C.c_void_p(0xC7), 0
    pool = ProverPool.__new__(ProverPool)
    pool._lib, pool._h, pool._jobs, pool._borrowed = lib, C.c_void_p(0x900), {}, []
    box = ProverBox.__new__(ProverBox)
    box._lib, box._h, box._jobs, box.devices = lib, C.c_void_p(0xB0), {}, [0]
    box._shapes = {WIRED: _key(), TABLES: _key(num_vars=0)}
    return ctx, pool, box


def _u64(n, seed):
    return (np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(seed)).reshape(-1, 4)


def _inputs():
    """Valid inputs, distinct in content: a wire table, public inputs, blinders, a witness, hints and a layout."""
    return SimpleNamespace(wires=_u64(5 * N * 4, 1).reshape(5, N, 4), pub=_u64(NUM_INPUTS * 4, 2), bl=_u64(17 * 4, 3),
                           wit=_u64(NUM_VARS * 4, 4), hint=LinkingHint(_u64((N + 2) * 4, 5), _u64(8, 6).reshape(-1)),
                           hint2=LinkingHint(_u64(12 * 4, 7), _u64(8, 8).reshape(-1)), lay=GroupLayout(4, 2, 3))


# ---- the refusal matrix ---------------------------------------------------------------------------------------------
# Each entry point is a function of one proof's (or link's) parts.  A batch or bundle entry point puts the parts in item
# (proof, link) 1, after a valid item 0, so the message must name that index.

def _entry_points():
    ctx, pool, box = _objects(_NoLibrary())
    srs, pk, x = _Srs(), _key(), _inputs()
    nokey = _key(num_vars=0)
    ok = lambda: [(x.hint, x.lay)]  # noqa: E731
    tables = {  # name: (where, exception, call(wires, pub, bl, links)), wires an array where the entry point takes one
        "prove_with_link_hint": ("prove_with_link_hint", ValueError,
                                 lambda w, p, b, _: PlonkKzgSnark.prove_with_link_hint(ctx, pk, w, p, b)),
        "prove_raw": ("prove_raw", ValueError, lambda w, p, b, _: prove_raw(ctx, pk, 0x7000, p, b)),
        "prove_batch": ("prove_batch: item 1", ValueError,
                        lambda w, p, b, _: PlonkKzgSnark.prove_batch(ctx, pk, [x.wires, w], [x.pub, p], [x.bl, b])),
        "prove_settlement": ("prove_settlement", _lib.B200Error,
                             lambda w, p, b, l: PlonkKzgSnark.prove_settlement(ctx, srs, pk, w, p, b, l)),
        "submit_prove": ("submit_prove", _lib.B200Error, lambda w, p, b, _: pool.submit_prove(pk, 0x7000, p, b)),
        "submit_prove_batch": ("submit_prove_batch: item 1", ValueError,
                               lambda w, p, b, _: pool.submit_prove_batch(pk, [x.wires, w], [x.pub, p], [x.bl, b])),
        "submit_bundle": ("submit_bundle: proof 1", _lib.B200Error,
                          lambda w, p, b, _: pool.submit_bundle(srs, [(pk, 0x7000, x.pub, x.bl), (pk, 0x7000, p, b)], [])),
        "submit_settlement": ("submit_settlement", _lib.B200Error,
                              lambda w, p, b, l: pool.submit_settlement(srs, pk, w, p, b, l)),
        "box.submit_prove": ("box.submit_prove", _lib.B200Error,
                             lambda w, p, b, _: box.submit_prove(C.c_void_p(WIRED), 0x7000, p, b)),
        "box.submit_bundle": ("box.submit_bundle: proof 1", _lib.B200Error,
                              lambda w, p, b, _: box.submit_bundle(None, [(WIRED, 0x7000, x.pub, x.bl), (WIRED, 0x7000, p, b)],
                                                                   [])),
        "box.submit_settlement": ("box.submit_settlement", _lib.B200Error,
                                  lambda w, p, b, l: box.submit_settlement(None, C.c_void_p(WIRED), w, p, b, l)),
    }
    witnesses = {  # name: (where, exception, call(key, witness, bl, links)); key is pk or the key without wiring
        "prove_witness": ("prove_witness", ValueError, lambda k, w, b, _: PlonkKzgSnark.prove_witness(ctx, k, w, b)),
        "prove_witness_batch": ("prove_witness_batch: item 1", ValueError,
                                lambda k, w, b, _: PlonkKzgSnark.prove_witness_batch(ctx, k, [x.wit, w], [x.bl, b])),
        "prove_settlement_witness": ("prove_settlement_witness", _lib.B200Error,
                                     lambda k, w, b, l: PlonkKzgSnark.prove_settlement_witness(ctx, srs, k, w, b, l)),
        "submit_prove_witness": ("submit_prove_witness", _lib.B200Error,
                                 lambda k, w, b, _: pool.submit_prove_witness(k, w, b)),
        "submit_prove_witness_batch": ("submit_prove_witness_batch: item 1", _lib.B200Error,
                                       lambda k, w, b, _: pool.submit_prove_witness_batch(k, [x.wit, w], [x.bl, b])),
        "submit_bundle_witness": ("submit_bundle_witness: proof 1", _lib.B200Error,
                                  lambda k, w, b, _: pool.submit_bundle_witness(srs, [(pk, x.wit, x.bl), (k, w, b)], [])),
        "submit_settlement_witness": ("submit_settlement_witness", _lib.B200Error,
                                      lambda k, w, b, l: pool.submit_settlement_witness(srs, k, w, b, l)),
        "box.submit_prove_witness": ("box.submit_prove_witness", _lib.B200Error,
                                     lambda k, w, b, _: box.submit_prove_witness(_box_key(k), w, b)),
        "box.submit_bundle_witness": ("box.submit_bundle_witness: proof 1", _lib.B200Error,
                                      lambda k, w, b, _: box.submit_bundle_witness(None, [(WIRED, x.wit, x.bl),
                                                                                          (_box_key(k), w, b)], [])),
        "box.submit_settlement_witness": ("box.submit_settlement_witness", _lib.B200Error,
                                          lambda k, w, b, l: box.submit_settlement_witness(None, _box_key(k), w, b, l)),
    }
    links = {  # name: (where, exception, call(hint, layout)) for the entry points that link two hints
        "link_proofs": ("link_proofs: the link", ValueError, lambda h, lay: link_proofs(ctx, srs, x.hint2, h, lay)),
        "link_proofs_batch": ("link_proofs_batch: item 1", ValueError,
                              lambda h, lay: link_proofs_batch(ctx, srs, [(x.hint2, x.hint, x.lay), (x.hint2, h, lay)])),
        "submit_link": ("submit_link: the link", ValueError, lambda h, lay: pool.submit_link(srs, x.hint2, h, lay)),
        "submit_link_batch": ("submit_link_batch: item 1", ValueError,
                              lambda h, lay: pool.submit_link_batch(srs, [(x.hint2, x.hint, x.lay), (x.hint2, h, lay)])),
    }
    # the settlements link a stored hint to the statement's own: link 1, after a valid link 0
    for name, (where, exc, call) in list(tables.items()):
        if "settlement" in name:
            links[name] = (where + ": link 1", exc, lambda h, lay, call=call: call(x.wires, x.pub, x.bl, ok() + [(h, lay)]))
    for name, (where, exc, call) in list(witnesses.items()):
        if "settlement" in name:
            links[name] = (where + ": link 1", exc, lambda h, lay, call=call: call(pk, x.wit, x.bl, ok() + [(h, lay)]))
    return x, pk, nokey, ok, tables, witnesses, links


def _box_key(k):
    return C.c_void_p(TABLES if k.num_vars == 0 else WIRED)


def _rows():
    x, pk, nokey, ok, tables, witnesses, links = _entry_points()
    bl16 = x.bl[:16]
    rows = []
    for name, (where, exc, call) in tables.items():
        rows.append((name, "16 blinders", exc, rf"{where} has 16 blinders, the prover draws 17",
                     lambda call=call: call(x.wires, x.pub, bl16, ok())))
        for n in (NUM_INPUTS - 1, NUM_INPUTS + 1):
            rows.append((name, f"{n} public inputs", exc, rf"{where} has {n} public inputs for a key with {NUM_INPUTS}",
                         lambda call=call, n=n: call(x.wires, _u64(4 * n, 9), x.bl, ok())))
        if name in ("prove_with_link_hint", "prove_batch", "submit_prove_batch") or "settlement" in name:
            rows.append((name, "wire table one row short", exc,
                         rf"{where}: the wire table has {5 * N - 1} elements, the key needs 5 x {N}",
                         lambda call=call: call(x.wires.reshape(-1, 4)[1:], x.pub, x.bl, ok())))
    for name, (where, exc, call) in witnesses.items():
        rows.append((name, "16 blinders", exc, rf"{where} has 16 blinders, the prover draws 17",
                     lambda call=call: call(pk, x.wit, bl16, ok())))
        rows.append((name, "witness one element short", exc,
                     rf"{where}: the witness has {NUM_VARS - 1} elements, the key takes {NUM_VARS}",
                     lambda call=call: call(pk, x.wit[1:], x.bl, ok())))
        first = where.replace("item 1", "item 0")  # a batch has one key: its first item is refused
        rows.append((name, "key without wiring", _lib.B200Error, rf"{first} holds no wiring",
                     lambda call=call: call(nokey, x.wit, x.bl, ok())))
    for name, (where, exc, call) in links.items():
        hint = "hint" if "settlement" in name else "hint_b"
        rows.append((name, "4-limb hint commitment", exc, rf"{where}'s {hint} commitment must be 8 limbs \(x \|\| y\), not 4",
                     lambda call=call: call(LinkingHint(x.hint.linking_wire_poly, x.hint.linking_wire_comm[:4]), x.lay)))
        rows.append((name, "size 0", exc, rf"{where}'s group of 0 roots does not fit polynomials of {N + 2} coefficients",
                     lambda call=call: call(x.hint, GroupLayout(4, 2, 0))))
        rows.append((name, "alignment 29", exc, rf"{where} has alignment 29 and offset 2 \(0 <= alignment <= 28",
                     lambda call=call: call(x.hint, GroupLayout(29, 2, 3))))
        rows.append((name, "size 2^a + 1", exc, rf"{where}'s group of 17 roots does not fit the 2\^4 roots of unity",
                     lambda call=call: call(x.hint, GroupLayout(4, 2, 17))))
    # the verifiers take a link as (comm_a, comm_b, proof, layout): link 1, after a valid link 0
    h, tau_h = _u64(16, 10).reshape(-1), _u64(16, 11).reshape(-1)
    verifiers = {
        "verify_each": lambda links: PlonkKzgSnark.verify_each(_objects(_NoLibrary())[0], [], [], [], links, g2=(h, tau_h)),
        "batch_verify": lambda links: PlonkKzgSnark.batch_verify(_objects(_NoLibrary())[0], [], [], [], links, g2=(h, tau_h)),
        "submit_verify": lambda links: _objects(_NoLibrary())[1].submit_verify([], [], [], links, g2=(h, tau_h)),
        "box.submit_verify": lambda links: _objects(_NoLibrary())[2].submit_verify([], [], [], links, combined=True,
                                                                                  g2=(h, tau_h)),
    }
    for name, call in verifiers.items():
        link = lambda lay: (x.hint.linking_wire_comm, x.hint2.linking_wire_comm, B200LinkProof(), lay)  # noqa: E731
        for a, size in ((4, 17), (0, 2), (28, (1 << 28) + 1), (4, 1 << 63)):
            rows.append((name, f"size {size} at alignment {a}", ValueError,
                         rf"{name}: link 1's group of {size} roots does not fit the 2\^{a} roots of unity",
                         lambda call=call, a=a, size=size: call([link(x.lay), link(GroupLayout(a, 5, size))])))
    _, pool, box = _objects(_NoLibrary())
    two = lambda k, ptr: [(k, ptr, x.pub, x.bl)] * 2  # noqa: E731
    outside = [(0, 1, x.lay), (1, 2, x.lay)]
    for name, call in (("submit_bundle", lambda: pool.submit_bundle(_Srs(), two(pk, 0x7000), outside)),
                       ("submit_bundle_witness", lambda: pool.submit_bundle_witness(_Srs(), [(pk, x.wit, x.bl)] * 2, outside)),
                       ("box.submit_bundle", lambda: box.submit_bundle(None, two(WIRED, 0x7000), outside)),
                       ("box.submit_bundle_witness",
                        lambda: box.submit_bundle_witness(None, [(WIRED, x.wit, x.bl)] * 2, outside))):
        rows.append((name, "link outside the bundle", _lib.B200Error,
                     rf"{name}: link 1 names proof \(1, 2\) of a bundle of 2", call))
    return rows


ROWS = _rows()


@pytest.mark.parametrize("row", ROWS, ids=[f"{r[0]}-{r[1]}" for r in ROWS])
def test_every_refusal_runs_before_the_library(row):
    _, _, exc, match, call = row
    with pytest.raises(Exception) as err:
        call()
    assert type(err.value) is exc, f"{type(err.value).__name__}: {err.value}"
    if exc is _lib.B200Error:
        assert err.value.code == INVALID
    assert re.search(match, str(err.value)), str(err.value)


# ---- what valid input sends to the library --------------------------------------------------------------------------

class _Recorder:
    """Stands in for the loaded library: records each call's arguments by the real signature and returns B200_OK.  A
    pointer is recorded as the name of the input array it points to, the contents of the item or entry array it points
    to, "out" for any other buffer, or None."""

    def __init__(self, known):
        self.lib, self.known, self.calls = _lib.load(), known, []

    def __getattr__(self, name):
        argtypes = getattr(self.lib, name).argtypes

        def call(*args):
            self.calls.append([name] + [self._arg(a, t) for a, t in zip(args, argtypes)])
            return _lib.B200_OK
        return call

    def _pointer(self, v):
        if v is None or isinstance(v, int):
            a = v or 0
        elif isinstance(v, C.c_void_p):
            a = v.value or 0
        else:
            obj = v._obj if type(v).__name__ == "CArgObject" else v.contents if isinstance(v, C._Pointer) else v
            if isinstance(obj, C.Array):
                return [self._struct(e) if isinstance(e, C.Structure) else e for e in obj]
            if isinstance(obj, C.Structure) and not isinstance(obj, (B200Proof, B200LinkProof)):
                return self._struct(obj)
            a = C.addressof(obj)
        return self.known.get(a, "out") if a else None

    def _struct(self, s):
        return {f: self._pointer(getattr(s, f)) if t is C.c_void_p else int(getattr(s, f)) for f, t in s._fields_}

    def _arg(self, v, t):
        return self._pointer(v) if t is C.c_void_p else int(getattr(v, "value", v))


def _record_calls():
    """{case: the library calls it made} for one valid input of every entry point."""
    known = {}
    rec = _Recorder(known)
    ctx, pool, box = _objects(rec)
    srs, pk, x = _Srs(), _key(), _inputs()
    for k, v in vars(x).items():
        for label, a in ((k, v), (k + ".poly", getattr(v, "linking_wire_poly", None)),
                         (k + ".comm", getattr(v, "linking_wire_comm", None))):
            if isinstance(a, np.ndarray):
                known[a.ctypes.data] = label
    known.update({0x7000: "wires@", 0x7100: "witness@", 0x7200: "poly@", ctx._h.value: "ctx", pool._h.value: "pool",
                  box._h.value: "box", srs._h.value: "srs", pk._h.value: "pk", WIRED: "box pk"})
    addr_hint = LinkingHint((0x7200, 30), x.hint2.linking_wire_comm)
    links = [(x.hint2, x.lay), (addr_hint, GroupLayout(5, 0, 7))]
    triples = [(x.hint2, x.hint, x.lay), (addr_hint, x.hint, GroupLayout(5, 1, 9))]
    bundle_links = [(0, 1, x.lay), (1, 0, GroupLayout(3, 1, 2))]
    wk = C.c_void_p(WIRED)
    cases = {
        "prove_with_link_hint": lambda: PlonkKzgSnark.prove_with_link_hint(ctx, pk, x.wires, x.pub, x.bl, want_challenges=True),
        "prove_raw": lambda: prove_raw(ctx, pk, 0x7000, x.pub, x.bl),
        "prove_witness": lambda: PlonkKzgSnark.prove_witness(ctx, pk, x.wit, x.bl, want_challenges=True),
        "prove_witness@": lambda: PlonkKzgSnark.prove_witness(ctx, pk, 0x7100, x.bl),
        "prove_batch": lambda: PlonkKzgSnark.prove_batch(ctx, pk, [x.wires, 0x7000], [x.pub, x.pub], [x.bl, x.bl],
                                                         link_hints=True, want_challenges=True),
        "prove_witness_batch": lambda: PlonkKzgSnark.prove_witness_batch(ctx, pk, [x.wit, 0x7100], [x.bl, x.bl],
                                                                         link_hints=True, want_challenges=True),
        "prove_settlement": lambda: PlonkKzgSnark.prove_settlement(ctx, srs, pk, x.wires, x.pub, x.bl, links),
        "prove_settlement_witness": lambda: PlonkKzgSnark.prove_settlement_witness(ctx, srs, pk, x.wit, x.bl, links),
        "link_proofs": lambda: link_proofs(ctx, srs, x.hint2, x.hint, x.lay),
        "link_proofs_batch": lambda: link_proofs_batch(ctx, srs, triples),
        "submit_prove": lambda: pool.submit_prove(pk, 0x7000, x.pub, x.bl, with_link_poly=True),
        "submit_prove_witness": lambda: pool.submit_prove_witness(pk, x.wit, x.bl, with_link_poly=True),
        "submit_prove_batch": lambda: pool.submit_prove_batch(pk, [x.wires, 0x7000], [x.pub, x.pub], [x.bl, x.bl],
                                                              link_hints=True),
        "submit_prove_witness_batch": lambda: pool.submit_prove_witness_batch(pk, [x.wit, 0x7100], [x.bl, x.bl]),
        "submit_bundle": lambda: pool.submit_bundle(srs, [(pk, 0x7000, x.pub, x.bl)] * 2, bundle_links),
        "submit_bundle_witness": lambda: pool.submit_bundle_witness(srs, [(pk, x.wit, x.bl), (pk, 0x7100, x.bl)],
                                                                    bundle_links),
        "submit_settlement": lambda: pool.submit_settlement(srs, pk, 0x7000, x.pub, x.bl, links),
        "submit_settlement_witness": lambda: pool.submit_settlement_witness(srs, pk, x.wit, x.bl, links),
        "submit_link": lambda: pool.submit_link(srs, x.hint2, x.hint, x.lay),
        "submit_link_batch": lambda: pool.submit_link_batch(srs, triples),
        "box.submit_prove": lambda: box.submit_prove(wk, 0x7000, x.pub, x.bl),
        "box.submit_prove_witness": lambda: box.submit_prove_witness(wk, 0x7100, x.bl, with_link_poly=True),
        "box.submit_bundle": lambda: box.submit_bundle(srs._h, [(WIRED, 0x7000, x.pub, x.bl)] * 2, bundle_links),
        "box.submit_bundle_witness": lambda: box.submit_bundle_witness(srs._h, [(WIRED, x.wit, x.bl)] * 2, bundle_links),
        "box.submit_settlement": lambda: box.submit_settlement(srs._h, wk, x.wires, x.pub, x.bl, links),
        "box.submit_settlement_witness": lambda: box.submit_settlement_witness(srs._h, wk, x.wit, x.bl, links),
    }
    out = {}
    for name, call in cases.items():
        rec.calls.clear()
        call()
        out[name] = json.loads(json.dumps(rec.calls))
    return out


def test_valid_input_reaches_the_library_unchanged():
    with open(GOLDEN) as f:
        want = json.load(f)
    got = _record_calls()
    assert sorted(got) == sorted(want)
    for name in want:
        assert got[name] == want[name], name


if __name__ == "__main__":  # writes the record the test compares against
    with open(GOLDEN, "w") as f:
        json.dump(_record_calls(), f, indent=1, sort_keys=True)
        f.write("\n")
