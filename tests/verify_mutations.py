"""Mutations of the verifiers' inputs, field by field: every one of them must be rejected.

Used by test_verify_encodings_cpu.py (the host verifiers, oracle proofs) and test_gpu_verify_encodings.py (the batch
verifier, device proofs).  An item is plain uint64 arrays, the bytes the C ABI takes:

    PlonkItem(k (5, 4), sel (13, 8), sig (5, 8), pi (n, 4), proof (144,))   verifying key, public inputs, b200_proof
    LinkItem(c1 (8,), c2 (8,), lp (16,), layout (alignment, offset, size))   b200_plonk_verify_link's arguments

Every field element is a Montgomery residue v = a 2^256 mod p in [0, p).  Each field is mutated on its own, into
  * an encoding outside the field: v + p, the largest v + m p below 2^256, and 2^256 - 1 (x and y of a point apart);
  * a wrong but canonical value: a point becomes the identity, -P, 2P or G; a scalar 0, r - 1 or a + 1;
and a link's layout moves by one in offset, size and alignment wherever the ABI takes the result."""
from collections import namedtuple

import numpy as np

import bn254_py as py

Q, R = py.Q, py.R
TOP = 1 << 256

PlonkItem = namedtuple("PlonkItem", "k sel sig pi proof")
LinkItem = namedtuple("LinkItem", "c1 c2 lp layout")
Mutation = namedtuple("Mutation", "label cls item")

NON_CANONICAL = ("plus_p", "max_multiple", "all_ones")
POINT_VALUES = ("identity", "neg", "double", "generator")
SCALAR_VALUES = ("zero", "minus_one", "plus_one")
LAYOUT = "layout"
CLASSES = NON_CANONICAL + POINT_VALUES + SCALAR_VALUES + (LAYOUT,)
MAX_ALIGNMENT = 28  # the largest alignment the link verifiers take

# b200_proof as uint64 words: the 13 G1 points (8 words each), then the 10 evaluations (4 words each)
PROOF_POINTS = ([("wires_poly_comms[%d]" % i, 8 * i) for i in range(5)] + [("prod_perm_poly_comm", 40)] +
                [("split_quot_poly_comms[%d]" % i, 48 + 8 * i) for i in range(5)] +
                [("opening_proof", 88), ("shifted_opening_proof", 96)])
PROOF_EVALS = ([("wires_evals[%d]" % i, 104 + 4 * i) for i in range(5)] +
               [("wire_sigma_evals[%d]" % i, 124 + 4 * i) for i in range(4)] + [("perm_next_eval", 140)])
PROOF_WORDS = 144
# b200_link_proof: quotient_commitment, opening_proof
LINK_POINTS = [("quotient_commitment", 0), ("opening_proof", 8)]


def to_int(words) -> int:
    return sum(int(w) << (64 * i) for i, w in enumerate(np.asarray(words, dtype=np.uint64).reshape(-1)))


def to_words(v: int) -> np.ndarray:
    assert 0 <= v < TOP
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def out_of_field(v: int, p: int) -> dict:
    """The three encodings of the Montgomery residue v (< p) that lie outside [0, p)."""
    assert 0 <= v < p
    return {"plus_p": v + p, "max_multiple": v + (TOP - 1 - v) // p * p, "all_ones": TOP - 1}


def point_values(xy) -> dict:
    """The canonical wrong values of the point with record xy (64 bytes, Montgomery); the identity is left out where
    the point is the identity, and so are -P and 2P, which are the identity too, and G where the point is G."""
    rec = np.asarray(xy, dtype=np.uint64).tobytes()
    p = None if not any(rec) else py.decode_g1_mont(rec, 0)
    out = {}
    if p is not None:
        out["identity"] = None
        out["neg"] = py.g1_neg(p)
        out["double"] = py.g1_add(p, p)
    if p != py.G1_GEN:
        out["generator"] = py.G1_GEN
    return {c: np.frombuffer(py.encode_g1_mont(v), dtype=np.uint64).copy() for c, v in out.items()}


def scalar_values(v_mont: int) -> dict:
    """The canonical wrong values of the Fr element v_mont (Montgomery): 0, r - 1 and a + 1, without the one it is."""
    a = py.from_mont(v_mont, R)
    out = {"zero": 0, "minus_one": R - 1, "plus_one": (a + 1) % R}
    return {c: py.to_mont(b, R) for c, b in out.items() if b != a}


def _point_mutations(label, words, off, make):
    """Mutations of the point at words[off:off + 8]; make(new words) builds the item."""
    out = []
    for coord, c_off in (("x", off), ("y", off + 4)):
        v = to_int(words[c_off:c_off + 4])
        for cls, enc in out_of_field(v, Q).items():
            w = words.copy()
            w[c_off:c_off + 4] = to_words(enc)
            out.append(("%s.%s:%s" % (label, coord, cls), cls, make(w)))
    for cls, rec in point_values(words[off:off + 8]).items():
        w = words.copy()
        w[off:off + 8] = rec
        out.append(("%s:%s" % (label, cls), cls, make(w)))
    return out


def _scalar_mutations(label, words, off, make):
    out = []
    v = to_int(words[off:off + 4])
    for cls, enc in list(out_of_field(v, R).items()) + list(scalar_values(v).items()):
        w = words.copy()
        w[off:off + 4] = to_words(enc)
        out.append(("%s:%s" % (label, cls), cls, make(w)))
    return out


def plonk_mutations(item: PlonkItem):
    """Every single-field mutation of a proof item: its 13 points, 10 evaluations, public inputs, and its verifying key's
    13 selector and 5 sigma commitments and 5 coset representatives k."""
    it = PlonkItem(*(np.ascontiguousarray(a, dtype=np.uint64) for a in item))
    assert it.proof.shape == (PROOF_WORDS,) and it.k.shape == (5, 4) and it.sel.shape == (13, 8)
    assert it.sig.shape == (5, 8) and it.pi.ndim == 2 and it.pi.shape[1] == 4
    out = []
    proof = lambda w: it._replace(proof=w)
    for name, off in PROOF_POINTS:
        out += _point_mutations("proof." + name, it.proof, off, proof)
    for name, off in PROOF_EVALS:
        out += _scalar_mutations("proof." + name, it.proof, off, proof)
    for label, attr, width, fn in (("pi", "pi", 4, _scalar_mutations), ("vk.k", "k", 4, _scalar_mutations),
                                   ("vk.selector_comms", "sel", 8, _point_mutations),
                                   ("vk.sigma_comms", "sig", 8, _point_mutations)):
        rows = getattr(it, attr)
        make = lambda w, attr=attr, shape=rows.shape: it._replace(**{attr: w.reshape(shape)})
        for i in range(rows.shape[0]):
            out += fn("%s[%d]" % (label, i), rows.reshape(-1), width * i, make)
    return [Mutation(*m) for m in _checked(it, out)]


def link_mutations(item: LinkItem):
    """Every single-field mutation of a link item: comm1, comm2, the proof's quotient commitment and opening, and the
    layout's offset, size and alignment +- 1 where the verifier takes it (size >= 1, alignment <= 28)."""
    it = LinkItem(np.ascontiguousarray(item.c1, dtype=np.uint64), np.ascontiguousarray(item.c2, dtype=np.uint64),
                  np.ascontiguousarray(item.lp, dtype=np.uint64), tuple(item.layout))
    assert it.c1.shape == (8,) and it.c2.shape == (8,) and it.lp.shape == (16,)
    out = []
    out += _point_mutations("link.comm1", it.c1, 0, lambda w: it._replace(c1=w))
    out += _point_mutations("link.comm2", it.c2, 0, lambda w: it._replace(c2=w))
    for name, off in LINK_POINTS:
        out += _point_mutations("link." + name, it.lp, off, lambda w: it._replace(lp=w))
    for j, name in enumerate(("alignment", "offset", "size")):
        for delta in (-1, 1):
            lay = list(it.layout)
            lay[j] += delta
            if min(lay) < 0 or lay[2] < 1 or lay[0] > MAX_ALIGNMENT:
                continue
            out.append(("link.layout.%s%+d" % (name, delta), LAYOUT, it._replace(layout=tuple(lay))))
    return [Mutation(*m) for m in _checked(it, out)]


def _bytes(item) -> bytes:
    return b"".join(a.tobytes() if isinstance(a, np.ndarray) else repr(a).encode() for a in item)


def _checked(honest, muts):
    """Every mutation changes the item, and no two of them are the same item."""
    seen = {_bytes(honest)}
    for label, cls, item in muts:
        assert cls in CLASSES, label
        b = _bytes(item)
        assert b not in seen, label
        seen.add(b)
    return muts


def representatives(muts, cls, count=3):
    """`count` mutations of class cls spread over the list (first, middle, last), for the small batches."""
    ms = [m for m in muts if m.cls == cls]
    assert ms, cls
    return [ms[(len(ms) - 1) * j // max(1, count - 1)] for j in range(count)]
