"""Test infrastructure: the verifiers' inputs at every domain size and link layout, with the tampered twin of each.

One known-tau SRS of 2^17 + 3 powers (conftest's SRS_2_16_TAU) and its G2 pair (H, tau H), H the reference's G2 record.
Proofs: a `synth` circuit at every n = 2^2 ... 2^17 with 0, 1 and 5 public inputs where the circuit has room for them
(num_inputs <= n - 2), and a circuit whose every row is public at 2^2, 2^3 and 2^5; each proved by the oracle.  Each
honest proof has these twins, every one of them refused:
  * eval_bit    one bit of one evaluation flipped (the evaluation stays below r);
  * last_input  the last public input plus one (where there are public inputs);
  * swap_wires  the first two wire commitments swapped;
  * next_key    the proof under the verifying key of the next size with as many public inputs (for 2^17 the size below;
                none for the all-public circuits, whose neighbours have another input count).
Links: every layout of `link_layouts.CASES`, proved by the oracle, with two twins: the layout one offset further
(accepted only where the roots stay the same, the whole subgroup, or the polynomials are equal) and C1 and C2 swapped
(accepted only for equal polynomials).

The device verifiers check items two to a warp, (2i, 2i+1), and either may leave early, so the proofs and the links are
each ordered in pairs that cycle through honest/tampered, tampered/honest, honest/honest and tampered/tampered."""
from __future__ import annotations

import os
import random
from dataclasses import dataclass, field

import numpy as np

import bn254_pairing_py as pr
import link_layouts as ll
from renegade_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987  # conftest's SRS_2_16_TAU
R, MONT = ll.R, ll.MONT
LOG_NS = range(2, 18)
INPUTS = (0, 1, 5)
ALL_PUBLIC = (2, 3, 5)  # log n of the circuits whose every row is a public input
SRS_LEN = (1 << 17) + 3
PROOF_TWINS = ("eval_bit", "last_input", "swap_wires", "next_key")
LINK_TWINS = ("shifted", "swapped")
PAIRS = (("H", "T"), ("T", "H"), ("H", "H"), ("T", "T"))


@dataclass
class ProofItem:
    name: str
    log_n: int
    num_inputs: int
    key: tuple           # (log_n, num_inputs) of the verifying key it is checked against
    pi: np.ndarray       # (num_inputs, 4) Montgomery
    proof: np.ndarray    # (144,) the b200_proof words
    kind: str            # "honest" or one of PROOF_TWINS
    want: bool


@dataclass
class LinkItem:
    name: str
    case: ll.Case
    c1: np.ndarray
    c2: np.ndarray
    lp: np.ndarray       # (16,) the b200_link_proof words
    layout: tuple        # (alignment, offset, size)
    kind: str            # "honest" or one of LINK_TWINS
    want: bool


@dataclass
class Key:
    log_n: int
    num_inputs: int
    k: np.ndarray
    pk: dict             # the oracle's key: coefficients and the 13 selector and 5 sigma commitments


@dataclass
class Sweep:
    tau: np.ndarray      # tau in Montgomery limbs
    srs: np.ndarray
    h: np.ndarray
    tau_h: np.ndarray
    keys: dict = field(default_factory=dict)     # (log_n, num_inputs) -> Key
    proofs: list = field(default_factory=list)   # in pair order
    links: list = field(default_factory=list)    # in pair order


def shapes():
    """(log_n, num_inputs) of every honest proof"""
    out = [(lg, ni) for lg in LOG_NS for ni in INPUTS if ni <= (1 << lg) - 2]
    return out + [(lg, 1 << lg) for lg in ALL_PUBLIC]


def all_public_circuit(log_n: int, seed: int) -> synth.SynthCircuit:
    """Every row an IO gate (q_O = 1, w4 = the row's public input, the other wires the zero variable)"""
    n = 1 << log_n
    rnd = random.Random(seed)
    pub = [rnd.randrange(R) for _ in range(n)]
    sel = [[0] * n for _ in range(synth.N_SELECTORS)]
    sel[synth.Q_O] = [1] * n
    wires = [[0] * n for _ in range(4)] + [pub]
    # wires 0-3 of every row hold the zero variable: one cycle through them; each public input stays in place
    zeros = [w * n + j for w in range(4) for j in range(n)]
    perm = np.empty(5 * n, dtype=np.uint64)
    for a, b in zip(zeros, zeros[1:] + zeros[:1]):
        perm[a] = b
    perm[4 * n:] = np.arange(4 * n, 5 * n, dtype=np.uint64)
    return synth.SynthCircuit(
        log_n=log_n, num_inputs=n, k=synth.to_mont_array([pow(5, i, R) for i in range(5)]),
        selectors=np.stack([synth.to_mont_array(c) for c in sel]), perm=perm,
        wires=np.stack([synth.to_mont_array(c) for c in wires]), pub_inputs=synth.to_mont_array(pub), n_gates=n,
        selectors_int=sel, wires_int=wires, pub_inputs_int=pub)


def circuit(log_n: int, num_inputs: int) -> synth.SynthCircuit:
    seed = 0x5EE9 + 64 * log_n + num_inputs
    if num_inputs == 1 << log_n:
        return all_public_circuit(log_n, seed)
    return synth.synth_circuit(log_n, num_inputs=num_inputs, seed=seed, fill=0.5)


def g2_pair():
    """(H, tau H): the reference's G2 record and its multiple by TAU"""
    raw = np.fromfile(os.path.join(ROOT, "tests", "golden", "srs_g2.bin"), dtype=np.uint64)
    h = raw[:16].copy()
    tau_h = pr.encode_g2_mont(pr.g2_mul(pr.decode_g2_mont(h.tobytes(), 0), TAU % R))
    return h, np.frombuffer(tau_h, dtype=np.uint64).copy()


def _commit(oracle, srs, vals):
    xy, inf = oracle.msm(srs[:len(vals)], oracle.ints_to_array(vals))
    return np.zeros(8, dtype=np.uint64) if inf else xy


def _plus_one(limbs) -> np.ndarray:
    """the Montgomery limbs of (value + 1)"""
    x = int.from_bytes(np.asarray(limbs, dtype=np.uint64).tobytes(), "little")
    return np.frombuffer(((x + MONT % R) % R).to_bytes(32, "little"), dtype=np.uint64).copy()


def proof_twins(sw: Sweep, it: ProofItem, j: int):
    """the tampered twins of honest proof `it`, the j-th honest proof"""
    out = []
    p = it.proof.copy()
    e = j % 10                                # which of the 10 evaluations
    word = 104 + 4 * e + (j // 10) % 3        # a limb below the top one: the value stays below r
    p[word] ^= np.uint64(1) << np.uint64((7 * j) % 64)
    out.append(("eval_bit", it.key, it.pi, p))
    if it.num_inputs:
        pi = it.pi.copy()
        pi[-1] = _plus_one(pi[-1])
        out.append(("last_input", it.key, pi, it.proof))
    p = it.proof.copy()
    p[0:8], p[8:16] = it.proof[8:16], it.proof[0:8]
    out.append(("swap_wires", it.key, it.pi, p))
    if it.num_inputs != 1 << it.log_n:
        nxt = (it.log_n + 1 if it.log_n < LOG_NS[-1] else it.log_n - 1, it.num_inputs)
        assert nxt in sw.keys
        out.append(("next_key", nxt, it.pi, it.proof))
    return [ProofItem(f"{it.name}:{kind}", it.log_n, it.num_inputs, key, pi, p, kind, False)
            for kind, key, pi, p in out]


def link_items(oracle, srs, c: ll.Case, seed: int):
    a1, a2 = ll.pair(oracle, c, seed)
    c1, c2 = _commit(oracle, srs, a1), _commit(oracle, srs, a2)
    rc, lp, _ = oracle.plonk_link(ll.to_mont(a1), ll.to_mont(a2), c1, c2, c.alignment, c.offset, c.size, srs)
    assert rc == 0, c.name
    lp = lp.to_array()
    lay = (c.alignment, c.offset, c.size)
    keeps = c.identical or c.size == 1 << c.alignment  # one offset further: the same roots, or nothing to divide
    return [LinkItem(c.name, c, c1, c2, lp, lay, "honest", True),
            LinkItem(f"{c.name}:shifted", c, c1, c2, lp, (c.alignment, c.offset + 1, c.size), "shifted", keeps),
            LinkItem(f"{c.name}:swapped", c, c2, c1, lp, lay, "swapped", c.identical)]


def pair_order(items):
    """items reordered so that consecutive pairs cycle through PAIRS while both kinds last; an even count"""
    honest = [x for x in items if x.want]
    tampered = [x for x in items if not x.want]
    out = []
    t = 0
    while honest or tampered:
        for want in PAIRS[t % len(PAIRS)]:
            src = (honest if want == "H" else tampered) or honest or tampered
            if src:
                out.append(src.pop(0))
        t += 1
    if len(out) % 2:
        out.append(out[0])
    return out


def pair_kinds(wants):
    """the pair kinds ("HT", "TH", "HH", "TT") of a verdict list, pair by pair"""
    return ["".join("H" if w else "T" for w in wants[i:i + 2]) for i in range(0, len(wants) - 1, 2)]


_CACHE = {}


def build(oracle) -> Sweep:
    """The sweep, built once per process"""
    if "sweep" in _CACHE:
        return _CACHE["sweep"]
    tau = oracle.int_to_limbs(TAU % R * MONT % R)
    h, tau_h = g2_pair()
    sw = Sweep(tau, oracle.srs_from_tau(tau, SRS_LEN), h, tau_h)
    honest = []
    for lg, ni in shapes():
        circ = circuit(lg, ni)
        pk = oracle.plonk_preprocess(lg, circ.selectors, circ.perm, circ.k, sw.srs)
        sw.keys[(lg, ni)] = Key(lg, ni, circ.k, pk)
        bl = synth.splitmix_blinders(0xB1 + 64 * lg + ni)
        rc, proof, _, _ = oracle.plonk_prove(lg, ni, circ.k, pk, circ.wires, circ.pub_inputs, bl, sw.srs)
        assert rc == 0, (lg, ni)
        honest.append(ProofItem(f"2^{lg}/{ni}", lg, ni, (lg, ni), circ.pub_inputs.reshape(-1, 4), proof.to_array(),
                                "honest", True))
    proofs = []
    for j, it in enumerate(honest):
        proofs += [it] + proof_twins(sw, it, j)
    sw.proofs = pair_order(proofs)
    links = []
    for i, c in enumerate(ll.CASES):
        links += link_items(oracle, sw.srs, c, seed=0x51 + i)
    sw.links = pair_order(links)
    _CACHE["sweep"] = sw
    return sw


def vk_parts(sw: Sweep, it: ProofItem):
    """(log_n, num_inputs, k, selector_comms, sigma_comms) of the key `it` is checked against"""
    key = sw.keys[it.key]
    return key.log_n, key.num_inputs, key.k, key.pk["selector_comms"], key.pk["sigma_comms"]
