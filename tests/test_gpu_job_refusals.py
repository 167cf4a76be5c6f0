"""GPU: every proof and link job refuses a malformed item in the same words on each layer that takes it.  For each job kind
(prove, prove_witness, prove_batch, prove_witness_batch, link, link_batch, bundle, bundle_witness, settlement,
settlement_witness) each required pointer of an item is NULL in turn, a witness job gets a key without wiring, a key with
public inputs gets none, and num_inputs differs from the key's where the ABI carries it.  The context call, the pool submit
and, for one case per kind, the box submit each return B200_ERR_INVALID, name the field in b200_last_error(), queue nothing,
write no output and launch no kernel."""
import ctypes as C

import numpy as np
import pytest

from renegade_b200 import _lib, synth
from renegade_b200.backend import PlonkKzgSnark, ProverBox, ProverPool
from test_gpu_prove_witness import TAU, load_srs
from test_gpu_verify_jobs import pool_stats

pytestmark = pytest.mark.gpu
INVALID = _lib.B200_ERR_INVALID
S = _lib.STRUCTS
LOG_N, NUM_INPUTS = 5, 2
ALIGNMENT, OFFSET, SIZE = 2, 1, 3  # a valid link group for polynomials of n + 2 coefficients
MARK = 0xEE


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def addr(x):
    return C.cast(C.pointer(x), C.c_void_p)


class Env:
    """A 2^5 circuit's keys with and without wiring on the session context, a one-worker pool and a one-device box with the
    same two keys, and every input a job reads."""

    def __init__(self, ctx, oracle, pyoracle):
        c = self.circ = synth.synth_circuit(LOG_N, num_inputs=NUM_INPUTS, seed=21)
        self.ctx, self.lib = ctx, ctx._lib
        self.bases = load_srs(ctx, oracle, pyoracle, c.n)
        self.pk = {"tables": PlonkKzgSnark.preprocess(ctx, self.bases, c.log_n, c.num_inputs, c.selectors, c.perm, c.k),
                   "wiring": PlonkKzgSnark.preprocess_wiring(ctx, self.bases, c.log_n, c.num_inputs, c.selectors, c.wire_vars,
                                                             c.num_vars, c.k)}
        self.pool = ProverPool(0, workers=1)
        self.box = ProverBox([0], workers_per_device=1)
        tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
        self.box_srs = self.box.load_srs(oracle.srs_from_tau(tau, c.n + 3))
        self.box_pk = {"tables": self.box.preprocess(self.box_srs, c.log_n, c.num_inputs, c.selectors, c.perm, c.k),
                       "wiring": self.box.preprocess_wiring(self.box_srs, c.log_n, c.num_inputs, c.selectors, c.wire_vars,
                                                            c.num_vars, c.k)}
        self.wires = np.ascontiguousarray(c.wires, dtype=np.uint64)
        self.pub = np.ascontiguousarray(c.pub_inputs, dtype=np.uint64)
        self.wit = np.ascontiguousarray(c.witness, dtype=np.uint64)
        self.bl = synth.splitmix_blinders(3)
        self.poly = np.zeros((c.n + 2, 4), dtype=np.uint64)
        self.comm = np.zeros(8, dtype=np.uint64)

    def free(self):
        for name in self.box_pk:
            self.box.free_pk(self.box_pk[name])
            self.pk[name].free()
        self.box.free_srs(self.box_srs)
        self.box.close()
        self.pool.close()
        self.bases.free()


@pytest.fixture(scope="module")
def env(ctx, oracle, pyoracle):
    e = Env(ctx, oracle, pyoracle)
    yield e
    e.free()


class Outs:
    """Every output a job may write, holding values that a refused call leaves as they are."""

    def __init__(self, n):
        self.proofs = [S["b200_proof"]() for _ in range(2)]
        self.link_proofs = [S["b200_link_proof"]() for _ in range(2)]
        self.polys = [np.full((n + 2, 4), MARK, dtype=np.uint64) for _ in range(2)]
        self.pubs = [np.full((NUM_INPUTS, 4), MARK, dtype=np.uint64) for _ in range(2)]
        self.etas = [np.full(4, MARK, dtype=np.uint64) for _ in range(2)]
        self.challenges = np.full((6, 4), MARK, dtype=np.uint64)
        self.statuses = (C.c_int * 2)(99, 99)
        self.ticket = C.c_uint64(7)

    def untouched(self):
        return (all(bytes(x) == bytes(C.sizeof(x)) for x in self.proofs + self.link_proofs) and
                all((a == MARK).all() for a in self.polys + self.pubs + self.etas + [self.challenges]) and
                list(self.statuses) == [99, 99] and self.ticket.value == 7)


def items(struct, k, fields, bad):
    """k items of `struct`: item i has fields(i), and item 1 also the malformed fields `bad`"""
    arr = (S[struct] * max(k, 1))()
    for i in range(k):
        arr[i] = S[struct](**{**fields(i), **(bad if i == 1 else {})})
    return arr


# Each kind: (env, outputs, the malformed fields) -> {layer: call}.  Keys of `bad` that are not fields of the item: "pk"
# (which key: "tables" or "wiring"), "k" (batch size) and "link.<field>" (a settlement link's field).
def prove(e, o, bad):
    f = {"pk": "tables", "wires": ptr(e.wires), "pub_inputs": ptr(e.pub), "num_inputs": NUM_INPUTS, "blinders": ptr(e.bl),
         "proof": addr(o.proofs[0]), **bad}
    args = (f["wires"], f["pub_inputs"], f["num_inputs"], f["blinders"], f["proof"], ptr(o.polys[0]), C.byref(o.ticket))
    return {"context": lambda: e.lib.b200_plonk_prove(e.ctx._h, e.pk[f["pk"]]._h, f["wires"], f["pub_inputs"], f["blinders"],
                                                      f["proof"], ptr(o.polys[0]), ptr(o.challenges)),
            "pool": lambda: e.lib.b200_pool_submit_prove(e.pool._h, e.pk[f["pk"]]._h, *args),
            "box": lambda: e.lib.b200_box_submit_prove(e.box._h, e.box_pk[f["pk"]], *args)}


def prove_witness(e, o, bad):
    f = {"pk": "wiring", "witness": ptr(e.wit), "blinders": ptr(e.bl), "proof": addr(o.proofs[0]), **bad}
    args = (f["witness"], f["blinders"], f["proof"], ptr(o.polys[0]))
    return {"context": lambda: e.lib.b200_plonk_prove_witness(e.ctx._h, e.pk[f["pk"]]._h, *args, ptr(o.challenges),
                                                              ptr(o.pubs[0])),
            "pool": lambda: e.lib.b200_pool_submit_prove_witness(e.pool._h, e.pk[f["pk"]]._h, *args, ptr(o.pubs[0]),
                                                                 C.byref(o.ticket)),
            "box": lambda: e.lib.b200_box_submit_prove_witness(e.box._h, e.box_pk[f["pk"]], *args, ptr(o.pubs[0]),
                                                               C.byref(o.ticket))}


def prove_batch(e, o, bad):
    bad = dict(bad)
    h, k = e.pk[bad.pop("pk", "tables")]._h, bad.pop("k", 2)
    arr = items("b200_prove_item", k, lambda i: {"wires": ptr(e.wires), "pub_inputs": ptr(e.pub), "blinders": ptr(e.bl),
                                                 "proof": addr(o.proofs[i]), "link_poly": ptr(o.polys[i])}, bad)
    return {"context": lambda: e.lib.b200_plonk_prove_batch(e.ctx._h, h, arr, k, o.statuses),
            "pool": lambda: e.lib.b200_pool_submit_prove_batch(e.pool._h, h, arr, k, o.statuses, C.byref(o.ticket))}


def prove_witness_batch(e, o, bad):
    bad = dict(bad)
    h, k = e.pk[bad.pop("pk", "wiring")]._h, bad.pop("k", 2)
    arr = items("b200_witness_item", k, lambda i: {"witness": ptr(e.wit), "blinders": ptr(e.bl), "proof": addr(o.proofs[i]),
                                                   "link_poly": ptr(o.polys[i]), "pub_inputs_out": ptr(o.pubs[i])}, bad)
    return {"context": lambda: e.lib.b200_plonk_prove_witness_batch(e.ctx._h, h, arr, k, o.statuses),
            "pool": lambda: e.lib.b200_pool_submit_prove_witness_batch(e.pool._h, h, arr, k, o.statuses, C.byref(o.ticket))}


def link_fields(e, o, i):
    n2 = e.circ.n + 2
    return {"a1": ptr(e.poly), "len1": n2, "a2": ptr(e.poly), "len2": n2, "comm1": ptr(e.comm), "comm2": ptr(e.comm),
            "alignment": ALIGNMENT, "offset": OFFSET, "size": SIZE, "proof": addr(o.link_proofs[i]), "eta": ptr(o.etas[i])}


def link(e, o, bad):
    f = {**link_fields(e, o, 0), **bad}
    args = [f[x] for x in ("a1", "len1", "a2", "len2", "comm1", "comm2", "alignment", "offset", "size", "proof")]
    return {"context": lambda: e.lib.b200_plonk_link(e.ctx._h, e.bases._h, *args, f["eta"]),
            "pool": lambda: e.lib.b200_pool_submit_link(e.pool._h, e.bases._h, *args, C.byref(o.ticket))}


def link_batch(e, o, bad):
    arr = items("b200_link_item", 2, lambda i: link_fields(e, o, i), bad)
    return {"context": lambda: e.lib.b200_plonk_link_batch(e.ctx._h, e.bases._h, arr, 2, o.statuses),
            "pool": lambda: e.lib.b200_pool_submit_link_batch(e.pool._h, e.bases._h, arr, 2, o.statuses, C.byref(o.ticket))}


def bundle_calls(e, o, name, key, fields, bad):
    """A bundle of two proofs without links: the pool reads each entry's key, the box its array of box keys.  "pk" names
    the key of both entries, or is None for a NULL key in entry 1."""
    struct = "b200_bundle_proof" if name == "bundle" else "b200_bundle_witness"
    bad = dict(bad)
    key = bad.pop("pk") if isinstance(bad.get("pk"), str) else key
    arr = items(struct, 2, lambda i: {"pk": e.pk[key]._h, **fields(i)}, bad)
    pks = (C.c_void_p * 2)(e.box_pk[key], e.box_pk[key])
    submit, box_submit = getattr(e.lib, "b200_pool_submit_" + name), getattr(e.lib, "b200_box_submit_" + name)
    return {"pool": lambda: submit(e.pool._h, e.bases._h, arr, 2, None, 0, C.byref(o.ticket)),
            "box": lambda: box_submit(e.box._h, e.box_srs, pks, arr, 2, None, 0, C.byref(o.ticket))}


def bundle(e, o, bad):
    return bundle_calls(e, o, "bundle", "tables",
                        lambda i: {"wires": ptr(e.wires), "pub_inputs": ptr(e.pub), "num_inputs": NUM_INPUTS,
                                   "blinders": ptr(e.bl), "proof": addr(o.proofs[i]), "link_poly": ptr(o.polys[i])}, bad)


def bundle_witness(e, o, bad):
    return bundle_calls(e, o, "bundle_witness", "wiring",
                        lambda i: {"witness": ptr(e.wit), "blinders": ptr(e.bl), "proof": addr(o.proofs[i]),
                                   "link_poly": ptr(o.polys[i]), "pub_inputs_out": ptr(o.pubs[i])}, bad)


def settlement_links(e, o, bad):
    f = {"hint_poly": ptr(e.poly), "hint_len": e.circ.n + 2, "hint_comm": ptr(e.comm), "alignment": ALIGNMENT,
         "offset": OFFSET, "size": SIZE, "proof": addr(o.link_proofs[0]), "eta": ptr(o.etas[0])}
    f.update({k[5:]: v for k, v in bad.items() if k.startswith("link.")})
    return (S["b200_settlement_link"] * 1)(S["b200_settlement_link"](**f)), {k: v for k, v in bad.items()
                                                                             if not k.startswith("link.")}


def settlement(e, o, bad):
    links, bad = settlement_links(e, o, bad)
    f = {"pk": "tables", "wires": ptr(e.wires), "pub_inputs": ptr(e.pub), "num_inputs": NUM_INPUTS, "blinders": ptr(e.bl),
         "proof": addr(o.proofs[0]), "link_poly": ptr(o.polys[0]), **bad}
    entry = S["b200_bundle_proof"](**{**f, "pk": e.pk[f["pk"]]._h})
    return {"context": lambda: e.lib.b200_plonk_prove_settlement(e.ctx._h, e.bases._h, e.pk[f["pk"]]._h, f["wires"], f["pub_inputs"],
                                                                 f["blinders"], f["proof"], f["link_poly"], links, 1, o.statuses),
            "pool": lambda: e.lib.b200_pool_submit_settlement(e.pool._h, e.bases._h, C.byref(entry), links, 1, o.statuses,
                                                              C.byref(o.ticket)),
            "box": lambda: e.lib.b200_box_submit_settlement(e.box._h, e.box_srs, e.box_pk[f["pk"]], C.byref(entry), links, 1,
                                                            o.statuses, C.byref(o.ticket))}


def settlement_witness(e, o, bad):
    links, bad = settlement_links(e, o, bad)
    f = {"pk": "wiring", "witness": ptr(e.wit), "blinders": ptr(e.bl), "proof": addr(o.proofs[0]),
         "link_poly": ptr(o.polys[0]), "pub_inputs_out": ptr(o.pubs[0]), **bad}
    entry = S["b200_bundle_witness"](**{**f, "pk": e.pk[f["pk"]]._h})
    return {"context": lambda: e.lib.b200_plonk_prove_settlement_witness(
                e.ctx._h, e.bases._h, e.pk[f["pk"]]._h, f["witness"], f["blinders"], f["proof"], f["link_poly"],
                f["pub_inputs_out"], links, 1, o.statuses),
            "pool": lambda: e.lib.b200_pool_submit_settlement_witness(e.pool._h, e.bases._h, C.byref(entry), links, 1,
                                                                      o.statuses, C.byref(o.ticket)),
            "box": lambda: e.lib.b200_box_submit_settlement_witness(e.box._h, e.box_srs, e.box_pk[f["pk"]], C.byref(entry),
                                                                    links, 1, o.statuses, C.byref(o.ticket))}


CTX_POOL, ALL = ("context", "pool"), ("context", "pool", "box")
# (kind, the malformed fields, the words every layer's message holds, the layers called)
CASES = [
    (prove, {"wires": None}, "NULL wires", CTX_POOL),
    (prove, {"pub_inputs": None}, "NULL pub_inputs", CTX_POOL),
    (prove, {"blinders": None}, "NULL blinders", ALL),
    (prove, {"proof": None}, "NULL proof", CTX_POOL),
    (prove, {"num_inputs": 1}, "num_inputs", ("pool", "box")),
    (prove_witness, {"witness": None}, "NULL witness", CTX_POOL),
    (prove_witness, {"blinders": None}, "NULL blinders", ALL),
    (prove_witness, {"proof": None}, "NULL proof", CTX_POOL),
    (prove_witness, {"pk": "tables"}, "holds no wiring", CTX_POOL),
    (prove_batch, {"wires": None}, "item 1 has a NULL wires", CTX_POOL),
    (prove_batch, {"pub_inputs": None}, "item 1 has a NULL pub_inputs", CTX_POOL),
    (prove_batch, {"blinders": None}, "item 1 has a NULL blinders", CTX_POOL),
    (prove_batch, {"proof": None}, "item 1 has a NULL proof", CTX_POOL),
    (prove_witness_batch, {"witness": None}, "item 1 has a NULL witness", CTX_POOL),
    (prove_witness_batch, {"blinders": None}, "item 1 has a NULL blinders", CTX_POOL),
    (prove_witness_batch, {"proof": None}, "item 1 has a NULL proof", CTX_POOL),
    (prove_witness_batch, {"pk": "tables"}, "holds no wiring", CTX_POOL),
    (prove_witness_batch, {"pk": "tables", "k": 0}, "holds no wiring", CTX_POOL),
    *[(link, {x: None}, f"NULL {x}", CTX_POOL) for x in ("a1", "a2", "comm1", "comm2", "proof")],
    *[(link_batch, {x: None}, f"item 1 has a NULL {x}", CTX_POOL) for x in ("a1", "a2", "comm1", "comm2", "proof")],
    (bundle, {"pk": None}, "proof 1 has a NULL pk", ("pool",)),
    (bundle, {"wires": None}, "proof 1 has a NULL wires", ("pool",)),
    (bundle, {"pub_inputs": None}, "proof 1 has a NULL pub_inputs", ("pool",)),
    (bundle, {"blinders": None}, "proof 1 has a NULL blinders", ("pool", "box")),
    (bundle, {"proof": None}, "proof 1 has a NULL proof", ("pool",)),
    (bundle, {"num_inputs": 3}, "proof 1: num_inputs", ("pool",)),
    (bundle_witness, {"witness": None}, "proof 1 has a NULL witness", ("pool",)),
    (bundle_witness, {"blinders": None}, "proof 1 has a NULL blinders", ("pool", "box")),
    (bundle_witness, {"proof": None}, "proof 1 has a NULL proof", ("pool",)),
    (bundle_witness, {"pk": "tables"}, "proof 0: the key holds no wiring", ("pool",)),
    (settlement, {"wires": None}, "NULL wires", CTX_POOL),
    (settlement, {"pub_inputs": None}, "NULL pub_inputs", CTX_POOL),
    (settlement, {"blinders": None}, "NULL blinders", ALL),
    (settlement, {"proof": None}, "NULL proof", CTX_POOL),
    (settlement, {"num_inputs": 1}, "num_inputs", ("pool",)),
    *[(settlement, {"link." + x: None}, f"link 0 has a NULL {x}", CTX_POOL) for x in ("hint_poly", "hint_comm", "proof")],
    (settlement_witness, {"witness": None}, "NULL witness", CTX_POOL),
    (settlement_witness, {"blinders": None}, "NULL blinders", ALL),
    (settlement_witness, {"proof": None}, "NULL proof", CTX_POOL),
    (settlement_witness, {"pk": "tables"}, "holds no wiring", CTX_POOL),
    *[(settlement_witness, {"link." + x: None}, f"link 0 has a NULL {x}", CTX_POOL) for x in ("hint_poly", "hint_comm", "proof")],
]


@pytest.mark.parametrize("kind,bad,words,layers", CASES,
                         ids=[f"{k.__name__}-{'-'.join(f'{a}={b}' for a, b in bad.items())}" for k, bad, _, _ in CASES])
def test_refused_before_any_device_work(env, kind, bad, words, layers):
    lib = env.lib
    box_pool = lib.b200_box_pool(env.box._h, 0)
    stats = env.pool.stats(), pool_stats(lib, box_pool)
    launches = lib.b200_kernel_launches()
    tails = {}
    for layer in layers:
        o = Outs(env.circ.n)
        lib.b200_pool_stats(None, None)  # a message of its own, so that a refusal without one shows
        assert kind(env, o, bad)[layer]() == INVALID, layer
        msg = lib.b200_last_error().decode()
        assert words in msg, (layer, msg)
        tails[layer] = msg.split(" ", 1)[1]  # without the entry point's name
        assert o.untouched(), layer
    assert len(set(tails.values())) == 1, tails  # the same words on every layer
    assert (env.pool.stats(), pool_stats(lib, box_pool)) == stats
    assert lib.b200_kernel_launches() == launches
