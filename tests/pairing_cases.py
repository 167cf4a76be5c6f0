"""Pairing checks whose verdicts follow from bilinearity, built without a GPU and without the product's pairing.

With G1 points a_j G and G2 points b_j H, prod_j e(a_j G, b_j H) = e(G, H)^(sum_j a_j b_j), and e(G, H) has order r, so a
check holds exactly when sum_j a_j b_j = 0 (mod r).  Every verdict here is predicted with Python integers, for any
number of pairs and any positions; a G1 or G2 identity is a = 0 or b = 0 and contributes 0.

* G2 points are b H for seeded b (`bn254_pairing_py.g2_mul` on the reference's H), plus H itself (b = 1), -H (b = r - 1),
  the same point in two slots and the identity record (128 zero bytes, b = 0).
* G1 points are a G (the C oracle's `g1_mul`); a = 0 is the identity record (64 zero bytes).
* A holding check picks one a to cancel the sum; its failing twin adds 1 to the a of a slot whose b is not 0.
* Degenerate G2 records without an algebraic verdict: a twist point outside the r-torsion.  Where its slot's G1 point is
  the identity the pair is skipped and the prediction stands; elsewhere only host and device can be compared.
* G1 records that must be refused: a coordinate moved to v + q, or x moved off the curve."""
import random

import numpy as np

import bn254_pairing_py as pr
import oracle_c

R, Q = pr.R, pr.Q
MAX_PAIRS = 8  # b200_pairing_check_many's kMaxPairs
G1_IDENTITY = np.zeros(8, dtype=np.uint64)
G2_IDENTITY = np.zeros(16, dtype=np.uint64)


def _mont(v: int) -> np.ndarray:
    return np.frombuffer(((v << 256) % Q).to_bytes(32, "little"), dtype="<u8").astype(np.uint64)


G1_GEN = np.concatenate([_mont(1), _mont(2)])  # G = (1, 2), the generator the verifiers use


class Points:
    """a -> the record of a G, b -> the record of b H; each computed once."""

    def __init__(self, h_record):
        self.h = pr.decode_g2_mont(np.asarray(h_record, dtype=np.uint64).tobytes(), 0)
        self._g1, self._g2 = {}, {}

    def g1(self, a: int) -> np.ndarray:
        a %= R
        if a not in self._g1:
            if a == 0:
                rec = G1_IDENTITY
            elif (a - 1) % R in self._g1 and (a - 1) % R:  # a failing twin: one addition instead of a multiplication
                rec, inf = oracle_c.g1_add(self._g1[(a - 1) % R], 0, G1_GEN, 0)
                assert not inf
            else:
                rec, inf = oracle_c.g1_mul(G1_GEN, 0, oracle_c.int_to_limbs(a))
                assert not inf
            self._g1[a] = rec
        return self._g1[a]

    def g2(self, b: int) -> np.ndarray:
        b %= R
        if b not in self._g2:
            self._g2[b] = G2_IDENTITY if b == 0 else np.frombuffer(pr.encode_g2_mont(pr.g2_mul(self.h, b)),
                                                                   dtype=np.uint64).copy()
        return self._g2[b]


def g2_scalars(m: int, kind: str, seed: int = 0) -> list:
    """The b_j of a check's m G2 points.  'distinct': seeded, pairwise distinct, none of 0, 1, r - 1.  'edges': H (b = 1)
    and -H (b = r - 1) first, then one seeded point in two slots, then seeded points.  'identity': 'distinct' with the
    identity record in the middle slot."""
    rng = random.Random(0x62A1 + 1000 * seed + m)
    b = [rng.randrange(2, R - 1) for _ in range(m)]
    if kind == "edges":
        b[:2] = [1, R - 1][:m]
        if m >= 4:
            b[3] = b[2]
    elif kind == "identity" and m:
        b[m // 2] = 0
    else:
        assert kind == "distinct", kind
    return b


def holds(a, b) -> bool:
    return sum(x * y for x, y in zip(a, b)) % R == 0


def _cancel_slot(b) -> int:
    """the last slot whose G2 point is not the identity"""
    return max(j for j in range(len(b)) if b[j] % R)


def _cancel(a, b, slot) -> list:
    """a with a[slot] chosen so that sum_j a_j b_j = 0"""
    a = list(a)
    a[slot] = 0
    a[slot] = -sum(x * y for x, y in zip(a, b)) * pow(b[slot], -1, R) % R
    return a


HOLD_KINDS = ("random", "identity", "opposite", "all_identity")


def holding_row(b, kind: str, rng: random.Random, pool) -> list:
    """G1 scalars of a check over b that holds.  'random': pool scalars, one slot cancelling; 'identity': the same with
    the identity in a seeded slot other than the cancelling one; 'opposite': P and -P against two slots of the same G2
    point, or P and P against Q and -Q, where b has such slots (elsewhere as 'random'); 'all_identity': every slot."""
    m = len(b)
    if kind == "all_identity" or not any(x % R for x in b):
        return [0] * m
    cs = _cancel_slot(b)
    a = [rng.choice(pool) for _ in range(m)]
    if kind == "identity" and m >= 2:
        a[rng.choice([j for j in range(m) if j != cs])] = 0
    if kind == "opposite":
        twins = [(i, k) for i in range(m) for k in range(i + 1, m) if b[i] % R and (b[i] - b[k]) * (b[i] + b[k]) % R == 0]
        if twins:
            i, k = twins[-1]
            a[k] = (R - a[i]) % R if b[i] == b[k] else a[i]
            rest = [j for j in range(m) if j not in (i, k) and b[j] % R]
            if rest:
                return _cancel(a, b, rest[-1])
            return a
    return _cancel(a, b, cs)


def failing_twin(a, b, slot: int) -> list:
    """a with 1 added to slot `slot` (whose b is not 0): the sum moves by b_slot, so the check fails"""
    assert b[slot] % R
    out = list(a)
    out[slot] = (out[slot] + 1) % R
    return out


class Sweep:
    """n holding checks over one set of G2 points and a failing twin of each, its failing slot cycling through the
    slots whose G2 point is not the identity (so each slot is the broken one somewhere)."""

    def __init__(self, pts: Points, b, n: int, seed: int = 0):
        self.pts, self.b, self.m = pts, list(b), len(b)
        rng = random.Random(0x5EE9 + 7919 * seed + self.m)
        pool = [rng.randrange(1, R) for _ in range(61)]
        live = [j for j in range(self.m) if b[j] % R]
        self.hold, self.fail = [], []
        for c in range(n):
            a = holding_row(b, HOLD_KINDS[c % len(HOLD_KINDS)], rng, pool)
            self.hold.append(a)
            self.fail.append(failing_twin(a, b, live[(c // len(HOLD_KINDS)) % len(live)]) if live else a)
        self.g2 = np.stack([pts.g2(x) for x in b]) if self.m else np.zeros((0, 16), dtype=np.uint64)

    def rows(self, n: int, failing) -> list:
        """scalars of the first n checks, the failing twin at each index of `failing`"""
        return [self.fail[c] if c in failing else self.hold[c] for c in range(n)]

    def g1(self, rows) -> np.ndarray:
        return g1_records(self.pts, rows, self.m)

    def predicted(self, rows) -> np.ndarray:
        return np.array([holds(a, self.b) for a in rows], dtype=bool)


def g1_records(pts: Points, rows, m: int) -> np.ndarray:
    """(n, m, 8) records of rows of G1 scalars"""
    out = np.zeros((len(rows), m, 8), dtype=np.uint64)
    for c, a in enumerate(rows):
        for j, x in enumerate(a):
            out[c, j] = pts.g1(x)
    return out


def placements(n: int) -> dict:
    """the indices of the failing checks of a batch of n: none, the first, 63 / 64 / 65 (either side of the pairing
    kernel's 64-thread block edge), the last, every odd index, all"""
    return {"none": set(), "first": {0}, "block_edge": {c for c in (63, 64, 65) if c < n}, "last": {n - 1},
            "alternating": set(range(1, n, 2)), "everywhere": set(range(n))}


def edge_rows(b, n: int, seed: int = 0) -> list:
    """n checks over b of every kind at once: each holding kind, failing twins at every live slot, the same G1 point in
    all m slots, P and -P in the first two slots (holds only against the same G2 point), all identities"""
    m = len(b)
    rng = random.Random(0xED6E + 101 * seed + m)
    pool = [rng.randrange(1, R) for _ in range(31)]
    live = [j for j in range(m) if b[j] % R]
    rows = []
    while len(rows) < n:
        c = len(rows)
        a = holding_row(b, HOLD_KINDS[c % len(HOLD_KINDS)], rng, pool)
        rows.append(a)
        if live:
            rows.append(failing_twin(a, b, live[c % len(live)]))
        p = rng.choice(pool)
        rows.append([p] * m)
        if m >= 2:
            rows.append([p, R - p] + [0] * (m - 2))
    return rows[:n]


# ---- degenerate G2 records and refused G1 records --------------------------------------------------------------------
def twist_point_record(seed: int) -> np.ndarray:
    """a seeded point of the twist y^2 = x^3 + 3 / (9 + u) outside the r-torsion"""
    from test_srs_check_cpu import oracle_in_subgroup, random_twist_point
    p = random_twist_point(random.Random(seed))
    assert not oracle_in_subgroup(p)
    return np.frombuffer(pr.encode_g2_mont(p), dtype=np.uint64).copy()


class TwistCase:
    """Checks over m G2 points whose slot t holds a twist point outside the r-torsion and the others b_j H.  `verdicts`
    is the prediction where slot t's G1 point is the identity (the pair is skipped, the others obey bilinearity) and
    None elsewhere."""

    def __init__(self, pts: Points, m: int, n: int, seed: int = 0):
        self.b = g2_scalars(m, "distinct", seed)
        self.t = m // 2
        self.b[self.t] = 0  # its algebraic stand-in: the identity in that slot
        self.g2 = np.stack([pts.g2(x) for x in self.b])
        self.g2[self.t] = twist_point_record(0x7157 + seed)
        rng = random.Random(0x7C + seed + m)
        pool = [rng.randrange(1, R) for _ in range(31)]
        rows = edge_rows(self.b, n, seed)
        for c in range(n):  # a G1 point against the twist point in every third check, the identity elsewhere
            rows[c] = list(rows[c])
            rows[c][self.t] = rng.choice(pool) if c % 3 == 0 else 0
        self.rows = rows
        self.g1 = g1_records(pts, rows, m)
        self.verdicts = [holds(a, self.b) if a[self.t] == 0 else None for a in rows]

    def recorded(self) -> list:
        """the host's verdicts as recorded: the prediction where there is one, and False for every check with a G1
        point against the twist point (on these seeded points no such product is one)"""
        return [v if v is not None else False for v in self.verdicts]


TWIST_CASES = [(1, 12), (2, 24), (5, 24), (8, 24), (8, 129)]  # (m, n) of the twist-point checks


def off_curve(rec: np.ndarray) -> np.ndarray:
    """x's lowest Montgomery limb moved by one: not on y^2 = x^3 + 3"""
    out = np.array(rec, dtype=np.uint64).copy()
    out[0] ^= np.uint64(1)
    assert not oracle_c.g1_on_curve(out)
    return out


def plus_q(rec: np.ndarray, coord: int) -> np.ndarray:
    """coordinate `coord` (0: x, 1: y) moved to v + q: the same residue, outside [0, q)"""
    out = np.array(rec, dtype=np.uint64).copy()
    v = int.from_bytes(out[4 * coord:4 * coord + 4].tobytes(), "little") + Q
    assert v < 1 << 256
    out[4 * coord:4 * coord + 4] = np.frombuffer(v.to_bytes(32, "little"), dtype="<u8")
    return out
