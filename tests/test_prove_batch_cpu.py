"""CPU checks of the batch prover's Python argument validation (`PlonkKzgSnark.prove_batch`,
`ProverPool.submit_prove_batch`): list lengths, wire-table shapes, public-input and blinder counts are refused with
ValueError before any device call, so a malformed batch never reaches the library."""
from types import SimpleNamespace

import numpy as np
import pytest

from renegade_b200.backend import PlonkKzgSnark, _prove_items


def key(log_n=3, num_inputs=2):
    # stands in for a ProvingKey: the checks read the shape only (a device call would fail on ctx=None)
    return SimpleNamespace(log_n=log_n, num_inputs=num_inputs, domain_size=1 << log_n, _h=None)


def args(k, log_n=3, num_inputs=2):
    n = 1 << log_n
    return ([np.zeros((5, n, 4), dtype=np.uint64)] * k, [np.zeros((num_inputs, 4), dtype=np.uint64)] * k,
            [np.zeros((17, 4), dtype=np.uint64)] * k)


@pytest.mark.parametrize("bad", ["lengths", "wires", "pub_inputs", "blinders"])
def test_malformed_batches_are_refused_before_the_device(bad):
    w, pi, bl = args(3)
    if bad == "lengths":
        pi = pi[:2]
    elif bad == "wires":
        w = w[:2] + [np.zeros((5, 4, 4), dtype=np.uint64)]
    elif bad == "pub_inputs":
        pi = pi[:1] + [np.zeros((3, 4), dtype=np.uint64)] + pi[2:]
    else:
        bl = bl[:2] + [np.zeros((16, 4), dtype=np.uint64)]
    with pytest.raises(ValueError):
        PlonkKzgSnark.prove_batch(None, key(), w, pi, bl)


def test_well_formed_batch_builds_one_item_per_witness():
    w, pi, bl = args(3, num_inputs=0)
    w[1] = 0xdead0000  # an address (device or pinned memory) is passed through unchecked
    items, keep = _prove_items(key(num_inputs=0), w, pi, bl, link_hints=True, want_challenges=False)
    assert len(keep) == 3
    assert items[1].wires == 0xdead0000 and items[0].pub_inputs is None
    assert all(items[i].link_poly and not items[i].challenges for i in range(3))
    assert keep[2][4].shape == (8 + 2, 4)  # the (n + 2)-coefficient link polynomial
