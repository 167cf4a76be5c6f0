"""CPU checks of the batch link prover's boundary (`link_proofs_batch`, `ProverPool.submit_link_batch`,
`b200_plonk_link_batch`, `b200_pool_submit_link_batch`): malformed triples are refused with ValueError before any device
call, well-formed ones become one b200_link_item each, NULL handles and item arrays come back as B200_ERR_INVALID, and a
pool cannot be made without a device (B200_ERR_NO_DEVICE, never a host fallback)."""
import ctypes as C

import numpy as np
import pytest

from renegade_b200.backend import GroupLayout, LinkingHint, ProverPool, _link_items, link_proofs_batch


class FakeBases:
    """stands in for a Bases: the checks read its length only (a device call would fail on _h=None)"""
    _h = None

    def __len__(self):
        return 100


def hint(n, comm_limbs=8):
    return LinkingHint(np.zeros((n, 4), dtype=np.uint64), np.zeros(comm_limbs, dtype=np.uint64))


def good():
    return [(hint(20), hint(12), GroupLayout(3, 6, 5)), (hint(9), hint(10), GroupLayout(4, 3, 1))]


@pytest.mark.parametrize("bad", ["size_zero", "size_is_len", "alignment", "offset", "srs_too_short", "comm", "limbs",
                                 "not_a_triple"])
def test_malformed_link_batches_are_refused_before_the_device(bad):
    t = good()
    a, b, lay = t[1]
    if bad == "size_zero":
        t[1] = (a, b, GroupLayout(4, 3, 0))
    elif bad == "size_is_len":
        t[1] = (a, b, GroupLayout(4, 3, 10))
    elif bad == "alignment":
        t[1] = (a, b, GroupLayout(29, 3, 1))
    elif bad == "offset":
        t[1] = (a, b, GroupLayout(4, -1, 1))
    elif bad == "srs_too_short":
        t[1] = (hint(101), b, lay)
    elif bad == "comm":
        t[1] = (a, hint(10, comm_limbs=4), lay)
    elif bad == "limbs":
        t[1] = (LinkingHint(np.zeros(9 * 4 + 1, dtype=np.uint64), a.linking_wire_comm), b, lay)
    else:
        t[1] = (a, b)
    with pytest.raises(ValueError, match="item 1"):
        link_proofs_batch(None, FakeBases(), t)  # ctx=None: reaching the library would raise AttributeError
    with pytest.raises(ValueError, match="item 1"):
        ProverPool.submit_link_batch(None, FakeBases(), t)


def test_well_formed_batch_builds_one_item_per_triple():
    t = good()
    t.append((LinkingHint((0xdead0000, 50), np.zeros(8, dtype=np.uint64)), hint(40), GroupLayout(5, 0, 7)))
    items, keep = _link_items(FakeBases(), t)
    assert len(keep) == 3
    assert [(items[i].len1, items[i].len2, items[i].size) for i in range(3)] == [(20, 12, 5), (9, 10, 1), (50, 40, 7)]
    assert items[2].a1 == 0xdead0000 and keep[2][0] is None  # an address (device or pinned memory) is passed through
    assert all(items[i].proof and items[i].eta and items[i].comm1 and items[i].comm2 for i in range(3))
    assert _link_items(FakeBases(), [])[1] == []


def test_null_handles_and_items():
    from renegade_b200 import _lib
    from renegade_b200.backend import B200LinkItem
    lib = _lib.load()
    st = (C.c_int * 2)()
    t = C.c_uint64(0)
    items = (B200LinkItem * 2)()  # every pointer NULL
    for k, arr in ((0, None), (2, None), (2, items)):
        assert lib.b200_plonk_link_batch(None, None, arr, k, st) == -1
        assert b"null argument" in lib.b200_last_error()
        assert lib.b200_pool_submit_link_batch(None, None, arr, k, st, C.byref(t)) == -1
        assert b"null argument" in lib.b200_last_error()
    assert lib.b200_pool_submit_link_batch(None, None, items, 2, st, None) == -1
    assert list(st) == [0, 0] and t.value == 0  # nothing written


def test_pool_without_a_device():
    import torch
    from renegade_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.b200_pool_create(0, 2, C.byref(h)) == -6 and not h.value
    assert b"no CPU fallback" in lib.b200_last_error()
