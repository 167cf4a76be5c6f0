"""The per-item verifier's and the device pairing checks' argument handling that runs before any device work: the Python
checks shared with batch_verify, the shape checks of pairing_check_many, and NULL handles in the C entry points."""
import ctypes as C

import numpy as np
import pytest

from renegade_b200 import _lib
from renegade_b200.backend import GroupLayout, PlonkKzgSnark, VerifyingKey, pairing_check_many


def _vk(h, tau_h):
    return VerifyingKey(6, 0, np.zeros((5, 4), np.uint64), np.zeros((13, 8), np.uint64), np.zeros((5, 8), np.uint64),
                        h, tau_h)


def test_python_checks_before_the_device():
    h, tau_h = np.zeros(16, np.uint64), np.ones(16, np.uint64)
    assert PlonkKzgSnark.verify_each(None, [], [], []) == []
    with pytest.raises(ValueError, match="one verifying key"):
        PlonkKzgSnark.verify_each(None, [_vk(h, tau_h)], [], [None])
    with pytest.raises(ValueError, match="share the G2 pair"):
        PlonkKzgSnark.verify_each(None, [_vk(h, tau_h), _vk(tau_h, h)], [np.zeros((0, 4), np.uint64)] * 2, [None] * 2)
    link = (np.zeros(8, np.uint64), np.zeros(8, np.uint64), None, GroupLayout(5, 0, 1))
    with pytest.raises(ValueError, match="need g2"):
        PlonkKzgSnark.verify_each(None, [], [], [], [link])


def test_pairing_check_many_shapes():
    g2 = np.zeros((2, 16), np.uint64)
    with pytest.raises(ValueError):
        pairing_check_many(None, np.zeros((2, 8), np.uint64), np.zeros((1, 2, 8), np.uint64))
    with pytest.raises(ValueError):
        pairing_check_many(None, g2, np.zeros((1, 3, 8), np.uint64))
    with pytest.raises(ValueError):
        pairing_check_many(None, g2, np.zeros((2, 8), np.uint64))
    with pytest.raises(ValueError, match="at most 8"):
        pairing_check_many(None, np.zeros((9, 16), np.uint64), np.zeros((1, 9, 8), np.uint64))


def test_null_handles():
    lib = _lib.load()
    g2 = np.zeros(16, np.uint64).ctypes.data_as(C.c_void_p)
    out = (C.c_uint8 * 4)()
    assert lib.b200_plonk_verify_each(None, None, 0, None, 0, None, 0, g2, g2, out) == _lib.B200_ERR_INVALID
    assert lib.b200_pairing_check_many(None, g2, 1, g2, 1, out) == _lib.B200_ERR_INVALID
    assert list(out) == [0] * 4  # nothing written


def test_entry_points_are_in_header_binding_and_ffi():
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "b200prover.h")).read()
    ffi = open(os.path.join(root, "shim", "gpu-prover", "src", "ffi.rs")).read()
    for name in ("b200_plonk_verify_each", "b200_pairing_check_many"):
        assert re.search(r"\bint " + name + r"\(", header)
        assert name in _lib.EXPORTS
        assert "pub fn " + name + "(" in ffi
