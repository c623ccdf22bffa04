"""The taxon look-up of the kept rows on the CPU warp emulator: with the dense row -> taxon array (what a narrow GPU context uses) and with
the SA walk, every read gets the same taxon, best score and match-id set, equal to the oracle's -- on the golden reads and on reads whose
kept intervals hold many rows and more than 20 distinct taxa (several waves of 32 rows, the stop on the 21st id)."""
import ctypes as C
import numpy as np
import pytest
import emu_row_tax
from helpers import Oracle, make_params, have_ref
from shared_core_db import make_shared_core_db
from test_kernel_logic_emulated import KjParams


@pytest.fixture(scope="module")
def emu(built, tmp_path_factory):
    return emu_row_tax.load(str(tmp_path_factory.mktemp("emu_row_tax")), KjParams)


@pytest.fixture(scope="module")
def shared_core(tmp_path_factory):
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    return make_shared_core_db(str(tmp_path_factory.mktemp("shared_core")))


def _classify(E, h, s1, o1, s2, o2):
    n = len(o1) - 1
    tax = np.zeros(n, np.uint64); best = np.zeros(n, np.uint32); ids = np.zeros((n, 21), np.uint64); nids = np.zeros(n, np.uint8)
    rc = E.kjemu_classify_ids(h, s1.ctypes.data, o1.ctypes.data, s2.ctypes.data if s2 is not None else None, o2.ctypes.data if s2 is not None else None,
                              n, tax.ctypes.data, best.ctypes.data, ids.ctypes.data, nids.ctypes.data, 4)
    assert rc == 0
    return tax, best, [tuple(int(x) for x in ids[i, :nids[i]]) for i in range(n)]


def _array_equals_walk(E, fmi, nodes, mode, s1, o1, s2, o2):
    P = make_params(mode)
    h = E.kjemu_create(fmi.encode(), nodes.encode(), C.byref(KjParams(**P))); assert h
    try:
        assert E.kjemu_use_row_tax(h, 1) == 1
        tax, best, ids = _classify(E, h, s1, o1, s2, o2)
        assert E.kjemu_use_row_tax(h, 0) == 0
        wtax, wbest, wids = _classify(E, h, s1, o1, s2, o2)
    finally:
        E.kjemu_destroy_row_tax(h)
    assert np.array_equal(tax, wtax) and np.array_equal(best, wbest)
    assert ids == wids, [i for i in range(len(ids)) if ids[i] != wids[i]][:5]
    otax, obest = Oracle(fmi, nodes).classify_batch(P, s1, o1, s2, o2)
    assert np.array_equal(tax, otax) and np.array_equal(best, obest)
    return ids


@pytest.mark.parametrize("mode", ["mem", "greedy"])
def test_row_tax_equals_walk_golden(emu, golden, mode):
    for tag in ("pe150", "se100"):
        names, s1, o1, s2, o2 = golden.reads(tag)
        _array_equals_walk(emu, golden.fmi, golden.nodes, mode, s1, o1, s2, o2)


@pytest.mark.parametrize("mode", ["mem", "greedy"])
def test_row_tax_equals_walk_many_ids(emu, shared_core, mode):
    fmi, nodes, s1, o1, s2, o2 = shared_core
    ids = _array_equals_walk(emu, fmi, nodes, mode, s1, o1, s2, o2)
    assert sum(len(x) == 21 for x in ids) > len(ids) // 4, "too few reads reach the stop on the 21st id"
