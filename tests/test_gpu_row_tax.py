"""The dense row -> taxon array on the GPU.  A default context of a narrow index carries the array; a KJ_FORCE_WIDE context of the same
index (64-bit kernels) does not, so it resolves every kept row with the SA walk.  Both give bit-identical taxa, best scores, dense taxon
indices and match-id sets, on the golden index, on a 2-fold scaled index, on a workload like bench.py's (1 M PE150 pairs), and on reads whose
kept intervals hold many rows and more than 20 distinct taxa (several waves of 32 rows, the stop on the 21st id)."""
import numpy as np
import pytest
from helpers import Oracle, SynthDB, build_fmi, have_ref, make_params
from shared_core_db import make_shared_core_db

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


def _outputs(clf, s1, o1, s2, o2):
    """taxon / best / dense taxon index through classify_device2, and the match-id sets through classify_verbose"""
    import torch
    n = len(o1) - 1
    dev = [None if a is None else torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else np.ascontiguousarray(a)).cuda()
           for a in (s1, o1, s2, o2)]
    d_tax = torch.zeros(n, dtype=torch.int64, device="cuda"); d_best = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_comp = torch.zeros(n, dtype=torch.int32, device="cuda")
    clf.classify_device2(*[None if t is None else t.data_ptr() for t in dev], n, d_tax.data_ptr(), d_best.data_ptr(), d_comp.data_ptr())
    torch.cuda.synchronize(); clf.check_errors()
    out = {"taxon": d_tax.cpu().numpy().view(np.uint64), "best": d_best.cpu().numpy().view(np.uint32), "taxon_index": d_comp.cpu().numpy().view(np.uint32)}
    vtax, vbest, ids = clf.classify_verbose(s1, o1, s2, o2)
    assert np.array_equal(vtax, out["taxon"]) and np.array_equal(vbest, out["best"])
    out["ids"] = ids
    return out


def _array_equals_walk(kb, monkeypatch, fmi, nodes, works, copies=1):
    """returns the array context's outputs per (mode, work)"""
    got = {}
    for mode in ("mem", "greedy"):
        arr = kb.Classifier(fmi, nodes, device=0, params=kb.make_params(mode), copies=copies)
        with monkeypatch.context() as m:
            m.setenv("KJ_FORCE_WIDE", "1")
            walk = kb.Classifier(fmi, nodes, device=0, params=kb.make_params(mode), copies=copies)
        try:
            for w, (s1, o1, s2, o2) in enumerate(works):
                a = _outputs(arr, s1, o1, s2, o2); b = _outputs(walk, s1, o1, s2, o2)
                for k in ("taxon", "best", "taxon_index"):
                    bad = np.nonzero(a[k] != b[k])[0]
                    assert len(bad) == 0, (mode, w, k, bad[:5])
                assert a["ids"] == b["ids"], (mode, w, [i for i in range(len(a["ids"])) if a["ids"][i] != b["ids"][i]][:5])
                got[(mode, w)] = a
        finally:
            arr.close(); walk.close()
    return got


def test_row_tax_equals_walk_golden(kb, golden, monkeypatch):
    _array_equals_walk(kb, monkeypatch, golden.fmi, golden.nodes, [golden.reads(t)[1:] for t in ("pe150", "se100")])


def test_row_tax_equals_walk_scaled(kb, golden, monkeypatch):
    """copies = 2: the scaled index is narrow and gets its own array (the transient base context of the construction does not)"""
    _array_equals_walk(kb, monkeypatch, golden.fmi, golden.nodes, [golden.reads(t)[1:] for t in ("pe150", "se100")], copies=2)


def test_row_tax_equals_walk_bench_like(kb, tmp_path, monkeypatch):
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    d = str(tmp_path); db = SynthDB(100000, 1); db.write(d + "/db.faa", d + "/nodes.dmp")
    fmi = build_fmi(d + "/db.faa", d + "/db", threads=16)
    _array_equals_walk(kb, monkeypatch, fmi, d + "/nodes.dmp", [db.reads(7, 0, 1 << 20, 150, True)])


def test_row_tax_equals_walk_many_ids(kb, tmp_path, monkeypatch):
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    fmi, nodes, s1, o1, s2, o2 = make_shared_core_db(str(tmp_path))
    got = _array_equals_walk(kb, monkeypatch, fmi, nodes, [(s1, o1, s2, o2)])
    orc = Oracle(fmi, nodes)
    for mode in ("mem", "greedy"):
        a = got[(mode, 0)]
        otax, obest = orc.classify_batch(make_params(mode), s1, o1, s2, o2)
        assert np.array_equal(a["taxon"], otax) and np.array_equal(a["best"], obest), mode
        assert sum(len(x) == 21 for x in a["ids"]) > len(a["ids"]) // 4, "too few reads reach the stop on the 21st id"
