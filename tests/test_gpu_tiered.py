"""Indexes with a host tier on the GPU (kj_create_tiered, Classifier(host_memory=)): a compact context whose records are split between HBM and
mapped pinned host memory (KJ_FORCE_COMPACT + KJ_TIER_DEVICE_RECORDS) gives bit-identical outputs to the plain compact context on every entry
point; its index checksums equal the compact context's and the host transcoder's; host_memory = 0 changes nothing; an index whose compact
construction does not fit in HBM is placed with a host tier without any hook, and one whose host tier exceeds the budget fails cleanly."""
import ctypes as C
import os
import numpy as np
import pytest
from helpers import Oracle, SynthDB, build_fmi, have_ref, make_params
from test_gpu_compact import MODES, _free, _outputs, _same

pytestmark = pytest.mark.gpu
HOST = 1 << 30


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


def _nb(bwtlen):
    return bwtlen // 128 + 1


def _split(split, nb):
    return {"0": 0, "1": 1, "half": nb // 2, "nb": nb}[split]


def _pair(kb, m, fmi, nodes, params, split, copies=1, **kw):
    """(plain compact context, tiered compact context split at `split` records of the final index)"""
    m.setenv("KJ_FORCE_COMPACT", "1")
    cpt = kb.Classifier(fmi, nodes, device=0, params=params, copies=copies, **kw)
    nd = _split(split, _nb(cpt.bwtlen)) if isinstance(split, str) else split
    m.setenv("KJ_TIER_DEVICE_RECORDS", str(nd))
    tie = kb.Classifier(fmi, nodes, device=0, params=params, copies=copies, host_memory=HOST, **kw)
    m.delenv("KJ_TIER_DEVICE_RECORDS")
    assert cpt.layout == 2 and cpt.host_bytes == 0
    assert tie.layout == (2 if nd >= _nb(tie.bwtlen) else 3) and tie.host_bytes > 0, (tie.layout, tie.host_bytes, nd)
    assert tie.index_bytes < cpt.index_bytes
    return cpt, tie


@pytest.mark.parametrize("split", ["0", "1", "half", "nb"])
def test_tiered_equals_compact_golden(kb, golden, monkeypatch, tmp_path, split):
    """MEM, two-kernel and single-kernel Greedy on the golden reads through kj_classify_device2, kj_classify, kj_classify2's dense indices,
    per-taxon counts, kj_classify_verbose and kj_classify_verbose2; name mode; kj_classify_multi; the file pipeline; protein input; long reads"""
    gold = os.path.dirname(golden.fmi); works = [golden.reads(t)[1:] for t in ("pe150", "se100")]
    db = SynthDB(800, 3); ps, po = db.protein_reads(42, 0, 400, 5, 5461); ls, lo = db.long_reads(55, 0, 6, 16384, 40000)
    for mode, env in MODES + [(dict(mode="mem", name_mode=True), {})]:
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            cpt, tie = _pair(kb, m, golden.fmi, golden.nodes, kb.make_params(**mode), split)
            try:
                for w, (s1, o1, s2, o2) in enumerate(works):
                    _same(_outputs(kb, cpt, s1, o1, s2, o2), _outputs(kb, tie, s1, o1, s2, o2), (split, mode, env, w))
                s1, o1, s2, o2 = works[0]
                a = kb.classify_multi([tie, cpt], s1, o1, s2, o2); b = cpt.classify(s1, o1, s2, o2)      # first shard on the tiered context
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
                if mode.get("name_mode") or env:
                    continue
                outs = []
                for clf in (cpt, tie):
                    o = str(tmp_path / ("o%d.tsv" % len(outs)))
                    clf.classify_files(os.path.join(gold, "pe150_1.fq.gz"), os.path.join(gold, "pe150_2.fq.gz"), o, verbose=True)
                    outs.append(open(o).read())
                assert outs[0] == outs[1] and len(outs[0]) > 1000
                for clf in (cpt, tie):
                    clf.set_max_read_len(kb.MAX_LONG_READ_LEN)
                _same(_outputs(kb, cpt, ls, lo, None, None, False), _outputs(kb, tie, ls, lo, None, None, False), (split, mode, "long"))
                for clf in (cpt, tie):
                    clf.set_params(kb.make_params(protein=True, **mode))
                _same(_outputs(kb, cpt, ps, po, None, None), _outputs(kb, tie, ps, po, None, None), (split, mode, "protein"))
            finally:
                cpt.close(); tie.close()


@pytest.mark.parametrize("split", ["0", "1", "half", "nb"])
def test_tiered_checksums_equal_compact_and_host_transcoder(kb, golden, monkeypatch, split):
    """records (HBM part, then host part: slot 0), superblock table, sa_tax, seq_tax, k-mer table, bwtlen, n_sa; layout 3 (2 when nothing is split)"""
    with monkeypatch.context() as m:
        cpt, tie = _pair(kb, m, golden.fmi, golden.nodes, kb.make_params("mem"), split)
        want = kb.host_index_checksums(golden.fmi, golden.nodes)
        a, b = cpt.debug_index_checksums(), tie.debug_index_checksums()
        cpt.close(); tie.close()
    keep = [0, 1, 2, 3, 4, 5, 7]
    assert np.array_equal(a[keep], b[keep]) and np.array_equal(b[keep], want[keep]), (a, b, want)
    assert int(b[6]) == (2 if split == "nb" else 3)


def test_tiered_equals_compact_bench_like(kb, tmp_path, monkeypatch):
    """1 M PE150 pairs on a 100 k-protein index, records split in half"""
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    d = str(tmp_path); db = SynthDB(100000, 1); db.write(d + "/db.faa", d + "/nodes.dmp")
    fmi = build_fmi(d + "/db.faa", d + "/db", threads=16)
    s1, o1, s2, o2 = db.reads(7, 0, 1 << 20, 150, True)
    for mode, env in MODES[:3]:
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            cpt, tie = _pair(kb, m, fmi, d + "/nodes.dmp", kb.make_params(**mode), "half")
            try:
                _same(_outputs(kb, cpt, s1, o1, s2, o2, False), _outputs(kb, tie, s1, o1, s2, o2, False), (mode, env))
            finally:
                cpt.close(); tie.close()


@pytest.mark.parametrize("copies", [2, 3])
def test_tiered_scaled_index(kb, monkeypatch, tmp_path, copies):
    """kj_create_tiered(K): the base context and the K-fold context both split (the scaled suffix array is resolved through the base's split
    records); the K-fold results and checksums equal the plain compact K-fold context's"""
    d = str(tmp_path); db = SynthDB(3000, 11 + copies); db.write(d + "/base.faa", d + "/nodes.dmp")
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    base = build_fmi(d + "/base.faa", d + "/base", threads=4); nodes = d + "/nodes.dmp"
    s1, o1, s2, o2 = db.reads(5, 0, 20000, 150, True)
    with monkeypatch.context() as m:
        m.setenv("KJ_BUILD_CHUNK_ROWS", "65536")
        small = kb.Classifier(base, nodes, device=0, params=kb.make_params("mem")); nb_base = _nb(small.bwtlen); small.close()
        cpt, tie = _pair(kb, m, base, nodes, kb.make_params("mem"), nb_base // 2, copies=copies)
        try:
            assert tie.layout == 3
            a, b = cpt.debug_index_checksums(), tie.debug_index_checksums()
            assert np.array_equal(a[[0, 1, 2, 3, 4, 5, 7]], b[[0, 1, 2, 3, 4, 5, 7]])
            for mode in ("mem", "greedy"):
                cpt.set_params(kb.make_params(mode)); tie.set_params(kb.make_params(mode))
                _same(_outputs(kb, cpt, s1, o1, s2, o2, False), _outputs(kb, tie, s1, o1, s2, o2, False), (copies, mode))
        finally:
            cpt.close(); tie.close()


def _create_tiered(kb, fmi, nodes, params, copies, host_bytes):
    """kj_create_tiered called directly (Classifier takes kj_create / kj_create_scaled for host_memory = 0)"""
    L = kb.lib(); clf = kb.Classifier.__new__(kb.Classifier); clf._ctx = C.c_void_p(); clf.params = params; clf.device = 0
    f = C.c_void_p(); t = C.c_void_p(); kb._check(L.kj_fmi_load(fmi.encode(), C.byref(f))); kb._check(L.kj_nodes_load(nodes.encode(), C.byref(t)))
    try:
        iv = kb.KjIndexView(); tv = kb.KjTaxonomyView(); L.kj_fmi_view(f, C.byref(iv)); L.kj_nodes_view(t, C.byref(tv))
        clf.bwtlen = int(iv.bwtlen) * copies; clf.nseq = int(iv.nseq) * copies
        kb._check(L.kj_create_tiered(C.byref(clf._ctx), 0, C.byref(params), C.byref(iv), C.byref(tv), copies, host_bytes))
    finally:
        L.kj_nodes_free(t); L.kj_fmi_free(f)
    return clf


@pytest.mark.parametrize("force", [None, "KJ_FORCE_WIDE", "KJ_FORCE_COMPACT"])
def test_zero_host_bytes_changes_nothing(kb, golden, monkeypatch, force):
    """host_bytes = 0: the layout, index_bytes and results of kj_create_scaled, also with the developer hook set"""
    s1, o1, s2, o2 = golden.reads("pe150")[1:]
    with monkeypatch.context() as m:
        if force:
            m.setenv(force, "1")
        m.setenv("KJ_TIER_DEVICE_RECORDS", "1")
        for copies in (1, 2):
            a = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"), copies=copies)
            b = _create_tiered(kb, golden.fmi, golden.nodes, kb.make_params("mem"), copies, 0)
            try:
                assert (a.layout, a.index_bytes, a.host_bytes) == (b.layout, b.index_bytes, b.host_bytes) and b.host_bytes == 0
                _same(_outputs(kb, a, s1, o1, s2, o2, False), _outputs(kb, b, s1, o1, s2, o2, False), (force, copies))
            finally:
                a.close(); b.close()


def _mem_available():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


def _rss():
    for line in open("/proc/self/status"):
        if line.startswith("VmRSS:"):
            return int(line.split()[1]) * 1024
    return 0


@pytest.fixture(scope="module")
def db7m(tmp_path_factory):
    """the 7 M-row reference-built index of test_gpu_compact.py"""
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    d = str(tmp_path_factory.mktemp("db7m"))
    db = SynthDB(24000, 77); db.write(d + "/db.faa", d + "/nodes.dmp")
    return db, build_fmi(d + "/db.faa", d + "/db", threads=min(16, os.cpu_count())), d + "/nodes.dmp"


def _overflow_copies(kb, fmi, nodes):
    """copies of the 7 M-row index whose compact construction needs ~15 % more than the free HBM (records 1.003 B, sa_tax 0.5 B per row)"""
    small = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"))
    free = _free(); n_base = small.bwtlen
    return small, max(2, int(1.15 * free / 1.52 / n_base))


def test_index_beyond_hbm_gets_a_host_tier(kb, db7m):
    """A scaled index whose compact construction does not fit in the free HBM, no hook: with a sufficient budget it is built with a host tier
    (layout 2 with the suffix-array arrays on the host, or 3), holds no more HBM than was free, and its MEM results equal the base index's.
    (One read of these 1 M pairs, read 647999, is classified on every K-fold index of this base -- the plain compact 2e10-row context held in
    HBM alone included -- and unclassified on the base itself; that difference predates the host tier and is allowed here.)"""
    db, fmi, nodes = db7m
    small, copies = _overflow_copies(kb, fmi, nodes)
    n = small.bwtlen * copies; need = int(0.55 * n) + (8 << 30)
    if _mem_available() < need + (16 << 30):
        small.close()
        pytest.skip("needs %d GB of MemAvailable for the host tier of a %.2g-row index" % ((need + (16 << 30)) >> 30, n))
    free = _free()
    big = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"), copies=copies, host_memory=need)
    try:
        assert big.layout in (2, 3) and big.host_bytes > 0 and big.index_bytes <= free, (big.layout, big.host_bytes, big.index_bytes, free)
        s1, o1, s2, o2 = db.reads(9, 0, 1 << 20, 150, True)
        a = small.classify(s1, o1, s2, o2); b = big.classify(s1, o1, s2, o2)
        bad = np.nonzero((a[0] != b[0]) | (a[1] != b[1]))[0]
        assert set(bad.tolist()) <= {647999}, bad[:10]
        assert (a[0] != 0).mean() > 0.5
    finally:
        small.close(); big.close()


def test_host_budget_too_small(kb, db7m):
    """The same index with a 1 GB budget: KJ_ERR_NOMEM naming the HBM free, the host bytes needed and the budget; device memory and the process's
    resident memory are back where they were"""
    db, fmi, nodes = db7m
    small, copies = _overflow_copies(kb, fmi, nodes); small.close()
    before, rss = _free(), _rss()
    with pytest.raises(kb.KaijuError, match=r"error -7: .*\d+ bytes of HBM are free, its host tier needs \d+ bytes of pinned host memory, the budget \(host_bytes\) is 1073741824 bytes"):
        kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"), copies=copies, host_memory=1 << 30)
    assert abs(_free() - before) <= (2 << 20)
    assert _rss() <= rss + (256 << 20)
