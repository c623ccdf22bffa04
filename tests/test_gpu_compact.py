"""The compact rank layout on the GPU (kj_layout.h).  The device build equals the host transcoder array for array; a KJ_FORCE_COMPACT context
gives bit-identical outputs to the default context on every classify path; kj_create_scaled builds the same compact arrays as the reference-built
K-fold index; a 64-bit index whose wide construction does not fit in HBM is built compact without any hook, one whose wide construction fits
stays wide, and one that fits neither way fails with KJ_ERR_NOMEM before it allocates anything large."""
import ctypes as C
import os
import numpy as np
import pytest
from helpers import Oracle, SynthDB, build_fmi, have_ref, make_params, make_quirk_db

pytestmark = pytest.mark.gpu
ST = 2048


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


def _free():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


@pytest.mark.parametrize("chunk", [None, 65536])
def test_compact_device_build_equals_host_transcoder(kb, golden, tmp_path, monkeypatch, chunk):
    """records (slot 0), superblock table (slot 1), sa_tax, seq_tax, k-mer table, layout 2 (slot 6): device == host, on the golden index and on
    the quirk index (bwtlen = 3 * 2^16), with the default chunk and with one superblock per chunk"""
    monkeypatch.setenv("KJ_FORCE_COMPACT", "1")
    if chunk:
        monkeypatch.setenv("KJ_BUILD_CHUNK_ROWS", str(chunk))
    idx = [(golden.fmi, golden.nodes)]
    if have_ref():
        fmi, nodes, _ = make_quirk_db(str(tmp_path), nprot=768); idx.append((fmi, nodes))
    for fmi, nodes in idx:
        want = kb.host_index_checksums(fmi, nodes)
        clf = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"))
        got = clf.debug_index_checksums()
        assert clf.layout == 2 and int(got[6]) == 2
        assert np.array_equal(got, want), (fmi, got, want)
        clf.close()


def _verbose2(kb, clf, s1, o1, s2, o2):
    L = kb.lib()
    L.kj_classify_verbose2.argtypes = [C.c_void_p] * 5 + [C.c_uint64] + [C.c_void_p] * 6 + [C.c_void_p, C.c_uint32, C.c_void_p]
    n = len(o1) - 1
    tax = np.zeros(n, np.uint64); best = np.zeros(n, np.uint32); ids = np.zeros((n, 21), np.uint64); nids = np.zeros(n, np.uint8)
    a = np.zeros((n, 20), np.uint32); na = np.zeros(n, np.uint8); frag = np.zeros((n, ST), np.uint8); flen = np.zeros(n, np.uint32)
    p2 = (s2.ctypes.data, o2.ctypes.data) if s2 is not None else (None, None)
    kb._check(L.kj_classify_verbose2(clf._ctx, s1.ctypes.data, o1.ctypes.data, p2[0], p2[1], n, tax.ctypes.data, best.ctypes.data,
                                     ids.ctypes.data, nids.ctypes.data, a.ctypes.data, na.ctypes.data, frag.ctypes.data, ST, flen.ctypes.data))
    # only the first nids / nacc / flen entries of a read are defined (the rest of its row is whatever the device buffer held)
    col = lambda m: np.arange(m.shape[1])[None, :]
    ids[col(ids) >= nids[:, None]] = 0; a[col(a) >= na[:, None]] = 0; frag[col(frag) >= flen[:, None]] = 0
    return tax, best, ids, nids, a, na, frag, flen


def _outputs(kb, clf, s1, o1, s2, o2, verbose2=True):
    import torch
    n = len(o1) - 1
    dev = [None if a is None else torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else np.ascontiguousarray(a)).cuda()
           for a in (s1, o1, s2, o2)]
    d_tax = torch.zeros(n, dtype=torch.int64, device="cuda"); d_best = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_comp = torch.zeros(n, dtype=torch.int32, device="cuda")
    clf.classify_device2(*[None if t is None else t.data_ptr() for t in dev], n, d_tax.data_ptr(), d_best.data_ptr(), d_comp.data_ptr())
    torch.cuda.synchronize(); clf.check_errors()
    out = {"taxon": d_tax.cpu().numpy().view(np.uint64), "best": d_best.cpu().numpy().view(np.uint32), "taxon_index": d_comp.cpu().numpy().view(np.uint32)}
    clf.counts_reset()
    tax, best = clf.classify(s1, o1, s2, o2)
    assert np.array_equal(tax, out["taxon"]) and np.array_equal(best, out["best"])
    out["counts"] = clf.counts()
    _, _, ids = clf.classify_verbose(s1, o1, s2, o2); out["ids"] = ids
    if verbose2:
        for k, v in zip(("v2tax", "v2best", "v2ids", "v2nids", "acc", "nacc", "frag", "flen"), _verbose2(kb, clf, s1, o1, s2, o2)):
            out[k] = v
    return out


def _same(a, b, what):
    for k in a:
        if k == "counts":
            assert np.array_equal(a[k][0], b[k][0]) and np.array_equal(a[k][1], b[k][1]), (what, k)
        elif k == "ids":
            assert a[k] == b[k], what
        else:
            bad = np.nonzero(np.asarray(a[k] != b[k]).reshape(len(a[k]), -1).any(axis=1))[0]
            assert len(bad) == 0, (what, k, bad[:5])


def _compact_equals_default(kb, monkeypatch, fmi, nodes, works, modes, copies=1, verbose2=True):
    for mode, env in modes:
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            ref = kb.Classifier(fmi, nodes, device=0, params=kb.make_params(**mode), copies=copies)
            m.setenv("KJ_FORCE_COMPACT", "1")
            cpt = kb.Classifier(fmi, nodes, device=0, params=kb.make_params(**mode), copies=copies)
            try:
                assert cpt.layout == 2 and ref.layout != 2
                for w, (s1, o1, s2, o2) in enumerate(works):
                    _same(_outputs(kb, ref, s1, o1, s2, o2, verbose2), _outputs(kb, cpt, s1, o1, s2, o2, verbose2), (mode, env, w))
            finally:
                ref.close(); cpt.close()


MODES = [(dict(mode="mem"), {}), (dict(mode="greedy"), {}), (dict(mode="greedy"), {"KJ_NO_SPLIT": "1"}), (dict(mode="greedy", e=5, s=40), {})]


def test_compact_equals_default_golden(kb, golden, monkeypatch, tmp_path):
    """MEM, two-kernel and single-kernel Greedy, on the golden reads: taxa, best values, dense indices, id sets, accession sets, fragment strings,
    per-taxon counts; and the file pipeline's output"""
    _compact_equals_default(kb, monkeypatch, golden.fmi, golden.nodes, [golden.reads(t)[1:] for t in ("pe150", "se100")], MODES)
    gold = os.path.dirname(golden.fmi); outs = []
    for force in (False, True):
        with monkeypatch.context() as m:
            if force:
                m.setenv("KJ_FORCE_COMPACT", "1")
            clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"))
            o = str(tmp_path / ("o%d.tsv" % force))
            clf.classify_files(os.path.join(gold, "pe150_1.fq.gz"), os.path.join(gold, "pe150_2.fq.gz"), o, verbose=True)
            outs.append(open(o).read()); clf.close()
    assert outs[0] == outs[1] and len(outs[0]) > 1000


def test_compact_equals_default_long_reads_and_protein(kb, golden, monkeypatch):
    """reads up to 16,383 bases (work space in global memory) and protein input (-p)"""
    db = SynthDB(800, 3)
    s, o = db.long_reads(41, 0, 200, 300, 16383)
    _compact_equals_default(kb, monkeypatch, golden.fmi, golden.nodes, [(s, o, None, None)], [(dict(mode="mem"), {}), (dict(mode="greedy"), {})])
    s, o = db.protein_reads(42, 0, 600, 5, 5461)
    _compact_equals_default(kb, monkeypatch, golden.fmi, golden.nodes, [(s, o, None, None)], [(dict(mode="mem", protein=True), {}), (dict(mode="greedy", protein=True), {})])


def test_compact_equals_default_bench_like(kb, tmp_path, monkeypatch):
    """1 M PE150 pairs on a 100 k-protein index"""
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    d = str(tmp_path); db = SynthDB(100000, 1); db.write(d + "/db.faa", d + "/nodes.dmp")
    fmi = build_fmi(d + "/db.faa", d + "/db", threads=16)
    _compact_equals_default(kb, monkeypatch, fmi, d + "/nodes.dmp", [db.reads(7, 0, 1 << 20, 150, True)], MODES[:3], verbose2=False)


@pytest.mark.parametrize("copies", [2, 3, 7])
def test_compact_scaled_index_equals_reference_built_kfold_index(kb, tmp_path, monkeypatch, copies):
    """kj_create_scaled(K) on the compact layout (a compact base context resolves the scaled suffix array) == the reference-built K-fold index"""
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    from test_gpu_build import kfold_fasta
    monkeypatch.setenv("KJ_FORCE_COMPACT", "1")
    monkeypatch.setenv("KJ_BUILD_CHUNK_ROWS", "65536")
    d = str(tmp_path)
    db = SynthDB(3000, 11 + copies); db.write(d + "/base.faa", d + "/nodes.dmp")
    kfold_fasta(d + "/base.faa", d + "/rep.faa", copies)
    base = build_fmi(d + "/base.faa", d + "/base", threads=4); rep = build_fmi(d + "/rep.faa", d + "/rep", threads=4)
    nodes = d + "/nodes.dmp"
    want = kb.host_index_checksums(rep, nodes)
    big = kb.Classifier(base, nodes, device=0, params=kb.make_params("mem"), copies=copies)
    got = big.debug_index_checksums()
    assert big.layout == 2 and np.array_equal(got[[0, 1, 3, 4, 5, 6]], want[[0, 1, 3, 4, 5, 6]]), (got, want)
    s1, o1, s2, o2 = db.reads(5, 0, 20000, 150, True)
    orc = Oracle(rep, nodes)
    for mode in ("mem", "greedy"):
        big.set_params(kb.make_params(mode))
        a = big.classify(s1, o1, s2, o2)
        otax, obest = orc.classify_batch(make_params(mode), s1, o1, s2, o2)
        assert np.array_equal(a[0], otax) and np.array_equal(a[1], obest), mode
    big.close()


@pytest.fixture(scope="module")
def db7m(tmp_path_factory):
    """the 7 M-row reference-built index of test_gpu_build.py::test_index_beyond_2_pow_32_rows"""
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    d = str(tmp_path_factory.mktemp("db7m"))
    db = SynthDB(24000, 77); db.write(d + "/db.faa", d + "/nodes.dmp")
    return db, build_fmi(d + "/db.faa", d + "/db", threads=min(16, os.cpu_count())), d + "/nodes.dmp"


def test_compact_chosen_for_2e10_rows(kb, db7m):
    """~2e10 rows: the wide construction does not fit in 80 GB, so the index is built compact without any hook; it holds at most 1.125 B per row
    next to sa_tax, seq_tax, the k-mer table and the taxonomy; MEM results equal the base index's and the oracle's"""
    if _free() < (40 << 30):
        pytest.skip("needs 40 GB of free HBM")
    db, fmi, nodes = db7m
    small = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"))
    copies = int(round(2e10 / small.bwtlen))
    big = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"), copies=copies)
    try:
        n = big.bwtlen
        assert big.layout == 2 and n > 1.9e10
        sa = ((n - 1) >> 3) * 4; seq = big.nseq * 4; kmer = 20 ** 6 * 16
        assert big.index_bytes <= 1.125 * n + sa + seq + kmer + (256 << 20), (big.index_bytes, n)
        s1, o1, s2, o2 = db.reads(9, 0, 200000, 150, True)
        a = small.classify(s1, o1, s2, o2); b = big.classify(s1, o1, s2, o2)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        otax, obest = Oracle(fmi, nodes).classify_batch(make_params("mem"), s1[:int(o1[5000])], o1[:5001], s2[:int(o2[5000])], o2[:5001])
        assert np.array_equal(a[0][:5000], otax) and np.array_equal(a[1][:5000], obest)
        assert (a[0] != 0).mean() > 0.5
    finally:
        small.close(); big.close()


def test_wide_stays_wide_at_bench_size(kb, db7m):
    """An index sized the way bench.py sizes configs[3] (copies at 4.72 B per row with 6 GB left free, ~1.2e10 rows) is built wide."""
    if _free() < (60 << 30):
        pytest.skip("needs 60 GB of free HBM")
    db, fmi, nodes = db7m
    small = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"))
    free = _free(); copies = max(2, int(round(1.2e10 / small.bwtlen)))
    while copies > 2 and copies * small.bwtlen * 4.72 > free - (6 << 30):
        copies -= 1
    big = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"), copies=copies)
    try:
        assert big.layout == 1, (copies, big.bwtlen)
    finally:
        small.close(); big.close()


def test_index_too_large_for_either_layout(kb, db7m):
    """~1.5e11 rows fit neither layout: KJ_ERR_NOMEM with the bytes needed and free, and nothing is left allocated"""
    db, fmi, nodes = db7m
    small = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"))
    copies = int(round(1.5e11 / small.bwtlen)); small.close()
    before = _free()
    with pytest.raises(kb.KaijuError, match=r"error -7: .*does not fit in HBM: building it needs \d+ bytes .*, \d+ bytes are free"):
        kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"), copies=copies)
    assert abs(_free() - before) <= (2 << 20)
