"""Indexes of every suffix-array shape (tests/index_shapes.py: SA exponents 0-7, every residue class of nseq and bwtlen modulo 2^exponent at
exponents 2 and 5, 5- and 6-byte samples) on the GPU: the device build against the host transcoder on every layout and with a host tier,
classification and the verbose columns against the oracle, the row -> taxon array against the walk, scaled indexes against the index the
reference builds for the K-fold FASTA, device-native index files, and the file pipeline against the reference CLI."""
import os
import subprocess
import numpy as np
import pytest
import index_shapes as S
from helpers import Oracle, ROOT, build_fmi, have_ref, make_params, run_ref_kaiju
from test_gpu_build import kfold_fasta

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_ref(), reason="oracle/_ref (index builder) not built")]
LAYOUTS = [("narrow", {}), ("wide", {"KJ_FORCE_WIDE": "1"}), ("compact", {"KJ_FORCE_COMPACT": "1"})]
NAMES = sorted(S.SMALL) + sorted(S.WIDE)


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


@pytest.fixture(scope="module")
def fam(built, tmp_path_factory):
    return S.build_family(str(tmp_path_factory.mktemp("shapes")), NAMES, nreads=1500, wide_reads=1000)


def _reads(x):
    """SE100-like (34 residues), PE150-like pairs, the reads that walk into the guard row, 2-10 kb reads"""
    se = S.pack(x.reads + x.guard_reads)
    pe = S.pairs(x.reads[:600] + x.guard_reads)
    return se, pe, S.pack(x.long_reads)


def _ctx(kb, x, env, monkeypatch, **kw):
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        return kb.Classifier(x.fmi, x.nodes, device=0, params=kb.make_params("mem"), **kw)


def _check_vs_oracle(kb, clf, orc, x, what):
    (ss, so), (p1, q1, p2, q2), (ls, lo) = _reads(x)
    for kw in (dict(mode="mem"), dict(mode="greedy", e=3)):
        clf.set_params(kb.make_params(**kw)); P = make_params(**kw)
        for tag, a in (("se", (ss, so, None, None)), ("pe", (p1, q1, p2, q2))):
            tax, best = clf.classify(*a); otax, obest = orc.classify_batch(P, *a)
            bad = np.nonzero((tax != otax) | (best != obest))[0]
            assert len(bad) == 0, (what, kw, tag, [(int(i), int(tax[i]), int(otax[i]), int(best[i]), int(obest[i])) for i in bad[:5]])
        clf.set_max_read_len(kb.MAX_LONG_READ_LEN)
        tax, best = clf.classify(ls, lo); otax, obest = orc.classify_batch(P, ls, lo)
        assert np.array_equal(tax, otax) and np.array_equal(best, obest), (what, kw, "long")
        clf.set_max_read_len(kb.MAX_READ_LEN)


@pytest.mark.parametrize("name", NAMES)
def test_device_build_and_classification(kb, fam, monkeypatch, name):
    """Per layout (narrow, KJ_FORCE_WIDE, KJ_FORCE_COMPACT): debug_index_checksums == host_index_checksums, MEM and Greedy == the oracle on
    SE, PE and 2-10 kb reads (the guard-row reads included); a tiered context split at 0, half and all records gives the compact checksums."""
    x = fam[name]; orc = Oracle(x.fmi, x.nodes)
    for lay, env in LAYOUTS:
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            want = kb.host_index_checksums(x.fmi, x.nodes)
        clf = _ctx(kb, x, env, monkeypatch)
        try:
            got = clf.debug_index_checksums()
            assert np.array_equal(got, want), (lay, got, want)
            _check_vs_oracle(kb, clf, orc, x, lay)
        finally:
            clf.close()
        if lay == "compact":
            nb = x.h["bwtlen"] // 128 + 1
            for nd in (0, nb // 2, nb):
                t = _ctx(kb, x, dict(env, KJ_TIER_DEVICE_RECORDS=str(nd)), monkeypatch, host_memory=1 << 30)
                try:
                    got = t.debug_index_checksums(); keep = [0, 1, 2, 3, 4, 5, 7]
                    assert np.array_equal(got[keep], want[keep]) and t.host_bytes > 0, (nd, got, want)
                    if nd == nb // 2:
                        _check_vs_oracle(kb, t, orc, x, "tiered")
                finally:
                    t.close()


@pytest.mark.parametrize("name", ["e2_n0_b3", "e5_n0_b17", "e7", "e0", "w5"])
def test_verbose_columns_on_walking_layouts(kb, fam, monkeypatch, tmp_path, name):
    """classify_verbose id sets on the wide and compact contexts (both walk for every row) == the oracle's and the reference CLI's column 5;
    the narrow context (row -> taxon array) gives the same."""
    x = fam[name]; orc = Oracle(x.fmi, x.nodes); fa = str(tmp_path / "r.fa"); S.write_fasta(fa, x.reads[:800])
    seq, off = S.pack(x.reads[:800])
    for kw in (dict(mode="mem"), dict(mode="greedy", e=3)):
        ref = run_ref_kaiju(x.nodes, x.fmi, fa, None, threads=1, **kw); P = make_params(**kw)
        outs = []
        for lay, env in LAYOUTS:
            clf = _ctx(kb, x, env, monkeypatch)
            try:
                clf.set_params(kb.make_params(**kw)); outs.append(clf.classify_verbose(seq, off))
            finally:
                clf.close()
        tax, best, ids = outs[1]
        for i in range(len(x.reads[:800])):
            assert (ref["r%d" % i][1], ref["r%d" % i][2], ref["r%d" % i][3] if tax[i] else ()) == (int(tax[i]), int(best[i]), ids[i] if tax[i] else ()), (kw, i)
        for i in np.nonzero(tax)[0][:200]:
            assert ids[i] == tuple(orc.classify_one(P, x.reads[i].encode())[2])
        for o in (outs[0], outs[2]):
            assert np.array_equal(o[0], tax) and np.array_equal(o[1], best) and o[2] == ids


@pytest.mark.parametrize("name", ["e0", "e5_n0_b17", "e7"])
def test_row_tax_equals_walk(kb, fam, monkeypatch, name):
    """The narrow context resolves taxa with its row -> taxon array, the KJ_FORCE_WIDE one with the SA walk: bit-identical results"""
    x = fam[name]; (ss, so), (p1, q1, p2, q2), _ = _reads(x)
    a, b = _ctx(kb, x, {}, monkeypatch), _ctx(kb, x, {"KJ_FORCE_WIDE": "1"}, monkeypatch)
    try:
        assert a.layout == 0 and b.layout == 1
        for kw in (dict(mode="mem"), dict(mode="greedy", e=3)):
            for c in (a, b):
                c.set_params(kb.make_params(**kw))
            for args in ((ss, so), (p1, q1, p2, q2)):
                r, s = a.classify(*args), b.classify(*args)
                assert np.array_equal(r[0], s[0]) and np.array_equal(r[1], s[1]), kw
    finally:
        a.close(); b.close()


@pytest.mark.parametrize("name", ["e0", "e5_n0_b17"])
@pytest.mark.parametrize("copies", [2, 3])
def test_scaled_index_equals_reference_built_kfold_index(kb, fam, tmp_path, name, copies):
    """kj_create_scaled(copies) == the index kaiju-mkbwt / -mkfmi build for the K-fold FASTA at the same exponent: array checksums (the sampled
    SA through classification) and MEM / Greedy results, the reads that start at the suffix of the K-fold index's last sampled row included.
    nseq = 128 with a bwtlen that is no multiple of 32 stays in the guard class at every K: there the scaled index resolves that row to its
    sequence's taxon where the reference-built index has no entry, and no result changes, because the other copies of the sequence lie in
    the same match interval and carry the same taxon."""
    x = fam[name]; d = str(tmp_path)
    kfold_fasta(x.faa, d + "/rep.faa", copies)
    rep = S._build_exp0(d + "/rep.faa", d + "/rep") if x.exp == 0 else build_fmi(d + "/rep.faa", d + "/rep", threads=4, exponent=x.exp)
    rx = S.fmi_header(rep); m = 1 << x.exp
    assert (rx["nseq"] % m == 0 and rx["bwtlen"] % m != 0) == (x.exp > 0)
    want = kb.host_index_checksums(rep, x.nodes)
    big = kb.Classifier(x.fmi, x.nodes, device=0, params=kb.make_params("mem"), copies=copies)
    ref_built = kb.Classifier(rep, x.nodes, device=0, params=kb.make_params("mem"))
    try:
        got = big.debug_index_checksums()
        assert np.array_equal(got[[0, 1, 3, 4, 5, 6]], want[[0, 1, 3, 4, 5, 6]]), (got, want)
        orc = Oracle(rep, x.nodes)
        extra = []
        if x.exp:                                   # reads that start at the suffix of the K-fold index's last sampled row (base row k' / K)
            import random
            from helpers import oracle_lib
            L = oracle_lib(); idx = L.ko_index_load(x.fmi.encode())
            iseq, pos = S.true_suffix(L, idx, x.h["alen"], (((rx["bwtlen"] - 1) >> x.exp) << x.exp) // copies); L.ko_index_free(idx)
            prot = x.prots[int(S.fmi_seq_names(x.fmi)[iseq][3:12])]; rnd = random.Random(copies)
            extra = [S._dna(prot[st:st + 40], rnd, 0.0) for st in range(pos, min(pos + m, len(prot) - 12))]
            assert extra
        ss, so = S.pack(x.reads + x.guard_reads + extra); p1, q1, p2, q2 = S.pairs(x.reads[:600] + extra)
        for kw in (dict(mode="mem"), dict(mode="greedy", e=3)):
            for c in (big, ref_built):
                c.set_params(kb.make_params(**kw))
            for args in ((ss, so), (p1, q1, p2, q2)):
                a, b = big.classify(*args), ref_built.classify(*args)
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (kw, np.nonzero(a[0] != b[0])[0][:5])
                o = orc.classify_batch(make_params(**kw), *args)
                assert np.array_equal(a[0], o[0]) and np.array_equal(a[1], o[1]), kw
    finally:
        big.close(); ref_built.close()


@pytest.mark.parametrize("name", ["e0", "e5_n0_b17", "e7", "w6"])
def test_native_index_file_roundtrip(kb, fam, tmp_path, name):
    """kj_native_index_write -> kj_create_from_native: the header passes kj_host_index_read's checks, same checksums and results as the context
    built from the .fmi (KJ_HOST_BUILD: the same host arrays, uploaded)."""
    x = fam[name]; p = str(tmp_path / "db.kjb")
    kb.write_native_index(x.fmi, x.nodes, p)
    a = kb.Classifier(p, None, device=0, params=kb.make_params("mem"))
    b = kb.Classifier(x.fmi, x.nodes, device=0, params=kb.make_params("mem"))
    try:
        assert np.array_equal(a.debug_index_checksums(), b.debug_index_checksums())
        (ss, so), (p1, q1, p2, q2), _ = _reads(x)
        for kw in (dict(mode="mem"), dict(mode="greedy", e=3)):
            for c in (a, b):
                c.set_params(kb.make_params(**kw))
            for args in ((ss, so), (p1, q1, p2, q2)):
                r, s = a.classify(*args), b.classify(*args)
                assert np.array_equal(r[0], s[0]) and np.array_equal(r[1], s[1]), kw
    finally:
        a.close(); b.close()


def test_file_pipeline_verbose_equals_reference_cli(fam, tmp_path):
    """`kaiju-b200 -v` == `kaiju -z 1 -v` byte for byte on the exponent-5 guard-class index"""
    x = fam["e5_n0_b17"]; fa = str(tmp_path / "r.fa"); S.write_fasta(fa, x.reads)
    for mode in (["-a", "mem"], ["-a", "greedy", "-e", "3"]):
        ours = subprocess.run([os.path.join(ROOT, "kaiju_b200", "kaiju-b200"), "-v", "-t", x.nodes, "-f", x.fmi, "-i", fa] + mode,
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
        ref = subprocess.run([os.path.join(ROOT, "oracle", "_ref", "kaiju"), "-z", "1", "-v", "-t", x.nodes, "-f", x.fmi, "-i", fa] + mode,
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True).stdout
        assert ours == ref and ours.count(b"\nC\t") > 500, mode
