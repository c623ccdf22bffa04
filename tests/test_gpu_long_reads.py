"""Reads longer than KJ_MAX_READ_LEN on the GPU (kj_set_max_read_len / Classifier(max_read_len=)): the long-read kernels against the oracle
through every classify entry point, mixed batches, the default limit, the memory budget of a long launch, and the file pipeline against the
reference binary."""
import ctypes as C
import gzip
import os
import numpy as np
import pytest
from helpers import Oracle, SynthDB, have_ref, make_params, pack_reads, run_ref_kaiju
from test_long_reads_emulated import SETS, SET_IDS, adversarial_reads

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


@pytest.fixture(scope="module")
def db():
    return SynthDB(800, 3)


@pytest.fixture(scope="module")
def lclf(kb, golden):
    c = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"), max_read_len=kb.MAX_LONG_READ_LEN)
    yield c
    c.close()


def kbp(kb, kw):
    kw = dict(kw); mode = kw.pop("mode")
    return kb.make_params(mode, **kw)


def oracle(golden, kw, s1, o1, s2=None, o2=None):
    return Oracle(golden.fmi, golden.nodes).classify_batch(make_params(**kw), s1, o1, s2, o2)


@pytest.mark.parametrize("kw", SETS, ids=SET_IDS)
def test_long_reads_match_oracle(kb, lclf, golden, db, tmp_path, kw):
    """SE reads of 16,384 to 300,000 bases, PE mates of 16,384 to 100,000, the adversarial reads of test_long_reads_emulated and protein reads of
    5,462 to 100,000 residues: bit-exact against the oracle."""
    lclf.set_params(kbp(kb, kw))
    batches = [db.long_reads(61, 0, 24, 16384, 300000), pack_reads(adversarial_reads(db, tmp_path))]
    for s, o in batches:
        t, b = lclf.classify(s, o); ot, ob = oracle(golden, kw, s, o)
        assert np.array_equal(t, ot) and np.array_equal(b, ob)
    s1, o1 = db.long_reads(62, 0, 12, 16384, 100000); s2, o2 = db.long_reads(63, 0, 12, 16384, 100000)
    t, b = lclf.classify(s1, o1, s2, o2); ot, ob = oracle(golden, kw, s1, o1, s2, o2)
    assert np.array_equal(t, ot) and np.array_equal(b, ob)
    lclf.set_params(kbp(kb, dict(kw, protein=True)))
    s, o = db.protein_reads(64, 0, 16, 5462, 100000)
    t, b = lclf.classify(s, o); ot, ob = oracle(golden, dict(kw, protein=True), s, o)
    assert np.array_equal(t, ot) and np.array_equal(b, ob)


@pytest.mark.parametrize("layout", ["KJ_FORCE_WIDE", "KJ_FORCE_COMPACT"])
def test_long_reads_on_wide_and_compact_indexes(kb, golden, db, monkeypatch, layout):
    monkeypatch.setenv(layout, "1")
    c = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"), max_read_len=200000)
    s, o = db.long_reads(65, 0, 12, 16384, 200000)
    for kw in (SETS[0], SETS[3]):
        c.set_params(kbp(kb, kw)); t, b = c.classify(s, o); ot, ob = oracle(golden, kw, s, o)
        assert np.array_equal(t, ot) and np.array_equal(b, ob), kw
    c.close()


def test_long_reads_through_every_entry_point(kb, lclf, golden, db, monkeypatch):
    """kj_classify2, kj_classify_verbose / verbose2 (against the short kernels on the same reads where those apply: the id sets), host-buffer
    chunking (KJ_CHUNK_READS), kj_classify_device / device2, kj_classify_multi with one context; per-taxon counts once per successful call."""
    import torch
    kw = SETS[0]; lclf.set_params(kbp(kb, kw))
    s, o = db.long_reads(66, 0, 40, 1000, 60000)
    ot, ob = oracle(golden, kw, s, o)
    monkeypatch.setenv("KJ_CHUNK_READS", "1024")
    t, b = lclf.classify(s, o); assert np.array_equal(t, ot) and np.array_equal(b, ob)
    monkeypatch.delenv("KJ_CHUNK_READS")
    t, b, ids = lclf.classify_verbose(s, o); assert np.array_equal(t, ot) and np.array_equal(b, ob)
    # the id sets of the reads the short kernels also take are the same on both paths
    short = np.nonzero(np.diff(o) <= 16383)[0]
    sc = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kbp(kb, kw))
    for i in short[:10]:
        st, sb, sids = sc.classify_verbose(s[o[i]:o[i + 1]], np.array([0, o[i + 1] - o[i]], np.uint64))
        assert st[0] == t[i] and sids[0] == ids[i]
    sc.close()
    ds = torch.from_numpy(s.copy()).cuda(); do = torch.from_numpy(o.astype(np.int64)).cuda()
    dt = torch.zeros(len(o) - 1, dtype=torch.int64, device="cuda"); db_ = torch.zeros(len(o) - 1, dtype=torch.int32, device="cuda")
    lclf.classify_device(ds.data_ptr(), do.data_ptr(), None, None, len(o) - 1, dt.data_ptr(), db_.data_ptr()); torch.cuda.synchronize()
    assert np.array_equal(dt.cpu().numpy().astype(np.uint64), ot) and np.array_equal(db_.cpu().numpy().astype(np.uint32), ob)
    lclf.counts_reset()
    tax = np.zeros(len(o) - 1, np.uint64); best = np.zeros(len(o) - 1, np.uint32)
    arr = (C.c_void_p * 1)(lclf._ctx)
    L = kb.lib(); L.kj_classify_multi.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_uint64, C.c_void_p, C.c_void_p]
    assert L.kj_classify_multi(arr, 1, s.ctypes.data, o.ctypes.data, None, None, len(o) - 1, tax.ctypes.data, best.ctypes.data) == 0
    assert np.array_equal(tax, ot)
    ids_, cnt = lclf.counts()
    assert int(np.sum(cnt)) == len(o) - 1


def test_mixed_batch_and_default_path(kb, golden, db):
    """Short reads in a batch that also holds long ones give the results of a short-only batch; a batch without long reads runs the default
    context's launches and geometry; raising the limit allocates nothing."""
    import torch
    from test_gpu_lifetime import free_bytes
    names, s1, o1, s2, o2 = golden.reads("se100")
    base = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"))
    t0, b0 = base.classify(s1, o1); l0 = base.kernel_launches; g0 = base.launch_geometry
    base.close()
    # device memory a first call takes: the same with the limit raised (nothing is sized for long reads unless a batch holds them)
    used = []
    for limit in (None, kb.MAX_LONG_READ_LEN):
        c = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"), max_read_len=limit)
        torch.cuda.synchronize(); f = free_bytes(torch); c.classify(s1, o1); torch.cuda.synchronize(); used.append(f - free_bytes(torch)); c.close()
    assert abs(used[0] - used[1]) <= (2 << 20), used
    raised = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"), max_read_len=kb.MAX_LONG_READ_LEN)
    t1, b1 = raised.classify(s1, o1)
    assert np.array_equal(t0, t1) and np.array_equal(b0, b1) and raised.kernel_launches == l0 and raised.launch_geometry == g0
    ls, lo = db.long_reads(67, 0, 4, 20000, 50000)
    reads = [bytes(s1[o1[i]:o1[i + 1]]) for i in range(len(o1) - 1)] + [bytes(ls[lo[i]:lo[i + 1]]) for i in range(4)]
    ms, mo = pack_reads([r.decode() for r in reads])
    t2, b2 = raised.classify(ms, mo)
    n = len(o1) - 1
    assert np.array_equal(t2[:n], t0) and np.array_equal(b2[:n], b0)
    ot, ob = oracle(golden, dict(mode="greedy"), ms, mo)
    assert np.array_equal(t2, ot) and np.array_equal(b2, ob)
    # the long reads get chunks of their own: a long read inside a stretch of short reads leaves the stretch on the short kernels
    reads = reads[:n // 2] + reads[n:n + 1] + reads[n // 2:n]
    ms, mo = pack_reads([r.decode() for r in reads])
    l3 = raised.kernel_launches; t3, b3 = raised.classify(ms, mo)
    ot, ob = oracle(golden, dict(mode="greedy"), ms, mo)
    assert np.array_equal(t3, ot) and np.array_equal(b3, ob)
    assert raised.kernel_launches > l3
    raised.close()


def test_limits(kb, golden):
    """The default refuses 16,384 bases; kj_set_max_read_len takes [16383, 1048575]; a read of exactly 1,048,575 bases completes and one base
    more is refused; a launch whose scratch does not fit the budget fails cleanly with KJ_ERR_NOMEM and the context stays usable."""
    c = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"))
    rng = np.random.default_rng(9)
    long = rng.choice(np.frombuffer(b"ACGT", np.uint8), 1048576)
    with pytest.raises(kb.KaijuError):
        c.classify(long[:16384], np.array([0, 16384], np.uint64))
    for bad in (16382, 1048576, 0):
        with pytest.raises(kb.KaijuError):
            c.set_max_read_len(bad)
    c.set_max_read_len(kb.MAX_LONG_READ_LEN)
    t, b = c.classify(long[:1048575], np.array([0, 1048575], np.uint64))
    ot, ob = oracle(golden, dict(mode="mem"), long[:1048575], np.array([0, 1048575], np.uint64))
    assert np.array_equal(t, ot) and np.array_equal(b, ob)
    with pytest.raises(kb.KaijuError):
        c.classify(long, np.array([0, 1048576], np.uint64))
    os.environ["KJ_LONG_BUDGET_MB"] = "64"
    try:
        with pytest.raises(kb.KaijuError, match="bytes of work space per warp"):
            c.classify(long[:500000], np.array([0, 500000], np.uint64))
    finally:
        del os.environ["KJ_LONG_BUDGET_MB"]
    names, s1, o1, s2, o2 = golden.reads("pe150")
    t, b = c.classify(s1, o1, s2, o2); ot, ob = oracle(golden, dict(mode="mem"), s1, o1, s2, o2)
    assert np.array_equal(t, ot) and np.array_equal(b, ob)
    c.close()


@pytest.mark.parametrize("verbose", [False, True])
@pytest.mark.parametrize("gz", [False, True])
def test_files_nanopore_like(kb, golden, db, tmp_path, verbose, gz):
    """kj_classify_files on a FASTQ of 1 kb to 300 kb reads: output equal to the reference binary's after sorting (verbose: the five columns the
    file pipeline writes), per-taxon counts equal."""
    if not have_ref():
        pytest.skip("oracle/_ref (reference binary) not available")
    s, o = db.long_reads(68, 0, 30, 1000, 300000)
    fq = str(tmp_path / ("r.fq.gz" if gz else "r.fq"))
    with (gzip.open(fq, "wt") if gz else open(fq, "w")) as f:
        for i in range(len(o) - 1):
            r = bytes(s[o[i]:o[i + 1]]).decode(); f.write("@r%d\n%s\n+\n%s\n" % (i, r, "I" * len(r)))
    c = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"), max_read_len=300000)
    c.counts_reset()
    out = str(tmp_path / "gpu.tsv"); ref = str(tmp_path / "ref.tsv")
    c.classify_files(fq, None, out, verbose=verbose)
    run_ref_kaiju(golden.nodes, golden.fmi, fq, mode="mem", verbose=verbose, out=ref)
    cols = (lambda l: "\t".join(l.split("\t")[:5])) if verbose else (lambda l: l)      # the file pipeline writes columns 1-5 of `kaiju -v`
    assert sorted(open(out).read().splitlines()) == sorted(cols(l) for l in open(ref).read().splitlines())
    ids, cnt = c.counts()
    want = {}
    for line in open(ref):
        p = line.split("\t"); want[int(p[2]) if p[0] == "C" else 0] = want.get(int(p[2]) if p[0] == "C" else 0, 0) + 1
    assert {int(i): int(n) for i, n in zip(ids, cnt)} == want
    c.close()
