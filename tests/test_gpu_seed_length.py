"""Greedy's seed length (-l) on the GPU: the sm_90a kernels against the reference's output at -l 9, 12 and 20 (tests/golden/make_golden_seed.py)
and against the oracle, at the k-mer widths production indexes use (6; 7 forced), on the fixed-profile two-kernel pair (PE150 at -m 11) and the
general kernels, the verbose kernels, the wide and compact layouts, the long-read kernels and the CLI.  The CPU counterpart, over the whole grid,
is tests/test_seed_length_emulated.py."""
import gzip
import os
import subprocess
import numpy as np
import pytest
from conftest import GOLD, ROOT
from helpers import Oracle, SynthDB, make_params

pytestmark = pytest.mark.gpu

SEEDS_GOLDEN = (9, 12, 20)


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


@pytest.fixture(scope="module")
def gclf(kb, golden):
    c = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"))
    yield c
    c.close()


def kbp(kb, kw, protein=False):
    return kb.make_params("greedy", m=kw.get("m", 11), e=kw.get("e", 3), s=kw.get("s", 65), seed=kw["seed"], E=kw.get("E", 0.01), protein=protein)


def same(tax, best, etax, ebest, what):
    bad = np.nonzero((tax != etax) | (best != ebest))[0]
    assert len(bad) == 0, (what, len(bad), [(int(i), int(tax[i]), int(etax[i]), int(best[i]), int(ebest[i])) for i in bad[:5]])


@pytest.mark.parametrize("tag", ["pe150", "se100"])
@pytest.mark.parametrize("seed", SEEDS_GOLDEN)
def test_gpu_seed_lengths_match_reference_golden(kb, gclf, golden, seed, tag):
    """PE150 at -m 11 runs the fixed-profile two-kernel pair, SE100 the general ones."""
    names, s1, o1, s2, o2 = golden.reads(tag)
    gclf.set_params(kbp(kb, dict(seed=seed)))
    tax, best = gclf.classify(s1, o1, s2, o2)
    etax, ebest, _ = golden.expected("greedy_l%d" % seed, tag)
    same(tax, best, etax, ebest, (seed, tag))


def test_gpu_seed_length_verbose_id_sets_match_reference(kb, gclf, golden):
    """kj_classify_verbose at -l 12: taxon, best and the id set == columns 3-5 of the reference's `kaiju -v -l 12`."""
    names, s1, o1, s2, o2 = golden.reads("pe150")
    gclf.set_params(kbp(kb, dict(seed=12)))
    tax, best, ids = gclf.classify_verbose(s1, o1, s2, o2)
    want = gzip.open(os.path.join(GOLD, "expected_v7_greedy_l12_pe150.tsv.gz"), "rt").read().splitlines()
    assert len(want) == len(names)
    for i, line in enumerate(want):
        p = line.split("\t")
        if p[0] == "C":
            assert (p[1], int(p[2]), int(p[3]), tuple(int(x) for x in p[4].split(",") if x)) == (names[i], int(tax[i]), int(best[i]), ids[i]), (line, ids[i])
        else:
            assert tax[i] == 0, line
    assert max(len(x) for x in ids) == 21


# (L, m, e, s): L below, at and above -m; m = 11 on PE150 selects the fixed-profile pair, the other m the general kernels
KMER_SETS = [dict(seed=7), dict(seed=12), dict(seed=40, m=20), dict(seed=12, m=9, e=5, s=50), dict(seed=7, m=7, e=8, s=50), dict(seed=24, m=11, e=8, s=40)]


@pytest.mark.parametrize("k", ["6", "7"])
def test_gpu_seed_lengths_at_production_kmer_widths(kb, golden, monkeypatch, k):
    """Greedy at k = 6 (indexes of >= 5e7 rows; -l 7 is L = k + 1) and k = 7, with L = k - 1 too: == the oracle and == the index's default table."""
    sets = KMER_SETS + [dict(seed=int(k) - 1), dict(seed=int(k) - 1, m=9, e=5, s=45)]
    ref = {}
    dflt = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"))
    for kw in sets:
        dflt.set_params(kbp(kb, kw))
        for tag in ("pe150", "se100"):
            _, s1, o1, s2, o2 = golden.reads(tag)
            ref[(str(kw), tag)] = dflt.classify(s1, o1, s2, o2)
    dflt.close()
    monkeypatch.setenv("KJ_KMER_K", k)
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"))
    orc = Oracle(golden.fmi, golden.nodes)
    for kw in sets:
        clf.set_params(kbp(kb, kw))
        for tag in ("pe150", "se100"):
            _, s1, o1, s2, o2 = golden.reads(tag)
            tax, best = clf.classify(s1, o1, s2, o2)
            otax, obest = orc.classify_batch(make_params("greedy", **kw), s1, o1, s2, o2)
            same(tax, best, otax, obest, (k, kw, tag, "oracle"))
            same(tax, best, *ref[(str(kw), tag)], (k, kw, tag, "default table"))
    clf.close()


@pytest.mark.parametrize("layout", ["KJ_FORCE_WIDE", "KJ_FORCE_COMPACT"])
def test_gpu_seed_lengths_on_wide_and_compact_layouts(kb, golden, monkeypatch, layout):
    monkeypatch.setenv(layout, "1")
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"))
    for seed in SEEDS_GOLDEN:
        clf.set_params(kbp(kb, dict(seed=seed)))
        for tag in ("pe150", "se100"):
            _, s1, o1, s2, o2 = golden.reads(tag)
            tax, best = clf.classify(s1, o1, s2, o2)
            etax, ebest, _ = golden.expected("greedy_l%d" % seed, tag)
            same(tax, best, etax, ebest, (layout, seed, tag))
    orc = Oracle(golden.fmi, golden.nodes); _, s1, o1, s2, o2 = golden.reads("pe150")
    for kw in (dict(seed=6, m=9, e=5, s=45), dict(seed=40, m=20)):
        clf.set_params(kbp(kb, kw))
        same(*clf.classify(s1, o1, s2, o2), *orc.classify_batch(make_params("greedy", **kw), s1, o1, s2, o2), (layout, kw))
    clf.close()


def test_gpu_seed_lengths_on_long_read_kernels(kb, golden):
    """Mates above 16,383 bases (the long-read kernels, max_read_len raised) and multi-block fragments of 1-16 kb reads and protein reads."""
    db = SynthDB(800, 3); orc = Oracle(golden.fmi, golden.nodes)
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"), max_read_len=40000)
    sl, ol = db.long_reads(61, 0, 12, 16384, 40000)
    ss, os_ = db.long_reads(62, 0, 300, 1000, 16383)
    sp, op = db.protein_reads(63, 0, 300, 50, 5461)
    for kw in (dict(seed=7), dict(seed=6, m=9, e=5, s=45), dict(seed=33, m=11, e=3, s=50), dict(seed=64, m=30, e=2)):
        clf.set_params(kbp(kb, kw))
        for s, o, what in ((sl, ol, "long kernels"), (ss, os_, "1-16 kb")):
            tax, best = clf.classify(s, o)
            otax, obest = orc.classify_batch(make_params("greedy", **kw), s, o)
            same(tax, best, otax, obest, (kw, what))
            assert (otax != 0).mean() > 0.4
        clf.set_params(kbp(kb, kw, protein=True))
        same(*clf.classify(sp, op), *orc.classify_batch(make_params("greedy", protein=True, **kw), sp, op), (kw, "protein"))
    clf.close()


@pytest.mark.parametrize("k", ["5", "6"])
def test_gpu_kmer_lower_bound_decides_below_the_last_active_block(kb, tmp_path, monkeypatch, k):
    """The one geometry in which the k-mer lower bound of a failed chain (j - k + 2) decides whether an open chain is completed
    (tests/test_seed_length_emulated.py::kdead_case), on the sm_90a kernels."""
    from helpers import have_ref, pack_reads
    from test_seed_length_emulated import kdead_case
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    fmi, nodes, reads, want = kdead_case(str(tmp_path), int(k))
    seq, off = pack_reads(reads); orc = Oracle(fmi, nodes)
    monkeypatch.setenv("KJ_KMER_K", k)
    clf = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("greedy"))
    for t, seed in enumerate((13, 16, 24)):
        kw = dict(seed=seed, m=11, e=0, s=40)
        clf.set_params(kb.make_params("greedy", m=11, e=0, s=40, seed=seed, seg=False, protein=True))
        otax, obest = orc.classify_batch(make_params("greedy", seg=False, protein=True, **kw), seq, off)
        same(*clf.classify(seq, off), otax, obest, (k, seed))
        assert otax[t] == want[t]
    clf.close()


def test_gpu_cli_seed_length_equals_reference_output(kb, golden, tmp_path):
    """kaiju-b200 -v -l 12 on the golden FASTQ == the reference's `kaiju -v -l 12` line for line (all seven columns); -l 12x is read as 12."""
    cli = os.path.join(ROOT, "kaiju_b200", "kaiju-b200")
    want = gzip.open(os.path.join(GOLD, "expected_v7_greedy_l12_pe150.tsv.gz"), "rt").read()
    for arg in ("12", "12x"):
        out = str(tmp_path / "o.tsv")
        subprocess.check_call([cli, "-t", golden.nodes, "-f", golden.fmi, "-i", os.path.join(GOLD, "pe150_1.fq.gz"), "-j", os.path.join(GOLD, "pe150_2.fq.gz"),
                               "-a", "greedy", "-l", arg, "-v", "-o", out], stderr=subprocess.DEVNULL)
        assert open(out).read().splitlines() == want.splitlines(), arg
