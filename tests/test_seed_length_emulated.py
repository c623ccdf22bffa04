"""Greedy's seed length (-l, kj_params.seed_length) on the CPU warp emulator against the oracle and the reference's own output.

The Greedy search of kj_core_greedy.h depends on the seed length L in several ways that each rest on an exactness argument: the k-mer
shortcut of kj_chain_start (only when L >= k), the lower bound of a chain that died inside the k-mer (j - k + 2, kj_chain_lbval), the
active end positions (j >= L - 1) of the 32-lane blocks and of the look-ahead block, the `i <= 1` break and the prefix minimum of the
recorded starts.  Which rule decides changes with how L compares to the k-mer width k, to 32 and to the fragment length, so L is crossed
here with k (KJ_KMER_K), the layouts, the one- and two-kernel Greedy, short, long and protein reads, and the checkpoint-quirk index.
The host transcoder builds k-mer tables of up to 6 letters; the 7-letter table exists on the device only (tests/test_gpu_seed_length.py).
Seeds 5 and 6 lie below the reference CLI's minimum of 7 but are valid kj_params: they put L right below k = 6 and k = 7."""
import gzip
import os
import random
import ctypes as C
import numpy as np
import pytest
import emu_compact
import test_kernel_logic_emulated as K
from conftest import GOLD
from helpers import Oracle, SynthDB, make_params

# (L, m, e, s): L below, at and above -m; e from 0 to 8; L = 51 lies above every fragment of the golden reads (at most 50 residues)
GRID = [dict(seed=5, m=9, e=3, s=50), dict(seed=6, m=11, e=3), dict(seed=7, m=7, e=8, s=50), dict(seed=8, m=11, e=0), dict(seed=9, m=9, e=3, s=55),
        dict(seed=11, m=11, e=5, s=50), dict(seed=12, m=9, e=3), dict(seed=16, m=12, e=5, s=60), dict(seed=24, m=11, e=8, s=40),
        dict(seed=40, m=20, e=3), dict(seed=51, m=11, e=3, s=40)]
SUBSET = [GRID[1], GRID[4], GRID[7], GRID[9]]
SEEDS_GOLDEN = (9, 12, 20)

emu = K.emu


@pytest.fixture(scope="module")
def emu_c(built, tmp_path_factory):
    return emu_compact.load(str(tmp_path_factory.mktemp("emu_compact")), K.KjParams)


_oracle_cache = {}


def oracle_for(golden, kw, tag):
    """the oracle's answer on a golden read set (it does not depend on the k-mer table or the layout)"""
    key = (tuple(sorted(kw.items())), tag)
    if key not in _oracle_cache:
        _, s1, o1, s2, o2 = golden.reads(tag)
        _oracle_cache[key] = Oracle(golden.fmi, golden.nodes).classify_batch(make_params("greedy", **kw), s1, o1, s2, o2)
    return _oracle_cache[key]


def check_golden(E, golden, kw, tags=("pe150", "se100")):
    for tag in tags:
        names, s1, o1, s2, o2 = golden.reads(tag)
        otax, obest = oracle_for(golden, kw, tag)
        tax, best = K.emu_classify(E, golden.fmi, golden.nodes, make_params("greedy", **kw), s1, o1, s2, o2)
        bad = np.nonzero((tax != otax) | (best != obest))[0]
        assert len(bad) == 0, (kw, tag, len(bad), [(names[i], int(tax[i]), int(otax[i]), int(best[i]), int(obest[i])) for i in bad[:5]])
        if kw["seed"] > 50:
            assert not otax.any()
        else:
            assert (otax != 0).mean() > (0.3 if kw["seed"] <= 33 or tag == "pe150" else -1)


@pytest.mark.parametrize("k", ["0", "3", "5", "6"])
def test_seed_grid_on_golden_reads(emu, golden, monkeypatch, k):
    """Every seed of the grid at k-mer widths 0 (no table), 3, 5 (the golden index's default) and 6 (indexes of >= 5e7 rows)."""
    monkeypatch.setenv("KJ_KMER_K", k)
    for kw in GRID:
        check_golden(emu, golden, kw)


@pytest.mark.parametrize("split", [False, True], ids=["one_kernel", "two_kernel"])
@pytest.mark.parametrize("layout", ["narrow", "KJ_FORCE_WIDE", "KJ_FORCE_COMPACT"])
def test_seed_lengths_on_every_layout(emu, emu_c, golden, monkeypatch, layout, split):
    """The 32-bit, 64-bit and compact instantiations, through the one-kernel Greedy and the front-end / search pair (KJ_EMU_SPLIT)."""
    if layout != "narrow":
        monkeypatch.setenv(layout, "1")
    if split:
        monkeypatch.setenv("KJ_EMU_SPLIT", "1")
    for kw in SUBSET:
        check_golden(emu_c if layout == "KJ_FORCE_COMPACT" else emu, golden, kw)


LONG_SEEDS = [dict(seed=6, m=11, e=3), dict(seed=7, m=7, e=8, s=50), dict(seed=16, m=12, e=5, s=60), dict(seed=33, m=11, e=3, s=50),
              dict(seed=40, m=20, e=3), dict(seed=64, m=30, e=2)]


@pytest.fixture(scope="module")
def long_sets():
    db = SynthDB(800, 3)
    return {False: db.long_reads(43, 0, 60, 1000, 16383), True: db.protein_reads(44, 0, 120, 50, 5461)}


@pytest.mark.parametrize("k", ["0", "6"])
def test_seed_lengths_on_long_and_protein_reads(emu, golden, long_sets, monkeypatch, k):
    """DNA reads of 1-16 kb and protein reads of up to 5,461 residues: fragments of many 32-lane blocks, where L meets the look-ahead
    block and the block edges (L = 33 and 64 start a fragment's search one or two blocks below its end)."""
    monkeypatch.setenv("KJ_KMER_K", k)
    orc = Oracle(golden.fmi, golden.nodes)
    for kw in LONG_SEEDS:
        for prot, (s, o) in long_sets.items():
            P = make_params("greedy", protein=prot, **kw)
            otax, obest = orc.classify_batch(P, s, o)
            rc, tax, best = K.emu_classify_rc(emu, golden.fmi, golden.nodes, P, s, o)
            bad = np.nonzero((tax != otax) | (best != obest))[0]
            assert rc == 0 and len(bad) == 0, (kw, prot, rc, [(int(i), int(tax[i]), int(otax[i]), int(best[i]), int(obest[i])) for i in bad[:5]])
            assert (otax != 0).mean() > 0.4


def test_seed_lengths_on_index_with_bwtlen_multiple_of_65536(emu, built, tmp_path, monkeypatch):
    """ix.mono = 0 (the reference's checkpoint quirk): no chain bounds, the general recorded-start rule, the 64-bit kernels."""
    from helpers import have_ref, make_quirk_db, pack_reads
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    fmi, nodes, reads = make_quirk_db(str(tmp_path))
    seq, off = pack_reads(reads); orc = Oracle(fmi, nodes)
    for k in ("5", "0"):
        monkeypatch.setenv("KJ_KMER_K", k)
        for kw in (dict(seed=6, m=11, e=3), dict(seed=9, m=9, e=5, s=40), dict(seed=16, m=11, e=3), dict(seed=40, m=20, e=8, s=40)):
            P = make_params("greedy", **kw); otax, obest = orc.classify_batch(P, seq, off)
            rc, tax, best = K.emu_classify_rc(emu, fmi, nodes, P, seq, off)
            assert rc == 0 and np.array_equal(tax, otax) and np.array_equal(best, obest), (k, kw)
            assert (otax != 0).mean() > (0.1 if kw["seed"] < 40 else -1)


@pytest.mark.parametrize("split", [False, True], ids=["one_kernel", "two_kernel"])
@pytest.mark.parametrize("seed", SEEDS_GOLDEN)
def test_seed_lengths_match_reference_golden(emu, golden, monkeypatch, seed, split):
    """The reference's own output at -l 9, 12, 20 (tests/golden/make_golden_seed.py)."""
    if split:
        monkeypatch.setenv("KJ_EMU_SPLIT", "1")
    for tag in ("pe150", "se100"):
        names, s1, o1, s2, o2 = golden.reads(tag)
        tax, best = K.emu_classify(emu, golden.fmi, golden.nodes, make_params("greedy", seed=seed), s1, o1, s2, o2)
        etax, ebest, _ = golden.expected("greedy_l%d" % seed, tag)
        bad = np.nonzero((tax != etax) | (best != ebest))[0]
        assert len(bad) == 0, [(names[i], int(tax[i]), int(etax[i]), int(best[i]), int(ebest[i])) for i in bad[:5]]


def test_seed_fixtures_differ_from_the_default_seed(golden):
    """The -l fixtures are not the -l 7 output under another name: the seed changes the result of some reads."""
    for tag in ("pe150", "se100"):
        d = golden.expected("greedy_default", tag)
        for seed in SEEDS_GOLDEN:
            e = golden.expected("greedy_l%d" % seed, tag)
            assert (d[0] != e[0]).sum() + (d[1] != e[1]).sum() > 0, (seed, tag)


def test_seed_length_verbose_columns_match_reference(emu, golden):
    """All seven columns of `kaiju -v -l 12` on PE150 (taxon, best, id set, accessions, fragment strings) from the emulated kernel logic."""
    import kaiju_b200 as kb
    L = kb.lib(); L.kj_fmi_accession.restype = C.c_char_p; L.kj_fmi_accession.argtypes = [C.c_void_p, C.c_uint32]
    f = C.c_void_p(); assert L.kj_fmi_load(golden.fmi.encode(), C.byref(f)) == 0
    emu.kjemu_classify_v2.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64] + [C.c_void_p] * 7 + [C.c_uint32, C.c_void_p, C.c_int]
    ST = 2048
    names, s1, o1, s2, o2 = golden.reads("pe150")
    kp = K.KjParams(**make_params("greedy", seed=12)); h = emu.kjemu_create(golden.fmi.encode(), golden.nodes.encode(), C.byref(kp)); assert h
    n = len(o1) - 1; tax = np.zeros(n, np.uint64); best = np.zeros(n, np.uint32); ids = np.zeros((n, 21), np.uint64); nids = np.zeros(n, np.uint8)
    acc = np.zeros((n, 20), np.uint32); nacc = np.zeros(n, np.uint8); frag = np.zeros((n, ST), np.uint8); flen = np.zeros(n, np.uint32)
    rc = emu.kjemu_classify_v2(h, s1.ctypes.data, o1.ctypes.data, s2.ctypes.data, o2.ctypes.data, n, tax.ctypes.data, best.ctypes.data, ids.ctypes.data,
                               nids.ctypes.data, acc.ctypes.data, nacc.ctypes.data, frag.ctypes.data, ST, flen.ctypes.data, 4)
    emu.kjemu_destroy(h); assert rc == 0
    want = gzip.open(os.path.join(GOLD, "expected_v7_greedy_l12_pe150.tsv.gz"), "rt").read().split("\n"); bad = []
    for i in range(n):
        line = "U\t%s\t0" % names[i] if not tax[i] else "C\t%s\t%d\t%d\t%s,\t%s\t%s" % (
            names[i], tax[i], best[i], ",".join(str(int(x)) for x in ids[i, :nids[i]]),
            "".join(L.kj_fmi_accession(f, int(a)).decode() + "," for a in acc[i, :nacc[i]]), bytes(frag[i, :flen[i]]).decode())
        if line != want[i]:
            bad.append((line[:160], want[i][:160]))
    L.kj_fmi_free(f)
    assert not bad, bad[:3]


def test_seed_length_drawn_with_the_other_parameters(emu, golden, monkeypatch):
    """Seeded sweep: L drawn together with -m, -e, -s, -E, SEG, the k-mer width and the one- / two-kernel Greedy; emulated kernel == oracle."""
    rnd = random.Random(12)
    orc = Oracle(golden.fmi, golden.nodes)
    monkeypatch.setenv("KJ_VARIANT_CAP", "65536")         # -e 8 at a low -s: a ring the library would enlarge and retry with (test_gpu_parity.py)
    for trial in range(14):
        kw = dict(seed=rnd.choice([5, 6, 7, 8, 10, 13, 17, 25, 31, 32, 33, 45]), m=rnd.choice([6, 9, 11, 12, 15, 25]), e=rnd.choice([0, 1, 2, 3, 5, 8]),
                  s=rnd.choice([30, 45, 65, 90]), E=rnd.choice([10.0, 0.01, 1e-6]), seg=rnd.random() < 0.7)
        env = dict(KJ_KMER_K=rnd.choice(["0", "3", "5", "6"]))
        if rnd.random() < 0.5:
            env["KJ_EMU_SPLIT"] = "1"
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        tag = rnd.choice(["pe150", "se100"])
        names, s1, o1, s2, o2 = golden.reads(tag)
        P = make_params("greedy", **kw)
        otax, obest = orc.classify_batch(P, s1, o1, s2, o2)
        tax, best = K.emu_classify(emu, golden.fmi, golden.nodes, P, s1, o1, s2, o2)
        bad = np.nonzero((tax != otax) | (best != obest))[0]
        assert len(bad) == 0, (kw, env, tag, [(names[i], int(tax[i]), int(otax[i]), int(best[i]), int(obest[i])) for i in bad[:5]])
        for k in env:
            monkeypatch.delenv(k)


def kdead_case(d, k, seeds=(13, 16, 24), n=40):
    """Protein reads of n residues on a purpose-built index in which the k-mer lower bound of kj_chain_lbval (a chain that died inside the k-mer
    starts at j - k + 2 or later) is what decides whether an open chain has to be completed.  That happens in one geometry only: a KDEAD chain is
    never directly below an open one, so the bound comes from lane 0 of the look-ahead block, below a block whose lowest lanes are inactive (j < L - 1).
    Read layout (p = n - 31 - k): junk, then A = a database segment of L letters at [p, p + L - 1] whose k-mer starting at p - 1 does not occur, then a
    letter c with A[1:] + c in another sequence.  The chain at p + L (start p + 1) is completed first; the chain at p + L - 1 (start exactly p, the bound,
    length exactly L) is recorded by maxMatches and wins: A starts with W (BLOSUM62 11), c is A (4).  Returns (fmi, nodes, reads, taxa of A's sequences)."""
    from helpers import build_fmi
    rnd = random.Random(40 + k); aa = "ACDEFGHIKLMNPQRSTVWY"
    rs = lambda m: "".join(rnd.choice(aa) for _ in range(m))
    prots = [(99, rs(300)) for _ in range(300)]; reads = []; want = []
    for t, L in enumerate(seeds):
        p = n - 31 - k
        assert p >= 2 and 9 <= L - p and p + L <= n - 1
        A = "W" + "".join(rnd.choice(aa[:-2]) for _ in range(L - 1))
        prots += [(100 + 2 * t, rs(30) + A + "G" + rs(30)), (101 + 2 * t, rs(30) + A[1:] + "A" + rs(30))]
        while True:
            r = rs(p) + A + "A" + rs(n - p - L - 1)
            if not any(r[p - 1:p - 1 + k] in s for _, s in prots):
                break
        reads.append(r); want.append(100 + 2 * t)
    with open(d + "/db.faa", "w") as f:
        for i, (tx, s) in enumerate(prots):
            f.write(">P%d_%d constructed sequence\n%s\n" % (i, tx, s))      # (kaiju-mkbwt sizes its buffer from the file size)
    with open(d + "/nodes.dmp", "w") as f:
        f.write("1\t|\t1\t|\tno rank\t|\n")
        for tx in sorted(set(tx for tx, _ in prots)):
            f.write("%d\t|\t1\t|\tspecies\t|\n" % tx)
    return build_fmi(d + "/db.faa", d + "/db", threads=2), d + "/nodes.dmp", reads, want


@pytest.mark.parametrize("k", ["5", "6"])
def test_kmer_lower_bound_decides_below_the_last_active_block(emu, built, tmp_path, monkeypatch, k):
    from helpers import have_ref, pack_reads
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    fmi, nodes, reads, want = kdead_case(str(tmp_path), int(k))
    seq, off = pack_reads(reads); orc = Oracle(fmi, nodes)
    monkeypatch.setenv("KJ_KMER_K", k)
    for seed in (13, 16, 24):
        P = make_params("greedy", m=11, e=0, s=40, seed=seed, seg=False, protein=True)
        otax, obest = orc.classify_batch(P, seq, off)
        rc, tax, best = K.emu_classify_rc(emu, fmi, nodes, P, seq, off)
        assert rc == 0 and np.array_equal(tax, otax) and np.array_equal(best, obest), (k, seed, tax, otax, best, obest)
        assert otax[(13, 16, 24).index(seed)] == want[(13, 16, 24).index(seed)], (k, seed, otax)      # the read built for this seed: A's taxon
