"""The long-read kernel instances (kj_classify_item<..., LONG = true>: 64-bit queue payloads, 32-bit match positions, prefix sums and SEG counts,
unclamped scores, the ranked fragment queue) on the CPU warp emulator (tests/emu/kj_emu_long.cpp) against the oracle: reads of 16,384 bases and
more, protein reads of 5,462 residues and more, on narrow, wide and compact indexes, and reads built to overflow each narrow field of the short
kernels.  The same build also runs the golden short-read sets (verbose columns, name mode): the long instances take any read length."""
import os
import numpy as np
import pytest
import emu_long
import test_kernel_logic_emulated as K
from conftest import GOLDEN_CONFIGS
from helpers import Oracle, SynthDB, have_ref, make_params, pack_reads, run_ref_kaiju

SETS = [dict(mode="mem"), dict(mode="mem", m=8, seg=False), dict(mode="greedy"), dict(mode="greedy", e=5, s=50)]
SET_IDS = ["mem_default", "mem_m8_X", "greedy_default", "greedy_e5_s50"]


@pytest.fixture(scope="module")
def emu(built, tmp_path_factory):
    return emu_long.load(str(tmp_path_factory.mktemp("emu_long")), K.KjParams)


@pytest.fixture(scope="module")
def db():
    return SynthDB(800, 3)


def check(emu, golden, P, s1, o1, s2=None, o2=None):
    otax, obest = Oracle(golden.fmi, golden.nodes).classify_batch(P, s1, o1, s2, o2)
    tax, best = K.emu_classify(emu, golden.fmi, golden.nodes, P, s1, o1, s2, o2)
    bad = np.nonzero((tax != otax) | (best != obest))[0]
    assert len(bad) == 0, [(int(i), int(tax[i]), int(otax[i]), int(best[i]), int(obest[i])) for i in bad[:5]]
    return otax, obest


@pytest.mark.parametrize("kw", SETS, ids=SET_IDS)
def test_long_reads_match_oracle(emu, golden, db, kw):
    """Single-end DNA reads of 16,384 to 60,000 bases and paired ones of 16,384 to 30,000 per mate."""
    s, o = db.long_reads(51, 0, 10, 16384, 60000)
    otax, _ = check(emu, golden, make_params(**kw), s, o)
    assert (otax != 0).mean() > 0.5
    s1, o1 = db.long_reads(52, 0, 6, 16384, 30000); s2, o2 = db.long_reads(53, 0, 6, 16384, 30000)
    check(emu, golden, make_params(**kw), s1, o1, s2, o2)


@pytest.mark.parametrize("kw", SETS, ids=SET_IDS)
def test_long_protein_reads_match_oracle(emu, golden, db, kw):
    """Protein input (-p) of 5,462 to 20,000 residues."""
    s, o = db.protein_reads(54, 0, 10, 5462, 20000)
    check(emu, golden, make_params(protein=True, **kw), s, o)


@pytest.mark.parametrize("layout", ["KJ_FORCE_WIDE", "KJ_FORCE_COMPACT"])
@pytest.mark.parametrize("kw", [SETS[0], SETS[3]], ids=[SET_IDS[0], SET_IDS[3]])
def test_long_reads_on_wide_and_compact_indexes(emu, golden, db, monkeypatch, layout, kw):
    monkeypatch.setenv(layout, "1")
    s, o = db.long_reads(55, 0, 6, 16384, 40000)
    check(emu, golden, make_params(**kw), s, o)


@pytest.mark.parametrize("cfg", sorted(GOLDEN_CONFIGS))
def test_long_instances_on_short_golden_reads(emu, golden, cfg):
    """Short reads through the long instances give the reference's golden outputs (a long launch takes the short reads of its batch too)."""
    K.test_emulated_kernel_matches_reference_golden(emu, golden, cfg, "pe150")


@pytest.mark.parametrize("cfg", ["mem_default", "mem_m5_noseg", "greedy_default", "greedy_e5_s40"])
def test_long_instances_verbose_columns(emu, golden, cfg):
    K.test_emulated_verbose_columns_match_reference(emu, golden, cfg)


@pytest.mark.parametrize("cfg", ["mem_default", "greedy_default"])
def test_long_instances_name_mode(emu, golden, cfg):
    K.test_emulated_name_frontend_matches_reference_kaijux(emu, golden, cfg)


CODON = {'A': 'GCT', 'R': 'CGT', 'N': 'AAT', 'D': 'GAT', 'C': 'TGT', 'Q': 'CAA', 'E': 'GAA', 'G': 'GGT', 'H': 'CAT', 'I': 'ATT',
         'L': 'CTG', 'K': 'AAA', 'M': 'ATG', 'F': 'TTT', 'P': 'CCT', 'S': 'TCT', 'T': 'ACT', 'W': 'TGG', 'Y': 'TAT', 'V': 'GTT'}


def db_proteins(db, d):
    """The proteins of the golden index (tests/golden/make_golden.py builds it from SynthDB(800, 3))."""
    faa = os.path.join(str(d), "db.faa"); db.write(faa, os.path.join(str(d), "nodes.dmp"))
    return ["".join(ch for ch in "".join(p.split("\n")[1:]) if ch in CODON) for p in open(faa).read().split(">")[1:]]


def adversarial_reads(db, d):
    """One read per narrow field of the short kernels:
    - a stop-free frame of ~21,000 residues of concatenated database proteins: matches start beyond array index 32,767 and the fragment's
      Greedy self-score exceeds 65,535;
    - a 70,000-residue stop-free low-complexity run followed by database protein in the same frame: SEG's counts exceed 65,535;
    - random DNA (hundreds of queue entries) followed by a database protein with a low-complexity block inside: SEG pieces are pushed
      behind the ranked entries (late entries)."""
    import random
    rnd = random.Random(5); prots = [p for p in db_proteins(db, d) if len(p) > 100]
    cat = "".join(prots)[:21000]
    r1 = "".join(CODON[c] for c in cat)
    r2 = "GCT" * 70000 + "".join(CODON[c] for c in "".join(prots[:3]))
    p = prots[4]; mid = len(p) // 2
    r3 = "".join(rnd.choice("ACGT") for _ in range(30000)) + "".join(CODON[c] for c in p[:mid] + "Q" * 60 + p[mid:])
    return [r1, r2, r3]


@pytest.mark.parametrize("kw", SETS, ids=SET_IDS)
def test_long_reads_overflowing_short_fields(emu, golden, db, tmp_path, kw):
    s, o = pack_reads(adversarial_reads(db, tmp_path))
    otax, obest = check(emu, golden, make_params(**kw), s, o)
    assert otax[0] != 0 and otax[2] != 0


def test_longest_admitted_read(emu, golden):
    """The emulator entry point admits KJ_MAX_LONG_READ_LEN bases and refuses one more (the library's limit is checked on the GPU)."""
    kp = K.KjParams(**make_params("mem"))
    import ctypes as C
    h = emu.kjemu_create(golden.fmi.encode(), golden.nodes.encode(), C.byref(kp)); assert h
    s = np.frombuffer(b"A" * 1048576, np.uint8); o = np.array([0, 1048576], np.uint64)
    tax = np.zeros(1, np.uint64); best = np.zeros(1, np.uint32)
    assert emu.kjemu_classify(h, s.ctypes.data, o.ctypes.data, None, None, 1, tax.ctypes.data, best.ctypes.data, 1) == -5
    emu.kjemu_destroy(h)


def seg_region_reads(db, d):
    """Stop-free frames whose low-complexity region is longer than the reference's 10,001-entry ln(n!) table, so that SEG's trim search uses
    Stirling's formula (s_lnfact): a database protein, then 12,000 or 20,000 residues drawn from two or three letters, then another protein."""
    import random
    rnd = random.Random(11); prots = [p for p in db_proteins(db, d) if len(p) > 100]
    out = []
    for k, (letters, weights, n) in enumerate((("AS", (3, 1), 12000), ("GSA", (5, 3, 1), 20000), ("KE", (1, 1), 15000))):
        lc = "".join(rnd.choices(letters, weights, k=n))
        out.append("".join(CODON[c] for c in prots[10 + k] + lc + prots[20 + k]))
    return out


def verbose_lines(kb_lib, fmi_handle, names, tax, best, ids, nids, acc, nacc, frag, flen):
    """The seven columns of `kaiju -v` from the arrays of kj_classify_verbose2."""
    lines = {}
    for i, name in enumerate(names):
        lines[name] = "U\t%s\t0" % name if not tax[i] else "C\t%s\t%d\t%d\t%s,\t%s\t%s" % (
            name, tax[i], best[i], ",".join(str(int(x)) for x in ids[i, :nids[i]]),
            "".join(kb_lib.kj_fmi_accession(fmi_handle, int(a)).decode() + "," for a in acc[i, :nacc[i]]), bytes(frag[i, :flen[i]]).decode())
    return lines


def reference_verbose(golden, reads, kw, d):
    fq = os.path.join(str(d), "long.fq")
    with open(fq, "w") as f:
        for i, r in enumerate(reads):
            f.write("@r%d\n%s\n+\n%s\n" % (i, r, "I" * len(r)))
    kw = dict(kw); mode = kw.pop("mode")
    out = os.path.join(str(d), "ref.tsv")
    run_ref_kaiju(golden.nodes, golden.fmi, fq, mode=mode, m=kw.get("m", 11), e=kw.get("e", 3), s=kw.get("s", 65), seg=kw.get("seg", True), out=out)
    return {l.split("\t")[1]: l for l in open(out).read().splitlines()}


@pytest.mark.parametrize("kw", SETS, ids=SET_IDS)
def test_long_reads_verbose_columns_match_reference_binary(emu, golden, db, tmp_path, kw):
    """All seven columns of `kaiju -v` (taxon, best, id set, accession set, matched fragment strings) for long reads, from the emulated long
    instances, equal the reference binary's: random long reads, the reads that overflow the short fields, and SEG regions longer than 10,000
    residues (the fragment strings show where SEG cut)."""
    import ctypes as C
    import kaiju_b200 as kb
    if not have_ref():
        pytest.skip("oracle/_ref (reference binary) not available")
    s0, o0 = db.long_reads(57, 0, 6, 16384, 40000)
    reads = [bytes(s0[o0[i]:o0[i + 1]]).decode() for i in range(len(o0) - 1)] + adversarial_reads(db, tmp_path) + seg_region_reads(db, tmp_path)
    want = reference_verbose(golden, reads, kw, tmp_path)
    L = kb.lib(); L.kj_fmi_accession.restype = C.c_char_p; L.kj_fmi_accession.argtypes = [C.c_void_p, C.c_uint32]
    f = C.c_void_p(); assert L.kj_fmi_load(golden.fmi.encode(), C.byref(f)) == 0
    emu.kjemu_classify_v2.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64] + [C.c_void_p] * 7 + [C.c_uint32, C.c_void_p, C.c_int]
    s, o = pack_reads(reads); n = len(reads); ST = 1 << 18
    kp = K.KjParams(**make_params(**kw)); h = emu.kjemu_create(golden.fmi.encode(), golden.nodes.encode(), C.byref(kp)); assert h
    tax = np.zeros(n, np.uint64); best = np.zeros(n, np.uint32); ids = np.zeros((n, 21), np.uint64); nids = np.zeros(n, np.uint8)
    acc = np.zeros((n, 20), np.uint32); nacc = np.zeros(n, np.uint8); frag = np.zeros((n, ST), np.uint8); flen = np.zeros(n, np.uint32)
    rc = emu.kjemu_classify_v2(h, s.ctypes.data, o.ctypes.data, None, None, n, tax.ctypes.data, best.ctypes.data, ids.ctypes.data, nids.ctypes.data,
                               acc.ctypes.data, nacc.ctypes.data, frag.ctypes.data, ST, flen.ctypes.data, 4)
    emu.kjemu_destroy(h); assert rc == 0
    got = verbose_lines(L, f, ["r%d" % i for i in range(n)], tax, best, ids, nids, acc, nacc, frag, flen)
    L.kj_fmi_free(f)
    bad = [(k, got[k][:200], want[k][:200]) for k in want if got[k] != want[k]]
    assert not bad, bad[:3]
    assert sum(1 for v in want.values() if v.startswith("C")) >= n // 2


@pytest.mark.parametrize("kw", [SETS[0], SETS[2]], ids=[SET_IDS[0], SET_IDS[2]])
def test_long_queue_pop_cost_does_not_grow_with_the_read(emu, golden, db, kw):
    """The emulator's counters (KjEmuStats lq_tops / lq_slots): queue slots read per look-up of the top entry do not follow the fragment count
    from 20 kb to 500 kb reads (25 times as many fragments).  The ranked run is read at its head; what is scanned is the SEG pieces still
    pending above the pop threshold (dead ones are dropped by the scan), a few per look-up at 500 kb."""
    import ctypes as C
    emu.kjemu_stats.argtypes = [C.c_void_p, C.c_int, C.c_int]
    per_top = {}
    for n in (20000, 500000):
        s, o = db.long_reads(71, 0, 2, n, n)
        buf = (C.c_ulonglong * 32)(); emu.kjemu_stats(buf, 32, 1)
        K.emu_classify(emu, golden.fmi, golden.nodes, make_params(**kw), s, o, None, None)
        k = emu.kjemu_stats(buf, 32, 1); assert k == 17
        tops, slots = int(buf[15]), int(buf[16])
        assert tops > 0
        per_top[n] = slots / tops
    assert per_top[500000] <= 0.25 * (500000 / 20000) * per_top[20000] and per_top[500000] < 16, per_top
