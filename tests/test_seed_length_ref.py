"""Pins the oracle against the UNMODIFIED reference binary (oracle/_ref/kaiju) in Greedy mode at seed lengths (-l) other than the default 7,
on a fresh seeded index, read by read: taxon, score and the column-5 id set of `kaiju -v`.  CPU only; skipped when oracle/_ref has not been
built.  The kernels are checked against the oracle at these seeds in tests/test_seed_length_emulated.py and tests/test_gpu_seed_length.py."""
import os, subprocess, tempfile
import pytest
from helpers import REF_DIR, SynthDB, build_fmi, Oracle, make_params, have_ref, read_fastq_packed, pack_reads, parse_kaiju_output

pytestmark = pytest.mark.skipif(not have_ref(), reason="oracle/_ref not built")


def run_ref_greedy(nodes, fmi, f1, f2, protein, kw):
    """`kaiju -a greedy -l <seed> -m -e -s -v` on f1 (and f2); returns {name: (C/U, taxon, best, ids)}"""
    cmd = [os.path.join(REF_DIR, "kaiju"), "-t", nodes, "-f", fmi, "-i", f1, "-z", "8", "-v", "-a", "greedy", "-l", str(kw["seed"]),
           "-m", str(kw.get("m", 11)), "-e", str(kw.get("e", 3)), "-s", str(kw.get("s", 65))] + (["-j", f2] if f2 else []) + (["-p"] if protein else [])
    return parse_kaiju_output(subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True).stdout.decode())


def _write_fasta(path, seq, off):
    with open(path, "w") as f:
        for i in range(len(off) - 1):
            f.write(">r%d\n%s\n" % (i, seq[int(off[i]):int(off[i + 1])].tobytes().decode()))


# Greedy at seed lengths (-l) other than the default 7: below, at and above the minimum match length -m, with 0 to 8 substitutions
SEED_SETS = [dict(seed=7, m=7, e=8, s=50), dict(seed=8, m=11, e=0), dict(seed=9, m=9, e=3, s=55), dict(seed=11, m=11, e=5, s=50),
             dict(seed=12, m=9, e=3), dict(seed=16, m=12, e=5, s=60), dict(seed=24, m=11, e=8, s=40), dict(seed=40, m=20, e=3, s=65)]
SEED_IDS = ["l%d_m%d_e%d" % (kw["seed"], kw["m"], kw["e"]) for kw in SEED_SETS]


@pytest.fixture(scope="module")
def work_seed(built):
    """A fresh index and four read sets: PE150, SE100, DNA reads of 300 b - 16 kb, protein reads (-p) of 5-1500 residues."""
    d = tempfile.mkdtemp(prefix="kjrefs_")
    db = SynthDB(3000, 13)
    db.write(d + "/db.faa", d + "/nodes.dmp")
    fmi = build_fmi(d + "/db.faa", d + "/db", threads=4)
    db.write_fastq(23, 0, 2000, 150, True, d + "/r1.fq", d + "/r2.fq")
    db.write_fastq(24, 0, 2000, 100, False, d + "/s.fq")
    ls, lo = db.long_reads(33, 0, 150, 300, 16383); ps, po = db.protein_reads(34, 0, 1000, 5, 1500)
    _write_fasta(d + "/long.fa", ls, lo); _write_fasta(d + "/prot.fa", ps, po)
    sets = {"pe150": (d + "/r1.fq", d + "/r2.fq", False), "se100": (d + "/s.fq", None, False), "long": (d + "/long.fa", None, False),
            "protein": (d + "/prot.fa", None, True)}
    return d, fmi, sets


def _packed(path):
    if path.endswith(".fq"):
        return read_fastq_packed(path)
    names, seqs = [], []
    for line in open(path).read().splitlines():
        if line.startswith(">"):
            names.append(line[1:])
        else:
            seqs.append(line)
    seq, off = pack_reads(seqs)
    return names, seq, off


def _ref_equals_oracle(d, fmi, f1, f2, protein, kw):
    """Read by read: the reference's taxon, score and column-5 id set (-v) == the oracle's.  Returns the number of classified reads."""
    ref = run_ref_greedy(d + "/nodes.dmp", fmi, f1, f2, protein, kw)
    names, s1, o1 = _packed(f1)
    s2 = o2 = None
    if f2:
        _, s2, o2 = _packed(f2)
    orc = Oracle(fmi, d + "/nodes.dmp"); P = make_params("greedy", protein=protein, **kw); ncls = 0
    for i, nm in enumerate(names):
        t, b, ids = orc.classify_one(P, s1[int(o1[i]):int(o1[i + 1])].tobytes(), s2[int(o2[i]):int(o2[i + 1])].tobytes() if f2 else None)
        r = ref[nm]
        assert (r[1], r[2], r[3] if r[1] else ()) == (t, b, tuple(sorted(ids)) if t else ()), (kw, nm, r, t, b, ids)
        ncls += t != 0
    return ncls


@pytest.mark.parametrize("kw", SEED_SETS, ids=SEED_IDS)
@pytest.mark.parametrize("tag", ["pe150", "se100", "long", "protein"])
def test_oracle_equals_reference_at_seed_lengths(work_seed, tag, kw):
    d, fmi, sets = work_seed
    f1, f2, protein = sets[tag]
    ncls = _ref_equals_oracle(d, fmi, f1, f2, protein, kw)
    assert ncls == 0 if tag == "se100" and kw["seed"] > 33 else ncls > 100       # SE100 fragments have at most 33 residues


def test_seed_length_above_every_fragment_classifies_nothing(work_seed):
    """-l 51 on PE150 / SE100 reads (fragments of at most 50 residues): maxMatches records no match, so no read is classified."""
    d, fmi, sets = work_seed
    for tag in ("pe150", "se100"):
        f1, f2, _ = sets[tag]
        assert _ref_equals_oracle(d, fmi, f1, f2, False, dict(seed=51, m=11, e=3, s=40)) == 0
