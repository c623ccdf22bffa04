"""A small DB in which one protein segment occurs in many sequences of distinct taxa, and reads taken from it: their kept suffix
intervals hold dozens of rows and more than 20 distinct taxa, so the taxon look-up runs several waves of 32 rows and stops on the
21st id, inside an interval or across two.  Needs oracle/_ref (index builder)."""
import random
import numpy as np
from helpers import build_fmi

AA = "ACDEFGHIKLMNPQRSTVWY"
CODON = {'A': 'GCT', 'R': 'CGT', 'N': 'AAT', 'D': 'GAT', 'C': 'TGT', 'Q': 'CAA', 'E': 'GAA', 'G': 'GGT', 'H': 'CAT', 'I': 'ATT',
         'L': 'CTG', 'K': 'AAA', 'M': 'ATG', 'F': 'TTT', 'P': 'CCT', 'S': 'TCT', 'T': 'ACT', 'W': 'TGG', 'Y': 'TAT', 'V': 'GTT'}


def _revcomp(s):
    return s[::-1].translate(str.maketrans("ACGT", "TGCA"))


def make_shared_core_db(d, seed=11, npairs=3000):
    """Sequences (taxon):  40 x flank + CORE (120 aa) + flank, 1000..1039 (genus 900); the first 12 of them carry a tail TAIL (60 aa)
    as well; 24 x flank + first half of CORE + flank, 2000..2023 (genus 901); 300 random background proteins, 3000..3049 (genus 902).
    Reads: PE150 pairs whose mates are 50-residue windows of CORE or TAIL (either strand, 1% base errors).
    Returns (fmi, nodes, seq1, off1, seq2, off2)."""
    rnd = random.Random(seed)
    prot = lambda n: "".join(rnd.choice(AA) for _ in range(n))
    core, tail = prot(120), prot(60)
    recs = []
    for i in range(40):
        recs.append(("C%d_%d" % (i, 1000 + i), prot(30) + core + prot(30) + (tail + prot(10) if i < 12 else "")))
    for i in range(24):
        recs.append(("H%d_%d" % (i, 2000 + i), prot(25) + core[:60] + prot(25)))
    for i in range(300):
        recs.append(("B%d_%d" % (i, 3000 + i % 50), prot(rnd.randrange(80, 400))))
    with open(d + "/db.faa", "w") as f:
        for name, s in recs:
            f.write(">%s\n%s\n" % (name, s))
    with open(d + "/nodes.dmp", "w") as f:
        f.write("1\t|\t1\t|\tno rank\t|\n")
        for g in (900, 901, 902):
            f.write("%d\t|\t1\t|\tgenus\t|\n" % g)
        for t in range(1000, 1040):
            f.write("%d\t|\t900\t|\tspecies\t|\n" % t)
        for t in range(2000, 2024):
            f.write("%d\t|\t901\t|\tspecies\t|\n" % t)
        for t in range(3000, 3050):
            f.write("%d\t|\t902\t|\tspecies\t|\n" % t)
    fmi = build_fmi(d + "/db.faa", d + "/db", threads=2)

    def mate():
        src = rnd.choice((core, core, tail))
        s0 = rnd.randrange(0, len(src) - 50 + 1)
        dna = "".join(CODON[c] for c in src[s0:s0 + 50])
        dna = "".join(ch if rnd.random() > 0.01 else rnd.choice("ACGT") for ch in dna)
        return _revcomp(dna) if rnd.random() < 0.5 else dna

    pairs = [(mate(), mate()) for _ in range(npairs)]
    pack = lambda rs: (np.frombuffer("".join(rs).encode(), dtype=np.uint8).copy(),
                       np.concatenate([[0], np.cumsum([len(r) for r in rs])]).astype(np.uint64))
    s1, o1 = pack([a for a, _ in pairs]); s2, o2 = pack([b for _, b in pairs])
    return fmi, d + "/nodes.dmp", s1, o1, s2, o2
