"""Small protein databases whose suffix-array shape is chosen: the SA exponent, nseq and bwtlen modulo 2^exponent, and the width of a
sample.  Built with the reference's own kaiju-mkbwt -e E / kaiju-mkfmi (oracle/_ref), for tests/test_index_shapes_emulated.py and
tests/test_gpu_index_shapes.py.

kaiju-mkbwt samples every row k >= nseq with k % 2^E == 0, entry (k >> E) - (((nseq - 1) >> E) + 1), but the header counts
ncheck = (bwtlen >> E) - (nseq >> E) samples (suffixArray.c:160, 206-216).  The two counts differ in two residue classes:
  nseq % 2^E == 0, bwtlen % 2^E != 0  ("guard"): the last sampled row has no entry; the device reads a guard entry ("no taxon") there;
  nseq % 2^E != 0, bwtlen % 2^E == 0: the header counts one entry more than is written, an entry no row addresses.
"""
import os
import random
import struct
import subprocess
import zlib
import numpy as np
from helpers import REF_DIR, build_fmi, oracle_lib

AA = "ACDEFGHIKLMNPQRSTVWY"
CODON = {'A': 'GCT', 'R': 'CGT', 'N': 'AAT', 'D': 'GAT', 'C': 'TGT', 'Q': 'CAA', 'E': 'GAA', 'G': 'GGT', 'H': 'CAT', 'I': 'ATT',
         'L': 'CTG', 'K': 'AAA', 'M': 'ATG', 'F': 'TTT', 'P': 'CCT', 'S': 'TCT', 'T': 'ACT', 'W': 'TGG', 'Y': 'TAT', 'V': 'GTT'}
NTAX = 7

# name: (exponent, nseq, bwtlen % 2^exponent, protein lengths [lo, hi), one long protein of this many residues or 0)
SMALL = {}
for _e, _q in ((2, 32), (5, 4)):
    _m = 1 << _e
    for _r in (0, 1, _m - 1):
        for _b in (0, _m // 2 + 1):
            SMALL["e%d_n%d_b%d" % (_e, _r, _b)] = (_e, _q * _m + _r, _b, (40, 200), 0)
SMALL.update({"e0": (0, 150, 0, (40, 200), 0), "e1": (1, 129, 0, (40, 200), 0), "e4": (4, 144, 9, (40, 200), 0), "e7": (7, 128, 77, (40, 300), 0)})
WIDE = {"w5": (5, 131072, 3, (12, 31), 16400), "w6": (5, 530000, 3, (5, 11), 1100000)}   # 5-byte and 6-byte samples


def fmi_header(path):
    """BWT + suffix-array header of a .fmi (bwt.c:40-45, suffixArray.c:261-277): bwtlen, nseq, ncheck, exponent, nbytes, sbits, pbits."""
    with open(path, "rb") as f:
        b = f.read(256)
    ln, nseq, alen = struct.unpack_from("<qii", b, 0)
    _, ncheck, exp, nbytes, sbits, pbits = struct.unpack_from("<qqiiii", b, 16 + alen)
    return dict(bwtlen=ln, nseq=nseq, ncheck=ncheck, exp=exp, nbytes=nbytes, sbits=sbits, pbits=pbits, sa_off=16 + alen + 52, alen=alen)


def fmi_seq_names(path):
    """The sequence names of a .fmi in the index's own sequence order (kaiju-mkbwt sorts the sequences; mkbwt.c:718)."""
    h = fmi_header(path)
    with open(path, "rb") as f:
        f.seek(h["sa_off"]); b = f.read(h["nseq"] * 256)
    out, o = [], 0
    for _ in range(h["nseq"]):
        out.append(b[o + 1:o + 1 + b[o]].decode()); o += 1 + b[o]
    return out


def _build_exp0(faa, prefix):
    """kaiju-mkfmi does not read the suffix array when the exponent is 0 ("the whole SA is saved", mkfmi.c:58-59) and then writes it from a
    null pointer (it dies).  The index it would write: run it with the .sa header's exponent set to 1 (the body is read and copied as it is;
    the header's check mask stays kaiju-mkbwt's 0), then set the exponent of the .fmi back to 0.  Every other byte is the reference tools'."""
    subprocess.check_call([os.path.join(REF_DIR, "kaiju-mkbwt"), "-n", "2", "-e", "0", "-a", AA, "-o", prefix, faa],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    with open(prefix + ".sa", "r+b") as f:                      # .sa header: len, ncheck, chpt_exp, ...
        f.seek(16); assert struct.unpack("<i", f.read(4))[0] == 0; f.seek(16); f.write(struct.pack("<i", 1))
    subprocess.check_call([os.path.join(REF_DIR, "kaiju-mkfmi"), prefix], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    h = fmi_header(prefix + ".fmi"); o = 16 + h["alen"]
    with open(prefix + ".fmi", "r+b") as f:                     # chpt_exp at +16, check (2^exp - 1) at +40 of the SA header
        f.seek(o + 40); assert struct.unpack("<q", f.read(8))[0] == 0
        f.seek(o + 16); assert struct.unpack("<i", f.read(4))[0] == 1; f.seek(o + 16); f.write(struct.pack("<i", 0))
    for ext in (".bwt", ".sa"):
        os.remove(prefix + ext)
    return prefix + ".fmi"


def true_suffix(L, idx, alen, k):
    """(sequence, position) of row k by LF steps back to the sequence start: no suffix-array sample involved (oracle FMindex)."""
    steps = 0
    while True:
        c = next(c for c in range(alen) if L.ko_fmindex(idx, c, k + 1) - L.ko_fmindex(idx, c, k) == 1)
        k = L.ko_fmindex(idx, c, k); steps += 1
        if c == 0:
            return int(k), steps - 1


def _dna(prot, rnd, mut=0.02):
    s = "".join(CODON[c] for c in prot)
    s = "".join(ch if rnd.random() > mut else rnd.choice("ACGT") for ch in s)
    return s[::-1].translate(str.maketrans("ACGT", "TGCA")) if rnd.random() < 0.5 else s


class ShapedIndex:
    """One database: .fmi + nodes.dmp, its header, the proteins, and reads back-translated from them (2 % mutations, half reverse-complemented).
    reads: random windows of proteins other than the one that holds the suffix of the guard row; guard_reads: windows that start at that suffix
    or up to 2^E - 1 residues to its right, so that their matches walk into the guard row (guard class only)."""

    def __init__(self, d, name, spec, seed, nreads):
        e, nseq, bres, (lo, hi), big = spec
        self.name, self.exp = name, e
        rnd = random.Random(seed); m = 1 << e
        lens = [rnd.randrange(lo, hi) for _ in range(nseq)]
        if big:
            lens[0] = big
        lens[-1] += (bres - sum(x + 1 for x in lens)) % m        # pad one protein to the wanted bwtlen residue
        self.prots = ["".join(rnd.choices(AA, k=x)) for x in lens]
        faa = os.path.join(d, name + ".faa"); self.nodes = os.path.join(d, "nodes.dmp")
        with open(faa, "w") as f:
            for i, p in enumerate(self.prots):
                f.write(">WP_%09d.1_%d\n%s\n" % (i, 100 + i % NTAX, p))
        if not os.path.exists(self.nodes):
            with open(self.nodes, "w") as f:
                f.write("1\t|\t1\t|\tno rank\t|\n" + "".join("%d\t|\t1\t|\tspecies\t|\n" % t for t in range(100, 100 + NTAX)))
        self.fmi = _build_exp0(faa, os.path.join(d, name)) if e == 0 else build_fmi(faa, os.path.join(d, name), threads=16, exponent=e)
        self.faa = faa
        self.h = fmi_header(self.fmi)
        n, s = self.h["bwtlen"], self.h["nseq"]
        self.guard = e > 0 and s % m == 0 and n % m != 0
        self.last_row = ((n - 1) >> e) << e
        self.written = ((n - 1) >> e) + 1 - (((s - 1) >> e) + 1)      # samples kaiju-mkbwt writes
        self.guard_seq, self.guard_pos, self.guard_reads = None, None, []
        if self.guard:
            L = oracle_lib(); idx = L.ko_index_load(self.fmi.encode())
            iseq, self.guard_pos = true_suffix(L, idx, self.h["alen"], self.last_row)
            L.ko_index_free(idx)
            self.guard_seq = int(fmi_seq_names(self.fmi)[iseq][3:12])
            p = self.prots[self.guard_seq]
            for j in sorted({0, 1, 2, m // 2, m - 1}):
                st = self.guard_pos + j
                if len(p) - st >= 12:
                    self.guard_reads.append(_dna(p[st:st + 40], rnd, 0.0))
        cand = [i for i, p in enumerate(self.prots) if len(p) >= 40 and i != self.guard_seq]
        self.reads = []
        for _ in range(nreads):
            p = self.prots[rnd.choice(cand)]; st = rnd.randrange(0, len(p) - 33)
            self.reads.append(_dna(p[st:st + 34], rnd))
        self.long_reads = []
        for _ in range(4):                                        # 2-10 kb: runs of ~40-residue windows of random proteins
            parts = []
            while sum(map(len, parts)) < rnd.randrange(2000, 10000):
                p = self.prots[rnd.choice(cand)]; st = rnd.randrange(0, len(p) - 33); parts.append(_dna(p[st:st + 40], rnd))
            self.long_reads.append("".join(parts))

    def residues(self):
        m = 1 << self.exp
        return self.h["nseq"] % m, self.h["bwtlen"] % m


def build_family(d, names, nreads=2000, wide_reads=1000):
    """{name: ShapedIndex} for the given names of SMALL and WIDE; asserts that every database has the shape it was planned for."""
    out = {}
    for name in names:
        spec = SMALL.get(name) or WIDE[name]
        for seed in range(zlib.crc32(name.encode()), zlib.crc32(name.encode()) + 8):     # until the guard row's suffix has 12 residues to read
            x = ShapedIndex(d, name, spec, seed, wide_reads if name in WIDE else nreads)
            if not x.guard or x.guard_reads:
                break
        e, nseq, bres = spec[:3]
        assert x.h["exp"] == e and x.h["nseq"] == nseq and x.residues() == (nseq % (1 << e), bres), (name, x.h)
        assert x.h["ncheck"] == (x.h["bwtlen"] >> e) - (nseq >> e), (name, x.h)
        if name in WIDE:
            assert x.h["nbytes"] == {"w5": 5, "w6": 6}[name], (name, x.h)
        if x.guard:
            assert x.written == x.h["ncheck"] + 1 and x.guard_reads, (name, x.h, x.guard_pos, len(x.prots[x.guard_seq]))
        out[name] = x
    planned = {(e, r, b != 0) for e in (2, 5) for r in (0, 1, (1 << e) - 1) for b in (0, 1)}
    got = {(x.exp, x.residues()[0], x.residues()[1] != 0) for x in out.values() if x.exp in (2, 5) and x.name in SMALL}
    if set(SMALL) <= set(names):
        assert planned <= got, planned - got
        assert {x.exp for x in out.values()} >= {0, 1, 2, 4, 5, 7}
    return out


def pack(reads):
    seq = np.frombuffer("".join(reads).encode(), dtype=np.uint8).copy()
    off = np.zeros(len(reads) + 1, np.uint64); off[1:] = np.cumsum([len(r) for r in reads])
    return seq, off


def pairs(reads):
    """PE-style pairs from a read list: mate 2 = the next read's reverse complement"""
    rc = [r[::-1].translate(str.maketrans("ACGT", "TGCA")) for r in reads[1:] + reads[:1]]
    return pack(reads) + pack(rc)


def write_fasta(path, reads):
    with open(path, "w") as f:
        for i, r in enumerate(reads):
            f.write(">r%d\n%s\n" % (i, r))
