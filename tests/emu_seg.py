"""The product's SEG filter on the CPU warp emulator (tests/emu/kj_emu_seg.cpp), compiled on first use into a directory of the caller's choosing;
the reference's SeqBufferSeg (oracle/_ref/libkaijuref.so) called the way the reference classifier sets it up; and the seeded sequence families
chosen for SEG's edges, which the emulated and the GPU tests share."""
import ctypes as C
import os
import random
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libkaijuref.so")
AA = "ACDEFGHIKLMNPQRSTVWY"
CODE = np.zeros(256, np.uint8)
CODE[np.frombuffer(AA.encode(), np.uint8)] = np.arange(1, 21, dtype=np.uint8)
COVERAGE = ("trim_minlen_1", "trim_minlen_n2_minus_50", "trim_long", "stirling", "level1_region", "merge", "raw_regions")


def load(out_dir):
    """ctypes handle of the emulated SEG, built into out_dir."""
    so = os.path.join(out_dir, "libkjemu_seg.so")
    if not os.path.exists(so):
        os.makedirs(out_dir, exist_ok=True)
        tmp = so + ".%d" % os.getpid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DKJ_EMU", "-o", tmp, os.path.join(HERE, "emu", "kj_emu_seg.cpp"), "-lz", "-lpthread"])
        os.replace(tmp, so)
    E = C.CDLL(so)
    E.kjemu_seg.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_uint32), C.c_void_p]
    E.kjemu_seg_cap.argtypes = [C.c_uint32, C.POINTER(C.c_uint32)]
    return E


def max_len_for(n):
    """The smallest batch profile (longest mate in bases) whose fragments hold n residues, but never below the PE150 profile."""
    return max(152, 3 * n)


def emu_seg(E, s, max_len, is_long, compact):
    """([(begin, end), ...], error flags, coverage counts) of kj_seg on the residue string s."""
    res = np.ascontiguousarray(CODE[np.frombuffer(s.encode(), np.uint8)])
    cap = len(s) // 4 + 16
    out = np.zeros(2 * cap, np.int32); cov = np.zeros(len(COVERAGE), np.uint64); err = C.c_uint32()
    ns = E.kjemu_seg(res.ctypes.data, len(s), max_len, int(is_long), int(compact), out.ctypes.data, cap, C.byref(err), cov.ctypes.data)
    if ns < 0:
        raise ValueError("fragment of %d residues does not fit the work space of max_len %d" % (len(s), max_len))
    return [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(ns)], int(err.value), [int(x) for x in cov]


def seg_cap(E, max_len):
    """(region capacity, longest fragment) of the work space for max_len"""
    mf = C.c_uint32(); cap = E.kjemu_seg_cap(max_len, C.byref(mf)); return cap, int(mf.value)


class RefSeg:
    """SeqBufferSeg with SegParametersNewAa and overlaps = 1 (the reference's Config.cpp), residues converted with AMINOACID_TO_NCBISTDAA."""

    def __init__(self, path=REF_SO):
        class SSeqRange(C.Structure):
            _fields_ = [("left", C.c_int), ("right", C.c_int)]

        class BlastSeqLoc(C.Structure):
            pass
        BlastSeqLoc._fields_ = [("next", C.POINTER(BlastSeqLoc)), ("ssr", C.POINTER(SSeqRange))]

        class SegParameters(C.Structure):   # blast_seg.h
            _fields_ = [("window", C.c_int), ("locut", C.c_double), ("hicut", C.c_double), ("period", C.c_int), ("hilenmin", C.c_int),
                        ("overlaps", C.c_ubyte), ("maxtrim", C.c_int), ("maxbogus", C.c_int)]
        R = self.R = C.CDLL(path)
        R.SegParametersNewAa.restype = C.c_void_p
        R.SeqBufferSeg.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.POINTER(BlastSeqLoc))]
        R.BlastSeqLocFree.restype = C.c_void_p; R.BlastSeqLocFree.argtypes = [C.POINTER(BlastSeqLoc)]
        self.sp = R.SegParametersNewAa()
        SegParameters.from_address(self.sp).overlaps = 1
        tab = (C.c_ubyte * 128).in_dll(R, "AMINOACID_TO_NCBISTDAA")
        self.tab = bytes(tab[i] for i in range(128)); self.Loc = BlastSeqLoc

    def __call__(self, s):
        """merged regions [(begin, end), ...] in the order of the returned list: ascending (s_SegToSeqLoc undoes s_SegSeq's prepending)"""
        conv = s.encode().translate(self.tab.ljust(256, b"\0")); locs = C.POINTER(self.Loc)()
        self.R.SeqBufferSeg(conv, len(s), 0, self.sp, C.byref(locs))
        out = []; p = locs
        while p:
            out.append((p.contents.ssr.contents.left, p.contents.ssr.contents.right)); p = p.contents.next
        if locs:
            self.R.BlastSeqLocFree(locs)
        return out


# ---------------------------------------------------------------------------------------------------------------------------------------------
# seeded sequence families
# ---------------------------------------------------------------------------------------------------------------------------------------------
def _rand(rnd, n, letters=AA):
    return "".join(rnd.choice(letters) for _ in range(n))


def _flanked(rnd, block, lo=0, hi=40):
    return _rand(rnd, rnd.randint(lo, hi)) + block + _rand(rnd, rnd.randint(lo, hi))


def _unit(rnd, k):
    return "".join(rnd.sample(AA, k)) if rnd.random() < 0.5 else _rand(rnd, k)


def block_of(rnd, kind, n):
    """A low-complexity block of n residues: homopolymer, period-2..4 repeat, 2-6 letter mixture, or a tie maker."""
    if kind == "homo":
        return rnd.choice(AA) * n
    if kind.startswith("period"):
        u = "".join(rnd.sample(AA, int(kind[6:])))
        return (u * (n // len(u) + 1))[:n]
    if kind == "mix":
        return _rand(rnd, n, rnd.sample(AA, rnd.randint(2, 6)))
    if kind == "palindrome":
        h = _rand(rnd, (n + 1) // 2, rnd.sample(AA, rnd.randint(2, 4)))
        return (h + h[::-1])[:n]
    if kind == "perm":                      # consecutive permutations of one multiset: windows of equal composition at many starts
        ms = list(_rand(rnd, rnd.randint(3, 8), rnd.sample(AA, rnd.randint(2, 4)))); out = ""
        while len(out) < n:
            rnd.shuffle(ms); out += "".join(ms)
        return out[:n]
    raise ValueError(kind)


KINDS = ("homo", "period2", "period3", "period4", "mix", "palindrome", "perm")


def families(seed=1, scale=1):
    """(family, sequence) pairs.  scale multiplies the counts of the cheap families."""
    rnd = random.Random(seed); out = []
    for _ in range(600 * scale):
        out.append(("uniform", _rand(rnd, rnd.randint(1, 400))))
    for p in range(1, 5):                                   # homopolymers and period-2..4 repeats of every run length 1-200 in random flanks
        for r in range(1, 201):
            for _ in range(scale):
                out.append(("period%d_run" % p, _flanked(rnd, block_of(rnd, "homo" if p == 1 else "period%d" % p, r))))
    for _ in range(1500 * scale):                           # 2-6 letter mixtures, bare and flanked
        n = rnd.choice([rnd.randint(12, 60), rnd.randint(40, 140), rnd.randint(100, 400)])
        b = block_of(rnd, "mix", n)
        out.append(("mixture", b if rnd.random() < 0.3 else _flanked(rnd, b)))
    for _ in range(700 * scale):                            # tie makers
        kind = rnd.choice(("palindrome", "perm", "period2"))
        out.append(("tie_" + kind, _flanked(rnd, block_of(rnd, kind, rnd.randint(8, 160)))))
    for _ in range(300 * scale):
        # b a^k b inside 15-40 residues of a 3-5 letter mixture: the hicut extent reaches into the mixtures, so the trim's shortest window
        # (n2 - 49) can be one longer than a^k, and then "b a^k" and "a^k b" tie at the same length, at two starts
        a, b = rnd.sample("AHIKLMNPQRSTVWY", 2); fl = "CDEFG"[:rnd.randint(3, 5)]
        k = rnd.choice([rnd.randint(30, 80), rnd.randint(100, 300)])
        out.append(("tie_minlen", _flanked(rnd, _rand(rnd, rnd.randint(15, 40), fl) + b + a * k + b + _rand(rnd, rnd.randint(15, 40), fl), 0, 20)))
    for _ in range(900 * scale):                            # two blocks 1-30 residues apart: merges and the left-trim recursion
        a = block_of(rnd, rnd.choice(KINDS), rnd.randint(6, 80)); b = block_of(rnd, rnd.choice(KINDS), rnd.randint(6, 80))
        out.append(("two_blocks", _flanked(rnd, a + _rand(rnd, rnd.randint(1, 30)) + b)))
    for n in (11, 12, 13, 51, 52, 127, 128, 129):           # block lengths around the trim's branch points
        for d in range(-3, 4):
            for kind in KINDS:
                for _ in range(2 * scale):
                    out.append(("edge_%d" % n, _flanked(rnd, block_of(rnd, kind, n + d), 0, 12)))
    return out


def nested(seed=3, count=800):
    """A weak low-complexity block, a short gap, then a strong homopolymer: the trim keeps the strong block, so the trigger window lies in
    the left trim and s_SegSeq recurses into it (the level-1 region)."""
    rnd = random.Random(seed); out = []
    for _ in range(count):
        a = block_of(rnd, rnd.choice(("homo", "period2", "mix")), rnd.randint(8, 25))
        gap = _rand(rnd, rnd.randint(0, 10), "".join(sorted(set(a))))
        out.append(("nested", _flanked(rnd, a + gap + block_of(rnd, "homo", rnd.randint(20, 200)), 0, 20)))
    return out


def stirling_tie(seed=4, count=4):
    """Windows of 9,999 and 10,000 residues whose probabilities are equal in exact arithmetic: a two-letter block of 9,999 residues with 499
    of letter b (none within 40 of its ends), followed by one more b.  s_Trim's choice between them rests on ln(10000!) being the table's
    entry rather than Stirling's value (the table holds n <= 10,000); the reference keeps the shorter window."""
    rnd = random.Random(seed); out = []
    for k in range(count):
        a, b = rnd.sample(AA, 2); foreign = [x for x in AA if x not in (a, b)]
        core = [a] * 9999
        for p in rnd.sample(range(40, 9999 - 40), 499):
            core[p] = b
        block = "".join(core) + b
        if k % 2:
            block = block[::-1]                           # the extra b on the left
        out.append(("stirling_tie", _rand(rnd, rnd.randint(0, 30), foreign) + block + _rand(rnd, rnd.randint(0, 30), foreign)))
    return out


def big_families(seed=2, long_only=False):
    """Regions of 5,461, 9,999-10,002 and 20,000 residues (and, for the long instances, 65,535, 65,536 and 70,000)."""
    rnd = random.Random(seed); out = []
    lens = [65535, 65536, 70000] if long_only else [5461, 9999, 10000, 10001, 10002, 20000]
    for n in lens:
        for kind in (("homo", "period2", "mix") if not long_only else ("homo", "mix")):
            out.append(("big_%d_%s" % (n, kind), _flanked(rnd, block_of(rnd, kind, n), 0, 30)))
    return out


def dense_search(E, n, seed, rounds, max_len=None, is_long=False):
    """Hill-climb on the raw region count the emulator reports for fragments of n residues: single-residue mutations of the best sequence so
    far, started from short repeats separated by single residues.  Returns (raw count, sequence)."""
    rnd = random.Random(seed); ml = max_len or max_len_for(n)
    best_s = None; best = -1
    for start in range(8):
        u = rnd.choice(AA) * rnd.randint(2, 5)
        s = ""
        while len(s) < n:
            s += u + rnd.choice(AA) if start % 2 else rnd.choice(AA) * rnd.randint(3, 7) + _rand(rnd, rnd.randint(1, 3))
        s = s[:n]; c = emu_seg(E, s, ml, is_long, False)[2][-1]
        if c > best:
            best, best_s = c, s
    for _ in range(rounds):
        t = list(best_s)
        for _ in range(rnd.randint(1, 3)):
            i = rnd.randrange(n); t[i] = rnd.choice(AA) if rnd.random() < 0.3 else t[rnd.randrange(n)]
        t = "".join(t); c = emu_seg(E, t, ml, is_long, False)[2][-1]
        if c >= best:
            best, best_s = c, t
    return best, best_s
