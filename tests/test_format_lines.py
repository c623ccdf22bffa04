"""The per-read output line of kj_classify_files (kaiju_b200/csrc/kj_format.h, the code kj_fmt_len / kj_fmt_write run) on the CPU, against a
restatement of the reference's ostream formatting: kaiju (ConsumerThread.cpp:527-536, 614-623, 724-739), kaijux / kaijup
(ConsumerThreadx.cpp:108-113, 182-187, 202-256; ConsumerThreadp.cpp:16-20, 66-94).  No GPU needed."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MAX_IDS, MAX_ACC = 21, 20
KAIJU, KAIJU_IDS, KAIJU_V, NAMES, NAMES_V = range(5)


class FmtIn(C.Structure):      # struct KjFmtIn
    _fields_ = [("fmt", C.c_int), ("tax", C.c_void_p), ("best", C.c_void_p), ("ids", C.c_void_p), ("nids", C.c_void_p), ("acc", C.c_void_p), ("nacc", C.c_void_p),
                ("frag", C.c_void_p), ("frag_stride", C.c_uint64), ("fraglen", C.c_void_p), ("gate", C.c_void_p), ("names", C.c_void_p), ("name_off", C.c_void_p),
                ("acc_str", C.c_void_p), ("acc_off", C.c_void_p), ("n_acc", C.c_uint64), ("lab_str", C.c_void_p), ("lab_off", C.c_void_p), ("n_lab", C.c_uint64),
                ("tax_id", C.c_void_p), ("n_present", C.c_uint32), ("n_tax", C.c_uint32)]


@pytest.fixture(scope="module")
def fmt_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("fmt") / "libkjfmt.so")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emu", "kj_emu_format.cpp")])
    L = C.CDLL(so)
    L.kjfmt_lines.restype = C.c_uint64; L.kjfmt_lines.argtypes = [C.POINTER(FmtIn), C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p]
    L.kjfmt_status.argtypes = [C.POINTER(FmtIn), C.c_uint64]
    L.kjfmt_self_score.restype = C.c_uint32; L.kjfmt_self_score.argtypes = [C.c_uint32]
    return L


def strtab(strings):
    off = np.zeros(len(strings) + 1, dtype=np.uint64); off[1:] = np.cumsum([len(s) for s in strings]) if strings else []
    return np.frombuffer(b"".join(strings) + b"\0", dtype=np.uint8), off


class Batch:
    """Per-read records -> the arrays kj_classify_files hands to the format pass (keeps them alive)."""

    def __init__(self, fmt, reads, accs=(), labels=(), tax_id=(), n_present=None):
        n = len(reads); self.keep = []
        stride = max([len(r.get("frag", b"")) for r in reads] + [16])
        tax = np.array([r["tax"] for r in reads], dtype=np.uint64); best = np.array([r.get("best", 0) for r in reads], dtype=np.uint32)
        ids = np.zeros((n, MAX_IDS), dtype=np.uint64); nids = np.zeros(n, dtype=np.uint8)
        acc = np.zeros((n, MAX_ACC), dtype=np.uint32); nacc = np.zeros(n, dtype=np.uint8)
        frag = np.zeros((n, stride), dtype=np.uint8); fraglen = np.zeros(n, dtype=np.uint32); gate = np.zeros(n, dtype=np.uint8)
        for i, r in enumerate(reads):
            ids[i, :len(r.get("ids", []))] = r.get("ids", []); nids[i] = len(r.get("ids", []))
            acc[i, :len(r.get("acc", []))] = r.get("acc", []); nacc[i] = len(r.get("acc", []))
            f = r.get("frag", b""); frag[i, :len(f)] = np.frombuffer(f, dtype=np.uint8) if f else []; fraglen[i] = len(f)
            gate[i] = r.get("gate", 0)
        names, name_off = strtab([r["name"] for r in reads]); name_off = name_off.astype(np.uint32)
        a_str, a_off = strtab(list(accs)); l_str, l_off = strtab(list(labels)); tid = np.array(list(tax_id) + [0], dtype=np.uint64)
        self.keep = [tax, best, ids, nids, acc, nacc, frag, fraglen, gate, names, name_off, a_str, a_off, l_str, l_off, tid]
        p = lambda a: a.ctypes.data
        self.s = FmtIn(fmt, p(tax), p(best), p(ids), p(nids), p(acc), p(nacc), p(frag), stride, p(fraglen), p(gate), p(names), p(name_off),
                       p(a_str), p(a_off), len(accs), p(l_str), p(l_off), len(labels), p(tid), len(tax_id) if n_present is None else n_present, len(tax_id))
        self.n = n


def run(L, batch):
    out = {}
    for nl in (1, 32):
        buf = np.zeros(1 << 20, dtype=np.uint8); lens = np.zeros(batch.n, dtype=np.uint32)
        k = L.kjfmt_lines(C.byref(batch.s), batch.n, nl, buf.ctypes.data, lens.ctypes.data)
        out[nl] = bytes(buf[:k])
        assert int(lens.sum()) == k
    assert out[1] == out[32]
    return out[1]


# ---- the reference's formatting, restated --------------------------------------------------------------------------------------------------
def ref_kaiju(fmt, r, accs):
    """ConsumerThread::doWork: "C\\t" << name << "\\t" << taxid [<< "\\t" << extraoutput] << "\\n", else "U\\t" << name << "\\t0\\n"."""
    if not r["tax"]:
        return b"U\t" + r["name"] + b"\t0\n"
    line = b"C\t" + r["name"] + b"\t" + str(r["tax"]).encode()
    if fmt >= KAIJU_IDS:
        line += b"\t" + str(r.get("best", 0)).encode() + b"\t" + b"".join(str(i).encode() + b"," for i in r.get("ids", []))
    if fmt == KAIJU_V:
        line += b"\t" + b"".join(accs[a] + b"," for a in r.get("acc", [])) + b"\t" + r.get("frag", b"")
    return line + b"\n"


def ref_names(fmt, r, label_of):
    """ConsumerThreadx/p::doWork: gate -> "U\\t<name>\\t0\\n"; extraoutput = best << "\\t" << names each "," << "\\t" [<< fragments each ","]."""
    if r.get("gate"):
        return b"U\t" + r["name"] + b"\t0\n"
    if not r["tax"] or not r.get("ids"):
        return b"U\t" + r["name"] + b"\n"
    return b"C\t" + r["name"] + b"\t" + str(r.get("best", 0)).encode() + b"\t" + b"".join(label_of(i) + b"," for i in r["ids"]) + b"\t" + \
        (r.get("frag", b"") if fmt == NAMES_V else b"") + b"\n"


def frag_list(rng, k, lo=11, hi=60):
    return b"".join(bytes(rng.choice(b"ACDEFGHIKLMNPQRSTVWY") for _ in range(rng.randint(lo, hi))) + b"," for _ in range(k))


def kaiju_reads(rng, n_acc):
    reads = [
        {"name": b"r0", "tax": 0},                                                                  # unclassified
        {"name": b"r1", "tax": 9606, "best": 42},                                                   # empty id / accession / fragment sets
        {"name": b"", "tax": 1, "best": 0, "ids": [1]},                                             # empty name
        {"name": b"r3", "tax": 2**64 - 1, "best": 2**32 - 1, "ids": list(range(10**12, 10**12 + 21)), "acc": list(range(20)), "frag": frag_list(rng, 40)},
        {"name": b"r4", "tax": 10, "best": 7, "ids": [3, 10, 99999], "acc": [n_acc - 1], "frag": frag_list(rng, 200, 30, 120)},
    ]
    for i in range(200):
        nid = rng.randint(0, 21); na = rng.randint(0, 20)
        reads.append({"name": b"read_%d" % i, "tax": rng.choice([0, rng.randint(1, 3 * 10**6)]), "best": rng.randint(0, 5000),
                      "ids": sorted(rng.sample(range(1, 10**7), nid)), "acc": sorted(rng.sample(range(n_acc), na)), "frag": frag_list(rng, rng.randint(0, 30))})
    return reads


@pytest.mark.parametrize("fmt", [KAIJU, KAIJU_IDS, KAIJU_V])
def test_kaiju_lines_equal_reference_formatting(fmt_lib, fmt):
    rng = random.Random(fmt)
    accs = [b"ACC%06d.%d" % (i, i % 3) for i in range(50)]
    reads = kaiju_reads(rng, len(accs))
    got = run(fmt_lib, Batch(fmt, reads, accs=accs))
    assert got == b"".join(ref_kaiju(fmt, r, accs) for r in reads)


@pytest.mark.parametrize("fmt", [NAMES, NAMES_V])
def test_name_lines_equal_reference_formatting(fmt_lib, fmt):
    """Labels by dense taxon index (two ascending runs of taxon ids, as the context keeps them), names with tabs, spaces and '/' (kaijup keeps
    them whole), both kinds of unclassified line, 21 labels, long fragment lists."""
    rng = random.Random(10 + fmt)
    tax_id = [1] + list(range(2, 400)) + [1000, 1001]            # nodes.dmp ids, then ids missing from it (n_present = 399)
    labels = [b""] + [b"seq_%d desc\twith tab" % i for i in range(398)] + [b"extra_a", b"extra_b/x"]
    dense = {t: k for k, t in enumerate(tax_id)}
    reads = [{"name": b"gated\tname /1", "tax": 0, "gate": 1}, {"name": b"gated but classified", "tax": 5, "ids": [5], "gate": 1},
             {"name": b"nomatch", "tax": 0}, {"name": b"tax but no ids", "tax": 7},
             {"name": b"max", "tax": 1, "best": 999, "ids": sorted(rng.sample(range(2, 400), 21)), "frag": frag_list(rng, 300)},
             {"name": b"missing", "tax": 1, "best": 3, "ids": [2, 1000, 1001, 5000]}]          # 5000: no such taxon -> empty label
    for i in range(300):
        k = rng.randint(0, 21)
        reads.append({"name": b"q%d extra\twords" % i, "tax": rng.choice([0, 1]), "best": rng.randint(11, 2000), "gate": int(rng.random() < 0.2),
                      "ids": sorted(rng.sample(tax_id, k)), "frag": frag_list(rng, rng.randint(0, 25))})
    got = run(fmt_lib, Batch(fmt, reads, labels=labels, tax_id=tax_id, n_present=399))
    label_of = lambda i: labels[dense[i]] if i in dense else b""
    assert got == b"".join(ref_names(fmt, r, label_of) for r in reads)
    for i, r in enumerate(reads[:4]):
        assert fmt_lib.kjfmt_status(C.byref(Batch(fmt, reads, labels=labels, tax_id=tax_id, n_present=399).s), i) == [0, 0, 1, 1][i]


def test_self_scores_are_blosum62_diagonal(fmt_lib):
    diag = dict(zip("ARNDCQEGHILKMFPSTWYV", [4, 5, 6, 6, 9, 5, 5, 6, 8, 4, 4, 5, 5, 6, 7, 4, 5, 11, 7, 4]))
    for c in range(256):
        assert fmt_lib.kjfmt_self_score(c) == diag.get(chr(c), 0)
