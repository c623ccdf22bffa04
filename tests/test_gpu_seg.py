"""SEG's region edges as the product's output shows them, against the reference binary.  A database of proteins with low-complexity blocks planted
between random stretches (homopolymers, period-2..4 repeats, 2-6 letter mixtures, tie makers, region-dense sequences; blocks of 12 to 10,500
residues) is built in the test; reads cover a block with flanks of varied length, as protein (-p) and as back-translated DNA, including one protein
read above 5,461 residues and one DNA read above 16,383 bases (the long kernels' kj_seg<true>).  In MEM the pieces between SEG regions match in
full, so column 7 of `-v` (the matched fragment strings) starts or ends at a region edge.  Checked: the CLI's `-v` output (file pipeline) and
kj_classify_verbose2 equal `kaiju -v` byte for byte, in MEM, Greedy -e 3 -s 65 and Greedy -e 0; the short reads' results equal the emulated
kernels'; turning SEG off changes a stated share of reads; a stated number of reads show a SeqBufferSeg region edge in column 7."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_seg as es
from conftest import ROOT
from helpers import REF_DIR, SynthDB, build_fmi, have_ref

pytestmark = pytest.mark.gpu
CODON = {'A': 'GCT', 'R': 'CGT', 'N': 'AAT', 'D': 'GAT', 'C': 'TGT', 'Q': 'CAA', 'E': 'GAA', 'G': 'GGT', 'H': 'CAT', 'I': 'ATT',
         'L': 'CTG', 'K': 'AAA', 'M': 'ATG', 'F': 'TTT', 'P': 'CCT', 'S': 'TCT', 'T': 'ACT', 'W': 'TGG', 'Y': 'TAT', 'V': 'GTT'}
CONFIGS = {"mem": ["-a", "mem"], "greedy_e3_s65": ["-a", "greedy", "-e", "3", "-s", "65"], "greedy_e0": ["-a", "greedy", "-e", "0", "-s", "65"]}
LIMIT = 40000                  # -L / max_read_len of the runs: admits the long protein read (a third of it in residues) and the long DNA read
# What this workload shows in the reference's own output (2,990 reads): -X changes every read's line in all three configurations, and a
# column-7 fragment starts or ends at a SeqBufferSeg region edge in 2,011 reads (MEM) and 1,775 reads (both Greedy configurations).
MIN_SEG_SHARE = 0.9            # share of reads whose line changes with -X
MIN_EDGE_READS = 1500          # reads (protein + DNA) with a column-7 fragment that starts or ends at a region edge


def make_workload(d, dense_blocks, seed=5, nprot=2000):
    """Write d/db.faa, d/nodes.dmp and the read files; returns {"prot": [(name, residues)], "dna": [(name, bases, residues of frame 0)]}."""
    rnd = random.Random(seed)
    SynthDB(nprot, seed).write(d + "/base.faa", d + "/nodes.dmp")
    recs = []; cur = None
    for line in open(d + "/base.faa").read().split("\n"):
        if line.startswith(">"):
            cur = [line, ""]; recs.append(cur)
        elif cur is not None:
            cur[1] += line.strip()
    lens = [rnd.randint(12, 60) for _ in range(6)] + [50, 51, 52, 53, 126, 127, 128, 129, 130] + [rnd.randint(131, 400)]
    prots = []; blocks = []
    for i, (h, p) in enumerate(recs):
        if i == 0:
            b = es.block_of(rnd, "mix", 10500)                   # one region above 10,000 residues: Stirling's ln(n!)
        elif i == 1:
            b = es.block_of(rnd, "period2", 6000)                # the long DNA read's block
        elif i < 2 + len(dense_blocks):
            b = dense_blocks[i - 2]
        else:
            b = es.block_of(rnd, rnd.choice(es.KINDS), rnd.choice(lens))
        a = rnd.randint(0, len(p)); q = p[:a] + b + p[a:]
        prots.append(q); blocks.append((a, a + len(b)))
        recs[i][1] = q
    with open(d + "/db.faa", "w") as f:
        for h, s in recs:
            f.write(h + "\n" + s + "\n")
    prot_reads = []; dna_reads = []
    for i, (q, (a, e)) in enumerate(zip(prots, blocks)):
        if i >= 2 and rnd.random() < 0.25:
            continue
        lo = max(0, a - rnd.choice([0, 1, 2, 5, 11, 12, 20, 40, 60])); hi = min(len(q), e + rnd.choice([0, 1, 2, 5, 11, 12, 20, 40, 60]))
        r = q[lo:hi]
        if i != 1:
            prot_reads.append(("p%d" % i, r))
        if i != 0:
            dna_reads.append(("d%d" % i, "".join(CODON[c] for c in r), r))
    for nm, rr in (("prot", [(n, s) for n, s in prot_reads]), ("dna", [(n, s) for n, s, _ in dna_reads])):
        with open("%s/%s.fq" % (d, nm), "w") as f:
            for n, s in rr:
                f.write("@%s\n%s\n+\n%s\n" % (n, s, "I" * len(s)))
    build_fmi(d + "/db.faa", d + "/db", threads=8)
    return {"prot": prot_reads, "dna": [(n, s, r) for n, s, r in dna_reads]}


def run_cli(binary, d, kind, cfg, seg, extra=()):
    cmd = [binary, "-t", d + "/nodes.dmp", "-f", d + "/db.fmi", "-i", "%s/%s.fq" % (d, kind), "-v", "-z", "8"] + CONFIGS[cfg] + list(extra)
    if kind == "prot":
        cmd += ["-p"]
    if not seg:
        cmd += ["-X"]
    txt = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout.decode()
    return {l.split("\t")[1]: l for l in txt.splitlines()}


def edge_reads(lines, residues, ref):
    """Names of classified reads with a column-7 fragment that starts right after or ends right before a SeqBufferSeg region of the read's
    protein sequence (the read itself for -p, frame 0 of the back-translation for DNA reads)."""
    out = set()
    for name, line in lines.items():
        p = line.split("\t")
        if p[0] != "C" or len(p) < 7 or name not in residues:
            continue
        s = residues[name]; regs = ref(s)
        starts = {e + 1 for _, e in regs}; ends = {b - 1 for b, _ in regs}
        for frag in p[6].split(","):
            if len(frag) < 11:
                continue
            at = s.find(frag)
            while at >= 0:
                if at in starts or at + len(frag) - 1 in ends:
                    out.add(name); break
                at = s.find(frag, at + 1)
    return out


@pytest.fixture(scope="module")
def work(built, tmp_path_factory):
    if not have_ref():
        pytest.skip("oracle/_ref (reference binary and index builder) not available")
    E = es.load(str(tmp_path_factory.mktemp("emu_seg")))
    dense = [es.dense_search(E, 200, 10 + k, 300)[1] for k in range(6)]
    d = str(tmp_path_factory.mktemp("segdb"))
    return d, make_workload(d, dense)


def verbose2_lines(kb, clf, fmi, names, reads):
    """kj_classify_verbose2 of single-end reads as `kaiju -v` lines (accession names through kj_fmi_accession)."""
    L = kb.lib()
    L.kj_classify_verbose2.argtypes = [C.c_void_p] * 5 + [C.c_uint64] + [C.c_void_p] * 6 + [C.c_void_p, C.c_uint32, C.c_void_p]
    L.kj_fmi_accession.restype = C.c_char_p; L.kj_fmi_accession.argtypes = [C.c_void_p, C.c_uint32]
    s = np.frombuffer("".join(reads).encode(), np.uint8).copy(); o = np.zeros(len(reads) + 1, np.uint64); o[1:] = np.cumsum([len(r) for r in reads])
    n = len(reads); ST = 1 << 16
    tax = np.zeros(n, np.uint64); best = np.zeros(n, np.uint32); ids = np.zeros((n, 21), np.uint64); nids = np.zeros(n, np.uint8)
    acc = np.zeros((n, 20), np.uint32); nacc = np.zeros(n, np.uint8); frag = np.zeros((n, ST), np.uint8); flen = np.zeros(n, np.uint32)
    kb._check(L.kj_classify_verbose2(clf._ctx, s.ctypes.data, o.ctypes.data, None, None, n, tax.ctypes.data, best.ctypes.data, ids.ctypes.data,
                                     nids.ctypes.data, acc.ctypes.data, nacc.ctypes.data, frag.ctypes.data, ST, flen.ctypes.data))
    f = C.c_void_p(); assert L.kj_fmi_load(fmi.encode(), C.byref(f)) == 0
    lines = {}
    for i, name in enumerate(names):
        lines[name] = "U\t%s\t0" % name if not tax[i] else "C\t%s\t%d\t%d\t%s,\t%s\t%s" % (
            name, tax[i], best[i], ",".join(str(int(x)) for x in ids[i, :nids[i]]),
            "".join(L.kj_fmi_accession(f, int(a)).decode() + "," for a in acc[i, :nacc[i]]), bytes(frag[i, :flen[i]]).decode())
    L.kj_fmi_free(f)
    return lines


def emu_lines(kb, d, cfg_params, names, reads, max_len):
    """Taxon and best of the emulated short-read kernels (tests/emu/libkjemu.so) for the reads of at most max_len characters."""
    E = C.CDLL(os.path.join(ROOT, "tests", "emu", "libkjemu.so"))
    E.kjemu_create.restype = C.c_void_p; E.kjemu_create.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p]; E.kjemu_destroy.argtypes = [C.c_void_p]
    E.kjemu_classify.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64, C.c_void_p, C.c_void_p, C.c_int]
    keep = [i for i, r in enumerate(reads) if len(r) <= max_len]
    rr = [reads[i] for i in keep]
    s = np.frombuffer("".join(rr).encode(), np.uint8).copy(); o = np.zeros(len(rr) + 1, np.uint64); o[1:] = np.cumsum([len(r) for r in rr])
    h = E.kjemu_create((d + "/db.fmi").encode(), (d + "/nodes.dmp").encode(), C.byref(cfg_params)); assert h
    tax = np.zeros(len(rr), np.uint64); best = np.zeros(len(rr), np.uint32)
    rc = E.kjemu_classify(h, s.ctypes.data, o.ctypes.data, None, None, len(rr), tax.ctypes.data, best.ctypes.data, os.cpu_count() or 4)
    E.kjemu_destroy(h); assert rc == 0
    return {names[i]: (int(tax[k]), int(best[k])) for k, i in enumerate(keep)}


def _params(kb, cfg, protein):
    if cfg == "mem":
        return kb.make_params("mem", protein=protein)
    return kb.make_params("greedy", e=3 if cfg == "greedy_e3_s65" else 0, s=65, protein=protein)


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_seg_edges_match_reference(built, work, cfg):
    import kaiju_b200 as kb
    d, W = work
    cli = os.path.join(ROOT, "kaiju_b200", "kaiju-b200"); ref_bin = os.path.join(REF_DIR, "kaiju"); ref = es.RefSeg()
    residues = {n: r for n, r in W["prot"]}; residues.update({n: r for n, _, r in W["dna"]})
    assert max(len(r) for _, r in W["prot"]) > 5461 and max(len(s) for _, s, _ in W["dna"]) > 16383
    edges = set(); changed = total = 0
    for kind in ("prot", "dna"):
        names = [x[0] for x in W[kind]]; reads = [x[1] for x in W[kind]]
        want = run_cli(ref_bin, d, kind, cfg, True)
        got = run_cli(cli, d, kind, cfg, True, ["-L", str(LIMIT)])
        bad = [(k, got.get(k, "")[:160], want[k][:160]) for k in want if got.get(k) != want[k]]
        assert not bad and len(got) == len(want) == len(names), (kind, len(bad), bad[:3])
        # the same through the C ABI (kj_classify_verbose2); the CLI and the ABI both return KJ_ERR_OVERFLOW as an error, never silently
        clf = kb.Classifier(d + "/db.fmi", d + "/nodes.dmp", device=0, params=_params(kb, cfg, kind == "prot"), max_read_len=LIMIT)
        v2 = verbose2_lines(kb, clf, d + "/db.fmi", names, reads)
        clf.close()
        bad = [(k, v2[k][:160], want[k][:160]) for k in want if v2[k] != want[k]]
        assert not bad, (kind, len(bad), bad[:3])
        emu = emu_lines(kb, d, _params(kb, cfg, kind == "prot"), names, reads, 5461 if kind == "prot" else 16383)
        bad = [k for k, (t, b) in emu.items() if (want[k].split("\t")[0] == "C") != (t != 0) or (t and want[k].split("\t")[2:4] != [str(t), str(b)])]
        assert not bad and len(emu) >= len(names) - 1, (kind, bad[:5])
        noseg = run_cli(cli, d, kind, cfg, False, ["-L", str(LIMIT)])
        if cfg == "mem":
            # Greedy with SEG off is not compared here: on reads that are long homopolymer runs matching many database proteins, the
            # reference's own Greedy -X line (taxon, score, id set) was not the same on two machines, so it is no fixed yardstick
            assert noseg == run_cli(ref_bin, d, kind, cfg, False)
        changed += sum(1 for k in want if noseg[k] != want[k]); total += len(want)
        edges |= edge_reads(want, residues, ref)
    share = changed / total
    print("\n%s: %d reads, -X changes %d (%.1f%%), %d reads show a SEG region edge in column 7" % (cfg, total, changed, 100 * share, len(edges)))
    assert share >= MIN_SEG_SHARE and len(edges) >= MIN_EDGE_READS, (share, len(edges))
