"""Indexes of every suffix-array shape a Kaiju database can have, on the CPU: SA exponents 0, 1, 2, 4, 5 (kaiju-mkbwt's default, nr's) and 7,
every residue class of nseq and bwtlen modulo 2^exponent at exponents 2 and 5, and samples of 5 and 6 bytes (tests/index_shapes.py).  The oracle
is pinned to the reference's own get_suffix / FMindex and CLI at these shapes, then the kernel source on the warp emulator and the host
transcoder are checked against it."""
import ctypes as C
import os
import numpy as np
import pytest
import emu_compact
import index_shapes as S
import test_kernel_logic_emulated as K
from helpers import Oracle, REF_DIR, have_ref, make_params, oracle_lib, run_ref_kaiju

pytestmark = pytest.mark.skipif(not have_ref(), reason="oracle/_ref (index builder) not built")
LAYOUTS = [{}, {"KJ_FORCE_WIDE": "1"}, {"KJ_FORCE_COMPACT": "1"}]
MODES = [dict(mode="mem"), dict(mode="greedy", e=3)]


@pytest.fixture(scope="module")
def fam(built, tmp_path_factory):
    return S.build_family(str(tmp_path_factory.mktemp("shapes")), list(S.SMALL) + list(S.WIDE), nreads=2000, wide_reads=600)


@pytest.fixture(scope="module")
def emu(built, tmp_path_factory):
    """the compact-capable emulator build (kj_emu.cpp + the compact instantiation): narrow, wide and compact by the descriptor's layout"""
    return emu_compact.load(str(tmp_path_factory.mktemp("emu_compact")), K.KjParams)


def _ref_lib(fmi):
    R = C.CDLL(os.path.join(REF_DIR, "libkaijuref.so")); libc = C.CDLL(None)
    libc.fopen.restype = C.c_void_p; libc.fopen.argtypes = [C.c_char_p, C.c_char_p]; libc.fclose.argtypes = [C.c_void_p]
    R.readIndexes.restype = C.c_void_p; R.readIndexes.argtypes = [C.c_void_p]

    class BWT(C.Structure):   # bwt/bwt.h:13-23
        _fields_ = [("len", C.c_long), ("nseq", C.c_int), ("bwt", C.c_void_p), ("alen", C.c_int), ("alphabet", C.c_char_p), ("f", C.c_void_p), ("s", C.c_void_p)]
    fp = libc.fopen(fmi.encode(), b"r"); b = BWT.from_address(R.readIndexes(fp)); libc.fclose(fp)
    R.FMindex.restype = C.c_long; R.FMindex.argtypes = [C.c_void_p, C.c_ubyte, C.c_long]
    R.get_suffix.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.POINTER(C.c_int), C.POINTER(C.c_long)]
    return R, b


def test_every_planned_shape_was_built(fam):
    """The fixture asserts each class as it builds it; here the union: the guard class at exponents 2, 4, 5, 7 and in the 5-byte index, the
    class whose header counts an entry no row addresses, exponent 0 (no walk), and samples of 5 and 6 bytes."""
    assert {x.exp for x in fam.values() if x.guard} >= {2, 4, 5, 7} and fam["w5"].guard
    assert any(x.written == x.h["ncheck"] - 1 for x in fam.values())
    assert fam["e0"].h["ncheck"] == fam["e0"].h["bwtlen"] - fam["e0"].h["nseq"]
    assert (fam["w5"].h["nbytes"], fam["w6"].h["nbytes"]) == (5, 6)
    assert fam["w5"].h["sbits"] + fam["w5"].h["pbits"] >= 33 and fam["w6"].h["sbits"] + fam["w6"].h["pbits"] >= 41


@pytest.mark.parametrize("name", sorted(S.SMALL))
def test_oracle_get_suffix_and_fmindex_equal_reference(fam, name):
    """ko_get_suffix == the reference's get_suffix for every row that holds a suffix of a sequence ([nseq, bwtlen)), and ko_fmindex == FMindex
    on every 7th row for every letter.  The last sampled row of a guard-class index is the exception: the reference's get_suffix decodes the
    bytes after its suffix-array array there (heap contents; a sequence number of the index only by chance), the oracle reports "no entry"
    (sequence -1), as the device reads its guard entry ("no taxon").  Reads that walk into that row are compared between the oracle and the
    kernels only (test_emulated_kernels_equal_oracle); the reference CLI is compared on reads that do not."""
    x = fam[name]; orc = Oracle(x.fmi, x.nodes); L = oracle_lib(); R, b = _ref_lib(x.fmi)
    n = x.h["bwtlen"]
    iseq = C.c_int(); pos = C.c_long(); oseq = C.c_int(); opos = C.c_int64()
    bad, walked = [], []
    R.get_suffix(b.f, b.s, x.last_row, C.byref(iseq), C.byref(pos)); past = iseq.value
    for k in range(x.h["nseq"], n):
        L.ko_get_suffix(orc.idx, k, C.byref(oseq), C.byref(opos))
        R.get_suffix(b.f, b.s, k, C.byref(iseq), C.byref(pos))
        if oseq.value == -1:                    # the walk from k ends on the guard row: the reference decodes the same bytes past its array
            walked.append(k)
            if iseq.value != past:
                bad.append((k, iseq.value, pos.value, oseq.value, opos.value))
        elif (iseq.value, pos.value) != (oseq.value, opos.value):
            bad.append((k, iseq.value, pos.value, oseq.value, opos.value))
    assert not bad, bad[:5]
    assert x.last_row in walked if x.guard else not walked, walked[:5]
    for k in list(range(0, n + 1, 7)) + [n - 1, n]:
        for c in range(x.h["alen"]):
            assert L.ko_fmindex(orc.idx, c, k) == R.FMindex(b.f, c, k), (k, c)


def _cli_v(x, fa, kw, out):
    """reference `kaiju -z 1 -v`: {name: (C/U, taxon, best, ids)} and {name: accession set}"""
    ref = run_ref_kaiju(x.nodes, x.fmi, fa, None, threads=1, out=out, **kw)
    acc = {}
    for line in open(out):
        p = line.rstrip("\n").split("\t")
        if p[0] == "C":
            acc[p[1]] = tuple(sorted(a for a in p[5].split(",") if a))
    return ref, acc


@pytest.mark.parametrize("name", sorted(S.SMALL) + sorted(S.WIDE))
def test_oracle_equals_reference_cli(fam, tmp_path, name):
    """taxon, best and the column-5 id set of `kaiju -z 1 -v` (MEM, Greedy -e 3) == the oracle on every read"""
    x = fam[name]; orc = Oracle(x.fmi, x.nodes); fa = str(tmp_path / "r.fa"); S.write_fasta(fa, x.reads)
    seq, off = S.pack(x.reads)
    for kw in MODES:
        ref, _ = _cli_v(x, fa, kw, str(tmp_path / "o.tsv"))
        P = make_params(**kw); tax, best = orc.classify_batch(P, seq, off)
        bad = [i for i in range(len(x.reads)) if (ref["r%d" % i][1], ref["r%d" % i][2]) != (int(tax[i]), int(best[i]))]
        assert not bad, (kw, [(i, ref["r%d" % i], int(tax[i]), int(best[i])) for i in bad[:5]])
        for i in np.nonzero(tax)[0][:300]:
            _, _, ids = orc.classify_one(P, x.reads[i].encode())
            assert tuple(ids) == ref["r%d" % i][3], (kw, i)
        assert (tax != 0).mean() > 0.5


def _emu_v2(E, x, P, seq, off):
    kp = K.KjParams(**P); h = E.kjemu_create(x.fmi.encode(), x.nodes.encode() if not P.get("name_mode") else None, C.byref(kp)); assert h
    n = len(off) - 1; tax = np.zeros(n, np.uint64); best = np.zeros(n, np.uint32); ids = np.zeros((n, 21), np.uint64); nids = np.zeros(n, np.uint8)
    acc = np.zeros((n, 20), np.uint32); nacc = np.zeros(n, np.uint8); frag = np.zeros((n, 2048), np.uint8); flen = np.zeros(n, np.uint32)
    E.kjemu_classify_v2.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64] + [C.c_void_p] * 7 + [C.c_uint32, C.c_void_p, C.c_int]
    rc = E.kjemu_classify_v2(h, seq.ctypes.data, off.ctypes.data, None, None, n, tax.ctypes.data, best.ctypes.data, ids.ctypes.data, nids.ctypes.data,
                             acc.ctypes.data, nacc.ctypes.data, frag.ctypes.data, 2048, flen.ctypes.data, 4)
    E.kjemu_destroy(h); assert rc == 0
    return tax, best, [tuple(int(v) for v in ids[i, :nids[i]]) for i in range(n)], [tuple(int(v) for v in acc[i, :nacc[i]]) for i in range(n)]


@pytest.mark.parametrize("name", sorted(S.SMALL) + sorted(S.WIDE))
def test_emulated_kernels_equal_oracle(fam, emu, monkeypatch, tmp_path, name):
    """The kernel source on the warp emulator, narrow / wide / compact (the last two resolve every taxon by the SA walk), MEM, Greedy in one kernel
    and in two (KJ_EMU_SPLIT): taxon and best == the oracle on the reads plus the reads that walk into the guard row; the id column == the
    oracle's, the accession column == the reference CLI's; name mode gives the same results on every layout."""
    import kaiju_b200 as kb
    x = fam[name]; orc = Oracle(x.fmi, x.nodes)
    reads = x.reads[:800] + x.guard_reads; seq, off = S.pack(reads)
    fa = str(tmp_path / "r.fa"); S.write_fasta(fa, x.reads[:800])
    L = kb.lib(); L.kj_fmi_accession.restype = C.c_char_p; L.kj_fmi_accession.argtypes = [C.c_void_p, C.c_uint32]
    f = C.c_void_p(); assert L.kj_fmi_load(x.fmi.encode(), C.byref(f)) == 0
    try:
        for kw in MODES:
            P = make_params(**kw); otax, obest = orc.classify_batch(P, seq, off)
            _, racc = _cli_v(x, fa, kw, str(tmp_path / "o.tsv"))
            names_ref = None
            for env in LAYOUTS:
                for split in ([False, True] if kw["mode"] == "greedy" else [False]):
                    with monkeypatch.context() as m:
                        for k, v in dict(env, **({"KJ_EMU_SPLIT": "1"} if split else {})).items():
                            m.setenv(k, v)
                        tax, best, ids, acc = _emu_v2(emu, x, P, seq, off)
                        bad = np.nonzero((tax != otax) | (best != obest))[0]
                        assert len(bad) == 0, (kw, env, split, [(int(i), int(tax[i]), int(otax[i]), int(best[i]), int(obest[i])) for i in bad[:5]])
                        for i in np.nonzero(otax)[0][:200]:
                            assert ids[i] == tuple(orc.classify_one(P, reads[i].encode())[2]), (kw, env, i)
                            if i < 800:
                                got = tuple(sorted(L.kj_fmi_accession(f, a).decode() for a in acc[i]))
                                assert got == racc["r%d" % i], (kw, env, i, got, racc["r%d" % i])
                        if not split:
                            nm = _emu_v2(emu, x, dict(P, name_mode=1), seq, off)
                            names_ref = names_ref or nm
                            assert np.array_equal(nm[0], names_ref[0]) and np.array_equal(nm[1], names_ref[1]) and nm[2] == names_ref[2], (kw, env)
    finally:
        L.kj_fmi_free(f)


def _mix(h, data):
    """kj_mix_bytes (kj_host.cpp)"""
    M = (1 << 64) - 1; i = 0; n = len(data)
    w = np.frombuffer(data[:n - n % 8], dtype="<u8")
    for v in w.tolist():
        h = ((h ^ v) * 0x9E3779B97F4A7C15) & M; h = ((h << 29) | (h >> 35)) & M
    i = n - n % 8
    v = int.from_bytes(data[i:] + b"\0" * (8 - (n - i)), "little") if i < n else 0
    h = ((h ^ v ^ n) * 0x9E3779B97F4A7C15) & M
    return ((h << 29) | (h >> 35)) & M


@pytest.mark.parametrize("name", ["w5", "w6", "e7", "e0"])
def test_host_transcoder_decodes_wide_samples(fam, name):
    """host_index_checksums succeeds for 5- and 6-byte samples, and its sa_tax is a plain decode of the .fmi's samples (big-endian, sequence =
    value >> pbits) mapped through the sequence taxa (dense taxon index: rank of the taxon among the sorted nodes.dmp ids)."""
    import kaiju_b200 as kb
    x = fam[name]; h = x.h
    got = kb.host_index_checksums(x.fmi, x.nodes)
    names = S.fmi_seq_names(x.fmi)
    with open(x.fmi, "rb") as f:
        f.seek(h["sa_off"] + sum(1 + len(s) for s in names) + 12 * h["nseq"]); raw = f.read(h["ncheck"] * h["nbytes"])
    a = np.frombuffer(raw, np.uint8).reshape(-1, h["nbytes"]).astype(np.uint64)
    val = np.zeros(len(a), np.uint64)
    for j in range(h["nbytes"]):
        val = (val << np.uint64(8)) | a[:, j]
    seq = (val >> np.uint64(h["pbits"])).astype(np.int64)
    assert seq.max() < h["nseq"] and len(seq) == h["ncheck"]
    dense = {t: i + 1 for i, t in enumerate(range(100, 100 + S.NTAX))}          # nodes.dmp ids sorted: 1, 100, ..., 106
    seq_tax = np.array([dense[int(s.rsplit("_", 1)[1])] for s in names], np.uint32)
    assert int(got[7]) == h["ncheck"] and int(got[5]) == h["bwtlen"]
    assert int(got[2]) == _mix(0x6b616a75 + 2, seq_tax[seq].astype("<u4").tobytes())
    assert int(got[3]) == _mix(0x6b616a75 + 3, seq_tax.astype("<u4").tobytes())
