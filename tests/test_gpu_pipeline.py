"""The host code that cuts a batch into pieces and runs the pieces concurrently, each piece boundary exercised with many pieces: the
host-buffer chunk pipeline (two streams, outputs at the chunk's offset, counts committed per call), the sub-batches of the two-kernel
Greedy path (two record buffers per slot), the two lanes of the file pipeline with batches of different read lengths, the variant-ring
overflow and its retry in a later piece, and the device-wide scans of the file parser beyond one scan round.  Every result is compared
bit for bit with the oracle, or with a single-piece path the other GPU tests pin to the oracle."""
import ctypes as C
import os
import numpy as np
import pytest
from helpers import Oracle, SynthDB, make_params, ROOT

pytestmark = pytest.mark.gpu

KJ_TAX_BAD = 0xffffffff
SCAN_ROUND = 1024 * 2048          # elements one kj_scan_blocks round covers (1024 threads x KJ_SCAN_TILE)
FQ_TILE = 2048                    # KJ_FQ_TILE: lines per tile of the FASTQ phase scan


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


@pytest.fixture(scope="module")
def orc(golden):
    return Oracle(golden.fmi, golden.nodes)


@pytest.fixture(scope="module")
def db(built):
    return SynthDB(800, 3)        # the proteins of the golden index


def unpack(seq, off):
    """Packed reads (bases + offsets) -> list of bytes."""
    return [seq[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


def pack_bytes(reads):
    """List of bytes -> (bases, offsets), the layout of Classifier.classify."""
    seq = np.frombuffer(b"".join(reads), dtype=np.uint8).copy()
    off = np.zeros(len(reads) + 1, np.uint64); off[1:] = np.cumsum([len(r) for r in reads])
    return seq, off


def fasta_record(name, read, width=0):
    """One FASTA record; width > 0 wraps the sequence at that many columns."""
    body = b"\n".join(read[k:k + width] for k in range(0, len(read), width)) if width and read else read
    return b">%s\n%s\n" % (name.encode(), body)


def fastq_record(name, read):
    return b"@%s\n%s\n+\n%s\n" % (name.encode(), read, b"I" * len(read))


def write_fasta(path, names, reads, width=0):
    with open(path, "wb") as f:
        f.write(b"".join(fasta_record(nm, r, width) for nm, r in zip(names, reads)))


def write_fastq(path, names, reads, blanks=None):
    """blanks: {record index: number of empty lines written after that record}."""
    blanks = blanks or {}
    with open(path, "wb") as f:
        f.write(b"".join(fastq_record(nm, r) + b"\n" * blanks.get(i, 0) for i, (nm, r) in enumerate(zip(names, reads))))


def kaiju_lines(names, tax):
    """The lines of kaiju's default output (no -v) for the given per-read taxon ids."""
    return ["C\t%s\t%d" % (nm, t) if t else "U\t%s\t0" % nm for nm, t in zip(names, (int(x) for x in tax))]


def histogram(tax):
    """{taxon id: reads}; 0 = unclassified (the layout of Classifier.counts())."""
    u, c = np.unique(np.asarray(tax, dtype=np.uint64), return_counts=True)
    return dict(zip(u.tolist(), c.tolist()))


_emu = None


def emu_lib():
    """The kernel logic on the CPU warp emulator (tests/emu/libkjemu.so, made by build())."""
    global _emu
    if _emu is None:
        E = C.CDLL(os.path.join(ROOT, "tests", "emu", "libkjemu.so"))
        E.kjemu_create.restype = C.c_void_p; E.kjemu_create.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p]
        E.kjemu_destroy.argtypes = [C.c_void_p]
        E.kjemu_classify.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64, C.c_void_p, C.c_void_p, C.c_int]
        _emu = E
    return _emu


def emu_status(fmi, nodes, params, seq, off, nthreads=8):
    """Status code of the emulated kernel logic on single-end reads (0, or KJ_ERR_OVERFLOW - 100 * error flags); honours KJ_VARIANT_CAP."""
    import kaiju_b200
    E = emu_lib()
    kp = kaiju_b200.KjParams(mode=params["mode"], min_fragment_length=params["min_fragment_length"], mismatches=params["mismatches"],
                             min_score=params["min_score"], seed_length=params["seed_length"], use_evalue=params["use_evalue"],
                             min_evalue=params["min_evalue"], seg=params["seg"], input_is_protein=params["input_is_protein"], name_mode=0)
    h = E.kjemu_create(fmi.encode(), nodes.encode(), C.byref(kp)); assert h
    seq = np.ascontiguousarray(seq, dtype=np.uint8); off = np.ascontiguousarray(off, dtype=np.uint64)
    n = len(off) - 1; tax = np.zeros(n, np.uint64); best = np.zeros(n, np.uint32)
    rc = E.kjemu_classify(h, seq.ctypes.data, off.ctypes.data, None, None, n, tax.ctypes.data, best.ctypes.data, nthreads)
    E.kjemu_destroy(h)
    return rc


def _same(what, got, want):
    bad = np.nonzero(np.asarray(got) != np.asarray(want))[0]
    assert len(bad) == 0, (what, "%d of %d differ" % (len(bad), len(want)), [(int(i), int(got[i]), int(want[i])) for i in bad[:5]])


def _counts(clf):
    ids, cnt = clf.counts()
    return dict(zip(ids.tolist(), cnt.tolist()))


def _from_compact(clf, comp):
    ids = clf.compact_ids()
    comp = np.asarray(comp).view(np.uint32)
    return np.where(comp == KJ_TAX_BAD, 0, ids[np.minimum(comp, len(ids) - 1)])


def _dev(*arrays):
    import torch
    return [None if a is None else torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda() for a in arrays]


def _ptr(t):
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. the two lanes of the file pipeline, batches with different longest reads
# ---------------------------------------------------------------------------------------------------------------------------------
LANE_CHUNK = 4 << 20
LANE_GROUPS = [(5000, 16000), (300, 500), (150, 150)] * 3       # read lengths of group g; one group per batch


def _lane_profile_fasta(db, path):
    """Single-end FASTA in groups of about one batch each (KJ_INGEST_CHUNK = LANE_CHUNK), longest reads first, three times over.  Batch w
    holds the complete records of file bytes [w, w + 1) * LANE_CHUNK; a FASTA record is complete once the next header line is in the batch.
    Where the next group has shorter reads, it starts early enough that the records carried over into the next batch are its own (the
    batch before gets a few of the shorter reads); where it has longer reads, it starts with the first record that crosses the edge.  So
    every batch's longest read is its group's.  Returns names, reads and the longest read of each batch."""
    pools = []
    for g, (lo, hi) in enumerate(LANE_GROUPS):
        if lo == hi:
            s, o, _, _ = db.reads(500 + g, 0, 40000, lo, False)
        else:
            s, o = db.long_reads(500 + g, 0, 16000 if hi <= 500 else 800, lo, hi)
        pools.append(unpack(s, o))
    names, reads, recs, used = [], [], [], [0] * len(LANE_GROUPS)
    pos, g = 0, 0
    while True:
        nm = "g%d_%d" % (g, used[g]); r = pools[g][used[g]]; t = fasta_record(nm, r, 80)
        if g + 1 < len(LANE_GROUPS):
            edge = (g + 1) * LANE_CHUNK; nxt = LANE_GROUPS[g + 1][1] + LANE_GROUPS[g + 1][1] // 80 + 64       # bytes of the next group's longest record
            if (pos + len(t) + 2 * nxt > edge) if LANE_GROUPS[g + 1][1] < LANE_GROUPS[g][1] else (pos + len(t) > edge):
                g += 1; continue
        elif pos + len(t) > len(LANE_GROUPS) * LANE_CHUNK:
            break
        names.append(nm); reads.append(r); recs.append(t); used[g] += 1; pos += len(t)
    with open(path, "wb") as f:
        f.write(b"".join(recs))
    # the batch of record i: where the header line of record i + 1 ends (the last record: the last batch)
    hdr_end = np.cumsum([0] + [len(t) for t in recs])[1:-1] + np.array([t.index(b"\n") for t in recs[1:]])
    batch = np.append(hdr_end // LANE_CHUNK, (pos - 1) // LANE_CHUNK)
    lens = np.array([len(r) for r in reads])
    return names, reads, [int(lens[batch == w].max()) for w in range(int(batch.max()) + 1)]


@pytest.mark.parametrize("kw", [dict(mode="greedy", e=3), dict(mode="mem")])
def test_file_lanes_with_alternating_read_lengths(kb, golden, orc, db, tmp_path, monkeypatch, kw):
    """kj_classify_files launches batch k + 1 on one lane while batch k runs on the other, each with run parameters from its own longest
    read.  Batches of 5-16 kb, 300-500 and 150-base reads alternate, each thousands of reads, so the warps of both lanes are busy at once:
    the per-warp scratch of one lane must not depend on the other lane's launch.  Output == Classifier.classify on every read == the oracle
    on a stratified subsample; counts() == the histogram of the output."""
    path = str(tmp_path / "lanes.fa")
    names, reads, batch_max = _lane_profile_fasta(db, path)
    assert len(batch_max) == len(LANE_GROUPS)
    for w, (lo, hi) in enumerate(LANE_GROUPS):
        assert lo <= batch_max[w] <= hi, (w, batch_max)
    seq, off = pack_bytes(reads); n = len(reads)
    monkeypatch.setenv("KJ_INGEST_CHUNK", str(LANE_CHUNK))
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params(**kw))
    out = str(tmp_path / "lanes.tsv")
    got_n, got_k = clf.classify_files(path, None, out)
    got = open(out).read().splitlines()
    counted = _counts(clf)
    tax = clf.classify(seq, off, want_best=False)
    want = kaiju_lines(names, tax)
    assert got_n == n and len(got) == n
    bad = [i for i in range(n) if got[i] != want[i]]
    assert not bad, ("%d of %d lines differ from Classifier.classify" % (len(bad), n), [(got[i], want[i]) for i in bad[:3]])
    # oracle: the first and last reads of every group and every 7th read
    first = {}
    for i, nm in enumerate(names):
        first.setdefault(nm.split("_")[0], []).append(i)
    sub = sorted(set(range(0, n, 7)) | {i for v in first.values() for i in v[:3] + v[-3:]})
    ss, so = pack_bytes([reads[i] for i in sub])
    otax, _ = orc.classify_batch(make_params(**kw), ss, so)
    _same("oracle", [int(tax[i]) for i in sub], otax)
    out_tax = np.array([int(l.split("\t")[2]) for l in got], dtype=np.uint64)
    assert counted == histogram(out_tax) and got_k == int((out_tax != 0).sum())
    assert 0.3 < got_k / n < 0.95
    clf.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. the host-buffer chunk pipeline
# ---------------------------------------------------------------------------------------------------------------------------------
def _ragged_pe150(db, n):
    """PE150 with empty mates, mates below the 3m length gate on one or both sides."""
    s1, o1, s2, o2 = db.reads(611, 0, n, 150, True)
    r1, r2 = unpack(s1, o1), unpack(s2, o2)
    for i in range(0, n, 97):
        r2[i] = b""
    for i in range(13, n, 89):
        r1[i] = r1[i][:20]
    for i in range(29, n, 211):
        r1[i] = r1[i][:30]; r2[i] = r2[i][:10]
    for i in range(41, n, 307):
        r1[i] = b""
    return pack_bytes(r1) + pack_bytes(r2)


@pytest.mark.parametrize("wide", [False, True])
def test_host_chunk_pipeline(kb, golden, orc, db, monkeypatch, wide):
    """KJ_CHUNK_READS = 1024 on 10,007 items: ten chunks alternate between the two streams.  classify, classify2_ptrs (dense indices in
    device memory), classify_verbose (id sets) and the per-taxon counts of two calls == the oracle for every read, MEM and Greedy."""
    import torch
    n = 10007
    monkeypatch.setenv("KJ_CHUNK_READS", "1024")
    if wide:
        monkeypatch.setenv("KJ_FORCE_WIDE", "1")
    work = {"pe150": _ragged_pe150(db, n), "se100": db.reads(612, 0, n, 100, False)}
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"))
    for kw in (dict(mode="mem"), dict(mode="greedy")):
        clf.set_params(kb.make_params(**kw)); P = make_params(**kw)
        for tag, (s1, o1, s2, o2) in work.items():
            what = (kw["mode"], tag, wide)
            otax, obest = orc.classify_batch(P, s1, o1, s2, o2)
            clf.counts_reset()
            k0 = clf.kernel_launches
            tax, best = clf.classify(s1, o1, s2, o2)
            assert clf.kernel_launches - k0 >= -(-n // 1024), what        # (at least) one launch per chunk
            _same(what + ("taxon",), tax, otax); _same(what + ("best",), best, obest)
            vtax, vbest, ids = clf.classify_verbose(s1, o1, s2, o2)
            _same(what + ("verbose taxon",), vtax, otax); _same(what + ("verbose best",), vbest, obest)
            r1 = unpack(s1, o1); r2 = unpack(s2, o2) if s2 is not None else None
            bad = []
            for i in range(n):
                want = tuple(sorted(orc.classify_one(P, r1[i], r2[i] if r2 else None)[2])) if otax[i] else ()
                if ids[i] != want:
                    bad.append((i, ids[i], want))
            assert not bad, (what, "id sets: %d differ" % len(bad), bad[:3])
            exp = {k: 2 * v for k, v in histogram(otax).items()}
            assert _counts(clf) == exp, what
            comp = torch.full((n,), -1, dtype=torch.int32, device="cuda")
            tax2 = np.zeros(n, np.uint64); best2 = np.zeros(n, np.uint32)
            clf.classify2_ptrs(s1.ctypes.data, o1.ctypes.data, None if s2 is None else s2.ctypes.data, None if o2 is None else o2.ctypes.data, n,
                               tax2.ctypes.data, best2.ctypes.data, comp.data_ptr())
            torch.cuda.synchronize()
            _same(what + ("classify2 taxon",), tax2, otax); _same(what + ("classify2 best",), best2, obest)
            _same(what + ("classify2 dense index",), _from_compact(clf, comp.cpu().numpy()), otax)
    clf.close()


def test_host_chunk_cut_by_bases(kb, golden, orc, db):
    """About 275 MB of 15-16.3 kb reads: the chunk is cut by KJ_CHUNK_BYTES (2^28 bases), not by its read count.  Result == the two halves
    of the batch classified separately (one chunk each) == the oracle on the 300 reads around the cut."""
    n = 17600
    s, o = db.long_reads(613, 0, n, 15000, 16300)
    assert int(o[-1]) > (1 << 28)
    cut = int(np.searchsorted(o[1:], np.uint64(1 << 28), side="right"))       # reads in the first chunk
    assert 150 <= cut <= n - 150 and cut != n // 2
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"))
    k0 = clf.kernel_launches
    tax, best = clf.classify(s, o)
    assert clf.kernel_launches - k0 == 3                                  # two chunks + the count commit
    h = n // 2
    for lo, hi in ((0, h), (h, n)):
        ht, hb = clf.classify(s[int(o[lo]):int(o[hi])], o[lo:hi + 1] - o[lo])
        _same(("half", lo), ht, tax[lo:hi]); _same(("half best", lo), hb, best[lo:hi])
    a, b = cut - 150, cut + 150
    otax, obest = orc.classify_batch(make_params("mem"), s[int(o[a]):int(o[b])], o[a:b + 1] - o[a])
    _same("oracle taxon", tax[a:b], otax); _same("oracle best", best[a:b], obest)
    assert (tax != 0).mean() > 0.5
    clf.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. the sub-batches of the two-kernel Greedy path
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wide", [False, True])
def test_greedy_sub_batches(kb, golden, orc, db, monkeypatch, wide):
    """KJ_SPLIT_SUB = 1024 / 1027 / 1031 on 9-10 k items: 9 or more sub-batches, so the two record buffers of a slot are each reused several
    times.  PE150 -m 11 (the fixed-profile kernels) and SE100 -m 12, through classify_device2 (three back-to-back calls of different n on a
    non-default stream, no synchronisation between them) and through classify with KJ_CHUNK_READS = 4096 (both slots in flight); then
    MEM and back (the record buffers are released and allocated again).  == the oracle == the single-kernel path (KJ_NO_SPLIT)."""
    import torch
    if wide:
        monkeypatch.setenv("KJ_FORCE_WIDE", "1")
    work = {"pe150_m11": (dict(mode="greedy"), db.reads(621, 0, 9601, 150, True), 150),
            "se100_m12": (dict(mode="greedy", m=12), db.reads(622, 0, 9973, 100, False), 100)}
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"))
    stream = torch.cuda.Stream()
    for tag, (kw, (s1, o1, s2, o2), rl) in work.items():
        n = len(o1) - 1; paired = s2 is not None
        otax, obest = orc.classify_batch(make_params(**kw), s1, o1, s2, o2)
        clf.set_params(kb.make_params(**kw))
        monkeypatch.setenv("KJ_NO_SPLIT", "1")
        ntax, nbest = clf.classify(s1, o1, s2, o2)
        monkeypatch.delenv("KJ_NO_SPLIT")
        _same((tag, wide, "single kernel"), ntax, otax); _same((tag, wide, "single kernel best"), nbest, obest)
        d = _dev(s1, o1, s2, o2); torch.cuda.synchronize()

        def device_calls(sizes):
            outs = []; sub = int(os.environ["KJ_SPLIT_SUB"])
            with torch.cuda.stream(stream):
                for m in sizes:
                    k0 = clf.kernel_launches
                    t = (torch.full((m,), -1, dtype=torch.int64, device="cuda"), torch.full((m,), -1, dtype=torch.int32, device="cuda"),
                         torch.full((m,), -1, dtype=torch.int32, device="cuda"))
                    clf.classify_device2(_ptr(d[0]), _ptr(d[1]), _ptr(d[2]), _ptr(d[3]), m, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(),
                                         rl, rl if paired else 0, stream.cuda_stream)
                    assert clf.kernel_launches - k0 == 2 * -(-m // sub), (m, sub)      # a front-end and a search launch per sub-batch
                    outs.append((m, t))
            stream.synchronize(); clf.check_errors()
            for m, (dt, dbst, dc) in outs:
                what = (tag, wide, os.environ.get("KJ_SPLIT_SUB"), m)
                _same(what + ("taxon",), dt.cpu().numpy().view(np.uint64), otax[:m]); _same(what + ("best",), dbst.cpu().numpy().view(np.uint32), obest[:m])
                _same(what + ("dense index",), _from_compact(clf, dc.cpu().numpy()), otax[:m])

        for sub in ("1024", "1027", "1031"):
            monkeypatch.setenv("KJ_SPLIT_SUB", sub)
            device_calls((n - 2077, n - 1000, n - 1531))
            monkeypatch.setenv("KJ_CHUNK_READS", "4096")
            tax, best = clf.classify(s1, o1, s2, o2)
            monkeypatch.delenv("KJ_CHUNK_READS")
            _same((tag, wide, sub, "host"), tax, otax); _same((tag, wide, sub, "host best"), best, obest)
        # MEM releases the record buffers; back in Greedy a larger call allocates them again
        clf.set_params(kb.make_params("mem")); clf.classify(s1[:int(o1[100])], o1[:101], None if s2 is None else s2[:int(o2[100])], None if o2 is None else o2[:101])
        clf.set_params(kb.make_params(**kw))
        device_calls((n,))
        monkeypatch.delenv("KJ_SPLIT_SUB")
    clf.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. variant-ring overflow in a later piece, and the retry
# ---------------------------------------------------------------------------------------------------------------------------------
RING_KW = dict(mode="greedy", e=8, s=30, m=9, seed=5, E=1e-9)
RING_CAP = "32"
RING_AT = 3300                        # position of the overflowing reads: chunk 3 (1024 reads per chunk), sub-batch 3 (1024 per sub-batch)


def _ring_workload(golden, db, monkeypatch):
    """3,500 SE100 reads that fit a 32-entry variant ring and, at RING_AT, 8 that overflow it but fit 128 entries (reads 5460-5485 of the
    seed-401 stream; checked here on the emulated kernel logic)."""
    s, o, _, _ = db.reads(401, 0, 5486, 100, False)
    r = unpack(s, o)
    clean, hot = r[:3500], [r[i] for i in (5460, 5461, 5462, 5463, 5464, 5471, 5479, 5485)]
    P = make_params(**RING_KW)
    monkeypatch.setenv("KJ_VARIANT_CAP", RING_CAP)
    assert emu_status(golden.fmi, golden.nodes, P, *pack_bytes(clean)) == 0
    for x in hot:
        assert emu_status(golden.fmi, golden.nodes, P, *pack_bytes([x]), nthreads=1) == -406        # KJ_ERR_OVERFLOW - 100 * flag 4
    monkeypatch.setenv("KJ_VARIANT_CAP", "128")
    assert emu_status(golden.fmi, golden.nodes, P, *pack_bytes(hot)) == 0
    monkeypatch.setenv("KJ_VARIANT_CAP", RING_CAP)
    reads = clean[:RING_AT] + hot + clean[RING_AT:]
    return ["r%d" % i for i in range(len(reads))], reads


def test_variant_ring_overflow_in_a_later_piece(kb, golden, orc, db, tmp_path, monkeypatch):
    """Reads that overflow the Greedy variant ring only in a later piece: chunk 3 of a host call (the call is repeated inside, counts are
    committed once), sub-batch 3 of a classify_device2 call (check_errors raises, the repeated call succeeds), a batch >= 2 of
    classify_files (the lanes are repeated, output and counts equal the oracle's)."""
    import torch
    names, reads = _ring_workload(golden, db, monkeypatch)
    seq, off = pack_bytes(reads); n = len(reads)
    otax, obest = orc.classify_batch(make_params(**RING_KW), seq, off)
    # host buffers, KJ_CHUNK_READS = 1024
    monkeypatch.setenv("KJ_CHUNK_READS", "1024")
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params(**RING_KW))
    tax, best = clf.classify(seq, off)
    _same("host taxon", tax, otax); _same("host best", best, obest)
    assert _counts(clf) == histogram(otax)
    clf.close()
    monkeypatch.delenv("KJ_CHUNK_READS")
    # device buffers, KJ_SPLIT_SUB = 1024
    monkeypatch.setenv("KJ_SPLIT_SUB", "1024")
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params(**RING_KW))
    ds, do = _dev(seq, off); dt = torch.zeros(n, dtype=torch.int64, device="cuda"); dbst = torch.zeros(n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    clf.classify_device(ds.data_ptr(), do.data_ptr(), None, None, n, dt.data_ptr(), dbst.data_ptr(), 100); torch.cuda.synchronize()
    with pytest.raises(kb.KaijuError, match="variant ring was enlarged"):
        clf.check_errors()
    clf.classify_device(ds.data_ptr(), do.data_ptr(), None, None, n, dt.data_ptr(), dbst.data_ptr(), 100); torch.cuda.synchronize()
    clf.check_errors()
    _same("device taxon", dt.cpu().numpy().view(np.uint64), otax); _same("device best", dbst.cpu().numpy().view(np.uint32), obest)
    clf.close()
    monkeypatch.delenv("KJ_SPLIT_SUB")
    # files, 64 KB batches: the overflowing reads sit at about 360 KB
    path = str(tmp_path / "ring.fa"); write_fasta(path, names, reads)
    monkeypatch.setenv("KJ_INGEST_CHUNK", "65536")
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params(**RING_KW))
    out = str(tmp_path / "ring.tsv")
    got_n, got_k = clf.classify_files(path, None, out)
    assert got_n == n and open(out).read().splitlines() == kaiju_lines(names, otax)
    assert _counts(clf) == histogram(otax) and got_k == int((otax != 0).sum())
    clf.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# 5. the device-wide scans of the file parser
# ---------------------------------------------------------------------------------------------------------------------------------
def _blank_lines(n, every):
    """1-3 empty lines after every `every`-th of n FASTQ records."""
    return {i: 1 + (i // every) % 3 for i in range(0, n, every)}


def test_parser_scans_beyond_one_round(kb, golden, db, tmp_path, monkeypatch):
    """KJ_INGEST_CHUNK = 64 MiB: one batch of more than 2,097,152 lines, so the scans over lines need a second round of block sums, and a
    FASTQ with blank lines between records runs the phase scan over more than 1,000 tiles.  Output == Classifier.classify on the packed
    reads, names in order."""
    monkeypatch.setenv("KJ_INGEST_CHUNK", str(64 << 20))
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"))
    # FASTA wrapped at 20 columns: 9 lines per 150-base read
    s, o, _, _ = db.reads(631, 0, 330000, 150, False); reads = unpack(s, o); names = ["a%d" % i for i in range(len(reads))]
    path = str(tmp_path / "wrapped.fa"); write_fasta(path, names, reads, width=20)
    text = open(path, "rb").read(); assert text.count(b"\n") > SCAN_ROUND and len(text) < (64 << 20); del text
    got_n, _ = clf.classify_files(path, None, str(tmp_path / "wrapped.tsv"))
    tax = clf.classify(s, o, want_best=False)
    assert got_n == len(reads) and open(tmp_path / "wrapped.tsv").read().splitlines() == kaiju_lines(names, tax)
    # FASTQ of 48-base reads with blank lines between records
    s, o, _, _ = db.reads(632, 0, 560000, 48, False); reads = unpack(s, o); names = ["q%d" % i for i in range(len(reads))]
    path = str(tmp_path / "blank.fq"); write_fastq(path, names, reads, _blank_lines(len(reads), 5))
    text = open(path, "rb").read(); lines = text.count(b"\n")
    assert lines > SCAN_ROUND and lines > 1000 * FQ_TILE and len(text) < (64 << 20); del text
    got_n, _ = clf.classify_files(path, None, str(tmp_path / "blank.tsv"))
    tax = clf.classify(s, o, want_best=False)
    assert got_n == len(reads) and open(tmp_path / "blank.tsv").read().splitlines() == kaiju_lines(names, tax)
    # small files of 2048 * 3 -+ 1 lines: the last line on either side of a tile edge
    monkeypatch.delenv("KJ_INGEST_CHUNK")
    s, o, _, _ = db.reads(633, 0, 1500, 100, False); reads = unpack(s, o); names = ["t%d" % i for i in range(len(reads))]
    tax = clf.classify(s, o, want_best=False)
    for lines in (3 * FQ_TILE - 1, 3 * FQ_TILE + 1):
        blanks = {i: 1 for i in range(3, 4 * len(reads), 10)[:lines - 4 * len(reads)]}
        path = str(tmp_path / ("edge%d.fq" % lines)); write_fastq(path, names, reads, blanks)
        assert open(path, "rb").read().count(b"\n") == lines
        got_n, _ = clf.classify_files(path, None, str(tmp_path / "edge.tsv"))
        assert got_n == len(reads) and open(tmp_path / "edge.tsv").read().splitlines() == kaiju_lines(names, tax), lines
    clf.close()
