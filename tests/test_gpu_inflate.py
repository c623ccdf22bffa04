"""BGZF input on the GPU: the inflate kernel against zlib on the files the emulator is checked on, and kj_classify_files on blocked gzip against the
same reads as plain text and as ordinary gzip -- byte-identical output, with the library reporting which path inflated the text.  The three
error cases run once each and only check that a bad block is reported; malformed input is explored on the CPU (test_inflate_emulated.py)."""
import gzip
import os

import numpy as np
import pytest

import emu_inflate as ei
from conftest import GOLD

pytestmark = pytest.mark.gpu
SMALL_CHUNK = "70000"              # KJ_INGEST_CHUNK: many rounds, each ending inside a block


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


@pytest.fixture(scope="module")
def clf_mem(kb, golden):
    c = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"))
    yield c
    c.close()


def gold_text(name):
    return gzip.open(os.path.join(GOLD, name)).read()


def three_ways(d, stem, text, level=6, block=ei.MAX_SLICE):
    """text as a plain file, an ordinary gzip file and a BGZF file"""
    paths = {k: str(d / ("%s.%s" % (stem, k))) for k in ("txt", "gz", "bgz")}
    open(paths["txt"], "wb").write(text)
    open(paths["gz"], "wb").write(gzip.compress(text, 1))
    open(paths["bgz"], "wb").write(ei.bgzf_write(text, level, block=block))
    return paths


def run(clf, out, in1, in2=None, verbose=False):
    n, k = clf.classify_files(in1, in2, str(out), verbose=verbose)
    return n, k, open(str(out), "rb").read(), clf.files_device_inflated_bytes


def test_kernel_equals_zlib_on_the_valid_set(clf_mem):
    for name, text, bg in ei.valid_files():
        assert clf_mem.debug_inflate_bgzf(bg, out_cap=len(text) + 16) == text, name
    text = gold_text("pe150_1.fq.gz")
    for block in (1000, 4096, 65280):
        assert clf_mem.debug_inflate_bgzf(ei.bgzf_write(text, 1, block=block), out_cap=len(text)) == text


@pytest.mark.parametrize("chunk", [None, SMALL_CHUNK])
@pytest.mark.parametrize("mode", ["mem", "greedy"])
def test_three_encodings_give_identical_output(kb, golden, tmp_path, monkeypatch, mode, chunk):
    if chunk:
        monkeypatch.setenv("KJ_INGEST_CHUNK", chunk)
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params(mode))
    try:
        t1, t2, ts = gold_text("pe150_1.fq.gz"), gold_text("pe150_2.fq.gz"), gold_text("se100.fq.gz")
        p1, p2, ps = three_ways(tmp_path, "m1", t1), three_ways(tmp_path, "m2", t2, level=1, block=30000), three_ways(tmp_path, "se", ts)
        for verbose in (False, True):
            ref_pe = run(clf, tmp_path / "pe.txt.out", p1["txt"], p2["txt"], verbose); ref_se = run(clf, tmp_path / "se.txt.out", ps["txt"], None, verbose)
            assert ref_pe[0] > 0 and ref_pe[1] > 0 and ref_pe[3] == 0 and ref_se[3] == 0
            for enc, want1, want2 in (("gz", 0, 0), ("bgz", len(t1) + len(t2), len(ts))):
                got = run(clf, tmp_path / ("pe.%s.out" % enc), p1[enc], p2[enc], verbose)
                assert got[:3] == ref_pe[:3] and got[3] == want1, (enc, verbose)
                got = run(clf, tmp_path / ("se.%s.out" % enc), ps[enc], None, verbose)
                assert got[:3] == ref_se[:3] and got[3] == want2, (enc, verbose)
        # one mate blocked, the other plain or ordinary gzip
        for other in ("txt", "gz"):
            got = run(clf, tmp_path / "mixed.out", p1["bgz"], p2[other], True)
            assert got[:3] == ref_pe[:3] and got[3] == len(t1)
    finally:
        clf.close()


def test_fasta_crlf_without_final_newline(clf_mem, golden, tmp_path, monkeypatch):
    monkeypatch.setenv("KJ_INGEST_CHUNK", SMALL_CHUNK)
    names, s1, o1, s2, o2 = golden.reads("se100")
    recs = [b">%s\r\n%s\r\n%s" % (names[i].encode(), s1[int(o1[i]):int(o1[i]) + 60].tobytes(), s1[int(o1[i]) + 60:int(o1[i + 1])].tobytes()) for i in range(len(names))]
    text = b"\r\n".join(recs)
    assert not text.endswith(b"\n")
    p = three_ways(tmp_path, "fa", text, block=5000)
    ref = run(clf_mem, tmp_path / "a.out", p["txt"])
    got = run(clf_mem, tmp_path / "b.out", p["bgz"])
    assert ref[0] == len(names) and got[:3] == ref[:3] and got[3] == len(text) and ref[3] == 0


def test_long_reads_span_many_blocks(kb, golden, tmp_path):
    """Records of 150 kb: one record runs through several blocks and several rounds of the reader."""
    rng = np.random.default_rng(5); names, s1, o1, s2, o2 = golden.reads("pe150")
    short = s1[:int(o1[200])].tobytes()
    recs = []
    for i in range(4):
        seq = bytearray(rng.choice(np.frombuffer(b"ACGT", np.uint8), 150000).tobytes()); seq[1000:1000 + len(short[:30000])] = short[:30000]
        recs.append(b"@long%d\n%s\n+\n%s\n" % (i, bytes(seq), b"I" * len(seq)))
    text = b"".join(recs)
    p = three_ways(tmp_path, "long", text)
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"), max_read_len=200000)
    try:
        ref = run(clf, tmp_path / "a.out", p["txt"]); got = run(clf, tmp_path / "b.out", p["bgz"])
        assert ref[0] == 4 and got[:3] == ref[:3] and got[3] == len(text)
    finally:
        clf.close()


def test_bgzf_followed_by_ordinary_gzip_falls_back_to_zlib(clf_mem, tmp_path, monkeypatch):
    monkeypatch.setenv("KJ_INGEST_CHUNK", SMALL_CHUNK)
    text = gold_text("se100.fq.gz"); cut = text.index(b"\n@", len(text) // 2) + 1
    a, b = text[:cut], text[cut:]
    open(tmp_path / "plain.fq", "wb").write(text)
    open(tmp_path / "cat.fq.gz", "wb").write(ei.bgzf_write(a, 6, block=20000) + gzip.compress(b))
    ref = run(clf_mem, tmp_path / "a.out", str(tmp_path / "plain.fq"))
    got = run(clf_mem, tmp_path / "b.out", str(tmp_path / "cat.fq.gz"))
    assert got[:3] == ref[:3] and got[3] == len(a)           # the blocked part on the device, the rest by zlib


def test_file_of_only_the_end_block(clf_mem, tmp_path):
    """An empty BGZF file.  Through zlib (the path such a file took before the device inflated BGZF) the call returns 0 reads, 0 classified and
    writes an empty output file; so it does now."""
    open(tmp_path / "empty.fq.gz", "wb").write(ei.EOF_BLOCK)
    assert run(clf_mem, tmp_path / "e.out", str(tmp_path / "empty.fq.gz")) == (0, 0, b"", 0)


def test_bad_blocks_are_reported_and_leave_no_state(kb, clf_mem, tmp_path):
    text, bg, bad_files = ei.corrupt_files()
    good = str(tmp_path / "good.fq.gz"); open(good, "wb").write(bg)
    ref = run(clf_mem, tmp_path / "ref.out", good)
    assert ref[0] == 400 and ref[3] == len(text)
    for name, data, offset in bad_files:          # each case once
        path = str(tmp_path / (name + ".fq.gz")); open(path, "wb").write(data)
        with pytest.raises(kb.KaijuError) as e:
            clf_mem.classify_files(path, None, str(tmp_path / "bad.out"))
        msg = str(e.value)
        assert "error -2" in msg and path in msg and ("offset %d" % offset) in msg, (name, msg)
        assert run(clf_mem, tmp_path / "again.out", good) == ref, name


def test_create_run_destroy_returns_memory(kb, golden, tmp_path, monkeypatch):
    """Device and pinned memory of the compressed staging go with the context: free device memory after the fourth cycle is where it was after
    the second (the first loads modules)."""
    torch = pytest.importorskip("torch")
    monkeypatch.setenv("KJ_INGEST_CHUNK", "65536")
    p1, p2 = three_ways(tmp_path, "m1", gold_text("pe150_1.fq.gz")), three_ways(tmp_path, "m2", gold_text("pe150_2.fq.gz"))
    free = []
    for _ in range(4):
        clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"))
        n, k = clf.classify_files(p1["bgz"], p2["bgz"], str(tmp_path / "o.tsv"))
        assert n > 0 and clf.files_device_inflated_bytes > 0
        clf.close()
        torch.cuda.synchronize(); free.append(torch.cuda.mem_get_info()[0])
    assert free[3] >= free[1] - (2 << 20), free
