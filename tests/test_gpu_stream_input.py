"""FASTA/FASTQ input from FIFOs, pipes and standard input in the file pipeline (kj_classify_files, kj_classify_files_multi, kaiju-b200): the output,
the read and classified totals, the per-taxon counts and the bytes the device inflated equal those of the same bytes read from regular files --
plain text, BGZF (still inflated on the device), gzip and multi-member gzip, single and paired, every output format, with the default chunk
and with many small batches.  A single writer that fills both FIFOs of a pair record by record finishes; a call that fails while a writer
stalls returns at once and leaves the context usable.  Writers are threads of this process (or the shell of a CLI run); every one is joined."""
import gzip
import os
import subprocess
import threading
import time

import pytest

import emu_inflate as ei
import emu_stream as es
from conftest import GOLD, ROOT

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "kaiju_b200", "kaiju-b200")
FMI, NODES = os.path.join(GOLD, "db.fmi"), os.path.join(GOLD, "nodes.dmp")
SMALL = "4096"                     # KJ_INGEST_CHUNK: about a hundred batches per golden file


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


@pytest.fixture(scope="module")
def ctxs(kb):
    """mem (with the accessions for OUT_KAIJU_V) and a name-mode context (OUT_NAMES)"""
    c = kb.Classifier(FMI, NODES, device=0, params=kb.make_params("mem"))
    c.set_output_strings(kb.STR_ACCESSION, kb.fmi_accessions(FMI))
    nm = kb.Classifier(FMI, NODES, device=0, params=kb.make_params("mem", name_mode=True))
    nm.set_output_strings(kb.STR_TAXON, [b"t%d" % k for k in range(len(nm.compact_ids()) - 1)])
    yield {"mem": c, "names": nm}
    c.close(); nm.close()


def text_of(name):
    return gzip.open(os.path.join(GOLD, name)).read()


def fasta(fq):
    lines = fq.split(b"\n")
    return b"".join(b">%s\n%s\n" % (lines[i][1:], lines[i + 1]) for i in range(0, len(lines) - 3, 4))


def multi_member(text):
    cuts = [0, 1, len(text) // 3, len(text) // 2, len(text)]
    return b"".join(gzip.compress(text[a:b], 6) for a, b in zip(cuts, cuts[1:]))


ENC = {"plain": lambda t: t, "bgzf1": lambda t: ei.bgzf_write(t, 1), "bgzf6": lambda t: ei.bgzf_write(t, 6, block=30000),
       "gzip1": lambda t: gzip.compress(t, 1), "multi": multi_member}


def timed(fn, timeout=120):
    """fn() on a thread, which must end within timeout seconds: its result, or the exception it raised"""
    res = []
    def body():
        try:
            res.append(("ok", fn()))
        except Exception as e:          # noqa: BLE001 (re-raised below)
            res.append(("err", e))
    t = threading.Thread(target=body, daemon=True); t.start(); t.join(timeout)
    assert not t.is_alive(), "the call did not return within %d s" % timeout
    if res[0][0] == "err":
        raise res[0][1]
    return res[0][1]


def run_files(c, paths, out, fmt):
    c.counts_reset(); n, k = c.classify_files(paths[0], paths[1] if len(paths) > 1 else None, out, fmt=fmt)
    return open(out, "rb").read(), n, k, list(c.counts(nonzero=False)[1]), c.files_device_inflated_bytes


def run_fifos(c, datas, d, tag, fmt, seed=0, call=None):
    """the same through FIFOs fed by writer threads (pauses inside the first record and after 64 KiB)"""
    fifos = []
    for i in range(len(datas)):
        p = os.path.join(d, "%s_%d.fifo" % (tag, i))
        if os.path.exists(p):
            os.unlink(p)
        os.mkfifo(p); fifos.append(p)
    ws = [es.Writer(x, seed + i, path=p, pauses=(20, 65536)) for i, (x, p) in enumerate(zip(datas, fifos))]
    for w in ws:
        w.start()
    try:
        out = os.path.join(d, tag + ".fifo.out")
        return timed(lambda: (call or run_files)(c, fifos, out, fmt))
    finally:
        for w in ws:
            w.finish()


def regular(datas, d, tag):
    paths = []
    for i, x in enumerate(datas):
        p = os.path.join(d, "%s_%d.in" % (tag, i)); open(p, "wb").write(x); paths.append(p)
    return paths


@pytest.mark.parametrize("chunk", [None, SMALL])
def test_streams_equal_files(kb, ctxs, tmp_path, monkeypatch, chunk):
    if chunk:
        monkeypatch.setenv("KJ_INGEST_CHUNK", chunk)
    se, p1, p2 = text_of("se100.fq.gz"), text_of("pe150_1.fq.gz"), text_of("pe150_2.fq.gz")
    inputs = {"se": [se], "pe": [p1, p2], "fasta": [fasta(se)]}
    d = str(tmp_path); checked = 0
    for enc, f in ENC.items():
        for kind, texts in inputs.items():
            fmts = [(kb.OUT_KAIJU, "mem")]
            if kind == "pe" and enc in ("plain", "bgzf6", "gzip1"):
                fmts += [(kb.OUT_KAIJU_IDS, "mem"), (kb.OUT_KAIJU_V, "mem"), (kb.OUT_NAMES, "names")]
            datas = [f(t) for t in texts]
            for fmt, ctx in fmts:
                tag = "%s_%s_%d" % (enc, kind, fmt)
                want = run_files(ctxs[ctx], regular(datas, d, tag), os.path.join(d, tag + ".out"), fmt)
                got = run_fifos(ctxs[ctx], datas, d, tag, fmt, seed=checked)
                assert want[1] > 0 and want[2] > 0 and want[0].count(b"\n") == want[1], tag
                assert got[0] == want[0], tag
                assert got[1:] == want[1:], (tag, got[1:3], want[1:3], got[4], want[4])
                assert want[4] == (sum(len(t) for t in texts) if enc.startswith("bgzf") else 0), tag
                checked += 1
    assert checked == 5 * 3 + 3 * 3


def interleaved(n, long_first):
    """n pairs with 150-base mates in one file and 100-base mates in the other"""
    import numpy as np
    rng = np.random.default_rng(9); p1, p2 = text_of("pe150_1.fq.gz").split(b"\n"), text_of("pe150_2.fq.gz").split(b"\n")
    acgt = np.frombuffer(b"ACGT", np.uint8); a, b = [], []
    for i in range(n):
        k = 4 * (i % (len(p1) // 4))
        s1 = p1[k + 1][:150] if i % 3 else rng.choice(acgt, 150).tobytes(); s2 = p2[k + 1][:100]
        if not long_first:
            s1, s2 = p1[k + 1][:100], p2[k + 1][:150]
        a.append(b"@pair%d/1\n%s\n+\n%s\n" % (i, s1, b"I" * len(s1))); b.append(b"@pair%d/2\n%s\n+\n%s\n" % (i, s2, b"I" * len(s2)))
    return a, b


class PairWriter(threading.Thread):
    """One writer for both FIFOs of a pair: opens file 2 first, then writes the records alternately, one mate to each FIFO."""
    def __init__(self, f1, f2, r1, r2):
        super().__init__(daemon=True); self.f1, self.f2, self.r1, self.r2 = f1, f2, r1, r2; self.error = None

    def run(self):
        try:
            fd2 = os.open(self.f2, os.O_WRONLY); fd1 = os.open(self.f1, os.O_WRONLY)
            try:
                for a, b in zip(self.r1, self.r2):
                    for fd, x in ((fd1, a), (fd2, b)):
                        mv = memoryview(x)
                        while len(mv):
                            mv = mv[os.write(fd, mv):]
            finally:
                os.close(fd1); os.close(fd2)
        except Exception as e:          # noqa: BLE001 (checked by the test)
            self.error = e


@pytest.mark.parametrize("chunk,long_first", [(None, True), (SMALL, True), (SMALL, False)])
def test_one_writer_interleaves_both_fifos(ctxs, tmp_path, monkeypatch, chunk, long_first):
    if chunk:
        monkeypatch.setenv("KJ_INGEST_CHUNK", chunk)
    c = ctxs["mem"]; d = str(tmp_path)
    r1, r2 = interleaved(30000, long_first)
    want = run_files(c, regular([b"".join(r1), b"".join(r2)], d, "ref"), d + "/ref.out", 0)
    f1, f2 = d + "/a.fifo", d + "/b.fifo"; os.mkfifo(f1); os.mkfifo(f2)
    w = PairWriter(f1, f2, r1, r2); w.start()
    try:
        got = timed(lambda: run_files(c, [f1, f2], d + "/got.out", 0), timeout=180)
    finally:
        w.join(60)
    assert not w.is_alive() and w.error is None, w.error
    assert want[1] == 30000 and got == want


def test_files_multi_two_contexts_on_one_device(kb, ctxs, tmp_path, monkeypatch):
    monkeypatch.setenv("KJ_INGEST_CHUNK", SMALL)
    other = kb.Classifier(FMI, NODES, device=0, params=kb.make_params("mem"))
    try:
        other.set_output_strings(kb.STR_ACCESSION, kb.fmi_accessions(FMI))
        c = ctxs["mem"]; d = str(tmp_path)
        def multi(_, paths, out, fmt):
            for x in (c, other):
                x.counts_reset()
            n, k = kb.classify_files_multi([c, other], paths[0], paths[1], out, fmt=fmt)
            return open(out, "rb").read(), n, k, list(c.counts(nonzero=False)[1] + other.counts(nonzero=False)[1]), c.files_device_inflated_bytes
        for enc in ("plain", "bgzf6"):
            datas = [ENC[enc](text_of("pe150_1.fq.gz")), ENC[enc](text_of("pe150_2.fq.gz"))]
            want = run_files(c, regular(datas, d, enc), d + "/%s.out" % enc, kb.OUT_KAIJU_V)
            got = run_fifos(None, datas, d, enc + "_multi", kb.OUT_KAIJU_V, call=multi)
            assert got == want, enc
    finally:
        other.close()


def cli(args, env=None, **kw):
    e = dict(os.environ); e.update(env or {})
    p = subprocess.run(args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e, timeout=180, **kw)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    return p.stdout


def test_cli_stdin_process_substitution_and_fifo_lists(built, tmp_path):
    d = str(tmp_path); base = [CLI, "-t", NODES, "-f", FMI, "-a", "mem", "-v"]
    se, p1, p2 = text_of("se100.fq.gz"), text_of("pe150_1.fq.gz"), text_of("pe150_2.fq.gz")
    fse, f1, f2 = regular([se, p1, p2], d, "cli")
    want_se = cli(base + ["-i", fse]); want_pe = cli(base + ["-i", f1, "-j", f2])
    assert want_se.count(b"\n") > 100 and want_pe.count(b"\n") > 100
    for data in (se, gzip.compress(se, 1), ei.bgzf_write(se, 6)):
        assert cli(base + ["-i", "/dev/stdin"], input=data) == want_se
    sh = "exec %s -i <(cat %s) -j <(cat %s) -o /dev/stdout" % (" ".join(base), f1, f2)
    assert cli(["bash", "-c", sh]) == want_pe
    # a list of two data sets, every input a FIFO, with many small batches
    fifos = [d + "/%s.fifo" % n for n in ("a1", "b1", "a2", "b2")]
    for p in fifos:
        os.mkfifo(p)
    datas = [p1, p2, ei.bgzf_write(p1, 1), gzip.compress(p2, 1)]
    ws = [es.Writer(x, i, path=p, pauses=(100,)) for i, (x, p) in enumerate(zip(datas, fifos))]
    for w in ws:
        w.start()
    try:
        cli(base + ["-i", fifos[0] + "," + fifos[2], "-j", fifos[1] + "," + fifos[3], "-o", d + "/o1.tsv," + d + "/o2.tsv"], {"KJ_INGEST_CHUNK": SMALL})
    finally:
        for w in ws:
            w.finish()
    assert open(d + "/o1.tsv", "rb").read() == want_pe and open(d + "/o2.tsv", "rb").read() == want_pe


def threads():
    return len(os.listdir("/proc/self/task"))


def test_errors_return_promptly_and_leave_the_context_usable(kb, ctxs, tmp_path, monkeypatch):
    monkeypatch.setenv("KJ_INGEST_CHUNK", SMALL)
    c = ctxs["mem"]; d = str(tmp_path)
    p1, p2 = text_of("pe150_1.fq.gz"), text_of("pe150_2.fq.gz")
    good = regular([p1, p2], d, "good")
    want = run_files(c, good, d + "/good.out", 0)
    assert run_fifos(c, [p1, p2], d, "warm", 0) == want
    base_threads = threads()
    recs2 = p2.split(b"\n")
    bad_names = p2.replace(b"@r300/2\n", b"@q300/2\n", 1)
    second = p1.index(b"\n@", 1) + 1; bad_header = p1[:second] + b"#" + p1[second + 1:]
    _, bg, bad_files = ei.corrupt_files()
    flipped, flipped_at = [(x, o) for n, x, o in bad_files if n == "flipped_bit"][0]
    # file 1 as BGZF with a damaged block about 240 kB into its text, which its reader meets while the parser waits for file 2
    late = bytearray(ei.bgzf_write(p1, 6, block=20000)); late_at = list(ei._block_ends(bytes(late)))[11]; late[late_at + 18 + 300] ^= 0x10
    assert bad_names != p2
    cases = [("more_reads", [p1, b"\n".join(recs2[:4 * 500]) + b"\n"], None, "contains more reads then file"),
             ("names", [p1, bad_names], None, "Read names are not identical"),
             ("bad_block", [flipped], None, "at compressed offset %d" % flipped_at),
             # file 1 is a corrupt BGZF stream; file 2's writer has written nothing, or part of its file, and keeps its FIFO open
             ("stall_empty", [flipped, b""], 60, "at compressed offset %d" % flipped_at),
             ("stall_part", [flipped, p2[:200000]], 60, "at compressed offset %d" % flipped_at),
             ("stall_late", [bytes(late), p2[:200000]], 60, "at compressed offset %d" % late_at),
             # file 1 is malformed text that the parser rejects once both sides have their first batch; file 2 stalls after 200 kB
             ("stall_parse", [bad_header, p2[:200000]], 60, "malformed FASTQ record")]
    for tag, datas, stall, msg in cases:
        fifos = []
        for i in range(len(datas)):
            p = "%s/%s_%d.fifo" % (d, tag, i); os.mkfifo(p); fifos.append(p)
        ws = [es.Writer(x, i, path=p, stall=stall if (stall and i == 1) else 0.0) for i, (x, p) in enumerate(zip(datas, fifos))]
        for w in ws:
            w.start()
        try:
            t0 = time.monotonic()
            with pytest.raises(kb.KaijuError) as e:
                timed(lambda: c.classify_files(fifos[0], fifos[1] if len(fifos) > 1 else None, d + "/bad.out"), timeout=30)
            assert "error -2" in str(e.value) and msg in str(e.value), (tag, str(e.value))
            assert time.monotonic() - t0 < 10, tag            # did not wait for the stalled writer (which holds its FIFO open for 60 s)
        finally:
            for w in ws:
                w.finish()
        assert threads() <= base_threads, tag
        assert run_files(c, good, d + "/again.out", 0) == want, tag
