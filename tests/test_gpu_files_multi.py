"""One input classified by several contexts (kj_classify_files_multi, kaiju_b200.classify_files_multi, kaiju-b200 -d 0,0 [-P] with fewer data
sets than devices): the output equals what one context writes, byte for byte, and the committed reference outputs where they exist; the read
and classified totals equal one context's; the contexts' count vectors sum to one context's.  On one GPU the contexts share device 0; on a
machine with two GPUs with peer access, the same holds across them."""
import ctypes as C
import gzip, os, random, re, subprocess
import numpy as np
import pytest
from conftest import ROOT, GOLD
from helpers import SynthDB
from emu_inflate import bgzf_write

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "kaiju_b200", "kaiju-b200")
FMI, NODES = os.path.join(GOLD, "db.fmi"), os.path.join(GOLD, "nodes.dmp")
PARAMS = {"mem_default": dict(mode="mem"), "greedy_default": dict(mode="greedy")}
XP = {"mem_default": ["-a", "mem"], "greedy_default": ["-a", "greedy", "-e", "3", "-s", "65"]}
TOPOLOGY = {"replicas_00": ("replicas", [0, 0]), "group_00": ("group", [0, 0]), "replicas_000": ("replicas", [0, 0, 0])}
SMALL = {"KJ_INGEST_CHUNK": "4096"}          # about a hundred batches per golden file: every context takes some


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


def expected(name):
    return gzip.open(os.path.join(GOLD, name), "rb").read().decode()


def same(got, want):
    assert got == want, [(a, b) for a, b in zip(got.split("\n"), want.split("\n")) if a != b][:3]


def inputs(d, tag, enc):
    """the golden reads as plain text, as they are (zlib gzip) or re-compressed as BGZF"""
    names = ["se100.fq.gz"] if tag == "se100" else ["pe150_1.fq.gz", "pe150_2.fq.gz"]
    out = []
    for k, nm in enumerate(names):
        src = os.path.join(GOLD, nm)
        if enc == "gzip":
            out.append(src)
        else:
            data = gzip.open(src, "rb").read(); dst = "%s/%s_%d%s" % (d, enc, k, ".fq.gz" if enc == "bgzf" else ".fq")
            open(dst, "wb").write(bgzf_write(data, 6) if enc == "bgzf" else data)
            out.append(dst)
    return out + [None] * (2 - len(out))


def contexts(kb, kind, devices, cfg, **kw):
    p = kb.make_params(**PARAMS[cfg])
    cs = kb.create_group(FMI, NODES, devices, params=p, **kw) if kind == "group" else [kb.Classifier(FMI, NODES, device=d, params=p, **kw) for d in devices]
    accs = kb.fmi_accessions(FMI)
    for c in cs:
        c.set_output_strings(kb.STR_ACCESSION, accs)
    return cs


def close(cs):
    for c in cs:
        c.close()


def one(kb, c, a, b, out, fmt):
    """kj_classify_files on one context: (text, reads, classified, counts)"""
    c.counts_reset(); n, k = c.classify_files(a, b, out, fmt=fmt)
    return open(out).read(), n, k, c.counts(nonzero=False)[1]


def multi(kb, cs, a, b, out, fmt):
    """kj_classify_files_multi: (text, reads, classified, the element-wise sum of the contexts' counts)"""
    for c in cs:
        c.counts_reset()
    n, k = kb.classify_files_multi(cs, a, b, out, fmt=fmt)
    ids = [c.counts(nonzero=False)[0] for c in cs]
    assert all(np.array_equal(x, ids[0]) for x in ids)
    return open(out).read(), n, k, sum(c.counts(nonzero=False)[1] for c in cs)


def check_equal(kb, cs, a, b, d, fmt, want_text=None):
    want = one(kb, cs[0], a, b, d + "/one.tsv", fmt)
    got = multi(kb, cs, a, b, d + "/multi.tsv", fmt)
    same(got[0], want[0])
    if want_text is not None:
        same(got[0], want_text)
    assert got[1:3] == want[1:3] and want[1] > 0
    assert np.array_equal(got[3], want[3]) and int(got[3].sum()) == want[1]
    return got


def _equal_on_golden(kb, monkeypatch, tmp_path, kind, devices, cfg):
    for k, v in SMALL.items():
        monkeypatch.setenv(k, v)
    d = str(tmp_path); cs = contexts(kb, kind, devices, cfg)
    try:
        for tag in ("se100", "pe150"):
            for enc in ("plain", "gzip", "bgzf"):
                a, b = inputs(d, tag, enc)
                for fmt in (kb.OUT_KAIJU, kb.OUT_KAIJU_IDS, kb.OUT_KAIJU_V):
                    check_equal(kb, cs, a, b, d, fmt, expected("expected_v7_%s_%s.tsv.gz" % (cfg, tag)) if fmt == kb.OUT_KAIJU_V else None)
    finally:
        close(cs)


@pytest.mark.parametrize("cfg", sorted(PARAMS))
@pytest.mark.parametrize("topology", sorted(TOPOLOGY))
def test_taxon_formats_equal_one_context(kb, monkeypatch, tmp_path, topology, cfg):
    """formats 0-2 on SE100 and PE150, plain / zlib gzip / BGZF: == one context, and format 2 == `kaiju -v`"""
    kind, devices = TOPOLOGY[topology]
    _equal_on_golden(kb, monkeypatch, tmp_path, kind, devices, cfg)


def cli(args, env=None, check=True):
    e = dict(os.environ); e.update(env or {})
    p = subprocess.run([CLI] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e)
    if check:
        assert p.returncode == 0, p.stderr.decode()
    return p


@pytest.mark.parametrize("devices", ["0,0", "0,0,0"])
def test_name_formats_equal_reference(built, tmp_path, devices):
    """formats 3 and 4 (kaijux, kaijux -v, kaijup, kaijup -v) through the CLI over replicas: == the reference's outputs"""
    d = str(tmp_path)
    for cfg in sorted(XP):
        for tag, enc in (("se100", "bgzf"), ("pe150", "plain")):
            a, b = inputs(d, tag, enc); i = ["-i", a] + (["-j", b] if b else [])
            for v, kind in (([], "x"), (["-v"], "xv")):
                same(cli(["-d", devices, "-M", "kaijux", "-f", FMI] + v + i + XP[cfg], SMALL).stdout.decode(), expected("expected_%s_%s_%s.tsv.gz" % (kind, cfg, tag)))
        for v, kind in (([], "p"), (["-v"], "pv")):
            same(cli(["-d", devices, "-M", "kaijup", "-f", FMI, "-i", os.path.join(GOLD, "prot.fa.gz")] + v + XP[cfg], SMALL).stdout.decode(), expected("expected_%s_%s.tsv.gz" % (kind, cfg)))


def _trace(stderr):
    m = re.search(r"KJ_FILES_TRACE contexts (\d+)  batches per context ([\d,]+)  writer held back at most (\d+)", stderr)
    assert m, stderr
    return [int(x) for x in m.group(2).split(",")], int(m.group(3))


@pytest.mark.parametrize("devices", ["0,0", "0,0,0"])
def test_out_of_order_batches_are_written_in_order(built, tmp_path, devices):
    """many small batches while ctxs[0] formats late (KJ_FILES_HOLD_MS): later batches complete first on the other contexts, the writer holds
    them back, and the output is unchanged"""
    d = str(tmp_path); a, b = inputs(d, "pe150", "plain")
    base = ["-v", "-t", NODES, "-f", FMI, "-i", a, "-j", b] + XP["greedy_default"]
    p = cli(["-d", devices] + base, dict(SMALL, KJ_FILES_TRACE="1", KJ_FILES_HOLD_MS="30"))
    same(p.stdout.decode(), expected("expected_v7_greedy_default_pe150.tsv.gz"))
    per, held = _trace(p.stderr.decode())
    assert len(per) == devices.count("0") and all(x > 0 for x in per) and sum(per) > 50, per
    assert held >= 1


def test_several_launches_per_batch(built, tmp_path):
    """formats 2 and 4 with a fragment-string budget of a few reads: every context classifies and formats each batch in several launches"""
    d = str(tmp_path); a, b = inputs(d, "pe150", "plain"); env = {"KJ_INGEST_CHUNK": "20000", "KJ_INGEST_BATCH": "60000", "KJ_FRAG_BUDGET": "50000", "KJ_FILES_TRACE": "1"}
    for cfg in sorted(XP):
        p = cli(["-d", "0,0", "-v", "-t", NODES, "-f", FMI, "-i", a, "-j", b] + XP[cfg], env)
        same(p.stdout.decode(), expected("expected_v7_%s_pe150.tsv.gz" % cfg))
        assert all(x > 0 for x in _trace(p.stderr.decode())[0])
        p = cli(["-d", "0,0,0", "-M", "kaijux", "-v", "-f", FMI, "-i", a, "-j", b] + XP[cfg], env)
        same(p.stdout.decode(), expected("expected_xv_%s_pe150.tsv.gz" % cfg))


def test_long_and_short_reads_mixed(kb, monkeypatch, tmp_path):
    """20-60 kb reads among short ones, with the read-length limit raised on every context: == one context, in MEM and Greedy"""
    db = SynthDB(800, 3); s, o = db.long_reads(91, 0, 12, 20000, 60000); sh, oh = db.long_reads(92, 0, 200, 100, 400)
    reads = [bytes(s[int(o[i]):int(o[i + 1])]).decode() for i in range(12)] + [bytes(sh[int(oh[i]):int(oh[i + 1])]).decode() for i in range(200)]
    random.Random(3).shuffle(reads)
    d = str(tmp_path); fq = d + "/l.fq"
    open(fq, "w").write("".join("@l%d\n%s\n+\n%s\n" % (i, r, "I" * len(r)) for i, r in enumerate(reads)))
    monkeypatch.setenv("KJ_INGEST_CHUNK", "65536")
    for cfg in sorted(PARAMS):
        cs = contexts(kb, "replicas", [0, 0], cfg, max_read_len=100000)
        try:
            for fmt in (kb.OUT_KAIJU_IDS, kb.OUT_KAIJU_V):
                check_equal(kb, cs, fq, None, d, fmt)
        finally:
            close(cs)


def test_errors_leave_the_contexts_usable(kb, monkeypatch, tmp_path):
    """every failure is reported once, prefixed with the device, and the same contexts then classify correctly"""
    d = str(tmp_path); a, b = inputs(d, "pe150", "plain"); want = expected("expected_v7_mem_default_pe150.tsv.gz")
    monkeypatch.setenv("KJ_INGEST_CHUNK", "4096")
    cs = contexts(kb, "replicas", [0, 0], "mem_default")

    def good():
        check_equal(kb, cs, a, b, d, kb.OUT_KAIJU_V, want)

    def fails(code, msg, *args, **kw):
        with pytest.raises(kb.KaijuError) as e:
            kb.classify_files_multi(cs, *args, **kw)
        assert ("error %d:" % code) in str(e.value) and msg in str(e.value), str(e.value)
        return str(e.value)

    try:
        good()
        # paired files whose names differ in the middle of the file
        lines = open(b).read().split("\n"); lines[4 * 1000] = "@renamed"; open(d + "/b_bad.fq", "w").write("\n".join(lines))
        m = fails(-2, "Read names are not identical between the two input files", a, d + "/b_bad.fq", d + "/x.tsv", fmt=kb.OUT_KAIJU_V)
        assert "device 0: " in m
        good()
        # a read over the limit
        r = "ACGT" * 5000; open(d + "/long.fq", "w").write(open(a).read() + "@long\n%s\n+\n%s\n" % (r, "I" * len(r)))
        fails(-5, "read longer than", d + "/long.fq", None, d + "/x.tsv")
        good()
        # fragment strings larger than the stride
        monkeypatch.setenv("KJ_FRAG_STRIDE", "16")
        fails(-6, "exceed frag_stride", a, b, d + "/x.tsv", fmt=kb.OUT_KAIJU_V)
        monkeypatch.delenv("KJ_FRAG_STRIDE")
        good()
        # argument checks, before any file is opened
        L = kb.lib(); arr = lambda xs: (C.c_void_p * max(1, len(xs)))(*[x._ctx for x in xs])
        for xs, n in ((cs, 0), ([cs[0]] * 9, 9)):
            assert L.kj_classify_files_multi(arr(xs), n, a.encode(), None, (d + "/arg.tsv").encode(), 0, None, None) == -1
        assert L.kj_classify_files_multi(arr(cs), 2, None, None, (d + "/arg.tsv").encode(), 0, None, None) == -1
        with pytest.raises(kb.KaijuError, match="listed twice"):
            kb.classify_files_multi([cs[0], cs[1], cs[0]], a, b, d + "/arg.tsv")
        other = kb.Classifier(FMI, NODES, device=0, params=kb.make_params("greedy"))
        try:
            with pytest.raises(kb.KaijuError, match="other kj_params"):
                kb.classify_files_multi(cs + [other], a, b, d + "/arg.tsv")
            other.set_params(kb.make_params("mem")); other.set_max_read_len(20000)
            with pytest.raises(kb.KaijuError, match="read-length limit"):
                kb.classify_files_multi(cs + [other], a, b, d + "/arg.tsv")
            with pytest.raises(kb.KaijuError, match="KJ_STR_ACCESSION"):      # the accession table is missing on the last context only
                other.set_max_read_len(kb.MAX_READ_LEN); kb.classify_files_multi(cs + [other], a, b, d + "/arg.tsv", fmt=kb.OUT_KAIJU_V)
            with pytest.raises(kb.KaijuError, match="name_mode"):
                kb.classify_files_multi(cs + [other], a, b, d + "/arg.tsv", fmt=kb.OUT_NAMES)
        finally:
            other.close()
        scaled = kb.Classifier(FMI, NODES, device=0, params=kb.make_params("mem"), copies=2)
        try:
            with pytest.raises(kb.KaijuError, match="another index"):
                kb.classify_files_multi(cs + [scaled], a, b, d + "/arg.tsv")
        finally:
            scaled.close()
        assert not os.path.exists(d + "/arg.tsv")
        good()
    finally:
        close(cs)


def _names_dmp(d):
    with open(d + "/names.dmp", "w") as f:
        for line in open(NODES):
            nid = line.split("\t|\t")[0].strip()
            f.write("%s\t|\ttaxon %s\t|\t\t|\tscientific name\t|\n" % (nid, nid))
    return d + "/names.dmp"


def test_cli_one_data_set_on_several_contexts(built, tmp_path):
    """-d 0,0 and -d 0,0 -P with one data set write the output and the -T table of -d 0 byte for byte; three data sets on -d 0,0,0,0 (fewer
    data sets than contexts) write each set's output and the table of -d 0"""
    d = str(tmp_path); names = _names_dmp(d); a, b = inputs(d, "pe150", "plain")
    base = ["-t", NODES, "-f", FMI, "-N", names, "-v"] + XP["greedy_default"]
    for tag, dev in (("one", ["-d", "0"]), ("rep", ["-d", "0,0"]), ("pool", ["-d", "0,0", "-P"])):
        cli(base + dev + ["-i", a, "-j", b, "-o", "%s/%s.tsv" % (d, tag), "-T", "%s/%s.table" % (d, tag)], SMALL)
    for ext in ("tsv", "table"):      # (the table's file column is the output file's name)
        want = open("%s/one.%s" % (d, ext)).read().replace(d + "/one.tsv", "OUT")
        for tag in ("rep", "pool"):
            assert open("%s/%s.%s" % (d, tag, ext)).read().replace("%s/%s.tsv" % (d, tag), "OUT") == want and len(want) > 100, (tag, ext)
    sets = [inputs(d, "se100", "plain")[0], os.path.join(GOLD, "se100.fq.gz"), a]
    for tag, dev in (("one", "0"), ("four", "0,0,0,0")):
        outs = ",".join("%s/%s_%d.tsv" % (d, tag, k) for k in range(3))
        cli(["-d", dev, "-t", NODES, "-f", FMI, "-N", names, "-i", ",".join(sets), "-o", outs, "-T", "%s/%s.table" % (d, tag)] + XP["mem_default"], SMALL)
    for k in range(3):
        assert open("%s/four_%d.tsv" % (d, k)).read() == open("%s/one_%d.tsv" % (d, k)).read()
    t1 = open(d + "/one.table").read(); t4 = open(d + "/four.table").read()
    for k in range(3):
        t1 = t1.replace("%s/one_%d.tsv" % (d, k), "OUT%d" % k); t4 = t4.replace("%s/four_%d.tsv" % (d, k), "OUT%d" % k)
    assert t1 == t4 and len(t1) > 100


def _peers(kb, n):
    import torch
    if kb.device_count() < n:
        pytest.skip("needs %d GPUs" % n)
    for x in range(n):
        for y in range(n):
            if x != y and not torch.cuda.can_device_access_peer(x, y):
                pytest.skip("GPUs %d and %d have no peer access" % (x, y))
    return list(range(n))


@pytest.mark.parametrize("kind", ["replicas", "group"])
def test_two_gpus(kb, monkeypatch, tmp_path, kind):
    """replicas [0, 1] and a group [0, 1]: as on one GPU"""
    devices = _peers(kb, 2)
    for cfg in sorted(PARAMS):
        _equal_on_golden(kb, monkeypatch, tmp_path, kind, devices, cfg)
