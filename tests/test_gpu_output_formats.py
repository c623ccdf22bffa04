"""Every output format of the file pipeline on the device (kj_classify_files KJ_OUT_KAIJU_V / KJ_OUT_NAMES / KJ_OUT_NAMES_V), byte for byte against
the reference: `kaijux -v` / `kaijup -v` against the committed outputs of tests/golden/make_golden_xv.py, BGZF input, batch and launch
boundaries, kaijup's reader rules, long reads, a tiered context and the errors."""
import gzip, os, random, shutil, subprocess
import pytest
from conftest import ROOT, GOLD
from helpers import SynthDB, REF_DIR, have_ref
from emu_inflate import bgzf_write

pytestmark = pytest.mark.gpu
XP = {"mem_default": ["-a", "mem"], "mem_m5_noseg": ["-a", "mem", "-m", "5", "-X"], "greedy_default": ["-a", "greedy", "-e", "3", "-s", "65"],
      "greedy_e5_s40": ["-a", "greedy", "-e", "5", "-s", "40"], "greedy_e0": ["-a", "greedy", "-e", "0"]}
CLI = os.path.join(ROOT, "kaiju_b200", "kaiju-b200")
FMI, NODES = os.path.join(GOLD, "db.fmi"), os.path.join(GOLD, "nodes.dmp")


def unz(src, dst):
    with gzip.open(src, "rb") as f, open(dst, "wb") as g:
        shutil.copyfileobj(f, g)
    return dst


def bgzf(src, dst):
    with gzip.open(src, "rb") as f:
        data = f.read()
    open(dst, "wb").write(bgzf_write(data, 6))
    return dst


def expected(name):
    return gzip.open(os.path.join(GOLD, name), "rb").read().decode()


def cli(args, env=None, check=True):
    e = dict(os.environ); e.update(env or {})
    p = subprocess.run([CLI] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e)
    if check:
        assert p.returncode == 0, p.stderr.decode()
    return p


def same(got, want):
    assert got == want, [(a, b) for a, b in zip(got.split("\n"), want.split("\n")) if a != b][:3]


def inputs(tag, d, enc=None):
    conv = (lambda s, n: bgzf(s, d + "/" + n + ".gz")) if enc == "bgzf" else (lambda s, n: unz(s, d + "/" + n))
    if tag == "se100":
        return ["-i", conv(GOLD + "/se100.fq.gz", "se.fq")]
    return ["-i", conv(GOLD + "/pe150_1.fq.gz", "a.fq"), "-j", conv(GOLD + "/pe150_2.fq.gz", "b.fq")]


@pytest.mark.parametrize("cfg", sorted(XP))
@pytest.mark.parametrize("tag", ["se100", "pe150"])
def test_kaijux_v_equals_reference(built, tmp_path, cfg, tag):
    out = cli(["-M", "kaijux", "-v", "-f", FMI] + inputs(tag, str(tmp_path)) + XP[cfg]).stdout.decode()
    want = expected("expected_xv_%s_%s.tsv.gz" % (cfg, tag))
    same(out, want)
    assert want.count("\nC\t") > 500


@pytest.mark.parametrize("cfg", sorted(XP))
def test_kaijup_v_equals_reference(built, tmp_path, cfg):
    cli(["-M", "kaijup", "-v", "-f", FMI, "-i", os.path.join(GOLD, "prot.fa.gz"), "-o", str(tmp_path / "o.tsv")] + XP[cfg])
    same(open(str(tmp_path / "o.tsv")).read(), expected("expected_pv_%s.tsv.gz" % cfg))


def _inflated(p):
    return int([l for l in p.stderr.decode().splitlines() if "inflated on the device" in l][0].split(": ")[1].split()[0])


@pytest.mark.parametrize("what", ["kaiju_v", "kaijux", "kaijup_v"])
def test_bgzf_input_is_inflated_on_the_device(built, tmp_path, what):
    d = str(tmp_path); env = {"KJ_CLI_TIMING": "1"}
    if what == "kaiju_v":
        p = cli(["-v", "-t", NODES, "-f", FMI] + inputs("pe150", d, "bgzf") + XP["greedy_default"], env); want = expected("expected_v7_greedy_default_pe150.tsv.gz")
    elif what == "kaijux":
        p = cli(["-M", "kaijux", "-f", FMI] + inputs("pe150", d, "bgzf") + XP["mem_default"], env); want = expected("expected_x_mem_default_pe150.tsv.gz")
    else:
        p = cli(["-M", "kaijup", "-v", "-f", FMI, "-i", bgzf(GOLD + "/prot.fa.gz", d + "/p.fa.gz")] + XP["greedy_e5_s40"], env); want = expected("expected_pv_greedy_e5_s40.tsv.gz")
    same(p.stdout.decode(), want)
    assert _inflated(p) > 0


@pytest.mark.parametrize("what", ["kaiju_v_mem", "kaiju_v_greedy", "kaijux_v", "kaijup_v"])
def test_batch_and_launch_boundaries(built, tmp_path, what):
    """Many small batches (KJ_INGEST_CHUNK / KJ_INGEST_BATCH) and a fragment-string budget of a few reads, so that every batch is classified
    in several launches and formatted in input order."""
    d = str(tmp_path); env = {"KJ_INGEST_CHUNK": "20000", "KJ_INGEST_BATCH": "60000", "KJ_FRAG_BUDGET": "300000"}
    if what.startswith("kaiju_v"):
        cfg = "mem_default" if what.endswith("mem") else "greedy_default"
        p = cli(["-v", "-t", NODES, "-f", FMI] + inputs("pe150", d) + XP[cfg], env); want = expected("expected_v7_%s_pe150.tsv.gz" % cfg)
    elif what == "kaijux_v":
        p = cli(["-M", "kaijux", "-v", "-f", FMI] + inputs("se100", d) + XP["greedy_e5_s40"], env); want = expected("expected_xv_greedy_e5_s40_se100.tsv.gz")
    else:
        p = cli(["-M", "kaijup", "-v", "-f", FMI, "-i", os.path.join(GOLD, "prot.fa.gz")] + XP["mem_m5_noseg"], env); want = expected("expected_pv_mem_m5_noseg.tsv.gz")
    same(p.stdout.decode(), want)


def _protein_reads(seed):
    db = SynthDB(800, 3); s, o = db.protein_reads(seed, 0, 300, 5, 300)
    return [bytes(s[int(o[i]):int(o[i + 1])]).decode() for i in range(300)]


def _kaijup_inputs(d):
    """Reader corner cases for kaijup: names with spaces, tabs and '/', reads without a fragment of length m next to reads that match nothing,
    lower case, FASTA with blank lines inside a sequence, CRLF headers; and a FASTQ protein file."""
    rng = random.Random(5); reads = _protein_reads(77); fa = []
    for i, r in enumerate(reads):
        name = ["q%d" % i, "q%d with spaces" % i, "q%d\twith\ttabs" % i, "q%d/1" % i, "q%d /2\tx" % i][i % 5]
        if i % 7 == 3:
            r = "XX".join("ACDEFGHIK"[: rng.randint(1, 9)] for _ in range(rng.randint(1, 6)))        # only pieces shorter than m: gated
        elif i % 7 == 5:
            r = "".join(rng.choice("ACDEFGHIKLMNPQRSTVWY") for _ in range(rng.randint(20, 80)))      # passes the gate, matches nothing
        elif i % 7 == 6:
            r = r.lower()
        if i % 4 == 1 and len(r) > 10:
            fa.append(">%s\n%s\n\n%s\n" % (name, r[:len(r) // 2], r[len(r) // 2:]))
        elif i % 9 == 2:
            fa.append(">%s\r\n%s\n" % (name, r))
        else:
            fa.append(">%s\n%s\n" % (name, r))
    open(d + "/p.fa", "w").write("".join(fa))
    open(d + "/p.fq", "w").write("".join("@%s\n%s\n+\n%s\n" % (["p%d x" % i, "p%d\t/y" % i][i % 2], r, "I" * len(r)) for i, r in enumerate(reads[:150])))
    return [d + "/p.fa", d + "/p.fq"]


@pytest.mark.parametrize("cfg", ["mem_default", "greedy_default", "greedy_e5_s40"])
def test_kaijup_reader_corner_cases_equal_reference(built, tmp_path, cfg):
    if not have_ref():
        pytest.skip("oracle/_ref (reference binary) not available")
    for f in _kaijup_inputs(str(tmp_path)):
        for v in ([], ["-v"]):
            want = subprocess.run([os.path.join(REF_DIR, "kaijup"), "-f", FMI, "-z", "1", "-i", f] + v + XP[cfg], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True).stdout.decode()
            got = cli(["-M", "kaijup", "-f", FMI, "-i", f] + v + XP[cfg]).stdout.decode()
            same(got, want)
            if f.endswith(".fa"):       # both kinds of unclassified line occur
                lines = got.splitlines()
                assert any(l.startswith("U\t") and l.endswith("\t0") for l in lines) and any(l.startswith("U\t") and not l.endswith("\t0") for l in lines)


def test_long_reads_verbose_equal_reference(built, tmp_path):
    """-v -L 100000 on 20-60 kb reads mixed with short ones: all seven columns equal `kaiju -v`."""
    if not have_ref():
        pytest.skip("oracle/_ref (reference binary) not available")
    db = SynthDB(800, 3); s, o = db.long_reads(91, 0, 12, 20000, 60000); sh, oh = db.long_reads(92, 0, 60, 100, 400)
    reads = [bytes(s[int(o[i]):int(o[i + 1])]).decode() for i in range(12)] + [bytes(sh[int(oh[i]):int(oh[i + 1])]).decode() for i in range(60)]
    random.Random(3).shuffle(reads)
    fq = str(tmp_path / "l.fq")
    open(fq, "w").write("".join("@l%d\n%s\n+\n%s\n" % (i, r, "I" * len(r)) for i, r in enumerate(reads)))
    for cfg in ("mem_default", "greedy_default"):
        want = subprocess.run([os.path.join(REF_DIR, "kaiju"), "-t", NODES, "-f", FMI, "-z", "1", "-v", "-i", fq] + XP[cfg], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True).stdout.decode()
        same(cli(["-v", "-L", "100000", "-t", NODES, "-f", FMI, "-i", fq] + XP[cfg]).stdout.decode(), want)


def test_tiered_context_prints_the_same_verbose_output(built, tmp_path, monkeypatch):
    """A context whose suffix-array arrays and part of its records are in the host tier: the same seven columns, and the accession table is
    counted in the host bytes."""
    import kaiju_b200 as kb
    d = str(tmp_path); i = inputs("pe150", d)
    monkeypatch.setenv("KJ_FORCE_COMPACT", "1"); monkeypatch.setenv("KJ_TIER_DEVICE_RECORDS", "3")
    c = kb.Classifier(FMI, NODES, device=0, params=kb.make_params("mem"), host_memory=1 << 30)
    monkeypatch.delenv("KJ_TIER_DEVICE_RECORDS")
    assert lib_layout(kb, c) == 3
    h0, d0 = int(kb.lib().kj_index_host_bytes(c._ctx)), int(kb.lib().kj_index_bytes(c._ctx))
    accs = kb.fmi_accessions(FMI)
    c.set_output_strings(kb.STR_ACCESSION, accs)
    table = sum(len(a) for a in accs)
    assert int(kb.lib().kj_index_host_bytes(c._ctx)) - h0 == max(table, 16) + 8 * (len(accs) + 1)
    assert int(kb.lib().kj_index_bytes(c._ctx)) == d0
    n, k = c.classify_files(i[1], i[3], d + "/o.tsv", fmt=kb.OUT_KAIJU_V)
    want = expected("expected_v7_mem_default_pe150.tsv.gz")
    same(open(d + "/o.tsv").read(), want)
    assert k == sum(l.startswith("C\t") for l in want.splitlines()) and n == want.count("\n")
    c.close()


def lib_layout(kb, c):
    return int(kb.lib().kj_index_layout(c._ctx))


def test_errors(built, tmp_path):
    import kaiju_b200 as kb
    d = str(tmp_path); i = inputs("se100", d)
    c = kb.Classifier(FMI, NODES, device=0, params=kb.make_params("mem"))
    c.set_output_strings(kb.STR_TAXON, [b"t%d" % k for k in range(len(c.compact_ids()) - 1)])
    for fmt, msg in ((kb.OUT_NAMES, "name_mode"), (kb.OUT_NAMES_V, "name_mode"), (kb.OUT_KAIJU_V, "KJ_STR_ACCESSION"), (5, "unknown output format")):
        with pytest.raises(kb.KaijuError) as e:
            c.classify_files(i[1], None, d + "/o.tsv", fmt=fmt)
        assert "error -1" in str(e.value) and msg in str(e.value)
        assert not os.path.exists(d + "/o.tsv")          # refused before anything is read or written
    with pytest.raises(kb.KaijuError, match="error -1"):
        c.set_output_strings(kb.STR_TAXON, [b"x"])        # not kj_counts_size() - 1 strings
    c.close()
    # a read whose fragment strings exceed the stride: KJ_ERR_OVERFLOW, the call fails (no truncated column)
    p = cli(["-v", "-t", NODES, "-f", FMI] + i + XP["mem_default"], {"KJ_FRAG_STRIDE": "16"}, check=False)
    assert p.returncode != 0 and b"exceed frag_stride" in p.stderr
    p = cli(["-M", "kaijux", "-T", d + "/t.tsv", "-f", FMI] + i, check=False)
    assert p.returncode != 0 and b"-T cannot be combined with -M" in p.stderr
