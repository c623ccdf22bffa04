"""Indexes spread over the HBM of a group of GPUs (kj_create_group, kaiju_b200.create_group, layout 4): group contexts whose compact records are
cut into segments (KJ_FORCE_COMPACT + KJ_SPREAD_RECORDS) give bit-identical outputs to the plain compact context on every entry point; their
index checksums equal the compact context's and the host transcoder's; the members can be destroyed in either order; a group too small for its
index fails cleanly; bad arguments are refused; the CLI's -P writes what one device writes.  On a machine with two or more GPUs with peer
access, the same holds across GPUs, and an index too large for one card's compact construction is built over two cards without any hook."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from helpers import SynthDB, build_fmi, have_ref
from test_gpu_compact import MODES, _free, _outputs, _same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "kaiju_b200", "kaiju-b200")


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


def _nb(bwtlen):
    return bwtlen // 128 + 1


def _counts(split, nb):
    """KJ_SPREAD_RECORDS for a named split: the record counts of every segment but the last"""
    return {"0": [0], "1": [1], "half": [nb // 2], "nb-1": [nb - 1], "nb": [nb], "empty-middle": [nb // 3, 0], "thirds": [nb // 3, nb // 3]}[split]


def _peers(kb, n):
    """n GPUs whose every pair has peer access, else skip"""
    import torch
    if kb.device_count() < n:
        pytest.skip("needs %d GPUs" % n)
    for a in range(n):
        for b in range(n):
            if a != b and not torch.cuda.can_device_access_peer(a, b):
                pytest.skip("GPUs %d and %d have no peer access" % (a, b))
    return list(range(n))


def _group(kb, m, fmi, nodes, params, devices, split, copies=1, **kw):
    """(plain compact context, the group's contexts) for the index cut at `split` (a name or a list of record counts)"""
    m.setenv("KJ_FORCE_COMPACT", "1")
    cpt = kb.Classifier(fmi, nodes, device=devices[0], params=params, copies=copies, **kw)
    counts = _counts(split, _nb(cpt.bwtlen)) if isinstance(split, str) else split
    if counts is not None:
        m.setenv("KJ_SPREAD_RECORDS", ",".join(str(x) for x in counts))
    grp = kb.create_group(fmi, nodes, devices, params=params, copies=copies, **kw)
    m.delenv("KJ_SPREAD_RECORDS", raising=False)
    assert cpt.layout == 2 and [g.layout for g in grp] == [4] * len(devices)
    assert all(g.host_bytes == 0 and g.index_bytes > 0 for g in grp) and all(g.bwtlen == cpt.bwtlen for g in grp)
    return cpt, grp


def _close(cpt, grp):
    cpt.close()
    for g in grp:
        g.close()


def _equal_everywhere(kb, m, golden, tmp_path, devices, split, modes):
    """every entry point of every member == the plain compact context, on the golden reads, protein input and long reads"""
    gold = os.path.dirname(golden.fmi); works = [golden.reads(t)[1:] for t in ("pe150", "se100")]
    db = SynthDB(800, 3); ps, po = db.protein_reads(42, 0, 400, 5, 5461); ls, lo = db.long_reads(55, 0, 6, 16384, 40000)
    for mode, env in modes:
        with m.context() as mm:
            for k, v in env.items():
                mm.setenv(k, v)
            cpt, grp = _group(kb, mm, golden.fmi, golden.nodes, kb.make_params(**mode), devices, split)
            try:
                for w, (s1, o1, s2, o2) in enumerate(works):
                    want = _outputs(kb, cpt, s1, o1, s2, o2)
                    for g in grp:
                        _same(want, _outputs(kb, g, s1, o1, s2, o2), (devices, split, mode, env, w))
                s1, o1, s2, o2 = works[0]
                a = kb.classify_multi(grp, s1, o1, s2, o2); b = cpt.classify(s1, o1, s2, o2)      # one batch sharded over the whole group
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
                if mode.get("name_mode") or env:
                    continue
                outs = []
                for clf in [cpt] + grp:
                    o = str(tmp_path / ("o%d.tsv" % len(outs)))
                    clf.classify_files(os.path.join(gold, "pe150_1.fq.gz"), os.path.join(gold, "pe150_2.fq.gz"), o, verbose=True)
                    outs.append(open(o).read())
                assert all(x == outs[0] for x in outs) and len(outs[0]) > 1000
                for clf in [cpt] + grp:
                    clf.set_max_read_len(kb.MAX_LONG_READ_LEN)
                want = _outputs(kb, cpt, ls, lo, None, None, False)
                for g in grp:
                    _same(want, _outputs(kb, g, ls, lo, None, None, False), (devices, split, mode, "long"))
                for clf in [cpt] + grp:
                    clf.set_params(kb.make_params(protein=True, **mode))
                want = _outputs(kb, cpt, ps, po, None, None)
                for g in grp:
                    _same(want, _outputs(kb, g, ps, po, None, None), (devices, split, mode, "protein"))
            finally:
                _close(cpt, grp)


@pytest.mark.parametrize("split", ["0", "1", "half", "nb-1", "nb"])
def test_group_of_two_on_one_gpu_equals_compact_golden(kb, golden, monkeypatch, tmp_path, split):
    """[0, 0], cut at records 0, 1, nb/2, nb-1, nb: kj_classify_device2, kj_classify, kj_classify2's dense indices, counts, kj_classify_verbose,
    kj_classify_verbose2, name mode, kj_classify_multi over the group, the file pipeline, long reads and protein input == the compact context"""
    modes = MODES + [(dict(mode="mem", name_mode=True), {})] if split == "half" else [MODES[0], MODES[1]]
    _equal_everywhere(kb, monkeypatch, golden, tmp_path, [0, 0], split, modes)


@pytest.mark.parametrize("split", ["empty-middle", "thirds"])
def test_group_of_three_on_one_gpu_equals_compact_golden(kb, golden, monkeypatch, tmp_path, split):
    """[0, 0, 0] with an empty middle segment, and in thirds"""
    _equal_everywhere(kb, monkeypatch, golden, tmp_path, [0, 0, 0], split, [MODES[0], MODES[1], (dict(mode="mem", name_mode=True), {})])


@pytest.mark.parametrize("devices,split", [([0, 0], "half"), ([0, 0, 0], "empty-middle"), ([0, 0], None)])
def test_group_checksums_equal_compact_and_host_transcoder(kb, golden, monkeypatch, devices, split):
    """records (the segments in group order: slot 0), superblock table, sa_tax, seq_tax, k-mer table, bwtlen, n_sa on every member; layout 4.
    split None: the library's own placement"""
    with monkeypatch.context() as m:
        cpt, grp = _group(kb, m, golden.fmi, golden.nodes, kb.make_params("mem"), devices, split)
        want = kb.host_index_checksums(golden.fmi, golden.nodes)
        a = cpt.debug_index_checksums(); got = [g.debug_index_checksums() for g in grp]
        _close(cpt, grp)
    keep = [0, 1, 2, 3, 4, 5, 7]
    assert np.array_equal(a[keep], want[keep]), (a, want)
    for b in got:
        assert np.array_equal(b[keep], a[keep]) and int(b[6]) == 4, (b, a)


@pytest.mark.parametrize("copies", [2, 3])
def test_group_scaled_index(kb, monkeypatch, tmp_path, copies):
    """create_group(copies=K) on [0, 0]: the K-fold index's checksums and MEM / Greedy results equal the plain compact K-fold context's"""
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    d = str(tmp_path); db = SynthDB(3000, 11 + copies); db.write(d + "/base.faa", d + "/nodes.dmp")
    base = build_fmi(d + "/base.faa", d + "/base", threads=4); nodes = d + "/nodes.dmp"
    s1, o1, s2, o2 = db.reads(5, 0, 20000, 150, True)
    with monkeypatch.context() as m:
        m.setenv("KJ_BUILD_CHUNK_ROWS", "65536")
        cpt, grp = _group(kb, m, base, nodes, kb.make_params("mem"), [0, 0], "half", copies=copies)
        try:
            a = cpt.debug_index_checksums()
            for g in grp:
                b = g.debug_index_checksums()
                assert np.array_equal(a[[0, 1, 2, 3, 4, 5, 7]], b[[0, 1, 2, 3, 4, 5, 7]])
            for mode in ("mem", "greedy"):
                for clf in [cpt] + grp:
                    clf.set_params(kb.make_params(mode))
                want = _outputs(kb, cpt, s1, o1, s2, o2, False)
                for g in grp:
                    _same(want, _outputs(kb, g, s1, o1, s2, o2, False), (copies, mode))
        finally:
            _close(cpt, grp)


@pytest.mark.parametrize("order", ["first", "last"])
def test_group_members_outlive_each_other(kb, golden, monkeypatch, order):
    """Destroying one member (the first or the last) leaves the index to the other, which classifies as before; the last close frees it all"""
    s1, o1, s2, o2 = golden.reads("pe150")[1:]
    before = _free()
    with monkeypatch.context() as m:
        cpt, grp = _group(kb, m, golden.fmi, golden.nodes, kb.make_params("mem"), [0, 0], "half")
    want = cpt.classify(s1, o1, s2, o2); cpt.close()
    gone, kept = (grp[0], grp[1]) if order == "first" else (grp[1], grp[0])
    gone.close()
    got = kept.classify(s1, o1, s2, o2)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    kept.close()
    assert abs(_free() - before) <= (64 << 20)


def test_group_too_small_fails_cleanly(kb, monkeypatch, tmp_path):
    """A K-fold index larger than the group's HBM: KJ_ERR_NOMEM naming the bytes needed and the bytes free on each device; nothing stays allocated"""
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    d = str(tmp_path); db = SynthDB(12000, 5); db.write(d + "/db.faa", d + "/nodes.dmp")
    fmi = build_fmi(d + "/db.faa", d + "/db", threads=min(16, os.cpu_count())); nodes = d + "/nodes.dmp"
    small = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem")); rows = small.bwtlen; small.close()
    copies = min(65536, int(2.0 * _free() / rows))          # ~2 rows per byte of free HBM: the records alone (1 B per row) do not fit
    assert rows * copies > 1.2 * _free(), (rows, copies)
    before = _free()
    with pytest.raises(kb.KaijuError, match=r"error -7: .*does not fit in the HBM of the group: it needs \d+ bytes .*free: device 0 \d+ bytes"):
        kb.create_group(fmi, nodes, [0, 0], params=kb.make_params("mem"), copies=copies)
    assert abs(_free() - before) <= (2 << 20)


def test_group_bad_arguments(kb, golden):
    """n = 0, n > 8 and a bad device ordinal are refused with KJ_ERR_ARG before anything is allocated"""
    L = kb.lib(); f = C.c_void_p(); t = C.c_void_p()
    kb._check(L.kj_fmi_load(golden.fmi.encode(), C.byref(f))); kb._check(L.kj_nodes_load(golden.nodes.encode(), C.byref(t)))
    try:
        iv = kb.KjIndexView(); tv = kb.KjTaxonomyView(); L.kj_fmi_view(f, C.byref(iv)); L.kj_nodes_view(t, C.byref(tv))
        p = kb.make_params("mem"); out = (C.c_void_p * 9)()
        for devs in ([], [0] * 9, [0, kb.device_count()], [-1]):
            arr = (C.c_int * max(1, len(devs)))(*devs)
            assert L.kj_create_group(out, len(devs), arr, C.byref(p), C.byref(iv), C.byref(tv), 1) == -1, devs
            assert all(x is None for x in out)
    finally:
        L.kj_nodes_free(t); L.kj_fmi_free(f)


def test_cli_pool_equals_one_device(kb, golden, tmp_path):
    """kaiju-b200 -d 0,0 -P under KJ_FORCE_COMPACT writes the output and the -T table of -d 0 byte for byte; -P with -H is refused"""
    gold = os.path.dirname(golden.fmi); d = str(tmp_path)
    with open(d + "/names.dmp", "w") as f:
        for line in open(golden.nodes):
            nid = line.split("\t|\t")[0].strip()
            f.write("%s\t|\ttaxon %s\t|\t\t|\tscientific name\t|\n" % (nid, nid))
    env = dict(os.environ, KJ_FORCE_COMPACT="1")
    base = ["-t", golden.nodes, "-f", golden.fmi, "-i", os.path.join(gold, "pe150_1.fq.gz"), "-j", os.path.join(gold, "pe150_2.fq.gz"), "-N", d + "/names.dmp", "-v"]
    for tag, dev in (("one", ["-d", "0"]), ("pool", ["-d", "0,0", "-P"])):
        subprocess.run([CLI] + base + dev + ["-o", "%s/%s.tsv" % (d, tag), "-T", "%s/%s.table" % (d, tag)], env=env, check=True)
    for ext in ("tsv", "table"):      # (the table's file column is the output file's name)
        a = open("%s/one.%s" % (d, ext)).read().replace(d + "/one.tsv", "OUT"); b = open("%s/pool.%s" % (d, ext)).read().replace(d + "/pool.tsv", "OUT")
        assert a == b and len(a) > 100, ext
    r = subprocess.run([CLI] + base + ["-d", "0,0", "-P", "-H", "1", "-o", d + "/x.tsv"], env=env, capture_output=True, text=True)
    assert r.returncode != 0 and "-P cannot be combined with -H" in r.stderr


def test_group_across_two_gpus_equals_compact(kb, golden, monkeypatch, tmp_path):
    """[0, 1], cut in half and by the library's own placement: every entry point == the plain compact context on GPU 0"""
    devices = _peers(kb, 2)
    _equal_everywhere(kb, monkeypatch, golden, tmp_path, devices, "half", MODES[:2])
    _equal_everywhere(kb, monkeypatch, golden, tmp_path, devices, None, MODES[:1])


def test_index_beyond_one_gpu_on_two(kb, tmp_path):
    """A scaled index whose compact construction does not fit on one card is built over [0, 1] without any hook; on 200 k PE150 pairs its MEM and
    Greedy results equal those of a kj_create_tiered context of the same index"""
    devices = _peers(kb, 2)
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    d = str(tmp_path); db = SynthDB(24000, 77); db.write(d + "/db.faa", d + "/nodes.dmp")
    fmi = build_fmi(d + "/db.faa", d + "/db", threads=min(16, os.cpu_count())); nodes = d + "/nodes.dmp"
    small = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem")); rows = small.bwtlen; small.close()
    copies = max(2, int(1.15 * _free() / 1.52 / rows))
    s1, o1, s2, o2 = db.reads(9, 0, 200000, 150, True)
    grp = kb.create_group(fmi, nodes, devices, params=kb.make_params("mem"), copies=copies)
    try:
        assert [g.layout for g in grp] == [4, 4] and all(g.index_bytes > (8 << 30) for g in grp)
        got = {}
        for mode in ("mem", "greedy"):
            for g in grp:
                g.set_params(kb.make_params(mode))
            got[mode] = kb.classify_multi(grp, s1, o1, s2, o2)
    finally:
        for g in grp:
            g.close()
    tie = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"), copies=copies, host_memory=int(0.7 * rows * copies) + (8 << 30))
    try:
        for mode in ("mem", "greedy"):
            tie.set_params(kb.make_params(mode)); want = tie.classify(s1, o1, s2, o2)
            assert np.array_equal(got[mode][0], want[0]) and np.array_equal(got[mode][1], want[1]), mode
    finally:
        tie.close()
