"""The compact spread layout (kj_layout.h, layout 4: compact records cut into contiguous segments over the HBM of a group of GPUs) on the CPU warp
emulator (tests/emu/kj_emu_spread.cpp): the KjSpreadIdx instances on a KJ_FORCE_COMPACT index cut by KJ_SPREAD_RECORDS -- two segments split at
records 0, 1, nb/2, nb-1 and nb, three segments with an empty middle one, eight segments -- against the golden outputs of the reference, the
oracle and the compact emulation: golden sets with verbose columns and name mode, protein input, long reads through the long instances, and the
3 * 2^16-row quirk index."""
import ctypes as C
import numpy as np
import pytest
import emu_compact
import emu_spread
import test_kernel_logic_emulated as K
from conftest import GOLDEN_CONFIGS
from helpers import Oracle, SynthDB, make_params

SPLITS = ["2:0", "2:1", "2:half", "2:nb-1", "2:nb", "3:empty-middle", "8:even"]


@pytest.fixture(scope="module")
def emu(built, tmp_path_factory):
    return emu_spread.load(str(tmp_path_factory.mktemp("emu_spread")), K.KjParams)


@pytest.fixture(scope="module")
def emu_long(built, tmp_path_factory):
    return emu_spread.load(str(tmp_path_factory.mktemp("emu_spread_long")), K.KjParams, long=True)


@pytest.fixture(scope="module")
def emu_cpt(built, tmp_path_factory):
    return emu_compact.load(str(tmp_path_factory.mktemp("emu_compact_ref")), K.KjParams)


def _layout(E, fmi, nodes):
    """(layout, segment starts first[0..n]) of the emulator context of (fmi, nodes)"""
    kp = K.KjParams(**make_params(mode="mem")); h = E.kjemu_create(fmi.encode(), nodes.encode(), C.byref(kp)); assert h
    n = C.c_uint(); first = (C.c_ulonglong * 9)(); lay = E.kjemu_layout(h, C.byref(n), first); E.kjemu_destroy(h)
    return lay, [int(first[g]) for g in range(n.value + 1)]


def counts_for(split, nb):
    """KJ_SPREAD_RECORDS for a split name: the record counts of every segment but the last"""
    g, where = split.split(":")
    if g == "2":
        return [{"0": 0, "1": 1, "half": nb // 2, "nb-1": nb - 1, "nb": nb}[where]]
    if g == "3":
        return [nb // 3, 0]
    return [nb // 8] * 7


def split_at(E, fmi, nodes, split, monkeypatch):
    """Sets KJ_SPREAD_RECORDS for `split` on the index of (fmi, nodes) and checks that the emulator context is spread that way."""
    monkeypatch.setenv("KJ_FORCE_COMPACT", "1"); monkeypatch.delenv("KJ_SPREAD_RECORDS", raising=False)
    lay, first = _layout(E, fmi, nodes)
    assert lay == 2
    nb = first[-1]; counts = counts_for(split, nb)
    monkeypatch.setenv("KJ_SPREAD_RECORDS", ",".join(str(x) for x in counts))
    lay, first = _layout(E, fmi, nodes)
    want = [0]
    for x in counts:
        want.append(min(nb, want[-1] + x))
    assert lay == 4 and first == want + [nb], (lay, first, want, nb)
    return first


def test_spread_emulated_segment_table(emu, golden, monkeypatch):
    """The splits the tests use: an empty first segment, an empty last one, an empty middle one, eight segments"""
    assert split_at(emu, golden.fmi, golden.nodes, "2:0", monkeypatch)[:2] == [0, 0]
    first = split_at(emu, golden.fmi, golden.nodes, "2:nb", monkeypatch); assert first[1] == first[2]
    first = split_at(emu, golden.fmi, golden.nodes, "3:empty-middle", monkeypatch); assert first[1] == first[2] < first[3]
    assert len(split_at(emu, golden.fmi, golden.nodes, "8:even", monkeypatch)) == 9


@pytest.mark.parametrize("split", SPLITS)
def test_spread_emulated_golden_sets(emu, golden, monkeypatch, split):
    """Every golden configuration, paired and single-end, and Greedy through the two-kernel path: == the reference's outputs."""
    split_at(emu, golden.fmi, golden.nodes, split, monkeypatch)
    for cfg in sorted(GOLDEN_CONFIGS):
        for tag in ("pe150", "se100"):
            K.test_emulated_kernel_matches_reference_golden(emu, golden, cfg, tag)
    for cfg in [c for c in sorted(GOLDEN_CONFIGS) if c.startswith("greedy")][:2]:
        K.test_emulated_two_kernel_greedy_matches_reference_golden(emu, golden, cfg, monkeypatch)
    monkeypatch.delenv("KJ_EMU_SPLIT", raising=False)


@pytest.mark.parametrize("split", SPLITS)
def test_spread_emulated_verbose_columns_and_name_mode(emu, golden, monkeypatch, split):
    """All seven `kaiju -v` columns (the SA walk's accessions read through the segments) and kaijux name mode."""
    split_at(emu, golden.fmi, golden.nodes, split, monkeypatch)
    for cfg in ("mem_default", "greedy_e5_s40"):
        K.test_emulated_verbose_columns_match_reference(emu, golden, cfg)
    for cfg in ("mem_default", "greedy_default"):
        K.test_emulated_name_frontend_matches_reference_kaijux(emu, golden, cfg)


@pytest.mark.parametrize("split", SPLITS)
def test_spread_emulated_equals_oracle_and_compact_emulation(emu, emu_cpt, golden, monkeypatch, split):
    """Seeded parameter sweep and protein input: spread == oracle == the compact emulation, read for read."""
    import random
    split_at(emu, golden.fmi, golden.nodes, split, monkeypatch)
    orc = Oracle(golden.fmi, golden.nodes); rnd = random.Random(12)
    names, s1, o1, s2, o2 = golden.reads("pe150")
    runs = []
    for _ in range(3):
        mode = rnd.choice(["mem", "greedy"]); kw = dict(mode=mode, m=rnd.choice([6, 9, 11, 15]), seg=rnd.random() < 0.7)
        if mode == "greedy":
            kw.update(e=rnd.choice([0, 1, 3, 5]), s=rnd.choice([40, 65, 80]))
        runs.append((make_params(**kw), s1, o1, s2, o2))
    db = SynthDB(800, 3); ps, po = db.protein_reads(42, 0, 300, 5, 5461)
    for kw in (dict(mode="mem"), dict(mode="greedy", e=5, s=40, E=1e-3)):
        runs.append((make_params(protein=True, **kw), ps, po, None, None))
    for P, a1, b1, a2, b2 in runs:
        otax, obest = orc.classify_batch(P, a1, b1, a2, b2)
        tax, best = K.emu_classify(emu, golden.fmi, golden.nodes, P, a1, b1, a2, b2)
        ctax, cbest = K.emu_classify(emu_cpt, golden.fmi, golden.nodes, P, a1, b1, a2, b2)
        assert np.array_equal(tax, otax) and np.array_equal(best, obest), P
        assert np.array_equal(tax, ctax) and np.array_equal(best, cbest), P


@pytest.mark.parametrize("split", SPLITS)
def test_spread_emulated_long_instances(emu_long, golden, monkeypatch, split):
    """Long DNA and protein reads through the spread long instances == the oracle; short golden reads through them == the reference."""
    split_at(emu_long, golden.fmi, golden.nodes, split, monkeypatch)
    db = SynthDB(800, 3); orc = Oracle(golden.fmi, golden.nodes)
    s, o = db.long_reads(55, 0, 4, 16384, 30000); ps, po = db.protein_reads(54, 0, 4, 5462, 12000)
    for P, a, b in ((make_params(mode="mem"), s, o), (make_params(mode="greedy", e=5, s=50), s, o), (make_params(mode="mem", protein=True), ps, po)):
        otax, obest = orc.classify_batch(P, a, b)
        tax, best = K.emu_classify(emu_long, golden.fmi, golden.nodes, P, a, b, None, None)
        assert np.array_equal(tax, otax) and np.array_equal(best, obest), P
    K.test_emulated_kernel_matches_reference_golden(emu_long, golden, "mem_default", "pe150")
    K.test_emulated_verbose_columns_match_reference(emu_long, golden, "greedy_default")


@pytest.mark.parametrize("split", SPLITS)
def test_spread_emulated_quirk_index(emu, built, monkeypatch, tmp_path, split):
    """bwtlen = 3 * 2^16: the reference's checkpoint quirk on segmented records (rank correction, k-mer table, SA walk) == the oracle."""
    from helpers import have_ref, make_quirk_db, pack_reads
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    fmi, nodes, reads = make_quirk_db(str(tmp_path), nprot=768)
    split_at(emu, fmi, nodes, split, monkeypatch)
    seq, off = pack_reads(reads); orc = Oracle(fmi, nodes)
    for kw in (dict(mode="mem"), dict(mode="greedy"), dict(mode="greedy", e=5, s=40)):
        P = make_params(**kw); otax, obest = orc.classify_batch(P, seq, off)
        rc, tax, best = K.emu_classify_rc(emu, fmi, nodes, P, seq, off)
        assert rc == 0 and np.array_equal(tax, otax) and np.array_equal(best, obest), kw
