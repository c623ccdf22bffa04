"""The product's SEG filter (kj_seg of kj_core.h: window classes, trigger loop, left-trim recursion, both trim searches, region merge) on the
CPU warp emulator, region by region against the reference's SeqBufferSeg, in all four instantiations (short/long kernels x the rolled and
unrolled window-class variants), on seeded sequence families chosen for SEG's edges.  Also: the region array of the work space (KJ_SEG_CAP)
never fills on region-dense sequences at the caps of three batch profiles."""
import os

import pytest

import emu_seg as es

pytestmark = pytest.mark.skipif(not os.path.exists(es.REF_SO), reason="oracle/_ref/libkaijuref.so not built (reference sources absent)")
INSTANCES = [(False, False), (False, True), (True, False), (True, True)]        # (LONG, compact)


@pytest.fixture(scope="module")
def E(tmp_path_factory):
    return es.load(str(tmp_path_factory.mktemp("emu_seg")))


@pytest.fixture(scope="module")
def ref():
    return es.RefSeg()


def _compare(E, ref, seqs, instances, max_len=None):
    """Compare every sequence in every instance; returns (comparisons, per-branch hit counts per instance, densest raw regions per residue,
    largest raw region count)."""
    cov = {inst: [0] * len(es.COVERAGE) for inst in instances}; n = 0; bad = []; dens = 0.0; raw_max = 0
    for fam, s in seqs:
        want = ref(s)
        for inst in instances:
            got, err, c = es.emu_seg(E, s, max_len or es.max_len_for(len(s)), *inst)
            n += 1
            if got != want or err:
                bad.append((fam, inst, len(s), want[:4], got[:4], err))
            cov[inst] = [a + b for a, b in zip(cov[inst], c)]
            raw_max = max(raw_max, c[-1]); dens = max(dens, c[-1] / len(s)) if s else dens
    assert not bad, "%d of %d SEG results differ from SeqBufferSeg, first: %s" % (len(bad), n, bad[:3])
    return n, cov, dens, raw_max


def test_seg_regions_match_reference(E, ref):
    seqs = es.families(1, scale=4) + es.nested(3) + es.stirling_tie(4) + es.big_families(2)
    n, cov, dens, _ = _compare(E, ref, seqs, INSTANCES)
    print("\nSEG: %d sequences, %d comparisons in 4 instances, 0 differences; densest raw regions per residue %.3f" % (len(seqs), n, dens))
    for inst in INSTANCES:
        print("  LONG=%d compact=%d: %s" % (inst[0], inst[1], ", ".join("%s %d" % kv for kv in zip(es.COVERAGE, cov[inst]))))
    assert len(seqs) >= 20000
    for inst in INSTANCES:
        c = dict(zip(es.COVERAGE, cov[inst]))
        # every branch many times: short trims of both minlen kinds, the sorted-composition trim, Stirling's ln(n!), the level-1 region, merges
        assert c["trim_minlen_1"] >= 10000 and c["trim_minlen_n2_minus_50"] >= 10000 and c["trim_long"] >= 2000, (inst, c)
        assert c["stirling"] >= 10 and c["level1_region"] >= 200 and c["merge"] >= 2000, (inst, c)


def test_seg_regions_beyond_16_bits(E, ref):
    """Regions of 65,535, 65,536 and 70,000 residues: the long kernels' 32-bit counts and result packing."""
    seqs = es.big_families(5, long_only=True)
    _, cov, _, _ = _compare(E, ref, seqs, [(True, False), (True, True)])
    for inst, c in cov.items():
        assert c[2] >= len(seqs) and c[3] >= len(seqs), (inst, c)


@pytest.fixture(scope="module")
def dense(E):
    """Region-dense fragments: hill-climbed on the raw region count at 51 and 200 residues."""
    return [es.dense_search(E, 51, seed, 1500, max_len=152) for seed in range(4)] + [es.dense_search(E, 200, 10 + seed, 800) for seed in range(4)]


@pytest.mark.parametrize("max_len", [152, 16384, 60000])
def test_seg_region_array_never_fills(E, ref, dense, max_len):
    """Region-dense sequences at the longest fragment of three batch profiles (PE150, protein reads of 5,461 residues, a long-read batch):
    the raw region count stays below KJ_SEG_CAP - 1, so error flag 8 (which fails the whole call) is never set, and the regions match."""
    cap, mf = es.seg_cap(E, max_len)
    seqs = []
    for raw, s in dense:
        seqs.append(("dense", (s * (mf // len(s) + 1))[:mf]))        # the dense pattern tiled over the whole fragment
        seqs.append(("dense", s[:mf]))
    n, cov, dens, raw_max = _compare(E, ref, seqs, INSTANCES if max_len <= 16384 else INSTANCES[2:], max_len)
    print("\nmax_len %d: longest fragment %d, region cap %d; densest raw regions per residue %.3f (hill climb), %.3f (at this length), "
          "most raw regions %d" % (max_len, mf, cap, max(r / len(s) for r, s in dense), dens, raw_max))
    assert raw_max < cap - 1
