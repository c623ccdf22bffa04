"""The compact rank layout (kj_layout.h: 5 bit-planes per 64 rows, midpoint counts, superblock table) on the CPU: the transcoder's rank query and
the kernels' rank / LF primitives against naive counting on BWTs whose lengths sit on and around the record and superblock edges, and the
emulated kernel logic on a KJ_FORCE_COMPACT index against the golden outputs and the oracle (the same sets as test_kernel_logic_emulated.py).
The emulator build is tests/emu/kj_emu_compact.cpp: it runs the compact instantiation where the descriptor says compact, as the library does."""
import ctypes as C
import numpy as np
import pytest
import emu_compact
import test_kernel_logic_emulated as K
from conftest import GOLDEN_CONFIGS
from helpers import Oracle, make_params


@pytest.fixture(scope="module")
def emu(built, tmp_path_factory):
    return emu_compact.load(str(tmp_path_factory.mktemp("emu_compact")), K.KjParams)

LENGTHS = sorted({65536 * m + d for m in (1, 2, 3) for d in (-1, 0, 1, 127, 128, 129)} | {128 * m for m in (1, 3, 511, 512, 513)} | {1, 63, 64, 65})


@pytest.fixture
def compact(monkeypatch):
    monkeypatch.setenv("KJ_FORCE_COMPACT", "1")


@pytest.mark.parametrize("alen", [21, 24])
def test_compact_rank_equals_naive_counting(emu, compact, monkeypatch, alen):
    """FMindex(c, k) = C[c] + #c in BWT[0, k) for every letter c < alen and every k in [0, bwtlen] (k = bwtlen included, also when bwtlen is a
    multiple of the record and superblock sizes), from the transcoder (host_rank) and the kernels' primitives; the LF step's letter and rank too."""
    monkeypatch.setenv("KJ_KMER_K", "0")
    rng = np.random.default_rng(alen)
    for n in LENGTHS:
        bwt = rng.integers(0, alen, n, dtype=np.uint8)
        bwt[rng.integers(0, n, max(1, n // 5000))] = 0            # a few terminators, as in a real BWT
        lay = C.c_int(-1)
        bad = emu.kjemu_rank_check(bwt.ctypes.data, n, alen, C.byref(lay))
        assert lay.value == 2 and bad == 0, (n, lay.value, bad)


def test_compact_rank_one_letter_runs(emu, compact, monkeypatch):
    """Records and superblocks that hold one letter only (the 16-bit midpoint count at its maximum, 65472)."""
    monkeypatch.setenv("KJ_KMER_K", "0")
    n = 3 * 65536 + 77
    bwt = np.full(n, 23, np.uint8); bwt[65536:2 * 65536] = 5; bwt[-50:] = 0
    lay = C.c_int(-1)
    assert emu.kjemu_rank_check(bwt.ctypes.data, n, 24, C.byref(lay)) == 0 and lay.value == 2


@pytest.mark.parametrize("cfg", sorted(GOLDEN_CONFIGS))
@pytest.mark.parametrize("tag", ["pe150", "se100"])
def test_compact_emulated_kernel_matches_reference_golden(emu, golden, compact, cfg, tag):
    K.test_emulated_kernel_matches_reference_golden(emu, golden, cfg, tag)


@pytest.mark.parametrize("cfg", [c for c in sorted(GOLDEN_CONFIGS) if c.startswith("greedy")])
def test_compact_emulated_two_kernel_greedy_matches_reference_golden(emu, golden, compact, cfg, monkeypatch):
    K.test_emulated_two_kernel_greedy_matches_reference_golden(emu, golden, cfg, monkeypatch)


def test_compact_emulated_kernel_matches_oracle_on_random_parameters(emu, golden, compact):
    K.test_emulated_kernel_matches_oracle_on_random_parameters(emu, golden)


@pytest.mark.parametrize("kw", [dict(mode="mem"), dict(mode="greedy"), dict(mode="mem", m=7, seg=False), dict(mode="greedy", e=5, s=40, E=1e-3)])
def test_compact_emulated_kernel_long_reads_and_protein_input(emu, golden, compact, kw):
    K.test_emulated_kernel_long_reads_and_protein_input(emu, golden, kw)


@pytest.mark.parametrize("cfg", sorted(K.XP_CONFIGS))
def test_compact_emulated_name_frontend_matches_reference_kaijux(emu, golden, compact, cfg):
    K.test_emulated_name_frontend_matches_reference_kaijux(emu, golden, cfg)


@pytest.mark.parametrize("cfg", ["mem_default", "mem_m5_noseg", "greedy_default", "greedy_e5_s40"])
def test_compact_emulated_verbose_columns_match_reference(emu, golden, compact, cfg):
    K.test_emulated_verbose_columns_match_reference(emu, golden, cfg)


def test_compact_emulated_kernel_on_quirk_index(emu, built, compact, tmp_path):
    """bwtlen = 3 * 2^16: the reference's checkpoint quirk on the compact layout (rank correction, k-mer table, SA walk) == the oracle."""
    from helpers import have_ref, make_quirk_db, pack_reads
    if not have_ref():
        pytest.skip("oracle/_ref (index builder) not available")
    fmi, nodes, reads = make_quirk_db(str(tmp_path), nprot=768)
    seq, off = pack_reads(reads); orc = Oracle(fmi, nodes)
    for kw in (dict(mode="mem"), dict(mode="greedy"), dict(mode="greedy", e=5, s=40)):
        P = make_params(**kw); otax, obest = orc.classify_batch(P, seq, off)
        rc, tax, best = K.emu_classify_rc(emu, fmi, nodes, P, seq, off)
        assert rc == 0 and np.array_equal(tax, otax) and np.array_equal(best, obest), kw


def test_native_index_file_refuses_compact_layout(built, golden, tmp_path, monkeypatch):
    """Device-native index files keep the narrow and wide layouts; a compact index is not written."""
    import kaiju_b200 as kb
    monkeypatch.setenv("KJ_FORCE_COMPACT", "1")
    with pytest.raises(kb.KaijuError, match="narrow and wide"):
        kb.write_native_index(golden.fmi, golden.nodes, str(tmp_path / "db.kjb"))
    assert kb.host_index_checksums(golden.fmi, golden.nodes)[6] == 2
