"""The context gives back every device allocation it makes.  Create / classify / destroy cycles through every classify path leave the free device
memory where it was; leaving Greedy mode returns the record buffers of the two-kernel path; the error returns of the file pipeline leave
nothing behind once the context is closed.  Free memory is read with cudaMemGetInfo (torch.cuda.mem_get_info): the torch tensors the test
needs exist before the first reading, so torch's caching allocator does not move it."""
import ctypes as C
import os
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# On an H100 80GB the free memory after each of these cycles was the same to the byte; one 2 MiB page of slack stays far below what a leak
# loses (a slot's staging or scratch buffers, a file reader's ring, the >= 256 MiB record buffers of the two-kernel Greedy path).
TOL = 2 << 20
ST = 2048                          # fragment-string stride of kj_classify_verbose2
FILE_CHUNK = "65536"               # KJ_INGEST_CHUNK: many small batches through the file pipeline


@pytest.fixture(scope="module")
def kb(built):
    import kaiju_b200
    return kaiju_b200


@pytest.fixture(scope="module")
def torch_dev():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.init()
    return torch


@pytest.fixture(scope="module")
def reads(golden, torch_dev):
    """PE150 golden reads on the host, and once more on the device with the output arrays of classify_device2."""
    torch = torch_dev
    names, s1, o1, s2, o2 = golden.reads("pe150")
    n = len(o1) - 1
    dev = [torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else np.ascontiguousarray(a)).cuda() for a in (s1, o1, s2, o2)]
    out = [torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")]
    torch.cuda.synchronize()
    return names, s1, o1, s2, o2, dev, out


def free_bytes(torch):
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def verbose2(kb, clf, s1, o1, s2, o2, acc):
    """kj_classify_verbose2 with fragment strings, and accession sets when `acc` (the context must carry accessions)."""
    L = kb.lib()
    L.kj_classify_verbose2.argtypes = [C.c_void_p] * 5 + [C.c_uint64] + [C.c_void_p] * 6 + [C.c_void_p, C.c_uint32, C.c_void_p]
    n = len(o1) - 1
    tax = np.zeros(n, np.uint64); best = np.zeros(n, np.uint32); ids = np.zeros((n, 21), np.uint64); nids = np.zeros(n, np.uint8)
    a = np.zeros((n, 20), np.uint32); na = np.zeros(n, np.uint8); frag = np.zeros((n, ST), np.uint8); flen = np.zeros(n, np.uint32)
    kb._check(L.kj_classify_verbose2(clf._ctx, s1.ctypes.data, o1.ctypes.data, s2.ctypes.data, o2.ctypes.data, n, tax.ctypes.data, best.ctypes.data,
                                     ids.ctypes.data, nids.ctypes.data, a.ctypes.data if acc else None, na.ctypes.data if acc else None,
                                     frag.ctypes.data, ST, flen.ctypes.data))
    assert flen.any()
    return tax


def make_clf(kb, golden, variant, native):
    if variant == "native":
        return kb.Classifier(native, None, device=0, params=kb.make_params("mem"))
    return kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"), copies=2 if variant == "scaled" else 1)


def one_cycle(kb, golden, reads, variant, native, tmp_path):
    """Create a context, classify through every path (MEM: classify, classify_verbose, kj_classify_verbose2, classify_device2; Greedy: the
    two-kernel path with its record buffers; classify_files on the paired FASTQ in small batches), close it."""
    from conftest import GOLD
    names, s1, o1, s2, o2, dev, out = reads
    n = len(o1) - 1
    clf = make_clf(kb, golden, variant, native)
    tax, _ = clf.classify(s1, o1, s2, o2)
    vtax, _, _ = clf.classify_verbose(s1, o1, s2, o2)
    assert np.array_equal(vtax, tax)
    assert np.array_equal(verbose2(kb, clf, s1, o1, s2, o2, acc=variant == "fmi"), tax)
    clf.classify_device2(*[t.data_ptr() for t in dev], n, out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr())
    assert np.array_equal(out[0].cpu().numpy().view(np.uint64), tax)
    clf.set_params(kb.make_params("greedy"))
    clf.classify(s1, o1, s2, o2)
    got, k = clf.classify_files(os.path.join(GOLD, "pe150_1.fq.gz"), os.path.join(GOLD, "pe150_2.fq.gz"), str(tmp_path / "o.tsv"))
    assert got == n and k > 0
    clf.close()


@pytest.fixture(scope="module")
def native_index(kb, golden, tmp_path_factory):
    path = str(tmp_path_factory.mktemp("native") / "golden.kjb")
    kb.write_native_index(golden.fmi, golden.nodes, path)
    return path


@pytest.mark.parametrize("variant", ["fmi", "scaled", "native"])
def test_create_use_destroy_returns_memory(kb, golden, reads, torch_dev, native_index, tmp_path, monkeypatch, variant):
    """One warm-up cycle (module loading, the primary context), then three more: free memory after the fourth is where it was after the
    second.  `scaled` builds the index through kj_create_scaled (copies = 2), `native` loads a device-native index file."""
    monkeypatch.setenv("KJ_INGEST_CHUNK", FILE_CHUNK)
    free = []
    for _ in range(4):
        one_cycle(kb, golden, reads, variant, native_index, tmp_path)
        free.append(free_bytes(torch_dev))
    print("free after each cycle (%s):" % variant, free)
    assert free[3] >= free[1] - TOL, ("lost %.1f MiB over two cycles" % ((free[1] - free[3]) / 2**20), free)


def test_leaving_greedy_returns_prep_records(kb, golden, reads, torch_dev):
    """set_params(mode="mem") after a Greedy call gives the record buffers of the two-kernel Greedy path back.  A first Greedy call grows the
    per-slot scratch, which a context keeps; the second one is measured."""
    names, s1, o1, s2, o2, dev, out = reads
    clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("greedy"))
    clf.classify(s1, o1, s2, o2)
    clf.set_params(kb.make_params("mem"))
    before = free_bytes(torch_dev)
    clf.set_params(kb.make_params("greedy"))
    clf.classify(s1, o1, s2, o2)
    during = free_bytes(torch_dev)
    clf.set_params(kb.make_params("mem"))
    after = free_bytes(torch_dev)
    clf.close()
    print("free before / during / after Greedy:", before, during, after)
    assert before - during >= 256 << 20          # the record buffers were allocated: at least 4 x 64 MiB
    assert after >= before - TOL, ("lost %.1f MiB" % ((before - after) / 2**20))


def test_file_errors_leave_nothing_behind(kb, golden, reads, torch_dev, tmp_path, monkeypatch):
    """kj_classify_files with a missing second input (fails while it opens the readers), and a paired run whose read names differ (fails in
    the parser thread, after its buffers exist): after close() the free memory is back where it was.  The first round is the warm-up."""
    names, s1, o1, s2, o2, dev, out = reads
    monkeypatch.setenv("KJ_INGEST_CHUNK", FILE_CHUNK)
    n = len(o1) - 1
    f1, f2 = str(tmp_path / "m1.fq"), str(tmp_path / "m2.fq")
    for path, seq, off, nm in ((f1, s1, o1, names), (f2, s2, o2, [x if i != n - 10 else x + "X" for i, x in enumerate(names)])):
        with open(path, "wb") as f:
            for i in range(n):
                r = seq[int(off[i]):int(off[i + 1])].tobytes()
                f.write(b"@%s\n%s\n+\n%s\n" % (nm[i].encode(), r, b"I" * len(r)))
    free = []
    for _ in range(2):
        clf = kb.Classifier(golden.fmi, golden.nodes, device=0, params=kb.make_params("mem"))
        with pytest.raises(kb.KaijuError, match="Could not open file"):
            clf.classify_files(f1, str(tmp_path / "missing.fq"), str(tmp_path / "x.tsv"))
        with pytest.raises(kb.KaijuError, match="not identical"):
            clf.classify_files(f1, f2, str(tmp_path / "x.tsv"))
        clf.close()
        free.append(free_bytes(torch_dev))
    print("free after each round:", free)
    assert free[1] >= free[0] - TOL, ("lost %.1f MiB" % ((free[0] - free[1]) / 2**20), free)
