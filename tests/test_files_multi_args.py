"""kj_classify_files_multi refuses a null argument or a context count outside 1..8 with KJ_ERR_ARG before it touches a device (no GPU needed)."""
import ctypes as C


def test_null_and_count_arguments(built, golden, tmp_path):
    import kaiju_b200 as kb
    L = kb.lib(); out = str(tmp_path / "o.tsv").encode(); fq = golden.fmi.encode()
    one = (C.c_void_p * 1)(None)
    assert L.kj_classify_files_multi(None, 1, fq, None, out, 0, None, None) == -1
    assert L.kj_classify_files_multi(one, 0, fq, None, out, 0, None, None) == -1
    assert L.kj_classify_files_multi(one, 1, fq, None, out, 0, None, None) == -1 and b"null context" in L.kj_last_error()
    assert L.kj_classify_files_multi(one, 1, None, None, out, 0, None, None) == -1
    assert L.kj_classify_files_multi((C.c_void_p * 9)(), 9, fq, None, out, 0, None, None) == -1 and b"outside 1..8" in L.kj_last_error()
    assert not (tmp_path / "o.tsv").exists()
