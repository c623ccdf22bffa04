"""The stream side of the file pipeline's reader (kaiju_b200/csrc/kj_stream.h) on the CPU, over real pipes and FIFOs fed by writer threads in
pieces of 1 byte to 1 MB with pauses (one inside a record, one inside a BGZF header): plain text, BGZF through the inflate emulator, BGZF followed
by ordinary gzip, multi-member gzip, the end block alone, an empty stream and streams shorter than the format probe give the text zlib (or the
input) gives; bad BGZF blocks give the message and offset the file reader gives; other gzip reads as gzread reads the same bytes from a file;
halt() ends a read that waits for a stalled writer.  The last test runs this module again on a harness built with the address and
undefined-behaviour sanitisers."""
import gzip
import os
import subprocess
import sys
import threading
import time
import zlib

import pytest

import emu_inflate as ei
import emu_stream as es

SANITIZE = bool(os.environ.get("KJ_EMU_INFLATE_SANITIZE"))
CHUNKS = [256, 70000, 16 << 20]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return es.load(str(tmp_path_factory.mktemp("emu_stream")), sanitize=SANITIZE)


def through_pipe(emu, data, chunk, seed=1, pauses=(), cap=None, fifo=None):
    """data written into a pipe (or the FIFO at path `fifo`, opened before its writer) by a writer thread; the reader's result"""
    if fifo:
        os.mkfifo(fifo); rfd = os.open(fifo, os.O_RDONLY | os.O_NONBLOCK); w = es.Writer(data, seed, path=fifo, pauses=pauses)
    else:
        rfd, wfd = os.pipe(); w = es.Writer(data, seed, fd=wfd, pauses=pauses)
    r = es.Reader(emu, rfd)
    w.start()
    try:
        return r.read(chunk, cap if cap is not None else 4 * len(data) + (1 << 20))
    finally:
        r.close(); w.finish()


def fq(n, seed):
    return ei.fastq_text(n, seed)


def test_plain_text(emu, tmp_path):
    text = fq(3000, 1); mid_record = text.index(b"\n+\n", 100000) - 40
    for k, chunk in enumerate(CHUNKS):
        rc, got, inflated, chunks, msg = through_pipe(emu, text, chunk, seed=k, pauses=(65536, mid_record), fifo=str(tmp_path / ("p%d" % k)) if k == 1 else None)
        assert rc == 0 and got == text and inflated == 0, (chunk, msg)
        assert chunks == len(text) // chunk + 1                 # full chunks, then the last one (maybe empty) with the end of the stream


def test_bgzf_blocks_through_the_emulated_inflate(emu):
    text = fq(2500, 2)
    for level, block in ((1, ei.MAX_SLICE), (6, 20000), (6, 777)):
        bg = ei.bgzf_write(text, level, block=block)
        second = next(iter(ei._block_ends(bg)))
        for chunk in (256, 70000, 200000):
            rc, got, inflated, _, msg = through_pipe(emu, bg, chunk, seed=level + chunk, pauses=(second + 7, second + 100, 65536, 65537))
            assert rc == 0 and got == text and inflated == len(text), (level, block, chunk, msg)


def test_bgzf_followed_by_ordinary_gzip(emu):
    text = fq(1500, 3); cut = text.index(b"\n@", len(text) // 2) + 1; a, b = text[:cut], text[cut:]
    data = ei.bgzf_write(a, 6, block=20000, eof=False) + gzip.compress(b, 1)
    for chunk in CHUNKS:
        rc, got, inflated, _, msg = through_pipe(emu, data, chunk, seed=chunk, pauses=(len(data) - len(b) // 3,))
        assert rc == 0 and got == text and inflated == len(a), (chunk, msg)


def test_multi_member_gzip(emu, tmp_path):
    text = fq(2000, 4); parts = [text[:1], text[1:70000], text[70000:300000], text[300000:]]
    data = b"".join(gzip.compress(p, lv) for p, lv in zip(parts, (1, 6, 9, 1)))
    assert zlib.decompressobj(31).decompress(data) == parts[0]            # one z_stream alone stops after the first member
    for chunk in CHUNKS:
        rc, got, inflated, _, msg = through_pipe(emu, data, chunk, seed=chunk, pauses=(len(gzip.compress(parts[0], 1)) + 1,))
        assert rc == 0 and got == text and inflated == 0, (chunk, msg)


def test_only_the_end_block_empty_and_short_streams(emu):
    cases = [(ei.EOF_BLOCK, b"", 0), (b"", b"", 0), (b"@r\nACGT\n+\nIIII", b"@r\nACGT\n+\nIIII", 0), (b"A", b"A", 0), (b"\x1f", None, 0),
             (ei.bgzf_write(fq(20, 5)), fq(20, 5), len(fq(20, 5))), (gzip.compress(fq(30, 6)), fq(30, 6), 0)]
    for data, want, want_inflated in cases:
        for chunk in (256, 70000):
            rc, got, inflated, chunks, msg = through_pipe(emu, data, chunk)
            if want is None:          # a lone 0x1f: a gzip header cut short, as for a file
                assert rc == 1 and msg == "truncated BGZF block in file <stream> at compressed offset 0", msg
                continue
            assert rc == 0 and got == want and inflated == want_inflated, (data[:20], chunk, msg)


def test_bad_blocks_give_the_file_readers_message(emu):
    text, bg, bad_files = ei.corrupt_files()
    for name, data, offset in bad_files:
        for chunk in (256, 70000):
            rc, got, _, _, msg = through_pipe(emu, data, chunk, seed=chunk, pauses=(offset + 9,))
            assert rc == 1 and msg.startswith({"truncated": "truncated BGZF block", "flipped_bit": "corrupt BGZF block", "wrong_crc": "corrupt BGZF block"}[name]), msg
            assert (" in file <stream> at compressed offset %d" % offset) in msg, (name, msg)
    bad = bytearray(ei.bgzf_write(text, 6, block=20000)); second = next(iter(ei._block_ends(bytes(bad)))); bad[second + 16:second + 18] = b"\x10\x00"
    rc, _, _, _, msg = through_pipe(emu, bytes(bad), 70000)
    assert rc == 1 and msg == "corrupt BGZF header in file <stream> at compressed offset %d" % second, msg


def test_gzip_stream_reads_as_gzread_reads_a_file(emu, tmp_path):
    """Trailing garbage, a member cut short, a lone byte behind a member, a damaged member and a wrong CRC: the stream gives what gzread gives
    from the same bytes in a file (the text, or an error where gzread returns -1)."""
    text = fq(800, 7); a, b = text[:100000], text[100000:]
    ga, gb = gzip.compress(a, 6), gzip.compress(b, 1)
    crc = bytearray(ga + gb); crc[-8] ^= 1
    damaged = bytearray(ga + gb); damaged[len(ga) + 400] ^= 0xff
    cases = {"garbage": ga + gb + b"not gzip at all", "cut": ga + gb[:len(gb) // 2], "lone_byte": ga + b"\x1f", "zeros": ga + b"\0" * 100,
             "crc": bytes(crc), "damaged": bytes(damaged), "header_only": ga + gb[:5]}
    for name, data in cases.items():
        path = str(tmp_path / (name + ".gz")); open(path, "wb").write(data)
        frc, ftext = es.gzread_file(emu, path, 4 * len(text))
        rc, got, _, _, msg = through_pipe(emu, data, 70000, seed=len(name))
        assert (rc, got if rc == 0 else None) == (frc, ftext if frc == 0 else None), (name, rc, frc, msg)
        if frc:
            assert msg == "read error in file <stream>", msg
    assert es.gzread_file(emu, str(tmp_path / "garbage.gz"), 4 * len(text)) == (0, text)


def test_halt_ends_a_read_that_waits_for_a_stalled_writer(emu, tmp_path):
    for kind in ("plain", "bgzf", "gzip", "no_writer"):
        data = {"plain": fq(50, 8), "bgzf": ei.bgzf_write(fq(50, 8))[:-100], "gzip": gzip.compress(fq(300, 8))[:-100], "no_writer": b""}[kind]
        fifo = str(tmp_path / kind); os.mkfifo(fifo); rfd = os.open(fifo, os.O_RDONLY | os.O_NONBLOCK)
        r = es.Reader(emu, rfd); w = es.Writer(data, 3, path=fifo, stall=30)
        if kind != "no_writer":
            w.start()
        res = []; t = threading.Thread(target=lambda: res.append(r.read(70000, 1 << 20))); t.start()
        try:
            time.sleep(0.3)
            assert t.is_alive() and not res, kind                  # waiting for the writer
            t0 = time.monotonic(); r.halt(); t.join(10)
            assert not t.is_alive() and time.monotonic() - t0 < 5, kind
            assert res[0][0] == -2, (kind, res[0])                   # KJ_STREAM_HALTED
        finally:
            t.join(10); r.close()
            if kind != "no_writer":
                w.finish()


@pytest.mark.skipif(SANITIZE, reason="this is the sanitised run")
def test_module_passes_under_address_and_undefined_sanitizers():
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__)], env=ei.sanitizer_env(),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
