"""The BGZF inflate kernel source on the CPU warp emulator against Python's zlib: every block type and compression setting, the block chain
walked across chunk boundaries, and malformed input -- which must end in an error code, never in an access outside the block's buffers.  The
last test runs this module once more on an emulator built with the address and undefined-behaviour sanitisers; that run is the evidence for
the bounds checks, and malformed input is only ever explored here, on the CPU."""
import ctypes as C
import gzip
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

import emu_inflate as ei
from conftest import GOLD

SANITIZE = bool(os.environ.get("KJ_EMU_INFLATE_SANITIZE"))
ERR = dict(input=1, btype=2, stored=3, lens=4, code=5, dist=6, output=7, isize=8, crc=9, bound=10, trailing=11)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return ei.load(str(tmp_path_factory.mktemp("emu_inflate")), sanitize=SANITIZE)


@pytest.fixture(scope="module")
def cases():
    return ei.valid_files()


def test_writer_produces_standard_gzip(cases):
    """Ties the fixture to the standard rather than to our reading of it."""
    for name, text, bg in cases:
        assert gzip.decompress(bg) == text, name
    assert ei.bgzf_block(b"") == ei.EOF_BLOCK


def test_valid_files_inflate_exactly(emu, cases):
    for name, text, bg in cases:
        got, bad = ei.inflate_file(emu, bg)
        assert bad is None, (name, bad)
        assert got == text, name


@pytest.mark.parametrize("block", [1, 7, 150, 4096, 65280])
def test_golden_fastq_reblocked(emu, block):
    text = gzip.open(os.path.join(GOLD, "se100.fq.gz")).read()
    if block < 100:
        text = text[:2000 if block == 1 else 20000]          # tens of thousands of tiny blocks add nothing
    got, bad = ei.inflate_file(emu, ei.bgzf_write(text, 6, block=block))
    assert bad is None and got == text


def walk(emu, buf, budget=1 << 62, max_blocks=1 << 40):
    a = np.frombuffer(buf, np.uint8) if len(buf) else np.zeros(1, np.uint8)
    tab = np.zeros((4096, 8), np.uint32); cons = C.c_uint64(); outb = C.c_uint64(); stop = C.c_int()
    n = emu.kjemu_bgzf_walk(a.ctypes.data, len(buf), budget, max_blocks, tab.ctypes.data, len(tab), C.byref(cons), C.byref(outb), C.byref(stop))
    return [tuple(int(x) for x in r) for r in tab[:n]], int(cons.value), int(outb.value), int(stop.value)


def test_header_walk_across_chunk_boundaries(emu):
    """Windows that end inside a header, a payload and a trailer: the walk takes the whole blocks and resumes at the partial one."""
    text = ei.fastq_text(300, 3); bg = ei.bgzf_write(text, 6, block=9000)
    whole, cons, outb, stop = walk(emu, bg)
    assert cons == len(bg) and outb == len(text) and stop == 1
    first_end = whole[1][0] - 18          # the second block's header starts where the first block ends
    for cut in (first_end + 5, first_end + 17, first_end + 500, 2 * first_end - 3, first_end - 4, 3):
        blocks, at, total = [], 0, 0
        for win in (cut, len(bg)):          # a short first window, then everything from where the walk stopped
            t, c, o, s = walk(emu, bg[at:at + win])
            blocks += [(r[0] + at, r[4], r[5], r[6]) for r in t]; at += c; total += o
            if win == cut:
                assert s == 2 and c <= cut
        assert at == len(bg) and total == len(text)
        assert blocks == [(r[0], r[4], r[5], r[6]) for r in whole]
    t, c, o, s = walk(emu, bg, budget=20000)                    # the inflated budget ends a round between blocks
    assert s == 0 and len(t) == 2 and o == 18000
    t, c, o, s = walk(emu, bg, max_blocks=3)
    assert s == 0 and len(t) == 3
    plain_gz = gzip.compress(b"xyz")
    assert walk(emu, bg + plain_gz)[3] == 3 and walk(emu, bg + plain_gz)[1] == len(bg)      # a member that is no BGZF block
    assert walk(emu, bg + b"trailing")[3] == 4
    bad = bytearray(ei.EOF_BLOCK); bad[16:18] = struct.pack("<H", 20)                         # BSIZE smaller than header + trailer
    assert walk(emu, bytes(bad))[3] == 5


def raw(emu, payload, isize, crc):
    a = np.frombuffer(payload, np.uint8); out = np.zeros(max(isize, 1), np.uint8)
    return emu.kjemu_inflate_raw(a.ctypes.data, len(payload), out.ctypes.data, isize, crc)


class Bits:
    """LSB-first bit writer for hand-made deflate streams."""
    def __init__(self):
        self.v = 0; self.n = 0

    def put(self, value, nbits):
        self.v |= value << self.n; self.n += nbits; return self

    def code(self, value, nbits):          # Huffman codes go in most significant bit first
        for k in range(nbits - 1, -1, -1):
            self.put((value >> k) & 1, 1)
        return self

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def test_crafted_blocks_are_rejected(emu):
    data = b"ACGTACGTAAACCCGGGTTT" * 50; crc = zlib.crc32(data)
    c = zlib.compressobj(6, zlib.DEFLATED, -15); good = c.compress(data) + c.flush()
    assert raw(emu, good, len(data), crc) == 0
    assert raw(emu, good, len(data), crc ^ 1) == ERR["crc"]
    assert raw(emu, good, len(data) - 1, crc) == ERR["output"]                 # output would pass ISIZE
    assert raw(emu, good, len(data) + 1, crc) == ERR["isize"]                  # ISIZE not reached
    assert raw(emu, good[:-3], len(data), crc) == ERR["input"]                 # no end-of-block inside the payload
    assert raw(emu, good + b"\x00", len(data), crc) == ERR["trailing"]
    assert raw(emu, Bits().put(1, 1).put(3, 2).bytes(), 0, 0) == ERR["btype"]
    assert raw(emu, b"\x01\x05\x00\xfa\xfe" + b"hello", 5, zlib.crc32(b"hello")) == ERR["stored"]        # LEN != ~NLEN
    assert raw(emu, b"\x01\x05\x00\xfa\xff" + b"hello", 5, zlib.crc32(b"hello")) == 0
    assert raw(emu, b"\x01\x05\x00\xfa\xff" + b"hell", 5, zlib.crc32(b"hello")) == ERR["input"]          # stored data passes the payload
    assert raw(emu, b"\x01\x05\x00\xfa\xff" + b"hello", 4, zlib.crc32(b"hell")) == ERR["output"]
    # fixed Huffman: a match at distance 1 as the first symbol reaches before the block (length code 257 = 0000001, distance code 0 = 00000)
    assert raw(emu, Bits().put(1, 1).put(1, 2).code(1, 7).code(0, 5).code(0, 7).bytes(), 3, 0) == ERR["dist"]
    # ... after one literal it is a legal overlapping copy: 'A' + 3 x 'A'
    lit_a = (0x30 + 65, 8)
    assert raw(emu, Bits().put(1, 1).put(1, 2).code(*lit_a).code(1, 7).code(0, 5).code(0, 7).bytes(), 4, zlib.crc32(b"AAAA")) == 0
    assert raw(emu, Bits().put(1, 1).put(1, 2).code(*lit_a).code(1, 7).code(30, 5).code(0, 7).bytes(), 4, 0) == ERR["code"]       # distance code 30
    assert raw(emu, Bits().put(1, 1).put(1, 2).code(*lit_a).code(0xC6, 8).bytes(), 4, 0) == ERR["code"]                        # length code 286
    # dynamic Huffman headers: too many literal/length codes; an over-subscribed and an incomplete code-length code; a repeat with nothing before it
    assert raw(emu, Bits().put(1, 1).put(2, 2).put(30, 5).put(0, 5).put(0, 4).bytes() + b"\x00" * 8, 0, 0) == ERR["lens"]
    over = Bits().put(1, 1).put(2, 2).put(0, 5).put(0, 5).put(0, 4)
    for _ in range(4):
        over.put(1, 3)                      # four codes of length 1
    assert raw(emu, over.bytes() + b"\x00" * 8, 0, 0) == ERR["lens"]
    inc = Bits().put(1, 1).put(2, 2).put(0, 5).put(0, 5).put(0, 4).put(2, 3).put(0, 3).put(0, 3).put(0, 3)      # one code of length 2
    assert raw(emu, inc.bytes() + b"\x00" * 8, 0, 0) == ERR["lens"]
    rep = Bits().put(1, 1).put(2, 2).put(0, 5).put(0, 5).put(0, 4).put(1, 3).put(1, 3).put(0, 3).put(0, 3).code(0, 1)   # symbols 16 and 17, one bit each; first symbol: 16
    assert raw(emu, rep.bytes() + b"\x00" * 8, 0, 0) == ERR["lens"]
    assert raw(emu, b"", 0, 0) == ERR["input"]


def test_truncated_and_corrupt_files(emu):
    """The three malformed files the GPU tests run (once each): a file cut inside a block, a flipped payload bit, a wrong CRC."""
    text, bg, bad_files = ei.corrupt_files()
    assert ei.inflate_file(emu, bg) == (text, None)
    for name, data, offset in bad_files:
        got, bad = ei.inflate_file(emu, data, cap=len(text) + 70000)
        assert got is None and bad[0] == offset, (name, bad)
        assert bad[1] == {"truncated": 102, "wrong_crc": ERR["crc"]}.get(name, bad[1]) and 1 <= bad[1] <= 102, (name, bad)


def test_random_bit_flips_never_pass_silently(emu):
    """A flipped bit in a payload either breaks the stream or is caught by the CRC; one in a trailer is a CRC or ISIZE error; none may
    touch memory outside the block's buffers (the sanitised run of this module checks that)."""
    rng = np.random.default_rng(11); text = ei.fastq_text(60, 9)
    files = [ei.bgzf_write(text, lv, st, block=3000) for lv, st in ((1, zlib.Z_DEFAULT_STRATEGY), (6, zlib.Z_DEFAULT_STRATEGY), (9, zlib.Z_FIXED), (0, zlib.Z_DEFAULT_STRATEGY))]
    flips = 60 if SANITIZE else 300
    for k in range(flips):
        f = bytearray(files[k % len(files)]); ends = list(ei._block_ends(bytes(f)))
        b = int(rng.integers(0, len(ends) - 1)); start = ends[b - 1] if b else 0
        pos = int(rng.integers(start + 18, ends[b])); f[pos] ^= 1 << int(rng.integers(0, 8))
        got, bad = ei.inflate_file(emu, bytes(f), cap=len(text) + 70000)
        if got is None:
            assert bad[0] == start and (1 <= bad[1] <= 11 or bad[1] == 105), (k, pos, bad)      # 105: an ISIZE above 65,536 stops the header walk
        else:
            assert got == text, (k, pos)          # the padding bits behind the last code of a block carry nothing


@pytest.mark.skipif(SANITIZE, reason="this is the sanitised run")
def test_module_passes_under_address_and_undefined_sanitizers():
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__)], env=ei.sanitizer_env(),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
