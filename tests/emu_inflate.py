"""The BGZF inflate code on the CPU warp emulator (tests/emu/kj_emu_inflate.cpp), compiled on first use into a directory of the caller's choosing,
and what the inflate tests share: a BGZF writer built on Python's zlib and the set of valid files both the emulator and the GPU are checked on."""
import ctypes as C
import os
import struct
import subprocess
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
MAX_SLICE = 65280


def load(out_dir, sanitize=False):
    """ctypes handle of the emulator, built into out_dir.  sanitize: built with the address and undefined-behaviour sanitisers (the process
    that loads it must have the sanitiser runtime preloaded, see sanitizer_env)."""
    so = os.path.join(out_dir, "libkjemu_inflate%s.so" % ("_san" if sanitize else ""))
    if not os.path.exists(so):
        os.makedirs(out_dir, exist_ok=True)
        tmp = so + ".%d" % os.getpid()
        flags = ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-fno-omit-frame-pointer"] if sanitize else ["-O2"]
        subprocess.check_call(["g++"] + flags + ["-std=c++17", "-fPIC", "-shared", "-DKJ_EMU", "-o", tmp, os.path.join(HERE, "emu", "kj_emu_inflate.cpp"),
                                                  os.path.join(ROOT, "kaiju_b200", "csrc", "kj_host.cpp"), "-lpthread"])
        os.replace(tmp, so)
    E = C.CDLL(so)
    E.kjemu_inflate_raw.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32]
    E.kjemu_bgzf_walk.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int)]
    E.kjemu_inflate_bgzf.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    return E


def sanitizer_env():
    """Environment of a Python process that can load the sanitised emulator."""
    libs = [subprocess.check_output(["gcc", "-print-file-name=lib%s.so" % n], text=True).strip() for n in ("asan", "ubsan")]
    return dict(os.environ, LD_PRELOAD=" ".join(libs), ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", UBSAN_OPTIONS="halt_on_error=1", KJ_EMU_INFLATE_SANITIZE="1")


def inflate_file(E, data, cap=None):
    """(text, None) or (None, (compressed offset of the first bad block, error code))"""
    buf = np.frombuffer(bytes(data), dtype=np.uint8) if len(data) else np.zeros(0, np.uint8)
    cap = cap if cap is not None else sum(struct.unpack("<I", data[i - 4:i])[0] for i in _block_ends(data)) + 16
    out = np.zeros(cap + 1, np.uint8); n = C.c_uint64(); off = C.c_uint64(); err = C.c_uint32()
    rc = E.kjemu_inflate_bgzf(buf.ctypes.data, len(buf), out.ctypes.data, cap, C.byref(n), C.byref(off), C.byref(err))
    if rc:
        return None, (int(off.value), int(err.value))
    return out[:n.value].tobytes(), None


def _block_ends(data):
    """End offsets of the blocks of a well-formed BGZF file (bad headers end the list: only used to size the output buffer)."""
    at = 0
    while at + 18 <= len(data) and data[at:at + 4] == b"\x1f\x8b\x08\x04" and data[at + 12:at + 14] == b"BC":
        at += struct.unpack("<H", data[at + 16:at + 18])[0] + 1
        if at > len(data):
            return
        yield at


def bgzf_block(raw, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, payload=None):
    """One BGZF block holding `raw` (at most 65,536 bytes); payload: a deflate stream to wrap instead of compressing raw."""
    if payload is None:
        c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy); payload = c.compress(raw) + c.flush()
    bsize = 18 + len(payload) + 8
    assert bsize <= 65536 and len(raw) <= 65536
    return b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", bsize - 1) + payload + struct.pack("<II", zlib.crc32(raw), len(raw))


def bgzf_write(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, block=MAX_SLICE, eof=True):
    """`data` as a BGZF file: slices of at most `block` bytes, one gzip member each, and the empty end-of-file block."""
    out = [bgzf_block(data[i:i + block], level, strategy) for i in range(0, len(data), block)]
    return b"".join(out) + (EOF_BLOCK if eof else b"")


def fastq_text(n, seed, read_len=150):
    rng = np.random.default_rng(seed)
    seqs = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=(n, read_len)); quals = rng.integers(35, 75, size=(n, read_len), dtype=np.uint8)
    return b"".join(b"@read%d/1\n%s\n+\n%s\n" % (i, seqs[i].tobytes(), quals[i].tobytes()) for i in range(n))


def valid_files():
    """(name, text, BGZF bytes) of every well-formed case both decoders must inflate exactly."""
    rng = np.random.default_rng(7)
    fq = fastq_text(700, 1)
    cases = []
    for lv in range(10):
        cases.append(("level%d" % lv, fq, bgzf_write(fq, lv)))
    for nm, st in (("fixed", zlib.Z_FIXED), ("huffman_only", zlib.Z_HUFFMAN_ONLY), ("rle", zlib.Z_RLE), ("filtered", zlib.Z_FILTERED)):
        cases.append((nm, fq, bgzf_write(fq, 6, st)))
    runs = b"".join(bytes([65 + i % 20]) * int(k) for i, k in enumerate(rng.integers(1, 700, 400)))[:200000]
    cases.append(("rle_runs", runs, bgzf_write(runs, 6, zlib.Z_RLE)))
    # several deflate blocks in one BGZF block: a full flush in the middle leaves an empty stored block behind it
    a, b = fq[:20000], fq[20000:45000]
    c = zlib.compressobj(6, zlib.DEFLATED, -15); pl = c.compress(a) + c.flush(zlib.Z_FULL_FLUSH) + c.compress(b) + c.flush()
    cases.append(("full_flush", a + b, bgzf_block(a + b, payload=pl) + EOF_BLOCK))
    noise = rng.integers(0, 256, MAX_SLICE, dtype=np.uint8).tobytes()
    cases.append(("random_stored", noise, bgzf_write(noise, 6)))
    # matches of length 258 at distance 32,768: a random 32 KiB window, then the same window again
    win = rng.integers(0, 256, 32768, dtype=np.uint8).tobytes()
    cases.append(("far_matches", win + win[:32000], bgzf_write(win + win[:32000], 9)))
    cases.append(("one_byte", b"A", bgzf_write(b"A")))
    cases.append(("empty_blocks", fq[:3000], EOF_BLOCK + bgzf_write(fq[:1500], eof=False) + EOF_BLOCK + bgzf_block(b"") + bgzf_write(fq[1500:3000]) + EOF_BLOCK))
    cases.append(("only_eof", b"", EOF_BLOCK))
    cases.append(("no_eof_block", fq[:5000], bgzf_write(fq[:5000], eof=False)))
    return cases


def corrupt_files():
    """(name, text, bytes, compressed offset of the block that must be reported) of the malformed files the GPU tests run once each, after the
    sanitised emulator has shown that they stay inside their buffers."""
    text = fastq_text(400, 5); bg = bgzf_write(text, 6, block=20000)
    second = next(iter(_block_ends(bg)))
    flipped = bytearray(bg); flipped[second + 18 + 200] ^= 0x10
    wrong = bytearray(bg); wrong[second - 8] ^= 0xff                      # the first block's CRC-32
    return text, bg, [("truncated", bg[:second + 300], second), ("flipped_bit", bytes(flipped), second), ("wrong_crc", bytes(wrong), 0)]
