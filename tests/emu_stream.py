"""The stream side of the file pipeline's reader on the CPU (tests/emu/kj_emu_stream.cpp), compiled on first use into a directory of the caller's
choosing, and what the stream tests share: writer threads that feed a pipe or a FIFO in random pieces with pauses."""
import ctypes as C
import os
import random
import subprocess
import threading
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def load(out_dir, sanitize=False):
    """ctypes handle of the harness, built into out_dir (sanitize: as emu_inflate.load)."""
    so = os.path.join(out_dir, "libkjemu_stream%s.so" % ("_san" if sanitize else ""))
    if not os.path.exists(so):
        os.makedirs(out_dir, exist_ok=True)
        tmp = so + ".%d" % os.getpid()
        flags = ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-fno-omit-frame-pointer"] if sanitize else ["-O2"]
        subprocess.check_call(["g++"] + flags + ["-std=c++17", "-fPIC", "-shared", "-DKJ_EMU", "-o", tmp, os.path.join(HERE, "emu", "kj_emu_stream.cpp"),
                                                  os.path.join(ROOT, "kaiju_b200", "csrc", "kj_host.cpp"), "-lz", "-lpthread"])
        os.replace(tmp, so)
    E = C.CDLL(so)
    E.kjemu_stream_new.restype = C.c_void_p; E.kjemu_stream_new.argtypes = [C.c_int]
    E.kjemu_stream_halt.argtypes = [C.c_void_p]; E.kjemu_stream_free.argtypes = [C.c_void_p]
    E.kjemu_stream_read.argtypes = [C.c_void_p, C.c_uint64, C.c_char_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                    C.c_char_p, C.c_uint64]
    E.kjemu_gzread_file.argtypes = [C.c_char_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    return E


class Reader:
    """One KjStream over descriptor fd (which it takes); read() runs the reader's logic to the end of the stream."""
    def __init__(self, E, fd):
        self.E = E; self.s = E.kjemu_stream_new(fd)
        assert self.s

    def read(self, chunk, cap, path="<stream>"):
        """(rc, text, device-inflated bytes, chunks, message)"""
        out = np.zeros(cap + 1, np.uint8); n = C.c_uint64(); inf = C.c_uint64(); ch = C.c_uint64(); msg = C.create_string_buffer(512)
        rc = self.E.kjemu_stream_read(self.s, chunk, path.encode(), out.ctypes.data, cap, C.byref(n), C.byref(inf), C.byref(ch), msg, len(msg))
        return rc, out[:n.value].tobytes(), int(inf.value), int(ch.value), msg.value.decode()

    def halt(self):
        self.E.kjemu_stream_halt(self.s)

    def close(self):
        self.E.kjemu_stream_free(self.s); self.s = None


def gzread_file(E, path, cap):
    """(rc, text) of gzread over a file: rc 0, or 1 where gzread returns -1"""
    out = np.zeros(cap + 1, np.uint8); n = C.c_uint64()
    rc = E.kjemu_gzread_file(path.encode(), out.ctypes.data, cap, C.byref(n))
    return rc, out[:n.value].tobytes()


def pieces(data, seed, pauses=(), max_piece=1 << 20):
    """data cut into pieces of 1 byte to max_piece bytes, each with a pause before it (seconds); the offsets in `pauses` start a piece that
    follows a pause of 0.05 s, so a reader finds the stream stalled exactly there."""
    rng = random.Random(seed); cuts = sorted(set(p for p in pauses if 0 < p < len(data))); out = []; at = 0
    while at < len(data):
        nxt = min([c for c in cuts if c > at] + [len(data)])
        size = min(nxt - at, rng.choice([1, rng.randint(1, 300), rng.randint(1, 70000), rng.randint(1, max_piece)]))
        out.append((0.05 if at in cuts else (0.002 if rng.random() < 0.05 else 0.0), data[at:at + size])); at += size
    return out


class Writer(threading.Thread):
    """Writes `data` in the pieces of pieces() to path (opened here: a FIFO's open waits for its reader) or to descriptor fd, then closes it.
    stall: seconds to keep the descriptor open after the last byte.  A reader that stops early ends the writer with BrokenPipeError."""
    def __init__(self, data, seed, path=None, fd=None, pauses=(), stall=0.0, max_piece=1 << 20):
        super().__init__(daemon=True)
        self.path, self.fd, self.stall = path, fd, stall
        self.parts = pieces(data, seed, pauses, max_piece); self.broken = False; self.error = None; self.release = threading.Event()

    def run(self):
        try:
            fd = self.fd if self.fd is not None else os.open(self.path, os.O_WRONLY)
            try:
                for pause, b in self.parts:
                    if pause:
                        time.sleep(pause)
                    mv = memoryview(b)
                    while len(mv):
                        mv = mv[os.write(fd, mv):]
                if self.stall:
                    self.release.wait(self.stall)
            finally:
                os.close(fd)
        except BrokenPipeError:
            self.broken = True
        except Exception as e:          # reported by the test that joins the writer
            self.error = e

    def finish(self, timeout=60):
        self.release.set(); self.join(0.5)
        if self.is_alive() and self.path:        # still in open(): the reader never opened the FIFO; open it for reading once so the writer ends
            try:
                os.close(os.open(self.path, os.O_RDONLY | os.O_NONBLOCK))
            except OSError:
                pass
        self.join(timeout)
        assert not self.is_alive(), "writer thread still running"
        assert self.error is None, self.error
