"""The CPU warp emulator on the compact spread layout (tests/emu/kj_emu_spread.cpp), compiled on first use into a directory of the caller's
choosing (test infrastructure: the library picks the spread instances on the device).  long=True builds the long-read instances."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def load(out_dir, params_type, long=False):
    """ctypes handle of the emulator, built into out_dir; params_type = the kj_params ctypes structure."""
    so = os.path.join(out_dir, "libkjemu_spread%s.so" % ("_long" if long else ""))
    if not os.path.exists(so):
        os.makedirs(out_dir, exist_ok=True)
        tmp = so + ".%d" % os.getpid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DKJ_EMU"] + (["-DKJ_EMU_SPREAD_LONG"] if long else []) +
                              ["-o", tmp, os.path.join(HERE, "emu", "kj_emu_spread.cpp"), os.path.join(ROOT, "kaiju_b200", "csrc", "kj_host.cpp"), "-lpthread"])
        os.replace(tmp, so)
    E = C.CDLL(so)
    E.kjemu_create.restype = C.c_void_p; E.kjemu_create.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(params_type)]
    E.kjemu_destroy.argtypes = [C.c_void_p]
    E.kjemu_classify.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64, C.c_void_p, C.c_void_p, C.c_int]
    E.kjemu_layout.restype = C.c_int; E.kjemu_layout.argtypes = [C.c_void_p, C.POINTER(C.c_uint), C.POINTER(C.c_ulonglong)]
    return E
