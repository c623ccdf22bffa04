"""Developer tool (CPU only): the UNMODIFIED reference binary (oracle/_ref/kaiju) against the kernel logic on the CPU warp emulator, directly,
on a fresh seeded workload of N read items per configuration (PE150, SE100, PE250 x MEM / Greedy parameter sets).  Usage: python tools/soak.py 1000000"""
import sys, time, numpy as np, ctypes as C, os, tempfile
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from conftest import ROOT
from helpers import *
from test_kernel_logic_emulated import KjParams
E = C.CDLL(os.path.join(ROOT, "tests", "emu", "libkjemu.so"))
E.kjemu_create.restype = C.c_void_p; E.kjemu_create.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(KjParams)]
E.kjemu_destroy.argtypes = [C.c_void_p]
E.kjemu_classify.argtypes = [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64, C.c_void_p, C.c_void_p, C.c_int]
d = tempfile.mkdtemp(prefix="kjsoak_")
db = SynthDB(60000, 21); db.write(d + "/db.faa", d + "/nodes.dmp"); fmi = build_fmi(d + "/db.faa", d + "/db", threads=8)
n = int(sys.argv[1])
for (rl, paired, seed) in ((150, True, 301), (100, False, 302), (250, True, 303)):
    fq1, fq2 = d + "/a.fq", d + "/b.fq"
    db.write_fastq(seed, 0, n, rl, paired, fq1, fq2 if paired else None)
    n1, s1, o1 = read_fastq_packed(fq1); s2 = o2 = None
    if paired: _, s2, o2 = read_fastq_packed(fq2)
    for kw in [dict(mode="mem"), dict(mode="greedy"), dict(mode="greedy", e=5, s=50), dict(mode="mem", m=8, seg=False)]:
        t0 = time.time(); ref = run_ref_kaiju(d + "/nodes.dmp", fmi, fq1, fq2 if paired else None, threads=8, **kw); t1 = time.time()
        P = make_params(**kw); kp = KjParams(**P); h = E.kjemu_create(fmi.encode(), (d + "/nodes.dmp").encode(), C.byref(kp))
        tax = np.zeros(n, dtype=np.uint64); best = np.zeros(n, dtype=np.uint32)
        rc = E.kjemu_classify(h, s1.ctypes.data, o1.ctypes.data, s2.ctypes.data if paired else None, o2.ctypes.data if paired else None, n, tax.ctypes.data, best.ctypes.data, 8); E.kjemu_destroy(h)
        bad = [i for i, nm in enumerate(n1) if (ref[nm][1], ref[nm][2]) != (int(tax[i]), int(best[i]))]
        print(rl, paired, kw, "rc", rc, "reference-vs-kernel-logic bad", len(bad), bad[:3], "ref %.0fs emu %.0fs" % (t1 - t0, time.time() - t1), flush=True)
