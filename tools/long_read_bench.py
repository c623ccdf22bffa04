"""Long-read throughput: bases/s of the GPU path per read-length bin (5, 20, 50, 200 kb, 1 Mb; MEM and Greedy) next to the reference
`kaiju -z <nproc>` on the same reads and host, and the cost of one long read inside a batch of short ones.  One JSON line per measurement.

Usage: python tools/long_read_bench.py [--bases-per-bin N] [--skip-cpu]
Reads come from the synthetic generator (tools/kjgen.c) against the golden index (tests/golden); the reference binary is oracle/_ref/kaiju."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bases-per-bin", type=int, default=4_000_000)
    ap.add_argument("--skip-cpu", action="store_true")
    a = ap.parse_args()
    import numpy as np
    import __graft_entry__ as ge
    ge.build()
    import kaiju_b200 as kb
    from conftest import Golden
    from helpers import REF_DIR, SynthDB, have_ref
    g = Golden(); db = SynthDB(800, 3); card = gpu_info(); nproc = os.cpu_count()
    d = tempfile.mkdtemp(prefix="kjlong_")
    for mode in ("mem", "greedy"):
        clf = kb.Classifier(g.fmi, g.nodes, device=0, params=kb.make_params(mode), max_read_len=kb.MAX_LONG_READ_LEN)
        for length in (5000, 20000, 50000, 200000, 1000000):
            n = max(2, a.bases_per_bin // length)
            s, o = db.long_reads(90 + length % 97, 0, n, length, length)
            clf.classify(s, o)                                            # warm-up: scratch sized, modules loaded
            t = time.perf_counter(); clf.classify(s, o); dt = time.perf_counter() - t
            rec = {"mode": mode, "read_len": length, "reads": n, "bases": int(o[-1]), "gpu_bases_per_s": o[-1] / dt, "gpu_s": dt, "gpu": card}
            if not a.skip_cpu and have_ref():
                fq = os.path.join(d, "r.fq")
                with open(fq, "w") as f:
                    for i in range(n):
                        r = bytes(s[o[i]:o[i + 1]]).decode(); f.write("@r%d\n%s\n+\n%s\n" % (i, r, "I" * len(r)))
                cmd = [os.path.join(REF_DIR, "kaiju"), "-t", g.nodes, "-f", g.fmi, "-i", fq, "-a", mode, "-z", str(nproc), "-o", os.path.join(d, "ref.out")]
                t = time.perf_counter(); subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL); ct = time.perf_counter() - t
                rec.update(cpu_bases_per_s=o[-1] / ct, cpu_s=ct, cpu_threads=nproc, gpu_over_cpu=ct / dt)
            print(json.dumps({k: (float(v) if isinstance(v, (np.floating, np.integer)) else v) for k, v in rec.items()}), flush=True)
        clf.close()
    # one long read inside a batch of short ones: the long read gets a chunk of its own, the short reads keep the short kernels
    clf = kb.Classifier(g.fmi, g.nodes, device=0, params=kb.make_params("mem"), max_read_len=kb.MAX_LONG_READ_LEN)
    s1, o1, _, _ = db.reads(95, 0, 1_000_000, 150, paired=False)
    ls, lo = db.long_reads(96, 0, 1, 1000000, 1000000)
    half = len(o1) // 2
    mixed = np.concatenate([s1[:o1[half]], ls, s1[o1[half]:]])
    mo = np.concatenate([o1[:half + 1], (o1[half:] + lo[-1])]).astype(np.uint64)
    for name, (s, o) in (("short_only", (s1, o1)), ("short_plus_one_1Mb_read", (mixed, mo)), ("one_1Mb_read", (ls, lo))):
        clf.classify(s, o); t = time.perf_counter(); clf.classify(s, o); dt = time.perf_counter() - t
        print(json.dumps({"mode": "mem", "batch": name, "reads": int(len(o) - 1), "s": dt, "gpu": card}), flush=True)
    clf.close()


if __name__ == "__main__":
    main()
