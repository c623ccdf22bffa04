#!/usr/bin/env python
"""Developer tool: what inflating BGZF input on the GPU buys.  One call measures, on the card whose name and power limit it prints,
  1. the inflate kernel alone: a whole BGZF file of synthetic PE150 FASTQ (>= 1 GB of text) through kj_debug_inflate_bgzf, CUDA events around the
     kernel, several launches after a warm-up, at deflate levels 1 and 6 (CRC-32 verification is part of the kernel and cannot be left out);
  2. file -> file through the CLI (first byte read -> last byte written, timed inside it): the same reads as plain text, `gzip -1`, BGZF level 1 and
     BGZF level 6, alternated over several rounds, outputs compared byte for byte.
Usage: python tools/inflate_bench.py [--pairs 4000000] [--nprot 200000] [--rounds 2] [--mode mem]"""
import argparse, hashlib, json, os, subprocess, sys, time
from multiprocessing import Pool
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def _pack(job):
    from emu_inflate import bgzf_write
    path, off, n, level = job
    with open(path, "rb") as f:
        f.seek(off); return bgzf_write(f.read(n), level, eof=False)


def write_bgzf(src, dst, level, pool):
    from emu_inflate import EOF_BLOCK, MAX_SLICE
    size = os.path.getsize(src); step = MAX_SLICE * 256
    with open(dst, "wb") as out:
        for part in pool.imap(_pack, [(src, o, min(step, size - o), level) for o in range(0, size, step)]):
            out.write(part)
        out.write(EOF_BLOCK)


def sha(path):
    h = hashlib.sha1()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nprot", type=int, default=200000); ap.add_argument("--mode", default="mem"); ap.add_argument("--pairs", type=int, default=4_000_000)
    ap.add_argument("--rounds", type=int, default=2); ap.add_argument("--launches", type=int, default=3); ap.add_argument("--workdir", default=os.environ.get("KJ_BENCH_DIR", "/tmp/kjbench"))
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("inflate_bench: no CUDA device (nothing is measured without one)")
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
    import kaiju_b200 as kb
    from helpers import SynthDB, build_fmi
    os.makedirs(a.workdir, exist_ok=True)
    db = SynthDB(a.nprot, 1); fmi = os.path.join(a.workdir, "synth_%d.fmi" % a.nprot); nodes = os.path.join(a.workdir, "synth_%d_nodes.dmp" % a.nprot)
    if not os.path.exists(fmi):
        faa = os.path.join(a.workdir, "synth_%d.faa" % a.nprot); db.write(faa, nodes); build_fmi(faa, os.path.join(a.workdir, "synth_%d" % a.nprot), threads=min(32, os.cpu_count()))
    plain = [os.path.join(a.workdir, "ib_%d_%d.fq" % (a.pairs, m)) for m in (1, 2)]
    if not os.path.exists(plain[0]):
        db.write_fastq(7, 0, a.pairs, 150, True, plain[0], plain[1])
    files = {"plain": plain, "gzip-1": [p + ".gz" for p in plain], "bgzf-1": [p + ".l1.bgz" for p in plain], "bgzf-6": [p + ".l6.bgz" for p in plain]}
    with Pool(os.cpu_count()) as pool:
        gz = [subprocess.Popen("gzip -1 -k -f " + p, shell=True) for p in plain if not os.path.exists(p + ".gz")]
        for p in plain:
            for lv in (1, 6):
                if not os.path.exists(p + ".l%d.bgz" % lv):
                    write_bgzf(p, p + ".l%d.bgz" % lv, lv, pool)
        for g in gz:
            assert g.wait() == 0
    text_bytes = sum(os.path.getsize(p) for p in plain)
    res = {"card": card, "pairs": a.pairs, "mode": a.mode, "text_GB": text_bytes / 1e9, "input_GB": {k: sum(os.path.getsize(p) for p in v) / 1e9 for k, v in files.items()}}

    # 1. the kernel alone
    clf = kb.Classifier(fmi, nodes, device=0, params=kb.make_params(a.mode))
    want = open(plain[0], "rb").read(); res["kernel"] = {}
    for lv in (1, 6):
        data = open(files["bgzf-%d" % lv][0], "rb").read(); ms = []
        for k in range(a.launches + 1):
            got = clf.debug_inflate_bgzf(data, out_cap=len(want))
            if k == 0:
                assert got == want, "the inflate kernel's text differs from the plain file"
            else:
                ms.append(clf.last_kernel_ms)
            del got
        res["kernel"]["bgzf-%d" % lv] = {"inflated_GB": len(want) / 1e9, "compressed_GB": len(data) / 1e9, "kernel_ms": ms, "inflated_GB_per_s": len(want) / 1e6 / min(ms)}
    clf.close(); del want, data

    # 2. file -> file through the CLI
    cli = [os.path.join(ROOT, "kaiju_b200", "kaiju-b200"), "-t", nodes, "-f", fmi, "-a", a.mode]
    for v in files.values():
        for p in v:
            open(p, "rb").read()                      # page cache warm for every encoding
    secs = {k: [] for k in files}; digest = {}; traces = {}
    for r in range(a.rounds + 1):                   # round 0 warms up
        for k, v in files.items():
            out = os.path.join(a.workdir, "ib_out_%s.tsv" % k)
            p = subprocess.run(cli + ["-i", v[0], "-j", v[1], "-o", out], stderr=subprocess.PIPE, text=True, check=True, env=dict(os.environ, KJ_CLI_TIMING="1", KJ_FILES_TRACE="1"))
            inner = [float(l.split(" classified, ")[1].split(" s")[0]) for l in p.stderr.splitlines() if " classified, " in l]
            infl = [int(l.split(": ")[1].split(" bytes")[0]) for l in p.stderr.splitlines() if "inflated on the device" in l and "KJ_FILES_TRACE" not in l]
            if r:
                secs[k].append(inner[0])
            traces[k] = [l for l in p.stderr.splitlines() if "KJ_FILES_TRACE" in l]
            assert infl[0] == (text_bytes if k.startswith("bgzf") else 0), (k, infl)
            if r == 0:
                digest[k] = sha(out)
    assert len(set(digest.values())) == 1, digest
    res["files"] = {k: {"seconds": s, "pairs_per_s": a.pairs / min(s), "text_GB_per_s": text_bytes / 1e9 / min(s)} for k, s in secs.items()}
    res["outputs_identical"] = True; res["trace_last_round"] = traces
    print(json.dumps(res))


if __name__ == "__main__":
    main()
