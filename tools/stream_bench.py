#!/usr/bin/env python
"""Developer tool: what reading the input from a FIFO costs against reading it from a regular file.  The workload of tools/inflate_bench.py
(synthetic PE150 pairs, a synthetic protein index, MEM): file -> file and FIFO -> file through the CLI (first byte read -> last byte written,
timed inside it) for plain text, BGZF level 1, BGZF level 6 and `gzip -1`.  In the FIFO arm one `cat` per mate copies the file (from the page
cache) into a FIFO.  The arms alternate; one warm-up round, then --rounds timed ones; every output is compared byte for byte with the first.
Prints the card's name and power limit from the same run, and one JSON line.
Usage: python tools/stream_bench.py [--pairs 4000000] [--nprot 100000] [--rounds 2] [--mode mem]"""
import argparse, json, os, subprocess, sys, tempfile
from multiprocessing import Pool
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nprot", type=int, default=100000); ap.add_argument("--mode", default="mem"); ap.add_argument("--pairs", type=int, default=4_000_000)
    ap.add_argument("--rounds", type=int, default=2); ap.add_argument("--workdir", default=os.environ.get("KJ_BENCH_DIR", "/tmp/kjbench"))
    a = ap.parse_args()
    from inflate_bench import sha, write_bgzf
    from helpers import SynthDB, build_fmi
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
    os.makedirs(a.workdir, exist_ok=True)
    db = SynthDB(a.nprot, 1); fmi = os.path.join(a.workdir, "synth_%d.fmi" % a.nprot); nodes = os.path.join(a.workdir, "synth_%d_nodes.dmp" % a.nprot)
    if not os.path.exists(fmi):
        faa = os.path.join(a.workdir, "synth_%d.faa" % a.nprot); db.write(faa, nodes); build_fmi(faa, os.path.join(a.workdir, "synth_%d" % a.nprot), threads=min(32, os.cpu_count()))
    plain = [os.path.join(a.workdir, "ib_%d_%d.fq" % (a.pairs, m)) for m in (1, 2)]
    if not os.path.exists(plain[0]):
        db.write_fastq(7, 0, a.pairs, 150, True, plain[0], plain[1])
    files = {"plain": plain, "bgzf-1": [p + ".l1.bgz" for p in plain], "bgzf-6": [p + ".l6.bgz" for p in plain], "gzip-1": [p + ".gz" for p in plain]}
    with Pool(os.cpu_count()) as pool:
        gz = [subprocess.Popen("gzip -1 -k -f " + p, shell=True) for p in plain if not os.path.exists(p + ".gz")]
        for p in plain:
            for lv in (1, 6):
                if not os.path.exists(p + ".l%d.bgz" % lv):
                    write_bgzf(p, p + ".l%d.bgz" % lv, lv, pool)
        for g in gz:
            assert g.wait() == 0
    text_bytes = sum(os.path.getsize(p) for p in plain)
    for v in files.values():
        for p in v:
            open(p, "rb").read()                          # page cache warm for every encoding
    cli = [os.path.join(ROOT, "kaiju_b200", "kaiju-b200"), "-t", nodes, "-f", fmi, "-a", a.mode]
    fifo_dir = tempfile.mkdtemp(prefix="kjstream_"); fifos = [os.path.join(fifo_dir, "m%d" % m) for m in (1, 2)]
    for f in fifos:
        os.mkfifo(f)
    secs = {(k, arm): [] for k in files for arm in ("file", "fifo")}; digest = {}; inflated = {}
    try:
        for r in range(a.rounds + 1):                 # round 0 warms up
            for k, v in files.items():
                for arm in ("file", "fifo"):
                    out = os.path.join(a.workdir, "sb_out_%s_%s.tsv" % (k, arm))
                    cats = [subprocess.Popen("exec cat '%s' > '%s'" % (p, f), shell=True) for p, f in zip(v, fifos)] if arm == "fifo" else []
                    try:
                        ins = v if arm == "file" else fifos
                        p = subprocess.run(cli + ["-i", ins[0], "-j", ins[1], "-o", out], stderr=subprocess.PIPE, text=True, env=dict(os.environ, KJ_CLI_TIMING="1"), timeout=600)
                    finally:
                        for c in cats:
                            c.wait(60)
                    assert p.returncode == 0 and all(c.returncode == 0 for c in cats), p.stderr[-2000:]
                    inner = [float(l.split(" classified, ")[1].split(" s")[0]) for l in p.stderr.splitlines() if " classified, " in l]
                    inflated[(k, arm)] = [int(l.split(": ")[1].split(" bytes")[0]) for l in p.stderr.splitlines() if "inflated on the device" in l][0]
                    if r:
                        secs[(k, arm)].append(inner[0])
                    else:
                        digest[(k, arm)] = sha(out)
    finally:
        for f in fifos:
            os.unlink(f)
        os.rmdir(fifo_dir)
    assert len(set(digest.values())) == 1, digest
    for k in files:
        assert inflated[(k, "file")] == inflated[(k, "fifo")] == (text_bytes if k.startswith("bgzf") else 0), (k, inflated)
    res = {"card": card, "pairs": a.pairs, "mode": a.mode, "text_GB": text_bytes / 1e9, "input_GB": {k: sum(os.path.getsize(p) for p in v) / 1e9 for k, v in files.items()},
           "runs": {"%s %s" % key: {"seconds": s, "pairs_per_s": a.pairs / min(s), "text_GB_per_s": text_bytes / 1e9 / min(s)} for key, s in secs.items()},
           "outputs_identical": True}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
