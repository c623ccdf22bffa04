#!/usr/bin/env python
"""Developer tool: what classifying one input file on several contexts costs or gains (kj_classify_files_multi).  One call measures file -> file
time, one context against N contexts, alternated over several rounds, outputs compared byte for byte, on the card whose name and power limit
it prints:
  1. the synth-viruses index of bench.py through the CLI: `-d 0` against `-d <devices>` (replicas) and `-d <devices> -P` (a group: the compact
     spread layout instead of the narrow one) (KJ_CLI_TIMING: first byte read -> last byte written, timed inside the CLI), MEM and Greedy;
  2. the same index scaled to --big-rows BWT rows (2.7e10 = 135 copies, compact layout) through the Python API: one group of the --devices,
     kj_classify_files on its first context against kj_classify_files_multi over all of them (host clock around the call, which returns after
     the last byte is written), MEM and Greedy.
With every device 0 (the default `0,0`), this is the cost of the multi-context machinery on one card; a gain needs distinct GPUs.
Usage: python tools/files_multi_bench.py [--devices 0,0] [--pairs 4000000] [--rounds 3] [--big-rows 2.7e10]"""
import argparse, hashlib, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

MODES = {"mem": ["-a", "mem", "-m", "11"], "greedy": ["-a", "greedy", "-e", "3", "-s", "65"]}


def sha(path):
    h = hashlib.sha1()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--devices", default="0,0"); ap.add_argument("--pairs", type=int, default=4_000_000); ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--nprot", type=int, default=680000); ap.add_argument("--big-rows", type=float, default=2.7e10)
    ap.add_argument("--workdir", default=os.environ.get("KJ_BENCH_DIR", "/tmp/kjbench"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("files_multi_bench: no CUDA device (nothing is measured without one)")
    devices = [int(x) for x in a.devices.split(",")]
    cards = subprocess.check_output(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip().splitlines()
    import bench
    import kaiju_b200 as kb
    db, fmi, nodes = bench.build_workload(a, 0)
    fq = [os.path.join(a.workdir, "fm_%d_%d.fq" % (a.pairs, m)) for m in (1, 2)]
    if not os.path.exists(fq[1]):
        db.write_fastq(7, 0, a.pairs, 150, True, fq[0], fq[1])
    for p in fq:
        open(p, "rb").read()                          # page cache warm
    res = {"cards": cards, "devices": devices, "pairs": a.pairs, "rounds": a.rounds, "text_GB": sum(os.path.getsize(p) for p in fq) / 1e9}

    # 1. the CLI on the synth-viruses index
    cli = [os.path.join(ROOT, "kaiju_b200", "kaiju-b200"), "-t", nodes, "-f", fmi, "-i", fq[0], "-j", fq[1]]
    # replicas: the same layout as `one` (narrow for this index), so the difference is the multi-context machinery; pool: a group (compact spread)
    arms = {"one": ["-d", str(devices[0])], "replicas": ["-d", a.devices], "pool": ["-d", a.devices, "-P"]}
    res["cli"] = {}
    for mode, mopt in MODES.items():
        secs = {k: [] for k in arms}; digest = {}
        for r in range(a.rounds + 1):                 # round 0 warms up
            for k, dopt in arms.items():
                out = os.path.join(a.workdir, "fm_out_%s.tsv" % k)
                p = subprocess.run(cli + mopt + dopt + ["-o", out], stderr=subprocess.PIPE, text=True, env=dict(os.environ, KJ_CLI_TIMING="1"))
                if p.returncode:
                    sys.exit("files_multi_bench: %s failed:\n%s" % (" ".join(mopt + dopt), p.stderr))
                inner = [float(l.split(" classified, ")[1].split(" s")[0]) for l in p.stderr.splitlines() if " classified, " in l]
                if r:
                    secs[k].append(inner[0])
                else:
                    digest[k] = sha(out)
        assert len(set(digest.values())) == 1, (mode, digest)
        res["cli"][mode] = {k: {"seconds": s, "pairs_per_s": a.pairs / min(s)} for k, s in secs.items()}
        for k in ("replicas", "pool"):
            res["cli"][mode][k + "_over_one"] = min(secs["one"]) / min(secs[k])

    # 2. the Python API on the scaled index (compact records), one group
    base = kb.Classifier(fmi, nodes, device=devices[0], params=kb.make_params("mem")); rows = base.bwtlen; base.close()
    copies = max(2, int(round(a.big_rows / rows)))
    grp = kb.create_group(fmi, nodes, devices, params=kb.make_params("mem", m=11), copies=copies)
    res["big"] = {"copies": copies, "bwt_rows": grp[0].bwtlen, "index_bytes": grp[0].index_bytes}
    try:
        for mode in MODES:
            for g in grp:
                g.set_params(kb.make_params(mode, m=11, e=3, s=65))
            secs = {"one": [], "multi": []}; digest = {}
            for r in range(a.rounds + 1):
                for k in ("one", "multi"):
                    out = os.path.join(a.workdir, "fm_big_%s.tsv" % k); t0 = time.perf_counter()
                    n, _ = grp[0].classify_files(fq[0], fq[1], out) if k == "one" else kb.classify_files_multi(grp, fq[0], fq[1], out)
                    dt = time.perf_counter() - t0
                    assert n == a.pairs
                    if r:
                        secs[k].append(dt)
                    else:
                        digest[k] = sha(out)
            assert digest["one"] == digest["multi"], (mode, digest)
            res["big"][mode] = {k: {"seconds": s, "pairs_per_s": a.pairs / min(s)} for k, s in secs.items()}
            res["big"][mode]["multi_over_one"] = min(secs["one"]) / min(secs["multi"])
    finally:
        for g in grp:
            g.close()
    res["outputs_identical"] = True
    res["cards_after"] = subprocess.check_output(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip().splitlines()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
