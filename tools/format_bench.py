#!/usr/bin/env python
"""Developer tool: the CLI file -> file (first byte read to last byte written, timed inside it) for each output mode, against another build of
the CLI (e.g. the parent commit's, built in a scratch directory), in one call on the card whose name and power limit it prints.
Synthetic PE150 pairs, plain and BGZF level 6, MEM and Greedy; default output, -v and -M kaijux; the two builds alternate, `--rounds` rounds
after one warm-up run of each (--warmup 0: none); the output files of the two builds are compared byte for byte.
Usage: python tools/format_bench.py --other DIR/kaiju-b200 [--pairs 4000000] [--nprot 20000] [--rounds 2]"""
import argparse, hashlib, json, os, subprocess, sys, time
from multiprocessing import Pool
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))


def sha(path):
    h = hashlib.sha1()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", required=True, help="the CLI to compare with (built from another commit)")
    ap.add_argument("--nprot", type=int, default=20000); ap.add_argument("--pairs", type=int, default=4_000_000); ap.add_argument("--rounds", type=int, default=2); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--modes", default="mem,greedy"); ap.add_argument("--outputs", default="default,v,kaijux"); ap.add_argument("--encodings", default="plain,bgzf6")
    ap.add_argument("--workdir", default=os.environ.get("KJ_BENCH_DIR", "/tmp/kjbench"))
    a = ap.parse_args()
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
    from helpers import SynthDB, build_fmi
    from inflate_bench import write_bgzf
    os.makedirs(a.workdir, exist_ok=True)
    db = SynthDB(a.nprot, 1); fmi = os.path.join(a.workdir, "synth_%d.fmi" % a.nprot); nodes = os.path.join(a.workdir, "synth_%d_nodes.dmp" % a.nprot)
    if not os.path.exists(fmi):
        faa = os.path.join(a.workdir, "synth_%d.faa" % a.nprot); db.write(faa, nodes); build_fmi(faa, os.path.join(a.workdir, "synth_%d" % a.nprot), threads=min(32, os.cpu_count()))
    plain = [os.path.join(a.workdir, "fb_%d_%d.fq" % (a.pairs, m)) for m in (1, 2)]
    if not os.path.exists(plain[0]):
        db.write_fastq(7, 0, a.pairs, 150, True, plain[0], plain[1])
    files = {"plain": plain, "bgzf6": [p + ".l6.bgz" for p in plain]}
    with Pool(os.cpu_count()) as pool:
        for p in plain:
            if not os.path.exists(p + ".l6.bgz"):
                write_bgzf(p, p + ".l6.bgz", 6, pool)
    for v in files.values():
        for p in v:
            open(p, "rb").read()                      # page cache warm
    arms = {"this": os.path.join(ROOT, "kaiju_b200", "kaiju-b200"), "other": os.path.abspath(a.other)}
    outs = {"default": [], "v": ["-v"], "kaijux": ["-M", "kaijux"]}

    def run(arm, mode, enc, out_kind):
        dst = os.path.join(a.workdir, "fb_out_%s_%s_%s_%s.tsv" % (arm, mode, enc, out_kind))
        cmd = [arms[arm], "-f", fmi, "-a", mode, "-i", files[enc][0], "-j", files[enc][1], "-o", dst] + outs[out_kind] + ([] if out_kind == "kaijux" else ["-t", nodes])
        t0 = time.perf_counter()
        p = subprocess.run(cmd, stderr=subprocess.PIPE, stdout=subprocess.DEVNULL, text=True, env=dict(os.environ, KJ_CLI_TIMING="1"))
        wall = time.perf_counter() - t0
        if p.returncode:
            raise SystemExit("%s failed: %s" % (" ".join(cmd), p.stderr[-2000:]))
        inner = [float(l.split(" classified, ")[1].split(" s")[0]) for l in p.stderr.splitlines() if " classified, " in l]
        return (inner[0] if inner else None), wall, dst

    res = {"card": card, "pairs": a.pairs, "nprot": a.nprot, "runs": {}}
    for mode in a.modes.split(","):
        for out_kind in a.outputs.split(","):
            for enc in a.encodings.split(","):
                key = "%s/%s/%s" % (mode, out_kind, enc); secs = {"this": [], "other": []}; walls = {"this": [], "other": []}; dig = {}
                for arm in ("this", "other") if a.warmup else ():
                    run(arm, mode, enc, out_kind)                                  # warm-up
                for r in range(a.rounds):
                    for arm in (("this", "other") if r % 2 == 0 else ("other", "this")):
                        s, w, dst = run(arm, mode, enc, out_kind); secs[arm].append(s); walls[arm].append(round(w, 3)); dig[arm] = sha(dst); os.remove(dst)
                # seconds: first byte read to last byte written, as the CLI reports it (None: that build does not report it for the mode);
                # wall_seconds: the whole process, index load and context construction included
                res["runs"][key] = {"seconds": secs, "wall_seconds": walls, "pairs_per_s": {k: (a.pairs / min(v) if v and None not in v else None) for k, v in secs.items()},
                                    "outputs_identical": dig["this"] == dig["other"]}
                print(key, json.dumps(res["runs"][key]), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
