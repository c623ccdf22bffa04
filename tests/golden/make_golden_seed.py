#!/usr/bin/env python
"""Golden fixtures for Greedy at seed lengths other than the default 7: runs the UNMODIFIED reference kaiju (oracle/_ref, built by
oracle/Makefile) with -a greedy -l L on the committed index and read sets.  Run in the build container:

    make -C oracle ref && python tests/golden/make_golden_seed.py

Outputs (the other fixtures are left alone):
    expected_greedy_l<L>_<tag>.tsv.gz   L = 9, 12, 20: status, name, taxon, best score, id set (the format of make_golden.py)
    expected_v7_greedy_l12_pe150.tsv.gz all seven columns of `kaiju -v -l 12`, the reference's output as it is"""
import gzip, os, shutil, subprocess, sys
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from helpers import REF_DIR, parse_kaiju_output   # noqa: E402

SEEDS = (9, 12, 20)


def plain(src, dst):
    with gzip.open(src, "rb") as f, open(dst, "wb") as g:
        shutil.copyfileobj(f, g)
    return dst


def run(inp, seed):
    """-z 1: the output lines come in input order"""
    return subprocess.run([os.path.join(REF_DIR, "kaiju"), "-t", os.path.join(HERE, "nodes.dmp"), "-f", os.path.join(HERE, "db.fmi"), "-z", "1", "-v",
                           "-a", "greedy", "-l", str(seed)] + inp, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True).stdout


def main():
    tmp = "/tmp/kj_seed"; os.makedirs(tmp, exist_ok=True)
    inputs = {"pe150": ["-i", plain(HERE + "/pe150_1.fq.gz", tmp + "/a.fq"), "-j", plain(HERE + "/pe150_2.fq.gz", tmp + "/b.fq")],
              "se100": ["-i", plain(HERE + "/se100.fq.gz", tmp + "/se.fq")]}
    for seed in SEEDS:
        for tag, inp in inputs.items():
            out = run(inp, seed).decode()
            res = parse_kaiju_output(out); names = [l.split("\t")[1] for l in out.splitlines()]
            with gzip.open(os.path.join(HERE, "expected_greedy_l%d_%s.tsv.gz" % (seed, tag)), "wt") as f:
                for nm in names:
                    r = res[nm]
                    f.write("%s\t%s\t%d\t%d\t%s\n" % (r[0], nm, r[1], r[2], ",".join(map(str, r[3]))))
            print("-l %d %s: %d of %d reads classified" % (seed, tag, sum(1 for nm in names if res[nm][0] == "C"), len(names)))
    with gzip.open(os.path.join(HERE, "expected_v7_greedy_l12_pe150.tsv.gz"), "wb") as g:
        g.write(run(inputs["pe150"], 12))


if __name__ == "__main__":
    main()
