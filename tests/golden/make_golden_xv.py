#!/usr/bin/env python
"""Golden fixtures for the fragment-string column of the name-reporting front-ends: runs the UNMODIFIED reference `kaijux -v` and `kaijup -v`
(oracle/_ref, built by oracle/Makefile) on the committed index and read sets, with the five configurations of make_golden_xp.py.  Run in the
build container after make_golden_xp.py (it writes prot.fa.gz):

    make -C oracle ref && python tests/golden/make_golden_xv.py

Outputs: expected_xv_<cfg>_<tag>.tsv.gz, expected_pv_<cfg>.tsv.gz -- the reference's output lines as they are (status, read name, best
length/score, database sequence names, matched fragment strings)."""
import gzip, os, subprocess, sys
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, HERE)
from helpers import REF_DIR   # noqa: E402
from make_golden_xp import XP_CONFIGS, plain   # noqa: E402


def main():
    tmp = "/tmp/kj_xv"; os.makedirs(tmp, exist_ok=True)
    fmi = os.path.join(HERE, "db.fmi")
    inputs = {"se100": ["-i", plain(HERE + "/se100.fq.gz", tmp + "/se.fq")],
              "pe150": ["-i", plain(HERE + "/pe150_1.fq.gz", tmp + "/a.fq"), "-j", plain(HERE + "/pe150_2.fq.gz", tmp + "/b.fq")]}
    prot = plain(HERE + "/prot.fa.gz", tmp + "/prot.fa")
    for cfg, flags in XP_CONFIGS.items():
        for tag, inp in inputs.items():
            out = subprocess.run([os.path.join(REF_DIR, "kaijux"), "-f", fmi, "-z", "1", "-v"] + inp + flags, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True).stdout
            with gzip.open(os.path.join(HERE, "expected_xv_%s_%s.tsv.gz" % (cfg, tag)), "wb") as g:
                g.write(out)
        out = subprocess.run([os.path.join(REF_DIR, "kaijup"), "-f", fmi, "-z", "1", "-v", "-i", prot] + flags, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True).stdout
        with gzip.open(os.path.join(HERE, "expected_pv_%s.tsv.gz" % cfg), "wb") as g:
            g.write(out)
    print("kaijux -v / kaijup -v outputs written")


if __name__ == "__main__":
    main()
