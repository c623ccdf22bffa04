"""Wide against compact rank layout on one GPU, with bench.py's workload (synth-viruses index, seeded PE150 pairs) and its timed loops.

  python tools/compact_bench.py [--rows 1.2e10] [--big-rows 2.7e10] [--reads 10000000] [--steps 5] [--warmup 3] [--rounds 3]

1. The index scaled to --rows (the size of bench.py's configs[3]): a wide context and a KJ_FORCE_COMPACT context, built alternately --rounds times
   each; MEM (-m 11) and Greedy (-e 3 -s 65) kernel-only (device buffers) and end-to-end (host buffers) pairs/s.  Results must be identical.
2. The index scaled to --big-rows (compact without any hook): the same, MEM results must equal those on the base index.
Also: bytes per row, index_bytes, device build ms, and the ptxas register / spill lines of the compact and wide classify kernels (ptxas.log of the
last in-tree build).  Prints one JSON line with the card name and power limit read in the same run.  Needs the in-tree build (build())."""
import argparse, json, os, re, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import bench


def ptxas_lines():
    """register / spill report of the 64-bit classify kernels: `y` = KjCompactIdx (compact), `m` = uint64_t (wide) in the mangled names"""
    p = os.path.join(ROOT, "kaiju_b200", "csrc", "ptxas.log")
    if not os.path.exists(p):
        return None
    out = {"compact": [], "wide": []}; cur = None
    for l in open(p):
        m = re.search(r"Compiling entry function '(_Z18kj_classify_kernelILi(\d)E([my])Lb(\d)ELb(\d)ELb(\d)ELi(\d)E\S*)'", l)
        if m:
            cur = ("compact" if m.group(3) == "y" else "wide", "mode%s gws%s fix%s vb%s role%s" % m.group(2, 4, 5, 6, 7)); continue
        if cur and ("registers" in l or "spill" in l):
            out[cur[0]].append("%s: %s" % (cur[1], l.split(":", 1)[-1].strip()))
            if "registers" in l:
                cur = None
    return out


def run_pair(kb, R, fmi, nodes, copies, force, steps, warmup, mode):
    """one context (wide / compact) of the scaled index: build, then kernel-only + end-to-end pairs/s in `mode`; returns (result, taxon, best)"""
    if force:
        os.environ["KJ_FORCE_COMPACT"] = "1"
    try:
        t0 = time.time()
        clf = kb.Classifier(fmi, nodes, device=0, params=kb.make_params(mode, m=11, e=3, s=65), copies=copies)
        create_s = time.time() - t0
    finally:
        os.environ.pop("KJ_FORCE_COMPACT", None)
    try:
        r = bench.measure(R, clf, steps, warmup, 1)
        tax = R.h_tax.numpy().view(np.uint64).copy(); best = R.h_best.numpy().view(np.uint32).copy()
        return {"layout": clf.layout, "value": r["value"], "e2e": r["e2e"]["value"], "kernel_ms": r["kernel_ms"], "bwt_rows": clf.bwtlen,
                "index_bytes": clf.index_bytes, "bytes_per_row": clf.index_bytes / clf.bwtlen, "device_build_ms": clf.index_build_ms, "create_s": create_s}, tax, best
    finally:
        clf.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1.2e10); ap.add_argument("--big-rows", type=float, default=2.7e10)
    ap.add_argument("--reads", type=int, default=10_000_000); ap.add_argument("--steps", type=int, default=5); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3); ap.add_argument("--nprot", type=int, default=680000)
    ap.add_argument("--workdir", default=os.environ.get("KJ_BENCH_DIR", "/tmp/kjbench"))
    args = ap.parse_args()
    import torch
    import kaiju_b200 as kb
    clock = bench.ClockSampler(0); card = clock.card()
    db, fmi, nodes = bench.build_workload(args, 0)
    R = bench.Runner(torch, None, 1, 0, *db.reads(7, 0, args.reads, 150, True))
    base = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem", m=11))
    bench.measure(R, base, 1, 1, 1)
    base_tax = R.h_tax.numpy().view(np.uint64).copy(); base_best = R.h_best.numpy().view(np.uint32).copy(); base_rows = base.bwtlen
    base.close()
    line = {"card": card, "reads": args.reads, "steps": args.steps, "warmup": args.warmup, "ptxas": ptxas_lines()}
    # 1. wide vs compact on the same scaled index, alternated
    copies = max(2, int(round(args.rows / base_rows)))
    runs = {}
    for mode in ("mem", "greedy"):
        ref = None
        for rnd in range(args.rounds):
            for name, force in (("wide", False), ("compact", True)):
                res, tax, best = run_pair(kb, R, fmi, nodes, copies, force, args.steps, args.warmup, mode)
                runs.setdefault("%s_%s" % (mode, name), []).append(res)
                if ref is None:
                    ref = (tax, best)
                res["diffs_vs_wide"] = int(((tax != ref[0]) | (best != ref[1])).sum())
                if mode == "mem":
                    res["diffs_vs_base"] = int(((tax != base_tax) | (best != base_best)).sum())
    line["scaled"] = {"copies": copies, "runs": runs}
    # 2. the refseq_ref-scale index: compact without a hook
    big_copies = max(2, int(round(args.big_rows / base_rows)))
    big = []
    for rnd in range(args.rounds):
        for mode in ("mem", "greedy"):
            res, tax, best = run_pair(kb, R, fmi, nodes, big_copies, False, args.steps, args.warmup, mode)
            if mode == "mem":
                res["diffs_vs_base"] = int(((tax != base_tax) | (best != base_best)).sum())
            res["mode"] = mode; big.append(res)
    line["big"] = {"copies": big_copies, "runs": big}
    line["card_after"] = clock.card()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
