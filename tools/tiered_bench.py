"""Classification with part of the compact index in pinned host memory (kj_create_tiered), with bench.py's workload (synth-viruses index,
seeded PE150 pairs) and its timed loops.

  python tools/tiered_bench.py [--rows 2.7e10] [--reads 2000000] [--steps 5] [--warmup 3] [--rounds 2] [--max-rows 1e11]

1. The index scaled to --rows (compact: its wide construction does not fit an 80 GB card), placed five ways, alternated over --rounds rounds:
   all in HBM (host_memory = 0); tier 1 only (the suffix-array taxon arrays on the host, KJ_TIER_DEVICE_RECORDS = nb); 10 %, 25 % and 50 % of
   the records on the host.  MEM (-m 11) and Greedy (-e 3 -s 65), kernel-only (device buffers) and end-to-end (host buffers) pairs/s.
2. The largest scaled index whose host tier fits in 80 % of MemAvailable (at most --max-rows), placed by the library alone (no hook).
Results must be identical across all placements (MEM: also equal to the base index's).  Reports index_bytes, host_bytes, the build time and
the HBM left free after classifying.  Prints one JSON line with the card name and power limit read in the same run.  Needs the in-tree build."""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import bench


def mem_available():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


def run_placement(kb, R, fmi, nodes, copies, host_memory, device_records, steps, warmup):
    """one context of the scaled index: build, then MEM and Greedy kernel-only + end-to-end pairs/s; returns ({mode: result}, {mode: (tax, best)})"""
    import torch
    if device_records is not None:
        os.environ["KJ_TIER_DEVICE_RECORDS"] = str(device_records)
    try:
        t0 = time.time()
        clf = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem", m=11), copies=copies, host_memory=host_memory)
        create_s = time.time() - t0
    finally:
        os.environ.pop("KJ_TIER_DEVICE_RECORDS", None)
    res, outs = {}, {}
    try:
        for mode in ("mem", "greedy"):
            clf.set_params(kb.make_params(mode, m=11, e=3, s=65))
            r = bench.measure(R, clf, steps, warmup, 1)
            outs[mode] = (R.h_tax.numpy().view(np.uint64).copy(), R.h_best.numpy().view(np.uint32).copy())
            res[mode] = {"value": r["value"], "e2e": r["e2e"]["value"], "kernel_ms": r["kernel_ms"]}
        torch.cuda.synchronize()
        res.update({"layout": clf.layout, "bwt_rows": clf.bwtlen, "index_bytes": clf.index_bytes, "host_bytes": clf.host_bytes,
                    "device_build_ms": clf.index_build_ms, "create_s": create_s, "hbm_free_after": torch.cuda.mem_get_info()[0]})
        return res, outs
    finally:
        clf.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=2.7e10); ap.add_argument("--max-rows", type=float, default=1e11)
    ap.add_argument("--reads", type=int, default=2_000_000); ap.add_argument("--steps", type=int, default=5); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2); ap.add_argument("--nprot", type=int, default=680000)
    ap.add_argument("--skip-largest", action="store_true")
    ap.add_argument("--workdir", default=os.environ.get("KJ_BENCH_DIR", "/tmp/kjbench"))
    args = ap.parse_args()
    import torch
    import kaiju_b200 as kb
    clock = bench.ClockSampler(0); card = clock.card()
    db, fmi, nodes = bench.build_workload(args, 0)
    R = bench.Runner(torch, None, 1, 0, *db.reads(7, 0, args.reads, 150, True))
    base = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem", m=11))
    bench.measure(R, base, 1, 1, 1)
    base_out = (R.h_tax.numpy().view(np.uint64).copy(), R.h_best.numpy().view(np.uint32).copy()); base_rows = base.bwtlen
    base.close()
    line = {"card": card, "reads": args.reads, "steps": args.steps, "warmup": args.warmup, "mem_available": mem_available()}
    copies = max(2, int(round(args.rows / base_rows))); nb = base_rows * copies // 128 + 1
    budget = int(0.8 * mem_available())
    placements = [("hbm", 0, None), ("tier1", budget, nb), ("host10", budget, nb - nb // 10), ("host25", budget, nb - nb // 4), ("host50", budget, nb - nb // 2)]
    runs, ref = {}, {}

    def check(res, outs):
        for mode, (tax, best) in outs.items():
            if mode not in ref:
                ref[mode] = (tax, best)
            res[mode]["diffs_vs_first"] = int(((tax != ref[mode][0]) | (best != ref[mode][1])).sum())
        res["mem"]["diffs_vs_base"] = int(((outs["mem"][0] != base_out[0]) | (outs["mem"][1] != base_out[1])).sum())

    for rnd in range(args.rounds):
        for name, host, nd in placements:
            res, outs = run_placement(kb, R, fmi, nodes, copies, host, nd, args.steps, args.warmup)
            check(res, outs); runs.setdefault(name, []).append(res)
            print(json.dumps({"placement": name, "round": rnd, **res}), file=sys.stderr, flush=True)
    line["scaled"] = {"copies": copies, "runs": runs}
    # 2. the largest index the host's memory allows beyond HBM (records 1.003 B + sa_tax 0.5 B per row, 4 GB of HBM kept free), no hook
    if not args.skip_largest:
        free = torch.cuda.mem_get_info()[0]
        rows = min(args.max_rows, (budget + free - (8 << 30)) / 1.51)
        big_copies = max(2, int(rows / base_rows))
        res, outs = run_placement(kb, R, fmi, nodes, big_copies, budget, None, args.steps, args.warmup)
        check(res, outs)
        line["largest"] = {"copies": big_copies, "budget": budget, **res}
    line["card_after"] = clock.card()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
