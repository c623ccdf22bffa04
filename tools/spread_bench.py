"""Classification against one index spread over the HBM of a group of GPUs (kj_create_group), with bench.py's workload (synth-viruses index,
seeded PE150 pairs) and its timed loops.

  python tools/spread_bench.py [--rows 2.7e10] [--reads 2000000] [--steps 5] [--warmup 3] [--rounds 1] [--skip-largest]

1. The index scaled to --rows (compact: its wide construction does not fit an 80 GB card), placed as: one GPU, compact (kj_create_scaled);
   the group [0, 0] (two segments on one GPU: the cost of selecting the segment alone); [0, 1] and [0, 1, 2, 3] where the machine has the GPUs
   and peer access between them.  For each, MEM (-m 11) and Greedy (-e 3 -s 65): kernel-only (device buffers) and end-to-end (host buffers)
   pairs/s of the group's first context on GPU 0, and end-to-end pairs/s of kj_classify_multi over all of the group's contexts.
2. With two or more GPUs: an index too large for one card's compact construction, over all GPUs with peer access (no hook).
Results must be identical across placements.  Prints one JSON line with the card name, power limit and the GPU interconnect (nvidia-smi topo -m)
read in the same run; configurations the machine cannot provide are reported as "not measured".  Needs the in-tree build."""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import bench


def topology():
    try:
        return subprocess.run(["nvidia-smi", "topo", "-m"], capture_output=True, text=True, timeout=60).stdout
    except Exception as e:      # the interconnect is reported, not required
        return "unavailable: %s" % e


def peer_group(torch, n):
    """[0, n) when the machine has n GPUs with peer access between every pair, else None"""
    if torch.cuda.device_count() < n:
        return None
    ok = all(a == b or torch.cuda.can_device_access_peer(a, b) for a in range(n) for b in range(n))
    return list(range(n)) if ok else None


def run(kb, R, make, steps, warmup, s1, o1, s2, o2):
    """contexts from make() (the first on GPU 0): build time, then per mode the first context's kernel-only / end-to-end pairs/s and the whole
    group's kj_classify_multi pairs/s; returns ({...}, {mode: (tax, best)})"""
    import torch
    t0 = time.time(); ctxs = make(); create_s = time.time() - t0
    res, outs = {"create_s": create_s, "layout": ctxs[0].layout, "bwt_rows": ctxs[0].bwtlen, "index_bytes": [c.index_bytes for c in ctxs],
                 "device_build_ms": ctxs[0].index_build_ms}, {}
    try:
        for mode in ("mem", "greedy"):
            for c in ctxs:
                c.set_params(kb.make_params(mode, m=11, e=3, s=65))
            r = bench.measure(R, ctxs[0], steps, warmup, 1)
            outs[mode] = (R.h_tax.numpy().view(np.uint64).copy(), R.h_best.numpy().view(np.uint32).copy())
            kb.classify_multi(ctxs, s1, o1, s2, o2)           # warm-up of every context
            t = time.time()
            for _ in range(steps):
                tax, best = kb.classify_multi(ctxs, s1, o1, s2, o2)
            multi = R.n * steps / (time.time() - t)
            assert np.array_equal(tax, outs[mode][0]) and np.array_equal(best, outs[mode][1]), "kj_classify_multi differs from the first context"
            res[mode] = {"kernel_only": r["value"], "e2e": r["e2e"]["value"], "kernel_ms": r["kernel_ms"], "group_e2e": multi}
        torch.cuda.synchronize()
        return res, outs
    finally:
        for c in ctxs:
            c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=2.7e10)
    ap.add_argument("--reads", type=int, default=2_000_000); ap.add_argument("--steps", type=int, default=5); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=1); ap.add_argument("--nprot", type=int, default=680000)
    ap.add_argument("--skip-largest", action="store_true")
    ap.add_argument("--workdir", default=os.environ.get("KJ_BENCH_DIR", "/tmp/kjbench"))
    args = ap.parse_args()
    import torch
    import kaiju_b200 as kb
    clock = bench.ClockSampler(0); card = clock.card()
    line = {"card": card, "gpus": torch.cuda.device_count(), "topology": topology(), "reads": args.reads, "steps": args.steps, "warmup": args.warmup}
    db, fmi, nodes = bench.build_workload(args, 0)
    s1, o1, s2, o2 = db.reads(7, 0, args.reads, 150, True)
    R = bench.Runner(torch, None, 1, 0, s1, o1, s2, o2)
    base = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem", m=11)); base_rows = base.bwtlen; base.close()
    copies = max(2, int(round(args.rows / base_rows)))
    P = kb.make_params("mem", m=11)
    placements = [("one_gpu_compact", lambda: [kb.Classifier(fmi, nodes, device=0, params=P, copies=copies)]),
                  ("group_0_0", lambda: kb.create_group(fmi, nodes, [0, 0], params=P, copies=copies))]
    for n in (2, 4):
        g = peer_group(torch, n)
        if g:
            placements.append(("group_0_%d" % (n - 1), lambda g=g: kb.create_group(fmi, nodes, g, params=P, copies=copies)))
        else:
            line["group_0_%d" % (n - 1)] = "not measured: the machine has no %d GPUs with peer access" % n
    runs, ref = {}, {}
    for rnd in range(args.rounds):
        for name, make in placements:
            res, outs = run(kb, R, make, args.steps, args.warmup, s1, o1, s2, o2)
            for mode, (tax, best) in outs.items():
                ref.setdefault(mode, (tax, best))
                res[mode]["diffs_vs_first"] = int(((tax != ref[mode][0]) | (best != ref[mode][1])).sum())
            runs.setdefault(name, []).append(res)
            print(json.dumps({"placement": name, "round": rnd, **res}), file=sys.stderr, flush=True)
    line["scaled"] = {"copies": copies, "runs": runs}
    # 2. beyond one card: records 1.003 B + sa_tax 0.5 B per row, over every GPU with peer access
    g = peer_group(torch, torch.cuda.device_count()) if torch.cuda.device_count() >= 2 else None
    if args.skip_largest:
        line["largest"] = "not measured: --skip-largest"
    elif not g:
        line["largest"] = "not measured: needs two or more GPUs with peer access"
    else:
        free = min(torch.cuda.mem_get_info(d)[0] for d in g)
        big = max(2, int(1.2 * free / 1.52 / base_rows))
        res, _ = run(kb, R, lambda: kb.create_group(fmi, nodes, g, params=P, copies=big), args.steps, args.warmup, s1, o1, s2, o2)
        line["largest"] = {"copies": big, "devices": g, **res}
    line["card_after"] = clock.card()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
