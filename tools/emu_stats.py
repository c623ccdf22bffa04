"""Developer tool (CPU only): counters of the chain-resolution loops on the CPU warp emulator (rounds / warp-steps / chains completed per read
item) next to an oracle check, on a seeded PE150 workload.  KJ_EMU_NOMONO=1 switches the bounds off (the round-1 behaviour: groups of 8).
The taxon look-up of the kept rows is counted twice, with the SA walk ("walk") and with the row -> taxon array ("row_tax"):
  id_reads / kept     : reads that reached the look-up / their kept intervals
  sa_waves            : waves of up to 32 rows
  sa_lf_steps         : LF steps, summed over the lanes
  sa_dep_steps        : LF steps the warp waits for (the slowest lane of each wave, summed)
  sa_dep_loads        : dependent global loads of the look-up: 2 per waited LF step + 1 per wave (the taxon load)
Usage: python tools/emu_stats.py [n_pairs] [nprot]"""
import sys, os, time, tempfile, ctypes as C, numpy as np
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
from helpers import SynthDB, build_fmi, Oracle, make_params
from test_kernel_logic_emulated import KjParams
import emu_row_tax
E = emu_row_tax.load(tempfile.mkdtemp(prefix="kjemu_row_tax_"), KjParams)      # the emulator with the row -> taxon array
n = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
nprot = int(sys.argv[2]) if len(sys.argv) > 2 else 60000
d = "/tmp/kjemu_stats_%d" % nprot; os.makedirs(d, exist_ok=True)
db = SynthDB(nprot, 21)
if not os.path.exists(d + "/db.fmi"):
    db.write(d + "/db.faa", d + "/nodes.dmp"); build_fmi(d + "/db.faa", d + "/db", threads=8)
fmi, nodes = d + "/db.fmi", d + "/nodes.dmp"
s1, o1, s2, o2 = db.reads(301, 0, n, 150, True)
orc = Oracle(fmi, nodes)
names = ["rounds", "round_steps", "lane_steps", "chains", "blocks", "lookaheads", "pops_frag", "pops_var", "var_steps", "var_pushed",
         "id_reads", "kept", "sa_waves", "sa_lf_steps", "sa_dep_steps", "lq_tops", "lq_slots"]
for kw in (dict(mode="mem"), dict(mode="greedy")):
    P = make_params(**kw); kp = KjParams(**P); h = E.kjemu_create(fmi.encode(), nodes.encode(), C.byref(kp))
    have_array = E.kjemu_use_row_tax(h, 1)          # built once here (it also appends the suffix array's guard entry, as the device does)
    otax, obest = orc.classify_batch(P, s1, o1, s2, o2)
    for lookup in ("walk", "row_tax"):
        if lookup == "row_tax" and not have_array:
            continue
        E.kjemu_use_row_tax(h, lookup == "row_tax")
        tax = np.zeros(n, dtype=np.uint64); best = np.zeros(n, dtype=np.uint32)
        buf = (C.c_ulonglong * 32)(); E.kjemu_stats(buf, 32, 1)
        t = time.time(); rc = E.kjemu_classify(h, s1.ctypes.data, o1.ctypes.data, s2.ctypes.data, o2.ctypes.data, n, tax.ctypes.data, best.ctypes.data, 8); dt = time.time() - t
        k = E.kjemu_stats(buf, 32, 1); c = {names[i]: buf[i] for i in range(k)}
        bad = int(((tax != otax) | (best != obest)).sum())
        per_pair = {x: round(c[x] / n, 2) for x in names}
        per_pair["sa_dep_loads"] = round((2 * c["sa_dep_steps"] + c["sa_waves"]) / n, 2)
        print(kw, lookup, "rc", rc, "bad", bad, "classified %.3f" % (otax != 0).mean(), "emu %.1fs" % dt, per_pair,
              "kept intervals per read that reached the look-up %.2f" % (c["kept"] / max(1, c["id_reads"])), flush=True)
    E.kjemu_destroy_row_tax(h)
