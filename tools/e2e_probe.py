import os, sys, time, numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import kaiju_b200 as kb
from helpers import SynthDB, build_fmi
wd = "/tmp/kjbench"; os.makedirs(wd, exist_ok=True)
db = SynthDB(680000, 1); fmi = wd + "/synth_680000.fmi"; nodes = wd + "/synth_680000_nodes.dmp"
if not os.path.exists(fmi):
    db.write(wd + "/synth_680000.faa", nodes); build_fmi(wd + "/synth_680000.faa", wd + "/synth_680000", threads=32)
n = 10_000_000
s1, o1, s2, o2 = db.reads(7, 0, n, 150, True)
clf = kb.Classifier(fmi, nodes, device=0, params=kb.make_params("mem"))
pin = lambda x: torch.from_numpy(x.view(np.int64) if x.dtype == np.uint64 else x).pin_memory()
h = [pin(x) for x in (s1, o1, s2, o2)]; d = [x.cuda() for x in h]
ht = torch.zeros(n, dtype=torch.int64).pin_memory(); hb = torch.zeros(n, dtype=torch.int32).pin_memory()
dt = torch.zeros(n, dtype=torch.int64, device="cuda"); dbst = torch.zeros(n, dtype=torch.int32, device="cuda")
for rep in range(3):
    clf.classify_device(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), n, dt.data_ptr(), dbst.data_ptr(), 150, 150); torch.cuda.synchronize()
    print("device path kernel_ms", clf.last_kernel_ms)
os.environ["KJ_TRACE"]="1"
for chunk in ("1048576",):
    os.environ["KJ_CHUNK_READS"] = chunk
    for rep in range(2):
        t = time.time(); clf.classify_ptrs(h[0].data_ptr(), h[1].data_ptr(), h[2].data_ptr(), h[3].data_ptr(), n, ht.data_ptr(), hb.data_ptr()); w = time.time() - t
        print("host path chunk", chunk, "wall_ms %.1f" % (w * 1e3), "last kernel_ms %.1f" % clf.last_kernel_ms)
