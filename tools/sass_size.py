#!/usr/bin/env python
"""Developer tool: static SASS size of the kernels in a cubin, attributed to source functions through the -lineinfo table
(the instruction-cache footprint is what limits the Greedy kernel: DESIGN.md §3).  Usage: tools/sass_size.py <cubin> [kernel-substring]"""
import re, subprocess, sys, os
cubin = sys.argv[1]; want = sys.argv[2] if len(sys.argv) > 2 else "kj_classify_kernelILi1EjLb0"
out = subprocess.run(["nvdisasm", "--print-line-info-inline", cubin], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout.decode(errors="replace")
csrc = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "kaiju_b200", "csrc")
fmap = {}
for fn in os.listdir(csrc):
    if fn.endswith((".h", ".cu")):
        cur = "(top:%s)" % fn; m = {}
        for i, l in enumerate(open(os.path.join(csrc, fn)).read().split("\n"), 1):
            mm = re.match(r"^(?:template <[^>]*>\s*)?(?:static )?(?:KJ_DEV|KJ_HD|__device__ __forceinline__|__device__ __noinline__|KJ_NOINLINE) .*?\b(kj_\w+|warp_\w+|lanemask_lt)\s*\(", l)
            if mm: cur = mm.group(1)
            if re.match(r"^(__global__|template <int MODE, class IdxT, bool GWS>)", l): cur = "(kernel body)"
            m[i] = cur
        fmap[fn] = m
sizes = {}; cur_fn = None; cur_src = ("?", 0); per = {}; chain = []; fresh = True
OWN = ("kj_core.h", "kj_core_greedy.h", "kj_device.cu", "kj_ingest.h")
for line in out.split("\n"):
    m = re.match(r"^\s*\.text\.(\S+):", line) or re.match(r"^(\S+):\s*$", line)
    mm = re.match(r'^\s*//## File "([^"]+)", line (\d+)', line)
    if mm:
        if fresh: chain = []; fresh = False
        chain.append((mm.group(1).split("/")[-1], int(mm.group(2))))
        # attribute to the innermost frame that lies in the kernels' own sources (not kj_warp.h / toolkit headers)
        own = [c for c in chain if c[0] in OWN]
        cur_src = own[0] if own else chain[0]
        continue
    m2 = re.match(r"^\.text\.(\S+):", line)
    if m2:
        cur_fn = m2.group(1); continue
    if re.match(r"^\s*\.section", line):
        cur_fn = None; continue
    if cur_fn and re.match(r"^\s+/\*[0-9a-f]+\*/\s+[@A-Z]", line):
        fresh = True
        sizes[cur_fn] = sizes.get(cur_fn, 0) + 1
        if want in cur_fn:
            f, l = cur_src; k = fmap.get(f, {}).get(l, f)
            per[k] = per.get(k, 0) + 1
for k, v in sorted(sizes.items(), key=lambda kv: -kv[1])[:14]:
    print("%7d instr %7.1f KB  %s" % (v, v * 16 / 1024, k[:90]))
print("--- attribution inside *%s*" % want)
for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:45]:
    print("%7d instr %6.1f KB  %s" % (v, v * 16 / 1024, k))
