#!/usr/bin/env python3
"""Time seeding (K0 + K1f + K1 + K1b) on the benchmark's workload and show where K1's (k_smem_c's) loop iterations go.

  python tools/k1_bench.py [--workdir DIR] [--ref-mbp 3000] [--reads 1000000] [--layout pe] [--repeats 5] [--lib PATH] [--json-out FILE]

Runs mem_process_seqs over bench.py's workload (made by bench.make_workload, shared with bench.py's work directory) with one lane
and one chunk, as bench.py's kernel-only passes do, and reads ms_smem from the device statistics after every call.  Prints one
JSON line with the GPU's name and power limit beside the numbers.

With a library built with `make NVEXTRA=-DBWAG_K1_CLOCKS` (pass it with --lib, or build it in place), the seeding driver times
K1f (k_smem_fwd) and k_smem_c with events of their own, and k_smem_c counts per lane its loop iterations by the kind of extension
each did (forward by a table lookup or by Occ blocks, backward a list or a mask candidate), how many of them looked up a pair of
table entries, and the clock64() cycles spent handing a finished read over and fetching the next.  The counters cost time: the
ms_smem of such a build is not the default build's."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402  (make_workload only)
from aln_bench import gpu_info  # noqa: E402

# bwag_k1_clocks words (include/bwa_b200_dev.h)
WORDS = ("iters", "fwd_table", "fwd_occ", "bwd_list", "bwd_mask", "pairs_fwd", "pairs_bwd", "turnover_cycles", "reads", "k1f_ns", "k1c_ns", "calls")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workdir", default=os.environ.get("BWA_B200_BENCH_DIR", "/tmp/bwa_b200_bench"))
    ap.add_argument("--ref-mbp", type=int, default=3000)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--read-len", type=int, default=150)
    ap.add_argument("--layout", default="pe", choices=["pe", "se"])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--lib", default=None, help="library to load (default: bwa_b200/libbwa_b200.so)")
    ap.add_argument("--json-out")
    a = ap.parse_args()
    paired = a.layout == "pe"
    fa, fqs = bench.make_workload(a.workdir, a.ref_mbp, a.reads, a.read_len, 1000, 0, paired)
    os.environ["BWA_B200_LANES"] = "1"
    os.environ["BWA_B200_CHUNK"] = str(1 << 30)
    import bwa_b200
    L = bwa_b200.lib(a.lib) if a.lib else bwa_b200.lib()
    if a.lib:
        bwa_b200._lib = L
    L.bwag_k1_clocks.argtypes = [C.c_void_p, C.c_int]
    idx = bwa_b200.Index(fa, L)
    idx.attach()
    opt = L.mem_opt_init()
    if paired:
        opt.contents.flag |= bwa_b200.MEM_F_PE
    batch = bwa_b200.ReadBatch(*fqs, library=L)

    def step():
        bwa_b200.mem_process_seqs(opt, idx, batch)
        batch.sam()

    step()                                          # warm-up: module load, buffer growth
    clocks = L.bwag_k1_clocks(None, 1) == 0
    ms = []
    for _ in range(a.repeats):
        idx.stats(reset=True)
        step()
        ms.append(idx.stats()["ms_smem"])
    res = dict(workload="%d %s reads of %d bp vs the %d Mbp random reference of bench.py, one lane, one chunk" % (a.reads, "paired" if paired else "single-end", a.read_len, a.ref_mbp),
               ms_smem=[round(x, 3) for x in ms], ms_smem_median=round(sorted(ms)[len(ms) // 2], 3), **gpu_info())
    if clocks:
        h = (C.c_uint64 * len(WORDS))()
        L.bwag_k1_clocks(h, 0)
        w = dict(zip(WORDS, h))
        calls = w["calls"] or 1
        steps = w["fwd_table"] + w["fwd_occ"] + w["bwd_list"] + w["bwd_mask"]
        res["calls_recorded"] = w["calls"]
        res["ms_k1f_per_call"] = round(w["k1f_ns"] / 1e6 / calls, 3)
        res["ms_k_smem_c_per_call"] = round(w["k1c_ns"] / 1e6 / calls, 3)
        per_call = {k: w[k] // calls for k in WORDS[:9]}
        per_call["warp_iters"] = w["iters"] // 32 // calls
        res["per_call"] = per_call
        res["lane_steps_per_warp_iter"] = round(steps / (w["iters"] / 32), 2) if w["iters"] else 0.0
        res["turnover_cycles_per_read"] = round(w["turnover_cycles"] / (w["reads"] or 1))
    line = json.dumps(res)
    print(line)
    if a.json_out:
        with open(a.json_out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
