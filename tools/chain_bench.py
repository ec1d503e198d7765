#!/usr/bin/env python3
"""Time the chaining kernel (K3) on the benchmark's workload and show where its time goes.

  python tools/chain_bench.py [--workdir DIR] [--ref-mbp 3000] [--reads 1000000] [--layout pe] [--repeats 5] [--lib PATH] [--json-out FILE]

Runs mem_process_seqs over bench.py's workload (made by bench.make_workload, shared with bench.py's work directory) with one lane
and one chunk, as bench.py's kernel-only passes do, and reads ms_chain from the device statistics after every call.  Prints one
JSON line with the GPU's name and power limit beside the numbers.

With a library built with `make NVEXTRA=-DBWAG_K3_CLOCKS` (pass it with --lib, or build it in place), k_chain records per read its
number of seeds and chains and the clock64() cycles of its chaining loop, mem_chain_flt and chain_emit; the tool then adds the
histograms of seeds and chains per read and the share of the lane-cycles spent on the reads of each seed count, which tells a
kernel whose time goes to the typical read from one whose time goes to a tail of big reads."""
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

N_TOT, N_CHN = 66, 34   # histogram bins of bwag_k3_clocks (include/bwa_b200_dev.h)


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
    L.bwag_k3_clocks.argtypes = [C.c_void_p, C.c_int]
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
    clocks = L.bwag_k3_clocks(None, 1) == 0
    ms = []
    for _ in range(a.repeats):
        idx.stats(reset=True)
        step()
        ms.append(idx.stats()["ms_chain"])
    res = dict(workload="%d %s reads of %d bp vs the %d Mbp random reference of bench.py, one lane, one chunk" % (a.reads, "paired" if paired else "single-end", a.read_len, a.ref_mbp),
               ms_chain=[round(x, 3) for x in ms], ms_chain_median=round(sorted(ms)[len(ms) // 2], 3), **gpu_info())
    if clocks:
        h = (C.c_uint64 * (4 * N_TOT + N_CHN))()
        L.bwag_k3_clocks(h, 0)
        reads = [h[4 * t] for t in range(N_TOT)]
        cyc = [h[4 * t + 1] + h[4 * t + 2] + h[4 * t + 3] for t in range(N_TOT)]
        n, c = sum(reads) or 1, sum(cyc) or 1
        res["calls_recorded"] = a.repeats
        res["seeds_per_read"] = {("%d" % t if t < 65 else ">64"): reads[t] for t in range(N_TOT) if reads[t]}
        res["chains_per_read"] = {("%d" % t if t < 33 else ">32"): h[4 * N_TOT + t] for t in range(N_CHN) if h[4 * N_TOT + t]}
        res["cycles_share_by_seeds"] = {("%d" % t if t < 65 else ">64"): round(cyc[t] / c, 4) for t in range(N_TOT) if reads[t]}
        res["cycles_per_read_by_seeds"] = {("%d" % t if t < 65 else ">64"): [round(h[4 * t + k] / reads[t]) for k in (1, 2, 3)] for t in range(N_TOT) if reads[t]}
        res["cycles_split"] = {k: round(sum(h[4 * t + i] for t in range(N_TOT)) / c, 4) for i, k in ((1, "chaining"), (2, "mem_chain_flt"), (3, "chain_emit"))}
        acc = 0
        for t in range(N_TOT):   # smallest seed count that covers 99 % of the reads
            acc += reads[t]
            if acc >= 0.99 * n:
                res["seeds_p99"] = t if t < 65 else ">64"
                break
    line = json.dumps(res)
    print(line)
    if a.json_out:
        with open(a.json_out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
