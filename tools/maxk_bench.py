#!/usr/bin/env python3
"""Timing of `bwa-b200 maxk` on the benchmark's data: `maxk -s` of the 3 Gbp random reference of bench.py against itself, and default
mode on the benchmark's 1 M single-end 150-bp reads (both made and indexed by bench.make_workload, shared with bench.py's work
directory).

  python tools/maxk_bench.py [--workdir DIR] [--ref-mbp 3000] [--reads 1000000] [--windows W1,W2,..] [--json-out FILE]

Per run: the wall time, and from BWA_B200_PROFILE the index load, the search kernel's time (CUDA events), the longest time one lane
spent on one window (device clock: whether long exact repeats bound the run), the binning kernel and the windows.  The reference is
not run here (about 1 us per base for -s on one core, DESIGN.md §7); tests/test_maxk.py compares the outputs.  Prints one JSON line
with the GPU name and power limit read in the same call.  Nothing is written to the repository."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402  (make_workload only)

CLI = os.path.join(ROOT, "bwa_b200", "bwa-b200")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=60).stdout
        name, power, clk = [x.strip() for x in q.splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clk)
    except Exception as e:   # noqa: BLE001 -- the numbers stay usable without it
        return dict(gpu_query_error=str(e))


def self_fasta(workdir, ref_mbp):
    """the FASTA of bench.make_workload's random reference (above 60 Mbp it indexes the contigs without writing one): the same
    contigs from the same seed, written once beside the index"""
    import gen_data
    fa, done = os.path.join(workdir, "ref_%d.self.fa" % ref_mbp), os.path.join(workdir, "ref_%d.self.fa.done" % ref_mbp)
    if not os.path.exists(done):
        contig_len = min(125_000_000, ref_mbp * 1_000_000)
        gen_data.write_fasta(fa, gen_data.random_contigs(max(1, (ref_mbp * 1_000_000) // contig_len), contig_len, 7))
        open(done, "w").write("ok")
    return fa


def run(args, window):
    env = dict(os.environ, BWA_B200_PROFILE="1")
    if window:
        env["BWA_B200_MAXK_WINDOW"] = str(window)
    with tempfile.TemporaryFile() as out:
        t0 = time.time()
        p = subprocess.run([CLI, "maxk"] + args, stdout=out, stderr=subprocess.PIPE, env=env)
        wall = time.time() - t0
        out.seek(0)
        text = out.read()
    err = p.stderr.decode()
    if p.returncode != 0:
        sys.stderr.write(err[-3000:])
        raise SystemExit("bwa-b200 maxk failed")
    hist = [int(l.split(b"\t")[1]) for l in text.split(b"\n") if l]
    r = dict(wall_s=round(wall, 3), bases=sum(hist), bases_at_255=hist[255])
    m = re.search(r"path: (.*)", err)
    r["path"] = m.group(1) if m else None
    m = re.search(r"\[prof\] maxk: (\d+) bases; index load ([\d.]+) s; search kernel ([\d.]+) ms, longest window ([\d.]+) ms, binning ([\d.]+) ms; "
                  r"list capacity (\d+), runs repeated (\d+);.*total ([\d.]+) s", err)
    if m:
        r.update(index_load_s=float(m.group(2)), kernel_s=round(float(m.group(3)) / 1e3, 3), longest_window_s=round(float(m.group(4)) / 1e3, 3),
                 binning_ms=float(m.group(5)), list_cap=int(m.group(6)), runs_repeated=int(m.group(7)),
                 ns_per_base_kernel=round(float(m.group(3)) * 1e6 / max(int(m.group(1)), 1), 3))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workdir", default=os.environ.get("BWA_B200_BENCH_DIR", "/tmp/bwa_b200_bench"))
    ap.add_argument("--ref-mbp", type=int, default=3000)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--windows", default="0", help="comma-separated BWA_B200_MAXK_WINDOW values for the self-run (0: the command's default)")
    ap.add_argument("--json-out")
    a = ap.parse_args()
    fa, (fq,) = bench.make_workload(a.workdir, a.ref_mbp, a.reads, 150, 1000, 0, False)
    res = dict(workload="maxk, %d Mbp random reference" % a.ref_mbp, **gpu_info())
    ref = self_fasta(a.workdir, a.ref_mbp)
    for w in (int(x) for x in a.windows.split(",")):
        res["self_s_window_%s" % (w or "default")] = run(["-s", fa + ".bwt", ref], w)
    res["reads_default"] = run([fa + ".bwt", fq], 0)
    line = json.dumps(res)
    print(line)
    if a.json_out:
        with open(a.json_out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
