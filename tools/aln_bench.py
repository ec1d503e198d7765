#!/usr/bin/env python3
"""End-to-end timing of `bwa-b200 aln` on the benchmark's workload: the 3 Gbp random reference of bench.py (made and indexed by
bench.make_workload, shared with bench.py's work directory) and 1 M single-end 100-bp reads, default options.

  python tools/aln_bench.py [--workdir DIR] [--ref-mbp 3000] [--reads 1000000] [--check-reads 20000] [--json-out FILE]

One command on the GPU box:
  - times `bwa-b200 aln -t <cpus> idx reads.fq > file` end to end, and splits it with BWA_B200_PROFILE (index load; busy time of the
    reader, device and writer threads, which overlap; reads that needed the second tier of queue memory);
  - runs the reference `bwa aln -t <cpus>` (all CPUs) on the first --check-reads reads, checks that its .sai is byte for byte the start
    of ours, and records its rate (its index load, measured on an empty input, is subtracted);
  - prints one JSON line with the GPU name, SM count and power limit (nvidia-smi).
Nothing is written to the repository; the output files live in a temporary directory."""
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
REF_BWA = os.path.join(ROOT, "oracle", "_ref", "bwa")


def gpu_info():
    info = {}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,memory.total", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=60).stdout
        name, power, mem = [x.strip() for x in q.splitlines()[0].split(",")]
        info.update(gpu=name, power_limit=power, memory=mem)
    except Exception as e:   # noqa: BLE001 -- the numbers stay usable without it
        info["gpu_query_error"] = str(e)
    try:
        import torch
        info["sm_count"] = torch.cuda.get_device_properties(0).multi_processor_count
    except Exception as e:   # noqa: BLE001
        info["sm_query_error"] = str(e)
    return info


def timed(cmd, out_path, env=None):
    t0 = time.time()
    with open(out_path, "wb") as o:
        p = subprocess.run(cmd, stdout=o, stderr=subprocess.PIPE, env=dict(os.environ, **(env or {})))
    dt = time.time() - t0
    if p.returncode != 0:
        sys.stderr.write(p.stderr.decode()[-3000:])
        raise SystemExit("command failed: %s" % " ".join(cmd))
    return dt, p.stderr.decode()


def head_records(fq, n, out):
    """the first n FASTQ records (4 lines each: gen_data writes no wrapped lines)"""
    with open(fq, "rb") as i, open(out, "wb") as o:
        for k, line in enumerate(i):
            if k >= 4 * n:
                break
            o.write(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workdir", default=os.environ.get("BWA_B200_BENCH_DIR", "/tmp/bwa_b200_bench"))
    ap.add_argument("--ref-mbp", type=int, default=3000)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--check-reads", type=int, default=20_000)
    ap.add_argument("--json-out")
    a = ap.parse_args()
    fa, (fq,) = bench.make_workload(a.workdir, a.ref_mbp, a.reads, 100, 1000, 0, False)
    t = str(os.cpu_count() or 1)   # -t only changes the header; the same value on both sides keeps the bytes comparable
    res = dict(workload="aln, %d Mbp random reference, %d single-end 100-bp reads, default options" % (a.ref_mbp, a.reads), cpus=int(t), **gpu_info())
    with tempfile.TemporaryDirectory() as d:
        ours = os.path.join(d, "ours.sai")
        wall, err = timed([CLI, "aln", "-t", t, fa, fq], ours, env={"BWA_B200_PROFILE": "1"})
        m = re.search(r"\[prof\] aln: index load ([\d.]+) s; busy time of the reader ([\d.]+) s, the device ([\d.]+) s, the writer ([\d.]+) s; (\d+) reads in tier 2; total ([\d.]+) s", err)
        res.update(wall_s=round(wall, 3), output_bytes=os.path.getsize(ours))
        if m:
            load, rd, dev, wr, t2, tot = (float(x) for x in m.groups())
            res.update(index_load_s=load, reader_busy_s=rd, device_busy_s=dev, writer_busy_s=wr, tier2_reads=int(t2), after_load_s=round(tot - load, 3),
                       reads_per_s_after_load=round(a.reads / max(tot - load, 1e-9)))
        res["reads_per_s_end_to_end"] = round(a.reads / wall)
        # the reference on the first check-reads reads, and on no reads (its index load)
        sub, empty = os.path.join(d, "sub.fq"), os.path.join(d, "empty.fq")
        head_records(fq, a.check_reads, sub)
        open(empty, "w").close()
        t_load, _ = timed([REF_BWA, "aln", "-t", t, fa, empty], os.path.join(d, "ref0.sai"))
        t_ref, _ = timed([REF_BWA, "aln", "-t", t, fa, sub], os.path.join(d, "ref.sai"))
        want = open(os.path.join(d, "ref.sai"), "rb").read()
        with open(ours, "rb") as f:
            got = f.read(len(want))
        res.update(ref_reads=a.check_reads, ref_index_load_s=round(t_load, 3), ref_s=round(t_ref - t_load, 3),
                   ref_reads_per_s=round(a.check_reads / max(t_ref - t_load, 1e-9)), identical_to_reference=got == want)
    line = json.dumps(res)
    print(line)
    if a.json_out:
        with open(a.json_out, "w") as f:
            f.write(line + "\n")
    return 0 if res["identical_to_reference"] else 1


if __name__ == "__main__":
    sys.exit(main())
