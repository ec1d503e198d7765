#!/usr/bin/env python3
"""End-to-end timing of `bwa-b200 samse` on the benchmark's workload: the 3 Gbp random reference of bench.py (made and indexed by
bench.make_workload, shared with bench.py's work directory) and 1 M single-end 100-bp reads, default options.

  python tools/samse_bench.py [--workdir DIR] [--ref-mbp 3000] [--reads 1000000] [--check-reads 20000] [--json-out FILE]

One command on the GPU box:
  - makes the .sai with `bwa-b200 aln`, outside the timed region;
  - times `bwa-b200 samse idx reads.sai reads.fq > file` end to end, and splits it with BWA_B200_PROFILE (index load; busy time of the
    reader, device and writer threads, which overlap; hits sent to the suffix array; global alignments);
  - runs the reference `bwa samse` on the first --check-reads reads with the .sai of those reads, checks that its SAM without @PG is
    byte for byte the start of ours (the hit choice draws its random numbers in read order, so the first records do not depend on the
    rest of the input), and records its rate with its per-group .bwt/.sa load INCLUDED: the reference reloads them for every group of
    262144 reads, so that load is part of how it runs (its one-time .ann/.pac load is measured on an empty input and subtracted);
  - prints one JSON line with the GPU name, SM count and power limit (nvidia-smi).
Nothing is written to the repository; the output files live in a temporary directory."""
import argparse
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402  (make_workload only)
from aln_bench import gpu_info, head_records, timed  # noqa: E402

CLI = os.path.join(ROOT, "bwa_b200", "bwa-b200")
REF_BWA = os.path.join(ROOT, "oracle", "_ref", "bwa")


def strip_pg(b):
    return b"\n".join(l for l in b.split(b"\n") if not l.startswith(b"@PG"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workdir", default=os.environ.get("BWA_B200_BENCH_DIR", "/tmp/bwa_b200_bench"))
    ap.add_argument("--ref-mbp", type=int, default=3000)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--check-reads", type=int, default=20_000)
    ap.add_argument("--json-out")
    a = ap.parse_args()
    fa, (fq,) = bench.make_workload(a.workdir, a.ref_mbp, a.reads, 100, 1000, 0, False)
    res = dict(workload="samse, %d Mbp random reference, %d single-end 100-bp reads, .sai of bwa-b200 aln with default options" % (a.ref_mbp, a.reads),
               ref_rate_note="the reference's rate includes its .bwt/.sa load, which it repeats for every group of 262144 reads", **gpu_info())
    with tempfile.TemporaryDirectory() as d:
        sai, ours = os.path.join(d, "reads.sai"), os.path.join(d, "ours.sam")
        timed([CLI, "aln", fa, fq], sai)
        wall, err = timed([CLI, "samse", fa, sai, fq], ours, env={"BWA_B200_PROFILE": "1"})
        m = re.search(r"\[prof\] samse: index load ([\d.]+) s; busy time of the reader ([\d.]+) s, the device ([\d.]+) s, the writer ([\d.]+) s; "
                      r"(\d+) hits sent to bwt_sa; (\d+) global alignments; total ([\d.]+) s", err)
        res.update(wall_s=round(wall, 3), output_bytes=os.path.getsize(ours))
        if m:
            load, rd, dev, wr, nsa, nglb, tot = (float(x) for x in m.groups())
            res.update(index_load_s=load, reader_busy_s=rd, device_busy_s=dev, writer_busy_s=wr, sa_hits=int(nsa), global_alignments=int(nglb),
                       after_load_s=round(tot - load, 3), reads_per_s_after_load=round(a.reads / max(tot - load, 1e-9)))
        res["reads_per_s_end_to_end"] = round(a.reads / wall)
        # the reference on the first check-reads reads (their own .sai), and on no reads (its one-time load)
        sub, empty, sub_sai, empty_sai = (os.path.join(d, x) for x in ("sub.fq", "empty.fq", "sub.sai", "empty.sai"))
        head_records(fq, a.check_reads, sub)
        open(empty, "w").close()
        timed([CLI, "aln", fa, sub], sub_sai)
        timed([CLI, "aln", fa, empty], empty_sai)
        t_load, _ = timed([REF_BWA, "samse", fa, empty_sai, empty], os.path.join(d, "ref0.sam"))
        t_ref, _ = timed([REF_BWA, "samse", fa, sub_sai, sub], os.path.join(d, "ref.sam"))
        want = strip_pg(open(os.path.join(d, "ref.sam"), "rb").read())
        with open(ours, "rb") as f:
            got = strip_pg(f.read(len(want) + 4096))[:len(want)]
        res.update(ref_reads=a.check_reads, ref_startup_s=round(t_load, 3), ref_s=round(t_ref - t_load, 3),
                   ref_reads_per_s=round(a.check_reads / max(t_ref - t_load, 1e-9)), identical_to_reference=got == want)
    line = json.dumps(res)
    print(line)
    if a.json_out:
        with open(a.json_out, "w") as f:
            f.write(line + "\n")
    return 0 if res["identical_to_reference"] else 1


if __name__ == "__main__":
    sys.exit(main())
