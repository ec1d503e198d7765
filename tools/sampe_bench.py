#!/usr/bin/env python3
"""End-to-end timing of `bwa-b200 sampe` on the benchmark's workload: the 3 Gbp random reference of bench.py (made and indexed by
bench.make_workload, shared with bench.py's work directory) and 1 M pairs of 100-bp reads, insert N(400, 50), default options.

  python tools/sampe_bench.py [--workdir DIR] [--ref-mbp 3000] [--pairs 1000000] [--check-pairs 20000] [--json-out FILE]

One command on the GPU box:
  - makes the two .sai files with `bwa-b200 aln`, outside the timed region;
  - times `bwa-b200 sampe idx 1.sai 2.sai 1.fq 2.fq > file` end to end and splits it with BWA_B200_PROFILE: index load; busy time of
    the reader, device and writer threads (they overlap, so the largest bounds the command); rows resolved, pairing candidates
    sorted, mate local and global alignments, gapped refinements; and the host part of the device thread (pairing and XA, the
    mate-rescue decisions), which is where the device thread does not wait for the GPU;
  - runs the reference `bwa sampe` and ours on the first --check-pairs pairs (the insert-size model is made per group, so the first
    pairs of a larger run are not comparable) and checks that the SAM without @PG is identical; records the reference's rate with its
    per-group .bwt/.sa load included (its one-time load, measured on an empty input, subtracted);
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
PROF = (r"\[prof\] sampe: index load ([\d.]+) s; busy time of the reader ([\d.]+) s, the device ([\d.]+) s, the writer ([\d.]+) s; "
        r"(\d+) rows sent to bwt_sa; (\d+) pairing candidates sorted; (\d+) mate local alignments, (\d+) mate global alignments; "
        r"(\d+) gapped refinements; host part of the device thread: pairing and XA ([\d.]+) s, mate-rescue decisions ([\d.]+) s; total ([\d.]+) s")


def strip_pg(b):
    return b"\n".join(l for l in b.split(b"\n") if not l.startswith(b"@PG"))


def n_records(fq):
    with open(fq, "rb") as f:
        return sum(1 for _ in f) // 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workdir", default=os.environ.get("BWA_B200_BENCH_DIR", "/tmp/bwa_b200_bench"))
    ap.add_argument("--ref-mbp", type=int, default=3000)
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--check-pairs", type=int, default=20_000)
    ap.add_argument("--json-out")
    a = ap.parse_args()
    fa, fqs = bench.make_workload(a.workdir, a.ref_mbp, 2 * a.pairs, 100, 1000, 0, True)
    pairs = n_records(fqs[0])
    res = dict(workload="sampe, %d Mbp random reference, %d pairs of 100-bp reads, insert N(400, 50), .sai of bwa-b200 aln with default options" % (a.ref_mbp, pairs),
               ref_rate_note="the reference's rate includes its .bwt/.sa load, which it repeats for every group of 262144 pairs", **gpu_info())
    with tempfile.TemporaryDirectory() as d:
        sai = [os.path.join(d, "r%d.sai" % k) for k in (1, 2)]
        ours = os.path.join(d, "ours.sam")
        for s, fq in zip(sai, fqs):
            timed([CLI, "aln", fa, fq], s)
        wall, err = timed([CLI, "sampe", fa, sai[0], sai[1], fqs[0], fqs[1]], ours, env={"BWA_B200_PROFILE": "1"})
        m = re.search(PROF, err)
        res.update(wall_s=round(wall, 3), output_bytes=os.path.getsize(ours))
        if m:
            g = m.groups()
            load, rd, dev, wr = (float(x) for x in g[:4])
            nrow, nsort, nloc, nglb, nref = (int(x) for x in g[4:9])
            tpair, tsw, tot = (float(x) for x in g[9:])
            busy = {"reader": rd, "device": dev, "writer": wr}
            res.update(index_load_s=load, reader_busy_s=rd, device_busy_s=dev, writer_busy_s=wr, bound_by=max(busy, key=busy.get),
                       rows=nrow, pairs_sorted_candidates=nsort, mate_local_alignments=nloc, mate_global_alignments=nglb,
                       gapped_refinements=nref, host_pairing_xa_s=tpair, host_rescue_decisions_s=tsw,
                       after_load_s=round(tot - load, 3), pairs_per_s_after_load=round(pairs / max(tot - load, 1e-9)))
        res["pairs_per_s_end_to_end"] = round(pairs / wall)
        # the reference and ours on the first check-pairs pairs, and the reference on no pairs (its one-time load)
        sub = [os.path.join(d, "sub_%d.fq" % k) for k in (1, 2)]
        ssai = [os.path.join(d, "sub_%d.sai" % k) for k in (1, 2)]
        empty, esai = os.path.join(d, "empty.fq"), os.path.join(d, "empty.sai")
        open(empty, "w").close()
        timed([CLI, "aln", fa, empty], esai)
        for k in range(2):
            head_records(fqs[k], a.check_pairs, sub[k])
            timed([CLI, "aln", fa, sub[k]], ssai[k])
        t_load, _ = timed([REF_BWA, "sampe", fa, esai, esai, empty, empty], os.path.join(d, "ref0.sam"))
        t_ref, _ = timed([REF_BWA, "sampe", fa, ssai[0], ssai[1], sub[0], sub[1]], os.path.join(d, "ref.sam"))
        timed([CLI, "sampe", fa, ssai[0], ssai[1], sub[0], sub[1]], os.path.join(d, "sub.sam"))
        want = strip_pg(open(os.path.join(d, "ref.sam"), "rb").read())
        got = strip_pg(open(os.path.join(d, "sub.sam"), "rb").read())
        res.update(ref_pairs=a.check_pairs, ref_startup_s=round(t_load, 3), ref_s=round(t_ref - t_load, 3),
                   ref_pairs_per_s=round(a.check_pairs / max(t_ref - t_load, 1e-9)), identical_to_reference=got == want)
    line = json.dumps(res)
    print(line)
    if a.json_out:
        with open(a.json_out, "w") as f:
            f.write(line + "\n")
    return 0 if res["identical_to_reference"] else 1


if __name__ == "__main__":
    sys.exit(main())
