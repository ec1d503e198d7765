#!/usr/bin/env python3
"""End-to-end timing of `bwa-b200 pemerge` against the reference's `bwa pemerge -t 16` on the same input.

  python tools/pemerge_bench.py [--pairs 1000000] [--threads 16] [--seed 7] [--json-out FILE]

Data (generated before anything is timed, from a seed): a 10 Mbp random reference, pairs of 2 x 150 bp with inserts drawn from
N(250, 60) (at least 20 bp; a read longer than its insert runs into random bases), 1 % substitutions, random qualities 2-41.
One command on the GPU box:
  - times `bwa-b200 pemerge r1.fq r2.fq > file` end to end, and records the busy time of its reader, device and writer threads, which
    overlap (BWA_B200_PROFILE);
  - times `bwa pemerge -t THREADS` on the same files and checks that both outputs and count lines are identical;
  - prints one JSON line with the GPU name, its power limit, the SM count and the host's CPU count.
Nothing is written to the repository; the files live in a temporary directory."""
import argparse
import hashlib
import json
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from aln_bench import gpu_info, timed  # noqa: E402

CLI = os.path.join(ROOT, "bwa_b200", "bwa-b200")
REF_BWA = os.path.join(ROOT, "oracle", "_ref", "bwa")
L = 150


def make_pairs(d, n, seed):
    rng = np.random.default_rng(seed)
    ref = rng.integers(0, 4, 10_000_000, dtype=np.uint8)
    ins = np.clip(np.rint(rng.normal(250, 60, n)), 20, 1000).astype(np.int64)
    pos = rng.integers(0, len(ref) - 1001, n)
    j = np.arange(L)[None, :]
    inside = j < ins[:, None]
    r1 = np.where(inside, ref[np.minimum(pos[:, None] + j, len(ref) - 1)], rng.integers(0, 4, (n, L), dtype=np.uint8))
    r2 = np.where(inside, 3 - ref[np.clip(pos[:, None] + ins[:, None] - 1 - j, 0, len(ref) - 1)], rng.integers(0, 4, (n, L), dtype=np.uint8))
    paths = []
    for mate, r in ((1, r1), (2, r2)):
        sub = rng.random((n, L)) < 0.01
        r = np.where(sub, (r + rng.integers(1, 4, (n, L), dtype=np.uint8)) % 4, r).astype(np.uint8)
        qual = rng.integers(2 + 33, 41 + 34, (n, L), dtype=np.uint8)
        name = np.zeros((n, 12), dtype=np.uint8)   # "@r0000001/1\n"
        name[:, 0] = ord("@"); name[:, 1] = ord("r")
        k = np.arange(n)
        for p in range(7):
            name[:, 8 - p] = ord("0") + (k // 10 ** p) % 10
        name[:, 9] = ord("/"); name[:, 10] = ord("0") + mate; name[:, 11] = 10
        nl = np.full((n, 1), 10, dtype=np.uint8)
        rec = np.concatenate([name, np.frombuffer(b"ACGT", dtype=np.uint8)[r], nl, np.full((n, 1), ord("+"), dtype=np.uint8), nl, qual, nl], axis=1)
        path = os.path.join(d, "r%d.fq" % mate)
        rec.tofile(path)
        paths.append(path)
    return paths


def digest(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    return h.hexdigest()


def counts(err):
    return [l for l in err.split("\n") if re.match(r"^ *\d+ (successful|low-scoring|pairs )", l)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--json-out")
    a = ap.parse_args()
    res = dict(workload="pemerge, %d pairs of 2 x %d bp, insert N(250, 60), 1 %% substitutions, random qualities 2-41" % (a.pairs, L),
               cpus=os.cpu_count(), **gpu_info())
    with tempfile.TemporaryDirectory() as d:
        r1, r2 = make_pairs(d, a.pairs, a.seed)
        ours, theirs = os.path.join(d, "ours.fq"), os.path.join(d, "ref.fq")
        timed([CLI, "pemerge", r1, r2], ours)   # warm-up: module load and page cache
        wall, err = timed([CLI, "pemerge", r1, r2], ours, env={"BWA_B200_PROFILE": "1"})
        m = re.search(r"\[prof\] pemerge: busy time of the reader ([\d.]+) s, the device ([\d.]+) s, the writer ([\d.]+) s", err)
        res.update(wall_s=round(wall, 3), pairs_per_s=round(a.pairs / wall), output_bytes=os.path.getsize(ours))
        if m:
            res.update(reader_busy_s=float(m.group(1)), device_busy_s=float(m.group(2)), writer_busy_s=float(m.group(3)))
        t_ref, err_ref = timed([REF_BWA, "pemerge", "-t", str(a.threads), r1, r2], theirs)
        res.update(ref_threads=a.threads, ref_wall_s=round(t_ref, 3), ref_pairs_per_s=round(a.pairs / t_ref),
                   merged=int(counts(err_ref)[0].split()[0]) if counts(err_ref) else None,
                   identical_to_reference=digest(ours) == digest(theirs) and counts(err) == counts(err_ref))
    line = json.dumps(res)
    print(line)
    if a.json_out:
        with open(a.json_out, "w") as f:
            f.write(line + "\n")
    return 0 if res["identical_to_reference"] else 1


if __name__ == "__main__":
    sys.exit(main())
