#!/usr/bin/env python3
"""Wall time of each step of `bwa index` as a command of its own: fa2pac, pac2bwt, bwtupdate, fa2pac -f, bwt2sa.

  python tools/index_steps_bench.py [--small-mbp 100] [--large-mbp 3000] [--skip-ref] [--skip-large] [--json-out FILE]

  - on a --small-mbp uniform-random reference (4 contigs, tools/gen_data.py seed 13): the chain of `bwa-b200` and the chain of the
    reference's `bwa` (oracle/_ref/bwa), with a byte-for-byte check of the five files;
  - on the --large-mbp benchmark reference (24 contigs, seed 7): the chain of `bwa-b200` alone (the reference's `bwt2sa` alone is
    one dependent LF step per base on one core), with the peak device memory each device step reports;
  - one JSON line with the GPU name and power limit (nvidia-smi) beside the numbers.
Everything it writes lives in a temporary directory."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_data  # noqa: E402

CLI = os.path.join(ROOT, "bwa_b200", "bwa-b200")
REF_BWA = os.path.join(ROOT, "oracle", "_ref", "bwa")
EXTS = ("pac", "ann", "amb", "bwt", "sa")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,memory.total", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=60).stdout
        name, power, mem = [x.strip() for x in q.splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=power, memory=mem)
    except Exception as e:   # noqa: BLE001 -- the numbers stay usable without it
        return dict(gpu_query_error=str(e))


def chain(binary, d, fa):
    """the five steps in directory d; per step: wall seconds and the peak device memory it reports (GB)"""
    out = {}
    for name, args in (("fa2pac", ["fa2pac", fa]), ("pac2bwt", ["pac2bwt", fa + ".pac", fa + ".bwt"]), ("bwtupdate", ["bwtupdate", fa + ".bwt"]),
                       ("fa2pac_f", ["fa2pac", "-f", fa]), ("bwt2sa", ["bwt2sa", fa + ".bwt", fa + ".sa"])):
        t0 = time.time()
        p = subprocess.run([binary] + args, cwd=d, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)
        dt = time.time() - t0
        if p.returncode != 0:
            sys.stderr.write(p.stderr[-3000:])
            raise SystemExit("%s %s failed" % (binary, name))
        m = re.search(r"peak device memory ([0-9.]+) GB", p.stderr)
        out[name] = {"s": round(dt, 2)}
        if m:
            out[name]["peak_gb"] = float(m.group(1))
        m = re.search(r"(\d+) rulers (\d+) rows apart", p.stderr)
        if m:
            out[name].update(rulers=int(m.group(1)), stride=int(m.group(2)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small-mbp", type=int, default=100)
    ap.add_argument("--large-mbp", type=int, default=3000)
    ap.add_argument("--skip-ref", action="store_true", help="do not run the reference's chain")
    ap.add_argument("--skip-large", action="store_true")
    ap.add_argument("--json-out")
    a = ap.parse_args()
    res = dict(gpu_info())
    with tempfile.TemporaryDirectory() as tmp:
        mine, ref = os.path.join(tmp, "mine"), os.path.join(tmp, "ref")
        os.mkdir(mine)
        os.mkdir(ref)
        gen_data.write_fasta(os.path.join(mine, "r.fa"), gen_data.random_contigs(4, a.small_mbp * 250000, 13))
        shutil.copy(os.path.join(mine, "r.fa"), os.path.join(ref, "r.fa"))
        res["small_mbp"] = a.small_mbp
        res["small_bwa_b200"] = chain(CLI, mine, "r.fa")
        if not a.skip_ref:
            res["small_bwa"] = chain(REF_BWA, ref, "r.fa")
            res["small_identical"] = all(open(os.path.join(mine, "r.fa." + e), "rb").read() == open(os.path.join(ref, "r.fa." + e), "rb").read() for e in EXTS)
        shutil.rmtree(mine)
        shutil.rmtree(ref)
        if not a.skip_large:
            big = os.path.join(tmp, "big")
            os.mkdir(big)
            n_ctg = 24
            gen_data.write_fasta(os.path.join(big, "g.fa"), gen_data.random_contigs(n_ctg, a.large_mbp * 1000000 // n_ctg, 7))
            res["large_mbp"] = a.large_mbp
            res["large_bwa_b200"] = chain(CLI, big, "g.fa")
    line = json.dumps(res)
    print(line)
    if a.json_out:
        with open(a.json_out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
