"""K3 on chip: reads with at most K3S_CAP seeds are chained with their workspace in shared memory (k_chain_sm), the others in HBM
(k_chain over the list k_chain_sm leaves), and batches with the long-read seed filter entirely in HBM (k_chain, K6, K3b).  SAM is
compared byte for byte with the reference's `bwa mem`; the `[prof] chain:` line says which path each read took."""
import os
import re
import subprocess

import pytest

from conftest import CUSIMBIN, ROOT, ref_sam, strip_pg

GPUBIN = os.path.join(ROOT, "bwa_b200", "bwa-b200")
CAP = 16   # K3S_CAP (bwa_b200/csrc/cuda/bwag_kernels.h)


def run_prof(binary, args, env=None):
    """SAM without @PG, and (reads on chip, reads in HBM, CAP) summed over the batches' [prof] chain: lines"""
    r = subprocess.run([binary, "mem", "-v", "1"] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900,
                       env=dict(os.environ, BWA_B200_PROFILE="1", **(env or {})))
    err = r.stderr.decode()
    assert r.returncode == 0, err[-2000:]
    lines = re.findall(r"\[prof\] chain: (\d+) reads on chip, (\d+) in HBM, CAP (\d+) seeds", err)
    assert lines, "no [prof] chain: line:\n" + err[-2000:]
    caps = {int(x[2]) for x in lines}
    assert caps == {CAP}, caps
    return strip_pg(r.stdout), sum(int(x[0]) for x in lines), sum(int(x[1]) for x in lines)


def write_fq(path, reads):
    with open(path, "w") as f:
        for name, seq in reads:
            f.write("@%s\n%s\n+\n%s\n" % (name, seq, "I" * len(seq)))


def revcomp(s):
    return s[::-1].translate(str.maketrans("ACGT", "TGCA"))


def crafted(data, tmp_path):
    """Reads whose seed counts sit at and just past CAP, reads whose chains share a position (B-tree duplicates) and reads whose
    chains weigh the same (introsort order among equal keys), on the repeat-rich reference."""
    import gen_data
    fa = data.ref("stress")
    seq = gen_data.read_fasta(fa)[0].tobytes().decode()
    L = len(seq) - 400
    reads = []
    # exact copies of one 1-kb family member: every seed occurs at each family copy -> many chains of equal weight, many at equal
    # positions after the family's copies are merged; slide the window to vary the number of copies each seed sees
    for k in range(24):
        p = (200_000 + 997 * k) % L
        reads.append(("fam%d" % k, seq[p:p + 150]))
    # tandem-ish and chimeric reads: two halves from far apart, the second reverse-complemented
    for k in range(24):
        a, b = (50_000 + 4093 * k) % L, (600_000 - 3071 * k) % L
        reads.append(("chim%d" % k, seq[a:a + 75] + revcomp(seq[b:b + 75])))
    # short pieces glued from several places: the number of SMEMs, hence seeds, grows with the number of pieces
    for n_pieces in range(1, 12):
        for k in range(3):
            starts = [(20_000 + 7919 * (j + 13 * k + 3 * n_pieces)) % L for j in range(n_pieces)]
            parts = [seq[x:x + 24] for x in starts]
            reads.append(("glue%d_%d" % (n_pieces, k), "".join(parts)))
    reads = [(n, s) for n, s in reads if len(s) >= 30 and "N" not in s]
    fq = str(tmp_path / "crafted.fq")
    write_fq(fq, reads)
    return fa, [fq]


def cases(data, tmp_path, name):
    if name == "random_se":
        return data.reads("c1", tag="oc", n=300, seed=41), "all"
    if name == "random_pe":
        return data.reads("c1", tag="ocpe", n=150, seed=42, paired=True), "all"
    if name == "stress_pe":
        return data.reads("stress", tag="ocst", n=200, seed=43, paired=True, err=(0.016, 0.002, 0.002), chimeric=0.05), "both"
    if name == "crafted":
        return crafted(data, tmp_path), "both"
    raise KeyError(name)


NAMES = ["random_se", "random_pe", "stress_pe", "crafted"]


def check(binary, data, tmp_path, name):
    (fa, fqs), expect = cases(data, tmp_path, name)
    args = ["-K", "100000000", "-t", "2", fa] + fqs
    sam, on_chip, hbm = run_prof(binary, args)
    assert sam == ref_sam(args)
    if expect == "all":   # random reference: nearly every read has few seeds
        assert on_chip > 0 and hbm <= on_chip // 50, (on_chip, hbm)
    else:
        assert on_chip > 0 and hbm > 0, (on_chip, hbm)


@pytest.mark.parametrize("name", NAMES)
def test_chain_onchip_emulated(data, tmp_path, name):
    check(CUSIMBIN, data, tmp_path, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_chain_onchip_gpu(data, tmp_path, name):
    check(GPUBIN, data, tmp_path, name)


def test_chain_onchip_cap_boundary(data):
    """One read per batch (-K 150): each batch's [prof] line says whether its read had more than CAP seeds.  The repeat-rich
    reads with 2 % error spread over both sides of CAP (their seed counts run from a few to well past it), and every read's SAM
    must equal the reference's whichever path it took."""
    fa, (fq,) = data.reads("stress", tag="occap", n=120, seed=44, err=(0.016, 0.002, 0.002), chimeric=0.05)
    args = ["-K", "150", "-t", "1", fa, fq]
    sam, on_chip, hbm = run_prof(CUSIMBIN, args)
    assert sam == ref_sam(args)
    assert on_chip + hbm == 120 and on_chip > 0 and hbm > 0, (on_chip, hbm)


def test_chain_long_reads_take_hbm(data):
    """Reads long enough for the seed-level filter: the whole batch is chained in HBM and K3b reads the workspace back."""
    fa, fqs = data.reads("two", tag="oclong", n=6, length=1000, seed=45)
    args = ["-K", "100000000", "-t", "2", fa] + fqs
    sam, on_chip, hbm = run_prof(CUSIMBIN, args)
    assert sam == ref_sam(args)
    assert on_chip == 0 and hbm == 6
