"""`bwa-b200 fastmap` against the reference's `bwa fastmap` (oracle/_ref/bwa): stdout byte for byte and the exit status, on the
emulated kernels (tests/_build/bwa-b200-cusim) and on the GPU.  Cases: datasets of short, chimeric and long noisy reads; edge reads
(empty, all N, N runs, lowercase, IUPAC codes, 1 base, across a contig junction and its reverse complement, a whole contig,
multi-line FASTA, names with comments); the options -w -l -i -I -L -p; gzip, stdin and FASTA input; batches of 1 and 1000 bases
(BWA_B200_FASTMAP_CHUNK) and interval pools that overflow (BWA_B200_TEST_SMALL_POOLS, the repeat path); 2^16-symbol Occ
superblocks; an index kept resident by `bwa-b200 shm`; the errors of the command line."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import bwa_b200
from conftest import CUSIMBIN, REF_BWA, ROOT, TESTBIN

GPUBIN = bwa_b200.CLI_PATH


def _run(cmd, env=None, stdin=None):
    e = dict(os.environ, **(env or {}))
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1800, env=e, input=stdin)


def _same(binary, args, env=None, stdin=None):
    """stdout and exit status of `binary fastmap args` equal those of `bwa fastmap args`; returns the run"""
    want = _run([REF_BWA, "fastmap"] + args, stdin=stdin)
    got = _run([binary, "fastmap"] + args, env=env, stdin=stdin)
    assert got.returncode == want.returncode, (args, got.stderr.decode()[-2000:])
    if got.stdout != want.stdout:
        a, b = want.stdout.split(b"\n"), got.stdout.split(b"\n")
        k = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
        raise AssertionError("%r: line %d differs:\n  bwa      %r\n  bwa-b200 %r" % (args, k, a[k][:300] if k < len(a) else None, b[k][:300] if k < len(b) else None))
    return got


def _datasets(data, n_c1, n_two, n_stress, n_2k, n_10k):
    noisy = (0.08, 0.01, 0.01)   # 10 % error
    return [data.reads("c1", tag="fm_c1_%d" % n_c1, n=n_c1, seed=61),
            data.reads("two", tag="fm_two_%d" % n_two, n=n_two, seed=62),
            data.reads("stress", tag="fm_st_%d" % n_stress, n=n_stress, seed=63, err=(0.016, 0.002, 0.002), chimeric=0.05),
            data.reads("two", tag="fm_2k_%d" % n_2k, n=n_2k, length=2000, seed=64, err=noisy),
            data.reads("c1", tag="fm_10k_%d" % n_10k, n=n_10k, length=10000, seed=65, err=noisy)]


def _revcomp(s):
    return s[::-1].translate(str.maketrans("ACGTacgtN", "TGCAtgcaN"))


def _edge_files(tmp_path):
    """a three-contig reference (indexed by `bwa index`) and the edge reads, as FASTQ and as multi-line FASTA"""
    rng = np.random.default_rng(71)
    rand = lambda n: "".join("ACGT"[i] for i in rng.integers(0, 4, n))
    ctg = [rand(6000), rand(2500), rand(800)]
    ctg[2] = ctg[0][1000:1400] + ctg[2][400:]   # a repeat: two occurrences
    fa = str(tmp_path / "edge.fa")
    with open(fa, "w") as f:
        for i, s in enumerate(ctg):
            f.write(">ctg%d desc %d\n%s\n" % (i + 1, i, "\n".join(s[k:k + 70] for k in range(0, len(s), 70))))
    subprocess.run([REF_BWA, "index", fa], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    a, b = ctg[0], ctg[1]
    junction = a[-60:] + b[:60]
    reads = [("empty", ""), ("alln", "N" * 120), ("nrun", a[100:160] + "N" * 15 + a[175:260]),
             ("lower comment with spaces", a[300:420].lower()), ("mixedcase\tand tab", a[500:560] + a[560:620].lower()),
             ("iupac", a[700:750] + "RYKM" + a[754:800] + "SWBDHV" + a[806:850]), ("one", "A"), ("oneN", "N"), ("oneg", "g"),
             ("junction", junction), ("junction_rc", _revcomp(junction)), ("whole", b), ("whole_rc", _revcomp(ctg[2])),
             ("repeat", a[1050:1200]), ("repeat_rc", _revcomp(a[1100:1350])), ("dash", a[2000:2050] + "-" + a[2051:2100]),
             ("tail", a[-1:] + b[:1] + "ACGT"), ("x", "N" * 7 + a[3000:3005] + "N")]
    fq, fasta = str(tmp_path / "edge.fq"), str(tmp_path / "edge_reads.fa")
    with open(fq, "w") as f:
        for name, s in reads:
            f.write("@%s\n%s\n+\n%s\n" % (name, s, "I" * len(s)))
    with open(fasta, "w") as f:
        for name, s in reads:
            f.write(">%s\n%s\n" % (name, "\n".join(s[k:k + 37] for k in range(0, len(s), 37))))
    return fa, [fq, fasta]


OPTIONS = [["-w", "0"], ["-w", "1"], ["-w", "5"], ["-w", "-1"], ["-l", "0"], ["-l", "1"], ["-l", "40"], ["-l", "-1"],
           ["-i", "0"], ["-i", "2"], ["-i", "10"], ["-I", "1"], ["-I", "5"], ["-I", "50"],
           ["-I", "1", "-l", "10"], ["-I", "5", "-l", "10"], ["-I", "50", "-l", "10"], ["-L", "30"], ["-p"], ["-p", "-w", "1", "-I", "3"]]


def _check_datasets(binary, data, sizes):
    for fa, fqs in _datasets(data, *sizes):
        _same(binary, [fa] + fqs)


def _check_edges(binary, tmp_path):
    fa, inputs = _edge_files(tmp_path)
    for f in inputs:
        for extra in ([], ["-p"], ["-l", "1", "-w", "-1"], ["-l", "0", "-i", "2"], ["-I", "2", "-l", "5"]):
            _same(binary, extra + [fa, f])


def _check_options(binary, data, n_stress):
    fa, fqs = data.reads("stress", tag="fm_st_%d" % n_stress, n=n_stress, seed=63, err=(0.016, 0.002, 0.002), chimeric=0.05)
    for extra in OPTIONS:
        _same(binary, extra + [fa] + fqs)


# ---------------------------------------------------------------------------------------------------- emulated kernels (CPU)

def test_fastmap_datasets_emulated(data):
    _check_datasets(CUSIMBIN, data, (2000, 300, 500, 50, 20))


def test_fastmap_edge_reads_emulated(tmp_path):
    _check_edges(CUSIMBIN, tmp_path)


def test_fastmap_options_emulated(data):
    _check_options(CUSIMBIN, data, 300)


def test_fastmap_input_forms_emulated(data, tmp_path):
    fa, fqs = data.reads("two", tag="fm_two_300", n=300, seed=62)
    raw = open(fqs[0], "rb").read()
    gz = str(tmp_path / "r.fq.gz")
    with gzip.open(gz, "wb") as f:
        f.write(raw)
    _same(CUSIMBIN, [fa, gz])
    _same(CUSIMBIN, [fa, "-"], stdin=raw)
    fasta = str(tmp_path / "r.fa")
    lines = raw.decode().split("\n")
    with open(fasta, "w") as f:
        for k in range(0, len(lines) - 3, 4):
            f.write(">" + lines[k][1:] + "\n" + lines[k + 1] + "\n")
    _same(CUSIMBIN, ["-p", fa, fasta])


def test_fastmap_batches_emulated(data):
    """the same bytes whatever the batch size, and when the interval pool of K1 overflows and the stage is repeated"""
    fa, fqs = data.reads("stress", tag="fm_st_300", n=300, seed=63, err=(0.016, 0.002, 0.002), chimeric=0.05)
    outs = set()
    for env in ({"BWA_B200_FASTMAP_CHUNK": "1"}, {"BWA_B200_FASTMAP_CHUNK": "1000"}, {}, {"BWA_B200_TEST_SMALL_POOLS": "1", "BWA_B200_PROFILE": "1"}):
        r = _same(CUSIMBIN, ["-l", "5", fa] + fqs, env=env)
        outs.add(r.stdout)
        if "BWA_B200_TEST_SMALL_POOLS" in env:
            assert b"seeding repeated" in r.stderr
            assert b"[prof] fastmap:" in r.stderr
    assert len(outs) == 1


def _sb16(binary, data):
    if not os.path.exists(binary):
        subprocess.run(["make", "-C", ROOT, "sb16" if "cusim" in binary else "sb16-cuda"], check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    fa, fqs = data.reads("c1", tag="fm_sb16", n=400, seed=66)
    for extra in ([], ["-w", "-1", "-l", "10"], ["-I", "5"]):
        _same(binary, extra + [fa] + fqs)


def test_fastmap_small_superblocks_emulated(data):
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-cusim-sb16"), data)


def _resident(binary, data, tmp_path, n):
    fa, fqs = data.reads("two", tag="fm_res%d" % n, n=n, seed=67)
    env = {"BWA_B200_SHM_DIR": str(tmp_path)}
    try:
        r = _run([binary, "shm", fa], env=env)
        assert r.returncode == 0, r.stderr.decode()[-2000:]
        r = _same(binary, ["-w", "-1", fa] + fqs, env=env)
        assert b"using the index resident on the GPU" in r.stderr
        assert b".bwt" not in r.stderr                  # the FM-index files were not opened
    finally:
        _run([binary, "shm", "-d"], env=env)
    assert not [f for f in os.listdir(str(tmp_path)) if f.endswith(".resident")]


def test_fastmap_resident_index_emulated(data, tmp_path):
    _resident(CUSIMBIN, data, tmp_path, 60)


def test_fastmap_errors(data, tmp_path):
    fa, fqs = data.reads("two", tag="fm_two_300", n=300, seed=62)
    for args in ([], [fa], ["-x", fa] + fqs, [str(tmp_path / "missing")] + fqs):
        r = _same(CUSIMBIN, args)
        assert r.returncode != 0 and r.stdout == b""
    r = _run([TESTBIN, "fastmap", fa] + fqs)   # the host pipeline over the CPU oracle stages: no device SMEM lister
    assert r.returncode != 0 and r.stdout == b""
    assert b"no device SMEM lister" in r.stderr


# ---------------------------------------------------------------------------------------------------- H100

@pytest.mark.gpu
def test_fastmap_datasets_gpu(data):
    _check_datasets(GPUBIN, data, (2000, 300, 500, 50, 20))


@pytest.mark.gpu
def test_fastmap_edge_reads_gpu(tmp_path):
    _check_edges(GPUBIN, tmp_path)


@pytest.mark.gpu
def test_fastmap_options_gpu(data):
    _check_options(GPUBIN, data, 3000)


@pytest.mark.gpu
def test_fastmap_small_superblocks_gpu(data):
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-sb16"), data)


@pytest.mark.gpu
def test_fastmap_resident_index_gpu(data, tmp_path):
    _resident(GPUBIN, data, tmp_path, 2000)


@pytest.mark.gpu
def test_fastmap_100mbp_gpu(tmp_path):
    """a 100 Mbp random reference indexed by `bwa-b200 index`; 200 000 reads of 150 bp and 1 000 of 10 kbp"""
    import gen_data
    contigs = gen_data.random_contigs(4, 25_000_000, 81)
    fa = str(tmp_path / "ref100.fa")
    gen_data.write_fasta(fa, contigs)
    r = _run([GPUBIN, "index", fa])
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    fq = str(tmp_path / "reads.fq")
    short, _ = gen_data.gen_reads(contigs, 200_000, 150, 82)
    long_, _ = gen_data.gen_reads(contigs, 1000, 10000, 83, err=(0.08, 0.01, 0.01), prefix="L")
    gen_data.write_fastq(fq, short + long_)
    del contigs, short, long_
    for extra in ([], ["-w", "1000", "-l", "25", "-i", "2"]):
        _same(GPUBIN, extra + [fa, fq])
