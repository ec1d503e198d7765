"""`bwa-b200 maxk` against the reference's `bwa maxk` (oracle/_ref/bwa): stdout byte for byte and the exit status, on the emulated
kernels (tests/_build/bwa-b200-cusim) and on the GPU.  Cases: read sets of 150-bp, 2-kbp and 10-kbp reads and each reference
against itself, with and without -s; the edge queries of test_fastmap.py as FASTQ, multi-line FASTA, gzip and stdin; windows of
1, 7 and more bases than any sequence (BWA_B200_MAXK_WINDOW) and one sequence per batch (BWA_B200_MAXK_CHUNK); references on
which some base occurs fewer than min_intv times (one window per sequence); interval lists that outgrow their scratch
(BWA_B200_TEST_SMALL_POOLS); 2^16-symbol Occ superblocks; the errors of the command line."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import bwa_b200
from conftest import CUSIMBIN, REF_BWA, ROOT, TESTBIN
from test_fastmap import _edge_files

GPUBIN = bwa_b200.CLI_PATH


def _run(cmd, env=None, stdin=None):
    e = dict(os.environ, **(env or {}))
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=3600, env=e, input=stdin)


def _same(binary, args, env=None, stdin=None):
    """stdout and exit status of `binary maxk args` equal those of `bwa maxk args`; returns the run"""
    want = _run([REF_BWA, "maxk"] + args, stdin=stdin)
    got = _run([binary, "maxk"] + args, env=env, stdin=stdin)
    assert got.returncode == want.returncode, (args, env, got.stderr.decode()[-2000:])
    assert got.stdout == want.stdout, (args, env, [(a, b) for a, b in zip(want.stdout.split(b"\n"), got.stdout.split(b"\n")) if a != b][:5])
    return got


def _read_sets(data):
    noisy = (0.08, 0.01, 0.01)
    return [data.reads("c1", tag="mk_c1_2000", n=2000, seed=91),
            data.reads("two", tag="mk_two_300", n=300, seed=92),
            data.reads("stress", tag="mk_st_500", n=500, seed=93, err=(0.016, 0.002, 0.002), chimeric=0.05),
            data.reads("two", tag="mk_2k_50", n=50, length=2000, seed=94, err=noisy),
            data.reads("c1", tag="mk_10k_20", n=20, length=10000, seed=95, err=noisy)]


def _check_read_sets(binary, data):
    for fa, (fq,) in _read_sets(data):
        for extra in ([], ["-s"]):
            r = _same(binary, extra + [fa + ".bwt", fq], env={"BWA_B200_PROFILE": "1"})
            assert b"[prof] maxk: path: windows of 1024 bases" in r.stderr   # every base occurs twice or more: windows
    return True


def _check_self(binary, data):
    for name in ("c1", "two", "stress"):
        fa = data.ref(name)
        for extra in ([], ["-s"]):
            r = _same(binary, extra + [fa + ".bwt", fa])
            if name == "stress":   # the repeat family and tandem repeats reach 255, the N runs bin 0
                hist = [int(l.split(b"\t")[1]) for l in r.stdout.split(b"\n") if l]
                assert hist[0] > 0 and hist[255] > 0


def _check_edges(binary, tmp_path):
    fa, inputs = _edge_files(tmp_path)
    raw = open(inputs[0], "rb").read()
    gz = str(tmp_path / "edge.fq.gz")
    with gzip.open(gz, "wb") as f:
        f.write(raw)
    for extra in ([], ["-s"]):
        for f in inputs + [gz]:
            _same(binary, extra + [fa + ".bwt", f])
        _same(binary, extra + [fa + ".bwt", "-"], stdin=raw)


def _check_windows(binary, data, tmp_path):
    """the same bytes whatever the window and the batch"""
    fa, (fq,) = data.reads("stress", tag="mk_st_100", n=100, seed=96, err=(0.016, 0.002, 0.002), chimeric=0.05)
    efa, inputs = _edge_files(tmp_path)
    for env in ({"BWA_B200_MAXK_WINDOW": "1"}, {"BWA_B200_MAXK_WINDOW": "7"}, {"BWA_B200_MAXK_WINDOW": "1000000000"},
                {"BWA_B200_MAXK_CHUNK": "1"}, {"BWA_B200_MAXK_CHUNK": "1", "BWA_B200_MAXK_WINDOW": "7"}):
        for extra in ([], ["-s"]):
            _same(binary, extra + [fa + ".bwt", fq], env=env)
            _same(binary, extra + [efa + ".bwt", inputs[1]], env=env)
    two = data.ref("two")
    for env in ({"BWA_B200_MAXK_WINDOW": "64"}, {"BWA_B200_MAXK_WINDOW": "1000000000"}, {"BWA_B200_MAXK_CHUNK": "1"}):
        _same(binary, ["-s", two + ".bwt", two], env=env)


def _rare_base_refs(tmp_path):
    """an A/T reference with one C (C and G occur once: -s fails the base-count condition) and one without C or G (default mode
    fails it too), each indexed by `bwa index`; queries: the reference itself and reads with substitutions and Ns"""
    rng = np.random.default_rng(97)
    out = []
    for tag, one_c in (("at1c", True), ("at", False)):
        s = list("AT"[i] for i in rng.integers(0, 2, 6000))
        if one_c:
            s[3217] = "C"
        s = "".join(s)
        fa = str(tmp_path / (tag + ".fa"))
        with open(fa, "w") as f:
            f.write(">%s\n%s\n" % (tag, "\n".join(s[k:k + 60] for k in range(0, len(s), 60))))
        subprocess.run([REF_BWA, "index", fa], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        fq = str(tmp_path / (tag + ".fq"))
        with open(fq, "w") as f:
            for k in range(40):
                p = int(rng.integers(0, len(s) - 300))
                r = list(s[p:p + 300])
                for _ in range(int(rng.integers(0, 6))):
                    r[int(rng.integers(0, 300))] = "ACGTN"[int(rng.integers(0, 5))]
                if k == 0:
                    r = list(s[3100:3400])   # across the C
                f.write("@r%d\n%s\n+\n%s\n" % (k, "".join(r), "I" * 300))
        out.append((fa, fq))
    return out


def _check_rare_bases(binary, tmp_path):
    for fa, fq in _rare_base_refs(tmp_path):
        for extra in ([], ["-s"]):
            for q in (fq, fa):
                r = _same(binary, extra + [fa + ".bwt", q], env={"BWA_B200_PROFILE": "1", "BWA_B200_MAXK_WINDOW": "7"})
                fails = extra == ["-s"] or fa.endswith("at.fa")
                assert (b"path: one window per sequence" in r.stderr) == fails, (fa, extra, r.stderr.decode()[-500:])


def _check_overflow(binary, tmp_path):
    """a query with a 1.5 kbp exact repeat and a tandem repeat: its interval lists outgrow the forced small scratch and the batch is run again"""
    rng = np.random.default_rng(98)
    rand = lambda n: "".join("ACGT"[i] for i in rng.integers(0, 4, n))
    rep, unit = rand(1500), rand(3)
    ctg = [rand(3000) + rep + rand(2000) + unit * 400 + rand(1000), rand(2500) + rep + rand(3000)]
    fa = str(tmp_path / "rep.fa")
    with open(fa, "w") as f:
        for i, s in enumerate(ctg):
            f.write(">c%d\n%s\n" % (i, s))
    subprocess.run([REF_BWA, "index", fa], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    for extra in ([], ["-s"]):
        for env in ({}, {"BWA_B200_MAXK_WINDOW": "1000000000"}):
            r = _same(binary, extra + [fa + ".bwt", fa], env=dict(env, BWA_B200_TEST_SMALL_POOLS="1", BWA_B200_PROFILE="1"))
            assert b"runs repeated 0;" not in r.stderr, r.stderr.decode()[-500:]


def _sb16(binary, data):
    if not os.path.exists(binary):
        subprocess.run(["make", "-C", ROOT, "sb16" if "cusim" in binary else "sb16-cuda"], check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    fa, (fq,) = data.reads("c1", tag="mk_sb16", n=400, seed=99)
    for extra in ([], ["-s"]):
        _same(binary, extra + [fa + ".bwt", fq])
    _same(binary, ["-s", fa + ".bwt", fa])


# ---------------------------------------------------------------------------------------------------- emulated kernels (CPU)

def test_maxk_read_sets_emulated(data):
    _check_read_sets(CUSIMBIN, data)


def test_maxk_self_emulated(data):
    _check_self(CUSIMBIN, data)


def test_maxk_edge_queries_emulated(tmp_path):
    _check_edges(CUSIMBIN, tmp_path)


def test_maxk_windows_and_batches_emulated(data, tmp_path):
    _check_windows(CUSIMBIN, data, tmp_path)


def test_maxk_rare_bases_emulated(tmp_path):
    _check_rare_bases(CUSIMBIN, tmp_path)


def test_maxk_list_overflow_emulated(tmp_path):
    _check_overflow(CUSIMBIN, tmp_path)


def test_maxk_small_superblocks_emulated(data):
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-cusim-sb16"), data)


def test_maxk_errors(data, tmp_path):
    fa, (fq,) = data.reads("two", tag="mk_two_300", n=300, seed=92)
    bwt = fa + ".bwt"
    for args in ([], [bwt], [str(tmp_path / "missing.bwt"), fq], [bwt, str(tmp_path / "missing.fq")], ["-x", bwt, fq]):
        r = _same(CUSIMBIN, args)
        if args[:1] != ["-x"]:   # the reference reports an unknown option and ignores it
            assert r.returncode == 1 and r.stdout == b""
    # where the reference crashes: a FASTA file and a .bwt without Occ checkpoints given as the index
    raw = str(tmp_path / "raw.bwt")
    subprocess.run([REF_BWA, "pac2bwt", fa + ".pac", raw], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    for index, why in ((fa, b"is not a"), (raw, b"has no Occ checkpoints")):
        r = _run([CUSIMBIN, "maxk", index, fq])
        assert r.returncode == 1 and r.stdout == b"" and why in r.stderr, r.stderr
    r = _run([TESTBIN, "maxk", bwt, fq])   # the host pipeline over the CPU oracle stages: no device SMEM search
    assert r.returncode == 1 and r.stdout == b""
    assert b"no device SMEM search" in r.stderr


# ---------------------------------------------------------------------------------------------------- H100

@pytest.mark.gpu
def test_maxk_read_sets_gpu(data):
    _check_read_sets(GPUBIN, data)


@pytest.mark.gpu
def test_maxk_self_gpu(data):
    _check_self(GPUBIN, data)


@pytest.mark.gpu
def test_maxk_edge_queries_gpu(tmp_path):
    _check_edges(GPUBIN, tmp_path)


@pytest.mark.gpu
def test_maxk_windows_and_batches_gpu(data, tmp_path):
    _check_windows(GPUBIN, data, tmp_path)


@pytest.mark.gpu
def test_maxk_rare_bases_gpu(tmp_path):
    _check_rare_bases(GPUBIN, tmp_path)


@pytest.mark.gpu
def test_maxk_list_overflow_gpu(tmp_path):
    _check_overflow(GPUBIN, tmp_path)


@pytest.mark.gpu
def test_maxk_small_superblocks_gpu(data):
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-sb16"), data)


@pytest.mark.gpu
def test_maxk_100mbp_self_gpu(tmp_path):
    """-s of a 100 Mbp reference (random contigs and the repeat-rich stress contigs) against itself; the reference takes ~100 s"""
    import gen_data
    contigs = gen_data.random_contigs(3, 30_000_000, 101) + gen_data.stress_contigs(10_000_000, 102)
    fa = str(tmp_path / "ref100.fa")
    gen_data.write_fasta(fa, contigs)
    del contigs
    r = _run([GPUBIN, "index", fa])
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    r = _same(GPUBIN, ["-s", fa + ".bwt", fa], env={"BWA_B200_PROFILE": "1"})
    assert b"path: windows of" in r.stderr


@pytest.mark.gpu
def test_maxk_3gbp_self_gpu():
    """-s of the benchmark's 3 Gbp reference against itself (made and indexed by bench.make_workload, shared with bench.py): it
    completes and its histogram counts every base; the reference is not run at this size (about an hour on one core)"""
    import bench
    import maxk_bench
    workdir = os.environ.get("BWA_B200_BENCH_DIR", "/tmp/bwa_b200_bench")
    fa, _ = bench.make_workload(workdir, 3000, 1_000_000, 150, 1000, 0, False)
    r = _run([GPUBIN, "maxk", "-s", fa + ".bwt", maxk_bench.self_fasta(workdir, 3000)], env={"BWA_B200_PROFILE": "1"})
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    hist = [int(l.split(b"\t")[1]) for l in r.stdout.split(b"\n") if l]
    assert len(hist) == 256 and sum(hist) == 3_000_000_000
