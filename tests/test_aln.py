"""`bwa-b200 aln` against the reference's `bwa aln` (oracle/_ref/bwa): stdout (the whole .sai) byte for byte and the exit status, on
the emulated kernels (tests/_build/bwa-b200-cusim) and on the GPU.  Cases: reads of 36-150 bp at the default error and at ~3 % error on
the c1/two references and on the repeat-rich stress reference; edge reads (empty, all N, more N than max_diff, N runs, lowercase, IUPAC,
1 base, around the seed length, across a contig junction and its reverse complement, a tandem repeat with an indel, exact 500-bp and
1000-bp reads with a fractional -n); the option matrix; gzip, stdin and FASTA input; batches of 1 and many reads and tiny first-tier
arenas (BWA_B200_ALN_CHUNK, BWA_B200_TEST_SMALL_POOLS); 2^16-symbol Occ superblocks; an index kept resident by `bwa-b200 shm`; the
errors; `bwa samse`/`bwa sampe` on our .sai files; AddressSanitizer; a 100 Mbp reference on the GPU."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import bwa_b200
from conftest import CUSIMBIN, REF_BWA, ROOT, TESTBIN

GPUBIN = bwa_b200.CLI_PATH
ASAN_BIN = os.path.join(ROOT, "tests", "_build", "bwa-b200-cusim-asan")


def _run(cmd, env=None, stdin=None):
    e = dict(os.environ, **(env or {}))
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=3600, env=e, input=stdin)


def _same(binary, args, env=None, stdin=None, ref_args=None):
    """stdout and exit status of `binary aln args` equal those of `bwa aln args`; returns the run"""
    want = _run([REF_BWA, "aln"] + (ref_args or args), stdin=stdin)
    got = _run([binary, "aln"] + args, env=env, stdin=stdin)
    assert got.returncode == want.returncode, (args, got.stderr.decode()[-2000:])
    if got.stdout != want.stdout:
        a, b = want.stdout, got.stdout
        k = next((i for i in range(min(len(a), len(b))) if a[i] != b[i]), min(len(a), len(b)))
        raise AssertionError("%r: .sai differs at byte %d of %d/%d (bwa / bwa-b200)" % (args, k, len(a), len(b)))
    return got


def _datasets(data, n):
    out = []
    for ref, seed in (("c1", 91), ("two", 92)):
        for length in (36, 50, 76, 100, 150):
            out.append(data.reads(ref, tag="aln_%d_%d" % (length, n), n=n, length=length, seed=seed + length))
            out.append(data.reads(ref, tag="aln_e3_%d_%d" % (length, n), n=n, length=length, seed=seed + 2 * length, err=(0.024, 0.003, 0.003)))
    out.append(data.reads("stress", tag="aln_st_%d" % n, n=n, length=100, seed=93, err=(0.016, 0.002, 0.002)))
    return out


def _revcomp(s):
    return s[::-1].translate(str.maketrans("ACGTacgtN", "TGCAtgcaN"))


def _edge_files(tmp_path):
    """a three-contig reference with a tandem repeat (indexed by `bwa index`) and the edge reads, as FASTQ and as FASTA"""
    rng = np.random.default_rng(97)
    rand = lambda n: "".join("ACGT"[i] for i in rng.integers(0, 4, n))
    unit = rand(7)
    ctg = [rand(6000), rand(2500) + unit * 40 + rand(500), rand(1200)]
    fa = str(tmp_path / "edge.fa")
    with open(fa, "w") as f:
        for i, s in enumerate(ctg):
            f.write(">ctg%d desc %d\n%s\n" % (i + 1, i, "\n".join(s[k:k + 70] for k in range(0, len(s), 70))))
    subprocess.run([REF_BWA, "index", fa], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    a, b = ctg[0], ctg[1]
    junction = a[-50:] + b[:50]
    tandem = b[2460:2500] + unit * 5 + unit[:3] + unit * 5 + b[2780:2800]   # an insertion of 3 bases inside the repeat
    reads = [("empty", ""), ("alln", "N" * 60), ("manyn", a[100:130] + "NNNNNN" + a[136:170]), ("nrun", a[200:240] + "N" * 2 + a[242:300]),
             ("lower", a[300:400].lower()), ("iupac", a[700:720] + "R" + a[721:740] + "Y" + a[741:760]), ("one", "A"), ("oneN", "N"),
             ("seed31", a[1000:1031]), ("seed32", a[1100:1132]), ("seed33", a[1200:1233]), ("junction", junction), ("junction_rc", _revcomp(junction)),
             ("tandem", tandem), ("tandem_rc", _revcomp(tandem)), ("dash", a[2000:2030] + "-" + a[2031:2060]),
             ("mm3", a[3000:3020] + "T" + a[3021:3040] + "G" + a[3041:3080]), ("exact500", a[4000:4500]), ("exact1000", a[4500:5500])]
    fq, fasta = str(tmp_path / "edge.fq"), str(tmp_path / "edge_reads.fa")
    with open(fq, "w") as f:
        for name, s in reads:
            f.write("@%s\n%s\n+\n%s\n" % (name, s, "I" * len(s)))
    with open(fasta, "w") as f:
        for name, s in reads:
            f.write(">%s\n%s\n" % (name, "\n".join(s[k:k + 37] for k in range(0, len(s), 37))))
    return fa, [fq, fasta]


OPTIONS = [["-n", "2"], ["-n", "0.01"], ["-o", "0"], ["-o", "2"], ["-e", "3"], ["-e", "-1"], ["-i", "0"], ["-d", "2"],
           ["-l", "20", "-k", "1"], ["-m", "50"], ["-M", "2", "-O", "9", "-E", "3"], ["-R", "2"], ["-q", "15"], ["-q", "15", "-I"],
           ["-B", "4"], ["-L", "-e", "4"], ["-t", "3"], ["-0", "-1"]]


def _quality_reads(data, tmp_path, n):
    """reads with varied qualities (for -q and -I: Phred+64 stays printable after -31) and Casava-style comments (for -Y)"""
    fa, fqs = data.reads("two", tag="aln_q_%d" % n, n=n, length=76, seed=94, err=(0.024, 0.003, 0.003))
    rng = np.random.default_rng(95)
    lines = open(fqs[0]).read().split("\n")
    out = str(tmp_path / "q.fq")
    with open(out, "w") as f:
        for k in range(0, len(lines) - 3, 4):
            L = len(lines[k + 1])
            q = "".join(chr(64 + int(x)) for x in np.clip(40 - np.arange(L) * rng.integers(0, 2) * 0.6 + rng.normal(0, 4, L), 2, 41))
            flag = "Y" if rng.random() < 0.3 else "N"
            f.write("%s 1:%s:0:ACGT\n%s\n+\n%s\n" % (lines[k].split()[0], flag, lines[k + 1], q))
    return fa, out


def _check_datasets(binary, data, n):
    for fa, fqs in _datasets(data, n):
        _same(binary, [fa] + fqs)


def _check_edges(binary, tmp_path):
    fa, inputs = _edge_files(tmp_path)
    for f in inputs:
        for extra in ([], ["-n", "0.04"], ["-n", "0.001"], ["-n", "3", "-o", "2", "-e", "2"], ["-l", "32"], ["-N", "-n", "2"]):
            _same(binary, extra + [fa, f])


def _check_options(binary, data, tmp_path, n):
    fa, fqs = data.reads("stress", tag="aln_st_%d" % n, n=n, length=100, seed=93, err=(0.016, 0.002, 0.002))
    for extra in OPTIONS:
        _same(binary, extra + [fa] + fqs)
    fa, fqs = data.reads("stress", tag="aln_st_small", n=40, length=50, seed=96, err=(0.016, 0.002, 0.002))
    _same(binary, ["-N"] + [fa] + fqs)
    fa, q = _quality_reads(data, tmp_path, n)
    for extra in (["-Y"], ["-q", "20", "-I"], ["-I", "-B", "5", "-Y"]):
        _same(binary, extra + [fa, q])
    out_got, out_want = str(tmp_path / "got.sai"), str(tmp_path / "want.sai")
    r = _same(binary, ["-f", out_got, fa, q], ref_args=["-f", out_want, fa, q])
    assert r.stdout == b"" and open(out_got, "rb").read() == open(out_want, "rb").read()


# ---------------------------------------------------------------------------------------------------- emulated kernels (CPU)

def test_aln_datasets_emulated(data):
    _check_datasets(CUSIMBIN, data, 150)


def test_aln_edge_reads_emulated(tmp_path):
    _check_edges(CUSIMBIN, tmp_path)


def test_aln_options_emulated(data, tmp_path):
    _check_options(CUSIMBIN, data, tmp_path, 150)


def test_aln_input_forms_emulated(data, tmp_path):
    fa, fqs = data.reads("two", tag="aln_100_150", n=150, length=100, seed=192)
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
    _same(CUSIMBIN, ["-q", "10", fa, fasta])


def test_aln_batches_emulated(data):
    """the same bytes whatever the batch size, and when nearly every read outgrows its first-tier arena and the hit pool"""
    fa, fqs = data.reads("stress", tag="aln_st_150", n=150, length=100, seed=93, err=(0.016, 0.002, 0.002))
    outs = set()
    for env in ({"BWA_B200_ALN_CHUNK": "1"}, {"BWA_B200_ALN_CHUNK": "7"}, {"BWA_B200_ALN_CHUNK": "100000"}, {"BWA_B200_TEST_SMALL_POOLS": "1", "BWA_B200_PROFILE": "1"}):
        r = _same(CUSIMBIN, [fa] + fqs, env=env)
        outs.add(r.stdout)
        if "BWA_B200_TEST_SMALL_POOLS" in env:
            line = next(l for l in r.stderr.decode().split("\n") if l.startswith("[prof] aln:"))
            n_tier2 = int(line.split(" reads in tier 2")[0].split()[-1])
            assert n_tier2 > 100, line
    assert len(outs) == 1


def _sb16(binary, data):
    if not os.path.exists(binary):
        subprocess.run(["make", "-C", ROOT, "sb16" if "cusim" in binary else "sb16-cuda"], check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    fa, fqs = data.reads("c1", tag="aln_sb16", n=200, length=76, seed=98, err=(0.024, 0.003, 0.003))
    for extra in ([], ["-n", "3", "-o", "2"]):
        _same(binary, extra + [fa] + fqs)


def test_aln_small_superblocks_emulated(data):
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-cusim-sb16"), data)


def _resident(binary, data, tmp_path, n):
    fa, fqs = data.reads("two", tag="aln_res%d" % n, n=n, length=100, seed=99)
    env = {"BWA_B200_SHM_DIR": str(tmp_path)}
    try:
        r = _run([binary, "shm", fa], env=env)
        assert r.returncode == 0, r.stderr.decode()[-2000:]
        r = _same(binary, [fa] + fqs, env=env)
        assert b"using the index resident on the GPU" in r.stderr
        assert b".bwt" not in r.stderr                  # the FM-index files were not opened
    finally:
        _run([binary, "shm", "-d"], env=env)
    assert not [f for f in os.listdir(str(tmp_path)) if f.endswith(".resident")]


def test_aln_resident_index_emulated(data, tmp_path):
    _resident(CUSIMBIN, data, tmp_path, 60)


def test_aln_errors(data, tmp_path):
    fa, fqs = data.reads("two", tag="aln_100_150", n=150, length=100, seed=192)
    for args in ([], [fa], ["-x", fa] + fqs, [str(tmp_path / "missing")] + fqs, [fa, str(tmp_path / "missing.fq")]):
        r = _same(CUSIMBIN, args)
        assert r.returncode != 0 and r.stdout == b""
    r = _run([CUSIMBIN, "aln", "-b", fa] + fqs)   # BAM input is refused
    assert r.returncode == 1 and r.stdout == b"" and b"BAM" in r.stderr
    r = _run([TESTBIN, "aln", fa] + fqs)   # the host pipeline over the CPU oracle stages: no device backtracking search
    assert r.returncode != 0 and r.stdout == b""
    assert b"no device backtracking search" in r.stderr


def _pipeline(binary, data, tmp_path):
    """`bwa samse` and `bwa sampe` give the same SAM on our .sai files as on the reference's"""
    fa, fqs = data.reads("two", tag="aln_pe", n=150, length=76, seed=100, paired=True, err=(0.024, 0.003, 0.003))
    sais = {}
    for who, b in (("ref", REF_BWA), ("got", binary)):
        for k, fq in enumerate(fqs):
            out = str(tmp_path / ("%s_%d.sai" % (who, k)))
            r = _run([b, "aln", "-f", out, fa, fq])
            assert r.returncode == 0, r.stderr.decode()[-2000:]
            sais[who, k] = out
    strip = lambda b: b"\n".join(l for l in b.split(b"\n") if not l.startswith(b"@PG"))
    for cmd in (lambda w: ["samse", fa, sais[w, 0], fqs[0]], lambda w: ["sampe", fa, sais[w, 0], sais[w, 1]] + fqs):
        want, got = _run([REF_BWA] + cmd("ref")), _run([REF_BWA] + cmd("got"))
        assert want.returncode == 0 and got.returncode == 0
        assert strip(got.stdout) == strip(want.stdout) and want.stdout.count(b"\n") > 150


def test_aln_samse_sampe_emulated(data, tmp_path):
    _pipeline(CUSIMBIN, data, tmp_path)


def test_aln_emulated_under_asan(data, tmp_path):
    r = subprocess.run(["make", "asan"], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0 or not os.path.exists(ASAN_BIN):
        pytest.skip("AddressSanitizer build not available: " + r.stdout.decode()[-300:])
    fa, fqs = data.reads("stress", tag="aln_st_asan", n=60, length=100, seed=101, err=(0.016, 0.002, 0.002))
    env = {"ASAN_OPTIONS": "detect_stack_use_after_return=0:detect_leaks=0"}   # fibers switch stacks by hand
    for extra_env in ({}, {"BWA_B200_TEST_SMALL_POOLS": "1"}):
        r = _same(ASAN_BIN, ["-n", "3", "-o", "2", fa] + fqs, env=dict(env, **extra_env))
        assert b"AddressSanitizer" not in r.stderr, r.stderr.decode()[-3000:]


# ---------------------------------------------------------------------------------------------------- H100

@pytest.mark.gpu
def test_aln_datasets_gpu(data):
    _check_datasets(GPUBIN, data, 2000)


@pytest.mark.gpu
def test_aln_edge_reads_gpu(tmp_path):
    _check_edges(GPUBIN, tmp_path)


@pytest.mark.gpu
def test_aln_options_gpu(data, tmp_path):
    _check_options(GPUBIN, data, tmp_path, 1000)


@pytest.mark.gpu
def test_aln_batches_gpu(data):
    fa, fqs = data.reads("stress", tag="aln_st_1000", n=1000, length=100, seed=93, err=(0.016, 0.002, 0.002))
    for env in ({"BWA_B200_ALN_CHUNK": "33"}, {"BWA_B200_TEST_SMALL_POOLS": "1"}):
        _same(GPUBIN, [fa] + fqs, env=env)


@pytest.mark.gpu
def test_aln_small_superblocks_gpu(data):
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-sb16"), data)


@pytest.mark.gpu
def test_aln_resident_index_gpu(data, tmp_path):
    _resident(GPUBIN, data, tmp_path, 2000)


@pytest.mark.gpu
def test_aln_samse_sampe_gpu(data, tmp_path):
    _pipeline(GPUBIN, data, tmp_path)


@pytest.mark.gpu
def test_aln_100mbp_gpu(tmp_path):
    """a 100 Mbp random reference indexed by `bwa-b200 index`; 200 000 reads of 100 bp against `bwa aln -t <cpus>`"""
    import gen_data
    contigs = gen_data.random_contigs(4, 25_000_000, 81)
    fa = str(tmp_path / "ref100.fa")
    gen_data.write_fasta(fa, contigs)
    r = _run([GPUBIN, "index", fa])
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    fq = str(tmp_path / "reads.fq")
    reads, _ = gen_data.gen_reads(contigs, 200_000, 100, 102)
    gen_data.write_fastq(fq, reads)
    del contigs, reads
    t = str(os.cpu_count() or 1)
    _same(GPUBIN, ["-t", t, fa, fq], env={"BWA_B200_PROFILE": "1"})
