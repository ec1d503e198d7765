"""`bwa-b200 samse` against the reference's `bwa samse` (oracle/_ref/bwa) on the same .sai file, made by the reference's `bwa aln`:
stdout (without @PG) byte for byte and the exit status, on the emulated kernels (tests/_build/bwa-b200-cusim) and on the GPU.  Cases:
reads of 36-150 bp at the default error and at ~3 % error on the c1/two references and on the repeat-rich stress reference, with .sai
files from a matrix of `aln` options (many gapped hits, fractional and integer -n, quality trimming, -I, barcodes, -Y, -R, -N); the
samse options (-n on the repeats: XA lists, gapped XA hits, too many hits; -r; -f); edge reads (a junction between contigs, the start
of a contig on the reverse strand, N runs in the reference for XN and XT:N, an exact 5000-bp read, empty, all-N and FASTA input);
handcrafted .sai files (COMPREAD cleared, bad magic, truncated, trailing records, BAM input); gzip and stdin; batch sizes;
2^16-symbol Occ superblocks; an index kept resident by `bwa-b200 shm`; AddressSanitizer; `bwa-b200 aln` into `bwa-b200 samse`;
the errors; a 100 Mbp reference on the GPU."""
import gzip
import os
import struct
import subprocess

import numpy as np
import pytest

import bwa_b200
from conftest import CUSIMBIN, REF_BWA, ROOT, TESTBIN, strip_pg

GPUBIN = bwa_b200.CLI_PATH
ASAN_BIN = os.path.join(ROOT, "tests", "_build", "bwa-b200-cusim-asan")


def _run(cmd, env=None, stdin=None):
    e = dict(os.environ, **(env or {}))
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=3600, env=e, input=stdin)


def _sai(tmp_path, fa, fq, aln_args=(), who=REF_BWA):
    out = str(tmp_path / ("%08x.sai" % (abs(hash((fa, fq, tuple(aln_args), who))) & 0xffffffff)))
    if not os.path.exists(out):
        r = _run([who, "aln", "-f", out] + list(aln_args) + [fa, fq])
        assert r.returncode == 0, r.stderr.decode()[-2000:]
    return out


def _same(binary, args, env=None, stdin=None, ref_args=None):
    """stdout without @PG and exit status of `binary samse args` equal those of `bwa samse args`; returns the run"""
    want = _run([REF_BWA, "samse"] + (ref_args or args), stdin=stdin)
    got = _run([binary, "samse"] + args, env=env, stdin=stdin)
    assert got.returncode == want.returncode, (args, got.stderr.decode()[-2000:])
    a, b = strip_pg(want.stdout), strip_pg(got.stdout)
    if a != b:
        la, lb = a.split(b"\n"), b.split(b"\n")
        k = next((i for i in range(min(len(la), len(lb))) if la[i] != lb[i]), min(len(la), len(lb)))
        raise AssertionError("%r: SAM differs at line %d of %d/%d:\nbwa      %r\nbwa-b200 %r" % (
            args, k, len(la), len(lb), la[k][:600] if k < len(la) else None, lb[k][:600] if k < len(lb) else None))
    return got


def _datasets(data, n):
    out = []
    for ref, seed in (("c1", 191), ("two", 192)):
        for length in (36, 76, 100, 150):
            out.append(data.reads(ref, tag="se_%d_%d" % (length, n), n=n, length=length, seed=seed + length))
            out.append(data.reads(ref, tag="se_e3_%d_%d" % (length, n), n=n, length=length, seed=seed + 2 * length, err=(0.024, 0.003, 0.003)))
    out.append(data.reads("stress", tag="se_st_%d" % n, n=n, length=100, seed=193, err=(0.016, 0.002, 0.002)))
    return out


def _check_datasets(binary, data, tmp_path, n):
    for fa, fqs in _datasets(data, n):
        for aln_args in ([], ["-o", "2", "-e", "3"]):
            _same(binary, [fa, _sai(tmp_path, fa, fqs[0], aln_args), fqs[0]])


def _quality_reads(data, tmp_path, n):
    """reads with varied qualities (for -q and -I: Phred+64 stays printable after -31) and Casava-style comments (for -Y)"""
    fa, fqs = data.reads("two", tag="se_q_%d" % n, n=n, length=76, seed=194, err=(0.024, 0.003, 0.003))
    rng = np.random.default_rng(195)
    lines = open(fqs[0]).read().split("\n")
    out = str(tmp_path / "q.fq")
    with open(out, "w") as f:
        for k in range(0, len(lines) - 3, 4):
            L = len(lines[k + 1])
            q = "".join(chr(64 + int(x)) for x in np.clip(40 - np.arange(L) * rng.integers(0, 2) * 0.6 + rng.normal(0, 4, L), 2, 41))
            flag = "Y" if rng.random() < 0.3 else "N"
            name = lines[k].split()[0] + ("/1" if k % 8 == 0 else "")
            f.write("%s 1:%s:0:ACGT\n%s\n+\n%s\n" % (name, flag, lines[k + 1], q))
    return fa, out


ALN_OPTIONS = [["-o", "2", "-e", "3"], ["-n", "0.01"], ["-n", "2"], ["-R", "2"], ["-N", "-n", "2"], ["-q", "15"]]
QUAL_OPTIONS = [["-q", "15"], ["-q", "15", "-I"], ["-B", "4"], ["-Y"], ["-I", "-B", "5", "-Y", "-q", "20"]]


def _check_options(binary, data, tmp_path, n):
    fa, fqs = data.reads("stress", tag="se_st_%d" % n, n=n, length=100, seed=193, err=(0.016, 0.002, 0.002))
    for aln_args in ALN_OPTIONS:
        _same(binary, [fa, _sai(tmp_path, fa, fqs[0], aln_args), fqs[0]])
    sai = _sai(tmp_path, fa, fqs[0], ["-o", "2", "-e", "3"])
    for extra in (["-n", "0"], ["-n", "1"], ["-n", "10"], ["-n", "100"], ["-h", "-r", "@RG\\tID:x\\tSM:y"]):
        _same(binary, extra + [fa, sai, fqs[0]])
    fa2, q = _quality_reads(data, tmp_path, n)
    for aln_args in QUAL_OPTIONS:
        _same(binary, [fa2, _sai(tmp_path, fa2, q, aln_args), q])
    out_got, out_want = str(tmp_path / "got.sam"), str(tmp_path / "want.sam")
    r = _same(binary, ["-f", out_got, fa, sai, fqs[0]], ref_args=["-f", out_want, fa, sai, fqs[0]])
    assert r.stdout == b"" and strip_pg(open(out_got, "rb").read()) == strip_pg(open(out_want, "rb").read())


def _revcomp(s):
    return s[::-1].translate(str.maketrans("ACGTacgtN", "TGCAtgcaN"))


def _edge_files(tmp_path):
    """a three-contig reference with a tandem repeat (indexed by `bwa index`) and the edge reads, as FASTQ and as FASTA
    (the fixture of tests/test_aln.py)"""
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


def _pac_bases(fa, beg, end):
    """the forward reference bases [beg, end) as `bwa index` packed them (holes hold random bases there)"""
    raw = np.fromfile(fa + ".pac", dtype=np.uint8)
    k = np.arange(beg, end)
    return "".join("ACGT"[int(c)] for c in (raw[k >> 2] >> ((~k & 3) << 1)) & 3)


def _hole_files(tmp_path):
    """two contigs with N runs of 5 and 20 bases; reads over the holes (XN, and XT:N past 10), at a contig's first base on the
    reverse strand, across the junction, a gapped read near a hole, and an exact 5000-bp read"""
    rng = np.random.default_rng(131)
    rand = lambda n: "".join("ACGT"[i] for i in rng.integers(0, 4, n))
    c1 = rand(3000) + "N" * 5 + rand(3000) + "N" * 20 + rand(4000)
    c2 = rand(9000)
    fa = str(tmp_path / "holes.fa")
    with open(fa, "w") as f:
        f.write(">h1\n%s\n>h2\n%s\n" % (c1, c2))
    subprocess.run([REF_BWA, "index", fa], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    L1 = len(c1)
    full = _pac_bases(fa, 0, L1 + len(c2))
    reads = [("xn5", full[2960:3060]), ("xn5_rc", _revcomp(full[2950:3050])), ("xn20", full[5980:6080]), ("xn20_rc", _revcomp(full[5990:6110])),
             ("xn20_mm", full[5970:6000] + "A" + full[6001:6070]), ("start_rc", _revcomp(full[L1:L1 + 80])), ("start", full[L1:L1 + 80]),
             ("junction", full[L1 - 40:L1 + 40]), ("junction_rc", _revcomp(full[L1 - 30:L1 + 50])),
             ("gapped", full[7000:7040] + full[7043:7100]), ("gapped_ins", full[8000:8050] + "TT" + full[8050:8100]),
             ("long5000", full[L1 + 2000:L1 + 7000]), ("long5000_rc", _revcomp(full[L1 + 3000:L1 + 8000]))]
    fq = str(tmp_path / "holes.fq")
    with open(fq, "w") as f:
        for name, s in reads:
            f.write("@%s\n%s\n+\n%s\n" % (name, s, "".join(chr(35 + (i * 7) % 40) for i in range(len(s)))))
    return fa, fq


def _long_files(tmp_path):
    """reads of 17 000 bases and more, whose CIGAR runs reach 16384 bases: the reference keeps CIGAR entries in 16 bits with a 14-bit
    length, so its runs wrap there (a trimmed read's M, the M before a deletion near the end), on both strands"""
    rng = np.random.default_rng(141)
    ctg = "".join("ACGT"[i] for i in rng.integers(0, 4, 40000))
    fa = str(tmp_path / "long.fa")
    with open(fa, "w") as f:
        f.write(">long\n%s\n" % ctg)
    subprocess.run([REF_BWA, "index", fa], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    trimmed = ctg[1000:18000]
    gapped = ctg[20000:37000] + ctg[37003:37100]   # 17000M3D97M
    reads = [("trim17k", trimmed, "I" * 16900 + "#" * 100), ("trim17k_rc", _revcomp(trimmed), "I" * 16900 + "#" * 100),
             ("gap17k", gapped, "I" * len(gapped)), ("gap17k_rc", _revcomp(gapped), "I" * len(gapped))]
    fq = str(tmp_path / "long.fq")
    with open(fq, "w") as f:
        for name, s, q in reads:
            f.write("@%s\n%s\n+\n%s\n" % (name, s, q))
    return fa, fq


def _check_edges(binary, tmp_path):
    fa, inputs = _edge_files(tmp_path)
    for f in inputs:
        for aln_args in ([], ["-n", "3", "-o", "2", "-e", "2"], ["-l", "32"]):
            _same(binary, [fa, _sai(tmp_path, fa, f, aln_args), f])
    fa, fq = _hole_files(tmp_path)
    for aln_args in ([], ["-n", "25"], ["-n", "25", "-o", "2"]):
        r = _same(binary, [fa, _sai(tmp_path, fa, fq, aln_args), fq])
    assert b"XN:i:5" in r.stdout and b"XT:A:N" in r.stdout
    want = _run([REF_BWA, "samse", fa, _sai(tmp_path, fa, fq, []), fq]).stdout
    fa_l, fq_l = _long_files(tmp_path)
    _same(binary, [fa_l, _sai(tmp_path, fa_l, fq_l, ["-n", "3", "-q", "15"]), fq_l])
    assert any(l.split(b"\t")[1] == b"4" and l.split(b"\t")[2] != b"*" for l in want.split(b"\n") if l and not l.startswith(b"@"))


def _patched_sai(src, dst, fn):
    b = bytearray(open(src, "rb").read())
    fn(b)
    open(dst, "wb").write(bytes(b))
    return dst


def _check_handcrafted(binary, data, tmp_path):
    fa, fqs = data.reads("two", tag="se_hc", n=120, length=76, seed=196, err=(0.024, 0.003, 0.003))
    sai = _sai(tmp_path, fa, fqs[0], ["-o", "2"])
    raw = open(sai, "rb").read()

    def nocomp(b):
        mode = struct.unpack_from("<i", b, 16)[0]
        struct.pack_into("<i", b, 16, mode & ~2)
    _same(binary, [fa, _patched_sai(sai, str(tmp_path / "nocomp.sai"), nocomp), fqs[0]])
    r = _same(binary, [fa, _patched_sai(sai, str(tmp_path / "magic.sai"), lambda b: b.__setitem__(3, 2)), fqs[0]])
    assert r.returncode == 1 and r.stdout == b""
    for cut in (len(raw) - 7, 4 + 64 + 2, 10):
        trunc = str(tmp_path / ("trunc%d.sai" % cut))
        open(trunc, "wb").write(raw[:cut])
        r = _same(binary, [fa, trunc, fqs[0]])
        assert r.returncode == 1
    extra = str(tmp_path / "extra.sai")
    open(extra, "wb").write(raw + struct.pack("<i", 0) * 5 + raw[68:200])
    _same(binary, [fa, extra, fqs[0]])

    def bam(b):
        mode = struct.unpack_from("<i", b, 16)[0]
        struct.pack_into("<i", b, 16, mode | 0x20)
    r = _run([binary, "samse", fa, _patched_sai(sai, str(tmp_path / "bam.sai"), bam), fqs[0]])
    assert r.returncode == 1 and r.stdout == b"" and b"BAM" in r.stderr


def _check_input_forms(binary, data, tmp_path):
    fa, fqs = data.reads("two", tag="se_if", n=150, length=100, seed=197)
    sai = _sai(tmp_path, fa, fqs[0], [])
    raw = open(fqs[0], "rb").read()
    gz = str(tmp_path / "r.fq.gz")
    with gzip.open(gz, "wb") as f:
        f.write(raw)
    _same(binary, [fa, sai, gz])
    _same(binary, [fa, sai, "-"], stdin=raw)


# ---------------------------------------------------------------------------------------------------- emulated kernels (CPU)

def test_samse_datasets_emulated(data, tmp_path):
    _check_datasets(CUSIMBIN, data, tmp_path, 120)


def test_samse_options_emulated(data, tmp_path):
    _check_options(CUSIMBIN, data, tmp_path, 150)


def test_samse_edge_reads_emulated(tmp_path):
    _check_edges(CUSIMBIN, tmp_path)


def test_samse_handcrafted_sai_emulated(data, tmp_path):
    _check_handcrafted(CUSIMBIN, data, tmp_path)


def test_samse_input_forms_emulated(data, tmp_path):
    _check_input_forms(CUSIMBIN, data, tmp_path)


def test_samse_batches_emulated(data, tmp_path):
    """the same bytes whatever the batch size: the hit choice draws its random numbers in read order"""
    fa, fqs = data.reads("stress", tag="se_st_150", n=150, length=100, seed=193, err=(0.016, 0.002, 0.002))
    sai = _sai(tmp_path, fa, fqs[0], ["-o", "2", "-e", "3"])
    outs = set()
    for env in ({"BWA_B200_SAMSE_CHUNK": "1"}, {"BWA_B200_SAMSE_CHUNK": "7"}, {"BWA_B200_SAMSE_CHUNK": "100000", "BWA_B200_PROFILE": "1"}):
        r = _same(CUSIMBIN, ["-n", "10", fa, sai, fqs[0]], env=env)
        outs.add(strip_pg(r.stdout))
        if "BWA_B200_PROFILE" in env:
            line = next(l for l in r.stderr.decode().split("\n") if l.startswith("[prof] samse:"))
            assert int(line.split(" global alignments")[0].split()[-1]) > 0, line
    assert len(outs) == 1


def _sb16(binary, data, tmp_path):
    if not os.path.exists(binary):
        subprocess.run(["make", "-C", ROOT, "sb16" if "cusim" in binary else "sb16-cuda"], check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    fa, fqs = data.reads("c1", tag="se_sb16", n=200, length=76, seed=198, err=(0.024, 0.003, 0.003))
    _same(binary, [fa, _sai(tmp_path, fa, fqs[0], ["-o", "2"]), fqs[0]])


def test_samse_small_superblocks_emulated(data, tmp_path):
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-cusim-sb16"), data, tmp_path)


def _resident(binary, data, tmp_path, n):
    fa, fqs = data.reads("two", tag="se_res%d" % n, n=n, length=100, seed=199)
    sai = _sai(tmp_path, fa, fqs[0], [])
    env = {"BWA_B200_SHM_DIR": str(tmp_path)}
    try:
        r = _run([binary, "shm", fa], env=env)
        assert r.returncode == 0, r.stderr.decode()[-2000:]
        r = _same(binary, [fa, sai, fqs[0]], env=env)
        assert b"using the index resident on the GPU" in r.stderr
        assert b".bwt" not in r.stderr
    finally:
        _run([binary, "shm", "-d"], env=env)
    assert not [f for f in os.listdir(str(tmp_path)) if f.endswith(".resident")]


def test_samse_resident_index_emulated(data, tmp_path):
    _resident(CUSIMBIN, data, tmp_path, 60)


def test_samse_errors(data, tmp_path):
    fa, fqs = data.reads("two", tag="se_if", n=150, length=100, seed=197)
    sai = _sai(tmp_path, fa, fqs[0], [])
    for args in ([], [fa, sai], ["-x", fa, sai] + fqs, [str(tmp_path / "missing"), sai] + fqs, [fa, str(tmp_path / "missing.sai")] + fqs):
        r = _same(CUSIMBIN, args)
        assert r.returncode != 0 and strip_pg(r.stdout) == b""
    r = _same(CUSIMBIN, [fa, sai, str(tmp_path / "missing.fq")])   # the header is out before the reads are opened
    assert r.returncode != 0
    r = _run([TESTBIN, "samse", fa, sai] + fqs)   # the host pipeline over the CPU oracle stages: no device samse, no records
    assert r.returncode != 0 and not [l for l in r.stdout.split(b"\n") if l and not l.startswith(b"@")]
    assert b"no device samse" in r.stderr


def _pipeline(binary, data, tmp_path, n):
    """`bwa-b200 aln | bwa-b200 samse` equals `bwa aln | bwa samse`"""
    fa, fqs = data.reads("two", tag="se_pipe_%d" % n, n=n, length=76, seed=200, err=(0.024, 0.003, 0.003))
    want = subprocess.run("%s aln -o 2 %s %s | %s samse %s - %s" % (REF_BWA, fa, fqs[0], REF_BWA, fa, fqs[0]), shell=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    got = subprocess.run("%s aln -o 2 %s %s | %s samse %s - %s" % (binary, fa, fqs[0], binary, fa, fqs[0]), shell=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert want.returncode == 0 and got.returncode == 0, got.stderr.decode()[-2000:]
    assert strip_pg(got.stdout) == strip_pg(want.stdout) and want.stdout.count(b"\n") > n


def test_samse_pipeline_emulated(data, tmp_path):
    _pipeline(CUSIMBIN, data, tmp_path, 150)


def test_samse_emulated_under_asan(data, tmp_path):
    r = subprocess.run(["make", "asan"], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0 or not os.path.exists(ASAN_BIN):
        pytest.skip("AddressSanitizer build not available: " + r.stdout.decode()[-300:])
    fa, fqs = data.reads("stress", tag="se_st_asan", n=60, length=100, seed=201, err=(0.016, 0.002, 0.002))
    env = {"ASAN_OPTIONS": "detect_stack_use_after_return=0:detect_leaks=0"}   # fibers switch stacks by hand
    r = _same(ASAN_BIN, ["-n", "10", fa, _sai(tmp_path, fa, fqs[0], ["-o", "2", "-e", "3"]), fqs[0]], env=env)
    assert b"AddressSanitizer" not in r.stderr, r.stderr.decode()[-3000:]


# ---------------------------------------------------------------------------------------------------- H100

@pytest.mark.gpu
def test_samse_datasets_gpu(data, tmp_path):
    _check_datasets(GPUBIN, data, tmp_path, 2000)


@pytest.mark.gpu
def test_samse_options_gpu(data, tmp_path):
    _check_options(GPUBIN, data, tmp_path, 1000)


@pytest.mark.gpu
def test_samse_edge_reads_gpu(tmp_path):
    _check_edges(GPUBIN, tmp_path)


@pytest.mark.gpu
def test_samse_handcrafted_sai_gpu(data, tmp_path):
    _check_handcrafted(GPUBIN, data, tmp_path)


@pytest.mark.gpu
def test_samse_batches_gpu(data, tmp_path):
    fa, fqs = data.reads("stress", tag="se_st_1000", n=1000, length=100, seed=193, err=(0.016, 0.002, 0.002))
    sai = _sai(tmp_path, fa, fqs[0], ["-o", "2", "-e", "3"])
    for env in ({"BWA_B200_SAMSE_CHUNK": "33"}, {"BWA_B200_SAMSE_CHUNK": "1000000"}):
        _same(GPUBIN, ["-n", "10", fa, sai, fqs[0]], env=env)


@pytest.mark.gpu
def test_samse_small_superblocks_gpu(data, tmp_path):
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-sb16"), data, tmp_path)


@pytest.mark.gpu
def test_samse_resident_index_gpu(data, tmp_path):
    _resident(GPUBIN, data, tmp_path, 2000)


@pytest.mark.gpu
def test_samse_pipeline_gpu(data, tmp_path):
    _pipeline(GPUBIN, data, tmp_path, 3000)


@pytest.mark.gpu
def test_samse_100mbp_gpu(tmp_path):
    """a 100 Mbp random reference indexed by `bwa-b200 index`; 200 000 reads of 100 bp, their .sai from `bwa-b200 aln`"""
    import gen_data
    contigs = gen_data.random_contigs(4, 25_000_000, 81)
    fa = str(tmp_path / "ref100.fa")
    gen_data.write_fasta(fa, contigs)
    r = _run([GPUBIN, "index", fa])
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    fq = str(tmp_path / "reads.fq")
    reads, _ = gen_data.gen_reads(contigs, 200_000, 100, 102, err=(0.016, 0.002, 0.002))
    gen_data.write_fastq(fq, reads)
    del contigs, reads
    sai = str(tmp_path / "reads.sai")
    r = _run([GPUBIN, "aln", "-f", sai, "-o", "2", fa, fq])
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    _same(GPUBIN, [fa, sai, fq], env={"BWA_B200_PROFILE": "1"})


@pytest.mark.gpu
def test_samse_sai_ends_in_second_group_gpu(data, tmp_path):
    """a .sai that ends inside the second group of 262144 reads: the header and the whole first group are printed, then exit 1"""
    fa, fqs = data.reads("c1", tag="se_2groups", n=270_000, length=36, seed=202)
    sai = str(tmp_path / "two_groups.sai")
    r = _run([GPUBIN, "aln", "-f", sai, fa, fqs[0]])
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    raw = open(sai, "rb").read()
    cut = str(tmp_path / "cut.sai")
    open(cut, "wb").write(raw[:len(raw) - 1000])
    r = _same(GPUBIN, [fa, cut, fqs[0]])
    assert r.returncode == 1 and strip_pg(r.stdout).count(b"\n") > 262144
