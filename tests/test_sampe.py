"""`bwa-b200 sampe` against the reference's `bwa sampe` (oracle/_ref/bwa) on the same two .sai files: stdout (without @PG) byte
for byte and the exit status, on the emulated kernels (tests/_build/bwa-b200-cusim) and on the GPU.  Cases: paired reads of 36-150 bp
on the c1/two/stress references at the default error, at ~3 % error and with chimeric pairs (discordant pairs, mate rescue), inserts
of N(400, 50) and N(250, 80); .sai files from a matrix of `aln` options; the sampe options (-a, -o on the repeats, -n/-N, -c, -s,
-A, -r, -f, -P); the insert-size model's failure paths; unmapped reads with a mapped mate, with and without trimming; handcrafted
inputs (COMPREAD cleared, bad magic, truncated and trailing .sai records, BAM bit, mismatched names, unequal read files, an over-long
combined barcode); gzip; batch sizes; `bwa-b200 aln` into `bwa-b200 sampe`."""
import gzip
import os
import struct
import subprocess

import numpy as np
import pytest

import bwa_b200
from conftest import CUSIMBIN, REF_BWA, ROOT, TESTBIN, strip_pg
from test_samse import _hole_files, _pac_bases, _revcomp

GPUBIN = bwa_b200.CLI_PATH
ASAN_BIN = os.path.join(ROOT, "tests", "_build", "bwa-b200-cusim-asan")
TSAN_BIN = os.path.join(ROOT, "tests", "_build", "bwa-b200-tsan")


def _run(cmd, env=None):
    e = dict(os.environ, **(env or {}))
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=3600, env=e)


def _sai(tmp_path, fa, fq, aln_args=(), who=REF_BWA):
    out = str(tmp_path / ("%08x.sai" % (abs(hash((fa, fq, tuple(aln_args), who))) & 0xffffffff)))
    if not os.path.exists(out):
        r = _run([who, "aln", "-f", out] + list(aln_args) + [fa, fq])
        assert r.returncode == 0, r.stderr.decode()[-2000:]
    return out


def _same(binary, args, env=None, want_rc=None):
    """stdout without @PG and exit status of `binary sampe args` equal those of `bwa sampe args`"""
    want = _run([REF_BWA, "sampe"] + args)
    got = _run([binary, "sampe"] + args, env=env)
    assert got.returncode == want.returncode, (args, got.stderr.decode()[-2000:])
    if want_rc is not None:
        assert got.returncode == want_rc
    a, b = strip_pg(want.stdout), strip_pg(got.stdout)
    if a != b:
        la, lb = a.split(b"\n"), b.split(b"\n")
        k = next((i for i in range(min(len(la), len(lb))) if la[i] != lb[i]), min(len(la), len(lb)))
        raise AssertionError("%r: SAM differs at line %d of %d/%d:\nbwa      %r\nbwa-b200 %r" % (
            args, k, len(la), len(lb), la[k][:600] if k < len(la) else None, lb[k][:600] if k < len(lb) else None))
    return got


def _pair_files(data, tmp_path, ref, tag, n, length, seed, err=(0.008, 0.001, 0.001), chimeric=0.0, ins=(400, 50)):
    import gen_data
    fa = data.ref(ref)
    base = str(tmp_path / ("%s_%s" % (ref, tag)))
    outs = [base + "_1.fq", base + "_2.fq"]
    if not os.path.exists(outs[1]):
        contigs = gen_data.read_fasta(fa)
        r1, r2 = gen_data.gen_reads(contigs, n, length, seed, err=err, paired=True, ins_mean=ins[0], ins_sd=ins[1], chimeric=chimeric)
        gen_data.write_fastq(outs[0], r1)
        gen_data.write_fastq(outs[1], r2)
    return fa, outs


def _pe(binary, tmp_path, fa, fqs, aln_args=((), ()), sampe_args=(), env=None, who=REF_BWA):
    s1 = _sai(tmp_path, fa, fqs[0], aln_args[0], who)
    s2 = _sai(tmp_path, fa, fqs[1], aln_args[1], who)
    return _same(binary, list(sampe_args) + [fa, s1, s2, fqs[0], fqs[1]], env=env)


def _datasets(data, tmp_path, n):
    out = []
    for ref, seed in (("c1", 291), ("two", 292)):
        for length in (36, 76, 100, 150):
            out.append(_pair_files(data, tmp_path, ref, "pe_%d" % length, n, length, seed + length))
            out.append(_pair_files(data, tmp_path, ref, "pe_e3_%d" % length, n, length, seed + 2 * length, err=(0.024, 0.003, 0.003), chimeric=0.1))
    out.append(_pair_files(data, tmp_path, "two", "pe_ins250", n, 100, 293, ins=(250, 80), chimeric=0.05))
    out.append(_pair_files(data, tmp_path, "stress", "pe_st", n, 100, 294, err=(0.016, 0.002, 0.002), chimeric=0.05))
    return out


def _check_datasets(binary, data, tmp_path, n):
    for fa, fqs in _datasets(data, tmp_path, n):
        for aln_args in ([], ["-o", "2", "-e", "3"]):
            _pe(binary, tmp_path, fa, fqs, (aln_args, aln_args))


def _check_options(binary, data, tmp_path, n):
    fa, fqs = _pair_files(data, tmp_path, "two", "pe_opt", n, 100, 295, err=(0.02, 0.003, 0.003), chimeric=0.1)
    for args in (["-a", "200"], ["-a", "1000"], ["-n", "0", "-N", "0"], ["-n", "10", "-N", "20"], ["-c", "1e-3"], ["-s"], ["-A"], ["-P"],
                 ["-r", "@RG\\tID:x\\tSM:y"]):
        _pe(binary, tmp_path, fa, fqs, sampe_args=args)
    for aln in ((["-n", "0.01"], ["-n", "0.01"]), (["-n", "2"], ["-n", "2"]), (["-Y"], ["-Y"]), (["-R", "2"], ["-R", "2"])):
        _pe(binary, tmp_path, fa, fqs, aln)
    st, sfq = _pair_files(data, tmp_path, "stress", "pe_st_o", n, 76, 296, err=(0.016, 0.002, 0.002))
    for args in (["-o", "10"], ["-n", "10", "-N", "20"]):
        _pe(binary, tmp_path, st, sfq, sampe_args=args)


def _check_edges(binary, data, tmp_path):
    # fewer than 20 pairs: "too few good pairs", the -a path and no rescue
    fa, fqs = _pair_files(data, tmp_path, "two", "pe_few", 12, 100, 297, chimeric=0.3)
    _pe(binary, tmp_path, fa, fqs)
    # batch sizes change no byte
    fa, fqs = _pair_files(data, tmp_path, "two", "pe_chunk", 300, 76, 299, err=(0.024, 0.003, 0.003), chimeric=0.1)
    for chunk in ("1", "7", "1000"):
        _pe(binary, tmp_path, fa, fqs, env={"BWA_B200_SAMPE_CHUNK": chunk})
    # -f
    out = str(tmp_path / "pe_f.sam")
    s1, s2 = _sai(tmp_path, fa, fqs[0]), _sai(tmp_path, fa, fqs[1])
    r = _run([binary, "sampe", "-f", out, fa, s1, s2, fqs[0], fqs[1]])
    assert r.returncode == 0 and r.stdout == b""
    want = _run([REF_BWA, "sampe", fa, s1, s2, fqs[0], fqs[1]])
    assert strip_pg(open(out, "rb").read()) == strip_pg(want.stdout)
    # gzip input
    gz = [str(tmp_path / ("pe_gz_%d.fq.gz" % k)) for k in (1, 2)]
    for src, dst in zip(fqs, gz):
        with open(src, "rb") as f, gzip.open(dst, "wb") as g:
            g.write(f.read())
    _same(binary, [fa, s1, s2, gz[0], gz[1]])
    return fa, fqs, s1, s2


def _check_handcrafted(binary, data, tmp_path):
    fa, fqs = _pair_files(data, tmp_path, "two", "pe_hand", 60, 76, 300, chimeric=0.2)
    s1, s2 = _sai(tmp_path, fa, fqs[0]), _sai(tmp_path, fa, fqs[1])
    b1, b2 = open(s1, "rb").read(), open(s2, "rb").read()

    def put(name, blob):
        p = str(tmp_path / name)
        with open(p, "wb") as f:
            f.write(blob)
        return p
    nocomp = lambda b: b[:4] + b[4:16] + struct.pack("<i", struct.unpack("<i", b[16:20])[0] & ~2) + b[20:]
    _same(binary, [fa, put("nc1.sai", nocomp(b1)), put("nc2.sai", nocomp(b2)), fqs[0], fqs[1]])
    _same(binary, [fa, put("bad1.sai", b"SAI\2" + b1[4:]), s2, fqs[0], fqs[1]], want_rc=1)
    _same(binary, [fa, s1, put("bad2.sai", b"SAI\2" + b2[4:]), fqs[0], fqs[1]], want_rc=1)
    _same(binary, [fa, put("tr1.sai", b1[:len(b1) - 40]), s2, fqs[0], fqs[1]], want_rc=1)
    _same(binary, [fa, s1, put("tr2.sai", b2[:len(b2) - 40]), fqs[0], fqs[1]], want_rc=1)
    _same(binary, [fa, put("tail1.sai", b1 + b"\0" * 64), s2, fqs[0], fqs[1]])
    bam = lambda b: b[:16] + struct.pack("<i", struct.unpack("<i", b[16:20])[0] | 0x20) + b[20:]
    r = _run([binary, "sampe", fa, s1, put("bam2.sai", bam(b2)), fqs[0], fqs[1]])
    assert r.returncode == 1 and r.stdout == b"" and b"BAM" in r.stderr
    # only one file with COMPREAD cleared: each end's rseq follows its own .sai
    _same(binary, [fa, put("nc1only.sai", nocomp(b1)), s2, fqs[0], fqs[1]])
    _same(binary, [fa, s1, put("nc2only.sai", nocomp(b2)), fqs[0], fqs[1]])
    # a negative hit count in either file: the earlier groups out, then [fread] and exit 1
    neg = lambda b: b[:68] + struct.pack("<i", -1) + b[72:]
    _same(binary, [fa, put("neg1.sai", neg(b1)), s2, fqs[0], fqs[1]], want_rc=1)
    _same(binary, [fa, s1, put("neg2.sai", neg(b2)), fqs[0], fqs[1]], want_rc=1)
    # mismatched names: the pair is printed, then the command fails
    lines = open(fqs[1]).read().split("\n")
    lines[4 * 30] = lines[4 * 30].split()[0] + "x"
    mm = put("mm_2.fq", "\n".join(lines).encode())
    _same(binary, [fa, s1, s2, fqs[0], mm], want_rc=1)
    # a shorter second file: the pairs up to its end
    short2 = put("short_2.fq", ("\n".join(open(fqs[1]).read().split("\n")[:4 * 40]) + "\n").encode())
    _same(binary, [fa, s1, s2, fqs[0], short2], want_rc=0)
    # a shorter first file: an error before the group is printed
    short1 = put("short_1.fq", ("\n".join(open(fqs[0]).read().split("\n")[:4 * 40]) + "\n").encode())
    r = _run([binary, "sampe", fa, s1, s2, short1, fqs[1]])
    assert r.returncode != 0 and b"fewer reads" in r.stderr


def _check_own_aln(binary, data, tmp_path):
    fa, fqs = _pair_files(data, tmp_path, "two", "pe_own", 200, 100, 301, err=(0.02, 0.003, 0.003), chimeric=0.1)
    _pe(binary, tmp_path, fa, fqs, who=binary)


def _write_pairs(path_base, pairs, qual=None):
    """pairs: (name, seq1, seq2[, qual1, qual2]); returns the two FASTQ paths"""
    outs = [path_base + "_1.fq", path_base + "_2.fq"]
    with open(outs[0], "w") as f1, open(outs[1], "w") as f2:
        for p in pairs:
            name, a, b = p[:3]
            qa, qb = (p[3], p[4]) if len(p) > 3 else ((qual or "I") * len(a), (qual or "I") * len(b))
            f1.write("@%s\n%s\n+\n%s\n" % (name, a, qa))
            f2.write("@%s\n%s\n+\n%s\n" % (name, b, qb))
    return outs


def _contig(data, ref):
    return _pac_bases(data.ref(ref), 0, 400000)


def _frag_pair(ctg, rng, length, ins):
    p = int(rng.integers(1000, len(ctg) - ins - 1000))
    frag = ctg[p:p + ins]
    return frag[:length], _revcomp(frag)[:length]


def _check_crafted(binary, data, tmp_path):
    rng = np.random.default_rng(311)
    rand = lambda n: "".join("ACGT"[i] for i in rng.integers(0, 4, n))
    fa = data.ref("c1")
    ctg = _contig(data, "c1")
    # inserts shorter than the longest read: "upper bound is smaller than read length" (60-bp pairs with 60-64-bp inserts, and two
    # unmappable 150-bp pairs that set max_len)
    pairs = [("s%d" % i,) + _frag_pair(ctg, rng, 60, 60 + i % 5) for i in range(80)] + [("long%d" % i, rand(150), rand(150)) for i in range(2)]
    fqs = _write_pairs(str(tmp_path / "ub"), pairs)
    r = _pe(binary, tmp_path, fa, fqs)
    assert b"upper bound is smaller than read length" in r.stderr
    # quality trimming: low-quality tails; unmapped mates (random bases) with mapped partners, trimmed and untrimmed; -q differs per end
    pairs = []
    for i in range(120):
        a, b = _frag_pair(ctg, rng, 100, int(rng.normal(400, 50)))
        if i % 4 == 0:
            b = rand(100)
        qa = "I" * (100 - 15 * (i % 3)) + "#" * (15 * (i % 3))
        qb = "I" * (100 - 20 * (i % 2)) + "#" * (20 * (i % 2))
        pairs.append(("q%d" % i, a, b, qa, qb))
    fqs = _write_pairs(str(tmp_path / "trim"), pairs)
    r = _pe(binary, tmp_path, fa, fqs, (["-q", "15"], ["-q", "25"]))
    assert b"XC:i:" in r.stdout
    # the same in Phred+64 (-I)
    fqs64 = _write_pairs(str(tmp_path / "trim64"), [(p[0], p[1], p[2], "".join(chr(ord(c) + 31) for c in p[3]), "".join(chr(ord(c) + 31) for c in p[4])) for p in pairs])
    _pe(binary, tmp_path, fa, fqs64, (["-I", "-q", "15"], ["-I", "-q", "15"]))
    # barcodes (-B 4 on both ends): both reads carry the pair's concatenated barcode
    pairs = [("b%d" % i, rand(4) + a, rand(4) + b) for i, (a, b) in enumerate(_frag_pair(ctg, rng, 76, int(rng.normal(400, 50))) for _ in range(60))]
    fqs = _write_pairs(str(tmp_path / "bc"), pairs)
    r = _pe(binary, tmp_path, fa, fqs, (["-B", "4"], ["-B", "4"]))
    assert b"BC:Z:" in r.stdout
    # a combined barcode over 63 bases is refused, naming the pair
    pairs = [("l%d" % i, rand(40) + a, rand(40) + b) for i, (a, b) in enumerate(_frag_pair(ctg, rng, 76, 400) for _ in range(5))]
    fqs = _write_pairs(str(tmp_path / "bclong"), pairs)
    r = _run([binary, "sampe", fa, _sai(tmp_path, fa, fqs[0], ["-B", "40"]), _sai(tmp_path, fa, fqs[1], ["-B", "40"]), fqs[0], fqs[1]])
    assert r.returncode == 1 and b"l0" in r.stderr and b"barcodes" in r.stderr
    # reads of 1000 bp, half of end 1 chimeric: mate rescue of long reads runs K6's 16-bit path
    import gen_data
    r1, r2 = gen_data.gen_reads(gen_data.read_fasta(fa), 24, 1000, 312, paired=True, ins_mean=2500, ins_sd=100, chimeric=0.5)
    base = str(tmp_path / "kb")
    gen_data.write_fastq(base + "_1.fq", r1)
    gen_data.write_fastq(base + "_2.fq", r2)
    _pe(binary, tmp_path, fa, [base + "_1.fq", base + "_2.fq"])
    # the N-run reference of the samse tests: pairs over the holes (XN, XT:N), across the junction, at the second contig's start on the
    # reverse strand, plus ordinary pairs for the model
    hfa, _ = _hole_files(tmp_path)
    L1 = 3000 + 5 + 3000 + 20 + 4000
    full = _pac_bases(hfa, 0, L1 + 9000)
    pairs = [("xn5", full[2960:3060], _revcomp(full[3300:3400])), ("xn20", full[5700:5800], _revcomp(full[5990:6090])),
             ("junction", full[L1 - 60:L1 + 40], _revcomp(full[L1 + 250:L1 + 350])), ("start_rc", _revcomp(full[L1:L1 + 80]), full[L1 + 300:L1 + 380]),
             ("start_fr", full[L1:L1 + 80], _revcomp(full[L1 + 300:L1 + 380]))]
    for i in range(40):
        p = int(rng.integers(L1 + 500, L1 + 8400))
        pairs.append(("h%d" % i, full[p:p + 80], _revcomp(full[p + 320:p + 400])))
    fqs = _write_pairs(str(tmp_path / "holes_pe"), pairs)
    for aln in ([], ["-n", "25"]):
        r = _pe(binary, tmp_path, hfa, fqs, (aln, aln))
    assert b"XN:i:" in r.stdout


def _resident(binary, data, tmp_path):
    fa, fqs = _pair_files(data, tmp_path, "two", "pe_res", 100, 100, 313, chimeric=0.1)
    env = {"BWA_B200_SHM_DIR": str(tmp_path)}
    try:
        r = _run([binary, "shm", fa], env=env)
        assert r.returncode == 0, r.stderr.decode()[-2000:]
        r = _pe(binary, tmp_path, fa, fqs, env=env)
        assert b"using the index resident on the GPU" in r.stderr
    finally:
        _run([binary, "shm", "-d"], env=env)


def _sb16(binary, data, tmp_path):
    if not os.path.exists(binary):
        subprocess.run(["make", "-C", ROOT, "sb16" if "cusim" in binary else "sb16-cuda"], check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    fa, fqs = _pair_files(data, tmp_path, "c1", "pe_sb16", 150, 76, 314, err=(0.024, 0.003, 0.003), chimeric=0.1)
    _pe(binary, tmp_path, fa, fqs)


def test_sampe_crafted_emulated(built, data, tmp_path):
    _check_crafted(CUSIMBIN, data, tmp_path)


def test_sampe_resident_and_sb16_emulated(built, data, tmp_path):
    _resident(CUSIMBIN, data, tmp_path)
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-cusim-sb16"), data, tmp_path)


def test_sampe_sanitizers(built, data, tmp_path):
    """AddressSanitizer over the emulated kernels and the host; ThreadSanitizer over the host pipeline (its device half is the stub)"""
    for target, path in (("asan", ASAN_BIN), ("tsan", TSAN_BIN)):
        r = subprocess.run(["make", "-C", ROOT, target], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        assert r.returncode == 0 and os.path.exists(path), r.stderr.decode()[-2000:]
    fa, fqs = _pair_files(data, tmp_path, "two", "pe_san", 120, 100, 315, err=(0.02, 0.003, 0.003), chimeric=0.15)
    env = {"ASAN_OPTIONS": "detect_stack_use_after_return=0:detect_leaks=0"}   # fibers switch stacks by hand
    r = _pe(ASAN_BIN, tmp_path, fa, fqs, env=dict(env, BWA_B200_SAMPE_CHUNK="7"))
    assert b"AddressSanitizer" not in r.stderr
    s1, s2 = _sai(tmp_path, fa, fqs[0]), _sai(tmp_path, fa, fqs[1])
    r = _run([TSAN_BIN, "sampe", fa, s1, s2, fqs[0], fqs[1]], env={"BWA_B200_SAMPE_CHUNK": "7"})
    assert r.returncode == 1 and b"no device sampe" in r.stderr and b"ThreadSanitizer" not in r.stderr, r.stderr.decode()[-3000:]


def test_sampe_emulator(built, data, tmp_path):
    _check_datasets(CUSIMBIN, data, tmp_path, 150)
    _check_options(CUSIMBIN, data, tmp_path, 150)
    _check_edges(CUSIMBIN, data, tmp_path)
    _check_handcrafted(CUSIMBIN, data, tmp_path)
    _check_own_aln(CUSIMBIN, data, tmp_path)


def test_sampe_testbin_has_no_device(built, data, tmp_path):
    fa, fqs = _pair_files(data, tmp_path, "two", "pe_tb", 20, 76, 302)
    s1, s2 = _sai(tmp_path, fa, fqs[0]), _sai(tmp_path, fa, fqs[1])
    r = _run([TESTBIN, "sampe", fa, s1, s2, fqs[0], fqs[1]])
    assert r.returncode == 1 and b"no device sampe" in r.stderr


@pytest.mark.gpu
def test_sampe_gpu(built, data, tmp_path):
    _check_datasets(GPUBIN, data, tmp_path, 2000)
    _check_options(GPUBIN, data, tmp_path, 2000)
    _check_edges(GPUBIN, data, tmp_path)
    _check_handcrafted(GPUBIN, data, tmp_path)
    _check_own_aln(GPUBIN, data, tmp_path)
    _check_crafted(GPUBIN, data, tmp_path)
    _resident(GPUBIN, data, tmp_path)
    _sb16(os.path.join(ROOT, "tests", "_build", "bwa-b200-sb16"), data, tmp_path)


@pytest.mark.gpu
def test_sampe_gpu_two_groups(built, data, tmp_path):
    """262144 + 10 pairs: the second group is too small for the model and takes the first group's (last_ii)"""
    fa, fqs = _pair_files(data, tmp_path, "c1", "pe_big", 262144 + 10, 76, 303)
    _pe(GPUBIN, tmp_path, fa, fqs)
    s1, s2 = _sai(tmp_path, fa, fqs[0]), _sai(tmp_path, fa, fqs[1])
    b2 = open(s2, "rb").read()
    cut = str(tmp_path / "cut2.sai")
    with open(cut, "wb") as f:
        f.write(b2[:len(b2) - 200])
    _same(GPUBIN, [fa, s1, cut, fqs[0], fqs[1]], want_rc=1)
