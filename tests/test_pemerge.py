"""`bwa-b200 pemerge` against the reference's `bwa pemerge` (oracle/_ref/bwa): stdout byte for byte, the nine count lines of stderr
and the exit status, on the emulated kernels (tests/_build/bwa-b200-cusim) and on the GPU.  The pairs come from a seeded generator over
a random reference: inserts from 20 bp to beyond twice the read length, 0-5 % substitutions, indels inside the overlap, short-period
repeats across the overlap, low qualities, N in either read and at the same overlap position in both, lowercase and IUPAC letters,
mates of 36-300 bp and pairs of ~1000 and ~5000 bp.  Each dataset must reach every outcome of the reference (its own counts say so).
Also covered: the options, the input forms (two files, interleaved, gzip, stdin, FASTA, FASTA with FASTQ, odd and unequal counts,
empty reads, read-number suffixes, a quality below '!'), batch sizes, the stub binary, AddressSanitizer and
`pemerge -m | aln | samse` against the reference's three commands."""
import gzip
import os
import re
import subprocess

import numpy as np
import pytest

import bwa_b200
from conftest import CUSIMBIN, REF_BWA, ROOT, TESTBIN, strip_pg

GPUBIN = bwa_b200.CLI_PATH
ASAN_BIN = os.path.join(ROOT, "tests", "_build", "bwa-b200-cusim-asan")
MESSAGES = ("successful merges", "low-scoring pairs", "pairs where the best SW alignment is not an overlap (long left end)",
            "pairs where the best SW alignment is not an overlap (long right end)", "pairs with large 2nd best SW score",
            "pairs with gapped overlap", "pairs where the end-to-end alignment is inconsistent with SW",
            "pairs potentially with tandem overlaps", "pairs with high sum of errors")
COUNT_RE = re.compile(rb"^ *(\d+) (.*)$")


def _run(cmd, env=None, stdin=None):
    e = dict(os.environ, **(env or {}))
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=3600, env=e, input=stdin)


def _counts(stderr):
    """the nine count lines, in order"""
    out = []
    for line in stderr.split(b"\n"):
        m = COUNT_RE.match(line)
        if m and m.group(2).decode() in MESSAGES:
            out.append((MESSAGES.index(m.group(2).decode()), int(m.group(1)), line))
    return out


def _same(binary, args, env=None, stdin=None):
    """stdout, the count lines and the exit status of `binary pemerge args` equal those of `bwa pemerge args`; returns the counts"""
    want = _run([REF_BWA, "pemerge"] + args, stdin=stdin)
    got = _run([binary, "pemerge"] + args, env=env, stdin=stdin)
    assert got.returncode == want.returncode, (args, got.stderr.decode()[-2000:], want.stderr.decode()[-2000:])
    if got.stdout != want.stdout:
        la, lb = want.stdout.split(b"\n"), got.stdout.split(b"\n")
        k = next((i for i in range(min(len(la), len(lb))) if la[i] != lb[i]), min(len(la), len(lb)))
        raise AssertionError("%r: output differs at line %d of %d/%d:\nbwa      %r\nbwa-b200 %r" % (
            args, k, len(la), len(lb), la[k - 1:k + 1] if k < len(la) else None, lb[k - 1:k + 1] if k < len(lb) else None))
    cw, cg = _counts(want.stderr), _counts(got.stderr)
    assert [c[2] for c in cg] == [c[2] for c in cw], (args, got.stderr.decode()[-2000:])
    return [c[1] for c in cw]


# ---------------------------------------------------------------------------------------------------- data

COMP = str.maketrans("ACGTNacgtn", "TGCANtgcan")


def _rc(s):
    return s.translate(COMP)[::-1]


class _Gen:
    def __init__(self, seed, ref_len=300_000):
        self.rng = np.random.default_rng(seed)
        self.ref = self.rand(ref_len)

    def rand(self, n):
        return "".join("ACGT"[i] for i in self.rng.integers(0, 4, n))

    def mutate(self, s, rate):
        s = list(s)
        for k in np.nonzero(self.rng.random(len(s)) < rate)[0]:
            s[k] = "ACGT"[("ACGT".index(s[k]) + int(self.rng.integers(1, 4))) % 4] if s[k] in "ACGT" else s[k]
        return "".join(s)

    def qual(self, n, lo=2, hi=41):
        return "".join(chr(33 + int(x)) for x in self.rng.integers(lo, hi + 1, n))

    def pair(self, l1, l2, ins, kind):
        r = self.rng
        if kind == "repeat":   # a short-period repeat across the overlap
            unit = self.rand(int(r.integers(1, 7)))
            frag = (unit * (ins // len(unit) + 2))[:ins]
            if r.random() < 0.5:   # anchored on one side by unique sequence
                k = int(r.integers(0, ins // 2 + 1))
                frag = self.rand(k) + frag[k:]
        else:
            p = int(r.integers(0, len(self.ref) - ins))
            frag = self.ref[p:p + ins]
        s1 = frag[:l1] if ins >= l1 else frag + self.rand(l1 - ins)
        f2 = _rc(frag)
        s2 = f2[:l2] if ins >= l2 else f2 + self.rand(l2 - ins)
        rate = float(r.choice([0, 0, 0.005, 0.01, 0.02, 0.03, 0.05]))
        s1, s2 = self.mutate(s1, rate), self.mutate(s2, rate)
        if kind == "indel" and len(s2) > 20:   # inside the overlap: read 2's middle
            k = int(r.integers(5, len(s2) - 5))
            s2 = s2[:k] + self.rand(int(r.integers(1, 4))) + s2[k:] if r.random() < 0.5 else s2[:k] + s2[k + int(r.integers(1, 4)):]
        if r.random() < 0.1:   # N in either read
            for _ in range(int(r.integers(1, 4))):
                if r.random() < 0.5:
                    k = int(r.integers(0, len(s1))); s1 = s1[:k] + "N" + s1[k + 1:]
                else:
                    k = int(r.integers(0, len(s2))); s2 = s2[:k] + "N" + s2[k + 1:]
        lo = max(0, ins - l2)
        if r.random() < 0.08 and lo < min(l1, ins):   # N at the same overlap position of both reads
            x = int(r.integers(lo, min(l1, ins)))
            j = ins - 1 - x
            s1 = s1[:x] + "N" + s1[x + 1:]
            if 0 <= j < len(s2):
                s2 = s2[:j] + "N" + s2[j + 1:]
        if r.random() < 0.05:
            s1 = s1.lower() if r.random() < 0.5 else s1[:len(s1) // 2] + s1[len(s1) // 2:].lower()
        if r.random() < 0.05:
            s2 = s2.lower()
        if r.random() < 0.05:   # IUPAC letters
            for _ in range(3):
                s = s1 if r.random() < 0.5 else s2
                k = int(r.integers(0, len(s)))
                s = s[:k] + "RYKMSWBDHV"[int(r.integers(0, 10))] + s[k + 1:]
                if r.random() < 0.5 and s is not s2:
                    s1 = s
                else:
                    s2 = s
        low = r.random() < 0.15
        q1 = self.qual(len(s1), 2, 12 if low else 41)
        q2 = self.qual(len(s2), 2, 12 if low else 41)
        return s1, q1, s2, q2

    def pairs(self, n, long_pairs=True):
        r = self.rng
        out = []
        for i in range(n):
            kind = str(r.choice(["normal"] * 6 + ["indel", "repeat", "repeat"]))
            if r.random() < 0.5:
                l1 = l2 = 150
            else:
                l1, l2 = int(r.integers(36, 301)), int(r.integers(36, 301))
            m = max(l1, l2)
            u = r.random()
            if u < 0.15:
                ins = int(r.integers(20, m + 1))                    # read-through
            elif u < 0.25:
                ins = int(r.integers(l1 + l2, 2 * m + 150))          # no overlap
            else:
                ins = int(r.integers(m, l1 + l2))                    # overlap
            ins = max(ins, 20)
            out.append(self.pair(l1, l2, ins, kind))
        if long_pairs:   # K6's lane kernel: ~1000 and ~5000 bp
            for l, ins in ((1000, 1600), (1000, 1100), (5000, 8000), (4800, 5200)):
                out.append(self.pair(l, l, ins, "normal"))
        names = []
        for i in range(len(out)):
            suf = str(r.choice(["/1", "/1", "/1", "", "/3"]))
            names.append(("pair%d" % i, suf, "/2" if suf == "/1" else suf))
        return [(nm[0] + nm[1], s1, q1, nm[0] + nm[2], s2, q2) for nm, (s1, q1, s2, q2) in zip(names, out)]


def _fq(recs, fasta=False, comment=True):
    out = []
    for k, (name, seq, qual) in enumerate(recs):
        c = " c%d" % k if comment and k % 3 == 0 else ""
        out.append((">%s%s\n%s\n" % (name, c, seq)) if fasta or qual is None else ("@%s%s\n%s\n+\n%s\n" % (name, c, seq, qual)))
    return "".join(out)


def _write(path, text, gz=False):
    if gz:
        with gzip.open(path, "wb") as f:
            f.write(text.encode("latin-1"))
    else:
        with open(path, "wb") as f:
            f.write(text.encode("latin-1"))
    return str(path)


def _files(tmp_path, pairs, tag, **kw):
    r1 = _write(tmp_path / ("%s_1.fq" % tag), _fq([(p[0], p[1], p[2]) for p in pairs], **kw))
    r2 = _write(tmp_path / ("%s_2.fq" % tag), _fq([(p[3], p[4], p[5]) for p in pairs], **kw))
    return r1, r2


def _dataset(tmp_path, seed, n):
    return _files(tmp_path, _Gen(seed).pairs(n), "d%d_%d" % (seed, n))


# ---------------------------------------------------------------------------------------------------- checks

def _check_datasets(binary, tmp_path, n, seeds=(11, 12)):
    for seed in seeds:
        r1, r2 = _dataset(tmp_path, seed, n)
        cnt = _same(binary, [r1, r2])
        assert all(c > 0 for c in cnt[:8]), cnt          # every outcome but -8 at the default -Q
        cnt = _same(binary, ["-Q", "20", r1, r2])
        assert all(c > 0 for c in cnt), cnt              # and -8 with a small -Q


OPTIONS = [["-m"], ["-u"], ["-mu"], ["-T", "0"], ["-T", "1"], ["-T", "30"], ["-T", "200"], ["-Q", "0"], ["-Q", "20"], ["-Q", "1000"],
           ["-t", "0"], ["-t", "4"], ["-t", "300"], ["-T", "-3", "-Q", "-1"], ["-m", "-T", "0", "-Q", "5"], ["-u", "-t", "0"]]


def _check_options(binary, tmp_path, n):
    r1, r2 = _dataset(tmp_path, 13, n)
    for opt in OPTIONS:
        _same(binary, opt + [r1, r2])


def _check_inputs(binary, tmp_path, n):
    pairs = _Gen(14).pairs(n, long_pairs=False)
    r1, r2 = _files(tmp_path, pairs, "in")
    # interleaved, gzip, stdin
    inter = _write(tmp_path / "inter.fq", _fq([x for p in pairs for x in ((p[0], p[1], p[2]), (p[3], p[4], p[5]))]))
    _same(binary, [inter])
    _same(binary, ["-m", inter])
    gz1 = _write(tmp_path / "in_1.fq.gz", open(r1, "rb").read().decode("latin-1"), gz=True)
    gz2 = _write(tmp_path / "in_2.fq.gz", open(r2, "rb").read().decode("latin-1"), gz=True)
    _same(binary, [gz1, gz2])
    _same(binary, ["-", r2], stdin=open(r1, "rb").read())
    _same(binary, ["-"], stdin=open(inter, "rb").read())
    # FASTA, and FASTA with FASTQ
    f1, f2 = _files(tmp_path, pairs, "fa", fasta=True)
    _same(binary, [f1, f2])
    _same(binary, ["-Q", "10", f1, f2])
    _same(binary, [f1, r2])
    _same(binary, [r1, f2])
    # an odd count at the end; unequal files both ways
    odd = _write(tmp_path / "odd.fq", _fq([x for p in pairs[:21] for x in ((p[0], p[1], p[2]), (p[3], p[4], p[5]))][:41]))
    _same(binary, [odd])
    short2 = _write(tmp_path / "short_2.fq", _fq([(p[3], p[4], p[5]) for p in pairs[:n // 2]]))
    short1 = _write(tmp_path / "short_1.fq", _fq([(p[0], p[1], p[2]) for p in pairs[:n // 3]]))
    _same(binary, [r1, short2])
    _same(binary, [short1, r2])
    _same(binary, ["-t", "0", short1, r2])


def _check_edges(binary, tmp_path):
    """empty reads in either mate or both, read-number suffixes, a quality below '!', FASTQ with an empty read"""
    g = _Gen(15)
    base = g.pairs(12, long_pairs=False)
    recs = []
    for k, p in enumerate(base):
        n1, s1, q1, n2, s2, q2 = p
        if k == 1:
            s1, q1 = "", ""        # empty read 1
        elif k == 3:
            s2, q2 = "", ""        # empty read 2
        elif k == 5:
            s1 = q1 = s2 = q2 = ""   # both empty
        elif k == 7:
            q1 = " " + q1[1:]      # a quality character below '!'
            q2 = q2[:-1] + "\x1f"
        recs.append((n1, s1, q1, n2, s2, q2))
    names = [("e/1", "e/2"), ("f/2", "f/1"), ("g/3", "g/3"), ("h", "h"), ("i/1", "i"), ("j/9", "j/8")]
    for k, (a, b) in enumerate(names):
        p = recs[k]
        recs[k] = (a, p[1], p[2], b, p[4], p[5])
    r1, r2 = _files(tmp_path, recs, "edge")
    for opt in ([], ["-m"], ["-u"], ["-T", "0"], ["-T", "0", "-m"], ["-T", "-2", "-Q", "-1"], ["-T", "0", "-Q", "-1"], ["-t", "0"], ["-t", "0", "-m"]):
        _same(binary, opt + [r1, r2])
    f1, f2 = _files(tmp_path, recs, "edgefa", fasta=True)
    for opt in ([], ["-T", "0"], ["-T", "0", "-m"]):
        _same(binary, opt + [f1, f2])
        _same(binary, opt + [f1, r2])


def _check_errors(binary, tmp_path):
    r1, r2 = _files(tmp_path, _Gen(16).pairs(10, long_pairs=False), "err")
    _same(binary, [])                                           # the usage, exit 1
    _same(binary, [str(tmp_path / "missing.fq"), r2])           # file 1 missing: the reference's message and status
    got = _run([binary, "pemerge", r1, str(tmp_path / "missing.fq")])   # file 2 missing: the reference crashes; a message here
    assert got.returncode == 1 and got.stdout == b"" and b"missing.fq" in got.stderr
    got = _run([binary, "pemerge", "-t", "-1", r1, r2])         # negative -t: the reference crashes; refused here
    assert got.returncode == 1 and got.stdout == b""


def _check_batches(binary, tmp_path, n):
    r1, r2 = _dataset(tmp_path, 17, n)
    want = _run([REF_BWA, "pemerge", r1, r2])
    for chunk in ("1", "7", "1000"):
        _same(binary, [r1, r2], env={"BWA_B200_PEMERGE_CHUNK": chunk})
        _same(binary, ["-Q", "20", r1, r2], env={"BWA_B200_PEMERGE_CHUNK": chunk})
    got = _run([binary, "pemerge", r1, r2], env={"BWA_B200_PROFILE": "1"})
    assert got.stdout == want.stdout and b"[prof] pemerge:" in got.stderr


def _pipeline(binary, tmp_path, n):
    """`bwa-b200 pemerge -m | bwa-b200 aln | bwa-b200 samse` equals the reference's three commands"""
    g = _Gen(18, ref_len=200_000)
    fa = str(tmp_path / "pm_ref.fa")
    with open(fa, "w") as f:
        f.write(">chr1\n%s\n" % "\n".join(g.ref[k:k + 70] for k in range(0, len(g.ref), 70)))
    assert _run([REF_BWA, "index", fa]).returncode == 0
    r1, r2 = _files(tmp_path, g.pairs(n, long_pairs=False), "pipe")
    outs = []
    for who in (REF_BWA, binary):
        m = _run([who, "pemerge", "-m", r1, r2])
        assert m.returncode == 0, m.stderr.decode()[-2000:]
        fq = _write(tmp_path / ("merged_%d.fq" % len(outs)), m.stdout.decode("latin-1"))
        sai = str(tmp_path / ("merged_%d.sai" % len(outs)))
        a = _run([who, "aln", "-f", sai, fa, fq])
        assert a.returncode == 0, a.stderr.decode()[-2000:]
        s = _run([who, "samse", fa, sai, fq])
        assert s.returncode == 0, s.stderr.decode()[-2000:]
        outs.append(strip_pg(s.stdout))
    assert outs[0] == outs[1] and outs[0].count(b"\n") > n // 4


# ---------------------------------------------------------------------------------------------------- emulated kernels

def test_pemerge_datasets_emulated(built, tmp_path):
    _check_datasets(CUSIMBIN, tmp_path, 400, seeds=(11,))


def test_pemerge_options_emulated(built, tmp_path):
    _check_options(CUSIMBIN, tmp_path, 150)


def test_pemerge_inputs_emulated(built, tmp_path):
    _check_inputs(CUSIMBIN, tmp_path, 60)


def test_pemerge_edges_emulated(built, tmp_path):
    _check_edges(CUSIMBIN, tmp_path)


def test_pemerge_errors_emulated(built, tmp_path):
    _check_errors(CUSIMBIN, tmp_path)


def test_pemerge_batches_emulated(built, tmp_path):
    _check_batches(CUSIMBIN, tmp_path, 120)


def test_pemerge_pipeline_emulated(built, tmp_path):
    _pipeline(CUSIMBIN, tmp_path, 150)


def test_pemerge_stub_binary(built, tmp_path):
    r1, r2 = _files(tmp_path, _Gen(19).pairs(5, long_pairs=False), "stub")
    r = _run([TESTBIN, "pemerge", r1, r2])   # the host pipeline over the CPU oracle stages: no device pemerge, no records
    assert r.returncode != 0 and r.stdout == b"" and b"no device pemerge" in r.stderr


def test_pemerge_emulated_under_asan(built, tmp_path):
    r = subprocess.run(["make", "asan"], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0 or not os.path.exists(ASAN_BIN):
        pytest.skip("AddressSanitizer build not available: " + r.stdout.decode()[-300:])
    r1, r2 = _files(tmp_path, _Gen(20).pairs(80), "asan")
    env = {"ASAN_OPTIONS": "detect_stack_use_after_return=0:detect_leaks=0"}   # fibers switch stacks by hand
    for opt in ([], ["-Q", "20", "-T", "0"]):
        want = _run([REF_BWA, "pemerge"] + opt + [r1, r2])
        got = _run([ASAN_BIN, "pemerge"] + opt + [r1, r2], env=env)
        assert b"AddressSanitizer" not in got.stderr, got.stderr.decode()[-3000:]
        assert got.returncode == 0 and got.stdout == want.stdout


# ---------------------------------------------------------------------------------------------------- H100

@pytest.mark.gpu
def test_pemerge_datasets_gpu(tmp_path):
    _check_datasets(GPUBIN, tmp_path, 3000, seeds=(11, 12, 21))


@pytest.mark.gpu
def test_pemerge_options_gpu(tmp_path):
    _check_options(GPUBIN, tmp_path, 2000)


@pytest.mark.gpu
def test_pemerge_inputs_gpu(tmp_path):
    _check_inputs(GPUBIN, tmp_path, 500)


@pytest.mark.gpu
def test_pemerge_edges_gpu(tmp_path):
    _check_edges(GPUBIN, tmp_path)
    _check_errors(GPUBIN, tmp_path)


@pytest.mark.gpu
def test_pemerge_batches_gpu(tmp_path):
    _check_batches(GPUBIN, tmp_path, 2000)


@pytest.mark.gpu
def test_pemerge_pipeline_gpu(tmp_path):
    _pipeline(GPUBIN, tmp_path, 3000)


@pytest.mark.gpu
def test_pemerge_300k_pairs_gpu(tmp_path):
    """300 000 pairs of 2 x 150 bp: several device batches and K6 launches"""
    g = _Gen(22)
    rng = g.rng
    recs1, recs2 = [], []
    for i in range(300_000):
        ins = int(np.clip(rng.normal(250, 60), 20, 600))
        p = int(rng.integers(0, len(g.ref) - ins))
        frag = g.ref[p:p + ins]
        s1 = frag[:150] if ins >= 150 else frag + "A" * (150 - ins)
        f2 = _rc(frag)
        s2 = f2[:150] if ins >= 150 else f2 + "A" * (150 - ins)
        if i % 7 == 0:
            s1 = g.mutate(s1, 0.02)
        recs1.append(("r%d/1" % i, s1, g.qual(150)))
        recs2.append(("r%d/2" % i, s2, g.qual(150)))
    r1 = _write(tmp_path / "big_1.fq", _fq(recs1, comment=False))
    r2 = _write(tmp_path / "big_2.fq", _fq(recs2, comment=False))
    _same(GPUBIN, [r1, r2], env={"BWA_B200_PEMERGE_CHUNK": "65536"})
    _same(GPUBIN, ["-t", "8", r1, r2])
