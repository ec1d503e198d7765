"""The steps of `bwa index` as commands (`fa2pac`, `pac2bwt`, `pac2bwtgen`, `bwtupdate`, `bwt2sa`) against the reference's own
commands, byte for byte, on the emulated kernels (tests/_build/bwa-b200-cusim) and on the GPU; their refusals (exit 1, no
output); and the chain fa2pac -> pac2bwt -> bwtupdate -> fa2pac -f -> bwt2sa against `bwa index`, `bwa-b200 index` and `mem`.
BWA_B200_BWT2SA_STRIDE forces the distance between the rulers of bwt2sa: 1 (every row a ruler), a middle value, and one
larger than the text (a single lane walks the whole cycle)."""
import gzip
import os
import shutil
import subprocess
import time

import numpy as np
import pytest

from conftest import CUSIMBIN, REF_BWA, ROOT, run_sam
from test_index_cli import SMALL, _fasta

GPUBIN = os.path.join(ROOT, "bwa_b200", "bwa-b200")
EXTS = ("pac", "ann", "amb", "bwt", "sa")
BINS = [pytest.param(CUSIMBIN, id="emulated"), pytest.param(GPUBIN, id="gpu", marks=pytest.mark.gpu)]
SA_CASES = ["holes", "len1001", "len63", "repeat20k"]


def _run(args, cwd=None, env=None, check=True):
    r = subprocess.run(args, cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1800)
    if check:
        assert r.returncode == 0, (args, r.stderr.decode()[-2000:])
    return r


def _env(stride=None):
    env = dict(os.environ)
    env.pop("BWA_B200_BWT2SA_STRIDE", None)
    if stride:
        env["BWA_B200_BWT2SA_STRIDE"] = str(stride)
    return env


def _same(a, b):
    assert open(a, "rb").read() == open(b, "rb").read(), (a, b)


def _dirs(tmp_path, name, gz=False):
    """Two directories with the case's FASTA: ref/ for the reference's commands, mine/ for ours."""
    text = _fasta(name)
    fn = name + (".fa.gz" if gz else ".fa")
    out = []
    for d in ("ref", "mine"):
        p = tmp_path / d
        p.mkdir(exist_ok=True)
        if gz:
            with gzip.open(str(p / fn), "wt") as f:
                f.write(text)
        else:
            (p / fn).write_text(text)
        out.append(str(p))
    return out[0], out[1], fn


def _both(binary, ref, mine, args, env=None):
    _run([REF_BWA] + args, cwd=ref)
    _run([binary] + args, cwd=mine, env=env)


def _seq_len(bwt):
    return int(np.frombuffer(open(bwt, "rb").read(40), dtype="<u8")[4])


# ---------------------------------------------------------------------------------------------- fa2pac (host only)

@pytest.mark.parametrize("name", SMALL + ["repeat20k"])
def test_fa2pac(tmp_path, name):
    ref, mine, fn = _dirs(tmp_path, name)
    for opts, prefix in (([], None), (["-f"], None), ([], "dbl"), (["-f"], "fwd")):
        _both(CUSIMBIN, ref, mine, ["fa2pac"] + opts + [fn] + ([prefix] if prefix else []))
        for ext in ("pac", "ann", "amb"):
            f = (prefix or fn) + "." + ext
            _same(os.path.join(ref, f), os.path.join(mine, f))


def test_fa2pac_gzip(tmp_path):
    ref, mine, fn = _dirs(tmp_path, "holes", gz=True)
    for opts in ([], ["-f"]):
        _both(CUSIMBIN, ref, mine, ["fa2pac"] + opts + [fn, "p" + "".join(opts)])
        for ext in ("pac", "ann", "amb"):
            _same(os.path.join(ref, "p%s.%s" % ("".join(opts), ext)), os.path.join(mine, "p%s.%s" % ("".join(opts), ext)))


def test_usage(tmp_path):
    for cmd in ("fa2pac", "pac2bwt", "pac2bwtgen", "bwtupdate", "bwt2sa"):
        r = _run([CUSIMBIN, cmd], check=False)
        assert r.returncode == 1 and b"Usage: bwa-b200 " + cmd.encode() in r.stderr, (cmd, r.stderr)
    r = _run([CUSIMBIN], check=False)
    for cmd in (b"fa2pac", b"pac2bwt", b"pac2bwtgen", b"bwtupdate", b"bwt2sa"):
        assert b"bwa-b200 " + cmd + b" " in r.stderr


def test_oracle_build_has_no_device_steps(tmp_path):
    """The test binary over the CPU oracle stages (no kernels) says so and writes nothing."""
    from conftest import TESTBIN
    ref, mine, fn = _dirs(tmp_path, "len1001")
    _run([CUSIMBIN, "fa2pac", fn], cwd=mine)
    r = _run([TESTBIN, "pac2bwt", fn + ".pac", "x.bwt"], cwd=mine, check=False)
    assert r.returncode == 1 and b"no device" in r.stderr and not os.path.exists(os.path.join(mine, "x.bwt"))


# ---------------------------------------------------------------------------------------------- pac2bwt, bwtupdate, bwt2sa

def _steps(binary, tmp_path, name, intvs=(1, 2, 32, 64), strides=(1, 16, 1 << 20)):
    """pac2bwt (-d) / pac2bwtgen on the doubled and the forward-only .pac, bwtupdate, a second bwtupdate, and bwt2sa at each
    interval under each ruler stride: every file the reference's."""
    ref, mine, fn = _dirs(tmp_path, name)
    for kind, opts in (("dbl", []), ("fwd", ["-f"])):
        _both(binary, ref, mine, ["fa2pac"] + opts + [fn, kind])
        _both(binary, ref, mine, ["pac2bwt", kind + ".pac", kind + ".bwt"])
        _same(os.path.join(ref, kind + ".bwt"), os.path.join(mine, kind + ".bwt"))
        for cmd in (["pac2bwt", "-d"], ["pac2bwtgen"]):
            _run([binary] + cmd + [kind + ".pac", kind + ".2.bwt"], cwd=mine)
            _same(os.path.join(ref, kind + ".bwt"), os.path.join(mine, kind + ".2.bwt"))
        raw = open(os.path.join(mine, kind + ".bwt"), "rb").read()
        _run([REF_BWA, "bwtupdate", kind + ".bwt"], cwd=ref)
        r = _run([binary, "bwt2sa", kind + ".bwt", "x.sa"], cwd=mine, check=False)   # a raw .bwt: refused
        assert r.returncode == 1 and b"bwtupdate" in r.stderr and not os.path.exists(os.path.join(mine, "x.sa")), r.stderr
        _run([binary, "bwtupdate", kind + ".bwt"], cwd=mine)
        _same(os.path.join(ref, kind + ".bwt"), os.path.join(mine, kind + ".bwt"))
        upd = open(os.path.join(mine, kind + ".bwt"), "rb").read()
        assert upd != raw
        r = _run([binary, "bwtupdate", kind + ".bwt"], cwd=mine, check=False)   # already updated: refused, file unchanged
        assert r.returncode != 0 and b"already" in r.stderr
        assert open(os.path.join(mine, kind + ".bwt"), "rb").read() == upd
        n = _seq_len(os.path.join(mine, kind + ".bwt"))
        for intv in list(intvs) + [1 << (n.bit_length() + 1)]:
            sa = "%s.i%d.sa" % (kind, intv)
            _run([REF_BWA, "bwt2sa", "-i", str(intv), kind + ".bwt", sa], cwd=ref)
            for stride in strides:
                _run([binary, "bwt2sa", "-i", str(intv), kind + ".bwt", sa], cwd=mine, env=_env(stride))
                _same(os.path.join(ref, sa), os.path.join(mine, sa))
        assert not [f for f in os.listdir(mine) if ".tmp" in f]


@pytest.mark.parametrize("binary", BINS)
@pytest.mark.parametrize("name", SA_CASES)
def test_steps(binary, tmp_path, name):
    _steps(binary, tmp_path, name)


@pytest.mark.parametrize("binary", BINS)
@pytest.mark.parametrize("name", [n for n in SMALL if n not in SA_CASES])
def test_steps_small(binary, tmp_path, name):
    _steps(binary, tmp_path, name, intvs=(32,), strides=(None,))


# ---------------------------------------------------------------------------------------------- refusals

def _lf_one_cycle(raw_bwt):
    """Whether the LF mapping of a raw .bwt (primary, L2, words) is one cycle of n + 1 rows (bwt.c:53-59)."""
    hdr = np.frombuffer(raw_bwt[:40], dtype="<u8")
    primary, n = int(hdr[0]), int(hdr[4])
    words = np.frombuffer(raw_bwt[40:], dtype="<u4")
    sym = ((words[:, None] >> (2 * (15 - np.arange(16, dtype=np.uint32)))) & 3).reshape(-1)[:n].astype(np.int64)
    L2 = np.concatenate([[0], hdr[1:5].astype(np.int64)])
    occ = np.zeros((4, n), dtype=np.int64)
    for c in range(4):
        occ[c] = np.cumsum(sym == c)
    lf = np.zeros(n + 1, dtype=np.int64)
    for k in range(n + 1):
        if k != primary:
            kp = k - (k > primary)
            lf[k] = L2[sym[kp]] + occ[sym[kp], kp]
    k, steps = 0, 0
    while True:
        k = lf[k]
        steps += 1
        if k == 0:
            return steps == n + 1


def _swap(raw_bwt, i, j):
    b = bytearray(raw_bwt)
    words = np.frombuffer(bytes(b[40:]), dtype="<u4").copy()
    get = lambda p: int(words[p >> 4] >> (2 * (15 - (p & 15))) & 3)

    def put(p, c):
        sh = 2 * (15 - (p & 15))
        words[p >> 4] = (int(words[p >> 4]) & ~(3 << sh) & 0xffffffff) | (c << sh)
    a, c = get(i), get(j)
    put(i, c)
    put(j, a)
    return bytes(b[:40]) + words.tobytes(), a != c


@pytest.mark.parametrize("binary", BINS)
def test_refusals(binary, tmp_path):
    ref, mine, fn = _dirs(tmp_path, "holes")
    _run([binary, "fa2pac", fn], cwd=mine)
    _run([binary, "pac2bwt", fn + ".pac", "raw.bwt"], cwd=mine)
    raw = open(os.path.join(mine, "raw.bwt"), "rb").read()
    shutil.copy(os.path.join(mine, "raw.bwt"), os.path.join(mine, "upd.bwt"))
    _run([binary, "bwtupdate", "upd.bwt"], cwd=mine)
    for intv in ("0", "3", "-4"):
        r = _run([binary, "bwt2sa", "-i", intv, "upd.bwt", "x.sa"], cwd=mine, check=False)
        assert r.returncode == 1 and b"power of two" in r.stderr and not os.path.exists(os.path.join(mine, "x.sa")), r.stderr
    r = _run([binary, "bwt2sa", "raw.bwt", "x.sa"], cwd=mine, check=False)
    assert r.returncode == 1 and not os.path.exists(os.path.join(mine, "x.sa"))
    open(os.path.join(mine, "empty.pac"), "wb").write(b"\x00\x00")
    r = _run([binary, "pac2bwt", "empty.pac", "x.bwt"], cwd=mine, check=False)
    assert r.returncode == 1 and b"empty" in r.stderr and not os.path.exists(os.path.join(mine, "x.bwt"))
    # two BWT symbols swapped, then updated: refused if that split the LF cycle, else the reference's .sa
    rng = np.random.default_rng(5)
    n = _seq_len(os.path.join(mine, "raw.bwt"))
    split = kept = 0
    for t in range(12):
        bad, differ = _swap(raw, int(rng.integers(0, n)), int(rng.integers(0, n)))
        if not differ:
            continue
        b = "swap%d.bwt" % t
        for d in (ref, mine):
            open(os.path.join(d, b), "wb").write(bad)
        _run([binary, "bwtupdate", b], cwd=mine)
        _run([REF_BWA, "bwtupdate", b], cwd=ref)
        _same(os.path.join(ref, b), os.path.join(mine, b))
        r = _run([binary, "bwt2sa", b, b + ".sa"], cwd=mine, env=_env(16), check=False)
        if _lf_one_cycle(bad):
            kept += 1
            assert r.returncode == 0, r.stderr
            _run([REF_BWA, "bwt2sa", b, b + ".sa"], cwd=ref)
            _same(os.path.join(ref, b + ".sa"), os.path.join(mine, b + ".sa"))
        else:
            split += 1
            assert r.returncode == 1 and b"not the BWT of any text" in r.stderr, r.stderr
            assert not os.path.exists(os.path.join(mine, b + ".sa"))
    assert split > 0
    assert not [f for f in os.listdir(mine) if ".tmp" in f]


def test_bwtupdate_failure_leaves_input(tmp_path):
    """A .bwt of the wrong size for its L2 is refused and left as it was."""
    p = tmp_path / "x.bwt"
    data = np.array([0, 1, 2, 3, 100], dtype="<u8").tobytes() + b"\x00" * 12
    p.write_bytes(data)
    r = _run([CUSIMBIN, "bwtupdate", str(p)], check=False)
    assert r.returncode == 1 and p.read_bytes() == data
    assert os.listdir(str(tmp_path)) == ["x.bwt"]


# ---------------------------------------------------------------------------------------------- the chain

def _chain(binary, d, fa, env=None, times=None):
    """fa2pac -> pac2bwt -> bwtupdate -> fa2pac -f -> bwt2sa in directory d: the five index files of fa"""
    steps = (["fa2pac", fa], ["pac2bwt", fa + ".pac", fa + ".bwt"], ["bwtupdate", fa + ".bwt"], ["fa2pac", "-f", fa], ["bwt2sa", fa + ".bwt", fa + ".sa"])
    for s in steps:
        t0 = time.time()
        r = _run([binary] + s, cwd=d, env=env)
        if times is not None:
            times.append((s[0] + (" -f" if "-f" in s else ""), time.time() - t0, r.stderr.decode()))


def _chain_equals_index(binary, tmp_path, data, ref_name):
    fa, fqs = data.reads(ref_name, "idxsteps", 1000, paired=True)
    d = str(tmp_path / "chain")
    os.mkdir(d)
    shutil.copy(fa, os.path.join(d, "c.fa"))
    _chain(binary, d, "c.fa")
    os.mkdir(str(tmp_path / "idx"))
    shutil.copy(fa, str(tmp_path / "idx" / "c.fa"))
    _run([binary, "index", "c.fa"], cwd=str(tmp_path / "idx"))
    for ext in EXTS:
        _same(fa + "." + ext, os.path.join(d, "c.fa." + ext))
        _same(fa + "." + ext, str(tmp_path / "idx" / ("c.fa." + ext)))
    mine = os.path.join(d, "c.fa")
    assert run_sam(binary, [mine] + fqs) == run_sam(binary, [fa] + fqs)
    # the same output from an index whose .sa was re-made at another interval
    def aln_samse(idx):
        sai = idx + ".sai"
        with open(sai, "wb") as f:
            subprocess.run([binary, "aln", idx, fqs[0]], stdout=f, stderr=subprocess.DEVNULL, check=True)
        r = _run([binary, "samse", idx, sai, fqs[0]])
        return b"\n".join(l for l in r.stdout.split(b"\n") if not l.startswith(b"@PG"))
    want_mem, want_se = run_sam(binary, [mine] + fqs), aln_samse(mine)
    for intv in (16, 64):
        _run([binary, "bwt2sa", "-i", str(intv), "c.fa.bwt", "c.fa.sa"], cwd=d)
        assert np.frombuffer(open(mine + ".sa", "rb").read(48), dtype="<u8")[5] == intv
        assert run_sam(binary, [mine] + fqs) == want_mem
        assert aln_samse(mine) == want_se


@pytest.mark.parametrize("binary", BINS)
def test_chain_equals_index(binary, tmp_path, data):
    _chain_equals_index(binary, tmp_path, data, "two")


# ---------------------------------------------------------------------------------------------- large references (GPU)

def _md5(path):
    import hashlib
    h = hashlib.md5()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    return h.hexdigest()


@pytest.mark.gpu
def test_chain_gpu_100mbp(tmp_path):
    """100 Mbp uniform-random reference (4 contigs): our chain against the reference's chain, file for file, with the wall
    time of each step of both."""
    import gen_data
    ref, mine = str(tmp_path / "ref"), str(tmp_path / "mine")
    os.mkdir(ref)
    os.mkdir(mine)
    gen_data.write_fasta(os.path.join(ref, "r.fa"), gen_data.random_contigs(4, 25000000, 13))
    shutil.copy(os.path.join(ref, "r.fa"), os.path.join(mine, "r.fa"))
    t_ref, t_mine = [], []
    _chain(REF_BWA, ref, "r.fa", times=t_ref)
    _chain(GPUBIN, mine, "r.fa", env=_env(), times=t_mine)
    print("100 Mbp chain, wall seconds (bwa / bwa-b200): " + "; ".join("%s %.1f / %.1f" % (a[0], a[1], b[1]) for a, b in zip(t_ref, t_mine)))
    for ext in EXTS:
        _same(os.path.join(ref, "r.fa." + ext), os.path.join(mine, "r.fa." + ext))


@pytest.mark.gpu
@pytest.mark.timeout(3600)
def test_steps_gpu_3gbp(tmp_path):
    """The benchmark's 3 Gbp reference (tools/gen_data.py, seed 7, 24 x 125 Mbp): pac2bwt + bwtupdate + bwt2sa give the .bwt and
    .sa of `bwa-b200 index` (whose output is pinned to `bwa index`), by md5.  Prints each step's wall time and peak device memory."""
    import gen_data
    fa = str(tmp_path / "g3.fa")
    gen_data.write_fasta(fa, gen_data.random_contigs(24, 125000000, 7))
    t0 = time.time()
    _run([GPUBIN, "index", "-p", str(tmp_path / "idx"), fa])
    t_index = time.time() - t0
    times = []
    _chain(GPUBIN, str(tmp_path), "g3.fa", env=_env(), times=times)
    lines = ["%s %.1f s (%s)" % (s, t, "; ".join(l for l in e.splitlines() if "device memory" in l)) for s, t, e in times]
    print("3 Gbp: bwa-b200 index %.1f s; steps: %s" % (t_index, " | ".join(lines)))
    for ext in EXTS:
        assert _md5(str(tmp_path / "idx") + "." + ext) == _md5(fa + "." + ext), ext
