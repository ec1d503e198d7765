"""k_smem_c looks up two short-string table entries in one iteration where a lane's next two extensions are both lookups (the
first steps of a forward sweep, two mask candidates of a backward step).  Its seed-stage buffers (every interval, every suffix-array
position) and the reference-equivalent Occ-block touch count must stay the CPU oracle's, on the inputs where pairing has edges:
ambiguous bases inside the table's reach, reads shorter than the table depth, a seed length below, at and above the depth, long
reads with many re-seeding calls, batches smaller than a warp or finishing all at once, and the small-scratch repeat path."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ORACLE_SO, ROOT
from stage_abi import SeedPar, seed_stage

BACKENDS = [pytest.param("emu", id="emu"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)]
ENC = np.full(256, 4, dtype=np.uint8)
for _i, _ch in enumerate(b"ACGT"):
    ENC[_ch] = _i


def _lib(backend):
    if backend == "emu":
        return C.CDLL(os.path.join(ROOT, "tests/_build/libbwa_b200_cusim.so"), mode=C.RTLD_LOCAL)
    import bwa_b200
    return bwa_b200.lib()


def _depth(backend):
    return 8 if backend == "emu" else 12   # the emulator builds the table one fiber per entry: keep it small there


def _codes(seqs):
    off = np.zeros(len(seqs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    return ENC[np.frombuffer(b"".join(bytes(s) for s in seqs), dtype=np.uint8)].copy(), off


def _par(m):
    return SeedPar(m, int(m * 1.5 + .499), 10, 500, 20)


def _same(backend, fa, seqs, par, depth):
    import bwa_b200
    L = bwa_b200.lib()
    idx = L.bwa_idx_load(fa.encode(), 7).contents
    l_pac = C.cast(idx.bns, C.POINTER(C.c_int64))[0]
    codes, off = _codes(seqs)
    O = C.CDLL(ORACLE_SO, mode=C.RTLD_LOCAL)
    t = []
    want = seed_stage(O, idx.bwt, l_pac, idx.pac, codes, off, par, touches=t)
    got = seed_stage(_lib(backend), idx.bwt, l_pac, idx.pac, codes, off, par, ktab=depth, touches=t)
    assert got == want
    assert t[0] == t[1], t
    return want


def _ref(data, name):
    import gen_data
    fa = data.ref(name)
    return fa, gen_data.read_fasta(fa)[0]


@pytest.mark.parametrize("backend", BACKENDS)
def test_small_and_synchronous_batches(data, backend):
    """Fewer reads than a warp; then 64 exact reads of equal length, whose lanes run the same steps and finish together."""
    fa, c = _ref(data, "c1")
    rng = np.random.default_rng(41)
    few = [c[p:p + 150] for p in rng.integers(0, len(c) - 150, 5)]
    _same(backend, fa, few, _par(19), _depth(backend))
    same_len = [c[p:p + 150] for p in rng.integers(0, len(c) - 150, 64)]
    assert sum(len(r) for r in _same(backend, fa, same_len, _par(19), _depth(backend))) >= 64


@pytest.mark.parametrize("backend", BACKENDS)
def test_ambiguous_bases_and_short_reads_within_table_reach(data, backend):
    """An N at every position of the first and last table-depth bases (a pair must not look past it), reads of 1 to depth + 2
    bases, and reads that end right after the depth."""
    fa, c = _ref(data, "c1")
    d = _depth(backend)
    rng = np.random.default_rng(42)
    seqs = []
    for pos in list(range(d + 2)) + [149 - k for k in range(d + 2)]:
        p = int(rng.integers(0, len(c) - 150))
        s = c[p:p + 150].copy()
        s[pos] = ord("N")
        seqs.append(s)
    for ln in range(1, d + 3):
        p = int(rng.integers(0, len(c) - ln))
        seqs.append(c[p:p + ln].copy())
    s = c[3000:3150].copy(); s[d - 1] = s[d] = ord("N"); seqs.append(s)
    seqs.append(np.frombuffer(b"N" * 40, dtype=np.uint8).copy())
    for m in (5, 19):
        _same(backend, fa, seqs, _par(m), d)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("below", [3, 0, -7], ids=["seed_below_depth", "seed_at_depth", "seed_above_depth"])
def test_seed_length_against_table_depth(data, backend, below):
    """min_seed_len below, equal to and above the table depth: mask candidates are the strings of at most min(depth,
    min_seed_len) bases, forward lookups those of at most the depth."""
    fa, fqs = data.reads("stress", tag="k1p", n=96, seed=43, err=(0.016, 0.002, 0.002), chimeric=0.05)
    seqs = [l.strip() for i, l in enumerate(open(fqs[0], "rb")) if i % 4 == 1]
    seqs = [np.frombuffer(s, dtype=np.uint8) for s in seqs]
    d = _depth(backend)
    _same(backend, fa, seqs, _par(d - below), d)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("length,n", [(300, 24), (1000, 6)])
def test_long_repeat_reads(data, backend, length, n):
    """300- and 1000-bp reads of the repeat-rich reference with errors and chimeras: many re-seeding calls per read."""
    fa, fqs = data.reads("stress", tag="k1p%d" % length, n=n, length=length, seed=44, err=(0.02, 0.004, 0.004), chimeric=0.1)
    seqs = [np.frombuffer(l.strip(), dtype=np.uint8) for i, l in enumerate(open(fqs[0], "rb")) if i % 4 == 1]
    _same(backend, fa, seqs, _par(19), _depth(backend))


@pytest.mark.parametrize("backend", BACKENDS)
def test_small_scratch_repeats_the_stage(data, backend, monkeypatch):
    """BWA_B200_TEST_SMALL_K1: lists and result arrays overflow, the stage is repeated with larger scratch, same buffers."""
    monkeypatch.setenv("BWA_B200_TEST_SMALL_K1", "1")
    fa, fqs = data.reads("stress", tag="k1ps", n=64, seed=45, err=(0.016, 0.002, 0.002), chimeric=0.05)
    seqs = [np.frombuffer(l.strip(), dtype=np.uint8) for i, l in enumerate(open(fqs[0], "rb")) if i % 4 == 1]
    _same(backend, fa, seqs, _par(19), _depth(backend))
