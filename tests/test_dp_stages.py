"""The extension stage (K4, bwag_extend) and the global-alignment stage (K5, bwag_global) against the CPU oracle, call by call.

The inputs are recorded from the host glue over the oracle stages (tests/_build/bwa-b200-oracle with
BWA_B200_TEST_DUMP_STAGES): chains, seeds and CIGAR requests exactly as the reference's logic builds them, for each option
set.  Each recording is replayed through liboracle.so and through the library under test -- the CUDA kernels under the SIMT
emulator (tests/_build/libbwa_b200_cusim.so) without a GPU, libbwa_b200.so with -m gpu -- and every region (all fields of
bwag_xreg_t) and every alignment (score, NM, CIGAR words, MD bytes) must be equal.  The option sets reach the edges of the
arithmetic that depends on them: the band, cal_max_gap, max_ins / max_del with gap extensions of 0 (divisions by zero that
the reference's x86 build truncates to INT_MIN), the lane kernel's 13-bit cells and its shared-memory limit.  The kernel routes
are forced one by one and the BWA_B200_PROFILE lines show that each was taken."""
import ctypes as C
import glob
import os
import re
import subprocess

import numpy as np
import pytest

import bwa_b200
from conftest import CUSIMBIN, ORACLE_SO, ROOT, TESTBIN, ref_sam, run_sam

CUSIM_SO = os.path.join(ROOT, "tests", "_build", "libbwa_b200_cusim.so")
TARGETS = [pytest.param("emu", id="emu"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)]


class SwPar(C.Structure):
    _fields_ = [(k, C.c_int) for k in ("a", "b", "o_del", "e_del", "o_ins", "e_ins", "w", "zdrop", "pen_clip5", "pen_clip3")] + [("mat", C.c_int8 * 25)]


class RegsOut(C.Structure):
    _fields_ = [("n_regs", C.c_void_p), ("regs", C.c_void_p)]


class GalnOut(C.Structure):
    _fields_ = [("res", C.c_void_p), ("cigar", C.c_void_p), ("md", C.c_void_p)]


XCHAIN = np.dtype([("rmax0", "<i8"), ("rmax1", "<i8"), ("seed_off", "<i4"), ("n_seeds", "<i4")])
XSEED = np.dtype([("rbeg", "<i8"), ("qbeg", "<i4"), ("len", "<u4")])
XREG = np.dtype([("rb", "<i8"), ("re", "<i8")] + [(k, "<i4") for k in ("qb", "qe", "score", "truesc", "w", "seedcov", "seedlen0", "chain")])
GTASK = np.dtype([("rb", "<i8"), ("re", "<i8")] + [(k, "<i4") for k in ("read", "qb", "qe", "w", "truesc", "mode")])
GRES = np.dtype([(k, "<i4") for k in ("score", "n_cigar", "NM", "l_md")] + [("cigar_off", "<i8"), ("md_off", "<i8")])
G_REG2ALN, G_SCORE = 0, 1


# ---------------------------------------------------------------------------------------------------- libraries and index
_libs = {}


def _lib(name):
    if name not in _libs:
        if name == "oracle":
            L = C.CDLL(ORACLE_SO, mode=C.RTLD_LOCAL)
        elif name == "emu":
            L = C.CDLL(CUSIM_SO, mode=C.RTLD_LOCAL)
        else:
            L = bwa_b200.lib()
        L.bwag_ctx_create.restype = C.c_void_p
        L.bwag_ctx_create.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
        L.bwag_batch_begin.restype = C.c_void_p
        L.bwag_batch_begin.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.bwag_batch_end.argtypes = [C.c_void_p]
        L.bwag_extend.argtypes = [C.c_void_p, C.POINTER(SwPar), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(RegsOut)]
        L.bwag_global.argtypes = [C.c_void_p, C.POINTER(SwPar), C.c_int, C.c_void_p, C.POINTER(GalnOut)]
        L.bwag_last_error.restype = C.c_char_p
        _libs[name] = L
    return _libs[name]


_ctx = {}


def _context(name, fa):
    """a context of library `name` over the index of fa (index loaded once, by the product library's host code)"""
    if (name, fa) not in _ctx:
        if ("idx", fa) not in _ctx:
            idx = bwa_b200.lib().bwa_idx_load(fa.encode(), 7).contents
            _ctx["idx", fa] = (idx.bwt, C.cast(idx.bns, C.POINTER(C.c_int64))[0], idx.pac)
        bwt, l_pac, pac = _ctx["idx", fa]
        ctx = _lib(name).bwag_ctx_create(-1, bwt, l_pac, pac)
        assert ctx, _lib(name).bwag_last_error()
        _ctx[name, fa] = ctx
    return _ctx[name, fa]


def _l_pac(fa):
    _context("oracle", fa)
    return _ctx["idx", fa][1]


# ---------------------------------------------------------------------------------------------------- recordings
def _parse(path):
    buf = open(path, "rb").read()
    h = np.frombuffer(buf, "<i8", 8)
    kind, n, n_codes, n_items, n_seeds, par_size, item_size = (int(x) for x in h[:7])
    assert par_size == C.sizeof(SwPar) and item_size == (XCHAIN if kind == 1 else GTASK).itemsize, path
    pos = 64
    rec = {"kind": kind, "file": os.path.basename(path), "par": SwPar.from_buffer_copy(buf[pos:pos + par_size])}
    pos += par_size

    def take(dtype, count):
        nonlocal pos
        a = np.frombuffer(buf, dtype, count, pos).copy()
        pos += a.nbytes
        return a
    rec["off"] = take("<i8", n + 1)
    rec["codes"] = take("u1", n_codes)
    if kind == 1:
        rec["chain_off"] = take("<i4", n + 1)
        rec["chains"] = take(XCHAIN, n_items)
        rec["seeds"] = take(XSEED, n_seeds)
    else:
        rec["tasks"] = take(GTASK, n_items)
    assert pos == len(buf), path
    return rec


def record(tmp_path, fa, fqs, opts, tag="rec"):
    """the inputs of every bwag_extend / bwag_global call of `bwa-b200 mem opts` over the oracle stages: (extensions, global alignments)"""
    d = tmp_path / tag
    d.mkdir()
    env = dict(os.environ, BWA_B200_TEST_DUMP_STAGES=str(d))
    p = subprocess.run([TESTBIN, "mem", "-v", "1", "-K", "100000000", "-t", "2"] + opts + [fa] + fqs, env=env,
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, timeout=600)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    ext = [_parse(f) for f in sorted(glob.glob(str(d / "extend-*.bin")))]
    glb = [_parse(f) for f in sorted(glob.glob(str(d / "global-*.bin")))]
    assert ext and glb, "nothing recorded"
    return ext, glb


# ---------------------------------------------------------------------------------------------------- replay
def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def run_extend(name, fa, rec):
    L = _lib(name)
    n = len(rec["off"]) - 1
    b = L.bwag_batch_begin(_context(name, fa), n, _ptr(rec["codes"]), _ptr(rec["off"]))
    assert b
    out = RegsOut()
    par = SwPar.from_buffer_copy(rec["par"])
    rc = L.bwag_extend(b, C.byref(par), _ptr(rec["chain_off"]), _ptr(rec["chains"]), len(rec["seeds"]), _ptr(rec["seeds"]), C.byref(out))
    assert rc == 0, (name, L.bwag_last_error())
    n_regs = np.frombuffer(C.string_at(out.n_regs, 4 * n), "<i4").copy()
    regs = np.frombuffer(C.string_at(out.regs, XREG.itemsize * len(rec["seeds"])), XREG).copy() if len(rec["seeds"]) else np.zeros(0, XREG)
    L.bwag_batch_end(b)
    return n_regs, regs


def run_global(name, fa, rec):
    L = _lib(name)
    n, nt = len(rec["off"]) - 1, len(rec["tasks"])
    b = L.bwag_batch_begin(_context(name, fa), n, _ptr(rec["codes"]), _ptr(rec["off"]))
    assert b
    out = GalnOut()
    par = SwPar.from_buffer_copy(rec["par"])
    rc = L.bwag_global(b, C.byref(par), nt, _ptr(rec["tasks"]), C.byref(out))
    assert rc == 0, (name, L.bwag_last_error())
    res = np.frombuffer(C.string_at(out.res, GRES.itemsize * nt), GRES).copy()
    got = []
    for r in res:
        cig = np.frombuffer(C.string_at(out.cigar + 4 * int(r["cigar_off"]), 4 * int(r["n_cigar"])), "<u4") if r["n_cigar"] > 0 else np.zeros(0, "<u4")
        md = C.string_at(out.md + int(r["md_off"]), int(r["l_md"])) if r["l_md"] > 0 else b""
        got.append((int(r["score"]), int(r["n_cigar"]), int(r["NM"]), int(r["l_md"]), tuple(int(x) for x in cig), md))
    L.bwag_batch_end(b)
    return got


def _par_str(p):
    return "a=%d b=%d o_del=%d e_del=%d o_ins=%d e_ins=%d w=%d zdrop=%d clip=%d,%d" % (p.a, p.b, p.o_del, p.e_del, p.o_ins, p.e_ins, p.w, p.zdrop, p.pen_clip5, p.pen_clip3)


def _read_str(rec, r):
    return "".join("ACGTN"[c] for c in rec["codes"][rec["off"][r]:rec["off"][r + 1]])


def compare_extend(target, fa, rec, label):
    """every read with chains: n_regs and each bwag_xreg_t equal; returns the number of regions compared"""
    wn, wr = run_extend("oracle", fa, rec)
    gn, gr = run_extend(target, fa, rec)
    co, bad, n_cmp = rec["chain_off"], [], 0
    for r in range(len(co) - 1):
        if co[r + 1] == co[r]:
            continue
        base = int(rec["chains"][co[r]]["seed_off"])
        k = int(wn[r])
        n_cmp += k
        if gn[r] != k or wr[base:base + k].tobytes() != gr[base:base + max(int(gn[r]), 0)].tobytes():
            bad.append(r)
    if bad:
        r = bad[0]
        base = int(rec["chains"][co[r]]["seed_off"])
        ch = rec["chains"][co[r]:co[r + 1]]
        pytest.fail("%s (%s): regions of %d of %d reads differ (%s, %s)\nfirst: read %d (%d bp) %s\nchains %s\nseeds %s\nwant %d: %s\ngot  %d: %s" % (
            label, rec["file"], len(bad), int(np.count_nonzero(co[1:] > co[:-1])), _par_str(rec["par"]), target, r, rec["off"][r + 1] - rec["off"][r],
            _read_str(rec, r), ch.tolist(), rec["seeds"][ch[0]["seed_off"]:ch[-1]["seed_off"] + ch[-1]["n_seeds"]].tolist(),
            wn[r], wr[base:base + wn[r]].tolist(), gn[r], gr[base:base + max(int(gn[r]), 0)].tolist()))
    return n_cmp


def compare_global(target, fa, rec, label):
    want = run_global("oracle", fa, rec)
    got = run_global(target, fa, rec)
    bad = [t for t in range(len(want)) if want[t] != got[t]]
    if bad:
        t = bad[0]
        tk = rec["tasks"][t]
        pytest.fail("%s (%s): %d of %d alignments differ (%s, %s)\nfirst: task %d %s\nread %d: %s\nwant %s\ngot  %s" % (
            label, rec["file"], len(bad), len(want), _par_str(rec["par"]), target, t, tk, tk["read"], _read_str(rec, int(tk["read"])), want[t], got[t]))
    return len(want)


def compare_recording(target, fa, ext, glb, label):
    n_regs = sum(compare_extend(target, fa, r, label) for r in ext)
    n_aln = sum(compare_global(target, fa, r, label) for r in glb)
    return n_regs, n_aln


# ---------------------------------------------------------------------------------------------------- option sets and read sets
STRESS_ERR = (0.016, 0.002, 0.002)
# name -> (reference, reads(kw) on the emulator, on the GPU)
READS = {
    "se150": ("stress", dict(tag="dp150", length=150, seed=41, err=STRESS_ERR, chimeric=0.1), 80, 3000),
    "se36": ("c1", dict(tag="dp36", length=36, seed=42), 80, 3000),
    "se400": ("c1", dict(tag="dp400", length=400, seed=43, err=STRESS_ERR, chimeric=0.1), 24, 1000),
    "l1k": ("two", dict(tag="dp1k", length=1000, seed=44, err=STRESS_ERR, chimeric=0.2), 6, 200),
    "l8k": ("two", dict(tag="dp8k", length=8000, seed=45, err=(0.02, 0.05, 0.03)), 1, 12),
    "se292": ("c1", dict(tag="dp292", length=292, seed=46, err=STRESS_ERR), 24, 1000),
    "se388": ("c1", dict(tag="dp388", length=388, seed=47, err=STRESS_ERR), 16, 800),
    "se392": ("c1", dict(tag="dp392", length=392, seed=48, err=STRESS_ERR), 16, 800),
}

# (id, read set, options, K4 kernel the profile must show or None)
CASES = [
    ("default", "se150", [], None),
    ("E0", "se150", ["-E", "0"], None),
    ("E0_1", "se150", ["-E", "0,1"], None),
    ("E1_0", "se150", ["-E", "1,0"], None),
    ("O0", "se150", ["-O", "0"], None),
    ("O0_E0", "se150", ["-O", "0", "-E", "0"], None),
    ("B40_O60_E10", "se150", ["-B", "40", "-O", "60", "-E", "10"], None),
    ("L0", "se150", ["-L", "0"], None),
    ("L100", "se150", ["-L", "100"], None),
    ("d0", "se150", ["-d", "0"], None),
    ("d1", "se150", ["-d", "1"], None),
    ("d100000", "se150", ["-d", "100000"], None),
    ("w0", "se150", ["-w", "0"], None),
    ("w1", "se150", ["-w", "1"], None),
    ("w500", "se150", ["-w", "500"], None),
    ("se36", "se36", [], None),
    ("se36_E0", "se36", ["-E", "0"], None),
    ("se400", "se400", [], None),
    ("l1k", "l1k", [], None),
    ("l1k_E0", "l1k", ["-O", "0", "-E", "0"], None),
    ("pacbio", "l8k", ["-x", "pacbio"], None),
    ("ont2d", "l1k", ["-x", "ont2d"], None),
    # 13-bit cells of the lane kernel: 292 x 28 = 8176 < 8192 takes it, 292 x 29 = 8468 does not
    ("A28_292bp", "se292", ["-A", "28"], "lane"),
    ("A29_292bp", "se292", ["-A", "29"], "warp"),
    # the lane kernel's row of (read length + 10) x 128 lanes x 4 bytes in at most 200 KB of shared memory: 388 bp fit, 392 bp do not
    ("lane_smem_388bp", "se388", [], "lane"),
    ("lane_smem_392bp", "se392", [], "warp"),
]


def _reads(data, target, rs):
    ref, kw, n_emu, n_gpu = READS[rs]
    kw = dict(kw, tag=kw["tag"] + ("g" if target == "gpu" else "e"))
    return data.reads(ref, n=n_gpu if target == "gpu" else n_emu, **kw)


def _k4_kernels(err):
    return set(re.findall(r"\[prof\] extension: (lane-per-read kernel|warp-per-read kernel \w+)", err))


@pytest.mark.parametrize("target", TARGETS)
@pytest.mark.parametrize("case,rs,opts,k4", CASES, ids=[c[0] for c in CASES])
def test_stages_equal_oracle(data, tmp_path, monkeypatch, capfd, target, case, rs, opts, k4):
    fa, fqs = _reads(data, target, rs)
    ext, glb = record(tmp_path, fa, fqs, opts)
    monkeypatch.setenv("BWA_B200_PROFILE", "1")
    capfd.readouterr()
    n_regs, n_aln = compare_recording(target, fa, ext, glb, "%s %s" % (case, " ".join(opts)))
    assert n_regs > 0 and n_aln > 0
    if k4 is not None:
        ks = _k4_kernels(capfd.readouterr().err)
        if k4 == "lane":
            assert "lane-per-read kernel" in ks, ks
        else:
            assert "lane-per-read kernel" not in ks and "warp-per-read kernel k_extend_sm_fast" in ks, ks


# kernel routes: environment -> the K4 and K5 kernels the profile lines must name
ROUTES = [
    ("default", {}, ["lane-per-read kernel for reads with chains 0..8", "warp-per-read kernel k_extend_sm_fast"], ["warp-per-request kernel k_global_sm_fast"]),
    ("k4_warp", {"BWA_B200_K4_LANE": "0"}, ["warp-per-read kernel k_extend_sm_fast (scratch in shared memory, lean row sweep) for reads with chains 0.."], []),
    ("k4_global_scratch", {"BWA_B200_K4_LANE": "0", "BWA_B200_K4_SM": "0"}, ["warp-per-read kernel k_extend_fast (scratch in global memory, lean row sweep)"], []),
    ("first_sweep", {"BWA_B200_K4_FAST": "0", "BWA_B200_K5_FAST": "0"}, ["warp-per-read kernel k_extend_sm (scratch in shared memory, first row sweep)"],
     ["warp-per-request kernel k_global_sm (scratch in shared memory, first row sweep)"]),
    ("global_scratch_first_sweep", {"BWA_B200_K4_SM": "0", "BWA_B200_K5_SM": "0", "BWA_B200_K4_FAST": "0", "BWA_B200_K5_FAST": "0"},
     ["warp-per-read kernel k_extend (scratch in global memory, first row sweep)"], ["warp-per-request kernel k_global (scratch in global memory, first row sweep)"]),
    ("k4_split", {"BWA_B200_K4_LANE_MAXCHAINS": "1"}, ["lane-per-read kernel for reads with chains 0..1", "warp-per-read kernel k_extend_sm_fast (scratch in shared memory, lean row sweep) for reads with chains 2.."], []),
    ("k5_lane", {"BWA_B200_K5_LANE": "1"}, [], ["lane-per-request kernel made"]),
    ("k5_global_scratch", {"BWA_B200_K5_SM": "0"}, [], ["warp-per-request kernel k_global_fast (scratch in global memory, lean row sweep)"]),
]


_route_cache = {}


def _route_recordings(data, tmp_path_factory, target):
    """150-bp reads of the repeat-rich reference (reads with one chain and with several, so that a split between the lane and
    the warp kernel has work on both sides; more than 64 CIGAR requests per call), with the default options and with -E 0"""
    if target not in _route_cache:
        fa, fqs = _reads(data, target, "se150")
        _route_cache[target] = (fa, [(opts,) + record(tmp_path_factory.mktemp("route"), fa, fqs, opts) for opts in ([], ["-E", "0"])])
    return _route_cache[target]


@pytest.mark.parametrize("target", TARGETS)
@pytest.mark.parametrize("route,env,k4,k5", ROUTES, ids=[r[0] for r in ROUTES])
def test_routes_equal_oracle(data, tmp_path_factory, monkeypatch, capfd, target, route, env, k4, k5):
    fa, recs = _route_recordings(data, tmp_path_factory, target)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("BWA_B200_PROFILE", "1")
    for opts, ext, glb in recs:
        if route == "k4_split":
            assert any(np.any(np.diff(r["chain_off"]) >= 2) and np.any(np.diff(r["chain_off"]) == 1) for r in ext)
        if route == "k5_lane":
            assert max(len(r["tasks"]) for r in glb) >= 64
        capfd.readouterr()
        compare_recording(target, fa, ext, glb, "route %s, %s" % (route, " ".join(opts) or "defaults"))
        err = capfd.readouterr().err
        for s in k4 + k5:
            assert s in err, (s, err[-3000:])
        if route == "k4_warp" or route == "k4_global_scratch":
            assert "lane-per-read kernel" not in err
        if route == "k5_lane":
            assert re.search(r"lane-per-request kernel made [1-9]\d* of", err), err[-3000:]


# ---------------------------------------------------------------------------------------------------- hand-written inputs
def _ref_codes(fa):
    import gen_data
    tab = np.full(256, 4, dtype=np.uint8)
    for i, ch in enumerate(b"ACGT"):
        tab[ch] = i
    return [tab[c] for c in gen_data.read_fasta(fa)]


def _revcomp(s):
    r = s[::-1].copy()
    r[r < 4] = 3 - r[r < 4]
    return r


def _sw_par(a=1, b=4, o_del=6, e_del=1, o_ins=6, e_ins=1, w=100, zdrop=100, clip5=5, clip3=5):
    p = SwPar(a, b, o_del, e_del, o_ins, e_ins, w, zdrop, clip5, clip3)
    for i in range(5):
        for j in range(5):
            p.mat[i * 5 + j] = -1 if (i == 4 or j == 4) else (a if i == j else -b)
    return p


def _batch(reads):
    off = np.zeros(len(reads) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(r) for r in reads])
    return off, np.concatenate(reads).astype(np.uint8)


PARS = [("defaults", {}), ("E0", dict(e_del=0, e_ins=0)), ("E0_1", dict(e_del=0)), ("O0_E0", dict(o_del=0, e_del=0, o_ins=0, e_ins=0)),
        ("w0", dict(w=0)), ("w1", dict(w=1)), ("B40_O60_E10", dict(b=40, o_del=60, e_del=10, o_ins=60, e_ins=10))]


def _global_tasks(fa):
    """reads cut from the 2-contig reference (forward and reverse strand, with mismatches, indels and Ns) and requests over them"""
    ref = _ref_codes(fa)
    fwd = np.concatenate(ref)
    l_pac = len(fwd)
    assert l_pac == _l_pac(fa)
    c0 = len(ref[0])
    rng = np.random.default_rng(7)
    reads, tasks = [], []

    def add_read(s):
        reads.append(s.astype(np.uint8))
        return len(reads) - 1

    def task(r, qb, qe, rb, re_, w, truesc, mode):
        tasks.append((rb, re_, r, qb, qe, w, truesc, mode))

    def both(r, qb, qe, rb, re_, w, truesc=10000):
        task(r, qb, qe, rb, re_, w, truesc, G_REG2ALN)
        task(r, qb, qe, rb, re_, w, truesc, G_SCORE)
    p = 5000
    exact = fwd[p:p + 120].copy()
    r = add_read(exact)
    for w in (0, 1, 4):
        both(r, 0, 120, p, p + 120, w)                     # gap-free: the diagonal when w is 0
    mm = exact.copy(); mm[[3, 50, 119]] = (mm[[3, 50, 119]] + 1) % 4
    r = add_read(mm)
    for w in (0, 1):
        both(r, 0, 120, p, p + 120, w)
    r = add_read(fwd[p + 7:p + 8].copy())                  # qlen 1
    both(r, 0, 1, p + 7, p + 8, 0); both(r, 0, 1, p + 5, p + 9, 1); both(r, 0, 1, p + 6, p + 8, 0)
    # indels: a 6-base and a second 6-base insertion, then a 12-base deletion (offsets 6 and 12 from the diagonal: bands 4, 8, 16 each
    # gain) -- with truesc far above every score the band doubles until the third try
    s = fwd[20000:20200]
    ins1, ins2 = rng.integers(0, 4, 6), rng.integers(0, 4, 6)
    ind = np.concatenate([s[:40], ins1, s[40:80], ins2, s[80:120], s[132:200]])
    r = add_read(ind)
    for w in (1, 4):
        both(r, 0, len(ind), 20000, 20200, w)
    task(r, 0, len(ind), 20000, 20200, 4, 0, G_REG2ALN)     # truesc reached at once: a single try
    task(r, 10, len(ind) - 10, 20010, 20190, 2, 10000, G_REG2ALN)
    # reverse strand windows ([2 l_pac - end, 2 l_pac - beg) holds the reverse complement of [beg, end))
    rc = _revcomp(fwd[30000:30150]); rc[[10, 11, 80]] = (rc[[10, 11, 80]] + 2) % 4
    r = add_read(rc)
    for w in (0, 1, 5):
        both(r, 0, 150, 2 * l_pac - 30150, 2 * l_pac - 30000, w)
    rci = np.concatenate([rc[:60], rc[63:]])
    r = add_read(rci)
    both(r, 0, len(rci), 2 * l_pac - 30150, 2 * l_pac - 30000, 2)
    # windows ending at the end of the first contig, at l_pac (end of the forward strand), and starting at l_pac
    r = add_read(fwd[c0 - 100:c0].copy())
    both(r, 0, 100, c0 - 100, c0, 1); both(r, 0, 100, c0 - 103, c0, 3)
    r = add_read(fwd[l_pac - 90:l_pac].copy())
    both(r, 0, 90, l_pac - 90, l_pac, 0); both(r, 0, 90, l_pac - 95, l_pac, 2)
    r = add_read(_revcomp(fwd[l_pac - 80:l_pac]))
    both(r, 0, 80, l_pac, l_pac + 80, 1); both(r, 0, 80, l_pac, l_pac + 84, 3)
    r = add_read(fwd[0:70].copy())                         # the first base of the reference
    both(r, 0, 70, 0, 70, 0); both(r, 0, 70, 0, 73, 2)
    # reads with N: single, a run, all N
    nn = fwd[40000:40130].copy(); nn[[0, 64, 129]] = 4
    r = add_read(nn)
    both(r, 0, 130, 40000, 40130, 0); both(r, 0, 130, 40000, 40132, 3)
    nr = fwd[41000:41130].copy(); nr[50:70] = 4
    r = add_read(nr)
    both(r, 0, 130, 41000, 41130, 1)
    r = add_read(np.full(40, 4, np.uint8))
    both(r, 0, 40, 42000, 42040, 1)
    # a clipped part of a read (qb > 0) against a shifted window
    r = add_read(fwd[43000:43150].copy())
    both(r, 30, 140, 43030, 43140, 1); both(r, 30, 140, 43028, 43142, 4)
    off, codes = _batch(reads)
    return off, codes, np.array(tasks, dtype=GTASK)


@pytest.mark.parametrize("target", TARGETS)
@pytest.mark.parametrize("pname,pkw", PARS, ids=[p[0] for p in PARS])
def test_handwritten_global_tasks(data, target, pname, pkw):
    fa = data.ref("two")
    off, codes, tasks = _global_tasks(fa)
    rec = {"file": "hand-written", "par": _sw_par(**pkw), "off": off, "codes": codes, "tasks": tasks}
    assert compare_global(target, fa, rec, "hand-written global tasks, " + pname) == len(tasks)


def _ext_inputs(fa, l_pac):
    """reads from the 1-Mbp reference with hand-placed chains: one seed at the read's start, one at its end, one covering it whole, several
    seeds ordered as the host orders them (ascending score << 32 | index, the last one extended first), a reverse-strand chain, and a
    chain whose window starts at the first base of the reference"""
    fwd = _ref_codes(fa)[0]
    reads, chains, seeds, chain_off = [], [], [], [0]

    def read(s, chs):   # chs: (rmax0, rmax1, [(rbeg, qbeg, len), ...]) per chain
        reads.append(s.astype(np.uint8))
        for rmax0, rmax1, sds in chs:
            chains.append((rmax0, rmax1, len(seeds), len(sds)))
            for key in sorted((ln << 32 | k) for k, (rb, qb, ln) in enumerate(sds)):
                rb, qb, ln = sds[key & 0xffffffff]
                seeds.append((rb, qb, ln))
        chain_off.append(len(chains))
    p = 300000
    s = fwd[p:p + 150].copy(); s[[20, 75, 140]] = (s[[20, 75, 140]] + 1) % 4
    w0, w1 = p - 300, p + 450
    read(s, [(w0, w1, [(p, 0, 19)])])                       # seed at qbeg 0
    read(s, [(w0, w1, [(p + 121, 121, 29)])])               # seed ending at the read's end
    read(fwd[p:p + 150].copy(), [(w0, w1, [(p, 0, 150)])])  # seed covering the whole read
    t = np.concatenate([fwd[p + 500:p + 560], fwd[p + 563:p + 650], fwd[p + 650:p + 660]])
    read(t, [(p + 200, p + 960, [(p + 500, 0, 40), (p + 563, 60, 25), (p + 600, 97, 50), (p + 520, 20, 25)]),
             (p + 200, p + 960, [(p + 610, 107, 40)])])     # several seeds, and two chains of one read
    rc = _revcomp(fwd[p + 2000:p + 2150]); rc[30] = (rc[30] + 1) % 4
    rb = 2 * l_pac - (p + 2150)
    read(rc, [(rb - 300, rb + 450, [(rb + 40, 40, 60)])])   # reverse strand
    read(fwd[0:150].copy(), [(0, 450, [(0, 0, 30), (100, 100, 30)])])   # window starting at the first base
    n4 = fwd[p + 3000:p + 3150].copy(); n4[[0, 1, 149]] = 4
    read(n4, [(p + 2700, p + 3450, [(p + 3010, 10, 100)])])
    off, codes = _batch(reads)
    return {"file": "hand-written", "off": off, "codes": codes, "chain_off": np.array(chain_off, dtype="<i4"),
            "chains": np.array(chains, dtype=XCHAIN), "seeds": np.array(seeds, dtype=XSEED)}


@pytest.mark.parametrize("target", TARGETS)
@pytest.mark.parametrize("route", [{}, {"BWA_B200_K4_LANE": "0"}, {"BWA_B200_K4_LANE": "0", "BWA_B200_K4_SM": "0", "BWA_B200_K4_FAST": "0"}], ids=["lane", "warp", "warp_global_first"])
@pytest.mark.parametrize("pname,pkw", PARS, ids=[p[0] for p in PARS])
def test_handwritten_extensions(data, monkeypatch, target, route, pname, pkw):
    fa = data.ref("c1")
    rec = _ext_inputs(fa, _l_pac(fa))
    rec["par"] = _sw_par(**pkw)
    for k, v in route.items():
        monkeypatch.setenv(k, v)
    assert compare_extend(target, fa, rec, "hand-written extensions, " + pname) > 0


# ---------------------------------------------------------------------------------------------------- whole SAM, and the source
SAM_OPTS = [["-E", "0"], ["-E", "0,1"], ["-O", "0", "-E", "0"]]


@pytest.mark.parametrize("target", TARGETS)
@pytest.mark.parametrize("opts", SAM_OPTS, ids=["E0", "E0_1", "O0_E0"])
@pytest.mark.parametrize("paired", [False, True], ids=["se", "pe"])
def test_zero_gap_extension_sam(data, target, opts, paired):
    """bwa-b200 mem with gap extensions of 0, SAM against the reference: the only test that reaches the cal_max_gap of the chaining
    kernel (K3), which runs on the default (device-chaining) path"""
    if target == "gpu":
        kw = dict(tag="gpe", n=3000, seed=4, paired=True) if paired else dict(tag="gse", n=4000, seed=3, chimeric=0.05)
        binary = bwa_b200.CLI_PATH
    else:
        kw = dict(tag="cspe", n=60, seed=34, paired=True) if paired else dict(tag="cs", n=120, seed=33, chimeric=0.05)
        binary = CUSIMBIN
    fa, fqs = data.reads("stress", err=STRESS_ERR, **kw)
    args = opts + ["-K", "100000000", "-t", "4", fa] + fqs
    assert run_sam(binary, args) == ref_sam(args)


def test_no_raw_double_to_int_casts_in_device_code():
    """(int) of a double is cvt.rzi.s32.f64 on the device, which saturates where the reference's x86 build gives INT_MIN: the
    reference's band and gap formulas go through bwag_trunc_i32 instead"""
    bad = []
    for f in sorted(glob.glob(os.path.join(ROOT, "bwa_b200", "csrc", "cuda", "*.c*"))):
        for i, line in enumerate(open(f), 1):
            if re.search(r"\(int\)\s*\(+\s*\(double\)", line):
                bad.append("%s:%d: %s" % (os.path.basename(f), i, line.strip()))
    assert not bad, "\n".join(bad)
