"""Stage 4's SAM text (k_tail_sam) for records that do not fit a lane's slot of shared memory: 1000- and 2000-bp reads, short and
long reads in one batch, ~200-character contig names and a long read group, single- and paired-end.  Records that fit their slot
are copied out by the warp, the others are written straight to the text pool; both must give the reference's bytes, and stage 4
must take every read without handing any back.  CPU: the SIMT emulator; -m gpu: the H100."""
import subprocess

import pytest

import bwa_b200
from conftest import CUSIMBIN, REF_BWA, ref_sam
from test_tail import _counts

LONG_NAME = "contig_" + "abcdefghij" * 19 + "_"   # + the contig number: 198-200 characters
LONG_RG = "@RG\\tID:" + "grp" * 70 + "\\tSM:sample"


@pytest.fixture(scope="module")
def long_names(tmp_path_factory):
    import gen_data
    d = tmp_path_factory.mktemp("tail_text")
    contigs = gen_data.random_contigs(3, 200000, 17)
    fa = str(d / "ref.fa")
    gen_data.write_fasta(fa, contigs, prefix=LONG_NAME)
    subprocess.run([REF_BWA, "index", fa], check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    return d, fa, contigs


def _reads(d, contigs, tag, parts, paired):
    """parts: (number, length, insert) per read length; the kinds alternate in the files so that a warp sees both."""
    import gen_data
    sets = []
    for k, (n, length, ins) in enumerate(parts):
        r1, r2 = gen_data.gen_reads(contigs, n, length, 100 + k, err=(0.004, 0.0, 0.0), paired=paired, ins_mean=ins, ins_sd=ins // 20,
                                    prefix="%s%d_" % (tag, k))
        sets.append((r1, r2))
    outs = []
    for e in range(2 if paired else 1):
        recs = []
        for i in range(max(n for n, _, _ in parts)):
            for s in sets:
                if i < len(s[e]):
                    recs.append(s[e][i])
        out = str(d / ("%s_%d.fq" % (tag, e + 1)))
        gen_data.write_fastq(out, recs)
        outs.append(out)
    return outs, sum(n for n, _, _ in parts) * (2 if paired else 1)


def _check(binary, long_names, scale):
    d, fa, contigs = long_names
    # A slot is max_len + 176 + the read group's length, rounded up to 16 and capped at TAIL_SLOT_MAX (512) bytes.  A record is
    # its SEQ, about 100 bytes of fields and tags, one ~200-character contig name (RNEXT is "=") and the read group id.
    cases = (("pe1k", [(8 * scale, 1000, 2500)], True, ["-R", LONG_RG]),              # slot 512: every record overflows
             # 150-bp records (~450 bytes) fit the 512-byte slot, 2000-bp ones overflow; alone, reads this long skip stage 4 (mean > 1500 bp)
             ("pe2k", [(8 * scale, 150, 400), (4 * scale, 2000, 4500)], True, []),
             ("pemix", [(16 * scale, 150, 2500), (4 * scale, 1000, 2500)], True, []),  # both paths in one warp; one insert-size model: no mate rescue
             ("se150", [(24 * scale, 150, 0)], False, []),                             # slot 336: the contig name alone makes every record overflow
             ("semix", [(16 * scale, 100, 0), (6 * scale, 300, 0), (3 * scale, 2000, 0)], False, ["-R", LONG_RG]))   # slot 512, the read group makes all overflow
    for tag, parts, paired, extra in cases:
        fqs, n_reads = _reads(d, contigs, tag, parts, paired)
        args = extra + ["-K", "100000000", "-t", "4", fa] + fqs
        sam, took, handed, _ = _counts(binary, args)
        assert sam == ref_sam(args), tag
        assert took == n_reads and handed == 0, (tag, took, handed)

    # chunks of different read lengths on several lanes at once: each launch sizes its slots from its own chunk
    fqs, n_reads = _reads(d, contigs, "selanes", [(40 * scale, 100, 0)], False)
    fq2, n2 = _reads(d, contigs, "selanes_long", [(40 * scale, 300, 0)], False)
    with open(fqs[0], "a") as o, open(fq2[0]) as i:
        o.write(i.read())
    args = ["-K", "100000000", "-t", "4", fa, fqs[0]]
    sam, took, handed, _ = _counts(binary, args, {"BWA_B200_CHUNK": str(8 * scale), "BWA_B200_LANES": "3"})
    assert sam == ref_sam(args)
    assert took == n_reads + n2 and handed == 0, (took, handed)


def test_tail_text_emulated(long_names):
    _check(CUSIMBIN, long_names, 1)


@pytest.mark.gpu
def test_tail_text_gpu(long_names):
    _check(bwa_b200.CLI_PATH, long_names, 40)
