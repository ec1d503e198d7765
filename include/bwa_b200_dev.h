/* bwa_b200_dev.h -- device-batch entry points (C ABI) of the H100 seed-and-extend path.
 *
 * These are the calls the host glue (mem_process_seqs) makes where the reference's worker threads
 * call bwt_smem1/bwt_seed_strategy1/bwt_sa (bwamem.c:140-188,309), mem_chain2aln/ksw_extend2
 * (bwamem.c:658-812, ksw.c:416) and bwa_gen_cigar2/ksw_global2 (bwa.c:148, ksw.c:540) once per read.
 * Here each is ONE call per batch; the work runs in hand-written sm_90a kernels.  Plain pointers and
 * sizes only.  Every function returns 0 on success and a non-zero CUDA/driver error otherwise; there
 * is no CPU implementation behind them in the product library.
 *
 * Host-visible result buffers are owned by the batch object (pinned memory) and stay valid until the
 * next call of the same stage on that batch or bwag_batch_end().
 */
#ifndef BWA_B200_DEV_H
#define BWA_B200_DEV_H

#include "bwa_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct bwag_ctx bwag_ctx_t;     /* one per (GPU, index): FM-index + SA + pac resident in HBM */
typedef struct bwag_batch bwag_batch_t; /* the reads of one mem_process_seqs call, resident in HBM */

/* ---- index residency ------------------------------------------------------------------------ */
/* Size in bytes of the device index blob for this index (header + Occ/BWT blocks + SA + pac). */
size_t bwag_blob_bytes(const bwt_t *bwt, int64_t l_pac);
/* Fill a device blob (d_blob: device pointer, >= bwag_blob_bytes) from the host index
 * (bwt_restore_bwt/bwt_restore_sa layout, bwt.c:421-462; pac: bwa.c:308). */
int bwag_blob_fill(int device, void *d_blob, const bwt_t *bwt, int64_t l_pac, const uint8_t *pac);
/* Create a context over a filled blob (e.g. after an NCCL broadcast of the blob).  own_blob!=0: the
 * context frees the blob with cudaFree on destroy. */
bwag_ctx_t *bwag_ctx_from_blob(int device, void *d_blob, int own_blob);
/* Convenience: allocate + fill + create.  device < 0 -> current device. */
bwag_ctx_t *bwag_ctx_create(int device, const bwt_t *bwt, int64_t l_pac, const uint8_t *pac);
void bwag_ctx_destroy(bwag_ctx_t *ctx);
/* Replace the every-32nd-row suffix-array sample by a denser one computed on the device (values are
 * exact; only the number of LF steps per bwt_sa changes).  intv must be a power of two <= 32; 0 = choose from the device's
 * memory: the densest interval >= 2 whose sample takes at most an eighth of it. */
int bwag_ctx_densify_sa(bwag_ctx_t *ctx, int intv);

/* Short-string table: the bi-intervals (bwtintv_t x[0..2]) of ALL strings of 1..depth bases, so that a bwt_extend
 * (bwt.c:262-275) whose result is that short costs one 16-byte lookup instead of two Occ blocks (results unchanged;
 * two thirds of a read's extensions qualify at depth 12).  depth 0 = choose from the index size: floor(log4(BWT length)) - 2,
 * i.e. as deep as strings still occur a few dozen times (14 at 3 Gbp: 358 M entries, 5.7 GB); depth < 0 = remove the table;
 * depth <= 14.  Entries also carry the reference-equivalent Occ-block touch counts of the extensions they replace (forward chain,
 * last backward step), so the stage's occ_touches counter is what the reference would count, table or not. */
int bwag_ctx_build_ktab(bwag_ctx_t *ctx, int depth);

/* Verify the resident FM-index against the resident text: for rows first, first + stride, ... the BWT symbol must be the text base
 * before the row's suffix-array value, and the row's suffix must sort strictly before the next row's (stride 1: every row = a
 * complete check of .bwt/.sa against .pac; seconds for 3 Gbp).  out[4]: rows checked, BWT/text/SA mismatches, order violations,
 * suffix pairs equal over 8192 bases (undecided).  For indexes that did not come from `bwa index` (bwa_b200/index_build.py). */
int bwag_ctx_verify(bwag_ctx_t *ctx, uint64_t first, uint64_t stride, uint64_t out[4]);

/* Build the index files of a reference on the device (`bwa-b200 index`): the BWT of T = forward + reverse complement of
 * the l_pac bases in pac (2 bits per base, first base in the top bits: the .pac layout), with its Occ checkpoints every 128
 * symbols and the suffix array sampled every 32nd row, byte for byte what `bwa index` writes (bwtindex.c:150-172, 267-330).
 * Uses only the device memory cudaMemGetInfo reports free and fails (bwag_last_error says why) rather than oversubscribe.
 * BWA_B200_INDEX_BUCKET_BASES=k (1..6) sorts each bucket of suffixes with the same first k bases on its own, and
 * BWA_B200_INDEX_GROUP_SUFFIXES=m caps a group of buckets at m suffixes (tests: many buckets and groups on tiny references). */
typedef struct {
	uint64_t primary, seq_len, L2[5];
	uint64_t bwt_size;          /* u32 words of bwt[]: the .bwt file after its five u64 header words (primary, L2[1..4]) */
	uint32_t *bwt;
	uint64_t n_sa;              /* sa[r] = SA[32 r]; sa[0] = seq_len (the .sa file holds sa[1 ..]) */
	uint64_t *sa;
	uint64_t peak_device_bytes; /* most device memory the build held at once */
	uint64_t n_groups, max_group; /* groups of buckets sorted one after the other, and the most suffixes in one */
} bwag_built_index_t;
int bwag_index_build(int device, const uint8_t *pac, int64_t l_pac, bwag_built_index_t *out);
void bwag_built_index_free(bwag_built_index_t *x);

/* The steps of `bwa index` as commands of their own (bwtindex.c:64-208).  Each fails (bwag_last_error says why) rather than
 * oversubscribe the device memory cudaMemGetInfo reports free.
 * bwag_pac2bwt (`bwa-b200 pac2bwt`, `pac2bwtgen`): the BWT of the seq_len bases of pac (the .pac layout) taken as they are, by the
 * sorter of bwag_index_build: primary, L2 and the '$'-less BWT, 16 symbols per word (first in the top bits), no Occ checkpoints;
 * the raw .bwt of bwt_pac2bwt.  out->bwt is malloc'ed; the caller frees it. */
typedef struct {
	uint64_t primary, seq_len, L2[5];
	uint64_t bwt_size;          /* (seq_len + 15) / 16 words */
	uint32_t *bwt;
	uint64_t peak_device_bytes;
} bwag_raw_bwt_t;
int bwag_pac2bwt(int device, const uint8_t *pac, uint64_t seq_len, bwag_raw_bwt_t *out);
/* bwag_bwtupdate (`bwa-b200 bwtupdate`): the (seq_len + 15) / 16 raw words with the Occ checkpoints interleaved as
 * bwt_bwtupdate_core does (bwtindex.c:150-172): (seq_len + 15) / 16 + ((seq_len + 127) / 128 + 1) * 8 words into out */
int bwag_bwtupdate(int device, const uint32_t *raw, uint64_t seq_len, uint32_t *out, uint64_t *peak_device_bytes);
/* bwag_bwt2sa (`bwa-b200 bwt2sa`): the suffix array sampled every intv-th row (intv a power of two) from an updated BWT alone
 * (bwt_cal_sa, bwt.c:62-84): sa[r] = SA[r intv] for r < (seq_len + intv) / intv, sa[0] = seq_len.  Ranks the cycle of the LF
 * mapping in parallel from rulers every `stride` rows (BWA_B200_BWT2SA_STRIDE forces it); fails if LF is not one cycle of
 * seq_len + 1 rows, i.e. if bwt is not the BWT of any text. */
typedef struct { uint64_t stride, n_rulers, peak_device_bytes; } bwag_bwt2sa_stats_t;
int bwag_bwt2sa(int device, const bwt_t *bwt, int intv, uint64_t *sa, bwag_bwt2sa_stats_t *st);

/* Residency across processes (SURVEY.md 8-f3; the reference's counterpart is `bwa shm`, bwashm.c:16-122, which parks the index
 * in POSIX shared memory so that later `bwa mem` runs skip the load).  Device memory lives and dies with its process, so here a
 * process that keeps the index resident (`bwa-b200 shm idxbase`) EXPORTS it -- CUDA IPC handles of the blob, the dense suffix-array
 * sample and the short-string table, written to `path` -- and any other process on the same GPU IMPORTS it: a context over the
 * exporter's memory, ready in milliseconds, nothing read from the index files and nothing uploaded.  bwag_ctx_import returns NULL
 * (bwag_last_error says why) if the file is missing or stale (exporter gone, other device, other index size). */
int bwag_ctx_export(bwag_ctx_t *ctx, const char *path);
bwag_ctx_t *bwag_ctx_import(const char *path, int64_t l_pac);
void bwag_ctx_unexport(const char *path);   /* remove what bwag_ctx_export left behind (the exporter calls it before it exits) */

/* on != 0: batches begun from now on run the first formulation of the extension / global-alignment row sweeps and do no
 * short-string table lookups (same results, the configuration measured in round 1); 0: the defaults again.  The host's
 * start-up self-check compares the two on a few hundred reads drawn from the reference and stays on the baseline if
 * they ever disagree. */
void bwag_ctx_baseline(bwag_ctx_t *ctx, int on);
int bwag_is_emulator(void);   /* 0: CUDA device; 1: the CPU SIMT emulator of the tests; 2: the CPU oracle stages (tests) */
const char *bwag_last_error(void);

/* Page-locked host memory for buffers that are handed to the stage calls (reads, extension work, tasks):
 * copies from such memory are DMA transfers instead of staged driver copies.  Plain malloc memory works too. */
void *bwag_host_alloc(size_t bytes);
void bwag_host_free(void *p);

/* ---- batch ------------------------------------------------------------------------------------ */
/* codes: concatenated reads, one byte per base, values 0..4 (bwamem.c:1087-1088); off[n_reads+1]. */
bwag_batch_t *bwag_batch_begin(bwag_ctx_t *ctx, int n_reads, const uint8_t *codes, const int64_t *off);
void bwag_batch_end(bwag_batch_t *b);

/* ---- stage 1: SMEM seeding + suffix-array lookup (replaces mem_collect_intv + bwt_sa) --------- */
typedef struct {
	int min_seed_len;        /* opt->min_seed_len */
	int split_len;           /* (int)(min_seed_len*split_factor+.499)  bwamem.c:144 */
	int split_width;         /* opt->split_width */
	int max_occ;             /* opt->max_occ */
	uint64_t max_mem_intv;   /* opt->max_mem_intv */
} bwag_seed_par_t;

typedef struct {
	const int64_t *intv_beg;   /* [n_reads] first interval of each read in intv[] */
	const int32_t *intv_n;     /* [n_reads] number of intervals of each read */
	const bwtintv_t *intv;     /* per read: sorted by info, exactly smem_aux_t.mem after bwamem.c:187 */
	const int64_t *seed_beg;   /* [n_intv] first seed of each interval in rbeg[]; it has min(x[2], max_occ) seeds */
	const int64_t *rbeg;       /* bwt_sa(x[0]+k) for k = 0, step, 2*step ... (bwamem.c:304-309) */
	int64_t n_intv, n_seeds;   /* pool sizes (reads may sit in the pools in any order) */
} bwag_seeds_t;

int bwag_seed(bwag_batch_t *b, const bwag_seed_par_t *par, bwag_seeds_t *out);   /* out == NULL: keep the results in HBM only */

/* ---- SMEM listing of `bwa fastmap` (replaces the smem_next loop of main_fastmap, fastmap.c:443-475) ------------------------
 * Per read: every SMEM of every bwt_smem1a call in the reference's order (bwamem_extra.c:86-96, bwt.c:289-351), those at least
 * min_len long (compared as the reference does, unsigned: min_len < 0 lists nothing), each as its EM line of fastmap.c:457-473
 * ("EM\tbeg\tend\tx[2]", then "\tname:+pos" for each of the x[2] occurrences if x[2] <= (uint64_t)max_iwidth, else "\t*\n";
 * then "\n").  The SQ and "//" lines are the caller's.  Needs bwag_ctx_set_contigs (the contig names).  Reads of 2^23 bases or
 * more are refused (bwag_last_error names the first).  BWAG_UNSUPPORTED from the CPU oracle of the tests. */
typedef struct {
	int min_len;             /* -l */
	int min_intv;            /* -i (values below 1 act as 1, bwt.c:297) */
	uint64_t max_intv;       /* -I (0: off) */
	int max_iwidth;          /* -w */
} bwag_fastmap_par_t;
typedef struct {
	const char *text;        /* the EM lines of all reads, in read order */
	const int64_t *off;      /* [n_reads+1]: read r's lines are text[off[r], off[r+1]) */
} bwag_fastmap_t;
int bwag_fastmap(bwag_batch_t *b, const bwag_fastmap_par_t *par, bwag_fastmap_t *out);

/* ---- longest-match histogram of `bwa maxk` (replaces the smem_next loop of main_maxk, maxk.c:34-55) ----------------------------
 * bwag_ctx_create_occ: a context over an updated .bwt alone (bwt_restore_bwt): the Occ blocks, no suffix array, no text; NULL
 * (bwag_last_error says why) without a device.  bwag_maxk: per base of each of the batch's sequences, the longest match of the
 * reference's chain of bwt_smem1a calls (min_intv as given, max_intv 0) that covers it, capped at 255 (0 for N and for bases no
 * match covers); hist[v] += the number of bases of value v.  window > 0: each sequence is cut into windows of that many bases
 * that run in parallel, which gives the reference's bytes only when each of the four bases occurs at least min_intv times in the
 * BWT (L2[c+1] - L2[c] >= min_intv; the caller checks); window <= 0: one window per sequence, the reference's chain as it runs.
 * BWAG_UNSUPPORTED from the CPU oracle of the tests. */
typedef struct {
	int64_t window, n_windows;   /* the window used (whole-sequence windows: the longest sequence) and the batch's windows */
	int list_cap, n_repeat;      /* interval-list entries per lane, and the runs repeated because a list outgrew them */
	double ms_kernel, ms_hist;   /* CUDA-event time of the search (all runs) and of the binning */
	double max_window_ms;        /* the longest time one lane spent on one window (device clock) */
	uint64_t occ_touches;        /* Occ blocks touched as the reference counts them (bwt.c:194-197) */
} bwag_maxk_stats_t;
bwag_ctx_t *bwag_ctx_create_occ(int device, const bwt_t *bwt);
int bwag_maxk(bwag_batch_t *b, int min_intv, int64_t window, uint64_t hist[256], bwag_maxk_stats_t *st);

/* ---- BWA-backtrack search of `bwa aln` (replaces bwa_cal_sa_reg_gap + bwt_match_gap, bwtaln.c:83-126, bwtgap.c:109-264) -------
 * The batch's codes are the searched bases of each read in input order (after barcode removal and quality trimming).  Per read:
 * the widths of the reversed read (and of its seed), then the bounded-difference backtracking search with the reference's
 * priority queue, top-2 stop, duplicate check and width shadowing; its hits in the order the reference appends them.  Reads of
 * 65536 bases or more are refused.  BWAG_UNSUPPORTED from the CPU oracle of the tests. */
#define BWAG_ALN_GAPE    0x01   /* the mode bits of gap_opt_t that the search reads (bwtaln.h:94-98) */
#define BWAG_ALN_LOGGAP  0x04
#define BWAG_ALN_NONSTOP 0x10
typedef struct {
	int s_mm, s_gapo, s_gape;    /* -M -O -E (non-negative) */
	int mode;                    /* BWAG_ALN_* bits */
	int indel_end_skip, max_del_occ, max_entries;   /* -i -d -m */
	int max_gapo;                /* -o clamped to the max_diff of the longest read of the reference's 262144-read group (bwtaln.c:91-94) */
	int max_gape, max_seed_diff, seed_len, max_top2;   /* -e -k -l -R */
	const int8_t *max_diff;      /* [n_reads] -n, or bwa_cal_maxdiff of the read's length (host libm) */
} bwag_aln_par_t;
/* one hit in the .sai layout (bwt_aln1_t on x86-64, bwtaln.h:43-46): bits = n_mm | n_gapo << 8 | n_gape << 16 | score << 24 |
 * n_ins << 44 | n_del << 54, then the suffix-array interval [k, l] */
typedef struct { uint64_t bits, k, l; } bwag_aln1_t;
typedef struct {
	const int32_t *n_aln;        /* [n_reads] */
	const int64_t *off;          /* [n_reads+1]: read r's hits are aln[off[r], off[r+1]) */
	const bwag_aln1_t *aln;
	int64_t n_tier2;             /* reads whose queue outgrew the small per-lane arena and were searched again with a large one */
} bwag_aln_t;
int bwag_aln(bwag_batch_t *b, const bwag_aln_par_t *par, bwag_aln_t *out);

/* ---- stage 2: chain -> alignment regions (replaces the mem_chain2aln loop + ksw_extend2) ------ */
typedef struct {
	int a, b, o_del, e_del, o_ins, e_ins, w, zdrop, pen_clip5, pen_clip3;
	int8_t mat[25];
} bwag_sw_par_t;

#define BWAG_UNSUPPORTED 77           /* returned by a stage an implementation does not provide */
#define BWAG_DECLINED    78           /* returned by a stage that does not run in the context's current mode (stage 4 while bwag_ctx_baseline is on) */
#define BWAG_XSEED_ZEROKEY 0x80000000u   /* the seed's sort key (score<<32|index) is 0, see bwamem.c:720 */
typedef struct { int64_t rbeg; int32_t qbeg; uint32_t len; } bwag_xseed_t;  /* seeds of a chain in ks_introsort_64 order (bwamem.c:688-691) */
typedef struct { int64_t rmax0, rmax1; int32_t seed_off, n_seeds; } bwag_xchain_t; /* rmax after bns_fetch_seq clamping (bwamem.c:668-685) */
typedef struct { int64_t rb, re; int32_t qb, qe, score, truesc, w, seedcov, seedlen0, chain; } bwag_xreg_t;

typedef struct {
	const int32_t *n_regs;     /* [n_reads] */
	const bwag_xreg_t *regs;   /* regs of read r: regs[reg_base(r) ... + n_regs[r]), reg_base(r) = chains[chain_off[r]].seed_off */
} bwag_regs_t;

int bwag_extend(bwag_batch_t *b, const bwag_sw_par_t *par,
                const int32_t *chain_off /* [n_reads+1] */, const bwag_xchain_t *chains,
                int64_t n_seeds, const bwag_xseed_t *seeds, bwag_regs_t *out);

/* ---- stages 2a+2: chaining on the device, fused with the extension (replaces mem_chain's chaining loop,
 * mem_chain_flt and the mem_chain2aln loop: bwamem.c:299-334, 353-411, 658-812).  Requires a preceding
 * bwag_seed(b, par, NULL) on the same batch (results stay in HBM).  Valid for reads for which
 * mem_flt_chained_seeds is inactive (bwamem.c:626-628); the caller checks that. ------------------------ */
typedef struct {
	int w, max_chain_gap, max_occ, min_seed_len, min_chain_weight, max_chain_extend;
	float mask_level, drop_ratio;
} bwag_chain_par_t;
typedef struct { int n_seqs; const int64_t *offset; const int32_t *len; const uint8_t *is_alt; } bwag_contigs_t;  /* bntann1_t columns (bntseq.h:41-50) */
typedef struct { bwag_xreg_t r; int32_t rid; float frac_rep; } bwag_creg_t;   /* region + contig and repeat fraction of its chain */
typedef struct {
	const int32_t *n_regs;     /* [n_reads] */
	const int64_t *reg_beg;    /* [n_reads] first region of each read in regs[] */
	const bwag_creg_t *regs;
} bwag_cregs_t;
int bwag_chain_extend(bwag_batch_t *b, const bwag_chain_par_t *cp, const bwag_sw_par_t *sp, const bwag_contigs_t *ctg, bwag_cregs_t *out);   /* out == NULL: the regions stay in HBM (for bwag_tail_regs) */

/* The raw regions of a selection of reads after bwag_chain_extend(b, ..., NULL) left them in HBM: what a caller needs to run its own
 * post-processing for the reads stage 4 hands back without aligning them again.  out->n_regs / reg_beg are indexed by position in sel[]. */
int bwag_fetch_cregs(bwag_batch_t *b, int n_sel, const int32_t *sel, bwag_cregs_t *out);

/* ---- stage 3: banded global alignment -> CIGAR/NM/MD (replaces bwa_gen_cigar2 + ksw_global2) -- */
#define BWAG_G_REG2ALN 0   /* the do-while of mem_reg2aln (bwamem.c:1144-1152): up to 3 band doublings, CIGAR+NM+MD */
#define BWAG_G_SCORE   1   /* one bwa_gen_cigar2 call, score only (mem_patch_reg, bwamem.c:454) */
typedef struct { int64_t rb, re; int32_t read, qb, qe, w, truesc, mode; } bwag_gtask_t;
typedef struct { int32_t score, n_cigar, NM, l_md; int64_t cigar_off, md_off; } bwag_gres_t;

typedef struct {
	const bwag_gres_t *res;    /* [n_tasks] */
	const uint32_t *cigar;     /* pool; task t: cigar[res[t].cigar_off ... + n_cigar) , len<<4|op */
	const char *md;            /* pool; task t: md[res[t].md_off ... + l_md), NUL-terminated (l_md counts the NUL) */
} bwag_galn_t;

int bwag_global(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, const bwag_gtask_t *tasks, bwag_galn_t *out);

/* ---- K6: batched local Smith-Waterman with start recovery (replaces ksw_align2, ksw.c:379-401, in mem_matesw
 * bwamem_pair.c:137-206 and mem_seed_sw bwamem.c:597-622).  Same numbers as the reference's striped SSE2 kernels (score, te, qe,
 * score2, te2, tb, qb); xtra as ksw.h:29-33.  The query of a task is a stretch of the batch's reads (optionally
 * reverse-complemented) or bytes of `pool`; the target a window of the reference (doubled coordinates) or bytes of `pool`. ---- */
#define BWAG_SW_XBYTE  0x10000u
#define BWAG_SW_XSTOP  0x20000u
#define BWAG_SW_XSUBO  0x40000u
#define BWAG_SW_XSTART 0x80000u
#define BWAG_SWF_QREV  1    /* query = reverse complement of the given stretch */
#define BWAG_SWF_TREF  2    /* target = reference positions [t_beg, t_beg + tlen) */
#define BWAG_SWF_QREAD 4    /* query = batch codes [q_beg, q_beg + qlen) (offset into the batch's concatenated reads) */
typedef struct { int64_t t_beg, q_beg; int32_t tlen, qlen; uint32_t xtra; int32_t flags; } bwag_swtask_t;
typedef struct { int32_t score, te, qe, score2, te2, tb, qb; } bwag_swres_t;
/* pool (host pointer, pool_bytes) may be NULL when every task reads the batch and the reference; results: pinned, valid until the
 * next call on this batch */
int bwag_localsw(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, const bwag_swtask_t *tasks, const uint8_t *pool, size_t pool_bytes, const bwag_swres_t **out);

/* ---- stage 4: the reference's per-read work AFTER the extension, on the device, for the reads whose post-processing is
 * "simple" (bwag_tail.cu): mem_sort_dedup_patch, one CIGAR request per region, mem_pestat's per-pair candidate
 * (bwag_tail_regs); mem_mark_primary_se, mem_approx_mapq_se, the mate-rescue trigger test, mem_pair, mem_sam_pe's pair
 * logic, mem_reg2aln and the SAM record (bwag_tail_sam).  Reads that leave the simple case come back flagged and are
 * aligned by the caller's host-side post-processing instead.  Both need bwag_ctx_set_contigs once per context and a
 * preceding bwag_chain_extend(b, ..., NULL) (regions stay in HBM).  BWAG_UNSUPPORTED from the CPU oracle of the tests. ---- */
int bwag_ctx_set_contigs(bwag_ctx_t *ctx, int n_seqs, const int64_t *offset, const int32_t *len, const uint8_t *is_alt, const char *const *names);
/* pe_is (PE only, else NULL is stored): [n_reads/2] per-pair insert-size candidates, pinned; cflag: [n_reads], non-zero =
 * the read left the simple path already here (too many regions, ALT contig, a region merge that needs an alignment) */
int bwag_tail_regs(bwag_batch_t *b, const mem_opt_t *opt, const bwag_sw_par_t *sp, const uint64_t **pe_is, const uint8_t **cflag);
#define BWAG_REC_TEXT    1u    /* the record's text is in the pool */
#define BWAG_REC_QREV    2u    /* the quality string goes in reversed */
#define BWAG_REC_COMPLEX 4u    /* no text: the read needs the host-side post-processing (reason in bits 8-15) */
enum { BWAG_CX_MANY = 1, BWAG_CX_ALT, BWAG_CX_PATCH, BWAG_CX_CAP, BWAG_CX_RESCUE, BWAG_CX_PAIR, BWAG_CX_XA, BWAG_CX_MULTI, BWAG_CX_CIGAR, BWAG_CX_LONG };
/* one read's record: name + text[off, off+len_a) + QUAL + text[off+len_a, off+len_a+len_b) + [\t comment] + \n */
typedef struct { int64_t off; int32_t len_a, len_b; uint32_t flags; int32_t pad; } bwag_samrec_t;
typedef struct { const bwag_samrec_t *rec; const char *text; int64_t n_text, n_complex; } bwag_sam_t;
/* pair_tab[d]: the insert-size term of a pair's score for distances pes[d].low..pes[d].high (bwamem_pair.c:266), NULL = orientation
 * unusable; log_tab: log(i) for i < 4096; both from the host's libm so that the integer decisions are the host's */
int bwag_tail_sam(bwag_batch_t *b, const mem_opt_t *opt, const mem_pestat_t pes[4], const double *const pair_tab[4], const double *log_tab,
                  int64_t n_processed, const char *rg_id, bwag_sam_t *out);

/* ---- single-end SAM of `bwa samse` (replaces bwa_cal_pac_pos, bwa_refine_gapped and bwa_print_sam1 with no mate,
 * bwase.c:112-499) -------------------------------------------------------------------------------------------------------------
 * The batch's codes are the whole reads after barcode removal (0..5, as nst_nt4_table gives them).  The caller has chosen each
 * read's hit and its XA candidates (bwa_aln2seq_core, host, in read order: its random draws are serial) and its mapping quality.
 * Per read, on the device: the positions of the chosen hit and of its candidates (bwa_sa2pos through the resident suffix array),
 * the candidates that stay in XA, the banded global alignment of every gapped hit (ksw_global with the fix-ups of
 * bwa_refine_gapped_core), MD and NM (bwa_cal_md1), the trimming correction (bwa_correct_trimmed) and the SAM record in the
 * stage-4 layout (bwag_samrec_t; part B holds no trailing newline).  Needs bwag_ctx_set_contigs and bwag_ctx_set_ambs.
 * BWAG_UNSUPPORTED from the CPU oracle of the tests. */
#define BWAG_SE_COMPREAD 0x02   /* gap_opt_t mode bit: NM (else CM) and a complemented rseq */
typedef struct {
	uint64_t sa;                 /* the chosen suffix-array row */
	int32_t len;                 /* bases searched (after quality trimming); the whole read is in the batch's codes */
	int32_t clip_len;            /* XC:i: is printed when it is below the read's length */
	int32_t ref_shift;           /* n_del - n_ins of the chosen hit */
	uint8_t type, n_mm, n_gapo, n_gape;   /* 0 no match, 1 unique, 2 repeat; the chosen hit's differences */
	uint32_t c1, c2;             /* X0 and X1: best and second-best hit counts (28 bits each, as bwa_seq_t keeps them) */
	uint8_t mapq, l_bc, pad[2];
	int32_t n_multi;             /* XA candidates: par->multi[multi_beg, multi_beg + n_multi), in bwa_aln2seq_core's order */
	int64_t multi_beg;
	int64_t bc_off;              /* the barcode: par->bc[bc_off, bc_off + l_bc) */
} bwag_se_read_t;
typedef struct { uint64_t sa; int32_t ref_shift; uint8_t gap, mm, pad[2]; } bwag_se_hit_t;   /* gap = n_gapo + n_gape (8 bits) */
typedef struct {
	int mode;                    /* BWAG_SE_COMPREAD */
	int max_top2;                /* X1 is printed when X0 <= max_top2 */
	const char *rg_id;           /* NULL or "": no RG tag */
	const bwag_se_read_t *reads; /* [n_reads] */
	const bwag_se_hit_t *multi; int64_t n_multi;
	const char *bc; int64_t l_bc;
} bwag_samse_par_t;
/* the holes of the reference (bns->ambs): bns_cnt_ambi counts the N bases under an alignment for XN and XT */
int bwag_ctx_set_ambs(bwag_ctx_t *ctx, int n_holes, const int64_t *offset, const int32_t *len);
/* *past_end: -1, or the first read of the batch whose gapped alignment window runs past the end of the forward strand (the
 * reference aborts on its assert there, bwase.c:180); the call then fails.  n_sa, n_glb: SA rows resolved, global alignments run. */
int bwag_samse(bwag_batch_t *b, const bwag_samse_par_t *par, bwag_sam_t *out, int *past_end, int64_t *n_sa, int64_t *n_glb);

/* ---- paired-end SAM of `bwa sampe` (bwape.c:260-711, with bwa_print_sam1 of a pair) --------------------------------------------
 * The host chooses the hits (serial random draws), infers the insert size, pairs and picks XA; the device resolves the suffix-array
 * rows, runs the mate rescue's alignments and writes the records.  BWAG_UNSUPPORTED from the CPU oracle of the tests.
 * bwag_pe_sa2pos: n_rows rows, resolved once through the resident suffix array, then bwa_sa2pos with the two reference lengths
 * ref_len[2k], ref_len[2k + 1] of row k into pos[2k], pos[2k + 1] ((uint64_t)-1: across the strand boundary) and strand[]. */
int bwag_pe_sa2pos(bwag_batch_t *b, int64_t n_rows, const uint64_t *rows, const int32_t *ref_len, int64_t *pos, uint8_t *strand);
/* the mate rescue's global alignment (bwa_sw_core, bwape.c:434): ksw_global, scores bwa_fill_scmat(1, 3), gaps 5/1, band 50, of
 * pool[q_beg, q_beg + qlen) against the forward reference [t_beg, t_beg + tlen); the raw CIGAR (len << 4 | op) at res[i].cig_off of
 * *cig.  Results pinned, valid until the next call on this batch. */
typedef struct { int64_t t_beg, q_beg; int32_t tlen, qlen; } bwag_pe_gtask_t;
typedef struct { int32_t score, n_cigar; int64_t cig_off; } bwag_pe_gres_t;
int bwag_pe_global(bwag_batch_t *b, int n_tasks, const bwag_pe_gtask_t *tasks, const uint8_t *pool, size_t pool_bytes, const bwag_pe_gres_t **res, const uint32_t **cig);
/* the pair's records.  reads[2i] and reads[2i + 1] are the two ends of pair i; their type 3 is a mate-rescued hit (BWA_TYPE_MATESW),
 * whose CIGAR (16-bit entries) the caller gives; the caller's positions are the final ones before the gapped refinement, and its XA
 * lists hold only the candidates kept (positions in mpos / mstrand). */
typedef struct {
	int64_t cig_off; int32_t n_cig;   /* type 3: par->cig[cig_off, cig_off + n_cig) */
	uint8_t flag;                     /* extra_flag: 0x1, 0x2 (proper pair), 0x40 / 0x80 */
	uint8_t seq_q;                    /* SM: the single-end mapping quality */
	uint8_t comp, pad;                /* comp: the read's rseq is complemented (COMPREAD of its own .sai) */
} bwag_pe_read_t;
typedef struct {
	int mode, max_top2;               /* mode: NM (COMPREAD) or CM, from .sai 2 as in the reference */
	int comp[2];                      /* per end: its rseq complemented (COMPREAD of that end's .sai) */
	const char *rg_id;
	const bwag_se_read_t *reads; const bwag_pe_read_t *pe;      /* [n_reads] */
	const int64_t *pos; const uint8_t *strand;                  /* [n_reads]; an unmapped read's strand is 0 */
	const bwag_se_hit_t *multi; const int64_t *mpos; const uint8_t *mstrand; int64_t n_multi;
	const uint32_t *cig; int64_t n_cig;
	const char *bc; int64_t l_bc;
} bwag_sampe_par_t;
/* past_end as bwag_samse; n_glb: gapped refinements run */
int bwag_sampe(bwag_batch_t *b, const bwag_sampe_par_t *par, bwag_sam_t *out, int *past_end, int64_t *n_glb);

/* ---- read-pair merging of `bwa pemerge` (bwa_pemerge and the printing loop, pemerge.c:59-215) ------------------------------------
 * No index is involved: the batch comes from a context made by bwag_ctx_create_bare (a stream and buffers, no index), and its "codes"
 * are the reads' raw sequence bytes, read 1 of pair i as read 2i and read 2 as read 2i + 1.  Per pair, on the device: the codes and
 * qualities, the local alignment of read 2's reverse complement against read 1 (K6: ksw_align with KSW_XSTART | KSW_XSUBO, scores
 * bwa_fill_scmat(5, 4), gaps 2/17), the reference's eight tests in its order, the merged read and the records print_bseq writes,
 * whole (names included), in pair order.  cnt[k]: pairs whose bwa_pemerge returned -k.  BWAG_UNSUPPORTED from the CPU oracle of the
 * tests. */
bwag_ctx_t *bwag_ctx_create_bare(int device);   /* device < 0: the current one; NULL (bwag_last_error says why) without a device */
typedef struct {
	int T;                       /* minimum score: 5 x the minimum overlap (-T) */
	int q_thres;                 /* -Q */
	int q_def;                   /* the quality of every base of a read without qualities (20) */
	int flag;                    /* 1: print merged pairs, 2: unmerged ones */
	int merge;                   /* 0: try no pair (the reference with -t 0): every count 0, every pair printed as it came */
	const uint8_t *qual;         /* raw quality bytes at the offsets of the batch's reads (any bytes where has_qual is 0) */
	const uint8_t *has_qual;     /* [n_reads] the read has a quality string (a FASTQ read that is not empty) */
	const char *names;           /* the reads' names after trim_readno, back to back */
	const int64_t *name_off;     /* [n_reads + 1] */
} bwag_pemerge_par_t;
typedef struct { const char *text; int64_t n_text; int64_t cnt[9]; } bwag_pemerge_t;   /* text: pinned, valid until the next call on the batch */
int bwag_pemerge(bwag_batch_t *b, const bwag_pemerge_par_t *par, bwag_pemerge_t *out);

/* ---- work / time counters for the roofline ---------------------------------------------------- */
typedef struct {
	uint64_t occ_touches;      /* 64-byte Occ blocks touched by bwt_extend (1 or 2 per call, bwt.c:194-197) */
	uint64_t sa_touches;       /* 64-byte blocks touched by LF steps in bwt_sa */
	uint64_t sa_touches_algo;  /* reserved (LF steps the files' sa_intv=32 sample would have needed); not filled yet, reads 0 */
	uint64_t ext_cells;        /* sum over ksw_extend2 rows of (end-beg) */
	uint64_t glb_cells;        /* sum over ksw_global2 rows of (end-beg) */
	double ms_smem, ms_sa, ms_extend, ms_global;   /* CUDA-event time of the kernels, accumulated */
	double ms_h2d, ms_d2h;
	uint64_t n_launch;         /* kernels launched */
	uint64_t h2d_bytes, d2h_bytes;   /* bytes copied host->device / device->host by the stage calls */
	double ms_chain;           /* CUDA-event time of the chaining kernel */
	double ms_tail;            /* CUDA-event time of the stage-4 kernels (de-duplication/requests, pairing/SAM records) */
	uint64_t tail_reads, tail_complex;   /* reads that went through stage 4 / that it handed back to the host-side post-processing */
	double ms_localsw;         /* CUDA-event time of K6 (local Smith-Waterman: mate rescue) */
	uint64_t sw_tasks;         /* local alignments K6 computed */
} bwag_stats_t;
void bwag_stats_get(bwag_ctx_t *ctx, bwag_stats_t *s);
void bwag_stats_reset(bwag_ctx_t *ctx);
/* builds with -DBWAG_K3_CLOCKS only (else returns -1): copies the chaining kernel's cycle histograms (BWAG_K3CLK_WORDS words) to out,
 * then clears them if reset.  Words 4t..4t+3, t = seeds per read (0..64, 65: more): reads, cycles of the chaining loop, of
 * mem_chain_flt, of chain_emit; words 264+c, c = chains per read (0..32, 33: more): reads. */
#define BWAG_K3CLK_WORDS (4 * 66 + 34)
int bwag_k3_clocks(uint64_t *out, int reset);
/* builds with -DBWAG_K1_CLOCKS only (else returns -1): copies the seeding kernel k_smem_c's counters (BWAG_K1CLK_WORDS words) to out,
 * then clears them if reset.  Summed over lanes: loop iterations (a warp's count times 32), iterations that extended forward by a
 * table lookup / by Occ blocks, backward a list candidate / a mask candidate, those of them that looked up a pair (forward, backward),
 * clock64() cycles spent handing a finished read over and fetching the next, reads fetched.  Then the CUDA-event time of K1f
 * (k_smem_fwd) and of k_smem_c in nanoseconds, and the seeding calls. */
enum { BWAG_K1CLK_ITERS, BWAG_K1CLK_FWD_TAB, BWAG_K1CLK_FWD_OCC, BWAG_K1CLK_BWD_LIST, BWAG_K1CLK_BWD_MASK, BWAG_K1CLK_PAIR_FWD,
       BWAG_K1CLK_PAIR_BWD, BWAG_K1CLK_TURN_CYC, BWAG_K1CLK_READS, BWAG_K1CLK_LANE_WORDS,
       BWAG_K1CLK_K1F_NS = BWAG_K1CLK_LANE_WORDS, BWAG_K1CLK_K1C_NS, BWAG_K1CLK_CALLS, BWAG_K1CLK_WORDS };
int bwag_k1_clocks(uint64_t *out, int reset);

#ifdef __cplusplus
}
#endif
#endif
