/* bb_host.h -- internal interfaces of the host glue of libbwa_b200 (C).
 *
 * The host side keeps what the reference keeps per read around its kernels: chaining and chain
 * filtering, region de-duplication, primary marking, MAPQ, pairing and SAM text.  Everything that
 * walks the FM-index or fills a DP matrix is behind include/bwa_b200_dev.h (CUDA).
 */
#ifndef BB_HOST_H
#define BB_HOST_H

#include "bwa_b200.h"
#include "bwa_b200_dev.h"
#include "bb_util.h"
#include "bb_str.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- sequence / coordinate helpers (bb_index.c) ---- */
extern unsigned char bb_nt4_table[256];
static inline int bb_pac_get(const uint8_t *pac, int64_t k) { return pac[k >> 2] >> ((~k & 3) << 1) & 3; }
static inline int64_t bb_depos(const bntseq_t *bns, int64_t pos, int *is_rev)
{
	*is_rev = pos >= bns->l_pac;
	return *is_rev ? (bns->l_pac << 1) - 1 - pos : pos;
}
int bb_pos2rid(const bntseq_t *bns, int64_t pos_f);
int bb_intv2rid(const bntseq_t *bns, int64_t rb, int64_t re);
uint8_t *bb_get_seq(int64_t l_pac, const uint8_t *pac, int64_t beg, int64_t end, int64_t *len);
uint8_t *bb_fetch_seq(const bntseq_t *bns, const uint8_t *pac, int64_t *beg, int64_t mid, int64_t *end, int *rid);
void bb_clamp_to_contig(const bntseq_t *bns, int64_t *beg, int64_t mid, int64_t *end, int *rid);

/* ---- device residency keyed by host index pointer (bb_process.c) ---- */
bwag_ctx_t *bb_device_attach(const bwt_t *bwt, const bntseq_t *bns, const uint8_t *pac);
void bb_device_release(const bwt_t *bwt);
void bb_device_adopt(const bwt_t *bwt, bwag_ctx_t *ctx);
void bb_device_adopt2(const bwt_t *bwt, const bntseq_t *bns, const uint8_t *pac, bwag_ctx_t *ctx);

/* ---- chaining (bb_chain.c) ---- */
typedef struct { int64_t rbeg; int32_t qbeg, len; int score; } bb_seed_t;
typedef struct {
	int n, m, first, rid;
	uint32_t w, kept, is_alt;
	float frac_rep;
	int64_t pos;
	bb_seed_t *seeds;
} bb_chain_t;
typedef BB_VEC(bb_chain_t) bb_chain_v;

typedef struct bb_chainer bb_chainer_t; /* per-thread scratch: ordered map + seed arena */
bb_chainer_t *bb_chainer_new(void);
void bb_chainer_free(bb_chainer_t *c);
/* Chains of one read from its sorted SA intervals and their suffix-array positions.  Output chains
 * (and their seed arrays) live in the chainer's arena until the next call. */
void bb_chain_build(bb_chainer_t *c, const mem_opt_t *opt, const bntseq_t *bns, int l_query,
                    int n_intv, const bwtintv_t *intv, const int64_t *seed_beg, const int64_t *rbeg, bb_chain_v *out);
int bb_chain_weight(const bb_chain_t *c);
int bb_chain_filter(const mem_opt_t *opt, int n, bb_chain_t *a);
void bb_chain_seed_sw(const mem_opt_t *opt, const bntseq_t *bns, const uint8_t *pac, int l_query, const uint8_t *query, int n, bb_chain_t *a);
int bb_cal_max_gap(const mem_opt_t *opt, int qlen);

/* ---- local Smith-Waterman used by mate rescue and seed filtering (bb_localsw.c) ---- */
#define BB_SW_XBYTE  0x10000
#define BB_SW_XSTOP  0x20000
#define BB_SW_XSUBO  0x40000
#define BB_SW_XSTART 0x80000
typedef struct { int score, te, qe, score2, te2, tb, qb; } bb_swr_t;
bb_swr_t bb_local_sw(int qlen, uint8_t *query, int tlen, uint8_t *target, const int8_t *mat, int o_del, int e_del, int o_ins, int e_ins, int xtra);

/* ---- global-alignment service with memoisation (bb_process.c) ---- */
typedef struct {
	int64_t rb, re;
	int32_t qb, qe, w, truesc, mode;
	int32_t score, n_cigar, NM, l_md;
	uint32_t *cigar; /* malloc'd: n_cigar ops followed by the MD string */
	int done;
} bb_galn_t;
typedef BB_VEC(bb_galn_t) bb_galn_v;
/* Look up / request an alignment for a read.  Returns the cached entry, or NULL after recording the
 * request (the caller then abandons this read's current pass; it is re-run after the next device round). */
typedef struct {
	bb_galn_v memo;
	int pending;     /* requests recorded in this pass */
	int in_arena;    /* memo.a lives in the batch's bump arena (nothing to free) */
	bb_galn_t inl;   /* storage of the first entry: most reads need exactly one alignment */
} bb_gcache_t;
const bb_galn_t *bb_gcache_get(bb_gcache_t *gc, int mode, int qb, int qe, int64_t rb, int64_t re, int w, int truesc);

/* a region array whose storage belongs to a batch-wide block: mem_alnreg_v.m carries this flag and the real
 * capacity equals n; whoever needs to grow it must move it to the heap first (bb_regs_make_room) */
#define BB_BORROWED ((size_t)1 << 62)
void bb_regs_make_room(mem_alnreg_v *v);

/* ---- regions (bb_reg.c) ---- */
int bb_sort_dedup_patch(const mem_opt_t *opt, const bntseq_t *bns, bb_gcache_t *gc, int l_query, int n, mem_alnreg_t *a);
int bb_mark_primary_se(const mem_opt_t *opt, int n, mem_alnreg_t *a, int64_t id);
void bb_reorder_primary5(int T, mem_alnreg_v *a);
int bb_approx_mapq_se(const mem_opt_t *opt, const mem_alnreg_t *a);

/* ---- SAM (bb_sam.c) ---- */
typedef struct {
	const mem_opt_t *opt;
	const bntseq_t *bns;
	const uint8_t *pac;
	bb_gcache_t *gc;   /* of the read being formatted */
	int dry;           /* pass that only discovers which alignments are needed: skip text */
	/* optional bump area (the caller's stack) for the CIGAR+MD copies bb_reg2aln hands out: most records need ~40 bytes
	 * for a few hundred nanoseconds, not a malloc/free pair.  bb_cigar_free() releases only what did not fit. */
	uint32_t *scratch;
	int scratch_cap, scratch_used;   /* in 32-bit words */
} bb_samctx_t;
static inline void bb_cigar_free(const bb_samctx_t *sc, uint32_t *cigar)
{
	if (cigar && !(sc->scratch && cigar >= sc->scratch && cigar < sc->scratch + sc->scratch_cap)) free(cigar);
}
int bb_reg2aln_band(const mem_opt_t *opt, const mem_alnreg_t *ar);
mem_aln_t bb_reg2aln(bb_samctx_t *sc, int l_query, const char *query, const mem_alnreg_t *ar);
void bb_encode_bases(char *seq, uint8_t *dst, int n);   /* ASCII (or codes) -> codes 0..5 in place, 0..4 into dst */
void bb_codes_to_text(char *dst, const uint8_t *codes, int n, int rev);   /* SEQ column: "ACGTN" / reverse complement */
void bb_copy_text(char *dst, const char *src, int n, int rev);             /* QUAL column: copy / reverse */
void bb_aln2sam(const mem_opt_t *opt, const bntseq_t *bns, bb_str_t *str, bseq1_t *s, int n, const mem_aln_t *list, int which, const mem_aln_t *m_);
void bb_reg2sam(bb_samctx_t *sc, bseq1_t *s, mem_alnreg_v *a, int extra_flag, const mem_aln_t *m);
char **bb_gen_alt(bb_samctx_t *sc, const mem_alnreg_v *a, int l_query, const char *query);

int bb_selfcheck_status(void);   /* start-up self-check of the device kernels: 0 not run, 1 passed, 2 differed (running on the baseline kernels) */

/* ---- paired-end (bb_pair.c) ---- */
uint64_t bb_pestat_pair(const mem_opt_t *opt, int64_t l_pac, const mem_alnreg_v *r0, const mem_alnreg_v *r1);
void bb_pestat_from_pairs(const mem_opt_t *opt, long n_pairs, const uint64_t *v, mem_pestat_t pes[4]);
/* Mate-rescue alignments come from the device (K6, bwag_localsw) the way global alignments do: a per-pair cache; a miss records
 * a request and the pair's rescue pass is abandoned (return -1) and replayed after the device has served the batch's requests. */
typedef struct { int64_t rb, re; int32_t which, is_rev, done; bb_swr_t res; } bb_swent_t;   /* which: the read of the pair that is the query */
typedef struct { BB_VEC(bb_swent_t) v; int pending, probe; } bb_swcache_t;   /* probe: the pass only collects the requests of every anchor (nothing is applied) */
int bb_matesw(const mem_opt_t *opt, const bntseq_t *bns, const uint8_t *pac, const mem_pestat_t pes[4], const mem_alnreg_t *a, int l_ms, const uint8_t *ms, mem_alnreg_v *ma, bb_swcache_t *swc, int which);
int bb_sam_pe(bb_samctx_t sc[2], const mem_pestat_t pes[4], uint64_t id, bseq1_t s[2], mem_alnreg_v a[2], int rescue_done);
int bb_rescue_pe(const mem_opt_t *opt, const bntseq_t *bns, const uint8_t *pac, const mem_pestat_t pes[4], bseq1_t s[2], mem_alnreg_v a[2], bb_swcache_t *swc);   /* swc == NULL: align on the host (SSE2) */

/* ---- an index that stays on the GPU between runs (bb_resident.c) ---- */
bwaidx_t *bb_idx_from_resident(const char *prefix);
int bb_shm_main(int argc, char *argv[]);

/* ---- FASTA/FASTQ input (bb_fastq.c) ---- */
typedef struct bb_fq bb_fq_t;
bb_fq_t *bb_fq_open(const char *fn);
bb_fq_t *bb_fq_open_range(const char *fn, int64_t beg, int64_t end);
void bb_fq_close(bb_fq_t *f);
int bb_fq_read1(bb_fq_t *f, const bb_str_t **name, const bb_str_t **comment, const bb_str_t **seq);
const bb_str_t *bb_fq_qual(const bb_fq_t *f);

/* ---- `bwa-b200 index` (bb_index_build.c) ---- */
int bb_index_main(int argc, char *argv[]);

/* ---- the .pac/.ann/.amb of a FASTA file, and whole-file writes (bb_pac.c) ---- */
typedef struct {
	int64_t l_pac;
	uint8_t *pac;
	size_t m_pac;              /* bytes allocated */
	BB_VEC(bntann1_t) anns;
	BB_VEC(bntamb1_t) ambs;
} bb_packed_t;
void bb_pack_add(bb_packed_t *P, const bb_str_t *name, const bb_str_t *comment, const bb_str_t *seq);
void bb_pack_add_revcomp(bb_packed_t *P);
int bb_pack_dump(const bb_packed_t *P, const char *prefix, const char *where);
void bb_pack_free(bb_packed_t *P);
int bb_write_whole(const char *fn, const void *a, size_t bytes, const void *b, size_t b_bytes, const char *where);
int bb_write_index_file(const char *prefix, const char *ext, const void *a, size_t bytes, const void *b, size_t b_bytes, const char *where);

/* ---- `bwa-b200 fa2pac`, `pac2bwt`, `pac2bwtgen`, `bwtupdate`, `bwt2sa` (bb_index_steps.c) ---- */
int bb_fa2pac_main(int argc, char *argv[]);
int bb_pac2bwt_main(int argc, char *argv[]);
int bb_pac2bwtgen_main(int argc, char *argv[]);
int bb_bwtupdate_main(int argc, char *argv[]);
int bb_bwt2sa_main(int argc, char *argv[]);
/* a .bwt file alone, raw or updated (bb_index.c): primary, L2, seq_len = L2[4], bwt_size and the words; no suffix array */
bwt_t *bb_bwt_restore(const char *fn);
/* (bb_index_steps.c) a .bwt file of a non-empty text, raw (updated = 0) or with its Occ checkpoints (updated = 1); NULL after a
 * message otherwise */
bwt_t *bb_read_bwt(const char *fn, int updated, const char *where);

/* ---- `bwa-b200 maxk` (bb_maxk.c) ---- */
int bb_maxk_main(int argc, char *argv[]);

/* ---- `bwa-b200 fastmap` (bb_fastmap.c) ---- */
int bb_fastmap_main(int argc, char *argv[]);

/* ---- `bwa-b200 aln` (bb_aln.c) ---- */
int bb_aln_main(int argc, char *argv[]);

/* ---- the reads of `aln` and `samse` (bb_seqio.c): bwa_read_seq, bwaseqio.c:151-221 ---- */
#define BB_MODE_COMPREAD 0x02      /* the mode bits of gap_opt_t (bwtaln.h:94-103) */
#define BB_MODE_CFY      0x08
#define BB_MODE_BAM      0x20
#define BB_MODE_IL13     0x200
#define BB_MAX_BCLEN     63        /* BWA_MAX_BCLEN */
#define BB_MIN_RDLEN     35        /* BWA_MIN_RDLEN: quality trimming stops here */
typedef struct {
	int n;
	int64_t *off;              /* [n+1] first base of each read in codes[] */
	uint8_t *codes;            /* keep == 0: the searched bases, 0..4; keep != 0: the whole read after the barcode, 0..5 (nst_nt4_table) */
	int32_t *len;              /* [n] bases searched (after quality trimming) */
	int max_len;               /* the most bases searched in one read */
	int64_t *name, *qual, *bc; /* keep != 0: [n] offsets into text (NUL-terminated strings); qual / bc -1: none */
	bb_str_t text;
} bb_reads_t;
/* gap_opt_t (bwtaln.h:105-115): the 64 bytes after "SAI\1" in a .sai file */
typedef struct {
	int32_t s_mm, s_gapo, s_gape;
	int32_t mode;                 /* bits 24-31: barcode length */
	int32_t indel_end_skip, max_del_occ, max_entries;
	float fnr;
	int32_t max_diff, max_gapo, max_gape;
	int32_t max_seed_diff, seed_len;
	int32_t n_threads;
	int32_t max_top2;
	int32_t trim_qual;
} aln_opt_t;
_Static_assert(sizeof(aln_opt_t) == 64, "gap_opt_t is 16 four-byte fields");
_Static_assert(offsetof(aln_opt_t, mode) == 12 && offsetof(aln_opt_t, fnr) == 28 && offsetof(aln_opt_t, max_diff) == 32, "gap_opt_t layout");
_Static_assert(offsetof(aln_opt_t, seed_len) == 48 && offsetof(aln_opt_t, n_threads) == 52 && offsetof(aln_opt_t, trim_qual) == 60, "gap_opt_t layout");
/* up to n_max reads (one group of the reference); NULL at the end of the input.  A read with max_len or more bases to search is
 * fatal (`who` names the command). */
bb_reads_t *bb_read_group(bb_fq_t *fq, int mode, int trim_qual, int n_max, int keep, int max_len, const char *who);
void bb_reads_free(bb_reads_t *g);

/* ---- `bwa-b200 samse` (bb_samse.c), and the parts of bwase.c that `sampe` uses too ---- */
int bb_samse_main(int argc, char *argv[]);
/* bwase_initialize's g_log_n, and a private erand48 state seeded as srand48(bns->seed) seeds drand48: the same sequence, which
 * nothing else in the process can disturb */
typedef struct { unsigned short rng[3]; int log_n[256]; } bb_aln2seq_t;
void bb_aln2seq_init(bb_aln2seq_t *s, const bntseq_t *bns);
/* the hit bwa_aln2seq_core chooses from a read's .sai records (bwase.c:22-48): one draw per best-score interval, a second when it
 * is taken.  sa, ref_shift, score and the differences are the last interval taken; they stay untouched when none is. */
typedef struct { uint64_t sa; int ref_shift, score; uint32_t c1, c2; uint8_t type, n_mm, n_gapo, n_gape; } bb_hit_t;
void bb_choose_hit(bb_aln2seq_t *s, int n_aln, const bwag_aln1_t *aln, bb_hit_t *h);
/* bwa_approx_mapQ (bwase.c:101-110) of a read of len bases searched, with the max_diff of opt (samse: its .sai; sampe: .sai 2) */
int bb_approx_mapq(const bb_aln2seq_t *s, const aln_opt_t *opt, int len, const bb_hit_t *h);
void bb_upload_holes(bwag_ctx_t *ctx, const bntseq_t *bns, const char *who);   /* bwag_ctx_set_ambs; fatal on failure */
/* one SAM record: read r's name + part A + QUAL (reversed under BWAG_REC_QREV, "*" without) + part B + "\n" */
void bb_splice_sam(bb_str_t *s, const bb_reads_t *rd, int r, const bwag_samrec_t *rec, const char *text);

/* ---- `bwa-b200 sampe` (bb_sampe.c) ---- */
int bb_sampe_main(int argc, char *argv[]);

/* ---- `bwa-b200 pemerge` (bb_pemerge.c) ---- */
int bb_pemerge_main(int argc, char *argv[]);

#ifdef __cplusplus
}
#endif
#endif
