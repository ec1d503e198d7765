/* bb_process.c -- mem_process_seqs: the drop-in boundary (reference bwamem.c:1191-1264).
 *
 * The reference runs, per read and on a CPU thread, seeding -> chaining -> extension -> (PE stats) ->
 * CIGAR -> SAM.  Here a batch goes through the same stages, but every stage that walks the FM-index
 * or fills a DP matrix is ONE device call for the whole batch (include/bwa_b200_dev.h):
 *
 *   host  encode reads to 0..4 codes in place (bwamem.c:1087), pack, upload
 *   GPU   bwag_seed    : SMEM intervals + suffix-array positions of every read
 *   host  chain, filter chains (bb_chain.c), lay out extension work             [threads]
 *   GPU   bwag_extend  : mem_chain2aln loops with banded extension
 *   host  dedup/patch regions (bb_reg.c), insert-size model, mate rescue        [threads]
 *   GPU   bwag_global  : banded global alignment -> CIGAR/NM/MD (as many rounds as the host asks)
 *   host  MAPQ, pairing, SAM text (bb_sam.c, bb_pair.c)                          [threads]
 *
 * Host steps that need a global alignment (mem_patch_reg, mem_reg2aln) look it up in a per-read
 * cache; a miss records a request and abandons that read's pass, and the pass is repeated after the
 * device has served all requests of the batch.  There is no CPU implementation of the device stages.
 */
#include <pthread.h>
#include <assert.h>
#include <math.h>
#include <malloc.h>
#include <unistd.h>
#include "bb_host.h"
#if defined(__SSE2__)
#include <emmintrin.h>
#endif

/* ---------------------------------------------------------------- large host buffers
 * A batch needs a few buffers of tens to hundreds of MB (codes, per-read state, extension work).  glibc
 * serves those with mmap and returns them with munmap, i.e. every batch would page-fault them in again
 * (with 100+ threads touching them at once, that costs more than the GPU stages).  Freed blocks are
 * therefore parked here and handed out again; small allocations stay with malloc, whose arenas are told
 * once not to trim (the same pages are recycled batch after batch). */
typedef struct { void *p; size_t cap; int pinned; } bigblk_t;
#define N_BIG 256
static bigblk_t g_big[N_BIG];
static pthread_mutex_t g_big_mu = PTHREAD_MUTEX_INITIALIZER;
static int g_malloc_tuned;

static void *big_alloc_x(size_t bytes, int pinned);
static void *big_alloc(size_t bytes) { return big_alloc_x(bytes, 0); }
/* pinned: page-locked (bwag_host_alloc) for buffers the device stages read; cached the same way */
static void *big_alloc_x(size_t bytes, int pinned)
{
	int i, best = -1;
	void *p = 0;
	pthread_mutex_lock(&g_big_mu);
	if (!g_malloc_tuned) { mallopt(M_TRIM_THRESHOLD, 1 << 30); mallopt(M_TOP_PAD, 64 << 20); mallopt(M_MMAP_THRESHOLD, 32 << 20); g_malloc_tuned = 1; }
	for (i = 0; i < N_BIG; ++i)
		if (g_big[i].p && g_big[i].pinned == pinned && g_big[i].cap >= bytes && (best < 0 || g_big[i].cap < g_big[best].cap)) best = i;
	if (best >= 0 && g_big[best].cap <= bytes * 4 + (64u << 20)) { p = g_big[best].p; g_big[best].p = 0; }
	pthread_mutex_unlock(&g_big_mu);
	if (!p) {
		size_t cap = bytes + bytes / 8 + 4096;
		size_t *q = 0;
		if (pinned && cap >= (1u << 20)) q = bwag_host_alloc(cap + 16);
		if (q) q[1] = 1; else { q = bb_malloc(cap + 16); q[1] = 0; }
		q[0] = cap;
		return q + 2;
	}
	return p;
}

static void big_free(void *p)
{
	size_t *q;
	int i;
	if (!p) return;
	q = (size_t *)p - 2;
	if (q[0] < (1u << 20)) { if (q[1]) bwag_host_free(q); else free(q); return; }
	pthread_mutex_lock(&g_big_mu);
	for (i = 0; i < N_BIG; ++i) if (!g_big[i].p) { g_big[i].p = p; g_big[i].cap = q[0]; g_big[i].pinned = (int)q[1]; p = 0; break; }
	pthread_mutex_unlock(&g_big_mu);
	if (p) { if (q[1]) bwag_host_free(q); else free(q); }
}

/* phase timer: BWA_B200_PROFILE=1 prints the wall time of every phase of a batch to stderr */
static int g_prof = -1;
static double g_t_last;
static void ph(const char *name)
{
	double t;
	if (g_prof <= 0) return;     /* set once by diag_init(); the timer is only meaningful with one call in flight */
	t = bb_realtime();
	if (name) fprintf(stderr, "[prof] %-16s %9.2f ms\n", name, 1e3 * (t - g_t_last));
	g_t_last = t;
}

/* BWA_B200_TRACE=1: one line per (lane, chunk, phase) with start/end in ms since the batch began */
static int g_trace = -1;
static double g_trace_t0;
static double trace_now(void) { return 1e3 * (bb_realtime() - g_trace_t0); }
#define PH(j, name) do { if ((j)->lane == 0) ph(name); if (g_trace > 0) { double t_ = trace_now(); fprintf(stderr, "[trace] lane %d chunk %d %-12s %8.1f -> %8.1f\n", (j)->lane, (j)->chunk_id, name, (j)->t_last, t_); (j)->t_last = t_; } } while (0)
#define TRACE(j, name, t_start) do { if (g_trace > 0) fprintf(stderr, "[trace] lane %d chunk %d %-12s %8.1f -> %8.1f\n", (j)->lane, (j)->chunk_id, name, t_start, trace_now()); } while (0)

/* ---------------------------------------------------------------- device residency */
typedef struct { const bwt_t *bwt; bwag_ctx_t *ctx; } dev_slot_t;
static dev_slot_t g_dev[8];
static pthread_mutex_t g_dev_mu = PTHREAD_MUTEX_INITIALIZER;

/* The on-disk suffix-array sample keeps every 32nd row (bwa index); the device derives a denser one from it in about a
 * second, which cuts the LF walk of every seed lookup from ~15.5 steps to ~0.5 (every 2nd row) or ~3.5 (every 8th row)
 * without changing any result.  By default the interval is chosen from the device's memory (bwag_ctx_densify_sa with 0):
 * a 3 Gbp reference on an 80 GB H100 gets every 8th row (6 GB; every 2nd row would be 24 GB and leave too little for the
 * batches of three calls in flight), smaller references every 2nd row.  It is derived in two stages (32 -> 8 -> intv) so
 * that each stage walks only a few steps per row.  BWA_B200_SA_INTV overrides (32 keeps the disk sample); a stage that
 * does not fit the free device memory is skipped silently and the previous sample stays. */
static void densify_default(bwag_ctx_t *ctx)
{
	const char *e = getenv("BWA_B200_SA_INTV");
	if (!e) bwag_ctx_densify_sa(ctx, 0);
	else {
		int intv = atoi(e);
		if (intv > 0 && intv < 8) bwag_ctx_densify_sa(ctx, 8);
		if (intv > 0) bwag_ctx_densify_sa(ctx, intv);   /* a refusal (interval not below the current one, no memory) leaves the context as it was */
	}
	{   /* short-string table (include/bwa_b200_dev.h): BWA_B200_KTAB = depth, 0 = none; default: from the index size */
		const char *k = getenv("BWA_B200_KTAB");
		int depth = k ? atoi(k) : 0;
		if (!k || depth > 0) bwag_ctx_build_ktab(ctx, depth);
	}
}

/* Start-up self-check.  The lean row sweeps of K4/K5 and the short-string table of K1 compute exactly what the first
 * formulations compute; to make a platform-specific fault in them visible (and harmless) the moment an index goes to the
 * device, a few hundred reads drawn from the reference itself (with substitutions, small insertions and deletions, both
 * strands) are aligned twice -- defaults, then baseline (bwag_ctx_baseline) -- and the SAM records compared.  Any
 * difference: a warning on stderr and the context stays on the baseline, whose parity the GPU tests check.
 * BWA_B200_SELFCHECK = number of reads (default 192 on a CUDA device, 0 = off; off by default in the test emulator). */
static __thread bwag_ctx_t *tl_attach_override;   /* the self-check aligns through mem_process_seqs while the registry lock is held */
static int g_selfcheck_status;                    /* 0 not run, 1 passed, 2 differed: running on the baseline */
int bb_selfcheck_status(void) { return __atomic_load_n(&g_selfcheck_status, __ATOMIC_RELAXED); }

static bseq1_t *selfcheck_reads(const bntseq_t *bns, const uint8_t *pac, int n, int len)
{
	bseq1_t *seqs = bb_calloc((size_t)n, sizeof(bseq1_t));
	uint64_t rng = 0x9e3779b97f4a7c15ULL;
	int i, k;
	for (i = 0; i < n; ++i) {
		char *s = bb_malloc((size_t)len + 8), name[32];
		int l = 0;
		int64_t pos;
		rng = rng * 6364136223846793005ULL + 1442695040888963407ULL;
		pos = (int64_t)((rng >> 11) % (uint64_t)(bns->l_pac - len - 8));
		for (k = 0; k < len + 4 && l < len; ++k) {
			int c = pac[(pos + k) >> 2] >> ((~(pos + k) & 3) << 1) & 3;
			if (k == 17 + i % 23 || k == len - 9 - i % 11) c = (c + 1 + i % 3) & 3;      /* two substitutions */
			if (i % 3 == 1 && (k == len / 2 || k == len / 2 + 1)) continue;            /* a 2-base deletion */
			if (i % 5 == 2 && k == len / 3) { s[l++] = "ACGT"[(c + 2) & 3]; if (l < len) s[l++] = "ACGT"[(c + 1) & 3]; if (l < len) s[l++] = "ACGT"[c]; }   /* a 3-base insertion */
			if (l < len) s[l++] = "ACGT"[c];
		}
		if (i & 1) {   /* reverse complement */
			for (k = 0; k < l / 2; ++k) { char t = s[k]; s[k] = s[l - 1 - k]; s[l - 1 - k] = t; }
			for (k = 0; k < l; ++k) s[k] = s[k] == 'A' ? 'T' : s[k] == 'C' ? 'G' : s[k] == 'G' ? 'C' : 'A';
		}
		s[l] = 0;
		snprintf(name, sizeof(name), "selfcheck%d", i);
		seqs[i].l_seq = l; seqs[i].seq = s; seqs[i].name = bb_malloc(strlen(name) + 1); strcpy(seqs[i].name, name);
	}
	return seqs;
}
static void selfcheck_free(bseq1_t *seqs, int n) { int i; for (i = 0; i < n; ++i) { free(seqs[i].seq); free(seqs[i].name); free(seqs[i].sam); } free(seqs); }

static void device_selfcheck(bwag_ctx_t *ctx, const bwt_t *bwt, const bntseq_t *bns, const uint8_t *pac)
{
	const char *e = getenv("BWA_B200_SELFCHECK");
	int n = e ? atoi(e) : (bwag_is_emulator() ? 0 : 192), i, differ = 0;
	const int len = 120;
	bseq1_t *a, *b;
	mem_opt_t *opt;
	if (n <= 0 || bwag_is_emulator() == 2 || bns->l_pac < 4 * len) return;
	opt = mem_opt_init();
	opt->n_threads = 2;
	a = selfcheck_reads(bns, pac, n, len); b = selfcheck_reads(bns, pac, n, len);
	tl_attach_override = ctx;
	mem_process_seqs(opt, bwt, bns, pac, 0, n, a, 0);
	bwag_ctx_baseline(ctx, 1);
	mem_process_seqs(opt, bwt, bns, pac, 0, n, b, 0);
	tl_attach_override = 0;
	if (getenv("BWA_B200_SELFCHECK_INJECT") && a[0].sam && a[0].sam[0]) a[0].sam[strlen(a[0].sam) / 2] ^= 1;   /* test hook: pretend a difference */
	for (i = 0; i < n; ++i) if (!a[i].sam || !b[i].sam || strcmp(a[i].sam, b[i].sam) != 0) { ++differ; if (differ == 1 && bwa_verbose >= 1) fprintf(stderr, "[W::bwa_b200] self-check: first differing record\n  default : %s  baseline: %s", a[i].sam ? a[i].sam : "(none)\n", b[i].sam ? b[i].sam : "(none)\n"); }
	if (differ) {
		/* a difference is a fault of this platform or build: stop (every failure of this library is fatal, as in the reference),
		 * unless the caller asked to continue on the baseline kernels (BWA_B200_SELFCHECK_FALLBACK=1) */
		if (!(getenv("BWA_B200_SELFCHECK_FALLBACK") && atoi(getenv("BWA_B200_SELFCHECK_FALLBACK"))))
			bb_fatal("bwa_b200 self-check", "%d of %d records differ between the default kernels and the baseline kernels; set BWA_B200_SELFCHECK_FALLBACK=1 to run on the baseline kernels", differ, n);
		fprintf(stderr, "[W::bwa_b200] start-up self-check: %d of %d records differ between the default kernels and the baseline; staying on the baseline kernels\n", differ, n);
		__atomic_store_n(&g_selfcheck_status, 2, __ATOMIC_RELAXED);
	} else {
		bwag_ctx_baseline(ctx, 0);
		__atomic_store_n(&g_selfcheck_status, 1, __ATOMIC_RELAXED);
	}
	selfcheck_free(a, n); selfcheck_free(b, n);
	free(opt);
}

/* stage 4 needs the contig table (offsets, lengths, ALT flags, names) next to the index */
static void set_contigs(bwag_ctx_t *ctx, const bntseq_t *bns)
{
	int c, n = bns->n_seqs, rc;
	int64_t *off = bb_malloc(sizeof(int64_t) * ((size_t)n + 1));
	int32_t *len = bb_malloc(sizeof(int32_t) * ((size_t)n + 1));
	uint8_t *alt = bb_malloc((size_t)n + 1);
	const char **names = bb_malloc(sizeof(char *) * ((size_t)n + 1));
	for (c = 0; c < n; ++c) { off[c] = bns->anns[c].offset; len[c] = bns->anns[c].len; alt[c] = !!bns->anns[c].is_alt; names[c] = bns->anns[c].name; }
	rc = bwag_ctx_set_contigs(ctx, n, off, len, alt, names);
	if (rc != 0 && rc != BWAG_UNSUPPORTED) bb_fatal("bb_device_attach", "cannot place the contig table on the GPU: %s", bwag_last_error());
	free(off); free(len); free(alt); free(names);
}

bwag_ctx_t *bb_device_attach(const bwt_t *bwt, const bntseq_t *bns, const uint8_t *pac)
{
	int i;
	bwag_ctx_t *ctx = 0;
	if (tl_attach_override) return tl_attach_override;
	pthread_mutex_lock(&g_dev_mu);
	for (i = 0; i < 8; ++i) if (g_dev[i].bwt == bwt && g_dev[i].ctx) { ctx = g_dev[i].ctx; break; }
	if (!ctx) {
		for (i = 0; i < 8 && g_dev[i].ctx; ++i) {}
		if (i == 8) bb_fatal("bb_device_attach", "too many resident indexes");
		ctx = bwag_ctx_create(-1, bwt, bns->l_pac, pac);
		if (!ctx) bb_fatal("bb_device_attach", "cannot place the index on the GPU: %s", bwag_last_error());
		densify_default(ctx);
		set_contigs(ctx, bns);
		g_dev[i].bwt = bwt; g_dev[i].ctx = ctx;
		device_selfcheck(ctx, bwt, bns, pac);   /* other callers wait for the verdict */
	}
	pthread_mutex_unlock(&g_dev_mu);
	return ctx;
}

/* register a context created elsewhere (e.g. from an NCCL-broadcast blob) for this host index; with bns/pac given the
 * start-up self-check runs here as it does in bb_device_attach.  The slot becomes visible only when the context is ready. */
void bb_device_adopt2(const bwt_t *bwt, const bntseq_t *bns, const uint8_t *pac, bwag_ctx_t *ctx)
{
	int i;
	pthread_mutex_lock(&g_dev_mu);
	for (i = 0; i < 8 && g_dev[i].ctx; ++i) {}
	if (i == 8) bb_fatal("bb_device_adopt", "too many resident indexes");
	densify_default(ctx);
	if (bns) set_contigs(ctx, bns);
	g_dev[i].bwt = bwt; g_dev[i].ctx = ctx;
	if (bns && pac) device_selfcheck(ctx, bwt, bns, pac);
	pthread_mutex_unlock(&g_dev_mu);
}
void bb_device_adopt(const bwt_t *bwt, bwag_ctx_t *ctx) { bb_device_adopt2(bwt, 0, 0, ctx); }

void bb_device_release(const bwt_t *bwt)
{
	int i;
	pthread_mutex_lock(&g_dev_mu);
	for (i = 0; i < 8; ++i)
		if (g_dev[i].bwt == bwt && g_dev[i].ctx) { bwag_ctx_destroy(g_dev[i].ctx); g_dev[i].ctx = 0; g_dev[i].bwt = 0; }
	pthread_mutex_unlock(&g_dev_mu);
}

/* ---------------------------------------------------------------- alignment cache */
/* Caches that outgrow their inline slot take their array from a per-thread bump arena of the chunk being processed:
 * a million small mallocs released later by other threads cost more than the alignments they describe. */
typedef struct memo_blk { struct memo_blk *next; size_t used, cap; } memo_blk_t;
typedef struct { memo_blk_t *head; } memo_arena_t;
static __thread memo_arena_t *tl_memo;
static void *memo_alloc(size_t bytes)
{
	memo_arena_t *ar = tl_memo;
	memo_blk_t *b;
	void *p;
	if (!ar) return 0;
	bytes = (bytes + 15) & ~(size_t)15;
	b = ar->head;
	if (!b || b->used + bytes > b->cap) {
		size_t cap = bytes > (1u << 18) ? bytes : (1u << 18);
		b = bb_malloc(sizeof(memo_blk_t) + cap);
		b->next = ar->head; b->used = 0; b->cap = cap;
		ar->head = b;
	}
	p = (char *)(b + 1) + b->used;
	b->used += bytes;
	return p;
}
static void memo_arenas_free(memo_arena_t *ars, int n)
{
	int i;
	if (!ars) return;
	for (i = 0; i < n; ++i) { memo_blk_t *b = ars[i].head, *nx; for (; b; b = nx) { nx = b->next; free(b); } }
	free(ars);
}
const bb_galn_t *bb_gcache_get(bb_gcache_t *gc, int mode, int qb, int qe, int64_t rb, int64_t re, int w, int truesc)
{
	size_t i;
	bb_galn_t e;
	for (i = 0; i < gc->memo.n; ++i) {
		const bb_galn_t *g = &gc->memo.a[i];
		if (g->mode == mode && g->qb == qb && g->qe == qe && g->rb == rb && g->re == re && g->w == w && g->truesc == truesc) {
			if (g->done) return g;
			++gc->pending;
			return 0;
		}
	}
	memset(&e, 0, sizeof(e));
	e.mode = mode; e.qb = qb; e.qe = qe; e.rb = rb; e.re = re; e.w = w; e.truesc = truesc;
	if (gc->memo.a == 0) { gc->memo.a = &gc->inl; gc->memo.m = 1; gc->memo.n = 0; }
	if (gc->memo.n == gc->memo.m) { /* leave the inline slot for the heap */
		size_t m = gc->memo.m < 4 ? 4 : gc->memo.m << 1;
		bb_galn_t *na = memo_alloc(m * sizeof(bb_galn_t));
		int arena = na != 0;
		if (!na) na = bb_malloc(m * sizeof(bb_galn_t));
		memcpy(na, gc->memo.a, gc->memo.n * sizeof(bb_galn_t));
		if (gc->memo.a != &gc->inl && !gc->in_arena) free(gc->memo.a);
		gc->memo.a = na; gc->memo.m = m; gc->in_arena = arena;
	}
	gc->memo.a[gc->memo.n++] = e;
	++gc->pending;
	return 0;
}

static void gcache_free(bb_gcache_t *gc) /* CIGAR/MD bytes live in per-round blocks owned by the job */
{
	if (gc->memo.a != &gc->inl && !gc->in_arena) free(gc->memo.a);
	gc->memo.a = 0; gc->memo.n = gc->memo.m = 0; gc->in_arena = 0;
}

/* ---------------------------------------------------------------- batch state */
typedef struct {
	mem_alnreg_v regs;   /* regions after de-duplication (and mate rescue), pristine */
	bb_gcache_t gc;
	int done;            /* SAM written */
	int dedup_done;
	int n_raw;           /* regions straight from the extension stage */
} rstate_t;

typedef struct { /* per-thread output of the chaining step */
	bb_chainer_t *chainer;
	bb_chain_v chains;
	BB_VEC(bwag_xchain_t) xc;
	BB_VEC(bwag_xseed_t) xs;
	BB_VEC(int) c_rid;
	BB_VEC(float) c_frac;
	BB_VEC(uint64_t) srt;
} tls_t;

typedef struct { int tid; int64_t c0, s0; int nc, ns; } rslice_t; /* where read i's chains sit in its thread's buffers */

typedef struct job_s {
	const mem_opt_t *opt;
	const bwt_t *bwt;
	const bntseq_t *bns;
	const uint8_t *pac;
	const mem_pestat_t *pes;
	int64_t n_processed;
	int n;
	bseq1_t *seqs;
	int64_t *off;
	uint8_t *codes;
	rstate_t *rs;
	/* stage 1 results */
	bwag_seeds_t seeds;
	/* chaining */
	tls_t *tls;
	rslice_t *slice;
	/* flattened extension work */
	int32_t *chain_off;
	bwag_xchain_t *xchains;
	bwag_xseed_t *xseeds;
	int *chain_rid;
	float *chain_frac;
	int64_t n_xchains, n_xseeds;
	bwag_regs_t xregs;
	bwag_cregs_t cregs; int have_cregs;   /* regions from the fused device chain+extend stage */
	int pass_dry;
	void **blocks; int n_blocks, m_blocks;   /* CIGAR/MD storage of each device round (a read whose regions merge one after
	                                          * the other, bwamem.c:463-515, can need one round per merge: no fixed bound) */
	mem_alnreg_t *reg_pool; int64_t *reg_off;   /* SE: regions of all reads in one block */
	double t_last;
	memo_arena_t *arenas;    /* one bump arena per parallel id for the alignment caches of this chunk */
	uint64_t *pe_is;         /* PE: this chunk's slice of the per-pair insert-size candidates */
	int lane, chunk_id;      /* which lane (device batch object) runs this chunk */
	bwag_batch_t *batch;
	bwag_sw_par_t swp;
	/* device tail (stage 4): the chunk's reads are post-processed on the device; reads it hands back go through `sub` jobs,
	 * which are ordinary jobs over copies of their bseq1_t records */
	int tail;                      /* 1: bwag_tail_regs ran for this chunk */
	int no_tail;                   /* the caller wants the regions on the host (mem_align1) */
	bb_swcache_t *swc;             /* PE: per pair, the mate-rescue alignments asked from / served by K6 */
	const uint8_t *cflag;          /* [n] from bwag_tail_regs: non-zero = the read left the simple path before pairing */
	struct job_s *sub0, *sub1;     /* reads handed back by bwag_tail_regs (aligned up to regions before the insert-size model) / by bwag_tail_sam */
	int *sub_map;                  /* sub job only: index of each of its reads in the parent chunk */
	const int64_t *ids;            /* sub job only: global index (n_processed + position) of each read: the hash tie-breaks depend on it */
	int32_t *pre_n; int64_t *pre_beg; bwag_creg_t *pre_regs;   /* sub job only: the raw regions of its reads, taken over from the parent chunk's device stages */
	const struct tail_shared_s *ts;
} job_t;

/* Bases to codes, in place (the caller's buffer, bwamem.c:1087: seq[i] < 4 ? seq[i] : nst_nt4_table[seq[i]]) and into the
 * device staging buffer (codes above 4 -- the table's '-' -> 5 -- become 4 there: every kernel treats > 3 as N).
 * 16 bases per step with SSE2 compares where available; the scalar loop is the specification (tests/test_cabi.py). */
void bb_encode_bases(char *seq, uint8_t *dst, int n)
{
	int k = 0;
#if defined(__SSE2__)
	const __m128i c3 = _mm_set1_epi8(3), c4 = _mm_set1_epi8(4), c5 = _mm_set1_epi8(5), fold = _mm_set1_epi8((char)0xDF), zero = _mm_setzero_si128();
	const __m128i cA = _mm_set1_epi8('A'), cC = _mm_set1_epi8('C'), cG = _mm_set1_epi8('G'), cT = _mm_set1_epi8('T'), cD = _mm_set1_epi8('-');
	const __m128i one = _mm_set1_epi8(1), two = _mm_set1_epi8(2);
	for (; k + 16 <= n; k += 16) {
		const __m128i v = _mm_loadu_si128((const __m128i *)(seq + k));
		const __m128i small = _mm_cmpeq_epi8(_mm_subs_epu8(v, c3), zero);      /* already a code 0..3 */
		const __m128i u = _mm_and_si128(v, fold);
		const __m128i isA = _mm_cmpeq_epi8(u, cA), isC = _mm_cmpeq_epi8(u, cC), isG = _mm_cmpeq_epi8(u, cG), isT = _mm_cmpeq_epi8(u, cT);
		const __m128i acgt = _mm_or_si128(_mm_or_si128(isA, isC), _mm_or_si128(isG, isT));
		const __m128i code = _mm_or_si128(_mm_and_si128(isC, one), _mm_or_si128(_mm_and_si128(isG, two), _mm_and_si128(isT, c3)));
		const __m128i other = _mm_or_si128(_mm_and_si128(_mm_cmpeq_epi8(v, cD), c5), _mm_andnot_si128(_mm_cmpeq_epi8(v, cD), c4));
		__m128i r = _mm_or_si128(_mm_and_si128(acgt, code), _mm_andnot_si128(acgt, other));
		r = _mm_or_si128(_mm_and_si128(small, v), _mm_andnot_si128(small, r));
		_mm_storeu_si128((__m128i *)(seq + k), r);
		_mm_storeu_si128((__m128i *)(dst + k), _mm_min_epu8(r, c4));
	}
#endif
	for (; k < n; ++k) {
		unsigned char c = (unsigned char)seq[k];
		c = c < 4 ? c : bb_nt4_table[c];
		seq[k] = (char)c;
		dst[k] = c > 4 ? 4 : c;
	}
}

static void w_encode(void *d, long i, int tid)
{
	job_t *j = d;
	(void)tid;
	bb_encode_bases(j->seqs[i].seq, j->codes + j->off[i], j->seqs[i].l_seq);
}

static void w_chain(void *d, long i, int tid)
{
	job_t *j = d;
	tls_t *t = &j->tls[tid];
	const mem_opt_t *opt = j->opt;
	const bwag_seeds_t *sd = &j->seeds;
	int l_query = j->seqs[i].l_seq, n_chn, c;
	int64_t i0 = sd->intv_beg[i], i1 = i0 + sd->intv_n[i], l_pac = j->bns->l_pac;
	rslice_t *sl = &j->slice[i];
	const uint8_t *query = (const uint8_t *)j->seqs[i].seq;
	if (!t->chainer) t->chainer = bb_chainer_new();
	sl->tid = tid; sl->c0 = (int64_t)t->xc.n; sl->s0 = (int64_t)t->xs.n; sl->nc = sl->ns = 0;
	bb_chain_build(t->chainer, opt, j->bns, l_query, (int)(i1 - i0), sd->intv + i0, sd->seed_beg + i0, sd->rbeg, &t->chains);
	n_chn = bb_chain_filter(opt, (int)t->chains.n, t->chains.a);
	bb_chain_seed_sw(opt, j->bns, j->pac, l_query, query, n_chn, t->chains.a);
	for (c = 0; c < n_chn; ++c) { /* window and seed order of mem_chain2aln (bwamem.c:666-691) */
		const bb_chain_t *ch = &t->chains.a[c];
		bwag_xchain_t xc;
		int64_t rmax0 = l_pac << 1, rmax1 = 0;
		int k, rid;
		if (ch->n == 0) continue;
		for (k = 0; k < ch->n; ++k) {
			const bb_seed_t *s = &ch->seeds[k];
			int64_t b = s->rbeg - (s->qbeg + bb_cal_max_gap(opt, s->qbeg));
			int64_t e = s->rbeg + s->len + ((l_query - s->qbeg - s->len) + bb_cal_max_gap(opt, l_query - s->qbeg - s->len));
			if (b < rmax0) rmax0 = b;
			if (e > rmax1) rmax1 = e;
		}
		if (rmax0 < 0) rmax0 = 0;
		if (rmax1 > l_pac << 1) rmax1 = l_pac << 1;
		if (rmax0 < l_pac && l_pac < rmax1) {
			if (ch->seeds[0].rbeg < l_pac) rmax1 = l_pac; else rmax0 = l_pac;
		}
		bb_clamp_to_contig(j->bns, &rmax0, ch->seeds[0].rbeg, &rmax1, &rid);
		assert(rid == ch->rid);
		t->srt.n = 0;
		for (k = 0; k < ch->n; ++k) bb_vec_push(t->srt, (uint64_t)ch->seeds[k].score << 32 | (uint32_t)k);
		bb_sort_u64(t->srt.n, t->srt.a);
		xc.rmax0 = rmax0; xc.rmax1 = rmax1; xc.seed_off = (int32_t)(t->xs.n - sl->s0); xc.n_seeds = ch->n;
		for (k = 0; k < ch->n; ++k) {
			const bb_seed_t *s = &ch->seeds[(uint32_t)t->srt.a[k]];
			bwag_xseed_t xs;
			xs.rbeg = s->rbeg; xs.qbeg = s->qbeg; xs.len = (uint32_t)s->len | (t->srt.a[k] == 0 ? BWAG_XSEED_ZEROKEY : 0);
			bb_vec_push(t->xs, xs);
		}
		bb_vec_push(t->xc, xc);
		bb_vec_push(t->c_rid, ch->rid);
		bb_vec_push(t->c_frac, ch->frac_rep);
		++sl->nc; sl->ns += ch->n;
	}
}

static void w_flatten(void *d, long i, int tid)
{
	job_t *j = d;
	const rslice_t *sl = &j->slice[i];
	const tls_t *t = &j->tls[sl->tid];
	int64_t c0 = j->chain_off[i], s0, k;
	(void)tid;
	if (sl->nc == 0) return;
	s0 = j->xchains[c0].seed_off; /* pre-filled by the serial prefix pass with the read's global seed base */
	for (k = 0; k < sl->nc; ++k) {
		bwag_xchain_t xc = t->xc.a[sl->c0 + k];
		xc.seed_off += (int32_t)s0;
		j->xchains[c0 + k] = xc;
		j->chain_rid[c0 + k] = t->c_rid.a[sl->c0 + k];
		j->chain_frac[c0 + k] = t->c_frac.a[sl->c0 + k];
	}
	memcpy(j->xseeds + s0, t->xs.a + sl->s0, sizeof(bwag_xseed_t) * sl->ns);
}

/* regions of read i from the extension stage -> pristine mem_alnreg_t array */
static void load_raw_regs(job_t *j, long i, mem_alnreg_v *v)
{
	if (j->have_cregs) {
		const int n = j->cregs.n_regs[i];
		const bwag_creg_t *x = j->cregs.regs + j->cregs.reg_beg[i];
		int k;
		v->n = 0;
		if (j->reg_pool) { v->a = j->reg_pool + j->reg_off[i]; v->m = (size_t)n | BB_BORROWED; }
		else bb_vec_reserve(*v, (size_t)n + 4);
		for (k = 0; k < n; ++k) {
			mem_alnreg_t *a = &v->a[k];
			memset(a, 0, sizeof(*a));
			a->rb = x[k].r.rb; a->re = x[k].r.re; a->qb = x[k].r.qb; a->qe = x[k].r.qe;
			a->score = x[k].r.score; a->truesc = x[k].r.truesc; a->w = x[k].r.w;
			a->seedcov = x[k].r.seedcov; a->seedlen0 = x[k].r.seedlen0;
			a->rid = x[k].rid; a->frac_rep = x[k].frac_rep;
		}
		v->n = (size_t)n;
		return;
	}
	int64_t c0 = j->chain_off[i], c1 = j->chain_off[i + 1];
	int k, n = c1 > c0 ? j->xregs.n_regs[i] : 0;
	const bwag_xreg_t *x = c1 > c0 ? j->xregs.regs + j->xchains[c0].seed_off : 0;
	v->n = 0;
	if (j->reg_pool) { v->a = j->reg_pool + j->reg_off[i]; v->m = (size_t)n | BB_BORROWED; }
	else bb_vec_reserve(*v, (size_t)n + 4);
	for (k = 0; k < n; ++k) {
		mem_alnreg_t *a = &v->a[k];
		memset(a, 0, sizeof(*a));
		a->rb = x[k].rb; a->re = x[k].re; a->qb = x[k].qb; a->qe = x[k].qe;
		a->score = x[k].score; a->truesc = x[k].truesc; a->w = x[k].w;
		a->seedcov = x[k].seedcov; a->seedlen0 = x[k].seedlen0;
		a->rid = j->chain_rid[c0 + x[k].chain];
		a->frac_rep = j->chain_frac[c0 + x[k].chain];
	}
	v->n = (size_t)n;
}

static void w_zero_rs(void *d, long c, int tid)
{
	job_t *j = d;
	long b = c * 4096, e = b + 4096 <= j->n ? b + 4096 : (long)j->n + 1;
	(void)tid;
	if (c == ((long)j->n + 4095) / 4096 - 1) e = (long)j->n + 1;
	memset(j->rs + b, 0, (size_t)(e - b) * sizeof(rstate_t));
}

static void w_dedup(void *d, long i, int tid)
{
	job_t *j = d;
	rstate_t *r = &j->rs[i];
	int n;
	size_t k;
	if (r->dedup_done) return;
	tl_memo = j->arenas ? &j->arenas[tid] : 0;
	load_raw_regs(j, i, &r->regs);
	r->gc.pending = 0;
	n = bb_sort_dedup_patch(j->opt, j->bns, &r->gc, j->seqs[i].l_seq, (int)r->regs.n, r->regs.a);
	if (n < 0) return; /* a merge candidate needs a device alignment first */
	r->regs.n = (size_t)n;
	for (k = 0; k < r->regs.n; ++k) {
		mem_alnreg_t *p = &r->regs.a[k];
		if (p->rid >= 0 && j->bns->anns[p->rid].is_alt) p->is_alt = 1;
		/* Every region that can reach the output (or an XA list) will need its CIGAR: ask for all of them now, so
		 * that one device round serves the batch before the SAM pass (the K5 kernel is cheap; the host's time is not).
		 * The SAM pass still recovers through the cache-miss path if it ever needs something else. */
		bb_gcache_get(&r->gc, BWAG_G_REG2ALN, p->qb, p->qe, p->rb, p->re, bb_reg2aln_band(j->opt, p), p->truesc);
	}
	r->dedup_done = 1;
}

/* Test hook: BWA_B200_TEST_DUMP_STAGES=<dir> writes the inputs of every bwag_extend and bwag_global call to a file of its own in
 * <dir>, so that tests/test_dp_stages.py can replay them through two implementations of the stage ABI.  Every file is in the host's
 * byte order: eight int64 (kind 1 = extend, 2 = global; n_reads; bases; n_chains or n_tasks; n_seeds; and the sizes of
 * bwag_sw_par_t and of a chain or task), the bwag_sw_par_t, off[n_reads + 1], the bases (codes 0..4), then for an extension
 * chain_off[n_reads + 1], the chains and the seeds, for a global alignment the tasks. */
static void dump_stage(const job_t *j, const bwag_sw_par_t *swp, int kind, int64_t n_items, const void *items, size_t item_size)
{
	static int seq;
	const char *dir = getenv("BWA_B200_TEST_DUMP_STAGES");
	char path[4096];
	FILE *fp;
	if (!dir) return;
	snprintf(path, sizeof(path), "%s/%s-%d-%06d.bin", dir, kind == 1 ? "extend" : "global", (int)getpid(), __atomic_fetch_add(&seq, 1, __ATOMIC_RELAXED));
	if (!(fp = fopen(path, "wb"))) bb_fatal("mem_process_seqs", "cannot write %s", path);
	{
		const int64_t h[8] = { kind, j->n, j->off[j->n], n_items, kind == 1 ? j->n_xseeds : 0, (int64_t)sizeof(*swp), (int64_t)item_size, 0 };
		fwrite(h, sizeof(h), 1, fp);
	}
	fwrite(swp, sizeof(*swp), 1, fp);
	fwrite(j->off, sizeof(int64_t), (size_t)j->n + 1, fp);
	fwrite(j->codes, 1, (size_t)j->off[j->n], fp);
	if (kind == 1) fwrite(j->chain_off, sizeof(int32_t), (size_t)j->n + 1, fp);
	fwrite(items, item_size, (size_t)n_items, fp);
	if (kind == 1) fwrite(j->xseeds, sizeof(bwag_xseed_t), (size_t)j->n_xseeds, fp);
	if (fclose(fp) != 0) bb_fatal("mem_process_seqs", "cannot write %s", path);
}

/* serve every outstanding alignment request of the batch with one device call; returns #requests */
typedef struct { job_t *j; int64_t *off; bwag_gtask_t *tasks; const bwag_galn_t *out; int64_t *boff; char *block; } ground_t;

static void w_gcount(void *d, long i, int tid)
{
	ground_t *g = d;
	const bb_galn_v *m = &g->j->rs[i].gc.memo;
	size_t k;
	int c = 0;
	(void)tid;
	for (k = 0; k < m->n; ++k) c += !m->a[k].done;
	g->off[i + 1] = c;
}

static void w_gfill(void *d, long i, int tid)
{
	ground_t *g = d;
	const bb_galn_v *m = &g->j->rs[i].gc.memo;
	bwag_gtask_t *x = g->tasks + g->off[i];
	size_t k;
	(void)tid;
	if (g->off[i + 1] == g->off[i]) return;
	for (k = 0; k < m->n; ++k) {
		const bb_galn_t *e = &m->a[k];
		if (e->done) continue;
		x->rb = e->rb; x->re = e->re; x->read = (int32_t)i; x->qb = e->qb; x->qe = e->qe; x->w = e->w; x->truesc = e->truesc; x->mode = e->mode;
		++x;
	}
}

static void w_gstore(void *d, long i, int tid)
{
	ground_t *g = d;
	bb_galn_v *m = &g->j->rs[i].gc.memo;
	const bwag_gres_t *r = g->out->res + g->off[i];
	const int64_t *bo = g->boff + g->off[i];
	size_t k;
	(void)tid;
	if (g->off[i + 1] == g->off[i]) return;
	for (k = 0; k < m->n; ++k) {
		bb_galn_t *e = &m->a[k];
		if (e->done) continue;
		e->score = r->score; e->n_cigar = r->n_cigar; e->NM = r->NM; e->l_md = r->l_md > 0 ? r->l_md : 1;
		e->cigar = (uint32_t *)(g->block + *bo++);
		memcpy(e->cigar, g->out->cigar + r->cigar_off, 4 * (size_t)r->n_cigar);
		if (r->l_md > 0) memcpy((char *)(e->cigar + r->n_cigar), g->out->md + r->md_off, r->l_md);
		else *(char *)(e->cigar + r->n_cigar) = 0;
		e->done = 1;
		++r;
	}
}

static int64_t global_round(job_t *j, bwag_batch_t *batch, const bwag_sw_par_t *swp)
{
	ground_t g;
	bwag_galn_t out;
	int64_t i, t;
	int nt = j->opt->n_threads > 0 ? j->opt->n_threads : 1;
	g.j = j; g.out = &out;
	g.off = big_alloc(sizeof(int64_t) * ((size_t)j->n + 1));
	g.off[0] = 0;
	bb_parallel_for_lane(j->lane, nt, w_gcount, &g, j->n);
	for (i = 0; i < j->n; ++i) g.off[i + 1] += g.off[i];
	t = g.off[j->n];
	if (t == 0) { big_free(g.off); return 0; }
	g.tasks = big_alloc_x(sizeof(bwag_gtask_t) * (size_t)t, 1);
	bb_parallel_for_lane(j->lane, nt, w_gfill, &g, j->n);
	dump_stage(j, swp, 2, t, g.tasks, sizeof(bwag_gtask_t));
	if (bwag_global(batch, swp, (int)t, g.tasks, &out) != 0) bb_fatal("mem_process_seqs", "global-alignment stage failed: %s", bwag_last_error());
	g.boff = big_alloc(sizeof(int64_t) * ((size_t)t + 1));
	{
		int64_t x, tot = 0;
		for (x = 0; x < t; ++x) { g.boff[x] = tot; tot += ((int64_t)4 * out.res[x].n_cigar + (out.res[x].l_md > 0 ? out.res[x].l_md : 1) + 7) & ~(int64_t)7; }
		g.boff[t] = tot;
		if (j->n_blocks == j->m_blocks) { j->m_blocks = j->m_blocks ? j->m_blocks << 1 : 16; j->blocks = bb_realloc(j->blocks, sizeof(void *) * (size_t)j->m_blocks); }
		g.block = big_alloc((size_t)tot + 8);
		j->blocks[j->n_blocks++] = g.block;
	}
	bb_parallel_for_lane(j->lane, nt, w_gstore, &g, j->n);
	big_free(g.tasks); big_free(g.off); big_free(g.boff);
	return t;
}

static void w_rescue(void *d, long i, int tid)
{
	job_t *j = d;
	mem_alnreg_v a[2];
	tl_memo = j->arenas ? &j->arenas[tid] : 0;
	if (j->swc) {   /* alignments from the device (K6): work on copies; a pass that had to request one is void and is replayed later */
		bb_swcache_t *c = &j->swc[i];
		int e;
		if (c->pending < 0) { tl_memo = 0; return; }          /* this pair is done */
		for (e = 0; e < 2; ++e) {
			const mem_alnreg_v *src = &j->rs[i << 1 | e].regs;
			a[e].n = src->n; a[e].m = src->n + 4;
			a[e].a = bb_malloc(a[e].m * sizeof(mem_alnreg_t));
			if (src->n) memcpy(a[e].a, src->a, src->n * sizeof(mem_alnreg_t));
		}
		c->pending = 0;
		if (bb_rescue_pe(j->opt, j->bns, j->pac, j->pes, &j->seqs[i << 1], a, c) < 0) { free(a[0].a); free(a[1].a); }
		else {
			for (e = 0; e < 2; ++e) {
				mem_alnreg_v *dst = &j->rs[i << 1 | e].regs;
				if (!(dst->m & BB_BORROWED)) free(dst->a);
				*dst = a[e];
			}
			c->pending = -1;
			free(c->v.a); c->v.a = 0; c->v.n = c->v.m = 0;
		}
		tl_memo = 0;
		return;
	}
	a[0] = j->rs[i << 1].regs; a[1] = j->rs[i << 1 | 1].regs;
	bb_rescue_pe(j->opt, j->bns, j->pac, j->pes, &j->seqs[i << 1], a, 0);
	j->rs[i << 1].regs = a[0]; j->rs[i << 1 | 1].regs = a[1];
	tl_memo = 0;
}

/* serve the mate-rescue alignments the pairs of this chunk asked for with one launch of K6; returns the number served, -1 if the
 * stage library has no K6 */
static int g_no_dev_sw;
static long sw_round(job_t *j)
{
	const mem_opt_t *opt = j->opt;
	const long n_pairs = j->n >> 1;
	long i, t = 0, k;
	bwag_swtask_t *tasks;
	const bwag_swres_t *res = 0;
	int rc;
	for (i = 0; i < n_pairs; ++i) if (j->swc[i].pending > 0) { size_t x; for (x = 0; x < j->swc[i].v.n; ++x) t += !j->swc[i].v.a[x].done; }
	if (t == 0) return 0;
	tasks = big_alloc_x(sizeof(bwag_swtask_t) * (size_t)t, 1);
	for (i = 0, k = 0; i < n_pairs; ++i) if (j->swc[i].pending > 0) {
		size_t x;
		for (x = 0; x < j->swc[i].v.n; ++x) {
			const bb_swent_t *e = &j->swc[i].v.a[x];
			const long r = i << 1 | e->which;
			bwag_swtask_t *q = &tasks[k];
			if (e->done) continue;
			q->t_beg = e->rb; q->tlen = (int32_t)(e->re - e->rb); q->q_beg = j->off[r]; q->qlen = j->seqs[r].l_seq;
			q->xtra = BWAG_SW_XSUBO | BWAG_SW_XSTART | (j->seqs[r].l_seq * opt->a < 250 ? BWAG_SW_XBYTE : 0) | (uint32_t)(opt->min_seed_len * opt->a);
			q->flags = BWAG_SWF_QREAD | BWAG_SWF_TREF | (e->is_rev ? BWAG_SWF_QREV : 0);
			++k;
		}
	}
	rc = bwag_localsw(j->batch, &j->swp, (int)t, tasks, 0, 0, &res);
	if (rc == BWAG_UNSUPPORTED) { big_free(tasks); return -1; }
	if (rc != 0) bb_fatal("mem_process_seqs", "local-alignment stage (mate rescue) failed: %s", bwag_last_error());
	for (i = 0, k = 0; i < n_pairs; ++i) if (j->swc[i].pending > 0) {
		size_t x;
		for (x = 0; x < j->swc[i].v.n; ++x) {
			bb_swent_t *e = &j->swc[i].v.a[x];
			if (e->done) continue;
			e->res.score = res[k].score; e->res.te = res[k].te; e->res.qe = res[k].qe; e->res.score2 = res[k].score2; e->res.te2 = res[k].te2; e->res.tb = res[k].tb; e->res.qb = res[k].qb;
			e->done = 1;
			++k;
		}
	}
	big_free(tasks);
	return t;
}

#define STACK_REGS 8
/* scratch copy of a read's regions: on the caller's stack when small, else on the heap (freed by drop_regs) */
static void copy_regs(mem_alnreg_v *dst, const mem_alnreg_v *src, mem_alnreg_t *stack)
{
	dst->n = 0;
	if (src->n <= STACK_REGS) { dst->a = stack; dst->m = STACK_REGS; }
	else { dst->a = 0; dst->m = 0; bb_vec_reserve(*dst, src->n + 1); }
	memcpy(dst->a, src->a, src->n * sizeof(mem_alnreg_t));
	dst->n = src->n;
}
static void drop_regs(mem_alnreg_v *v, const mem_alnreg_t *stack) { if (v->a != stack) free(v->a); }

/* worker2 of the reference (bwamem.c:1217-1233) for read / pair i, on a scratch copy of the regions */
static void run_sam(job_t *j, long i, int dry)
{
	const mem_opt_t *opt = j->opt;
	if (!(opt->flag & MEM_F_PE)) {
		rstate_t *r = &j->rs[i];
		mem_alnreg_v w = {0, 0, 0};
		mem_alnreg_t st0[STACK_REGS];
		uint32_t cg[128];
		bb_samctx_t sc = { opt, j->bns, j->pac, &r->gc, dry, cg, 128, 0 };
		copy_regs(&w, &r->regs, st0);
		bb_mark_primary_se(opt, (int)w.n, w.a, j->ids ? j->ids[i] : j->n_processed + i);
		if (opt->flag & MEM_F_PRIMARY5) bb_reorder_primary5(opt->T, &w);
		bb_reg2sam(&sc, &j->seqs[i], &w, 0, 0);
		drop_regs(&w, st0);
	} else {
		mem_alnreg_v w[2] = {{0, 0, 0}, {0, 0, 0}};
		mem_alnreg_t st0[STACK_REGS], st1[STACK_REGS];
		uint32_t cg[2][128];
		bb_samctx_t sc[2] = { { opt, j->bns, j->pac, &j->rs[i << 1].gc, dry, cg[0], 128, 0 }, { opt, j->bns, j->pac, &j->rs[i << 1 | 1].gc, dry, cg[1], 128, 0 } };
		copy_regs(&w[0], &j->rs[i << 1].regs, st0); copy_regs(&w[1], &j->rs[i << 1 | 1].regs, st1);
		bb_sam_pe(sc, j->pes, (uint64_t)(j->ids ? j->ids[i << 1] >> 1 : (j->n_processed >> 1) + i), &j->seqs[i << 1], w, 1);
		drop_regs(&w[0], st0); drop_regs(&w[1], st1);
	}
}

static void w_sam(void *d, long i, int tid)
{
	job_t *j = d;
	int pe = !!(j->opt->flag & MEM_F_PE);
	rstate_t *r0 = pe ? &j->rs[i << 1] : &j->rs[i], *r1 = pe ? &j->rs[i << 1 | 1] : 0;
	int dry = j->pass_dry;
	if (r0->done) return;
	tl_memo = j->arenas ? &j->arenas[tid] : 0;
	for (;;) {
		r0->gc.pending = 0; if (r1) r1->gc.pending = 0;
		run_sam(j, i, dry);
		if (r0->gc.pending || (r1 && r1->gc.pending)) {
			if (!dry) { /* text built on incomplete data: discard */
				if (pe) { free(j->seqs[i << 1].sam); free(j->seqs[i << 1 | 1].sam); j->seqs[i << 1].sam = j->seqs[i << 1 | 1].sam = 0; }
				else { free(j->seqs[i].sam); j->seqs[i].sam = 0; }
			}
			return;
		}
		if (!dry) { r0->done = 1; if (r1) r1->done = 1; return; }
		dry = 0; /* everything this read needs is cached: produce the text now */
	}
}

static void sw_par_from_opt(const mem_opt_t *opt, bwag_sw_par_t *p)
{
	p->a = opt->a; p->b = opt->b; p->o_del = opt->o_del; p->e_del = opt->e_del; p->o_ins = opt->o_ins; p->e_ins = opt->e_ins;
	p->w = opt->w; p->zdrop = opt->zdrop; p->pen_clip5 = opt->pen_clip5; p->pen_clip3 = opt->pen_clip3;
	memcpy(p->mat, opt->mat, 25);
}

/* host chaining path: download intervals and seeds, chain and filter on the host, upload the extension work */
static void host_chain_extend(job_t *j, bwag_batch_t *batch, const bwag_sw_par_t *swp, const bwag_seed_par_t *sp_, int nt)
{
	const bwag_seed_par_t sp = *sp_;
	int n = j->n, t;
	int64_t i, nc = 0, ns = 0;
	if (bwag_seed(batch, &sp, &j->seeds) != 0) bb_fatal("mem_process_seqs", "seeding stage failed: %s", bwag_last_error());
	PH(j, "seed_stage");

	j->tls = bb_calloc(bb_parallel_ids(), sizeof(tls_t));
	j->slice = big_alloc(((size_t)n + 1) * sizeof(rslice_t));
	bb_parallel_for_lane(j->lane, nt, w_chain, j, n);
	PH(j, "chain");

	j->chain_off = big_alloc_x(sizeof(int32_t) * ((size_t)n + 1), 1);
	for (i = 0; i < n; ++i) { nc += j->slice[i].nc; ns += j->slice[i].ns; }
	j->n_xchains = nc; j->n_xseeds = ns;
	j->xchains = big_alloc_x(sizeof(bwag_xchain_t) * ((size_t)nc + 1), 1);
	j->xseeds = big_alloc_x(sizeof(bwag_xseed_t) * ((size_t)ns + 1), 1);
	j->chain_rid = big_alloc(sizeof(int) * ((size_t)nc + 1));
	j->chain_frac = big_alloc(sizeof(float) * ((size_t)nc + 1));
	for (i = 0, nc = ns = 0; i < n; ++i) {
		j->chain_off[i] = (int32_t)nc;
		if (j->slice[i].nc) j->xchains[nc].seed_off = (int32_t)ns; /* read's seed base, consumed by w_flatten */
		nc += j->slice[i].nc; ns += j->slice[i].ns;
	}
	j->chain_off[n] = (int32_t)nc;
	bb_parallel_for_lane(j->lane, nt, w_flatten, j, n);
	for (t = 0; t < bb_parallel_ids(); ++t) {
		tls_t *x = &j->tls[t];
		bb_chainer_free(x->chainer);
		free(x->chains.a); free(x->xc.a); free(x->xs.a); free(x->c_rid.a); free(x->c_frac.a); free(x->srt.a);
	}
	free(j->tls); j->tls = 0;
	big_free(j->slice); j->slice = 0;
	PH(j, "flatten");

	dump_stage(j, swp, 1, nc, j->xchains, sizeof(bwag_xchain_t));
	if (bwag_extend(batch, swp, j->chain_off, j->xchains, j->n_xseeds, j->xseeds, &j->xregs) != 0)
		bb_fatal("mem_process_seqs", "extension stage failed: %s", bwag_last_error());
	PH(j, "extend_stage");

}

/* ---------------------------------------------------------------- device tail (stage 4)
 * Chunks of short reads are post-processed on the device (include/bwa_b200_dev.h, stage 4): the host only splices each
 * record's text with what it alone has (read name, quality string, comment).  Reads the device hands back -- and whole
 * batches whose options reach into what it does not do (-a, -V, -5) -- take the host-side post-processing below.
 * BWA_B200_TAIL=0 switches the stage off. */
static int g_no_tail;   /* the stage library has no stage 4 (the CPU oracle of the tests) */
typedef struct tail_shared_s { double *ptab[4]; } tail_shared_t;   /* per call: the insert-size term of a pair's score by distance (bwamem_pair.c:266) */

static int tail_wanted(const job_t *j)
{
	static int env_ = -1;
	int env = __atomic_load_n(&env_, __ATOMIC_RELAXED);
	if (env < 0) { const char *e = getenv("BWA_B200_TAIL"); env = e ? atoi(e) != 0 : 1; __atomic_store_n(&env_, env, __ATOMIC_RELAXED); }
	if (!env || j->sub_map || j->no_tail || __atomic_load_n(&g_no_tail, __ATOMIC_RELAXED)) return 0;
	if (j->opt->flag & (MEM_F_ALL | MEM_F_REF_HDR | MEM_F_PRIMARY5)) return 0;
	if ((j->opt->flag & MEM_F_PE) && (j->n & 1)) return 0;
	/* long noisy reads (thousands of bases) have many regions, region merges and supplementary records: stage 4 would hand nearly all
	 * of them back after having made their CIGAR requests once already (the pacbio workload) */
	if (j->n > 0 && j->off && j->off[j->n] / j->n > 1500) return 0;
	return 1;
}

static void tail_tables(const mem_opt_t *opt, const mem_pestat_t pes[4], tail_shared_t *ts)
{
	int d;
	memset(ts, 0, sizeof(*ts));
	for (d = 0; d < 4; ++d) {
		const mem_pestat_t *pe = &pes[d];
		int64_t n = (int64_t)pe->high - pe->low + 1, k;
		if (pe->failed || n <= 0 || n > 65536) continue;
		ts->ptab[d] = bb_malloc((size_t)n * sizeof(double));
		for (k = 0; k < n; ++k) { double ns = ((pe->low + k) - pe->avg) / pe->std; ts->ptab[d][k] = .721 * log(2. * erfc(fabs(ns) * M_SQRT1_2)) * opt->a; }
	}
}
static void tail_tables_free(tail_shared_t *ts) { int d; for (d = 0; d < 4; ++d) { free(ts->ptab[d]); ts->ptab[d] = 0; } }

/* a job over the reads idx[0..n_sub) of chunk j (pairs stay together): copies of their records, their global indices */
static job_t *sub_job(job_t *j, int n_sub, const int *idx)
{
	job_t *s = bb_calloc(1, sizeof(job_t));
	int64_t *ids = bb_malloc(sizeof(int64_t) * ((size_t)n_sub + 1));
	int k;
	s->opt = j->opt; s->bwt = j->bwt; s->bns = j->bns; s->pac = j->pac; s->pes = j->pes; s->swp = j->swp; s->lane = j->lane; s->chunk_id = j->chunk_id;
	s->n = n_sub; s->seqs = bb_malloc(sizeof(bseq1_t) * ((size_t)n_sub + 1));
	s->sub_map = bb_malloc(sizeof(int) * ((size_t)n_sub + 1));
	for (k = 0; k < n_sub; ++k) { s->seqs[k] = j->seqs[idx[k]]; s->sub_map[k] = idx[k]; ids[k] = j->ids ? j->ids[idx[k]] : j->n_processed + idx[k]; }
	s->ids = ids;
	if (j->pe_is) s->pe_is = bb_calloc((size_t)(n_sub >> 1) + 1, sizeof(uint64_t));
	return s;
}
static void sub_job_done(job_t *j, job_t *s)   /* hand the records to the parent's reads */
{
	int k;
	for (k = 0; k < s->n; ++k) j->seqs[s->sub_map[k]].sam = s->seqs[k].sam;
	free(s->seqs); free(s->sub_map); free((void *)s->ids); free(s->pe_is); free(s->pre_n); free(s->pre_beg); free(s->pre_regs); free(s);
}
/* the sub job's reads were seeded, chained and extended as part of the parent chunk: take their raw regions over instead of doing it again */
static void sub_job_take_regs(job_t *j, job_t *s)
{
	bwag_cregs_t cr;
	int64_t tot = 0;
	int k, rc = bwag_fetch_cregs(j->batch, s->n, s->sub_map, &cr);
	if (rc == BWAG_UNSUPPORTED) return;
	if (rc != 0) bb_fatal("mem_process_seqs", "fetching regions failed: %s", bwag_last_error());
	for (k = 0; k < s->n; ++k) tot += cr.n_regs[k];
	s->pre_n = bb_malloc(sizeof(int32_t) * ((size_t)s->n + 1)); s->pre_beg = bb_malloc(sizeof(int64_t) * ((size_t)s->n + 1)); s->pre_regs = bb_malloc(sizeof(bwag_creg_t) * ((size_t)tot + 1));
	memcpy(s->pre_n, cr.n_regs, sizeof(int32_t) * (size_t)s->n); memcpy(s->pre_beg, cr.reg_beg, sizeof(int64_t) * (size_t)s->n);
	if (tot) { int64_t mx = 0; for (k = 0; k < s->n; ++k) if (cr.reg_beg[k] + cr.n_regs[k] > mx) mx = cr.reg_beg[k] + cr.n_regs[k]; memcpy(s->pre_regs, cr.regs, sizeof(bwag_creg_t) * (size_t)mx); }
}

typedef struct { job_t *j; const bwag_sam_t *out; } splice_t;
static void w_splice(void *d, long u, int tid)   /* one read (pair): name + part A + QUAL + part B [+ comment] + newline */
{
	const splice_t *sp = d;
	job_t *j = sp->j;
	const int pe = !!(j->opt->flag & MEM_F_PE), n_ends = pe ? 2 : 1;
	int e;
	(void)tid;
	for (e = 0; e < n_ends; ++e) {
		const long i = pe ? (u << 1 | e) : u;
		const bwag_samrec_t *r = &sp->out->rec[i];
		bseq1_t *s = &j->seqs[i];
		size_t l_name, l_com, l_qual;
		char *w;
		if (!(r->flags & BWAG_REC_TEXT)) continue;
		l_name = strlen(s->name); l_com = s->comment ? strlen(s->comment) + 1 : 0; l_qual = s->qual ? (size_t)s->l_seq : 1;
		w = s->sam = bb_malloc(l_name + (size_t)r->len_a + l_qual + (size_t)r->len_b + l_com + 2);
		memcpy(w, s->name, l_name); w += l_name;
		memcpy(w, sp->out->text + r->off, (size_t)r->len_a); w += r->len_a;
		if (s->qual) { bb_copy_text(w, s->qual, s->l_seq, !!(r->flags & BWAG_REC_QREV)); w += s->l_seq; } else *w++ = '*';
		memcpy(w, sp->out->text + r->off + r->len_a, (size_t)r->len_b); w += r->len_b;
		if (s->comment) { *w++ = '\t'; memcpy(w, s->comment, l_com - 1); w += l_com - 1; }
		*w++ = '\n'; *w = 0;
	}
	if (pe && (sp->out->rec[u << 1].flags & BWAG_REC_TEXT) && strcmp(j->seqs[u << 1].name, j->seqs[u << 1 | 1].name) != 0)
		bb_fatal("mem_sam_pe", "paired reads have different names: \"%s\", \"%s\"\n", j->seqs[u << 1].name, j->seqs[u << 1 | 1].name);
}

static bwag_batch_t *run_to_regs(job_t *j, bwag_ctx_t *ctx, const bwag_sw_par_t *swp);
static void job_finish(job_t *j, bwag_ctx_t *ctx);
static void job_free(job_t *j);
static void w_pe_pairs(void *d, long c, int tid);

/* first half of a tail chunk, after bwag_tail_regs: the reads it handed back are aligned up to regions the host-side way now,
 * because the insert-size model of the batch needs their pairs too */
static void tail_phase0(job_t *j, bwag_ctx_t *ctx)
{
	const int pe = !!(j->opt->flag & MEM_F_PE);
	int i, n_sub = 0, *idx;
	if (!pe) return;                       /* single-end: everything handed back is collected after bwag_tail_sam */
	for (i = 0; i < j->n; i += 2) if (j->cflag[i] || j->cflag[i + 1]) n_sub += 2;
	if (n_sub == 0) return;
	idx = bb_malloc(sizeof(int) * (size_t)n_sub);
	for (i = 0, n_sub = 0; i < j->n; i += 2) if (j->cflag[i] || j->cflag[i + 1]) { idx[n_sub++] = i; idx[n_sub++] = i + 1; }
	j->sub0 = sub_job(j, n_sub, idx);
	free(idx);
	sub_job_take_regs(j, j->sub0);
	j->sub0->batch = run_to_regs(j->sub0, ctx, &j->sub0->swp);
	bwag_batch_end(j->sub0->batch); j->sub0->batch = 0;
	if (j->pe_is) {
		int k;
		bb_parallel_for_lane(j->lane, j->opt->n_threads > 0 ? j->opt->n_threads : 1, w_pe_pairs, j->sub0, ((j->sub0->n >> 1) + 1023) / 1024);
		for (k = 0; k < j->sub0->n; k += 2) j->pe_is[j->sub0->sub_map[k] >> 1] = j->sub0->pe_is[k >> 1];
	}
	PH(j, "tail_sub0");
}

/* second half of a tail chunk: pairing + records on the device, text splice, then the reads that were handed back */
static void tail_finish(job_t *j, bwag_ctx_t *ctx)
{
	const mem_opt_t *opt = j->opt;
	const int nt = opt->n_threads > 0 ? opt->n_threads : 1, pe = !!(opt->flag & MEM_F_PE);
	const long n_units = pe ? j->n >> 1 : j->n;
	bwag_sam_t out;
	splice_t sp;
	int i, n_sub = 0, *idx;
	if (bwag_tail_sam(j->batch, opt, j->pes, j->ts ? (const double *const *)j->ts->ptab : 0, 0, j->n_processed, bwa_rg_id[0] ? bwa_rg_id : 0, &out) != 0)
		bb_fatal("mem_process_seqs", "stage 4 (records) failed: %s", bwag_last_error());
	PH(j, "tail_sam");
	sp.j = j; sp.out = &out;
	bb_parallel_for_lane(j->lane, nt, w_splice, &sp, n_units);
	PH(j, "splice");
	/* reads handed back here (mate rescue would align, XA, several records, ...): host-side post-processing from scratch */
#define HANDED_BACK(i_) ((out.rec[i_].flags & BWAG_REC_COMPLEX) && !(pe && j->sub0 && (j->cflag[(i_) & ~1] || j->cflag[(i_) | 1])))
	for (i = 0; i < j->n; ++i) if (HANDED_BACK(i)) ++n_sub;
	if (n_sub) {
		idx = bb_malloc(sizeof(int) * (size_t)n_sub);
		for (i = 0, n_sub = 0; i < j->n; ++i) if (HANDED_BACK(i)) idx[n_sub++] = i;
		j->sub1 = sub_job(j, n_sub, idx);
		free(idx);
		sub_job_take_regs(j, j->sub1);
	}
#undef HANDED_BACK
	bwag_batch_end(j->batch); j->batch = 0;   /* out.* is gone from here on */
	if (j->sub1) {
		free(j->sub1->pe_is); j->sub1->pe_is = 0;
		j->sub1->batch = run_to_regs(j->sub1, ctx, &j->sub1->swp);
		job_finish(j->sub1, ctx);
		sub_job_done(j, j->sub1); j->sub1 = 0;
	}
	if (j->sub0) { job_finish(j->sub0, ctx); sub_job_done(j, j->sub0); j->sub0 = 0; }
	PH(j, "tail_subs");
	job_free(j);
	PH(j, "cleanup");
}

/* stages up to de-duplicated regions for all reads of the job (worker1 of the reference) */
static bwag_batch_t *run_to_regs(job_t *j, bwag_ctx_t *ctx, const bwag_sw_par_t *swp)
{
	const mem_opt_t *opt = j->opt;
	bwag_batch_t *batch;
	bwag_seed_par_t sp;
	int nt = opt->n_threads > 0 ? opt->n_threads : 1, n = j->n;
	int64_t i, tot = 0;

	j->off = big_alloc_x(sizeof(int64_t) * ((size_t)n + 1), 1);
	for (i = 0; i < n; ++i) { j->off[i] = tot; tot += j->seqs[i].l_seq; }
	j->off[n] = tot;
	j->codes = big_alloc_x((size_t)tot + 16, 1);
	bb_parallel_for_lane(j->lane, nt, w_encode, j, n);
	PH(j, "encode");

	batch = bwag_batch_begin(ctx, n, j->codes, j->off);
	if (!batch) bb_fatal("mem_process_seqs", "cannot start a device batch: %s", bwag_last_error());
	PH(j, "batch_begin");
	sp.min_seed_len = opt->min_seed_len;
	sp.split_len = (int)(opt->min_seed_len * opt->split_factor + .499);
	sp.split_width = opt->split_width;
	sp.max_occ = opt->max_occ;
	sp.max_mem_intv = opt->max_mem_intv;
	{   /* chaining on the device, including the seed-level SW filter of long reads (mem_flt_chained_seeds, bwamem.c:626-641: K3 lists
	     * the alignments, K6 makes them, K3b applies them); on the host only if the stage is not provided */
		static int no_dev_chain = 0;   /* set once if the stage library has no device chaining (the CPU oracle of the tests) */
		int dev_chain = !__atomic_load_n(&no_dev_chain, __ATOMIC_RELAXED) && !(getenv("BWA_B200_DEVICE_CHAIN") && atoi(getenv("BWA_B200_DEVICE_CHAIN")) == 0);
		if (j->pre_n) {   /* regions inherited from the parent chunk */
			j->cregs.n_regs = j->pre_n; j->cregs.reg_beg = j->pre_beg; j->cregs.regs = j->pre_regs; j->have_cregs = 1;
			dev_chain = 0;
		}
		if (getenv("BWA_B200_DEVICE_SEEDSW") && atoi(getenv("BWA_B200_DEVICE_SEEDSW")) == 0)   /* A/B switch: long reads chain and filter on the host */
			for (i = 0; i < n && dev_chain; ++i) {
				int l = j->seqs[i].l_seq;
				double min_l = opt->min_chain_weight ? 1.1f * opt->min_chain_weight : 5.5f * log(l > 0 ? l : 1);
				if (l > 0 && !(min_l > 0.05f * l)) dev_chain = 0;
			}
		if (dev_chain) {
			bwag_chain_par_t cp;
			bwag_contigs_t ctg;
			int rc, c, n_seqs = j->bns->n_seqs;
			int64_t *c_off = bb_malloc(sizeof(int64_t) * n_seqs);
			int32_t *c_len = bb_malloc(sizeof(int32_t) * n_seqs);
			uint8_t *c_alt = bb_malloc(n_seqs);
			for (c = 0; c < n_seqs; ++c) { c_off[c] = j->bns->anns[c].offset; c_len[c] = j->bns->anns[c].len; c_alt[c] = !!j->bns->anns[c].is_alt; }
			ctg.n_seqs = n_seqs; ctg.offset = c_off; ctg.len = c_len; ctg.is_alt = c_alt;
			cp.w = opt->w; cp.max_chain_gap = opt->max_chain_gap; cp.max_occ = opt->max_occ; cp.min_seed_len = opt->min_seed_len;
			cp.min_chain_weight = opt->min_chain_weight; cp.max_chain_extend = opt->max_chain_extend; cp.mask_level = opt->mask_level; cp.drop_ratio = opt->drop_ratio;
			const int want_tail = tail_wanted(j);
			if (bwag_seed(batch, &sp, 0) != 0) bb_fatal("mem_process_seqs", "seeding stage failed: %s", bwag_last_error());
			PH(j, "seed_stage");
			rc = bwag_chain_extend(batch, &cp, swp, &ctg, want_tail ? 0 : &j->cregs);
			if (rc == 0 && want_tail) {   /* stage 4: de-duplication, CIGAR requests and K5 on the device; the regions never come to the host */
				const uint64_t *pis = 0;
				int rc2;
				PH(j, "chain_extend");
				rc2 = bwag_tail_regs(batch, opt, swp, &pis, &j->cflag);
				if (rc2 == 0) {
					free(c_off); free(c_len); free(c_alt);
					j->tail = 1;
					if (j->pe_is && pis) memcpy(j->pe_is, pis, sizeof(uint64_t) * (size_t)(n >> 1));
					PH(j, "tail_regs");
					return batch;
				}
				if (rc2 == BWAG_UNSUPPORTED) __atomic_store_n(&g_no_tail, 1, __ATOMIC_RELAXED);
				else if (rc2 != BWAG_DECLINED) bb_fatal("mem_process_seqs", "stage 4 (regions) failed: %s", bwag_last_error());
				rc = bwag_chain_extend(batch, &cp, swp, &ctg, &j->cregs);   /* host-side post-processing after all: bring the regions over */
			}
			free(c_off); free(c_len); free(c_alt);
			if (rc == BWAG_UNSUPPORTED) { __atomic_store_n(&no_dev_chain, 1, __ATOMIC_RELAXED); dev_chain = 0; }
			else if (rc == BWAG_DECLINED) dev_chain = 0;
			else if (rc != 0) bb_fatal("mem_process_seqs", "chain+extend stage failed: %s", bwag_last_error());
			else { j->have_cregs = 1; PH(j, "chain_extend"); }
		}
		if (!dev_chain && !j->pre_n) host_chain_extend(j, batch, swp, &sp, nt);
	}

	{ /* region arrays of all reads in one block; the rare array that must grow (mate rescue) moves to the heap */
		int64_t tot_regs = 0;
		j->reg_off = big_alloc(sizeof(int64_t) * ((size_t)n + 1));
		for (i = 0; i < n; ++i) { j->reg_off[i] = tot_regs; tot_regs += j->have_cregs ? j->cregs.n_regs[i] : (j->chain_off[i + 1] > j->chain_off[i] ? j->xregs.n_regs[i] : 0); }
		j->reg_pool = big_alloc(sizeof(mem_alnreg_t) * ((size_t)tot_regs + 1));
	}
	j->rs = big_alloc(((size_t)n + 1) * sizeof(rstate_t));
	j->arenas = bb_calloc(bb_parallel_ids(), sizeof(memo_arena_t));
	bb_parallel_for_lane(j->lane, nt, w_zero_rs, j, ((long)n + 4095) / 4096);
	for (;;) { /* de-duplicate; repeat for reads whose merge test needed a device alignment */
		int64_t left = 0;
		bb_parallel_for_lane(j->lane, nt, w_dedup, j, n);
		PH(j, "dedup");
		for (i = 0; i < n; ++i) left += !j->rs[i].dedup_done;
		if (global_round(j, batch, swp) == 0 && left) bb_fatal("mem_process_seqs", "internal error: pending reads without requests");
		PH(j, "global_round");
		if (left == 0) break;
	}
	return batch;
}

static void w_pe_pairs(void *d, long c, int tid)   /* insert-size candidates of 1024 pairs */
{
	job_t *j = d;
	long i, e = (c + 1) * 1024 < j->n >> 1 ? (c + 1) * 1024 : j->n >> 1;
	(void)tid;
	for (i = c * 1024; i < e; ++i) j->pe_is[i] = bb_pestat_pair(j->opt, j->bns->l_pac, &j->rs[i << 1].regs, &j->rs[i << 1 | 1].regs);
}

static void w_free(void *d, long i, int tid)
{
	job_t *j = d;
	(void)tid;
	if (!(j->rs[i].regs.m & BB_BORROWED)) free(j->rs[i].regs.a);
	gcache_free(&j->rs[i].gc);
}

static void job_free(job_t *j)
{
	if (j->rs) bb_parallel_for_lane(j->lane, j->opt->n_threads > 0 ? j->opt->n_threads : 1, w_free, j, j->n);
	memo_arenas_free(j->arenas, bb_parallel_ids()); j->arenas = 0;
	{ int b; for (b = 0; b < j->n_blocks; ++b) big_free(j->blocks[b]); free(j->blocks); j->blocks = 0; j->n_blocks = j->m_blocks = 0; }
	big_free(j->reg_pool); big_free(j->reg_off);
	big_free(j->rs); big_free(j->off); big_free(j->codes); big_free(j->chain_off); big_free(j->xchains); big_free(j->xseeds); big_free(j->chain_rid); big_free(j->chain_frac);
}

/* second half of a chunk: (PE: mate rescue,) SAM with as many device rounds as cache misses require */
static void job_finish(job_t *j, bwag_ctx_t *ctx)
{
	const mem_opt_t *opt = j->opt;
	int nt = opt->n_threads > 0 ? opt->n_threads : 1, pe = !!(opt->flag & MEM_F_PE);
	long n_units = pe ? j->n >> 1 : j->n;
	if (!j->batch) {
		j->batch = bwag_batch_begin(ctx, j->n, j->codes, j->off);
		if (!j->batch) bb_fatal("mem_process_seqs", "cannot start a device batch: %s", bwag_last_error());
	}
	if (pe && !(opt->flag & MEM_F_NO_RESCUE)) {   /* mate rescue; its local alignments are K6's, asked for pair by pair and served in rounds */
		static int env_ = -1;
		int env = __atomic_load_n(&env_, __ATOMIC_RELAXED);
		if (env < 0) { const char *e = getenv("BWA_B200_DEVICE_SW"); env = e ? atoi(e) != 0 : 1; __atomic_store_n(&env_, env, __ATOMIC_RELAXED); }
		if (env && !__atomic_load_n(&g_no_dev_sw, __ATOMIC_RELAXED)) j->swc = bb_calloc((size_t)n_units + 1, sizeof(bb_swcache_t));
		for (;;) {
			long left = 0, u, served;
			bb_parallel_for_lane(j->lane, nt, w_rescue, j, n_units);
			PH(j, "rescue");
			if (!j->swc) break;
			for (u = 0; u < n_units; ++u) left += j->swc[u].pending >= 0;
			if (left == 0) break;
			served = sw_round(j);
			PH(j, "sw_round");
			if (served < 0) {   /* no K6 behind this stage library (the CPU oracle of the tests): align on the host */
				__atomic_store_n(&g_no_dev_sw, 1, __ATOMIC_RELAXED);
				for (u = 0; u < n_units; ++u) free(j->swc[u].v.a);
				free(j->swc); j->swc = 0;
			} else if (served == 0) bb_fatal("mem_process_seqs", "internal error: unfinished mate rescue without requests");
		}
		if (j->swc) { free(j->swc); j->swc = 0; }
	}
	for (j->pass_dry = 0;; j->pass_dry = 0) { /* SAM; a read that misses an alignment is retried after a device round */
		long i, left = 0;
		bb_parallel_for_lane(j->lane, nt, w_sam, j, n_units);
		PH(j, "sam");
		for (i = 0; i < j->n; ++i) left += !j->rs[i].done;
		if (left == 0) break;
		if (global_round(j, j->batch, &j->swp) == 0) bb_fatal("mem_process_seqs", "internal error: unfinished reads without requests");
		PH(j, "global_round");
	}
	bwag_batch_end(j->batch); j->batch = 0;
	PH(j, "batch_end");
	job_free(j);
	PH(j, "cleanup");
}

static void w_encode(void *, long, int); static void w_chain(void *, long, int); static void w_flatten(void *, long, int); static void w_zero_rs(void *, long, int);
static void w_dedup(void *, long, int); static void w_gcount(void *, long, int); static void w_gfill(void *, long, int); static void w_gstore(void *, long, int);
static void w_rescue(void *, long, int); static void w_sam(void *, long, int); static void w_free(void *, long, int); static void w_pe_pairs(void *, long, int);
static pthread_once_t g_diag_once = PTHREAD_ONCE_INIT;
static void diag_init(void)   /* diagnostics switches are read once per process */
{
	g_prof = getenv("BWA_B200_PROFILE") != 0;
	g_trace = getenv("BWA_B200_TRACE") ? atoi(getenv("BWA_B200_TRACE")) : 0;
	bb_parallel_name(w_encode, "encode"); bb_parallel_name(w_chain, "chain"); bb_parallel_name(w_flatten, "flatten"); bb_parallel_name(w_zero_rs, "zero_rs");
	bb_parallel_name(w_dedup, "dedup"); bb_parallel_name(w_gcount, "g_count"); bb_parallel_name(w_gfill, "g_fill"); bb_parallel_name(w_gstore, "g_store");
	bb_parallel_name(w_rescue, "rescue"); bb_parallel_name(w_sam, "sam"); bb_parallel_name(w_free, "free"); bb_parallel_name(w_pe_pairs, "pe_pairs");
}

typedef struct { job_t *jobs; int n_jobs; volatile int next; bwag_ctx_t *ctx; int phase, lane, pe; } lane_arg_t;

static void *lane_main(void *a_)
{
	lane_arg_t *a = a_;
	for (;;) {
		int k = __sync_fetch_and_add(&a[-a->lane].next, 1);   /* the shared counter lives in lane 0's record */
		job_t *j;
		if (k >= a->n_jobs) break;
		j = &a->jobs[k];
		j->lane = a->lane; j->chunk_id = k;
		if (g_trace > 0) j->t_last = trace_now();
		if (a->phase == 0) {
			j->batch = run_to_regs(j, a->ctx, &j->swp);
			if (j->tail) {   /* stage 4 runs this chunk's post-processing on the device; its batch object stays alive (regions, CIGARs in HBM) */
				tail_phase0(j, a->ctx);
				if (!a->pe) tail_finish(j, a->ctx);
			} else if (a->pe) {   /* the insert-size model needs every chunk first; with few chunks each keeps its device batch (reads resident) for the second phase */
				if (a->n_jobs > 6) { bwag_batch_end(j->batch); j->batch = 0; }
				if (j->pe_is) { bb_parallel_for_lane(j->lane, j->opt->n_threads > 0 ? j->opt->n_threads : 1, w_pe_pairs, j, ((j->n >> 1) + 1023) / 1024); PH(j, "pe_pairs"); }
			}
			else job_finish(j, a->ctx);
		} else if (j->tail) tail_finish(j, a->ctx);
		else job_finish(j, a->ctx);
	}
	return 0;
}

static void run_lanes(job_t *jobs, int n_jobs, int n_lanes, bwag_ctx_t *ctx, int phase, int pe)
{
	lane_arg_t la[8];
	pthread_t th[8];
	int l;
	for (l = 0; l < n_lanes; ++l) { la[l].jobs = jobs; la[l].n_jobs = n_jobs; la[l].next = 0; la[l].ctx = ctx; la[l].phase = phase; la[l].lane = l; la[l].pe = pe; }
	for (l = 1; l < n_lanes; ++l) pthread_create(&th[l], 0, lane_main, &la[l]);
	lane_main(&la[0]);
	for (l = 1; l < n_lanes; ++l) pthread_join(th[l], 0);
}

/* The batch is cut into chunks that travel through the stages on `lanes` independent lanes (own CUDA stream and
 * device buffers, own host-thread pool): while one chunk sits in a GPU stage the other runs a host phase, so
 * kernels, PCIe copies and host work overlap.  BWA_B200_LANES / BWA_B200_CHUNK override the defaults. */
void mem_process_seqs(const mem_opt_t *opt, const bwt_t *bwt, const bntseq_t *bns, const uint8_t *pac,
                      int64_t n_processed, int n, bseq1_t *seqs, const mem_pestat_t *pes0)
{
	job_t *jobs;
	mem_pestat_t pes[4];
	bwag_ctx_t *ctx;
	double ctime = bb_cputime(), rtime = bb_realtime();
	static volatile int n_calls;   /* mem_process_seqs calls in flight (the command line keeps two) */
	int pe = !!(opt->flag & MEM_F_PE), n_lanes, n_jobs, k;
	long chunk = pe ? 1 << 18 : 1 << 17, start;
	uint64_t *pe_is = 0;
	const char *e;

	if (n <= 0) return;
	/* lanes of all calls share one GPU and one pool of host threads: about four in total is the sweet spot (tools/sweep_lanes.sh) */
	n_lanes = __sync_add_and_fetch(&n_calls, 1) >= 2 ? 2 : 3;
	if ((e = getenv("BWA_B200_LANES")) != 0) n_lanes = atoi(e);
	if ((e = getenv("BWA_B200_CHUNK")) != 0) chunk = atol(e);
	if (n_lanes < 1) n_lanes = 1;
	if (n_lanes > 8) n_lanes = 8;
	if (chunk < 2) chunk = 2;
	chunk &= ~1L;
	if (n <= chunk + chunk / 2) chunk = n;                 /* do not split off a small tail */
	n_jobs = (int)((n + chunk - 1) / chunk);
	if (n_lanes > n_jobs) n_lanes = n_jobs;
	ctx = bb_device_attach(bwt, bns, pac);
	jobs = bb_calloc((size_t)n_jobs, sizeof(job_t));
	for (k = 0, start = 0; k < n_jobs; ++k, start += chunk) {
		job_t *j = &jobs[k];
		j->opt = opt; j->bwt = bwt; j->bns = bns; j->pac = pac; j->pes = pes;
		j->n = (int)(start + chunk <= n ? chunk : n - start);
		j->seqs = seqs + start;
		j->n_processed = n_processed + start;
		sw_par_from_opt(opt, &j->swp);
	}
	if (pe && !pes0) {
		pe_is = big_alloc(sizeof(uint64_t) * ((size_t)(n >> 1) + 1));
		for (k = 0, start = 0; k < n_jobs; ++k, start += chunk) jobs[k].pe_is = pe_is + (start >> 1);
	}
	pthread_once(&g_diag_once, diag_init);
	ph(0);
	if (g_trace > 0) g_trace_t0 = bb_realtime();
	run_lanes(jobs, n_jobs, n_lanes, ctx, 0, pe);
	if (pe) {
		if (pes0) memcpy(pes, pes0, 4 * sizeof(mem_pestat_t));
		else {
			bb_pestat_from_pairs(opt, n >> 1, pe_is, pes);
		}
		big_free(pe_is);
		{
			tail_shared_t ts;
			int any = 0;
			for (k = 0; k < n_jobs; ++k) any |= jobs[k].tail;
			memset(&ts, 0, sizeof(ts));
			if (any) { tail_tables(opt, pes, &ts); for (k = 0; k < n_jobs; ++k) jobs[k].ts = &ts; }
			ph("pestat");
			if (g_trace > 0) fprintf(stderr, "[trace] pestat done %8.1f\n", trace_now());
			run_lanes(jobs, n_jobs, n_lanes, ctx, 1, pe);
			tail_tables_free(&ts);
		}
	}
	free(jobs);
	__sync_sub_and_fetch(&n_calls, 1);
	bb_parallel_report();
	if (g_trace > 0) fprintf(stderr, "[trace] batch done %8.1f\n", trace_now());
	if (bwa_verbose >= 3)
		fprintf(stderr, "[M::%s] Processed %d reads in %.3f CPU sec, %.3f real sec\n", __func__, n, bb_cputime() - ctime, bb_realtime() - rtime);
}

/* ---------------------------------------------------------------- single-read conveniences of the reference API */

mem_alnreg_v mem_align1(const mem_opt_t *opt, const bwt_t *bwt, const bntseq_t *bns, const uint8_t *pac, int l_seq, const char *seq_)
{
	job_t j;
	bseq1_t s;
	bwag_sw_par_t swp;
	bwag_batch_t *batch;
	mem_alnreg_v out;
	memset(&j, 0, sizeof(j)); memset(&s, 0, sizeof(s));
	s.l_seq = l_seq; s.seq = bb_malloc((size_t)l_seq + 1); memcpy(s.seq, seq_, l_seq);
	j.opt = opt; j.bwt = bwt; j.bns = bns; j.pac = pac; j.n = 1; j.seqs = &s; j.no_tail = 1;
	sw_par_from_opt(opt, &swp);
	batch = run_to_regs(&j, bb_device_attach(bwt, bns, pac), &swp);
	bwag_batch_end(batch);
	{   /* the caller owns (and frees) the array: never hand out a slice of the batch-wide region block */
		const mem_alnreg_v *r = &j.rs[0].regs;
		out.n = r->n; out.m = r->n + 4;
		out.a = bb_malloc(out.m * sizeof(mem_alnreg_t));
		if (r->n) memcpy(out.a, r->a, r->n * sizeof(mem_alnreg_t));
	}
	bb_mark_primary_se(opt, (int)out.n, out.a, lrand48());
	job_free(&j);
	free(s.seq);
	return out;
}

static const bwt_t *any_resident_bwt(const uint8_t *pac_unused)
{
	int i;
	(void)pac_unused;
	for (i = 0; i < 8; ++i) if (g_dev[i].ctx) return g_dev[i].bwt;
	return 0;
}

mem_aln_t mem_reg2aln(const mem_opt_t *opt, const bntseq_t *bns, const uint8_t *pac, int l_seq, const char *seq, const mem_alnreg_t *ar)
{
	/* needs the index on the device: the caller must have aligned with this index before (as example.c does) */
	job_t j;
	bseq1_t s;
	rstate_t rs;
	bwag_sw_par_t swp;
	bwag_batch_t *batch;
	bb_samctx_t sc = { opt, bns, pac, &rs.gc, 1 };
	mem_aln_t a;
	int64_t off[2] = {0, l_seq};
	int k;
	const bwt_t *bwt = any_resident_bwt(pac);
	if (!bwt) bb_fatal("mem_reg2aln", "no index resident on the GPU; call mem_align1/mem_process_seqs first");
	tl_memo = 0;
	memset(&j, 0, sizeof(j)); memset(&s, 0, sizeof(s)); memset(&rs, 0, sizeof(rs));
	s.l_seq = l_seq; s.seq = bb_malloc((size_t)l_seq + 1);
	for (k = 0; k < l_seq; ++k) { unsigned char c = (unsigned char)seq[k]; c = c < 5 ? c : bb_nt4_table[c]; s.seq[k] = (char)(c > 4 ? 4 : c); }
	a = bb_reg2aln(&sc, l_seq, s.seq, ar);
	if (rs.gc.pending) {
		free(a.cigar);
		j.opt = opt; j.bns = bns; j.pac = pac; j.n = 1; j.seqs = &s; j.rs = &rs;
		sw_par_from_opt(opt, &swp);
		batch = bwag_batch_begin(bb_device_attach(bwt, bns, pac), 1, (const uint8_t *)s.seq, off);
		if (!batch) bb_fatal("mem_reg2aln", "cannot start a device batch: %s", bwag_last_error());
		global_round(&j, batch, &swp);
		bwag_batch_end(batch);
		rs.gc.pending = 0;
		a = bb_reg2aln(&sc, l_seq, s.seq, ar);
	}
	{ int b; for (b = 0; b < j.n_blocks; ++b) big_free(j.blocks[b]); free(j.blocks); }
	gcache_free(&rs.gc);
	free(s.seq);
	return a;
}

/* release the SAM text of a batch the way the reference's caller does (fastmap.c:114-119), in one call */
static void w_free_sam(void *d, long c, int tid)
{
	bseq1_t *seqs = d;
	long i;
	(void)tid;
	for (i = c * 1024; i < (c + 1) * 1024; ++i) { free(seqs[i].sam); seqs[i].sam = 0; }
}
void bb_batch_free_sam(int n, bseq1_t *seqs)
{
	int i, full = n / 1024;
	bb_parallel_for(8, w_free_sam, seqs, full);   /* the records were allocated by many threads: free them in parallel too */
	for (i = full * 1024; i < n; ++i) { free(seqs[i].sam); seqs[i].sam = 0; }
}

/* total length of the SAM text of a batch; if dst != NULL the records are concatenated into it */
int64_t bb_batch_cat_sam(int n, const bseq1_t *seqs, char *dst)
{
	int64_t l = 0;
	int i;
	for (i = 0; i < n; ++i)
		if (seqs[i].sam) { size_t k = strlen(seqs[i].sam); if (dst) memcpy(dst + l, seqs[i].sam, k); l += (int64_t)k; }
	return l;
}

/* move the SAM pointers of a batch into a caller-owned array (so that a benchmark can release them outside its
 * timed region); returns the array, to be passed to bb_batch_free_detached */
char **bb_batch_detach_sam(int n, bseq1_t *seqs)
{
	char **p = bb_malloc(sizeof(char *) * ((size_t)n + 1));
	int i;
	for (i = 0; i < n; ++i) { p[i] = seqs[i].sam; seqs[i].sam = 0; }
	return p;
}

static void w_free_ptrs(void *d, long c, int tid)
{
	char **p = d;
	long i;
	(void)tid;
	for (i = c * 1024; i < (c + 1) * 1024; ++i) free(p[i]);
}
void bb_batch_free_detached(int n, char **p)
{
	int i, full = n / 1024;
	bb_parallel_for(8, w_free_ptrs, p, full);
	for (i = full * 1024; i < n; ++i) free(p[i]);
	free(p);
}
