/* bwag_mem.cu -- host drivers of `mem`'s device stages: seeding (K1, K1f, K1b, K2), chaining and extension (K3, K4),
 * the global alignments (K5, K5L), the local ones (K6) and stage 4 (bwag_tail.cu).  The kernels live in their own files. */
#include <math.h>
#include "bwag_drv.h"

#ifndef K1_COMPACT_DEFAULT
#define K1_COMPACT_DEFAULT 1   /* k_smem_c unless BWA_B200_K1_COMPACT=0 */
#endif
#define SEEDSW_MAXLEN 200   /* the seed-level filter aligns windows shorter than this on both axes (bwamem.c:591,612) */

/* K3 cycle histograms of a build with -DBWAG_K3_CLOCKS (tools/chain_bench.py): by seeds per read (0..64, then > 64) the reads and the
 * clock64() cycles of their chaining loop, mem_chain_flt and chain_emit, then the reads by chains per read (0..32, then > 32) */
#ifdef BWAG_K3_CLOCKS
static pthread_mutex_t g_k3clk_mu = PTHREAD_MUTEX_INITIALIZER;
static u64 g_k3clk[BWAG_K3CLK_WORDS];
#endif
extern "C" int bwag_k3_clocks(uint64_t *out, int reset)
{
#ifdef BWAG_K3_CLOCKS
	pthread_mutex_lock(&g_k3clk_mu);
	if (out) memcpy(out, g_k3clk, sizeof(g_k3clk));
	if (reset) memset(g_k3clk, 0, sizeof(g_k3clk));
	pthread_mutex_unlock(&g_k3clk_mu);
	return 0;
#else
	(void)out; (void)reset;
	return -1;
#endif
}
/* K1 counters of a build with -DBWAG_K1_CLOCKS (tools/k1_bench.py): BWAG_K1CLK_WORDS words, include/bwa_b200_dev.h */
#ifdef BWAG_K1_CLOCKS
static pthread_mutex_t g_k1clk_mu = PTHREAD_MUTEX_INITIALIZER;
static u64 g_k1clk[BWAG_K1CLK_WORDS];
#endif
extern "C" int bwag_k1_clocks(uint64_t *out, int reset)
{
#ifdef BWAG_K1_CLOCKS
	pthread_mutex_lock(&g_k1clk_mu);
	if (out) memcpy(out, g_k1clk, sizeof(g_k1clk));
	if (reset) memset(g_k1clk, 0, sizeof(g_k1clk));
	pthread_mutex_unlock(&g_k1clk_mu);
	return 0;
#else
	(void)out; (void)reset;
	return -1;
#endif
}
#ifdef BWAG_K3_CLOCKS
static void k3clk_add(const u32 *rec, int n)
{
	pthread_mutex_lock(&g_k3clk_mu);
	for (int r = 0; r < n; ++r, rec += 5) {
		const int t = rec[0] > 64 ? 65 : (int)rec[0], ch = rec[1] > 32 ? 33 : (int)rec[1];
		u64 *h = g_k3clk + 4 * t;
		h[0] += 1; h[1] += rec[2]; h[2] += rec[3]; h[3] += rec[4];
		g_k3clk[4 * 66 + ch] += 1;
	}
	pthread_mutex_unlock(&g_k3clk_mu);
}
#endif

/* ------------------------------------------------------------------------------------------------ stage 1 */

/* K1 (+ K1f, K1b, K2 for `mem`).  fm != NULL: K1 alone, in its fastmap form, with the same scratch sizing and repeats; the read's
 * matches stay in HBM (b->n_intv of them in the pool) */
int seed_impl(bwag_batch_t *b, const bwag_seed_par_t *par, const FmK1 *fm, bwag_seeds_t *out)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	const int n = b->n;
	/* pools: typical short reads need ~8 intervals / ~10 seeds each; long noisy reads against a large index pick up chance matches of
	 * their minimum seed length all along (measured: 10-kbp reads at 10 % error against 3 Gbp), hence the per-base terms */
	i64 cap_intv = (i64)n * 16 + b->total_bases / 4 + 1024, cap_seeds = (i64)n * 32 + b->total_bases / 2 + 4096;
	if (getenv("BWA_B200_TEST_SMALL_POOLS")) { cap_intv = n / 2 + 8; cap_seeds = n / 2 + 8; }   /* test hook: start with pools that overflow, so that the repeat-with-reported-sizes path runs */
	int cap_list = b->max_len + 1, cap_mem = 2 * b->max_len + 64;
	/* k_smem_c (compact candidate lists, bwag_smem.cu) needs the short-string table; BWA_B200_K1_COMPACT=0 selects k_smem */
	bool k1c = false;
#ifndef K1_PACKED8
	{
		const char *e = getenv("BWA_B200_K1_COMPACT");
		k1c = (e ? atoi(e) != 0 : K1_COMPACT_DEFAULT) && c->ix.ktab_k > 0 && !fm;   /* fastmap needs every match's interval (-I): k_smem */
	}
	/* k_smem_c checks every list and result append, so long reads start with scratch for what they typically need (a few
	 * candidates with an interval per list, a result per ~4 bases) instead of the worst case: more lanes fit the scratch budget.
	 * A lane that runs out sets a flag and the stage is repeated with the worst-case sizes. */
	if (k1c && b->max_len > 2048) { cap_list = 1024; cap_mem = b->max_len / 4 + 256; }
	if (k1c && getenv("BWA_B200_TEST_SMALL_K1")) { cap_list = 9; cap_mem = 3; }   /* test hook: the repeat-with-larger-scratch path (9: the shared slots + one entry of global tail) */
#endif
	SeedArgs a;
	memset(&a, 0, sizeof(a));
	for (int attempt = 0;; ++attempt) {
		const int groups_per_block = K1_THREADS;   /* one lane per read */
		/* shared memory of a block: the heads of both candidate lists + one read slot per lane (odd number of words) */
		int qstride = (((b->max_len + 6) >> 2) | 1) << 2;
		/* + a 2-bit packed copy of each read (the keys of the short-string table): 16 bases per word, one spare word, odd word count */
		int pstride = c->ix.ktab_k ? ((((b->max_len + 15) >> 4) + 1) | 1) << 2 : 0;
		int nstride = 0;
#ifdef K1_PACKED8   /* variant: packed read + N bitmap only, eight list entries per list in shared memory (bwag_smem.cu) */
		pstride = ((((b->max_len + 15) >> 4) + 1) | 1) << 2;
		nstride = (((b->max_len + 31) >> 5) | 1) << 2;
		qstride = 0;
#endif
		size_t smem = (size_t)2 * K1_SLOTS * K1_THREADS * 16 + (size_t)K1_THREADS * (qstride + pstride + nstride);
#ifdef K1_NO_QSMEM
		qstride = 0; pstride = 0; smem = (size_t)2 * K1_SLOTS * K1_THREADS * 16;
#endif
		bool want_pack = pstride != 0;
		if (k1c) {   /* list heads + the packed copy; reads too long for that are read in place (pstride = 0) */
			qstride = 0;
			smem = (size_t)2 * K1C_SLOTS * K1_THREADS * 16 + (size_t)K1_THREADS * pstride;
			if (smem > 44 * 1024) { pstride = 0; smem = (size_t)2 * K1C_SLOTS * K1_THREADS * 16; }   /* the shared copy must not cost a resident block (registers allow 5 per SM): reads up to ~350 bases */
		} else
		if (smem > K1_SMEM_MAX) { qstride = 0; pstride = 0; nstride = 0; want_pack = false; smem = (size_t)2 * K1_SLOTS * K1_THREADS * 16; }   /* very long reads stay in global memory */
		int grid;
#ifdef BWAG_CUSIM
		grid = 2;
#else
		{
			/* BWA_B200_K1_BLOCKS: resident blocks per SM K1 may take.  K1 waits on DRAM, K4/K5 on shared memory and the integer
			 * pipes: leaving room lets another lane's K4/K5 run beside it (chunks travel on independent streams) */
			static int cap = -1;
			int nb;
			if (cap < 0) { const char *e = getenv("BWA_B200_K1_BLOCKS"); cap = e ? atoi(e) : 0; }
#ifndef K1_PACKED8
			if (k1c) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_smem_c, K1_THREADS, smem));
			else
#endif
			if (fm) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_smem_fm, K1_THREADS, smem));
			else
			CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_smem, K1_THREADS, smem));
			if (cap > 0 && nb > cap) nb = cap;
			grid = b->ctx->n_sm * (nb > 0 ? nb : 1);
		}
#endif
		const int cap3 = fm ? 1 : b->max_len / (par->min_seed_len + 1) + 2;   /* fastmap: no third pass (and -l may be -1) */
		size_t per_group = (size_t)((k1c ? 2 : 4) * cap_list + 2 * cap_mem) * 16;   /* k_smem_c has no per-call result array */
		{   /* keep the per-group scratch within ~6 GB: very long reads get fewer groups */
			size_t budget = (size_t)6 << 30;
			i64 max_groups = (i64)(budget / per_group);
			if (max_groups < groups_per_block) max_groups = groups_per_block;
			if ((i64)grid * groups_per_block > max_groups) grid = (int)(max_groups / groups_per_block);
			i64 need_groups = ((i64)n + groups_per_block - 1) / groups_per_block;
			if (grid > need_groups) grid = (int)(need_groups > 0 ? need_groups : 1);
		}
		if (buf_reserve(&c->s_k1, per_group * (size_t)grid * groups_per_block)) return 1;
		if (buf_reserve(&c->s_k1f, 32 * (size_t)cap3 * (size_t)n + 64) || buf_reserve(&c->s_n3, sizeof(int) * (size_t)(n + 1))) return 1;
		const size_t pack_words = (size_t)(b->total_bases >> 4) + 2 * (size_t)n + 8, nmask_words = nstride ? (size_t)(b->total_bases >> 5) + 2 * (size_t)n + 8 : 0;
		if (want_pack && buf_reserve(&c->s_pack, 4 * (pack_words + nmask_words + (size_t)n + 8))) return 1;
		if (buf_reserve(&b->d_intv_beg, sizeof(i64) * (size_t)(n + 1)) || buf_reserve(&b->d_intv_n, sizeof(int) * (size_t)(n + 1)) ||
		    buf_reserve(&b->d_intv, 32 * (size_t)cap_intv) || buf_reserve(&b->d_seed_beg, 8 * (size_t)cap_intv) || buf_reserve(&b->d_rbeg, 8 * (size_t)cap_seeds)) return 1;
		a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p; a.n_reads = n;
		a.min_seed_len = par->min_seed_len; a.split_len = par->split_len; a.split_width = par->split_width; a.max_occ = par->max_occ; a.max_mem_intv = par->max_mem_intv;
		a.scratch = (Intv *)c->s_k1.p; a.cap_list = cap_list; a.cap_mem = cap_mem; a.qstride = qstride; a.pstride = pstride; a.nstride = nstride;
		a.post_copies3 = k1c ? 1 : 0;
		a.stage3 = (Intv *)c->s_k1f.p; a.cap3 = cap3; a.n3 = par->max_mem_intv ? (int *)c->s_n3.p : 0; a.next_read3 = &c->d_cnt->next_read3;
		a.intv_beg = (i64 *)b->d_intv_beg.p; a.intv_n = (int *)b->d_intv_n.p; a.intv = (bwtintv_t *)b->d_intv.p; a.seed_beg = (i64 *)b->d_seed_beg.p; a.rbeg = (i64 *)b->d_rbeg.p;
		a.cap_intv = cap_intv; a.cap_seeds = cap_seeds;
		a.next_read = &c->d_cnt->next_read; a.n_intv = &c->d_cnt->n_intv; a.n_seeds = &c->d_cnt->n_seeds; a.occ_touches = &c->d_cnt->occ_touches; a.flags = &c->d_cnt->flags;
		if (reset_counters(c)) return 1;
#ifdef BWAG_K1_CLOCKS   /* K1f and k_smem_c timed apart, and k_smem_c's counters */
		cudaEvent_t k1e[2];
		for (int e = 0; e < 2; ++e) CK(cudaEventCreate(&k1e[e]));
		CK(cudaMalloc((void **)&a.k1clk, 8 * BWAG_K1CLK_LANE_WORDS));
		CK(cudaMemsetAsync(a.k1clk, 0, 8 * BWAG_K1CLK_LANE_WORDS, c->stream));
#endif
		CK(cudaEventRecord(c->ev0, c->stream));
		if (want_pack) {   /* the packed copies K1's table lookups key on, and which reads have an ambiguous base */
			a.packed = (const u32 *)c->s_pack.p; a.nmask = nstride ? (const u32 *)c->s_pack.p + pack_words : 0; a.hasn = (const u32 *)c->s_pack.p + pack_words + nmask_words;
			BWAG_LAUNCH(k_pack_reads, (n + 127) / 128, 128, 0, c->stream, a.codes, a.off, n, (u32 *)c->s_pack.p, nstride ? (u32 *)c->s_pack.p + pack_words : (u32 *)0, (u32 *)c->s_pack.p + pack_words + nmask_words);
			CK(cudaGetLastError());
			++c->st.n_launch;
		}
#ifdef BWAG_K1_CLOCKS
		CK(cudaEventRecord(k1e[0], c->stream));
#endif
		if (a.n3) {   /* third pass first: K1 appends its seeds to the read's list */
			int g3 = b->ctx->grid_k1f;
			if (g3 > (n + K1F_THREADS - 1) / K1F_THREADS) g3 = (n + K1F_THREADS - 1) / K1F_THREADS;
			BWAG_LAUNCH(k_smem_fwd, g3, K1F_THREADS, 0, c->stream, c->ix, a);
			CK(cudaGetLastError());
			++c->st.n_launch;
		}
#ifdef BWAG_K1_CLOCKS
		CK(cudaEventRecord(k1e[1], c->stream));
#endif
#ifndef K1_PACKED8
		if (k1c) BWAG_LAUNCH(k_smem_c, grid, K1_THREADS, smem, c->stream, c->ix, a);
		else
#endif
		if (fm) BWAG_LAUNCH(k_smem_fm, grid, K1_THREADS, smem, c->stream, c->ix, a, fm->min_intv, fm->max_intv);
		else
		BWAG_LAUNCH(k_smem, grid, K1_THREADS, smem, c->stream, c->ix, a);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		if (!fm) {
			BWAG_LAUNCH(k_seed_post, (n + K1B_THREADS - 1) / K1B_THREADS, K1B_THREADS, 0, c->stream, a);   /* harmless if K1 overflowed: the run is repeated */
			CK(cudaGetLastError());
		}
		if (fetch_counters(c)) return 1;
		c->st.ms_smem += elapsed_at(c, "smem", __FILE__, __LINE__); c->st.n_launch += 2;
#ifdef BWAG_K1_CLOCKS
		{
			u64 h[BWAG_K1CLK_LANE_WORDS];
			float ms_f = 0, ms_c = 0;
			CK(cudaMemcpy(h, a.k1clk, sizeof(h), cudaMemcpyDeviceToHost));
			CK(cudaEventElapsedTime(&ms_f, k1e[0], k1e[1])); CK(cudaEventElapsedTime(&ms_c, k1e[1], c->ev1));
			CK(cudaFree(a.k1clk));
			a.k1clk = 0;
			for (int e = 0; e < 2; ++e) cudaEventDestroy(k1e[e]);
			if (k1c) {
				pthread_mutex_lock(&g_k1clk_mu);
				for (int w = 0; w < BWAG_K1CLK_LANE_WORDS; ++w) g_k1clk[w] += h[w];
				g_k1clk[BWAG_K1CLK_K1F_NS] += (u64)(ms_f * 1e6); g_k1clk[BWAG_K1CLK_K1C_NS] += (u64)(ms_c * 1e6); g_k1clk[BWAG_K1CLK_CALLS] += 1;
				pthread_mutex_unlock(&g_k1clk_mu);
			}
		}
#endif
		if (!(c->h_cnt->flags & 41u)) break;
		if (attempt >= 6) return set_err("seeding: output pools keep overflowing (intervals %llu, seeds %llu)", (unsigned long long)c->h_cnt->n_intv, (unsigned long long)c->h_cnt->n_seeds);
		if (c->h_cnt->flags & 1u) { /* pools too small: the counters say how much is needed */
			if ((i64)c->h_cnt->n_intv > cap_intv) cap_intv = (i64)c->h_cnt->n_intv + 1024;
			if ((i64)c->h_cnt->n_seeds > cap_seeds) cap_seeds = (i64)c->h_cnt->n_seeds + 4096;
		}
		if (c->h_cnt->flags & 8u) cap_mem = cap_mem * 4 < 2 * b->max_len + 64 || !k1c ? cap_mem * 4 : 2 * b->max_len + 64;
		if (c->h_cnt->flags & 32u) cap_list = b->max_len + 1;
		if (getenv("BWA_B200_PROFILE")) fprintf(stderr, "[prof] seeding repeated (flags %u): pools %lld intervals / %lld seeds, per-lane scratch %d list entries / %d results\n", c->h_cnt->flags, (long long)cap_intv, (long long)cap_seeds, cap_list, cap_mem);
	}
	c->st.occ_touches += c->h_cnt->occ_touches;
	const i64 n_intv = (i64)c->h_cnt->n_intv, n_seeds = (i64)c->h_cnt->n_seeds;
	if (fm) { b->n_intv = n_intv; b->n_seeds = 0; b->seeded = 0; return 0; }
	/* K2: resolve the BWT rows left in rbeg[] to suffix-array positions, in place */
	if (n_seeds > 0) {
		if (run_sa(b, (i64 *)b->d_rbeg.p, n_seeds) || fetch_counters(c)) return 1;
		c->st.ms_sa += elapsed_at(c, "sa", __FILE__, __LINE__); ++c->st.n_launch;
		c->st.sa_touches += c->h_cnt->sa_touches;
	}
	b->n_intv = n_intv; b->n_seeds = n_seeds; b->seeded = 1;
	if (!out) return 0;      /* results stay in HBM for bwag_chain_extend */
	if (hbuf_reserve(&b->h_intv_beg, sizeof(i64) * (size_t)(n + 1)) || hbuf_reserve(&b->h_intv_n, sizeof(int) * (size_t)(n + 1)) ||
	    hbuf_reserve(&b->h_intv, 32 * (size_t)(n_intv + 1)) || hbuf_reserve(&b->h_seed_beg, 8 * (size_t)(n_intv + 1)) || hbuf_reserve(&b->h_rbeg, 8 * (size_t)(n_seeds + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	D2H(c, b->h_intv_beg.p, b->d_intv_beg.p, sizeof(i64) * (size_t)n);
	D2H(c, b->h_intv_n.p, b->d_intv_n.p, sizeof(int) * (size_t)n);
	if (n_intv) D2H(c, b->h_intv.p, b->d_intv.p, 32 * (size_t)n_intv);
	if (n_intv) D2H(c, b->h_seed_beg.p, b->d_seed_beg.p, 8 * (size_t)n_intv);
	if (n_seeds) D2H(c, b->h_rbeg.p, b->d_rbeg.p, 8 * (size_t)n_seeds);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	out->intv_beg = (const int64_t *)b->h_intv_beg.p; out->intv_n = (const int32_t *)b->h_intv_n.p; out->intv = (const bwtintv_t *)b->h_intv.p;
	out->seed_beg = (const int64_t *)b->h_seed_beg.p; out->rbeg = (const int64_t *)b->h_rbeg.p; out->n_intv = n_intv; out->n_seeds = n_seeds;
	return 0;
}

extern "C" int bwag_seed(bwag_batch_t *b, const bwag_seed_par_t *par, bwag_seeds_t *out) { return seed_impl(b, par, 0, out); }

/* ------------------------------------------------------------------------------------------------ stage 2 */

/* K4 with its per-warp scratch in shared memory when that fits, else in global memory; n_units = reads to process */
static int k4_lane_maxchains(void) { const char *e = getenv("BWA_B200_K4_LANE_MAXCHAINS"); return e ? atoi(e) : 8; }

/* n_many: reads with more chains than the lane kernel takes, if the caller knows (K3 counts them), else -1 */
static int launch_extend(bwag_batch_t *b, ExtArgs &a, int n_units, int n_many = -1)
{
	Lane *c = &b->lane;
	const int wpb = K4_THREADS / 32;
	a.chain_lo = 0; a.chain_hi = 0x7fffffff;
	int per_warp = (8 * (a.cap_q + 2) + a.cap_r + a.cap_q + 15) & ~15;
	size_t smem = (size_t)per_warp * wpb;
	int grid = b->ctx->grid_k4, use_sm = smem <= K4_SMEM_MAX && !(getenv("BWA_B200_K4_SM") && atoi(getenv("BWA_B200_K4_SM")) == 0);
	/* the leaner row sweep (and its row cut-off) needs non-negative gap penalties (every real scoring scheme); BWA_B200_K4_FAST=0 forces the general one */
	const int fast = a.par.e_ins >= 0 && a.par.o_ins + a.par.e_ins >= 0 && a.par.e_del >= 0 && a.par.o_del + a.par.e_del >= 0 &&
	                 !c->baseline && !(getenv("BWA_B200_K4_FAST") && atoi(getenv("BWA_B200_K4_FAST")) == 0);
	{   /* short reads: one lane per read (bwag_extend_lane.cu) when every score fits its 13-bit cells and a block's columns fit shared memory */
		int maxsc = 0;
		for (int k = 0; k < 25; ++k) maxsc = maxsc > a.par.mat[k] ? maxsc : a.par.mat[k];
		const int lcols = a.cap_q - (a.min_seed > 0 && a.min_seed < a.cap_q ? a.min_seed - 3 : 0) + 2 + 8;   /* longest extension (read minus its shortest possible seed; cap_q rounds the read length up by <= 3) + column `end` + the chunk's spare columns (K4L_CH) */
		const size_t lsm = (size_t)lcols * K4L_THREADS * 4;
		const int lane_ok = fast && (i64)a.cap_q * maxsc < 8192 && a.par.a <= maxsc && lsm <= K4L_SMEM_MAX && !(getenv("BWA_B200_K4_LANE") && atoi(getenv("BWA_B200_K4_LANE")) == 0);
		if (lane_ok) {
			int lgrid = b->ctx->n_sm;
#ifndef BWAG_CUSIM
			{ int nb = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_extend_lane, K4L_THREADS, lsm)); lgrid = b->ctx->n_sm * (nb > 0 ? nb : 1); }
#else
			lgrid = 2;
#endif
			const i64 lneed = ((i64)n_units + K4L_THREADS - 1) / K4L_THREADS;
			if (lgrid > lneed) lgrid = (int)(lneed > 0 ? lneed : 1);
			/* a lane works through its read's chains one after the other, which is right for the usual one or two chains and hopeless for a
			 * read from a repeat family with hundreds (measured on the repeat-rich workload): those go to the warp-per-read kernel below */
			const int many = k4_lane_maxchains();
			ExtArgs la = a;
			la.eh = 0; la.rseq = 0; la.smem_per_warp = lcols;   /* here: the number of columns of a lane's row */
			la.chain_lo = 0; la.chain_hi = many;
			if (getenv("BWA_B200_PROFILE")) fprintf(stderr, "[prof] extension: lane-per-read kernel for reads with chains %d..%d, grid %d x %d, %zu bytes of shared memory per block\n", la.chain_lo, la.chain_hi, lgrid, K4L_THREADS, lsm);
			BWAG_LAUNCH(k_extend_lane, lgrid, K4L_THREADS, lsm, c->stream, c->ix, la);
			CK(cudaGetLastError());
			++c->st.n_launch;
			if (n_many == 0) return 0;                 /* no read is left for the warp-per-read kernel */
			CK(cudaMemsetAsync(a.next_read, 0, sizeof(int), c->stream));
			a.chain_lo = many + 1; a.chain_hi = 0x7fffffff;
		}
	}
#ifndef BWAG_CUSIM
	if (use_sm) { int nb = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fast ? k_extend_sm_fast : k_extend_sm, K4_THREADS, smem)); if (nb < 2) use_sm = 0; else grid = b->ctx->n_sm * nb; }
#endif
	i64 need = ((i64)n_units + wpb - 1) / wpb;
	if (grid > need) grid = (int)(need > 0 ? need : 1);
	if (getenv("BWA_B200_PROFILE"))
		fprintf(stderr, "[prof] extension: warp-per-read kernel %s (scratch in %s memory, %s row sweep) for reads with chains %d..%d, grid %d x %d\n",
		        use_sm ? (fast ? "k_extend_sm_fast" : "k_extend_sm") : (fast ? "k_extend_fast" : "k_extend"), use_sm ? "shared" : "global",
		        fast ? "lean" : "first", a.chain_lo, a.chain_hi, grid, K4_THREADS);
	if (!use_sm) {
		const size_t n_warps = (size_t)grid * wpb;
		if (buf_reserve(&c->s_eh, n_warps * 2 * (size_t)(a.cap_q + 2) * 4) || buf_reserve(&c->s_rseq, n_warps * (size_t)a.cap_r)) return 1;
		a.eh = (int *)c->s_eh.p; a.rseq = (uint8_t *)c->s_rseq.p; a.smem_per_warp = 0;
		if (fast) BWAG_LAUNCH(k_extend_fast, grid, K4_THREADS, 0, c->stream, c->ix, a);
		else BWAG_LAUNCH(k_extend, grid, K4_THREADS, 0, c->stream, c->ix, a);
	} else {
		a.eh = 0; a.rseq = 0; a.smem_per_warp = per_warp;
		if (fast) BWAG_LAUNCH(k_extend_sm_fast, grid, K4_THREADS, smem, c->stream, c->ix, a);
		else BWAG_LAUNCH(k_extend_sm, grid, K4_THREADS, smem, c->stream, c->ix, a);
	}
	CK(cudaGetLastError());
	return 0;
}


extern "C" int bwag_extend(bwag_batch_t *b, const bwag_sw_par_t *par, const int32_t *chain_off, const bwag_xchain_t *chains,
                           int64_t n_seeds, const bwag_xseed_t *seeds, bwag_regs_t *out)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	const int n = b->n;
	const i64 n_chains = chain_off[n];
	int cap_r = 16;
	for (i64 i = 0; i < n_chains; ++i) { i64 l = chains[i].rmax1 - chains[i].rmax0; if (l > cap_r) cap_r = (int)l; }
	cap_r = (cap_r + 15) & ~15;
	const int cap_q = (b->max_len + 3) & ~3;
	if (buf_reserve(&b->d_chain_off, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_chains, sizeof(bwag_xchain_t) * (size_t)(n_chains + 1)) ||
	    buf_reserve(&b->d_seeds, sizeof(bwag_xseed_t) * (size_t)(n_seeds + 1)) || buf_reserve(&b->d_regs, sizeof(bwag_xreg_t) * (size_t)(n_seeds + 1)) ||
	    buf_reserve(&b->d_nregs, 4 * (size_t)(n + 1))) return 1;
	if (buf_reserve(&b->d_chain_beg, 8 * (size_t)(n + 1)) || buf_reserve(&b->d_chain_cnt, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_reg_base, 8 * (size_t)(n + 1)) ||
	    hbuf_reserve(&b->h_tmp, 20 * (size_t)(n + 1))) return 1;
	i64 *h_cbeg = (i64 *)b->h_tmp.p, *h_rbase = h_cbeg + n + 1;
	int *h_ccnt = (int *)(h_rbase + n + 1);
	for (int r = 0; r < n; ++r) {   /* per read: its chains, and where its regions go (the slot range of its seeds) */
		h_cbeg[r] = chain_off[r]; h_ccnt[r] = chain_off[r + 1] - chain_off[r];
		h_rbase[r] = h_ccnt[r] ? chains[chain_off[r]].seed_off : 0;
	}
	if (reset_counters(c)) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	H2D(c, b->d_chain_beg.p, h_cbeg, 8 * (size_t)n);
	H2D(c, b->d_reg_base.p, h_rbase, 8 * (size_t)n);
	H2D(c, b->d_chain_cnt.p, h_ccnt, 4 * (size_t)n);
	if (n_chains) H2D(c, b->d_chains.p, chains, sizeof(bwag_xchain_t) * (size_t)n_chains);
	if (n_seeds) H2D(c, b->d_seeds.p, seeds, sizeof(bwag_xseed_t) * (size_t)n_seeds);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_h2d += elapsed_at(c, "h2d", __FILE__, __LINE__);
	ExtArgs a;
	memset(&a, 0, sizeof(a));
	a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p; a.n_reads = n; a.par = *par;
	a.chain_beg = (const i64 *)b->d_chain_beg.p; a.chain_cnt = (const int *)b->d_chain_cnt.p; a.reg_base = (const i64 *)b->d_reg_base.p;
	a.chains = (const bwag_xchain_t *)b->d_chains.p; a.seeds = (const bwag_xseed_t *)b->d_seeds.p;
	a.regs = (bwag_xreg_t *)b->d_regs.p; a.n_regs = (int32_t *)b->d_nregs.p;
	a.cap_q = cap_q; a.cap_r = cap_r;
	a.next_read = &c->d_cnt->next_read; a.cells = &c->d_cnt->ext_cells; a.flags = &c->d_cnt->flags;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (launch_extend(b, a, n)) return 1;
	CK(cudaEventRecord(c->ev1, c->stream));
	if (fetch_counters(c)) return 1;
	c->st.ms_extend += elapsed_at(c, "extend", __FILE__, __LINE__); ++c->st.n_launch;
	if (c->h_cnt->flags & 2u) return set_err("extension: a read or reference window exceeded the scratch capacity");
	c->st.ext_cells += c->h_cnt->ext_cells;
	if (hbuf_reserve(&b->h_regs, sizeof(bwag_xreg_t) * (size_t)(n_seeds + 1)) || hbuf_reserve(&b->h_nregs, 4 * (size_t)(n + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_seeds) D2H(c, b->h_regs.p, b->d_regs.p, sizeof(bwag_xreg_t) * (size_t)n_seeds);
	D2H(c, b->h_nregs.p, b->d_nregs.p, 4 * (size_t)n);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	out->n_regs = (const int32_t *)b->h_nregs.p; out->regs = (const bwag_xreg_t *)b->h_regs.p;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ stages 2a+2 fused */

/* K6 over n_tasks tasks that are in b->d_swtasks already (queries/targets: the batch's reads, the reference, or b->d_swpool);
 * results to b->d_swres.  max_q / max_t: no task is longer.  Records ev0/ev1 around the kernel; the caller fetches the counters. */
int localsw_on_device(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, int max_q, int max_t)
{
	Lane *c = &b->lane;
	const int cap_q = ((max_q > 16 ? max_q : 16) + 15) & ~15, cap_t = ((max_t > 16 ? max_t : 16) + 15) & ~15;
	const int cap_n = cap_q + 16;                                       /* query length rounded up to a whole number of vectors */
	/* warp per task (vectors in shared memory) when a block's share fits, else lane per task (everything in a global scratch slice) */
	const size_t w_smem = (size_t)(8 * cap_n + cap_q) * 4;
	const int warp_ok = w_smem <= K4_SMEM_MAX && !(getenv("BWA_B200_K6_WARP") && atoi(getenv("BWA_B200_K6_WARP")) == 0);
	const i64 per_thread = warp_ok ? (((i64)cap_t * 8 + cap_t + 63) & ~(i64)63) : (((i64)cap_n * 8 + (i64)cap_t * 8 + cap_q + cap_t + 63) & ~(i64)63);   /* per warp / per lane */
	int grid = b->ctx->n_sm * 16;
	if (warp_ok) {
#ifndef BWAG_CUSIM
		int nb = 0;
		CK(cudaFuncSetAttribute(k_localsw_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_localsw_warp, 128, w_smem));
		grid = b->ctx->n_sm * (nb > 0 ? nb : 1);
#else
		grid = 2;
#endif
		const i64 need = ((i64)n_tasks + 3) / 4;
		if (grid > need) grid = (int)need;
	} else {
		const i64 need = ((i64)n_tasks + 63) / 64;
		if (grid > need) grid = (int)need;
		const i64 max_threads = ((i64)4 << 30) / per_thread;            /* bound the scratch to ~4 GB */
		if ((i64)grid * 64 > max_threads) grid = (int)(max_threads / 64 > 0 ? max_threads / 64 : 1);
	}
	if (buf_reserve(&b->d_swres, sizeof(bwag_swres_t) * (size_t)n_tasks) || buf_reserve(&b->d_swscratch, (size_t)per_thread * (size_t)grid * (warp_ok ? 4 : 64)) ||
	    buf_reserve(&b->d_swpool, 16)) return 1;
	SwArgs a;
	memset(&a, 0, sizeof(a));
	a.tasks = (const bwag_swtask_t *)b->d_swtasks.p; a.n_tasks = n_tasks; a.par = *par;
	a.codes = (const uint8_t *)b->d_codes.p; a.pool = (const uint8_t *)b->d_swpool.p; a.res = (bwag_swres_t *)b->d_swres.p;
	a.scratch = (unsigned char *)b->d_swscratch.p; a.per_thread = per_thread; a.cap_n = cap_n; a.cap_q = cap_q; a.cap_t = cap_t;
	a.next_task = &c->d_cnt->next_task; a.flags = &c->d_cnt->flags;
	CK(cudaMemsetAsync(&c->d_cnt->next_task, 0, sizeof(int), c->stream));
	CK(cudaEventRecord(c->ev0, c->stream));
	if (warp_ok) BWAG_LAUNCH(k_localsw_warp, grid, 128, w_smem, c->stream, c->ix, a);
	else BWAG_LAUNCH(k_localsw, grid, 64, 0, c->stream, c->ix, a);
	CK(cudaGetLastError());
	CK(cudaEventRecord(c->ev1, c->stream));
	return 0;
}

extern "C" int bwag_localsw(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, const bwag_swtask_t *tasks, const uint8_t *pool, size_t pool_bytes, const bwag_swres_t **out)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	*out = 0;
	if (n_tasks <= 0) return 0;
	int max_q = 16, max_t = 16;
	for (int t = 0; t < n_tasks; ++t) { if (tasks[t].qlen > max_q) max_q = tasks[t].qlen; if (tasks[t].tlen > max_t) max_t = tasks[t].tlen; }
	if (buf_reserve(&b->d_swtasks, sizeof(bwag_swtask_t) * (size_t)n_tasks) || buf_reserve(&b->d_swpool, pool_bytes + 16) ||
	    hbuf_reserve(&b->h_swres, sizeof(bwag_swres_t) * (size_t)n_tasks)) return 1;
	if (reset_counters(c)) return 1;
	H2D(c, b->d_swtasks.p, tasks, sizeof(bwag_swtask_t) * (size_t)n_tasks);
	if (pool && pool_bytes) H2D(c, b->d_swpool.p, pool, pool_bytes);
	if (localsw_on_device(b, par, n_tasks, max_q, max_t)) return 1;
	D2H(c, b->h_swres.p, b->d_swres.p, sizeof(bwag_swres_t) * (size_t)n_tasks);
	if (fetch_counters(c)) return 1;
	c->st.ms_localsw += elapsed_at(c, "localsw", __FILE__, __LINE__); ++c->st.n_launch; c->st.sw_tasks += (u64)n_tasks;
	if (c->h_cnt->flags & 32u) return set_err("local alignment: a task exceeded the scratch capacity");
	*out = (const bwag_swres_t *)b->h_swres.p;
	return 0;
}
extern "C" int bwag_chain_extend(bwag_batch_t *b, const bwag_chain_par_t *cp, const bwag_sw_par_t *par, const bwag_contigs_t *ctg, bwag_cregs_t *out)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	if (!b->seeded) return set_err("bwag_chain_extend needs a preceding bwag_seed on the same batch");
	const int n = b->n;
	const i64 ns = b->n_seeds;
	if (ns >= ((i64)1 << 31)) return set_err("too many seeds in one batch for the 32-bit seed offsets; use smaller chunks");
	/* contig table: offsets (i64), lengths (int), ALT flags (byte) in one device buffer */
	const size_t ctg_bytes = (size_t)ctg->n_seqs * 13 + 64;
	if (buf_reserve(&b->d_ctg, ctg_bytes) || hbuf_reserve(&b->h_tmp, ctg_bytes)) return 1;
	{
		char *h = (char *)b->h_tmp.p;
		memcpy(h, ctg->offset, 8 * (size_t)ctg->n_seqs);
		memcpy(h + 8 * (size_t)ctg->n_seqs, ctg->len, 4 * (size_t)ctg->n_seqs);
		memcpy(h + 12 * (size_t)ctg->n_seqs, ctg->is_alt, (size_t)ctg->n_seqs);
	}
	if (buf_reserve(&b->s_bt, 88 * (size_t)(ns + 1)) || buf_reserve(&b->s_sn, 32 * (size_t)(ns + 1)) || buf_reserve(&b->s_ch, 48 * (size_t)(ns + 1)) ||
	    buf_reserve(&b->s_order, 4 * (size_t)(ns + 1)) || buf_reserve(&b->s_idx, 4 * (size_t)(ns + 1)) || buf_reserve(&b->s_keys, 8 * (size_t)(ns + 1)) ||
	    buf_reserve(&b->d_chains, sizeof(bwag_xchain_t) * (size_t)(ns + 1)) || buf_reserve(&b->d_seeds, sizeof(bwag_xseed_t) * (size_t)(ns + 1)) ||
	    buf_reserve(&b->d_regs, sizeof(bwag_xreg_t) * (size_t)(ns + 1)) || buf_reserve(&b->d_chain_rid, 4 * (size_t)(ns + 1)) || buf_reserve(&b->d_chain_frac, 4 * (size_t)(ns + 1)) ||
	    buf_reserve(&b->d_chain_beg, 8 * (size_t)(n + 1)) || buf_reserve(&b->d_chain_cnt, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_reg_base, 8 * (size_t)(n + 1)) ||
	    buf_reserve(&b->d_nregs, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_creg_beg, 8 * (size_t)(n + 1)) || buf_reserve(&b->d_k3big, 4 * (size_t)(n + 1))) return 1;
	if (reset_counters(c)) return 1;
	H2D(c, b->d_ctg.p, b->h_tmp.p, 13 * (size_t)ctg->n_seqs);
	ChainArgs k;
	memset(&k, 0, sizeof(k));
	k.off = (const i64 *)b->d_off.p; k.n_reads = n;
	k.intv_beg = (const i64 *)b->d_intv_beg.p; k.intv_n = (const int *)b->d_intv_n.p; k.intv = (const bwtintv_t *)b->d_intv.p;
	k.seed_beg = (const i64 *)b->d_seed_beg.p; k.rbeg = (const i64 *)b->d_rbeg.p;
	k.w = cp->w; k.max_chain_gap = cp->max_chain_gap; k.max_occ = cp->max_occ; k.min_seed_len = cp->min_seed_len; k.min_chain_weight = cp->min_chain_weight;
	k.max_chain_extend = cp->max_chain_extend; k.mask_level = cp->mask_level; k.drop_ratio = cp->drop_ratio;
	k.a = par->a; k.o_del = par->o_del; k.e_del = par->e_del; k.o_ins = par->o_ins; k.e_ins = par->e_ins;
	k.l_pac = c->ix.l_pac; k.n_seqs = ctg->n_seqs;
	k.ctg_off = (const i64 *)b->d_ctg.p; k.ctg_len = (const int *)((char *)b->d_ctg.p + 8 * (size_t)ctg->n_seqs); k.ctg_alt = (const uint8_t *)b->d_ctg.p + 12 * (size_t)ctg->n_seqs;
	k.s_bt = b->s_bt.p; k.s_sn = b->s_sn.p; k.s_ch = b->s_ch.p; k.s_order = (int *)b->s_order.p; k.s_idx = (int *)b->s_idx.p; k.s_keys = (u64 *)b->s_keys.p;
	k.xchains = (bwag_xchain_t *)b->d_chains.p; k.xseeds = (bwag_xseed_t *)b->d_seeds.p; k.chain_rid = (int *)b->d_chain_rid.p; k.chain_frac = (float *)b->d_chain_frac.p;
	k.chain_beg = (i64 *)b->d_chain_beg.p; k.reg_base = (i64 *)b->d_reg_base.p; k.n_chains = (int *)b->d_chain_cnt.p;
	k.max_rlen = &c->d_cnt->max_rlen; k.n_many = &c->d_cnt->n_many; k.many = k4_lane_maxchains();
	{   /* seed-level filter of long reads (mem_flt_chained_seeds, bwamem.c:626-641): threshold by read length, from the host's libm
	     * (the value is truncated to an int: bwamem.c:628); no table if no read of the chunk can be long enough */
		const int L = b->max_len;
		int any = 0;
		if (hbuf_reserve(&b->h_hsp, sizeof(int) * (size_t)(L + 2))) return 1;
		int *tab = (int *)b->h_hsp.p;
		for (int l = 0; l <= L; ++l) {
			const double min_l = cp->min_chain_weight ? 1.1f * cp->min_chain_weight : 5.5f * log((double)l);
			tab[l] = min_l > 0.05f * l ? -1 : (int)(par->a * min_l + .499);
			if (tab[l] >= 0 && l >= cp->min_seed_len) any = 1;
		}
		if (any && !(getenv("BWA_B200_DEVICE_SEEDSW") && atoi(getenv("BWA_B200_DEVICE_SEEDSW")) == 0)) {
			if (buf_reserve(&b->d_hsp, sizeof(int) * (size_t)(L + 2)) || buf_reserve(&b->d_flt_nchn, sizeof(int) * (size_t)(n + 1)) ||
			    buf_reserve(&b->d_swtasks, sizeof(bwag_swtask_t) * (size_t)(ns + 1))) return 1;
			H2D(c, b->d_hsp.p, tab, sizeof(int) * (size_t)(L + 1));
			k.hsp_tab = (const int *)b->d_hsp.p; k.flt_nchn = (int *)b->d_flt_nchn.p;
			k.sw_tasks = (bwag_swtask_t *)b->d_swtasks.p; k.n_swtasks = &c->d_cnt->n_swtasks;
		} else if (any) return BWAG_DECLINED;   /* switched off: the caller chains these reads on the host */
	}
#ifdef BWAG_K3_CLOCKS
	CK(cudaMalloc((void **)&k.k3clk, 20 * (size_t)(n + 1)));
#endif
	/* Without the long-read filter, k_chain_sm chains the reads with few seeds in shared memory and lists the others, which
	 * k_chain then takes with their workspace in HBM (grid-stride over the list, whose length only the device knows).  With the
	 * filter every read takes k_chain: K3b reads the HBM workspace back. */
	const int on_chip = !k.hsp_tab;
	int k3_grid = (n + K3_THREADS - 1) / K3_THREADS;
	if (on_chip) {
		k.big = (int *)b->d_k3big.p; k.n_big = &c->d_cnt->n_big;
		if (k3_grid > b->ctx->n_sm * 16) k3_grid = b->ctx->n_sm * 16;
	}
	CK(cudaEventRecord(c->ev0, c->stream));
	if (on_chip) {
		BWAG_LAUNCH(k_chain_sm, (n + K3S_THREADS - 1) / K3S_THREADS, K3S_THREADS, K3S_SMEM, c->stream, k);
		CK(cudaGetLastError());
	}
	BWAG_LAUNCH(k_chain, k3_grid > 0 ? k3_grid : 1, K3_THREADS, 0, c->stream, k);
	CK(cudaGetLastError());
	CK(cudaEventRecord(c->ev1, c->stream));
	if (fetch_counters(c)) return 1;
	c->st.ms_chain += elapsed_at(c, "chain", __FILE__, __LINE__); c->st.n_launch += 1 + on_chip;
	if (getenv("BWA_B200_PROFILE"))
		fprintf(stderr, "[prof] chain: %d reads on chip, %d in HBM, CAP %d seeds, %d blocks of %d threads per SM on chip\n",
		        on_chip ? n - c->h_cnt->n_big : 0, on_chip ? c->h_cnt->n_big : n, K3S_CAP, b->ctx->k3s_blocks, K3S_THREADS);
#ifdef BWAG_K3_CLOCKS
	{
		u32 *h = (u32 *)malloc(20 * (size_t)(n + 1));
		CK(cudaMemcpy(h, k.k3clk, 20 * (size_t)n, cudaMemcpyDeviceToHost));
		CK(cudaFree(k.k3clk));
		k.k3clk = 0;
		k3clk_add(h, n);
		free(h);
	}
#endif
	if (k.hsp_tab) {
		const int n_sw = (int)c->h_cnt->n_swtasks;
		if (n_sw > 0) {
			if (localsw_on_device(b, par, n_sw, SEEDSW_MAXLEN, SEEDSW_MAXLEN)) return 1;
			if (fetch_counters(c)) return 1;
			c->st.ms_localsw += elapsed_at(c, "localsw", __FILE__, __LINE__); ++c->st.n_launch; c->st.sw_tasks += (u64)n_sw;
			if (c->h_cnt->flags & 32u) return set_err("seed filter: a local alignment exceeded the scratch capacity");
		}
		k.sw_res = (const bwag_swres_t *)b->d_swres.p;
		CK(cudaEventRecord(c->ev0, c->stream));
		BWAG_LAUNCH(k_chain_emit, (n + K3_THREADS - 1) / K3_THREADS, K3_THREADS, 0, c->stream, k);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		if (fetch_counters(c)) return 1;
		c->st.ms_chain += elapsed_at(c, "chain", __FILE__, __LINE__); ++c->st.n_launch;
	}

	/* extension over the chains that K3 left in HBM; K3 reported the longest reference window */
	const int cap_q = (b->max_len + 3) & ~3;
	const int cap_r = (c->h_cnt->max_rlen + 16 + 15) & ~15;
	CK(cudaMemsetAsync(&c->d_cnt->next_read, 0, sizeof(int), c->stream));
	ExtArgs a;
	memset(&a, 0, sizeof(a));
	a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p; a.n_reads = n; a.par = *par;
	a.chain_beg = (const i64 *)b->d_chain_beg.p; a.chain_cnt = (const int *)b->d_chain_cnt.p; a.reg_base = (const i64 *)b->d_reg_base.p;
	a.chains = (const bwag_xchain_t *)b->d_chains.p; a.seeds = (const bwag_xseed_t *)b->d_seeds.p;
	a.regs = (bwag_xreg_t *)b->d_regs.p; a.n_regs = (int32_t *)b->d_nregs.p;
	a.cap_q = cap_q; a.cap_r = cap_r; a.min_seed = cp->min_seed_len;
	a.next_read = &c->d_cnt->next_read; a.cells = &c->d_cnt->ext_cells; a.flags = &c->d_cnt->flags;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (launch_extend(b, a, n, c->h_cnt->n_many)) return 1;
	CK(cudaEventRecord(c->ev1, c->stream));
	if (!out) {   /* the regions stay in HBM for bwag_tail_regs */
		if (fetch_counters(c)) return 1;
		c->st.ms_extend += elapsed_at(c, "extend", __FILE__, __LINE__); ++c->st.n_launch;
		if (c->h_cnt->flags & 2u) return set_err("extension: a read or reference window exceeded the scratch capacity");
		c->st.ext_cells += c->h_cnt->ext_cells;
		b->regs_on_device = 1;
		return 0;
	}
	/* dense copy of the regions (with contig id and repeat fraction of their chain) for the download */
	RegCompactArgs rc;
	rc.n_reads = n; rc.n_regs = (const int *)b->d_nregs.p; rc.regs = (const bwag_xreg_t *)b->d_regs.p; rc.reg_base = (const i64 *)b->d_reg_base.p;
	rc.chain_beg = (const i64 *)b->d_chain_beg.p; rc.chain_rid = (const int *)b->d_chain_rid.p; rc.chain_frac = (const float *)b->d_chain_frac.p;
	rc.out_beg = (i64 *)b->d_creg_beg.p; rc.total = &c->d_cnt->n_cig;
	/* the number of regions is not known before K4 ran: size the dense array by the number of seeds (upper bound) */
	if (buf_reserve(&b->d_cregs, sizeof(bwag_creg_t) * (size_t)(ns + 1))) return 1;
	rc.out = (bwag_creg_t *)b->d_cregs.p;
	BWAG_LAUNCH(k_regs_compact, (n + 127) / 128, 128, 0, c->stream, rc);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	c->st.ms_extend += elapsed_at(c, "extend", __FILE__, __LINE__); c->st.n_launch += 2;
	if (c->h_cnt->flags & 2u) return set_err("extension: a read or reference window exceeded the scratch capacity");
	c->st.ext_cells += c->h_cnt->ext_cells;
	const i64 n_regs = (i64)c->h_cnt->n_cig;
	if (hbuf_reserve(&b->h_cregs, sizeof(bwag_creg_t) * (size_t)(n_regs + 1)) || hbuf_reserve(&b->h_creg_beg, 8 * (size_t)(n + 1)) || hbuf_reserve(&b->h_nregs, 4 * (size_t)(n + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_regs) D2H(c, b->h_cregs.p, b->d_cregs.p, sizeof(bwag_creg_t) * (size_t)n_regs);
	D2H(c, b->h_creg_beg.p, b->d_creg_beg.p, 8 * (size_t)n);
	D2H(c, b->h_nregs.p, b->d_nregs.p, 4 * (size_t)n);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	out->n_regs = (const int32_t *)b->h_nregs.p; out->reg_beg = (const int64_t *)b->h_creg_beg.p; out->regs = (const bwag_creg_t *)b->h_cregs.p;
	return 0;
}

extern "C" int bwag_fetch_cregs(bwag_batch_t *b, int n_sel, const int32_t *sel, bwag_cregs_t *out)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	if (!b->regs_on_device) return set_err("bwag_fetch_cregs needs a preceding bwag_chain_extend(..., NULL) on the same batch");
	out->n_regs = 0; out->reg_beg = 0; out->regs = 0;
	if (n_sel <= 0) return 0;
	const i64 ns = b->n_seeds;
	if (buf_reserve(&b->d_cregs, sizeof(bwag_creg_t) * (size_t)(ns + 1)) || buf_reserve(&b->d_creg_beg, 8 * (size_t)(b->n + 1)) || buf_reserve(&b->d_sel, 8 * (size_t)(n_sel + 1))) return 1;
	if (reset_counters(c)) return 1;
	H2D(c, b->d_sel.p, sel, 4 * (size_t)n_sel);
	RegCompactArgs rc;
	rc.n_reads = b->n; rc.n_regs = (const int *)b->d_nregs.p; rc.regs = (const bwag_xreg_t *)b->d_regs.p; rc.reg_base = (const i64 *)b->d_reg_base.p;
	rc.chain_beg = (const i64 *)b->d_chain_beg.p; rc.chain_rid = (const int *)b->d_chain_rid.p; rc.chain_frac = (const float *)b->d_chain_frac.p;
	rc.out_beg = (i64 *)b->d_creg_beg.p; rc.total = &c->d_cnt->n_cig; rc.out = (bwag_creg_t *)b->d_cregs.p;
	int *d_out_n = (int *)b->d_sel.p + n_sel;
	BWAG_LAUNCH(k_regs_compact_sel, (n_sel + 127) / 128, 128, 0, c->stream, rc, (const int *)b->d_sel.p, n_sel, d_out_n);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	++c->st.n_launch;
	const i64 n_regs = (i64)c->h_cnt->n_cig;
	if (hbuf_reserve(&b->h_cregs, sizeof(bwag_creg_t) * (size_t)(n_regs + 1)) || hbuf_reserve(&b->h_creg_beg, 8 * (size_t)(n_sel + 1)) || hbuf_reserve(&b->h_nregs, 4 * (size_t)(n_sel + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_regs) D2H(c, b->h_cregs.p, b->d_cregs.p, sizeof(bwag_creg_t) * (size_t)n_regs);
	D2H(c, b->h_creg_beg.p, b->d_creg_beg.p, 8 * (size_t)n_sel);
	D2H(c, b->h_nregs.p, d_out_n, 4 * (size_t)n_sel);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	out->n_regs = (const int32_t *)b->h_nregs.p; out->reg_beg = (const int64_t *)b->h_creg_beg.p; out->regs = (const bwag_creg_t *)b->h_cregs.p;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ stage 3 */

/* K5 over n_tasks requests that already sit in b->d_tasks; results stay in b->d_res / d_cig / d_md, their pool sizes in *nc, *nm */
int run_global(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, int cap_q, int cap_r, i64 cap_z, i64 n_aln, i64 *nc_out, i64 *nm_out)
{
	Lane *c = &b->lane;
	cap_q = (cap_q + 3) & ~3; cap_r = (cap_r + 15) & ~15; cap_z = (cap_z + 15) & ~(i64)15;
	if (cap_q < 4) cap_q = 4;
	if (cap_r < 16) cap_r = 16;
	if (cap_z < 64) cap_z = 64;
	/* one task's CIGAR has at most lq+rlen ops, its MD at most 3 characters per reference base */
	const int cap_wcig = cap_q + cap_r + 4, cap_wmd = 3 * cap_r + cap_q + 16;
	int grid = b->ctx->grid_k5;
	/* H/E rows and the sequences in shared memory when a block's share fits (BWA_B200_K5_SM=0 keeps them in global memory) */
	const int k5_zsm = getenv("BWA_B200_K5_ZSM") ? atoi(getenv("BWA_B200_K5_ZSM")) & ~15 : 6144;   /* backtrack bytes per warp in shared memory */
	const int k5_per_warp = ((8 * (cap_q + 2) + cap_r + cap_q + 2 + 15) & ~15) + k5_zsm;
	const size_t k5_smem = (size_t)k5_per_warp * (K5_THREADS / 32);
	int k5_sm = k5_smem <= K4_SMEM_MAX && !(getenv("BWA_B200_K5_SM") && atoi(getenv("BWA_B200_K5_SM")) == 0);
	const int k5_fast = !c->baseline && !(getenv("BWA_B200_K5_FAST") && atoi(getenv("BWA_B200_K5_FAST")) == 0);   /* 0: the first formulation of the row sweep */
#ifndef BWAG_CUSIM
	if (k5_sm) { int nb = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k5_fast ? k_global_sm_fast : k_global_sm, K5_THREADS, k5_smem)); if (nb < 2) k5_sm = 0; else grid = b->ctx->n_sm * nb; }
#endif
	{
		i64 need = ((i64)n_tasks + (K5_THREADS / 32) - 1) / (K5_THREADS / 32);
		if (grid > need) grid = (int)(need > 0 ? need : 1);
		i64 max_warps = ((i64)8 << 30) / cap_z;    /* bound the per-warp backtrack scratch to ~8 GB */
		if (max_warps < K5_THREADS / 32) max_warps = K5_THREADS / 32;
		if ((i64)grid * (K5_THREADS / 32) > max_warps) grid = (int)(max_warps / (K5_THREADS / 32));
	}
	const size_t n_warps = (size_t)grid * (K5_THREADS / 32);
	if (buf_reserve(&c->s_eh, n_warps * 2 * (size_t)(cap_q + 2) * 4) || buf_reserve(&c->s_rseq, n_warps * (size_t)cap_r) ||
	    buf_reserve(&c->s_qseq, n_warps * (size_t)(cap_q + 2)) || buf_reserve(&c->s_z, n_warps * (size_t)cap_z) ||
	    buf_reserve(&c->s_wcig, n_warps * (size_t)cap_wcig * 4) || buf_reserve(&c->s_wmd, n_warps * (size_t)cap_wmd)) return 1;
	if (buf_reserve(&b->d_res, sizeof(bwag_gres_t) * (size_t)n_tasks)) return 1;
	/* K5L for batches of short reads (the requests it cannot take fall through to the warp kernel one by one).  Off by default: in
	 * its first form it takes 32 consecutive requests per warp, of which only the quarter that needs a DP is live, and it was slower
	 * than the warp kernel; it needs the requests compacted and bucketed by
	 * band first.  BWA_B200_K5_LANE=1 switches it on (exact: tests/test_tail.py runs both). */
	int k5_lane = !c->baseline && cap_q <= K5L_QWORDS * 4 && n_tasks >= 64 && getenv("BWA_B200_K5_LANE") && atoi(getenv("BWA_B200_K5_LANE")) != 0;
	const size_t k5l_smem = (size_t)K5L_RING * K5L_THREADS * 8 + (size_t)K5L_QWORDS * K5L_THREADS * 4;
	const i64 k5l_cap_z = (i64)(K5L_RING - 1) * (cap_r < 1024 ? cap_r : 1024);   /* cells per lane: the widest band it takes x the longest window */
	int k5l_grid = 0;
	if (k5_lane) {
#ifndef BWAG_CUSIM
		int nb = 0;
		CK(cudaFuncSetAttribute(k_global_lane, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k5l_smem));
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_global_lane, K5L_THREADS, k5l_smem));
		k5l_grid = b->ctx->n_sm * (nb > 0 ? nb : 1);
#else
		k5l_grid = 2;
#endif
		const i64 need = ((i64)n_tasks + K5L_THREADS - 1) / K5L_THREADS;
		if (k5l_grid > need) k5l_grid = (int)need;
		if (buf_reserve(&b->d_pre_n, 4 * (size_t)n_tasks) || buf_reserve(&b->d_pre_score, 4 * (size_t)n_tasks) || buf_reserve(&b->d_pre_cig, 4 * (size_t)K5L_MAXCIG * (size_t)n_tasks) ||
		    buf_reserve(&c->s_zl, (size_t)k5l_cap_z * (size_t)k5l_grid * K5L_THREADS)) return 1;
	}
	i64 cap_cig = n_aln * 6 + 1024, cap_md = n_aln * 24 + 4096;   /* typical short-read sizes; grown on demand */
	for (int attempt = 0;; ++attempt) {
		if (buf_reserve(&b->d_cig, 4 * (size_t)cap_cig) || buf_reserve(&b->d_md, (size_t)cap_md)) return 1;
		GlbArgs a;
		memset(&a, 0, sizeof(a));
		a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p; a.par = *par;
		a.tasks = (const bwag_gtask_t *)b->d_tasks.p; a.n_tasks = n_tasks;
		a.res = (bwag_gres_t *)b->d_res.p; a.cigar = (u32 *)b->d_cig.p; a.md = (char *)b->d_md.p;
		a.cap_cig = cap_cig; a.cap_md = cap_md; a.n_cig = &c->d_cnt->n_cig; a.n_md = &c->d_cnt->n_md;
		a.w_cig = (u32 *)c->s_wcig.p; a.w_md = (char *)c->s_wmd.p; a.cap_wcig = cap_wcig; a.cap_wmd = cap_wmd;
		a.eh = (int *)c->s_eh.p; a.rseq = (uint8_t *)c->s_rseq.p; a.qseq = (uint8_t *)c->s_qseq.p; a.z = (uint8_t *)c->s_z.p;
		a.cap_q = cap_q; a.cap_r = cap_r; a.cap_z = cap_z;
		a.next_task = &c->d_cnt->next_task; a.cells = &c->d_cnt->glb_cells; a.flags = &c->d_cnt->flags;
		if (reset_counters(c)) return 1;
		CK(cudaEventRecord(c->ev0, c->stream));
		if (k5_lane) {   /* DP + backtrack of the short-read CIGAR requests, one lane per request; the warp kernel then adds NM/MD and takes the rest */
			GlbLaneArgs la;
			memset(&la, 0, sizeof(la));
			la.codes = a.codes; la.off = a.off; la.par = *par; la.tasks = a.tasks; la.n_tasks = n_tasks;
			la.pre_n = (int *)b->d_pre_n.p; la.pre_score = (int *)b->d_pre_score.p; la.pre_cig = (u32 *)b->d_pre_cig.p;
			la.z = (uint8_t *)c->s_zl.p; la.cap_z = k5l_cap_z; la.next_task = &c->d_cnt->next_task; la.cells = &c->d_cnt->glb_cells; la.n_pre = &c->d_cnt->n_pre;
			BWAG_LAUNCH(k_global_lane, k5l_grid, K5L_THREADS, k5l_smem, c->stream, c->ix, la);
			CK(cudaGetLastError());
			CK(cudaMemsetAsync(&c->d_cnt->next_task, 0, sizeof(int), c->stream));
			a.pre_n = la.pre_n; a.pre_score = la.pre_score; a.pre_cig = la.pre_cig;
			++c->st.n_launch;
		}
		a.smem_per_warp = k5_sm ? k5_per_warp : 0; a.z_sm_bytes = k5_sm ? k5_zsm : 0;
		if (getenv("BWA_B200_PROFILE"))
			fprintf(stderr, "[prof] global alignment: warp-per-request kernel %s (scratch in %s memory, %s row sweep), %d requests, grid %d x %d\n",
			        k5_sm ? (k5_fast ? "k_global_sm_fast" : "k_global_sm") : (k5_fast ? "k_global_fast" : "k_global"), k5_sm ? "shared" : "global",
			        k5_fast ? "lean" : "first", n_tasks, grid, K5_THREADS);
		if (k5_sm && k5_fast) BWAG_LAUNCH(k_global_sm_fast, grid, K5_THREADS, k5_smem, c->stream, c->ix, a);
		else if (k5_sm) BWAG_LAUNCH(k_global_sm, grid, K5_THREADS, k5_smem, c->stream, c->ix, a);
		else if (k5_fast) BWAG_LAUNCH(k_global_fast, grid, K5_THREADS, 0, c->stream, c->ix, a);
		else BWAG_LAUNCH(k_global, grid, K5_THREADS, 0, c->stream, c->ix, a);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		if (fetch_counters(c)) return 1;
		c->st.ms_global += elapsed_at(c, "global", __FILE__, __LINE__); ++c->st.n_launch;
		if (k5_lane && getenv("BWA_B200_PROFILE")) fprintf(stderr, "[prof] global alignment: lane-per-request kernel made %u of %d CIGARs, grid %d x %d\n", c->h_cnt->n_pre, n_tasks, k5l_grid, K5L_THREADS);
		if (c->h_cnt->flags & 4u) return set_err("global alignment: a task exceeded the scratch capacity");
		if (!(c->h_cnt->flags & 16u)) break;
		if (attempt >= 3) return set_err("global alignment: output pools keep overflowing");
		cap_cig = (i64)c->h_cnt->n_cig + 1024; cap_md = (i64)c->h_cnt->n_md + 4096;
	}
	c->st.glb_cells += c->h_cnt->glb_cells;
	*nc_out = (i64)c->h_cnt->n_cig; *nm_out = (i64)c->h_cnt->n_md;
	return 0;
}

extern "C" int bwag_global(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, const bwag_gtask_t *tasks, bwag_galn_t *out)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	if (n_tasks <= 0) { out->res = 0; out->cigar = 0; out->md = 0; return 0; }
	i64 cap_z = 64, n_aln = 0, nc = 0, nm = 0;
	int cap_q = 4, cap_r = 16;
	for (int t = 0; t < n_tasks; ++t) {
		i64 lq = tasks[t].qe - tasks[t].qb, rl = tasks[t].re - tasks[t].rb;
		if (lq > cap_q) cap_q = (int)lq;
		if (rl > cap_r) cap_r = (int)rl;
		if (tasks[t].mode == BWAG_G_REG2ALN) { /* backtrack bytes of the widest band this task can reach */
			i64 d = rl > lq ? rl - lq : lq - rl, wmax = (i64)par->w << 2;
			if (d + 3 > wmax) wmax = d + 3;
			i64 ncol = lq < 2 * wmax + 1 ? lq : 2 * wmax + 1;
			if (ncol * rl > cap_z) cap_z = ncol * rl;
			++n_aln;
		}
	}
	if (buf_reserve(&b->d_tasks, sizeof(bwag_gtask_t) * (size_t)n_tasks)) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	H2D(c, b->d_tasks.p, tasks, sizeof(bwag_gtask_t) * (size_t)n_tasks);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_h2d += elapsed_at(c, "h2d", __FILE__, __LINE__);
	b->tail_ready = 0;   /* the request pool of a preceding bwag_tail_regs is gone */
	if (run_global(b, par, n_tasks, cap_q, cap_r, cap_z, n_aln, &nc, &nm)) return 1;
	if (hbuf_reserve(&b->h_res, sizeof(bwag_gres_t) * (size_t)n_tasks) || hbuf_reserve(&b->h_cig, 4 * (size_t)(nc + 1)) || hbuf_reserve(&b->h_md, (size_t)nm + 16)) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	D2H(c, b->h_res.p, b->d_res.p, sizeof(bwag_gres_t) * (size_t)n_tasks);
	if (nc) D2H(c, b->h_cig.p, b->d_cig.p, 4 * (size_t)nc);
	if (nm) D2H(c, b->h_md.p, b->d_md.p, (size_t)nm);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	out->res = (const bwag_gres_t *)b->h_res.p; out->cigar = (const uint32_t *)b->h_cig.p; out->md = (const char *)b->h_md.p;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ stage 4 */

#define TAIL_LOGN 4096
extern "C" int bwag_ctx_set_contigs(bwag_ctx_t *c, int n_seqs, const int64_t *offset, const int32_t *len, const uint8_t *is_alt, const char *const *names)
{
	CK(cudaSetDevice(c->device));
	size_t l_names = 0;
	for (int i = 0; i < n_seqs; ++i) l_names += strlen(names[i]);
	/* one block: offsets | lengths | name offsets | ALT flags | names | log table (8-byte aligned first) */
	const size_t o_off = 0, o_log = o_off + 8 * (size_t)n_seqs, o_len = o_log + 8 * TAIL_LOGN, o_noff = o_len + 4 * (size_t)n_seqs, o_alt = o_noff + 4 * ((size_t)n_seqs + 1), o_names = o_alt + (size_t)n_seqs, total = o_names + l_names + 16;
	char *h = (char *)malloc(total);
	if (!h) return set_err("out of memory");
	memset(h, 0, total);
	memcpy(h + o_off, offset, 8 * (size_t)n_seqs);
	memcpy(h + o_len, len, 4 * (size_t)n_seqs);
	memcpy(h + o_alt, is_alt, (size_t)n_seqs);
	{
		int *no = (int *)(h + o_noff), at = 0;
		for (int i = 0; i < n_seqs; ++i) { const size_t l = strlen(names[i]); no[i] = at; memcpy(h + o_names + at, names[i], l); at += (int)l; }
		no[n_seqs] = at;
		double *lt = (double *)(h + o_log);
		for (int i = 0; i < TAIL_LOGN; ++i) lt[i] = log((double)i);   /* the host's libm: log(0) = -inf included */
	}
	pthread_mutex_lock(&c->mu);
	if (c->tail.p) { cudaStreamSynchronize(c->lane.stream); cudaFree(c->tail.p); c->tail.p = 0; c->have_ctg = 0; }
	cudaError_t e = cudaMalloc(&c->tail.p, total);
	if (e == cudaSuccess) e = cudaMemcpy(c->tail.p, h, total, cudaMemcpyHostToDevice);
	free(h);
	if (e != cudaSuccess) { pthread_mutex_unlock(&c->mu); return set_err("contig table upload failed: %s", cudaGetErrorString(e)); }
	char *d = (char *)c->tail.p;
	c->tctg.l_pac = c->lane.ix.l_pac; c->tctg.n_seqs = n_seqs;
	c->tctg.off = (const i64 *)(d + o_off); c->tctg.len = (const int *)(d + o_len); c->tctg.alt = (const uint8_t *)(d + o_alt);
	c->tctg.names = d + o_names; c->tctg.name_off = (const int *)(d + o_noff);
	c->d_logtab = (const double *)(d + o_log);
	c->have_ctg = 1;
	pthread_mutex_unlock(&c->mu);
	return 0;
}

extern "C" int bwag_tail_regs(bwag_batch_t *b, const mem_opt_t *opt, const bwag_sw_par_t *sp, const uint64_t **pe_is, const uint8_t **cflag)
{
	Lane *c = &b->lane;
	const bwag_ctx_t *pc = b->ctx;
	CK(cudaSetDevice(pc->device));
	if (!pc->have_ctg) return BWAG_UNSUPPORTED;
	if (c->baseline) return BWAG_DECLINED;   /* the baseline of the start-up self-check is the host-side post-processing */
	if (!b->regs_on_device) return set_err("bwag_tail_regs needs a preceding bwag_chain_extend(..., NULL) on the same batch");
	const int n = b->n, pe = !!(opt->flag & MEM_F_PE);
	if (pe && (n & 1)) return set_err("paired-end batch with an odd number of reads");
	const i64 cap = b->n_seeds + 1;   /* regions <= seeds */
	if (buf_reserve(&b->d_dregs, sizeof(mem_alnreg_t) * (size_t)cap) || buf_reserve(&b->d_tasks, sizeof(bwag_gtask_t) * (size_t)cap) ||
	    buf_reserve(&b->d_dreg_beg, 8 * (size_t)(n + 1)) || buf_reserve(&b->d_dreg_n, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_task_beg, 8 * (size_t)(n + 1)) ||
	    buf_reserve(&b->d_cflag, (size_t)n + 16) || buf_reserve(&b->d_pe_is, 8 * (size_t)(n / 2 + 1))) return 1;
	TailRegsArgs a;
	memset(&a, 0, sizeof(a));
	a.n_reads = n; a.pe = pe; a.opt = *opt; a.ctg = pc->tctg;
	a.n_raw = (const int *)b->d_nregs.p; a.xregs = (const bwag_xreg_t *)b->d_regs.p; a.reg_base = (const i64 *)b->d_reg_base.p; a.chain_beg = (const i64 *)b->d_chain_beg.p;
	a.chain_rid = (const int *)b->d_chain_rid.p; a.chain_frac = (const float *)b->d_chain_frac.p;
	a.dregs = (mem_alnreg_t *)b->d_dregs.p; a.dreg_beg = (i64 *)b->d_dreg_beg.p; a.dreg_n = (int *)b->d_dreg_n.p; a.task_beg = (i64 *)b->d_task_beg.p; a.cflag = (uint8_t *)b->d_cflag.p;
	a.cap_dregs = cap; a.tasks = (bwag_gtask_t *)b->d_tasks.p; a.cap_tasks = cap; a.pe_is = (u64 *)b->d_pe_is.p;
	a.n_dregs = &c->d_cnt->t_dregs; a.n_tasks = &c->d_cnt->t_tasks; a.max_z = &c->d_cnt->t_max_z; a.max_lq = &c->d_cnt->t_max_lq; a.max_rl = &c->d_cnt->t_max_rl;
	if (reset_counters(c)) return 1;
	const int n_units = pe ? n >> 1 : n;
	CK(cudaEventRecord(c->ev0, c->stream));
	BWAG_LAUNCH(k_tail_regs, (n_units + 127) / 128, 128, 0, c->stream, a);
	CK(cudaGetLastError());
	CK(cudaEventRecord(c->ev1, c->stream));
	if (fetch_counters(c)) return 1;
	c->st.ms_tail += elapsed_at(c, "tail_regs", __FILE__, __LINE__); ++c->st.n_launch;
	const i64 n_tasks = (i64)c->h_cnt->t_tasks;
	if (n_tasks > cap || (i64)c->h_cnt->t_dregs > cap) return set_err("stage 4: more regions than seeds?");
	if (n_tasks >= ((i64)1 << 31)) return set_err("stage 4: too many alignment requests in one batch; use smaller chunks");
	const int cap_q = c->h_cnt->t_max_lq, cap_r = c->h_cnt->t_max_rl;
	const i64 cap_z = (i64)c->h_cnt->t_max_z;
	if (n_tasks > 0) {
		i64 nc = 0, nm = 0;
		if (run_global(b, sp, (int)n_tasks, cap_q, cap_r, cap_z, n_tasks, &nc, &nm)) return 1;
	}
	if (hbuf_reserve(&b->h_cflag, (size_t)n + 16) || hbuf_reserve(&b->h_pe_is, 8 * (size_t)(n / 2 + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	D2H(c, b->h_cflag.p, b->d_cflag.p, (size_t)n);
	if (pe) D2H(c, b->h_pe_is.p, b->d_pe_is.p, 8 * (size_t)(n / 2));
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	b->tail_ready = 1;
	if (pe_is) *pe_is = pe ? (const uint64_t *)b->h_pe_is.p : 0;
	if (cflag) *cflag = (const uint8_t *)b->h_cflag.p;
	return 0;
}

extern "C" int bwag_tail_sam(bwag_batch_t *b, const mem_opt_t *opt, const mem_pestat_t pes[4], const double *const pair_tab[4], const double *log_tab,
                             int64_t n_processed, const char *rg_id, bwag_sam_t *out)
{
	Lane *c = &b->lane;
	const bwag_ctx_t *pc = b->ctx;
	(void)log_tab;   /* the context keeps its own copy (bwag_ctx_set_contigs computes it with the same libm) */
	CK(cudaSetDevice(pc->device));
	if (!pc->have_ctg) return BWAG_UNSUPPORTED;
	if (!b->tail_ready) return set_err("bwag_tail_sam needs a preceding bwag_tail_regs on the same batch");
	const int n = b->n, pe = !!(opt->flag & MEM_F_PE);
	TailSamArgs g;
	memset(&g, 0, sizeof(g));
	g.n_reads = n; g.pe = pe; g.opt = *opt; g.ctg = pc->tctg; g.logtab = pc->d_logtab; g.n_processed = n_processed;
	size_t tab_bytes = 256;   /* read-group id first */
	if (pe) {
		memcpy(g.pes, pes, 4 * sizeof(mem_pestat_t));
		for (int d = 0; d < 4; ++d) if (pair_tab && pair_tab[d] && !pes[d].failed && pes[d].high >= pes[d].low) tab_bytes += 8 * ((size_t)pes[d].high - pes[d].low + 1);
	}
	if (buf_reserve(&b->d_ptab, tab_bytes) || hbuf_reserve(&b->h_ptab, tab_bytes)) return 1;
	{
		char *h = (char *)b->h_ptab.p;
		size_t at = 256;
		const size_t l_rg = rg_id ? strlen(rg_id) : 0;
		memset(h, 0, 256);
		if (l_rg > 255) return set_err("read-group id too long");
		if (l_rg) memcpy(h, rg_id, l_rg);
		g.rg = (const char *)b->d_ptab.p; g.l_rg = (int)l_rg;
		if (pe) for (int d = 0; d < 4; ++d) if (pair_tab && pair_tab[d] && !pes[d].failed && pes[d].high >= pes[d].low) {
			const size_t bytes = 8 * ((size_t)pes[d].high - pes[d].low + 1);
			memcpy(h + at, pair_tab[d], bytes);
			g.ptab[d] = (const double *)((char *)b->d_ptab.p + at);
			at += bytes;
		}
		H2D(c, b->d_ptab.p, h, tab_bytes);
	}
	g.codes = (const uint8_t *)b->d_codes.p; g.off = (const i64 *)b->d_off.p;
	g.dregs = (const mem_alnreg_t *)b->d_dregs.p; g.dreg_beg = (const i64 *)b->d_dreg_beg.p; g.dreg_n = (const int *)b->d_dreg_n.p; g.task_beg = (const i64 *)b->d_task_beg.p; g.cflag = (const uint8_t *)b->d_cflag.p;
	g.res = (const bwag_gres_t *)b->d_res.p; g.cigar = (const u32 *)b->d_cig.p; g.md = (const char *)b->d_md.p;
	if (buf_reserve(&b->d_rec, sizeof(bwag_samrec_t) * (size_t)(n + 1))) return 1;
	g.rec = (bwag_samrec_t *)b->d_rec.p;
	g.n_text = &c->d_cnt->t_text; g.n_complex = &c->d_cnt->t_complex;
	i64 cap_text = b->total_bases + 176 * (i64)n + 4096;
	const int n_units = pe ? n >> 1 : n;
	/* a slot holds SEQ and up to 176 bytes of the rest: the records of reads up to TAIL_SLOT_MAX - 176 - l_rg bases are staged */
	g.slot = (b->max_len + 176 + g.l_rg + 15) & ~15;
	if (g.slot > TAIL_SLOT_MAX) g.slot = TAIL_SLOT_MAX;
	const size_t sam_smem = (size_t)128 * g.slot;   /* <= TAIL_SAM_SMEM_MAX, the kernel's limit set once per context */
	for (int attempt = 0;; ++attempt) {
		if (buf_reserve(&b->d_text, (size_t)cap_text)) return 1;
		g.text = (char *)b->d_text.p; g.cap_text = cap_text;
		if (reset_counters(c)) return 1;
		CK(cudaEventRecord(c->ev0, c->stream));
		BWAG_LAUNCH(k_tail_sam, (n_units + 127) / 128, 128, sam_smem, c->stream, g);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		if (fetch_counters(c)) return 1;
		c->st.ms_tail += elapsed_at(c, "tail_sam", __FILE__, __LINE__); ++c->st.n_launch;
		if ((i64)c->h_cnt->t_text <= cap_text) break;
		if (attempt >= 2) return set_err("stage 4: the text pool keeps overflowing");
		cap_text = (i64)c->h_cnt->t_text + 4096;
	}
	const i64 n_text = (i64)c->h_cnt->t_text;
	if (hbuf_reserve(&b->h_rec, sizeof(bwag_samrec_t) * (size_t)(n + 1)) || hbuf_reserve(&b->h_text, (size_t)n_text + 16)) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	D2H(c, b->h_rec.p, b->d_rec.p, sizeof(bwag_samrec_t) * (size_t)n);
	if (n_text) D2H(c, b->h_text.p, b->d_text.p, (size_t)n_text);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	c->st.tail_reads += (u64)n; c->st.tail_complex += c->h_cnt->t_complex;
	out->rec = (const bwag_samrec_t *)b->h_rec.p; out->text = (const char *)b->h_text.p; out->n_text = n_text; out->n_complex = (int64_t)c->h_cnt->t_complex;
	return 0;
}
