/* bwag_aln.cu -- the BWA-backtrack search of `bwa aln` (bwa_cal_sa_reg_gap + bwt_match_gap, bwtaln.c:83-126, bwtgap.c:109-264),
 * one lane per read.
 *
 * A1 k_aln: persistent lanes take reads from an atomic counter.  Per read the lane computes the widths of the reversed read (and of
 * its seed: the first seed_len bases, reversed) with bwt_cal_width, then runs the backtracking search.  The reference keeps its
 * priority queue as one LIFO per score (aln_score = n_mm*s_mm + n_gapo*s_gapo + n_gape*s_gape) and always pops the top of the
 * lowest non-empty score; the pop order is the whole semantics, so any layout that pops the same entry gives the same hits.
 * Here the queue lives in the lane's arena of global memory:
 *   - nodes of 32 bytes (AlnNode): k, l, then i | last_diff_pos << 16, n_mm | n_gapo << 8 | n_gape << 16 | state << 24,
 *     n_ins | n_del << 16, and the index of the next node of the same score;
 *   - per score the index of its top node (heads[]) and one bit per non-empty score (mask[]) to find the next one after a pop;
 *   - popped nodes go to a free list; new nodes come from it or from a bump pointer at the bottom of the node array;
 *   - the read's hits (bwag_aln1_t, the .sai layout) grow downwards from the top of the same array.
 * When bump pointer and hits meet, the lane abandons the read and lists it for a second run with a larger arena (the search
 * is deterministic, so a restarted read gives the same hits).  A finished read's hits go to the batch's pool (atomicAdd); if the
 * pool is full the read is listed for another run too, after the pool has grown.
 * A2 k_aln_gather: the hits in read order, at the offsets of a one-block scan of the counts (k_fm_scan32). */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"
#include "bwag_drv.h"

#define A_M 0   /* states of a queue entry (bwtgap.c:11-13) */
#define A_I 1
#define A_D 2

__device__ __forceinline__ u64 aln_sel4(int c, u64 a0, u64 a1, u64 a2, u64 a3) { return c == 0 ? a0 : c == 1 ? a1 : c == 2 ? a2 : a3; }

/* bwt_2occ4(k, l) (bwt.c:189-220) on the 32-byte blocks: the ranks of all four symbols at k and at l (k <= l); k = (u64)-1 gives
 * zeros; one block load when both positions lie in the same 64-symbol block */
__device__ __forceinline__ void aln_occ2(const DevIndex &ix, u64 k, u64 l, u64 tk[4], u64 tl[4])
{
	const bool kv = k != (u64)-1;
	const u64 kp = k - (k >= ix.primary), lp = l - (l >= ix.primary);
	uint4 b0, b1, c0, c1;
	bwag_ld_block(ix.bwt + ((lp >> 6) << 1), b0, b1);
	if (kv && (kp >> 6) != (lp >> 6)) bwag_ld_block(ix.bwt + ((kp >> 6) << 1), c0, c1);
	else { c0 = b0; c1 = b1; }
	bwag_block_counts(ix, b0, b1, lp, tl);
	if (kv) bwag_block_counts(ix, c0, c1, kp, tk);
	else { tk[0] = tk[1] = tk[2] = tk[3] = 0; }
}

/* one backward step by base c (bwt_2occ, bwt.c:132-163): [k, l] -> [L2[c] + occ(k-1, c) + 1, L2[c] + occ(l, c)] */
__device__ __forceinline__ void aln_step(const DevIndex &ix, int c, u64 &k, u64 &l)
{
	u64 tk[4], tl[4];
	aln_occ2(ix, k - 1, l, tk, tl);
	const u64 L2 = aln_sel4(c, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]);
	k = L2 + aln_sel4(c, tk[0], tk[1], tk[2], tk[3]) + 1;
	l = L2 + aln_sel4(c, tl[0], tl[1], tl[2], tl[3]);
}

/* bwt_cal_width (bwtaln.c:57-81) of the string str[i] = q[n-1-i], i < n (the reversed read, or its reversed seed) */
__device__ void aln_width(const DevIndex &ix, int n, const uint8_t *q, u64 *ww, int *wb)
{
	u64 k = 0, l = ix.seq_len;
	int bid = 0;
	for (int i = 0; i < n; ++i) {
		const int c = q[n - 1 - i];
		if (c < 4) aln_step(ix, c, k, l);
		if (k > l || c > 3) { k = 0; l = ix.seq_len; ++bid; }
		ww[i] = l - k + 1;
		wb[i] = bid;
	}
	ww[n] = 0;
	wb[n] = ++bid;
}

__device__ __forceinline__ int aln_log2(u32 v)   /* int_log2, bwtgap.c:98-107 */
{
	return v ? 31 - __clz((int)v) : 0;
}

struct AlnQueue {
	int *heads; u64 *mask; AlnNode *nodes;
	int cap, bump, free_top, n_hits, n_entries, best, n_buckets;
};

/* gap_push (bwtgap.c:48-69); false: the arena is full */
__device__ __forceinline__ bool q_push(AlnQueue &q, int score, int i, u64 k, u64 l, int n_mm, int n_gapo, int n_gape, int n_ins, int n_del, int state, int is_diff)
{
	int x;
	if (q.free_top >= 0) { x = q.free_top; q.free_top = q.nodes[x].next; }
	else if (q.bump < q.cap - q.n_hits) x = q.bump++;
	else return false;
	AlnNode e;
	e.k = k; e.l = l;
	e.pos = (u32)i | (u32)(is_diff ? i : 0) << 16;
	e.cnt = (u32)(n_mm & 0xff) | (u32)(n_gapo & 0xff) << 8 | (u32)(n_gape & 0xff) << 16 | (u32)state << 24;   /* the entry's bit fields */
	e.id = (u32)(n_ins & 0xffff) | (u32)(n_del & 0xffff) << 16;
	e.next = q.heads[score];
	q.nodes[x] = e;
	q.heads[score] = x;
	q.mask[score >> 6] |= 1ull << (score & 63);
	++q.n_entries;
	if (q.best > score) q.best = score;
	return true;
}

/* gap_pop (bwtgap.c:71-84): the top of the lowest non-empty score */
__device__ __forceinline__ AlnNode q_pop(AlnQueue &q)
{
	const int b = q.best, x = q.heads[b];
	const AlnNode e = q.nodes[x];
	q.heads[b] = e.next;
	q.nodes[x].next = q.free_top; q.free_top = x;
	--q.n_entries;
	if (e.next < 0) {
		q.mask[b >> 6] &= ~(1ull << (b & 63));
		if (q.n_entries == 0) q.best = q.n_buckets;
		else {
			int w = (b + 1) >> 6;
			u64 m = q.mask[w] & (~0ull << ((b + 1) & 63));
			while (m == 0) m = q.mask[++w];
			const u32 lo = (u32)m;
			q.best = (w << 6) + (lo ? __ffs((int)lo) - 1 : 32 + __ffs((int)(u32)(m >> 32)) - 1);
		}
	}
	return e;
}

/* read r: 0 = searched (its n_hit hits are the top n_hit nodes, first hit at the very top), 1 = the arena is too small */
__device__ int aln_read(const DevIndex &ix, const AlnArgs &a, unsigned char *ar, const AlnLayout &L, int r, int &n_hit)
{
	const bwag_aln_par_t &p = a.par;
	const uint8_t *q = a.codes + a.off[r];
	const int len = (int)(a.off[r + 1] - a.off[r]);
	const int md = p.max_diff[r];
	u64 *ww = (u64 *)(ar + L.ww), *sw = (u64 *)(ar + L.sw);
	int *wb = (int *)(ar + L.wb), *sb = (int *)(ar + L.sb);
	n_hit = 0;
	{   /* too many N: no hit (bwtgap.c:121-127) */
		int nn = 0;
		for (int j = 0; j < len; ++j) nn += q[j] > 3;
		if (nn > md) return 0;
	}
	aln_width(ix, len, q, ww, wb);
	const bool has_seed = p.seed_len < len;
	if (has_seed) aln_width(ix, p.seed_len, q, sw, sb);
	const int sl = has_seed ? p.seed_len : 0x7fffffff;   /* local_opt.seed_len (bwtaln.c:112) */
	const bool gape = (p.mode & BWAG_ALN_GAPE) != 0, nonstop = (p.mode & BWAG_ALN_NONSTOP) != 0, loggap = (p.mode & BWAG_ALN_LOGGAP) != 0;
#define ALN_SCORE(m, o, e) ((m) * p.s_mm + (o) * p.s_gapo + (e) * p.s_gape)
	int best_score = ALN_SCORE(md + 1, p.max_gapo + 1, p.max_gape + 1), max_diff = md, best_cnt = 0;

	AlnQueue Q;
	Q.heads = (int *)(ar + L.heads); Q.mask = (u64 *)(ar + L.mask); Q.nodes = (AlnNode *)(ar + L.nodes);
	Q.cap = a.cap_nodes; Q.bump = 0; Q.free_top = -1; Q.n_hits = 0; Q.n_entries = 0; Q.n_buckets = a.n_buckets; Q.best = a.n_buckets;
	for (int s = 0; s < a.n_buckets; ++s) Q.heads[s] = -1;
	for (int s = 0; s < (a.n_buckets + 63) >> 6; ++s) Q.mask[s] = 0;
#define ALN_HIT(j) (*(bwag_aln1_t *)(Q.nodes + (Q.cap - 1 - (j))))   /* hit j, from the top of the node array down */
#define ALN_PUSH(i_, k_, l_, mm_, go_, ge_, in_, de_, st_, df_) \
	do { if (!q_push(Q, ALN_SCORE(mm_, go_, ge_), i_, k_, l_, mm_, go_, ge_, in_, de_, st_, df_)) return 1; } while (0)
	ALN_PUSH(len, (u64)0, ix.seq_len, 0, 0, 0, 0, 0, A_M, 0);

	while (Q.n_entries) {
		if (Q.n_entries > p.max_entries) break;
		const AlnNode e = q_pop(Q);
		u64 k = e.k, l = e.l;
		int i = (int)(e.pos & 0xffff);
		const int e_ldp = (int)(e.pos >> 16);
		const int e_mm = (int)(e.cnt & 0xff), e_go = (int)(e.cnt >> 8 & 0xff), e_ge = (int)(e.cnt >> 16 & 0xff), e_st = (int)(e.cnt >> 24);
		const int e_ins = (int)(e.id & 0xffff), e_del = (int)(e.id >> 16);
		const int e_score = ALN_SCORE(e_mm, e_go, e_ge);
		/* the entry's info>>21 (11 bits of the score) against best_score + s_mm, compared unsigned as in bwtgap.c:143 */
		if (!nonstop && ((u32)e_score & 0x7ffu) > (u32)(best_score + p.s_mm)) break;

		int m = max_diff - (e_mm + e_go);
		if (gape) m -= e_ge;
		if (m < 0) continue;
		int m_seed = 0;
		if (has_seed) {
			m_seed = p.max_seed_diff - (e_mm + e_go);
			if (gape) m_seed -= e_ge;
		}
		if (i > 0 && m < wb[i - 1]) continue;

		bool hit = i == 0;
		if (!hit && m == 0 && (e_st == A_M || gape || e_ge == p.max_gape)) {   /* no difference left: bwt_match_exact_alt */
			u64 kk = k, ll = l;
			int j = i - 1;
			for (; j >= 0; --j) {
				const int c = q[len - 1 - j];   /* seq[j] = complement of the reversed read */
				if (c > 3) break;
				aln_step(ix, 3 - c, kk, ll);
				if (kk > ll) break;
			}
			if (j >= 0 || (int)(ll - kk + 1) == 0) continue;   /* an N, no match, or the int return value is 0 */
			k = kk; l = ll; hit = true;
		}
		if (hit) {
			const int score = e_score;
			if (n_hit == 0) {
				best_score = score;
				const int best_diff = e_mm + e_go + (gape ? e_ge : 0);
				if (!nonstop) max_diff = best_diff + 1 > md ? md : best_diff + 1;   /* top2 behaviour */
			}
			if (score == best_score) best_cnt = (int)((u32)best_cnt + (u32)(l - k + 1));   /* int += u64, as the reference */
			else if (best_cnt > p.max_top2) break;
			bool add = true;
			if (e_go)   /* the same hit again: a gap in a tandem repeat */
				for (int j = 0; j < n_hit; ++j)
					if (ALN_HIT(j).k == k && ALN_HIT(j).l == l) { add = false; break; }
			if (add) {
				{   /* gap_shadow (bwtgap.c:86-96): x is an int there */
					const u64 x = (u64)(i64)(int)(l - k + 1);
					int jj = 0;
					for (int t = 0; t < e_ldp; ++t) {
						if (ww[t] > x) ww[t] -= x;
						else if (ww[t] == x) { wb[t] = 1; ww[t] = ix.seq_len - (u64)(++jj); }
					}
				}
				if (Q.bump >= Q.cap - Q.n_hits) return 1;
				bwag_aln1_t h;
				h.bits = (u64)(e_mm & 0xff) | (u64)(e_go & 0xff) << 8 | (u64)(e_ge & 0xff) << 16 | (u64)((u32)score & 0xfffff) << 24 |
				         (u64)(e_ins & 0x3ff) << 44 | (u64)(e_del & 0x3ff) << 54;
				h.k = k; h.l = l;
				ALN_HIT(n_hit) = h;
				++n_hit; ++Q.n_hits;
			}
			continue;
		}

		--i;
		u64 ck[4], cl[4];
		aln_occ2(ix, k - 1, l, ck, cl);
		const u64 occ = l - k + 1;
		bool allow_diff = true, allow_M = true;
		if (i > 0) {
			if (wb[i - 1] > m - 1) allow_diff = false;
			else if (wb[i - 1] == m - 1 && wb[i] == m - 1 && ww[i - 1] == ww[i]) allow_M = false;
			if (has_seed) {
				const int ii = i - (len - sl);
				if (ii > 0) {
					if (sb[ii - 1] > m_seed - 1) allow_diff = false;
					else if (sb[ii - 1] == m_seed - 1 && sb[ii] == m_seed - 1 && sw[ii - 1] == sw[ii]) allow_M = false;
				}
			}
		}
		/* indels */
		const int tmp = loggap ? aln_log2((u32)(e_ge + e_go)) / 2 + 1 : e_go + e_ge;
		if (allow_diff && i >= p.indel_end_skip + tmp && len - i >= p.indel_end_skip + tmp) {
			if (e_st == A_M) {
				if (e_go < p.max_gapo) {   /* gap open: insertion, then deletions */
					ALN_PUSH(i, k, l, e_mm, e_go + 1, e_ge, e_ins + 1, e_del, A_I, 1);
#pragma unroll
					for (int j = 0; j < 4; ++j) {
						const u64 kk = ix.L2[j] + ck[j] + 1, ll = ix.L2[j] + cl[j];
						if (kk <= ll) ALN_PUSH(i + 1, kk, ll, e_mm, e_go + 1, e_ge, e_ins, e_del + 1, A_D, 1);
					}
				}
			} else if (e_st == A_I) {
				if (e_ge < p.max_gape) ALN_PUSH(i, k, l, e_mm, e_go, e_ge + 1, e_ins + 1, e_del, A_I, 1);
			} else if (e_st == A_D) {
				if (e_ge < p.max_gape && (e_ge + e_go < max_diff || occ < (u64)(i64)p.max_del_occ)) {
#pragma unroll
					for (int j = 0; j < 4; ++j) {
						const u64 kk = ix.L2[j] + ck[j] + 1, ll = ix.L2[j] + cl[j];
						if (kk <= ll) ALN_PUSH(i + 1, kk, ll, e_mm, e_go, e_ge + 1, e_ins, e_del + 1, A_D, 1);
					}
				}
			}
		}
		/* mismatches */
		const int rc = q[len - 1 - i], si = rc > 3 ? 4 : 3 - rc;
		if (allow_diff && allow_M) {
#pragma unroll
			for (int j = 1; j <= 4; ++j) {
				const int c = (si + j) & 3, is_mm = j != 4 || si > 3;
				const u64 kk = aln_sel4(c, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]) + aln_sel4(c, ck[0], ck[1], ck[2], ck[3]) + 1;
				const u64 ll = aln_sel4(c, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]) + aln_sel4(c, cl[0], cl[1], cl[2], cl[3]);
				if (kk <= ll) ALN_PUSH(i, kk, ll, e_mm + is_mm, e_go, e_ge, e_ins, e_del, A_M, is_mm);
			}
		} else if (si < 4) {   /* exact match only */
			const u64 kk = aln_sel4(si, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]) + aln_sel4(si, ck[0], ck[1], ck[2], ck[3]) + 1;
			const u64 ll = aln_sel4(si, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]) + aln_sel4(si, cl[0], cl[1], cl[2], cl[3]);
			if (kk <= ll) ALN_PUSH(i, kk, ll, e_mm, e_go, e_ge, e_ins, e_del, A_M, 0);
		}
	}
#undef ALN_PUSH
#undef ALN_HIT
#undef ALN_SCORE
	return 0;
}

/* A1 */
__global__ void __launch_bounds__(ALN_THREADS) k_aln(DevIndex ix, AlnArgs a)
{
	const int lane = blockIdx.x * blockDim.x + threadIdx.x;
	if (lane >= a.n_lanes) return;
	unsigned char *ar = a.arena + (i64)lane * a.lane_bytes;
	const AlnLayout L = aln_layout(a.n_buckets, a.max_len, a.seed_cap, a.cap_nodes);
	const AlnNode *nodes = (const AlnNode *)(ar + L.nodes);
	for (;;) {
		const int w = atomicAdd(a.next, 1);
		if (w >= a.n_work) break;
		const int r = a.work ? a.work[w] : w;
		int n_hit = 0;
		u32 fail = aln_read(ix, a, ar, L, r, n_hit) ? 1u : 0u;
		if (!fail) {
			const u64 beg = atomicAdd(a.n_pool, (u64)n_hit);
			if (beg + (u64)n_hit > (u64)a.cap_pool) fail = 2;
			else {
				for (int j = 0; j < n_hit; ++j) a.pool[beg + j] = *(const bwag_aln1_t *)(nodes + (a.cap_nodes - 1 - j));
				a.n_aln[r] = n_hit; a.hit_beg[r] = (i64)beg;
			}
		}
		if (fail) {
			a.n_aln[r] = 0;
			atomicOr(a.flags, fail);
			a.redo[atomicAdd(a.n_redo, 1u)] = r;
		}
	}
}

/* A2: read r's hits to out[off[r] ..] */
__global__ void k_aln_gather(int n_reads, const int *n_aln, const i64 *hit_beg, const bwag_aln1_t *pool, const i64 *off, bwag_aln1_t *out)
{
	for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += gridDim.x * blockDim.x) {
		const int n = n_aln[r];
		const bwag_aln1_t *src = pool + hit_beg[r];
		bwag_aln1_t *dst = out + off[r];
		for (int j = 0; j < n; ++j) dst[j] = src[j];
	}
}

/* ------------------------------------------------------------------------------------------------ host driver */

#ifdef BWAG_CUSIM
#define ALN_BUDGET ((i64)256 << 20)   /* the emulator's device memory is the host's */
#else
#define ALN_BUDGET ((i64)6 << 30)     /* the lanes' arenas, next to the index (K1 takes as much) */
#endif
#define ALN_T1_NODES 4096             /* queue nodes per lane in tier 1 (fewer if the lanes do not fit the budget) */
#define ALN_T2_HITS 1024              /* tier 2: room for this many hits beyond max_entries + 9 queue entries, x4 per repeat at full size */

/* A1 over all reads with small arenas (tier 1), then over the reads it listed with larger arenas (tier 2, fewer lanes: 16 times
 * the nodes per round, up to max_entries + 9 entries and room for their hits), repeated while reads are listed (a full pool grows,
 * a full-size arena too small for the hits gets more room); then the scan of the counts and A2 */
extern "C" int bwag_aln(bwag_batch_t *b, const bwag_aln_par_t *par, bwag_aln_t *out)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	const int n = b->n;
	memset(out, 0, sizeof(*out));
	for (int r = 0; r < n; ++r)
		if (b->h_off[r + 1] - b->h_off[r] >= 65536) return set_err("read %d of the batch has %lld bases; reads of 65536 bases or more are not supported", r, (long long)(b->h_off[r + 1] - b->h_off[r]));
	if (par->s_mm < 0 || par->s_gapo < 0 || par->s_gape < 0) return set_err("negative penalties are not supported");
	if (par->seed_len < 0) return set_err("the seed length must not be negative");
	int md_max = 0;
	for (int r = 0; r < n; ++r) if (par->max_diff[r] > md_max) md_max = par->max_diff[r];
	/* every score pushed is below aln_score(max_diff+1, max_gapo+1, max_gape+1), the reference's number of stacks */
	const i64 n_buckets = (i64)(md_max + 1) * par->s_mm + (i64)((par->max_gapo > 0 ? par->max_gapo : 0) + 1) * par->s_gapo + (i64)((par->max_gape > 0 ? par->max_gape : 0) + 1) * par->s_gape + 1;
	if (n_buckets > (1 << 20)) return set_err("penalties too large: %lld queue scores", (long long)n_buckets);
	const int seed_cap = par->seed_len < b->max_len ? par->seed_len : b->max_len;
	const bool small = getenv("BWA_B200_TEST_SMALL_POOLS") != 0;   /* test hook: tier 1 and the pool too small for nearly every read */
	i64 cap_pool = small ? n / 8 + 1 : 2 * (i64)n + 1024;
	if (buf_reserve(&b->d_aln_md, (size_t)n + 16) || buf_reserve(&b->d_aln_n, 4 * ((size_t)n + 1)) || buf_reserve(&b->d_aln_beg, 8 * ((size_t)n + 1)) ||
	    buf_reserve(&b->d_aln_redo[0], 4 * ((size_t)n + 1)) || buf_reserve(&b->d_aln_redo[1], 4 * ((size_t)n + 1)) || buf_reserve(&b->d_aln_off, 8 * ((size_t)n + 1)) ||
	    buf_reserve(&b->d_aln_pool, sizeof(bwag_aln1_t) * (size_t)cap_pool) ||
	    hbuf_reserve(&b->h_aln_n, 4 * ((size_t)n + 1)) || hbuf_reserve(&b->h_aln_off, 8 * ((size_t)n + 1))) return 1;
	cap_pool = (i64)(b->d_aln_pool.cap / sizeof(bwag_aln1_t));
	if (n) H2D(c, b->d_aln_md.p, par->max_diff, (size_t)n);
	if (reset_counters(c)) return 1;
	int grid_lanes = 2 * ALN_THREADS;
#ifndef BWAG_CUSIM
	{
		int nb = 0;
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_aln, ALN_THREADS, 0));
		grid_lanes = b->ctx->n_sm * (nb > 0 ? nb : 1) * ALN_THREADS;
	}
#endif
	AlnArgs a;
	memset(&a, 0, sizeof(a));
	a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p;
	a.par = *par; a.par.max_diff = (const int8_t *)b->d_aln_md.p;
	a.n_buckets = (int)n_buckets; a.max_len = b->max_len; a.seed_cap = seed_cap;
	a.n_aln = (int *)b->d_aln_n.p; a.hit_beg = (i64 *)b->d_aln_beg.p;
	a.n_pool = &c->d_cnt->aln_pool; a.n_redo = &c->d_cnt->aln_redo; a.flags = &c->d_cnt->aln_flags; a.next = &c->d_cnt->aln_next;
	i64 cap_nodes = small ? 8 : ALN_T1_NODES, hit_room = ALN_T2_HITS;
	int lanes = n < grid_lanes ? (n > 0 ? n : 1) : grid_lanes;
	while (cap_nodes > 64 && lanes * aln_layout(a.n_buckets, a.max_len, seed_cap, cap_nodes).bytes > ALN_BUDGET) cap_nodes >>= 1;
	const int *work = 0;
	int n_work = n;
	for (int round = 0;; ++round) {
		const i64 lane_bytes = aln_layout(a.n_buckets, a.max_len, seed_cap, cap_nodes).bytes;
		if (lanes > ALN_BUDGET / lane_bytes) lanes = (int)(ALN_BUDGET / lane_bytes);
		if (lanes < 1) {
			int r = 0;
			if (work) CK(cudaMemcpy(&r, work, sizeof(int), cudaMemcpyDeviceToHost));
			return set_err("read %d of the batch needs a search queue of %lld entries, more than the device can give", r, (long long)cap_nodes);
		}
		if (buf_reserve(&b->d_aln_arena, (size_t)(lanes * lane_bytes))) return 1;
		a.work = work; a.n_work = n_work; a.arena = (unsigned char *)b->d_aln_arena.p; a.lane_bytes = lane_bytes;
		a.cap_nodes = (int)cap_nodes; a.n_lanes = lanes;
		a.pool = (bwag_aln1_t *)b->d_aln_pool.p; a.cap_pool = cap_pool;
		a.redo = (int *)b->d_aln_redo[round & 1].p;
		CK(cudaMemsetAsync(&c->d_cnt->aln_next, 0, sizeof(int), c->stream));
		CK(cudaMemsetAsync(&c->d_cnt->aln_redo, 0, 2 * sizeof(u32), c->stream));
		BWAG_LAUNCH(k_aln, (lanes + ALN_THREADS - 1) / ALN_THREADS, ALN_THREADS, 0, c->stream, c->ix, a);
		CK(cudaGetLastError());
		if (fetch_counters(c)) return 1;
		++c->st.n_launch;
		const u32 n_redo = c->h_cnt->aln_redo, flags = c->h_cnt->aln_flags;
		if (round == 0) out->n_tier2 = n_redo;
		if (n_redo == 0) break;
		if (flags & 2) {   /* the pool is full: it grows, the hits already in it stay */
			const i64 want = 2 * (i64)c->h_cnt->aln_pool + 1024;
			if (buf_grow_keep(c, &b->d_aln_pool, sizeof(bwag_aln1_t) * (size_t)cap_pool, sizeof(bwag_aln1_t) * (size_t)want)) return 1;
			cap_pool = (i64)(b->d_aln_pool.cap / sizeof(bwag_aln1_t));
		}
		/* tier 2 grows the arena 16-fold per round up to max_entries + 9 entries and the hit room: most listed reads need far
		 * less than the full size, and smaller arenas leave room for more lanes */
		const i64 queue_max = (i64)(par->max_entries > 0 ? par->max_entries : 0) + 9 + 1;
		if (round > 0 && (flags & 1) && cap_nodes >= queue_max + hit_room) hit_room *= 4;   /* a full-size arena overflowed: only its hits can have done that */
		cap_nodes = cap_nodes * 16 < queue_max + hit_room ? cap_nodes * 16 : queue_max + hit_room;
		if (cap_nodes > 0x7fffffff) cap_nodes = 0x7fffffff;
		work = (const int *)b->d_aln_redo[round & 1].p; n_work = (int)n_redo;
		lanes = n_work < grid_lanes ? n_work : grid_lanes;
	}
	/* A2 */
	BWAG_LAUNCH(k_fm_scan32, 1, FM_SCAN_THREADS, 0, c->stream, (const int *)b->d_aln_n.p, (i64)n, (i64 *)b->d_aln_off.p, &c->d_cnt->aln_total);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	const i64 total = (i64)c->h_cnt->aln_total;
	if (buf_reserve(&b->d_aln_out, sizeof(bwag_aln1_t) * ((size_t)total + 1)) || hbuf_reserve(&b->h_aln_out, sizeof(bwag_aln1_t) * ((size_t)total + 1))) return 1;
	if (n) BWAG_LAUNCH(k_aln_gather, fm_grid(b->ctx, n), 128, 0, c->stream, n, (const int *)b->d_aln_n.p, (const i64 *)b->d_aln_beg.p, (const bwag_aln1_t *)b->d_aln_pool.p,
	                   (const i64 *)b->d_aln_off.p, (bwag_aln1_t *)b->d_aln_out.p);
	CK(cudaGetLastError());
	c->st.n_launch += 2;
	if (n) D2H(c, b->h_aln_n.p, b->d_aln_n.p, 4 * (size_t)n);
	D2H(c, b->h_aln_off.p, b->d_aln_off.p, 8 * ((size_t)n + 1));
	if (total) D2H(c, b->h_aln_out.p, b->d_aln_out.p, sizeof(bwag_aln1_t) * (size_t)total);
	CK(stream_wait(c));
	out->n_aln = (const int32_t *)b->h_aln_n.p; out->off = (const int64_t *)b->h_aln_off.p; out->aln = (const bwag_aln1_t *)b->h_aln_out.p;
	return 0;
}
