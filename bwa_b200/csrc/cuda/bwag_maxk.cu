/* bwag_maxk.cu -- `bwa-b200 maxk`: per base of each sequence, the length of the longest match of the smem_next loop that covers it
 * (capped at 255), binned into the 256-bin histogram of maxk.c:11-66.
 *
 *   M1  k_maxk       persistent lanes; a lane takes one window [a, b) of one sequence with an atomicAdd and runs the chain of
 *                    bwt_smem1a calls (bwt.c:289-351, max_intv = 0) from the first base >= a while x < b, plus one call at the first
 *                    x >= b, on the query q[S, T) with S = max(0, a - MAXK_MARGIN) and T = min(len, b + MAXK_MARGIN).  Every match
 *                    paints max(cnt[j], min(end - start, 255)) over the part of it inside [a, b): no two lanes write the same byte;
 *   M2  k_maxk_hist  the batch's painted bytes into a 256 x u32 histogram per block, added to the batch's u64 one with one atomic
 *                    per bin per block.
 * Why windows give the reference's bytes (DESIGN.md §4.14): when each base occurs at least min_intv times in the BWT, cnt[j] is
 * min(255, the longest substring of the query that covers j and occurs >= min_intv times), whichever calls find it.  Cutting the
 * query MAXK_MARGIN = 255 bases outside the window leaves that value unchanged for every base of the window (a match the cut
 * shortens still covers the base with more than 255 bases), and bounds a lane's work and lists by W + 510 bases even inside an
 * exact repeat.  When the condition fails, the host passes one window per sequence: a = S = 0, b = T = len, the reference's chain.
 *
 * The lane keeps the bwt_smem1a state machine of K1 (bwag_smem.cu, smem_lane in its fastmap form with max_intv = 0): it advances
 * until it needs a bwt_extend, then the warp meets at one converged extend_step3 (bwag_ext.cuh).  The two interval lists of a call
 * keep their first MAXK_SLOTS entries in shared memory and the rest in per-lane global scratch of cap entries; a list that would
 * outgrow it sets a flag, abandons the window and reports its length, and the host runs the batch again with larger lists. */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"
#include "bwag_drv.h"
#include "bwag_ext.cuh"

#define MAXK_THREADS 128
#define MAXK_SLOTS 4             /* list entries per list in shared memory (32 bytes each) */
#define MAXK_MARGIN 255          /* bases of query kept on each side of a window */
#define MAXK_HIST_THREADS 256

struct MaxkCtr {
	int next_win; u32 flags; u32 need; u32 pad;
	u64 max_ns;                  /* the longest window, device-clock nanoseconds */
	u64 touches;                 /* Occ blocks as the reference counts them (bwt.c:194-197) */
	u64 hist[256];
};

struct MaxkArgs {
	const uint8_t *codes; const i64 *off; int n_seqs;
	const i64 *win_off;          /* [n_seqs + 1]: first window of each sequence */
	i64 n_win, window;
	int min_intv, cap;           /* cap: entries per list (the first MAXK_SLOTS in shared memory) */
	uint8_t *cnt;                /* one byte per base of the batch, zeroed */
	ulonglong2 *scratch;         /* per lane: 2 lists x cap entries x 32 bytes */
	MaxkCtr *ctr;
};

enum { MK_IDLE = 0, MK_FWD, MK_BWD, MK_NONE };

__device__ __forceinline__ u64 mk_now()
{
#ifdef BWAG_CUSIM
	return 0;
#else
	u64 t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return t;
#endif
}

__global__ void __launch_bounds__(MAXK_THREADS)
k_maxk(DevIndex ix, MaxkArgs a)
{
	/* [2 lists][MAXK_SLOTS][2 halves][MAXK_THREADS]: a warp's 16-byte accesses to one slot are consecutive */
	__shared__ ulonglong2 s_ent[2 * MAXK_SLOTS * 2 * MAXK_THREADS];
	const int tid = threadIdx.x;
	ulonglong2 *gl = a.scratch + ((i64)blockIdx.x * blockDim.x + tid) * (i64)(4 * a.cap);
#define MK_PTR(l, idx, h) ((idx) < MAXK_SLOTS ? &s_ent[((((l) * MAXK_SLOTS) + (idx)) * 2 + (h)) * MAXK_THREADS + tid] : &gl[(((l) * (i64)a.cap) + (idx)) * 2 + (h)])
#define MK_ST(l, idx, X0, X1, X2, E) do { ulonglong2 u_, v_; u_.x = (X0); u_.y = (X1); v_.x = (X2); v_.y = (u64)(E); *MK_PTR(l, idx, 0) = u_; *MK_PTR(l, idx, 1) = v_; } while (0)
#define MK_LD(l, idx, X0, X1, X2, E) do { const ulonglong2 u_ = *MK_PTR(l, idx, 0), v_ = *MK_PTR(l, idx, 1); X0 = u_.x; X1 = u_.y; X2 = v_.x; E = (int)v_.y; } while (0)

	i64 w = -1;
	int len = 0, wa = 0, wb = 0, S = 0, T = 0, x = 0, st = MK_IDLE;
	bool extra = false;
	const uint8_t *q = 0;
	uint8_t *cnt = 0;
	int sx = 0, i = 0, j = 0, n_prev = 0, n_curr = 0, pl = 0, rev_first = 0, ret = 0, last_start = 0, ikend = 0, pend = 0;
	bool m_any = false;
	u64 ik0 = 0, ik1 = 0, ik2 = 0, e0 = 0, e1 = 0, e2 = 0, curr_last_x2 = 0, touches = 0, t_win = 0, max_ns = 0;
	u32 overflow = 0, need_max = 0;
	const u64 min_intv = (u64)a.min_intv;

	/* a match [s, e) of this call: the part inside the window takes max(cnt, min(e - s, 255)) (maxk.c:44-49) */
#define PAINT(s_, e_) do { const int s0_ = (s_), e0_ = (e_), l_ = e0_ - s0_ < 255 ? e0_ - s0_ : 255; \
		for (int p_ = s0_ > wa ? s0_ : wa; p_ < (e0_ < wb ? e0_ : wb); ++p_) if (cnt[p_] < l_) cnt[p_] = (uint8_t)l_; } while (0)
	/* a list entry for the next step; a list longer than cap abandons the window (the host repeats the batch with longer lists) */
#define PUSH(X0, X1, X2, E) do { if (n_curr < a.cap) { MK_ST(pl ^ 1, n_curr, X0, X1, X2, E); ++n_curr; } \
		else { overflow = 1; need_max = need_max > (u32)n_curr + 1 ? need_max : (u32)n_curr + 1; x = T; extra = true; st = MK_IDLE; } } while (0)
#define TURN_AROUND() do { ret = ikend; pl ^= 1; n_prev = n_curr; n_curr = 0; rev_first = 1; i = sx - 1; j = 0; st = MK_BWD; } while (0)
#define CALL_DONE() do { x = ret; st = MK_IDLE; } while (0)

	for (;;) {
		bool need = false;
		int back = 0;
		for (;;) {
			if (st == MK_IDLE) {
				if (w >= 0) {                       /* the next call of the window's chain (smem_next, bwamem_extra.c:86-96) */
					while (x < T && q[x] > 3) ++x;
					if (x < T && !extra) {
						if (x >= wb) extra = true;  /* the one call at the first x >= b */
						sx = x;
						INIT_INTV(q[x], ik0, ik1, ik2);
						ikend = x + 1; i = x + 1; n_curr = 0; m_any = false; st = MK_FWD;
						continue;
					}
					const u64 dt = mk_now() - t_win;
					if (dt > max_ns) max_ns = dt;
				}
				w = atomicAdd(&a.ctr->next_win, 1);
				if (w >= a.n_win) { w = -1; st = MK_NONE; break; }
				int lo = 0, hi = a.n_seqs - 1;     /* the sequence r with win_off[r] <= w < win_off[r + 1] */
				while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (a.win_off[mid] <= w) lo = mid; else hi = mid - 1; }
				const i64 o = a.off[lo];
				len = (int)(a.off[lo + 1] - o);
				q = a.codes + o; cnt = a.cnt + o;
				const i64 wa64 = (w - a.win_off[lo]) * a.window;
				wa = (int)wa64; wb = wa64 + a.window < (i64)len ? (int)(wa64 + a.window) : len;
				S = wa > MAXK_MARGIN ? wa - MAXK_MARGIN : 0;
				T = (i64)wb + MAXK_MARGIN < (i64)len ? wb + MAXK_MARGIN : len;
				x = wa; extra = false;
				t_win = mk_now();
				continue;
			}
			if (st == MK_FWD) {                     /* bwt.c:305-322 */
				if (i < T && q[i] <= 3) { e0 = ik0; e1 = ik1; e2 = ik2; need = true; back = 0; break; }
				PUSH(ik0, ik1, ik2, ikend);         /* end of the query or an ambiguous base: the current interval is the last candidate */
				if (st == MK_FWD) TURN_AROUND();
				continue;
			}
			if (st == MK_BWD) {                     /* bwt.c:328-345 */
				const int c = i < S ? -1 : (q[i] > 3 ? -1 : (int)q[i]);
				if (c < 0) {                        /* nothing extends: only the first candidate in visiting order can be a match */
					if (!m_any || i + 1 < last_start) {
						const int pe = (int)MK_PTR(pl, rev_first ? n_prev - 1 : 0, 1)->y;
						PAINT(i + 1, pe);
					}
					CALL_DONE();
					continue;
				}
				if (j < n_prev) { MK_LD(pl, rev_first ? n_prev - 1 - j : j, e0, e1, e2, pend); need = true; back = 1; break; }
				if (n_curr == 0) { CALL_DONE(); continue; }
				pl ^= 1; n_prev = n_curr; n_curr = 0; rev_first = 0; --i; j = 0;
				continue;
			}
			break;   /* MK_NONE */
		}
		if (__all_sync(FULL_MASK, st == MK_NONE)) break;
		if (!need) continue;

		const int cq = (int)q[i];                   /* forward: its complement (bwt.c:309); backward: the base itself */
		u64 o_s, o_o, o_x2;
		{
			u32 ct;
			int t12;
			extend_step3(ix, back ? e0 : e1, back ? e1 : e0, e2, back ? cq : 3 - cq, false, 0, back, t12, o_s, o_o, o_x2, ct);
			touches += (u64)t12;
		}
		if (st == MK_FWD) {                         /* bwt.c:307-316 */
			if (o_x2 != ik2) {
				PUSH(ik0, ik1, ik2, ikend);
				if (st != MK_FWD) continue;
				if (o_x2 < min_intv) { TURN_AROUND(); continue; }
			}
			ik0 = o_o; ik1 = o_s; ik2 = o_x2; ikend = i + 1;
			++i;
		} else {                                    /* bwt.c:331-343 */
			if (o_x2 < min_intv) {
				if (n_curr == 0 && (!m_any || i + 1 < last_start)) { PAINT(i + 1, pend); m_any = true; last_start = i + 1; }
			} else if (n_curr == 0 || o_x2 != curr_last_x2) {
				PUSH(o_s, o_o, o_x2, pend);
				curr_last_x2 = o_x2;
			}
			++j;
		}
	}
#undef MK_PTR
#undef MK_ST
#undef MK_LD
#undef PAINT
#undef PUSH
#undef TURN_AROUND
#undef CALL_DONE
	/* one atomic per warp per counter */
	for (int d = 16; d; d >>= 1) {
		touches += __shfl_xor_sync(FULL_MASK, touches, d);
		const u64 m = __shfl_xor_sync(FULL_MASK, max_ns, d); max_ns = m > max_ns ? m : max_ns;
		const u32 n = __shfl_xor_sync(FULL_MASK, need_max, d); need_max = n > need_max ? n : need_max;
	}
	overflow = __reduce_or_sync(FULL_MASK, overflow);
	if ((tid & 31) == 0) {
		if (touches) atomicAdd(&a.ctr->touches, touches);
		if (max_ns) atomicMax(&a.ctr->max_ns, max_ns);
		if (overflow) { atomicOr(&a.ctr->flags, 1u); atomicMax((int *)&a.ctr->need, (int)need_max); }
	}
}

/* M2: bins of the painted bytes, one atomic per bin per block */
__global__ void __launch_bounds__(MAXK_HIST_THREADS) k_maxk_hist(const uint8_t *cnt, i64 n, u64 *hist)
{
	__shared__ u32 h[256];
	for (int k = threadIdx.x; k < 256; k += blockDim.x) h[k] = 0;
	__syncthreads();
	const i64 n16 = n >> 4;
	for (i64 k = (i64)blockIdx.x * blockDim.x + threadIdx.x; k < n16; k += (i64)gridDim.x * blockDim.x) {
		const uint4 v = reinterpret_cast<const uint4 *>(cnt)[k];
		const u32 wv[4] = { v.x, v.y, v.z, v.w };
		for (int t = 0; t < 4; ++t)
			for (int s = 0; s < 32; s += 8) atomicAdd(&h[wv[t] >> s & 255u], 1u);
	}
	for (i64 k = (n16 << 4) + (i64)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (i64)gridDim.x * blockDim.x) atomicAdd(&h[cnt[k]], 1u);
	__syncthreads();
	for (int k = threadIdx.x; k < 256; k += blockDim.x) if (h[k]) atomicAdd(&hist[k], (u64)h[k]);
}

/* ------------------------------------------------------------------------------------------------ host driver */

/* a context over the Occ blocks of an updated .bwt alone: no suffix array, no text, no short-string table */
extern "C" bwag_ctx_t *bwag_ctx_create_occ(int device, const bwt_t *bwt)
{
	bwag_ctx_t *c = bwag_ctx_create_bare(device);
	if (!c) return 0;
	void *d = 0;
	const size_t occ_bytes = (((size_t)bwt->bwt_size * 4 + 64) + 255) & ~(size_t)255;   /* what occ_upload clears */
	if (cudaMalloc(&d, occ_bytes) != cudaSuccess) { cudaGetLastError(); set_err("cannot allocate %.2f GB of device memory for the Occ blocks", (double)bwt->bwt_size * 4 / 1e9); bwag_ctx_destroy(c); return 0; }
	c->blob = d; c->own_blob = 1;
	DevIndex &ix = c->lane.ix;
	if (occ_upload(d, bwt, ix.sb)) { bwag_ctx_destroy(c); return 0; }
	ix.bwt = (const uint4 *)d;
	ix.primary = bwt->primary; ix.seq_len = bwt->seq_len;
	for (int k = 0; k < 5; ++k) ix.L2[k] = bwt->L2[k];
	for (int s = 0; s < BWAG_MAX_SB; ++s)
		for (int k = 0; k < 4; ++k) { ix.sbgt[s][k] = 0; for (int t = k + 1; t < 4; ++t) ix.sbgt[s][k] += ix.sb[s][t]; }
	return c;
}

extern "C" int bwag_maxk(bwag_batch_t *b, int min_intv, int64_t window, uint64_t hist[256], bwag_maxk_stats_t *out)
{
	Lane *c = &b->lane;
	const bwag_ctx_t *pc = b->ctx;
	CK(cudaSetDevice(pc->device));
	const int n = b->n;
	memset(out, 0, sizeof(*out));
	if (window <= 0 || window > (int64_t)b->max_len) window = b->max_len > 0 ? b->max_len : 1;
	if (buf_reserve(&b->d_mk_woff, 8 * ((size_t)n + 1)) || hbuf_reserve(&b->h_mk_woff, 8 * ((size_t)n + 1)) ||
	    buf_reserve(&b->d_mk_cnt, (size_t)b->total_bases + 16) || buf_reserve(&b->d_mk_ctr, sizeof(MaxkCtr)) || hbuf_reserve(&b->h_mk_ctr, sizeof(MaxkCtr))) return 1;
	i64 *woff = (i64 *)b->h_mk_woff.p;
	woff[0] = 0;
	for (int r = 0; r < n; ++r) woff[r + 1] = woff[r] + (b->h_off[r + 1] - b->h_off[r] + window - 1) / window;
	const i64 n_win = woff[n];
	H2D(c, b->d_mk_woff.p, woff, 8 * ((size_t)n + 1));
	int grid = 2;
#ifndef BWAG_CUSIM
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&grid, k_maxk, MAXK_THREADS, 0));
	grid = pc->n_sm * (grid > 0 ? grid : 1);
#endif
	if ((i64)grid * MAXK_THREADS > n_win) grid = (int)((n_win + MAXK_THREADS - 1) / MAXK_THREADS);
	if (grid < 1) grid = 1;
	/* list capacity: a list never holds more entries than the query has bases (window + 2 margins) */
	const char *e = getenv("BWA_B200_TEST_SMALL_POOLS");
	const i64 most = window + 2 * MAXK_MARGIN + 1;
	int cap = e && atoi(e) > 0 ? MAXK_SLOTS + 1 : (int)(most < 256 ? most : 256);
	if (cap < MAXK_SLOTS) cap = MAXK_SLOTS;
	MaxkArgs ma;
	memset(&ma, 0, sizeof(ma));
	ma.codes = (const uint8_t *)b->d_codes.p; ma.off = (const i64 *)b->d_off.p; ma.n_seqs = n;
	ma.win_off = (const i64 *)b->d_mk_woff.p; ma.n_win = n_win; ma.window = window; ma.min_intv = min_intv < 1 ? 1 : min_intv;
	ma.cnt = (uint8_t *)b->d_mk_cnt.p; ma.ctr = (MaxkCtr *)b->d_mk_ctr.p;
	MaxkCtr *hc = (MaxkCtr *)b->h_mk_ctr.p;
	for (;;) {
		if (buf_reserve(&b->d_mk_scratch, (size_t)grid * MAXK_THREADS * 4 * (size_t)cap * 16)) return 1;
		ma.cap = cap; ma.scratch = (ulonglong2 *)b->d_mk_scratch.p;
		CK(cudaMemsetAsync(b->d_mk_cnt.p, 0, (size_t)b->total_bases + 16, c->stream));
		CK(cudaMemsetAsync(b->d_mk_ctr.p, 0, sizeof(MaxkCtr), c->stream));
		CK(cudaEventRecord(c->ev0, c->stream));
		if (n_win > 0) BWAG_LAUNCH(k_maxk, grid, MAXK_THREADS, 0, c->stream, c->ix, ma);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		D2H(c, hc, b->d_mk_ctr.p, sizeof(MaxkCtr));
		CK(stream_wait(c));
		const double ms = elapsed_at(c, "maxk", __FILE__, __LINE__);
		out->ms_kernel += ms; c->st.ms_smem += ms; ++c->st.n_launch;
		if (!(hc->flags & 1)) break;
		++out->n_repeat;                            /* a list outgrew cap: again with lists twice as long as the longest asked for */
		i64 want = 2 * (i64)(hc->need > (u32)cap ? hc->need : (u32)cap);
		if (want > most) want = most;
		if (want <= cap) return set_err("maxk: an interval list of %u entries does not fit %d", hc->need, cap);
		cap = (int)want;
	}
	out->max_window_ms = (double)hc->max_ns / 1e6;
	out->occ_touches = hc->touches; c->st.occ_touches += hc->touches;
	out->n_windows = n_win; out->window = window; out->list_cap = cap;
	/* M2 */
	{
		const i64 n16 = (b->total_bases >> 4) + 1;
		i64 hg = (n16 + MAXK_HIST_THREADS - 1) / MAXK_HIST_THREADS;
		if (hg > (i64)pc->n_sm * 8) hg = (i64)pc->n_sm * 8;
		CK(cudaEventRecord(c->ev0, c->stream));
		BWAG_LAUNCH(k_maxk_hist, (int)(hg < 1 ? 1 : hg), MAXK_HIST_THREADS, 0, c->stream, (const uint8_t *)b->d_mk_cnt.p, (i64)b->total_bases, ((MaxkCtr *)b->d_mk_ctr.p)->hist);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		D2H(c, hc, b->d_mk_ctr.p, sizeof(MaxkCtr));
		CK(stream_wait(c));
		out->ms_hist = elapsed_at(c, "maxk_hist", __FILE__, __LINE__);
		++c->st.n_launch;
	}
	for (int k = 0; k < 256; ++k) hist[k] += hc->hist[k];
	return 0;
}
