/* bwag_extend.cu -- stage 2 kernel (K4): chains -> alignment regions.
 *
 * Replaces, per read, the loop over chains in mem_align1_core (bwamem.c:1096-1101), mem_chain2aln
 * (bwamem.c:658-812) and ksw_extend2 (ksw.c:416-515).
 *
 * Mapping to the machine.  Whether a seed is extended depends on the regions already produced by
 * earlier seeds and chains of the same read (bwamem.c:697-732), so one WARP owns a read and walks its
 * chains and seeds in the reference order; parallelism comes from the reads in flight (persistent
 * warps pulling read ids from an atomic counter) and, inside an extension, from the 32 lanes that
 * sweep a DP row together:
 *   - the DP is row-sequential because the band [beg,end) of row i+1 is trimmed from the finished
 *     row i (ksw.c:502-505); within a row, lanes own consecutive query columns;
 *   - H and E of a column depend on the previous row only through M (ksw.c:465-483), and F along the
 *     row is a max-plus prefix recurrence f[j+1] = max(f[j]-e_ins, t[j]) -> an inclusive warp scan
 *     with five shuffle steps per 32-column chunk and one carried value between chunks;
 *   - the row maximum / its right-most column, and the first / last non-zero cell for the band
 *     update, are warp reductions (REDUX);
 *   - cells are int32 here (exact for any read length); the H/E rows and the fetched reference window
 *     live in a per-warp scratch area that stays L1/L2 resident.
 * Integer-ALU bound; no tensor-core shape in this recurrence.
 */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"

#ifndef K4_MINB
#define K4_MINB 6   /* resident blocks per SM the lean kernels are compiled for (80 registers, as the first formulation) */
#endif
#define XSEED_DEAD 0x40000000u    /* set on a seed of the device copy when its extension was skipped (srt[k]=0, bwamem.c:727) */
#define XSEED_LEN(x) ((int)((x) & 0x3fffffffu))

__device__ __forceinline__ int imax2(int a, int b) { return a > b ? a : b; }
__device__ __forceinline__ int warp_max(int v) { return __reduce_max_sync(FULL_MASK, v); }
__device__ __forceinline__ int warp_min(int v) { return __reduce_min_sync(FULL_MASK, v); }

__device__ __forceinline__ int dev_cal_max_gap(const bwag_sw_par_t &p, int qlen) /* bwamem.c:647-654 */
{
	int l_del = bwag_trunc_i32((double)(qlen * p.a - p.o_del) / p.e_del + 1.);
	int l_ins = bwag_trunc_i32((double)(qlen * p.a - p.o_ins) / p.e_ins + 1.);
	int l = l_del > l_ins ? l_del : l_ins;
	l = l > 1 ? l : 1;
	return l < p.w << 1 ? l : p.w << 1;
}

/* Banded extension of query q[0..qlen) (q[j] = qp[j*qs]) against target t[0..tlen) (t[i] = tp[i*ts])
 * starting from score h0; exact restatement of ksw_extend2 (ksw.c:416-515) with lanes across columns.
 * H, E: per-warp int arrays of at least qlen+1 entries.  All lanes return the same values. */
__device__ __forceinline__ int warp_ksw_extend(int lane, int qlen, const uint8_t *qp, int qs, int tlen, const uint8_t *tp, int ts,
                               const int8_t *mat, int o_del, int e_del, int o_ins, int e_ins, int w, int end_bonus, int zdrop, int h0,
                               int *H, int *E, int *qle, int *tle, int *gtle, int *gscore_, int *max_off_, u64 *cells)
{
	const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
	int max, max_i, max_j, max_ie, gscore, max_off, beg, end;
	{   /* first row (ksw.c:431-433): H[0]=h0, then h0-oe_ins, decreasing by e_ins while positive; E = 0 */
		int H1 = h0 > oe_ins ? h0 - oe_ins : 0, maxsc = 0;
		for (int j = lane; j <= qlen; j += 32) {
			int v = j == 0 ? h0 : H1 - (j - 1) * e_ins;
			H[j] = v > 0 ? v : 0;
			E[j] = 0;
		}
		for (int k = 0; k < 25; ++k) maxsc = maxsc > mat[k] ? maxsc : mat[k];
		int max_ins = bwag_trunc_i32((double)(qlen * maxsc + end_bonus - o_ins) / e_ins + 1.); max_ins = max_ins > 1 ? max_ins : 1;
		w = w < max_ins ? w : max_ins;
		int max_del = bwag_trunc_i32((double)(qlen * maxsc + end_bonus - o_del) / e_del + 1.); max_del = max_del > 1 ? max_del : 1;
		w = w < max_del ? w : max_del;
	}
	__syncwarp();
	max = h0; max_i = max_j = -1; max_ie = -1; gscore = -1; max_off = 0;
	beg = 0; end = qlen;
	for (int i = 0; i < tlen; ++i) {
		const int8_t *srow = mat + tp[i * ts] * 5;
		int m = 0, mj = -1, nz_min = 0x7fffffff, nz_max = -1;   /* nz_*: warp-uniform, from ballots */
		if (beg < i - w) beg = i - w;
		if (end > i + w + 1) end = i + w + 1;
		if (end > qlen) end = qlen;
		int carry_h = 0;             /* H(i, j-1) entering the chunk; first column: ksw.c:456-459 */
		if (beg == 0) { carry_h = h0 - (o_del + e_del * (i + 1)); if (carry_h < 0) carry_h = 0; }
		int carry_f = 0;             /* F(i, j) entering the chunk */
		if (end > beg) *cells += (u64)(end - beg);
		for (int j0 = beg; j0 < end; j0 += 32) {
			const int j = j0 + lane;
			const bool act = j < end;
			int M = 0, e = 0, t, s, f, h, hp;
			if (act) {
				M = H[j]; e = E[j];
				M = M ? M + srow[qp[j * qs]] : 0;
			}
			t = M - oe_ins; t = t > 0 ? t : 0;        /* what this column offers to F of the columns on its right */
			if (!act) t = 0;
			s = t;                                     /* inclusive max-plus scan: s[l] = max_{k<=l} (t[k] - (l-k)*e_ins) */
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				int v = __shfl_up_sync(FULL_MASK, s, d) - d * e_ins;
				if (lane >= d && v > s) s = v;
			}
			{
				int sl = __shfl_up_sync(FULL_MASK, s, 1); /* s[l-1] */
				f = carry_f - lane * e_ins;
				if (lane > 0 && sl > f) f = sl;
				if (f < 0) f = 0;
			}
			h = M > e ? M : e; h = h > f ? h : f;
			if (!act) h = 0;
			hp = __shfl_up_sync(FULL_MASK, h, 1);
			if (lane == 0) hp = carry_h;
			{   /* carries: F entering column j0+32, and H of the last active column of this chunk */
				int la = end - 1 - j0; la = la < 31 ? la : 31;
				int s31 = __shfl_sync(FULL_MASK, s, 31);
				int cf = carry_f - 32 * e_ins;
				carry_f = s31 > cf ? s31 : cf; if (carry_f < 0) carry_f = 0;
				carry_h = __shfl_sync(FULL_MASK, h, la);
			}
			bool nz = false;
			if (act) {
				int te = M - oe_del; te = te > 0 ? te : 0;
				e -= e_del; e = e > te ? e : te;
				H[j] = hp; E[j] = e;
				if (h >= m) { m = h; mj = j; }         /* a lane's columns ascend, so ties keep the larger j (ksw.c:473-474) */
				nz = hp != 0 || e != 0;
			}
			{   /* first and last column whose stored cell is non-zero: chunks ascend, so the first ballot with a bit set holds the minimum */
				const u32 bal = __ballot_sync(FULL_MASK, nz);
				if (bal) { if (nz_min == 0x7fffffff) nz_min = j0 + __ffs(bal) - 1; nz_max = j0 + 31 - __clz(bal); }
			}
		}
		const int h1 = carry_h;                        /* H(i, end-1), or the first-column value if the row was empty */
		if (lane == 0) { H[end] = h1; E[end] = 0; }
		{
			int ma = warp_max(m);
			mj = warp_max(m == ma ? mj : -1);
			m = ma;
		}
		if ((end > beg ? end : beg) == qlen) {         /* ksw.c:486-489: ties go to the later row */
			max_ie = gscore > h1 ? max_ie : i;
			gscore = gscore > h1 ? gscore : h1;
		}
		if (m == 0) break;
		if (m > max) {
			int d = mj - i;
			max = m; max_i = i; max_j = mj;
			d = d < 0 ? -d : d;
			max_off = max_off > d ? max_off : d;
		} else if (zdrop > 0) {
			if (i - max_i > mj - max_j) { if (max - m - ((i - max_i) - (mj - max_j)) * e_del > zdrop) break; }
			else { if (max - m - ((mj - max_j) - (i - max_i)) * e_ins > zdrop) break; }
		}
		{   /* next band: first non-zero cell .. last non-zero cell + 2 (ksw.c:501-505; index `end` included) */
			int nb = nz_min == 0x7fffffff ? end : nz_min;
			int jl = nz_max;
			if (h1 != 0) jl = end;
			if (jl < 0) jl = nb - 1;
			beg = nb;
			end = jl + 2 < qlen ? jl + 2 : qlen;
		}
		__syncwarp();
	}
	__syncwarp();
	*qle = max_j + 1; *tle = max_i + 1; *gtle = max_ie + 1; *gscore_ = gscore; *max_off_ = max_off;
	return max;
}

/* The same extension for sane gap penalties (e_ins >= 0, o_ins + e_ins >= 0 -- every real scoring scheme), about half
 * the instructions per 32-column chunk:
 *   - H and E of a column sit side by side (one 64-bit load and store per cell);
 *   - no divergent code in the chunk: idle lanes of the last chunk load a clamped column and are masked by selects;
 *   - the F scan runs in slanted coordinates (value + column*e_ins), which makes it a plain max scan: one SHFL + one
 *     max per step, no decay constants, and no lane guards (a lane below the shuffle distance gets its own value back);
 *   - the F value entering the chunk is folded into lane 0's offer before the scan (max(t0, carry - e_ins)), so the
 *     scan result IS F of the next column and F of the next chunk's first column is its lane-31 value;
 *   - first / last non-zero stored cell are tracked per lane and reduced once per row;
 *   - CUT: the sweep stops at the first row after which no output can change (see the comment at the cut-off); the
 *     reference would go on to tlen = qlen + max_gap rows, i.e. about twice as many for a read that matches to its end.
 *     Needs non-negative deletion penalties as well.  `cells` then counts the cells actually computed.
 * q[j] = byte at qa + j*QS, t[i] = byte at ta + i*TS, H/E pair of column j at he + 8*j, mat[k] at ma + k.
 * Results are identical to warp_ksw_extend (and ksw_extend2) under the stated condition. */
template <class A, class AM, int QS, int TS, bool CUT>
__device__ __forceinline__ int warp_ksw_extend_fast(int lane, int qlen, typename A::addr qa, int tlen, typename A::addr ta,
                               typename AM::addr ma, int o_del, int e_del, int o_ins, int e_ins, int w, int end_bonus, int zdrop, int h0,
                               typename A::addr he, int *qle, int *tle, int *gtle, int *gscore_, int *max_off_, u64 *cells)
{
	const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
	int max, max_i, max_j, max_ie, gscore, max_off, beg, end, maxsc = 0;
	{   /* first row (ksw.c:431-433) */
		int H1 = h0 > oe_ins ? h0 - oe_ins : 0;
		for (int j = lane; j <= qlen; j += 32) {
			int v = j == 0 ? h0 : H1 - (j - 1) * e_ins;
			A::st_he(he + 8 * j, v > 0 ? v : 0, 0);
		}
		for (int k = 0; k < 25; ++k) { int v = AM::ld_s8(ma + k); maxsc = maxsc > v ? maxsc : v; }
		int max_ins = bwag_trunc_i32((double)(qlen * maxsc + end_bonus - o_ins) / e_ins + 1.); max_ins = max_ins > 1 ? max_ins : 1;
		w = w < max_ins ? w : max_ins;
		int max_del = bwag_trunc_i32((double)(qlen * maxsc + end_bonus - o_del) / e_del + 1.); max_del = max_del > 1 ? max_del : 1;
		w = w < max_del ? w : max_del;
	}
	__syncwarp();
	max = h0; max_i = max_j = -1; max_ie = -1; gscore = -1; max_off = 0;
	beg = 0; end = qlen;
	const int ne1 = -e_ins, noe_ins = -oe_ins, noe_del = -oe_del, ne_del = -e_del;
	const bool lane0 = lane == 0;
	const int le = lane * e_ins;
	const int pot0 = maxsc * (qlen - 1);            /* potential of a cell: its score + maxsc * (columns to its right) */
	for (int i = 0; i < tlen; ++i) {
		const typename AM::addr srow = ma + A::ld_u8(ta + i * TS) * 5;
		int m = 0, mj = -1, jmin = 0x7fffffff, jmax = -1, phi = 0;   /* per lane; reduced after the row */
		if (beg < i - w) beg = i - w;
		if (end > i + w + 1) end = i + w + 1;
		if (end > qlen) end = qlen;
		int carry_h = 0;             /* H(i, j-1) entering the chunk; first column: ksw.c:456-459 */
		if (beg == 0) { carry_h = h0 - (o_del + e_del * (i + 1)); if (carry_h < 0) carry_h = 0; }
		int carry_f = 0;             /* F(i, j0) entering the chunk */
		if (end > beg) *cells += (u64)(end - beg);
		for (int j0 = beg; j0 < end; j0 += 32) {
			const int j = j0 + lane;
			const bool act = j < end;
			const int jc = act ? j : end - 1;                  /* idle lanes re-read the last column; their results are masked */
			const int2 c = A::ld_he(he + 8 * jc);
			const int sc = AM::ld_s8(srow + A::ld_u8(qa + jc * QS));
			const int M = (act && c.x != 0) ? c.x + sc : 0;
			int t = __viaddmax_s32(M, noe_ins, 0);             /* what this column offers to F on its right; 0 for idle lanes */
			if (lane0) t = __viaddmax_s32(carry_f, ne1, t);
			/* inclusive max-plus scan in slanted coordinates: s[l] = max_{k<=l} (t[k] + k*e_ins) = F(i, j0+l+1) + l*e_ins, so
			 * the steps need no decay constants (and no lane guards: a lane below the distance gets its own value back) */
			int s = t + le;
			s = imax2(s, __shfl_up_sync(FULL_MASK, s, 1));
			s = imax2(s, __shfl_up_sync(FULL_MASK, s, 2));
			s = imax2(s, __shfl_up_sync(FULL_MASK, s, 4));
			s = imax2(s, __shfl_up_sync(FULL_MASK, s, 8));
			s = imax2(s, __shfl_up_sync(FULL_MASK, s, 16));
			int f = __shfl_up_sync(FULL_MASK, s, 1) - le + e_ins;
			if (lane0) f = carry_f;
			carry_f = __shfl_sync(FULL_MASK, s, 31) - 31 * e_ins;
			int h = __vimax3_s32(M, c.y, f);
			if (!act) h = 0;
			int hp = __shfl_up_sync(FULL_MASK, h, 1);
			if (lane0) hp = carry_h;
			{
				int la = end - 1 - j0; la = la < 31 ? la : 31;
				carry_h = __shfl_sync(FULL_MASK, h, la);           /* H of the chunk's last active column */
			}
			const int e = __vimax3_s32(c.y + ne_del, M + noe_del, 0);
			if (act) A::st_he(he + 8 * j, hp, e);
			if (act && h >= m) mj = j;                         /* a lane's columns ascend, so ties keep the larger j (ksw.c:473-474) */
			m = m > h ? m : h;
			phi = __viaddmax_s32(h, pot0 - maxsc * j, phi);
			if (act && (hp | e) != 0) { jmax = j; jmin = jmin < j ? jmin : j; }
		}
		const int h1 = carry_h;                        /* H(i, end-1), or the first-column value if the row was empty */
		if (lane0) A::st_he(he + 8 * end, h1, 0);
		{
			int ma_ = warp_max(m);
			mj = warp_max(m == ma_ ? mj : -1);
			m = ma_;
		}
		if ((end > beg ? end : beg) == qlen) {         /* ksw.c:486-489: ties go to the later row */
			max_ie = gscore > h1 ? max_ie : i;
			gscore = gscore > h1 ? gscore : h1;
		}
		if (m == 0) break;
		const bool falling = m <= max, to_end = end == qlen && end > beg;
		if (m > max) {
			int d = mj - i;
			max = m; max_i = i; max_j = mj;
			d = d < 0 ? -d : d;
			max_off = max_off > d ? max_off : d;
		} else if (zdrop > 0) {
			if (i - max_i > mj - max_j) { if (max - m - ((i - max_i) - (mj - max_j)) * e_del > zdrop) break; }
			else { if (max - m - ((mj - max_j) - (i - max_i)) * e_ins > zdrop) break; }
		}
		{   /* next band: first non-zero cell .. last non-zero cell + 2 (ksw.c:501-505; index `end` included) */
			const int nz_min = warp_min(jmin), nz_max = warp_max(jmax);
			int nb = nz_min == 0x7fffffff ? end : nz_min;
			int jl = nz_max;
			if (h1 != 0) jl = end;
			if (jl < 0) jl = nb - 1;
			beg = nb;
			end = jl + 2 < qlen ? jl + 2 : qlen;
		}
		if (CUT && falling && to_end) {
			/* Row cut-off.  ksw_extend2 keeps sweeping rows until tlen, Z-drop or an all-zero row, but once no cell can
			 * reach the best score again the outputs are final.  A cell's potential = score + maxsc * (columns to its
			 * right) bounds every score reachable from it (a diagonal step gains at most maxsc and uses up a column; E and
			 * F only lose: penalties are non-negative here; zero cells do not propagate, ksw.c:465).  This row covered
			 * every column from beg to the query's end, so all stored cells the later rows can read (fresh or stale) stem
			 * from it: every future score is <= max(phi over the row, the first-column entry below).  No future row maximum
			 * can exceed `max` (strictly needed: ksw.c:490) and no future H(i, qlen-1) can reach `gscore` (ties go to the
			 * later row, ksw.c:486-489), so max, max_i/j, max_off, gscore and max_ie cannot change any more. */
			int bound = warp_max(phi);
			if (beg == 0) { const int fc = h0 - (o_del + e_del * (i + 1)) + maxsc * qlen; bound = bound > fc ? bound : fc; }
			if (bound <= max && bound < gscore) break;
		}
		__syncwarp();
	}
	__syncwarp();
	*qle = max_j + 1; *tle = max_i + 1; *gtle = max_ie + 1; *gscore_ = gscore; *max_off_ = max_off;
	return max;
}

/* SM: the per-warp scratch (H/E rows, reference window, a copy of the read) lives in shared memory -- 32-bit
 * addressing and no L1 round trips in the row loop; chosen by the host whenever it fits (short reads) */
template <bool C, class X, class Y> struct SelT { typedef X type; };
template <class X, class Y> struct SelT<false, X, Y> { typedef Y type; };

template <bool SM, bool SANE>
__device__ __forceinline__ void extend_body(const DevIndex &ix, const ExtArgs &a)
{
	const int lane = threadIdx.x & 31;
	const i64 wid = ((i64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	int *H, *E;
	uint8_t *rseq, *qcopy = 0;
	if (SM) {
#ifdef BWAG_CUSIM
		unsigned char *dyn = cusim_dyn_smem;
#else
		extern __shared__ int4 k4_dyn[];
		unsigned char *dyn = reinterpret_cast<unsigned char *>(k4_dyn);
#endif
		unsigned char *mine = dyn + (size_t)(threadIdx.x >> 5) * a.smem_per_warp;
		H = reinterpret_cast<int *>(mine); E = H + a.cap_q + 2;
		rseq = reinterpret_cast<uint8_t *>(E + a.cap_q + 2);
		qcopy = rseq + a.cap_r;
	} else {
		H = a.eh + wid * (i64)(2 * (a.cap_q + 2)); E = H + a.cap_q + 2;
		rseq = a.rseq + wid * (i64)a.cap_r;
	}
	typedef typename SelT<SM, SmemAcc, PtrAcc>::type A;   /* how the lean sweep reaches the scratch; the matrix is always shared */
	typename A::addr he_a = A::make(H), rs_a = A::make(rseq), q_a = A::make(qcopy);
	if constexpr (SM && SANE) { BWAG_KEEP(he_a); BWAG_KEEP(rs_a); BWAG_KEEP(q_a); }
	const bwag_sw_par_t &p = a.par;
	__shared__ int8_t s_mat[32];
	if (threadIdx.x < 25) s_mat[threadIdx.x] = p.mat[threadIdx.x];
	__syncthreads();
	typename SmemAcc::addr mat_a = SmemAcc::make(s_mat);
	if constexpr (SANE) BWAG_KEEP(mat_a);
	u64 cells = 0;
	int overflow = 0;

	for (;;) {
		int rid = 0;
		if (lane == 0) rid = atomicAdd(a.next_read, 1);
		rid = __shfl_sync(FULL_MASK, rid, 0);
		if (rid >= a.n_reads) break;
		{ const int cc = a.chain_cnt[rid]; if (cc < a.chain_lo || cc > a.chain_hi) continue; }   /* another launch's read */
		const i64 c0 = a.chain_beg[rid], c1 = c0 + a.chain_cnt[rid];
		int n_regs = 0;
		if (c1 > c0) {
			const uint8_t *query = a.codes + a.off[rid];
			const int l_query = (int)(a.off[rid + 1] - a.off[rid]);
			bwag_xreg_t *regs = a.regs + a.reg_base[rid];
			if (l_query > a.cap_q) { overflow = 1; if (lane == 0) a.n_regs[rid] = 0; continue; }
			if (SM) {
				__syncwarp();
				if (SANE) { for (int x = lane; x < l_query; x += 32) A::st_u8(q_a + x, query[x]); }
				else { for (int x = lane; x < l_query; x += 32) qcopy[x] = query[x]; }
				__syncwarp();
				query = qcopy;
			} else if (SANE) q_a = A::make(query);
			for (i64 c = c0; c < c1; ++c) {
				const bwag_xchain_t ch = a.chains[c];
				bwag_xseed_t *seeds = const_cast<bwag_xseed_t *>(a.seeds) + ch.seed_off;
				const i64 rmax0 = ch.rmax0, rmax1 = ch.rmax1;
				const int rlen = (int)(rmax1 - rmax0);
				if (rlen > a.cap_r) { overflow = 1; continue; }
				__syncwarp();
				if (SANE) { for (int x = lane; x < rlen; x += 32) A::st_u8(rs_a + x, bwag_ref_base(ix, rmax0 + x)); }   /* bns_fetch_seq (bwamem.c:685) */
				else { for (int x = lane; x < rlen; x += 32) rseq[x] = (uint8_t)bwag_ref_base(ix, rmax0 + x); }
				__syncwarp();
				for (int k = ch.n_seeds - 1; k >= 0; --k) {
					const i64 s_rbeg = seeds[k].rbeg;
					const int s_qbeg = seeds[k].qbeg, s_len = XSEED_LEN(seeds[k].len);
					/* containment test against every region of this read so far (bwamem.c:697-713) */
					int hit = 0x7fffffff;
					for (int r = lane; r < n_regs; r += 32) {
						const bwag_xreg_t q = regs[r];
						if (s_rbeg < q.rb || s_rbeg + s_len > q.re || s_qbeg < q.qb || s_qbeg + s_len > q.qe) continue;
						if (s_len - q.seedlen0 > .1 * l_query) continue;
						int qd = s_qbeg - q.qb; i64 rd = s_rbeg - q.rb;
						int mg = dev_cal_max_gap(p, qd < rd ? qd : (int)rd);
						int w = mg < q.w ? mg : q.w;
						bool around = qd - rd < w && rd - qd < w;
						if (!around) {
							qd = q.qe - (s_qbeg + s_len); rd = q.re - (s_rbeg + s_len);
							mg = dev_cal_max_gap(p, qd < rd ? qd : (int)rd);
							w = mg < q.w ? mg : q.w;
							around = qd - rd < w && rd - qd < w;
						}
						if (around) { hit = r; break; }
					}
					hit = warp_min(hit);
					if (hit != 0x7fffffff) { /* contained: extend only if an overlapping extended seed sits on another diagonal (bwamem.c:718-729) */
						int other = 0;
						for (int t = k + 1 + lane; t < ch.n_seeds; t += 32) {
							const u32 tl_ = seeds[t].len;
							if (tl_ & (XSEED_DEAD | BWAG_XSEED_ZEROKEY)) continue;
							const int t_len = XSEED_LEN(tl_), t_qbeg = seeds[t].qbeg;
							const i64 t_rbeg = seeds[t].rbeg;
							if (t_len < s_len * .95) continue;
							if (s_qbeg <= t_qbeg && s_qbeg + s_len - t_qbeg >= s_len >> 2 && t_qbeg - s_qbeg != t_rbeg - s_rbeg) { other = 1; break; }
							if (t_qbeg <= s_qbeg && t_qbeg + t_len - s_qbeg >= s_len >> 2 && s_qbeg - t_qbeg != s_rbeg - t_rbeg) { other = 1; break; }
						}
						if (!__any_sync(FULL_MASK, other)) {
							if (lane == 0) seeds[k].len |= XSEED_DEAD;
							__syncwarp();
							continue;
						}
					}
					/* extend (bwamem.c:734-797) */
					bwag_xreg_t reg;
					int aw0 = p.w, aw1 = p.w;
					reg.score = reg.truesc = -1; reg.chain = (int)(c - c0); reg.seedlen0 = s_len; reg.seedcov = 0; reg.w = 0;
					if (s_qbeg) {   /* to the left: reversed query prefix against the reversed reference prefix */
						int qle, tle, gtle, gscore, moff;
						const int tl = (int)(s_rbeg - rmax0);
						for (int it = 0; it < 2; ++it) {
							int prev = reg.score;
							aw0 = p.w << it;
							if (SANE) reg.score = warp_ksw_extend_fast<A, SmemAcc, -1, -1, true>(lane, s_qbeg, q_a + (s_qbeg - 1), tl, rs_a + (tl - 1), mat_a, p.o_del, p.e_del, p.o_ins, p.e_ins,
							                            aw0, p.pen_clip5, p.zdrop, s_len * p.a, he_a, &qle, &tle, &gtle, &gscore, &moff, &cells);
							else reg.score = warp_ksw_extend(lane, s_qbeg, query + s_qbeg - 1, -1, tl, rseq + tl - 1, -1, s_mat, p.o_del, p.e_del, p.o_ins, p.e_ins,
							                            aw0, p.pen_clip5, p.zdrop, s_len * p.a, H, E, &qle, &tle, &gtle, &gscore, &moff, &cells);
							if (reg.score == prev || moff < (aw0 >> 1) + (aw0 >> 2)) break;
						}
						if (gscore <= 0 || gscore <= reg.score - p.pen_clip5) { reg.qb = s_qbeg - qle; reg.rb = s_rbeg - tle; reg.truesc = reg.score; }
						else { reg.qb = 0; reg.rb = s_rbeg - gtle; reg.truesc = gscore; }
					} else { reg.score = reg.truesc = s_len * p.a; reg.qb = 0; reg.rb = s_rbeg; }
					if (s_qbeg + s_len != l_query) {   /* to the right */
						int qle, tle, gtle, gscore, moff;
						const int sc0 = reg.score, qe = s_qbeg + s_len;
						const i64 re = s_rbeg + s_len - rmax0;
						for (int it = 0; it < 2; ++it) {
							int prev = reg.score;
							aw1 = p.w << it;
							if (SANE) reg.score = warp_ksw_extend_fast<A, SmemAcc, 1, 1, true>(lane, l_query - qe, q_a + qe, (int)(rmax1 - rmax0 - re), rs_a + (int)re, mat_a, p.o_del, p.e_del, p.o_ins, p.e_ins,
							                            aw1, p.pen_clip3, p.zdrop, sc0, he_a, &qle, &tle, &gtle, &gscore, &moff, &cells);
							else reg.score = warp_ksw_extend(lane, l_query - qe, query + qe, 1, (int)(rmax1 - rmax0 - re), rseq + re, 1, s_mat, p.o_del, p.e_del, p.o_ins, p.e_ins,
							                            aw1, p.pen_clip3, p.zdrop, sc0, H, E, &qle, &tle, &gtle, &gscore, &moff, &cells);
							if (reg.score == prev || moff < (aw1 >> 1) + (aw1 >> 2)) break;
						}
						if (gscore <= 0 || gscore <= reg.score - p.pen_clip3) { reg.qe = qe + qle; reg.re = rmax0 + re + tle; reg.truesc += reg.score - sc0; }
						else { reg.qe = l_query; reg.re = rmax0 + re + gtle; reg.truesc += gscore - sc0; }
					} else { reg.qe = l_query; reg.re = s_rbeg + s_len; }
					{   /* bases of this chain's seeds that lie inside the region (bwamem.c:800-805) */
						int cov = 0;
						for (int t = lane; t < ch.n_seeds; t += 32) {
							const int t_len = XSEED_LEN(seeds[t].len), t_qbeg = seeds[t].qbeg;
							const i64 t_rbeg = seeds[t].rbeg;
							if (t_qbeg >= reg.qb && t_qbeg + t_len <= reg.qe && t_rbeg >= reg.rb && t_rbeg + t_len <= reg.re) cov += t_len;
						}
						reg.seedcov = __reduce_add_sync(FULL_MASK, cov);
					}
					reg.w = aw0 > aw1 ? aw0 : aw1;
					if (lane == 0) regs[n_regs] = reg;
					++n_regs;
					__syncwarp();
				}
			}
		}
		if (lane == 0) a.n_regs[rid] = n_regs;
	}
	if (lane == 0 && cells) atomicAdd(a.cells, cells);
	if (overflow && lane == 0) atomicOr(a.flags, 2u);
}

/* k_extend*: any penalties (the first formulation); k_extend*_fast: e_ins >= 0 and o_ins + e_ins >= 0, chosen by the host */
__global__ void __launch_bounds__(K4_THREADS) k_extend(DevIndex ix, ExtArgs a) { extend_body<false, false>(ix, a); }
__global__ void __launch_bounds__(K4_THREADS) k_extend_sm(DevIndex ix, ExtArgs a) { extend_body<true, false>(ix, a); }
__global__ void __launch_bounds__(K4_THREADS, K4_MINB) k_extend_fast(DevIndex ix, ExtArgs a) { extend_body<false, true>(ix, a); }
__global__ void __launch_bounds__(K4_THREADS, K4_MINB) k_extend_sm_fast(DevIndex ix, ExtArgs a) { extend_body<true, true>(ix, a); }
