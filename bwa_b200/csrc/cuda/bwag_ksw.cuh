/* bwag_ksw.cuh -- the warp form of ksw_global2 (ksw.c:540-642) shared by K5 (bwag_global.cu) and samse's gapped refinement
 * (bwag_samse.cu): the banded row sweep with the direction bytes, and the backtrack that turns them into a CIGAR.
 * Both are force-inlined, so each kernel compiles them into its own body. */
#ifndef BWAG_KSW_CUH
#define BWAG_KSW_CUH
#include "bwag_dev.cuh"

#define NEG_INF (-0x40000000)

/* Banded global alignment score of q[0..qlen) vs t[0..tlen), band w; z != 0: record directions
 * (n_col bytes per row).  Restatement of ksw_global2 (ksw.c:552-611), lanes across columns. */
__device__ __forceinline__ int warp_ksw_global(int lane, int qlen, const uint8_t *q, int tlen, const uint8_t *t, const int8_t *mat,
                               int o_del, int e_del, int o_ins, int e_ins, int w, int *H, int *E, uint8_t *z, int n_col, u64 *cells)
{
	const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
	for (int j = lane; j <= qlen; j += 32) {
		H[j] = j == 0 ? 0 : (j <= w ? -(o_ins + e_ins * j) : NEG_INF);
		E[j] = NEG_INF;
	}
	__syncwarp();
	for (int i = 0; i < tlen; ++i) {
		const int8_t *srow = mat + t[i] * 5;
		const int beg = i > w ? i - w : 0, end = i + w + 1 < qlen ? i + w + 1 : qlen;
		int carry_h = beg == 0 ? -(o_del + e_del * (i + 1)) : NEG_INF;
		int carry_f = NEG_INF;
		uint8_t *zi = z ? z + (i64)i * n_col : 0;
		if (end > beg) *cells += (u64)(end - beg);
		for (int j0 = beg; j0 < end; j0 += 32) {
			const int j = j0 + lane;
			const bool act = j < end;
			int m = NEG_INF, e = NEG_INF, tt, s, f, h, hp;
			if (act) { m = H[j] + srow[q[j]]; e = E[j]; }
			tt = act ? m - oe_ins : -0x7f000000;       /* inactive lanes (only ever at the end of the last chunk) must not feed the scan */
			s = tt;
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				int v = __shfl_up_sync(FULL_MASK, s, d) - d * e_ins;
				if (lane >= d && v > s) s = v;
			}
			{
				int sl = __shfl_up_sync(FULL_MASK, s, 1);
				f = carry_f - lane * e_ins;
				if (lane > 0 && sl > f) f = sl;
			}
			uint8_t d;
			d = m >= e ? 0 : 1; h = m >= e ? m : e;
			d = h >= f ? d : 2; h = h >= f ? h : f;
			if (!act) h = NEG_INF;
			hp = __shfl_up_sync(FULL_MASK, h, 1);
			if (lane == 0) hp = carry_h;
			{
				int la = end - 1 - j0; la = la < 31 ? la : 31;
				int s31 = __shfl_sync(FULL_MASK, s, 31);
				int cf = carry_f - 32 * e_ins;
				carry_f = s31 > cf ? s31 : cf;
				carry_h = __shfl_sync(FULL_MASK, h, la);
			}
			if (act) {
				int te = m - oe_del;
				e -= e_del; d |= e > te ? 1 << 2 : 0; e = e > te ? e : te;
				d |= (f - e_ins) > tt ? 2 << 4 : 0;
				H[j] = hp; E[j] = e;
				if (zi) zi[j - beg] = d;
			}
		}
		if (lane == 0) { H[end] = carry_h; E[end] = NEG_INF; }
		__syncwarp();
	}
	return H[qlen];
}

/* The backtrack of ksw_global2 (ksw.c:613-627) over the direction bytes z (n_col per row) of a tlen x qlen sweep with band w:
 * the CIGAR (len << 4 | op) into cig, in order; returns its length.  One lane; the run being built stays in registers
 * (push_cigar merges equal ops). */
__device__ __forceinline__ int ksw_backtrack(const uint8_t *z, int n_col, int tlen, int qlen, int w, u32 *cig)
{
	int i = tlen - 1, k = (i + w + 1 < qlen ? i + w + 1 : qlen) - 1, which = 0, n = 0, run_op = -1, run_len = 0;
#define K5_PUSH(op_, len_) do { if ((op_) == run_op) run_len += (len_); else { if (run_op >= 0) cig[n++] = (u32)run_len << 4 | (u32)run_op; run_op = (op_); run_len = (len_); } } while (0)
	while (i >= 0 && k >= 0) {
		which = z[(i64)i * n_col + (k - (i > w ? i - w : 0))] >> (which << 1) & 3;
		if (which == 0) { K5_PUSH(0, 1); --i; --k; }
		else if (which == 1) { K5_PUSH(2, 1); --i; }
		else { K5_PUSH(1, 1); --k; }
	}
	if (i >= 0) K5_PUSH(2, i + 1);
	if (k >= 0) K5_PUSH(1, k + 1);
	if (run_op >= 0) cig[n++] = (u32)run_len << 4 | (u32)run_op;
#undef K5_PUSH
	for (int x = 0; x < n >> 1; ++x) { u32 tmp = cig[x]; cig[x] = cig[n - 1 - x]; cig[n - 1 - x] = tmp; }
	return n;
}

#endif
