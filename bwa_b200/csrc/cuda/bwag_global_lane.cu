/* bwag_global_lane.cu -- K5L: the banded global alignments of short-read CIGAR requests, one LANE per request.
 *
 * The warp-per-request kernel (bwag_global.cu) sweeps a DP row with 32 lanes; the requests of 150-bp reads have bands of 7..41
 * cells, so a row keeps one or two chunks of lanes busy for ~60 instructions each plus ~30 of per-row bookkeeping, and the serial
 * backtrack runs on one lane.
 * Here a lane runs ksw_global2's own scalar loop (ksw.c:552-611) and its backtrack (ksw.c:613-627) for one request; a warp works
 * on 32 requests in lock step, every loop bounded by the warp's maximum and predicated per lane.
 *   H/E of the band: a ring of K5L_RING (h, e) pairs per lane in shared memory, slot = column & (K5L_RING-1) -- row i touches
 *     columns [i-w, i+w+1], so 2w+2 <= K5L_RING suffices; layout [slot][thread], conflict-free;
 *   query codes: 4 per 32-bit shared word, [word][thread];
 *   direction bytes: per-lane slice of a global scratch, byte-interleaved by lane ([cell][lane]): lanes in step write one sector;
 *   the reference base of a row comes straight from the packed reference (one byte load per row).
 * Requests it does not take (no DP needed, band too wide for the ring, read longer than the query words, CIGAR longer than the
 * slot) are left to the warp kernel, which also turns every CIGAR -- made here or there -- into NM and MD.  The band-doubling
 * loop of mem_reg2aln (bwamem.c:1143-1152) runs here around the DP exactly as there.
 */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"

#define NEG_INF (-0x40000000)

__global__ void __launch_bounds__(K5L_THREADS, 2) k_global_lane(DevIndex ix, GlbLaneArgs a)
{
#ifdef BWAG_CUSIM
	unsigned char *dyn = cusim_dyn_smem;
#else
	extern __shared__ int4 k5l_dyn[];
	unsigned char *dyn = reinterpret_cast<unsigned char *>(k5l_dyn);
#endif
	int2 *ring = reinterpret_cast<int2 *>(dyn) + threadIdx.x;                                  /* slot s at ring[s * K5L_THREADS] */
	u32 *qw = reinterpret_cast<u32 *>(dyn + (size_t)K5L_RING * K5L_THREADS * 8) + threadIdx.x;   /* word k at qw[k * K5L_THREADS] */
	__shared__ int8_t s_mat[32];
	const bwag_sw_par_t &p = a.par;
	if (threadIdx.x < 25) s_mat[threadIdx.x] = p.mat[threadIdx.x];
	__syncthreads();
	const int lane = threadIdx.x & 31;
	const i64 wid = ((i64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	uint8_t *z = a.z + wid * a.cap_z * 32 + lane;     /* cell c of this lane at z[c * 32] */
	const int oe_del = p.o_del + p.e_del, oe_ins = p.o_ins + p.e_ins;
	u64 cells = 0;
	u32 n_pre = 0;

	for (;;) {
		int base = 0;
		if (lane == 0) base = atomicAdd(a.next_task, 32);
		base = __shfl_sync(FULL_MASK, base, 0);
		if (base >= a.n_tasks) break;
		const int tix = base + lane;
		bool live = tix < a.n_tasks;
		bwag_gtask_t tk;
		tk.rb = tk.re = 0; tk.read = 0; tk.qb = tk.qe = 0; tk.w = 0; tk.truesc = 0; tk.mode = BWAG_G_SCORE;
		if (live) tk = a.tasks[tix];
		const int lq = tk.qe - tk.qb, rlen = (int)(tk.re - tk.rb);
		const bool rev = tk.rb >= ix.l_pac;
		/* what this kernel takes: a CIGAR request over a valid window, short enough for the query words and the scratch */
		live = live && tk.mode == BWAG_G_REG2ALN && lq > 0 && rlen > 0 && !(tk.rb < ix.l_pac && tk.re > ix.l_pac) && tk.rb >= 0 && tk.re <= ix.l_pac << 1
		       && lq <= K5L_QWORDS * 4 && !(lq == rlen && (tk.w < p.w << 2 ? tk.w : p.w << 2) == 0);
		if (tix < a.n_tasks) a.pre_n[tix] = -1;
		if (!__any_sync(FULL_MASK, live)) continue;
		/* the query, in alignment order (reversed for reverse-strand hits: bwa.c:162-167), 4 codes per word */
		{
			const uint8_t *query = a.codes + a.off[tk.read] + tk.qb;
			const int nw = __reduce_max_sync(FULL_MASK, live ? (lq + 3) >> 2 : 0);
			for (int k = 0; k < nw; ++k) {
				u32 v = 0;
				if (live && k * 4 < lq) {
#pragma unroll
					for (int b = 0; b < 4; ++b) { const int x = k * 4 + b; if (x < lq) v |= (u32)query[rev ? lq - 1 - x : x] << (8 * b); }
				}
				qw[k * K5L_THREADS] = v;
			}
		}
		int w2 = tk.w, it = 0, last_sc = -(1 << 30), score = 0, n_cig = 0;
		u32 *cig = a.pre_cig + (i64)(live ? tix : 0) * K5L_MAXCIG;
		for (int round = 0; round < 3; ++round) {        /* the band-doubling loop; at most three alignments (bwamem.c:1150) */
			if (!__any_sync(FULL_MASK, live)) break;
			int w = 0, n_col = 0;
			if (live) {
				w2 = w2 < p.w << 2 ? w2 : p.w << 2;
				int max_gap, max_ins, max_del, min_w, d = rlen - lq;
				d = d < 0 ? -d : d;
				max_ins = bwag_trunc_i32((double)(((lq + 1) >> 1) * s_mat[0] - p.o_ins) / p.e_ins + 1.);
				max_del = bwag_trunc_i32((double)(((lq + 1) >> 1) * s_mat[0] - p.o_del) / p.e_del + 1.);
				max_gap = max_ins > max_del ? max_ins : max_del;
				max_gap = max_gap > 1 ? max_gap : 1;
				w = (max_gap + d + 1) >> 1;
				w = w < w2 ? w : w2;
				min_w = d + 3;
				w = w > min_w ? w : min_w;
				n_col = lq < 2 * w + 1 ? lq : 2 * w + 1;
				if (2 * w + 2 > K5L_RING || (i64)n_col * rlen > a.cap_z) live = false;   /* band or matrix too large: the warp kernel's */
			}
			/* ---- the DP (ksw.c:568-610) ---- */
			{
				const int n_init = __reduce_max_sync(FULL_MASK, live ? (lq < K5L_RING - 1 ? lq : K5L_RING - 1) : -1);
				for (int j = 0; j <= n_init; ++j)
					if (live && j <= lq && j < K5L_RING) ring[j * K5L_THREADS] = make_int2(j == 0 ? 0 : (j <= w ? -(p.o_ins + p.e_ins * j) : NEG_INF), NEG_INF);
			}
			const int rows = __reduce_max_sync(FULL_MASK, live ? rlen : 0);
			for (int i = 0; i < rows; ++i) {
				const bool on = live && i < rlen;
				int beg = 0, end = 0, h1 = NEG_INF, f = NEG_INF;
				const int8_t *srow = s_mat;
				if (on) {
					beg = i > w ? i - w : 0; end = i + w + 1 < lq ? i + w + 1 : lq;
					h1 = beg == 0 ? -(p.o_del + p.e_del * (i + 1)) : NEG_INF;
					srow = s_mat + bwag_ref_base(ix, rev ? tk.rb + (rlen - 1 - i) : tk.rb + i) * 5;
					cells += (u64)(end - beg);
				}
				uint8_t *zi = z + ((i64)i * n_col - beg) * 32;
				const int width = __reduce_max_sync(FULL_MASK, end - beg);
				for (int c = 0; c < width; ++c) {
					const int j = beg + c;
					if (on && j < end) {
						int2 *pe = ring + (j & (K5L_RING - 1)) * K5L_THREADS;
						const int2 he = *pe;
						int m = he.x, e = he.y, h, t;
						uint8_t d;
						m += srow[(qw[(j >> 2) * K5L_THREADS] >> (8 * (j & 3))) & 0xff];
						d = m >= e ? 0 : 1; h = m >= e ? m : e;
						d = h >= f ? d : 2; h = h >= f ? h : f;
						t = m - oe_del;
						e -= p.e_del;
						d |= e > t ? 1 << 2 : 0;
						e = e > t ? e : t;
						*pe = make_int2(h1, e);
						h1 = h;
						t = m - oe_ins;
						f -= p.e_ins;
						d |= f > t ? 2 << 4 : 0;
						f = f > t ? f : t;
						zi[(i64)j * 32] = d;
					}
				}
				if (on) ring[(end & (K5L_RING - 1)) * K5L_THREADS] = make_int2(h1, NEG_INF);
			}
			if (live) score = ring[(lq & (K5L_RING - 1)) * K5L_THREADS].x;
			/* ---- backtrack (ksw.c:613-627); the run being built stays in registers, equal neighbours merge ---- */
			{
				int i = rlen - 1, k = (i + w + 1 < lq ? i + w + 1 : lq) - 1, which = 0, n = 0, run_op = -1, run_len = 0;
				bool fits = true;
#define K5L_PUSH(op_, len_) do { if ((op_) == run_op) run_len += (len_); else { if (run_op >= 0) { if (n < K5L_MAXCIG) cig[n] = (u32)run_len << 4 | (u32)run_op; else fits = false; ++n; } run_op = (op_); run_len = (len_); } } while (0)
				while (__any_sync(FULL_MASK, live && i >= 0 && k >= 0)) {
					if (live && i >= 0 && k >= 0) {
						which = z[((i64)i * n_col + (k - (i > w ? i - w : 0))) * 32] >> (which << 1) & 3;
						if (which == 0) { K5L_PUSH(0, 1); --i; --k; }
						else if (which == 1) { K5L_PUSH(2, 1); --i; }
						else { K5L_PUSH(1, 1); --k; }
					}
				}
				if (live) {
					if (i >= 0) K5L_PUSH(2, i + 1);
					if (k >= 0) K5L_PUSH(1, k + 1);
					if (run_op >= 0) { if (n < K5L_MAXCIG) cig[n] = (u32)run_len << 4 | (u32)run_op; else fits = false; ++n; }
					if (!fits) live = false;           /* longer than the slot: the warp kernel redoes this request */
					else {
						for (int x = 0; x < n >> 1; ++x) { const u32 tmp = cig[x]; cig[x] = cig[n - 1 - x]; cig[n - 1 - x] = tmp; }
						n_cig = n;
					}
				}
#undef K5L_PUSH
			}
			/* ---- another round with twice the band? (bwamem.c:1150-1152) ---- */
			if (live) {
				bool more = !(score == last_sc || w2 == p.w << 2);
				if (more) { last_sc = score; w2 <<= 1; more = ++it < 3 && score < tk.truesc - p.a; }
				if (!more) {                        /* done: publish and retire the lane */
					a.pre_n[tix] = n_cig; a.pre_score[tix] = score; ++n_pre;
					live = false;
				}
			}
		}
	}
	if (cells) atomicAdd(a.cells, cells);
	if (n_pre) atomicAdd(a.n_pre, n_pre);
}
