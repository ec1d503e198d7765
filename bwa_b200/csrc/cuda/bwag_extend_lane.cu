/* bwag_extend_lane.cu -- stage 2 kernel for short reads (K4L): chains -> alignment regions, ONE LANE PER READ.
 *
 * Same contract as bwag_extend.cu (mem_chain2aln bwamem.c:658-812 with ksw_extend2 ksw.c:416-515 inside, per read, in
 * the reference's chain and seed order), different mapping.  The row sweep of bwag_extend.cu puts the 32 lanes of a warp
 * on consecutive query columns of ONE extension; for 150-bp reads a row is ~35 cells wide and ~80 instructions of per-row
 * bookkeeping (scan carries, reductions, band update) surround ~70 instructions of cell work, so the warp retires about one
 * cell per several issued instructions.  Here a
 * lane owns a read and runs ksw_extend2's own scalar loop, so a warp works on 32 extensions at once:
 *   - a DP column is one 32-bit shared-memory word of the lane: H (13 bits) | E (13 bits) | 8 x query code (6 bits), laid
 *     out [column][thread] -> conflict-free, one LDS + one STS per cell, the query base comes with the cell;
 *   - a cell is ~20 integer instructions: the substitution score is a funnel shift into the packed 5-byte matrix row of the
 *     row's reference base, H/E/F are DPX max-plus (__viaddmax_s32 / __vimax3_s32), the row maximum and its right-most
 *     column travel as one key (h << 16 | j) through one max;
 *   - lanes run in LOCK STEP through a small state machine: every iteration each lane in the DP does up to K4L_CH cells of
 *     its current row (then, if the row is complete, the reference's end-of-row logic: first-column carry, gscore, Z-drop,
 *     band trimming by its own two scanning loops, and the exact row cut-off of bwag_extend.cu); lanes that need a new
 *     extension / seed / chain / read run that (rare, divergent) code when enough of them wait or a few iterations passed;
 *   - persistent lanes pull reads from an atomic counter.
 * A lane's row has K4L_CH spare columns at its end (the masked cells read them).
 * Valid when every score fits 13 bits (max_len * max(mat) < 8192), gap penalties are non-negative (as the lean sweeps) and
 * a block's columns fit shared memory; the host picks bwag_extend.cu's kernels otherwise (long reads: rows are hundreds
 * of cells wide there and the warp-per-extension mapping is the right one).  Integer-ALU bound.
 */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"

#define XSEED_DEAD 0x40000000u
#define XSEED_LEN(x) ((int)((x) & 0x3fffffffu))
#define K4L_CH 8

enum { L_FETCH = 0, L_CHAIN, L_SEED, L_EXT_BEGIN, L_INIT, L_ROWS, L_EXT_END, L_DONE };

#ifdef BWAG_CUSIM
#define K4L_LD(addr) (*reinterpret_cast<const u32 *>(addr))
#define K4L_ST(addr, v) (*reinterpret_cast<u32 *>(addr) = (v))
typedef unsigned char *k4l_addr;
__device__ __forceinline__ u32 k4l_rc(u32 lo, u32 hi, u32 s) { return s >= 32 ? hi : __funnelshift_r(lo, hi, s); }
#else
__device__ __forceinline__ u32 k4l_ld(u32 a) { u32 v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void k4l_st(u32 a, u32 v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v)); }
#define K4L_LD(addr) k4l_ld(addr)
#define K4L_ST(addr, v) k4l_st(addr, v)
typedef u32 k4l_addr;
__device__ __forceinline__ u32 k4l_rc(u32 lo, u32 hi, u32 s) { return __funnelshift_rc(lo, hi, s); }
#endif
#define K4L_COL (K4L_THREADS * 4)            /* bytes between consecutive columns of a lane */
#define K4L_HE_MASK 0x03ffffffu
#define K4L_Q_MASK 0xfc000000u

__device__ __forceinline__ int k4l_max_gap(const bwag_sw_par_t &p, int qlen) /* cal_max_gap, bwamem.c:647-654 */
{
	int l_del = bwag_trunc_i32((double)(qlen * p.a - p.o_del) / p.e_del + 1.);
	int l_ins = bwag_trunc_i32((double)(qlen * p.a - p.o_ins) / p.e_ins + 1.);
	int l = l_del > l_ins ? l_del : l_ins;
	l = l > 1 ? l : 1;
	return l < p.w << 1 ? l : p.w << 1;
}

/* reference bases of up to 16 consecutive rows of an extension, 2 bits each, first row in the low bits: rows step by tdir from
 * doubled position p0, all on one strand (a chain's window never crosses l_pac), so they are 16 consecutive forward bases =
 * at most five bytes of pac, fetched together -- one memory round trip per 16 rows instead of one per row */
__device__ __forceinline__ u32 k4l_window(const DevIndex &ix, i64 p0, int tdir, int n)
{
	const bool rev = p0 >= ix.l_pac;
	const i64 f0 = rev ? (ix.l_pac << 1) - 1 - p0 : p0;       /* forward position of the first row */
	const int fdir = rev ? -tdir : tdir;
	const i64 lo = fdir > 0 ? f0 : f0 - (n - 1);               /* lowest forward position */
	const uint8_t *b = ix.pac + (lo >> 2);
	const int nb = (int)(((lo + n - 1) >> 2) - (lo >> 2)) + 1;  /* 1..5 bytes */
	unsigned long long v = 0;
#pragma unroll
	for (int k = 0; k < 5; ++k) v = v << 8 | (k < nb ? (unsigned long long)b[k] : 0ull);   /* first base of byte 0 in bits 39..38 */
	const int s0 = 38 - 2 * (int)(lo & 3);
	u32 w = 0;
	for (int k = 0; k < n; ++k) {
		const int m = fdir > 0 ? k : n - 1 - k;
		u32 c = (u32)(v >> (s0 - 2 * m)) & 3u;
		if (rev) c = 3u - c;
		w |= c << (2 * k);
	}
	return w;
}

__global__ void __launch_bounds__(K4L_THREADS, K4L_MINB) k_extend_lane(DevIndex ix, ExtArgs a)
{
#ifdef BWAG_CUSIM
	unsigned char *dyn = cusim_dyn_smem;
	const k4l_addr he0 = dyn + threadIdx.x * 4;
#else
	extern __shared__ int4 k4l_dyn[];
	const k4l_addr he0 = (u32)__cvta_generic_to_shared(k4l_dyn) + threadIdx.x * 4;
#endif
	__shared__ unsigned long long s_row[8];      /* matrix row of reference base t: byte q = mat[t*5+q] */
	const bwag_sw_par_t &p = a.par;
	if (threadIdx.x < 5) {
		unsigned long long v = 0;
		for (int q = 0; q < 5; ++q) v |= (unsigned long long)(uint8_t)p.mat[threadIdx.x * 5 + q] << (8 * q);
		s_row[threadIdx.x] = v;
	}
	__syncthreads();
	int maxsc = 0;
	for (int k = 0; k < 25; ++k) maxsc = maxsc > p.mat[k] ? maxsc : p.mat[k];
	const int o_del = p.o_del, e_del = p.e_del, o_ins = p.o_ins, e_ins = p.e_ins;
	const int noe_del = -(o_del + e_del), ne_del = -e_del, noe_ins = -(o_ins + e_ins), ne_ins = -e_ins, zdrop = p.zdrop;

	/* read / chain / seed */
	int st = L_FETCH, rid = -1, l_query = 0, n_regs = 0, k = 0, n_seeds = 0, c_idx = 0;
	i64 c = 0, c1 = 0, rmax0 = 0, rmax1 = 0, s_rbeg = 0;
	const uint8_t *query = 0;
	bwag_xreg_t *regs = 0;
	bwag_xseed_t *seeds = 0;
	int s_qbeg = 0, s_len = 0, phase = 0, it = 0, aw0 = 0, aw1 = 0, sc0 = 0, prev = 0;
	bwag_xreg_t reg;
	reg.rb = reg.re = 0; reg.qb = reg.qe = reg.score = reg.truesc = reg.w = reg.seedcov = reg.seedlen0 = reg.chain = 0;
	/* extension */
	int qlen = 0, tlen = 0, h0 = 0, w = 0, i = 0, beg = 0, end = 0, mx = 0, max_i = 0, max_j = 0, max_ie = 0, gscore = 0, max_off = 0, pot0 = 0;
	i64 tbase = 0; int tdir = 1, t_cur = 0; u32 tw = 0;
	/* row */
	int jcur = 0, f = 0, hp = 0, key = -1, jmin = 0x7fffffff, jmax = -1, phi = 0, H1 = 0;
	const uint8_t *qp = 0; int qs = 1;
	u32 rlo = 0, rhi = 0;
	u64 cells = 0;
	int overflow = 0, waited = 0;

	for (;;) {
		/* ---- divergent part: lanes that are not inside a DP advance their read's control flow ---- */
		const u32 want = __ballot_sync(FULL_MASK, st != L_ROWS && st != L_INIT && st != L_DONE);
		const bool go = want && (__popc(want) >= 4 || waited >= 6 || !__any_sync(FULL_MASK, st == L_ROWS || st == L_INIT));
		waited = go ? 0 : waited + 1;
		if (go && st != L_ROWS && st != L_INIT && st != L_DONE) {
			for (;;) {
				if (st == L_FETCH) {
					rid = atomicAdd(a.next_read, 1);
					if (rid >= a.n_reads) { rid = -1; st = L_DONE; break; }
					{ const int cc = a.chain_cnt[rid]; if (cc < a.chain_lo || cc > a.chain_hi) continue; }   /* another launch's read */
					c = a.chain_beg[rid]; c1 = c + a.chain_cnt[rid]; c_idx = 0; n_regs = 0;
					l_query = (int)(a.off[rid + 1] - a.off[rid]);
					query = a.codes + a.off[rid];
					regs = a.regs + a.reg_base[rid];
					if (l_query > a.cap_q) { overflow = 1; a.n_regs[rid] = 0; continue; }
					st = L_CHAIN;
				}
				if (st == L_CHAIN) {
					if (c >= c1) { a.n_regs[rid] = n_regs; st = L_FETCH; continue; }
					const bwag_xchain_t ch = a.chains[c];
					seeds = const_cast<bwag_xseed_t *>(a.seeds) + ch.seed_off;
					rmax0 = ch.rmax0; rmax1 = ch.rmax1; n_seeds = ch.n_seeds; k = n_seeds;
					st = L_SEED;
				}
				if (st == L_SEED) {
					if (--k < 0) { ++c; ++c_idx; st = L_CHAIN; continue; }
					s_rbeg = seeds[k].rbeg; s_qbeg = seeds[k].qbeg; s_len = XSEED_LEN(seeds[k].len);
					{   /* containment test against every region of this read so far (bwamem.c:697-713) */
						int hit = -1;
						for (int r = 0; r < n_regs; ++r) {
							const bwag_xreg_t q = regs[r];
							if (s_rbeg < q.rb || s_rbeg + s_len > q.re || s_qbeg < q.qb || s_qbeg + s_len > q.qe) continue;
							if (s_len - q.seedlen0 > .1 * l_query) continue;
							int qd = s_qbeg - q.qb; i64 rd = s_rbeg - q.rb;
							int mg = k4l_max_gap(p, qd < rd ? qd : (int)rd);
							int ww = mg < q.w ? mg : q.w;
							bool around = qd - rd < ww && rd - qd < ww;
							if (!around) {
								qd = q.qe - (s_qbeg + s_len); rd = q.re - (s_rbeg + s_len);
								mg = k4l_max_gap(p, qd < rd ? qd : (int)rd);
								ww = mg < q.w ? mg : q.w;
								around = qd - rd < ww && rd - qd < ww;
							}
							if (around) { hit = r; break; }
						}
						if (hit >= 0) {   /* contained: extend only if an overlapping extended seed sits on another diagonal (bwamem.c:718-729) */
							bool other = false;
							for (int t = k + 1; t < n_seeds && !other; ++t) {
								const u32 tl_ = seeds[t].len;
								if (tl_ & (XSEED_DEAD | BWAG_XSEED_ZEROKEY)) continue;
								const int t_len = XSEED_LEN(tl_), t_qbeg = seeds[t].qbeg;
								const i64 t_rbeg = seeds[t].rbeg;
								if (t_len < s_len * .95) continue;
								if (s_qbeg <= t_qbeg && s_qbeg + s_len - t_qbeg >= s_len >> 2 && t_qbeg - s_qbeg != t_rbeg - s_rbeg) other = true;
								else if (t_qbeg <= s_qbeg && t_qbeg + t_len - s_qbeg >= s_len >> 2 && s_qbeg - t_qbeg != s_rbeg - t_rbeg) other = true;
							}
							if (!other) { seeds[k].len |= XSEED_DEAD; continue; }
						}
					}
					reg.score = reg.truesc = -1; reg.chain = c_idx; reg.seedlen0 = s_len; reg.seedcov = 0; reg.w = 0;
					aw0 = aw1 = p.w; it = 0;
					if (s_qbeg) { phase = 0; prev = reg.score; st = L_EXT_BEGIN; }
					else { reg.score = reg.truesc = s_len * p.a; reg.qb = 0; reg.rb = s_rbeg; phase = 1; }
				}
				if (st == L_SEED || st == L_EXT_END) {   /* an extension result (L_EXT_END), or a seed that starts at the read's first base (L_SEED, phase 1) */
					bool right_done = false;
					if (st == L_EXT_END) {
						const int score = mx, qle = max_j + 1, tle = max_i + 1, gtle = max_ie + 1;
						const int aw = phase == 0 ? aw0 : aw1;
						reg.score = score;
						if (!(score == prev || max_off < (aw >> 1) + (aw >> 2)) && it == 0) { it = 1; prev = score; st = L_EXT_BEGIN; }   /* a wider band may do better (bwamem.c:741-748) */
						else if (phase == 0) {
							if (gscore <= 0 || gscore <= reg.score - p.pen_clip5) { reg.qb = s_qbeg - qle; reg.rb = s_rbeg - tle; reg.truesc = reg.score; }
							else { reg.qb = 0; reg.rb = s_rbeg - gtle; reg.truesc = gscore; }
							phase = 1; it = 0; st = L_SEED;
						} else {
							const int qe = s_qbeg + s_len;
							const i64 re = s_rbeg + s_len;
							if (gscore <= 0 || gscore <= reg.score - p.pen_clip3) { reg.qe = qe + qle; reg.re = re + tle; reg.truesc += reg.score - sc0; }
							else { reg.qe = l_query; reg.re = re + gtle; reg.truesc += gscore - sc0; }
							right_done = true; st = L_SEED;
						}
					}
					if (st == L_SEED && phase == 1 && !right_done) {   /* to the right, if the seed does not end the read */
						if (s_qbeg + s_len != l_query) { sc0 = reg.score; prev = reg.score; it = 0; st = L_EXT_BEGIN; }
						else { reg.qe = l_query; reg.re = s_rbeg + s_len; right_done = true; }
					}
					if (right_done) {   /* the region is complete (bwamem.c:800-808) */
						int cov = 0;
						for (int t = 0; t < n_seeds; ++t) {
							const int t_len = XSEED_LEN(seeds[t].len), t_qbeg = seeds[t].qbeg;
							const i64 t_rbeg = seeds[t].rbeg;
							if (t_qbeg >= reg.qb && t_qbeg + t_len <= reg.qe && t_rbeg >= reg.rb && t_rbeg + t_len <= reg.re) cov += t_len;
						}
						reg.seedcov = cov;
						reg.w = aw0 > aw1 ? aw0 : aw1;
						regs[n_regs++] = reg;
						phase = 0; st = L_SEED;
						continue;
					}
				}
				if (st == L_EXT_BEGIN) {   /* ksw_extend2's set-up (ksw.c:420-447) */
					int end_bonus;
					if (phase == 0) {
						aw0 = p.w << it; w = aw0; end_bonus = p.pen_clip5; h0 = s_len * p.a;
						qlen = s_qbeg; tlen = (int)(s_rbeg - rmax0);
						tbase = s_rbeg - 1; tdir = -1;
					} else {
						aw1 = p.w << it; w = aw1; end_bonus = p.pen_clip3; h0 = sc0;
						qlen = l_query - (s_qbeg + s_len); tlen = (int)(rmax1 - (s_rbeg + s_len));
						tbase = s_rbeg + s_len; tdir = 1;
					}
					{
						const int oe_ins = o_ins + e_ins;
						H1 = h0 > oe_ins ? h0 - oe_ins : 0;
						qp = phase == 0 ? query + s_qbeg - 1 : query + s_qbeg + s_len;
						qs = phase == 0 ? -1 : 1;
						int max_ins = bwag_trunc_i32((double)(qlen * maxsc + end_bonus - o_ins) / e_ins + 1.); max_ins = max_ins > 1 ? max_ins : 1;
						w = w < max_ins ? w : max_ins;
						int max_del = bwag_trunc_i32((double)(qlen * maxsc + end_bonus - o_del) / e_del + 1.); max_del = max_del > 1 ? max_del : 1;
						w = w < max_del ? w : max_del;
					}
					mx = h0; max_i = max_j = -1; max_ie = -1; gscore = -1; max_off = 0;
					beg = 0; end = qlen; i = 0;
					pot0 = maxsc * (qlen - 1);
					if (qlen + 1 + K4L_CH > a.smem_per_warp) { overflow = 1; st = L_EXT_END; continue; }   /* more columns than the launch provided (a seed shorter than min_seed): reported, the batch fails */
					if (tlen <= 0) { st = L_EXT_END; continue; }
					tw = k4l_window(ix, tbase, tdir, tlen < 16 ? tlen : 16);
					t_cur = (int)(tw & 3u); tw >>= 2;
					jcur = 0;
					st = L_INIT;   /* the first row's columns are written by the whole warp in the converged part below */
				}
				if (st == L_ROWS || st == L_INIT || st == L_DONE) break;
			}
		}
		if (__all_sync(FULL_MASK, st == L_DONE)) break;

		/* ---- converged part 1: the first row of a new extension (ksw.c:431-433).  Written by the WHOLE WARP for one lane at a time
		 * (lane l writes columns l, l + 32, ... of that lane's row): the ~40 columns of a 150-bp read's extension are two
		 * iterations of 32 lanes instead of 40 iterations of one ---- */
		for (u32 todo = __ballot_sync(FULL_MASK, st == L_INIT); todo; todo &= todo - 1) {
			const int src = __ffs((int)todo) - 1;
			const int lane = threadIdx.x & 31;
			const int s_qlen = __shfl_sync(FULL_MASK, qlen, src), s_h0 = __shfl_sync(FULL_MASK, h0, src), s_H1 = __shfl_sync(FULL_MASK, H1, src), s_qs = __shfl_sync(FULL_MASK, qs, src);
			const unsigned long long s_qp = __shfl_sync(FULL_MASK, (unsigned long long)(size_t)qp, src);
			const uint8_t *sq = reinterpret_cast<const uint8_t *>((size_t)s_qp);
			const k4l_addr row = he0 + (src - lane) * 4;            /* the row of lane `src` (same warp, same block) */
			for (int j = lane; j <= s_qlen; j += 32) {
				int v = j == 0 ? s_h0 : s_H1 - (j - 1) * e_ins;
				v = v > 0 ? v : 0;
				const u32 qc = j < s_qlen ? sq[j * s_qs] : 4;
				K4L_ST(row + j * K4L_COL, (u32)v | (qc > 4 ? 4u : qc) << 29);      /* 8 x code in the top six bits */
			}
			__syncwarp();
			if (lane == src) {   /* row 0: band, first-column carry (ksw.c:448-459) */
				if (end > w + 1) end = w + 1;
				if (end > qlen) end = qlen;
				hp = h0 - (o_del + e_del); if (hp < 0) hp = 0;
				f = 0; key = -1; jcur = 0; jmin = 0x7fffffff; jmax = -1; phi = 0;
				const unsigned long long rw = s_row[t_cur];
				rlo = (u32)rw; rhi = (u32)(rw >> 32);
				if (end > 0) cells += (u64)end;
				st = L_ROWS;
			}
		}
		/* ---- converged part 2: up to K4L_CH cells of the current row (ksw.c:460-484) ---- */
		if (st == L_ROWS) {
			int nact = end - jcur;
			nact = nact < K4L_CH ? nact : K4L_CH;
			k4l_addr ad = he0 + jcur * K4L_COL;
			u32 nzm = 0;
			int pot = pot0 - maxsc * jcur;
			/* straight-line code: cells past the row's end (only ever the tail of the chunk that ends the row) are computed on
			 * whatever their columns hold and masked -- no store, h1, the row maximum, the non-zero marks and the cut-off bound
			 * keep their values; F is dead by then */
#pragma unroll
			for (int cc = 0; cc < K4L_CH; ++cc) {
				const bool act = cc < nact;
				const u32 wd = K4L_LD(ad + cc * K4L_COL);
				const int H = (int)(wd & 0x1fffu), E = (int)(wd >> 13 & 0x1fffu);
				const int sc = (int)(int8_t)k4l_rc(rlo, rhi, wd >> 26);
				const int M = H ? H + sc : 0;
				const int h = __vimax3_s32(M, E, f);
				const int e = __viaddmax_s32(E, ne_del, __viaddmax_s32(M, noe_del, 0));
				f = __viaddmax_s32(f, ne_ins, __viaddmax_s32(M, noe_ins, 0));
				const int kk = act ? (h << 16) + (jcur + cc) : -1;
				key = key > kk ? key : kk;
				const u32 he = (u32)hp | (u32)e << 13;                   /* the stored cell: H(i, j-1), E(i+1, j) */
				if (act) K4L_ST(ad + cc * K4L_COL, (wd & K4L_Q_MASK) | he);
				nzm |= (act && he != 0) ? 1u << cc : 0u;
				phi = act ? __viaddmax_s32(h, pot - maxsc * cc, phi) : phi;    /* potential of the cell: score + maxsc per remaining column */
				hp = act ? h : hp;
			}
			if (nzm) {   /* first / last column of the row whose stored cell is non-zero: the next band (ksw.c:501-505) */
				const int lo = jcur + __ffs((int)nzm) - 1;
				jmax = jcur + 31 - __clz((int)nzm);
				jmin = jmin < lo ? jmin : lo;
			}
			if (nact > 0) jcur += nact;
		}
		/* ---- end of a row (ksw.c:485-506), then the next row's set-up ---- */
		if (st == L_ROWS && jcur >= end) {
			const int h1 = hp;
			{
				const k4l_addr ae = he0 + end * K4L_COL;
				K4L_ST(ae, (K4L_LD(ae) & K4L_Q_MASK) | (u32)h1);       /* eh[end].h = h1; eh[end].e = 0 */
			}
			const int m = key < 0 ? 0 : key >> 16, mj = key < 0 ? -1 : key & 0xffff;
			bool stop = false;
			if ((end > beg ? end : beg) == qlen) {                      /* ties go to the later row (ksw.c:486-489) */
				max_ie = gscore > h1 ? max_ie : i;
				gscore = gscore > h1 ? gscore : h1;
			}
			if (m == 0) stop = true;
			const bool falling = m <= mx, to_end = end == qlen && end > beg;
			if (!stop) {
				if (m > mx) {
					int d = mj - i;
					mx = m; max_i = i; max_j = mj;
					d = d < 0 ? -d : d;
					max_off = max_off > d ? max_off : d;
				} else if (zdrop > 0) {
					if (i - max_i > mj - max_j) { if (mx - m - ((i - max_i) - (mj - max_j)) * e_del > zdrop) stop = true; }
					else { if (mx - m - ((mj - max_j) - (i - max_i)) * e_ins > zdrop) stop = true; }
				}
			}
			if (!stop) {   /* next band: first non-zero stored cell .. last non-zero stored cell + 2, column `end` included (ksw.c:501-505) */
				const int nb = jmin == 0x7fffffff ? end : jmin;
				int jl = jmax;
				if (h1 != 0) jl = end;
				if (jl < 0) jl = nb - 1;
				beg = nb;
				end = jl + 2 < qlen ? jl + 2 : qlen;
				if (falling && to_end) {
					/* exact row cut-off (bwag_extend.cu): no later row can beat `mx` or reach `gscore` once every cell's potential
					 * (score + maxsc per remaining column) of the row just finished, and the first-column entry, are below them */
					int bound = phi;
					if (beg == 0) { const int fc = h0 - (o_del + e_del * (i + 1)) + maxsc * qlen; bound = bound > fc ? bound : fc; }
					if (bound <= mx && bound < gscore) stop = true;
				}
			}
			if (!stop && ++i >= tlen) stop = true;
			if (stop) st = L_EXT_END;
			else {   /* row i: band limits and first-column carry (ksw.c:448-459) */
				if (beg < i - w) beg = i - w;
				if (end > i + w + 1) end = i + w + 1;
				if (end > qlen) end = qlen;
				hp = 0;
				if (beg == 0) { hp = h0 - (o_del + e_del * (i + 1)); if (hp < 0) hp = 0; }
				f = 0; key = -1; jcur = beg; jmin = 0x7fffffff; jmax = -1; phi = 0;
				if ((i & 15) == 0) tw = k4l_window(ix, tbase + (i64)tdir * i, tdir, tlen - i < 16 ? tlen - i : 16);
				t_cur = (int)(tw & 3u); tw >>= 2;
				const unsigned long long rw = s_row[t_cur];
				rlo = (u32)rw; rhi = (u32)(rw >> 32);
				if (end > beg) cells += (u64)(end - beg);
			}
		}
	}
	for (int d = 16; d; d >>= 1) cells += __shfl_xor_sync(FULL_MASK, cells, d);
	if ((threadIdx.x & 31) == 0 && cells) atomicAdd(a.cells, cells);
	overflow = __any_sync(FULL_MASK, overflow);
	if (overflow && (threadIdx.x & 31) == 0) atomicOr(a.flags, 2u);
}
