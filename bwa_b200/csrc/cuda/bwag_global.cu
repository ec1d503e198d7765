/* bwag_global.cu -- stage 3 kernel (K5): banded global alignment -> CIGAR, NM, MD.
 *
 * Replaces bwa_gen_cigar2 (bwa.c:148-234) with ksw_global2 (ksw.c:540-642) and, in mode
 * BWAG_G_REG2ALN, the band-doubling loop of mem_reg2aln around it (bwamem.c:1143-1152).
 *
 * Mapping to the machine.  One warp per task (persistent warps, atomic task counter).  The DP is
 * swept row by row with the 32 lanes on consecutive query columns of the band, exactly like the
 * extension kernel: M/E per column depend on the previous row only, F along the row is a max-plus
 * prefix scan (shuffles), and the three direction bits of each cell (ksw.c:587-600) are derived per
 * lane from the scanned F.  One byte per cell goes to a per-warp backtrack matrix in global memory
 * (n_col x tlen, the only HBM traffic of the stage); the backtrack itself is a short serial walk
 * done by lane 0, after which NM/MD are produced from 32-base mismatch ballots.
 * The gap-free fast path of bwa_gen_cigar2 (equal lengths, band 0) never touches the DP.
 * Integer-ALU bound (cells), int32 cells with the reference's -2^30 sentinel.
 */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"
#include "bwag_ksw.cuh"   /* warp_ksw_global, ksw_backtrack */

/* The same sweep with about 40 % fewer instructions per 32-column chunk (see warp_ksw_extend_fast, bwag_extend.cu):
 * H/E side by side (64-bit accesses), no divergent code in the chunk (idle lanes load a clamped column and are masked),
 * F scanned in slanted coordinates (value + column*e_ins: a plain max scan without decay constants or lane guards) with
 * the F entering the chunk folded into lane 0's offer.  The direction bits still compare against lane 0's own offer.
 * q[j] at qa + j, t[i] at ta + i, the H/E pair of column j at he + 8*j, mat[k] at ma + k.  Exact for any penalties. */
template <class A, class AM>
__device__ __forceinline__ int warp_ksw_global_fast(int lane, int qlen, typename A::addr qa, int tlen, typename A::addr ta, typename AM::addr ma,
                               int o_del, int e_del, int o_ins, int e_ins, int w, typename A::addr he, uint8_t *z, int n_col, u64 *cells)
{
	const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
	for (int j = lane; j <= qlen; j += 32) A::st_he(he + 8 * j, j == 0 ? 0 : (j <= w ? -(o_ins + e_ins * j) : NEG_INF), NEG_INF);
	__syncwarp();
	const bool lane0 = lane == 0;
	const int le = lane * e_ins;
	for (int i = 0; i < tlen; ++i) {
		const typename AM::addr srow = ma + A::ld_u8(ta + i) * 5;
		const int beg = i > w ? i - w : 0, end = i + w + 1 < qlen ? i + w + 1 : qlen;
		int carry_h = beg == 0 ? -(o_del + e_del * (i + 1)) : NEG_INF;
		int carry_f = NEG_INF;
		uint8_t *zi = z ? z + (i64)i * n_col - beg : 0;
		if (end > beg) *cells += (u64)(end - beg);
		for (int j0 = beg; j0 < end; j0 += 32) {
			const int j = j0 + lane;
			const bool act = j < end;
			const int jc = act ? j : end - 1;
			const int2 c = A::ld_he(he + 8 * jc);
			const int m = c.x + AM::ld_s8(srow + A::ld_u8(qa + jc));
			const int tt = act ? m - oe_ins : -0x7f000000;     /* idle lanes (only at the end of the last chunk) must not feed the scan */
			int s = tt;
			if (lane0) s = __viaddmax_s32(carry_f, -e_ins, s);
			s += le;
			{ const int v = __shfl_up_sync(FULL_MASK, s, 1); s = s > v ? s : v; }
			{ const int v = __shfl_up_sync(FULL_MASK, s, 2); s = s > v ? s : v; }
			{ const int v = __shfl_up_sync(FULL_MASK, s, 4); s = s > v ? s : v; }
			{ const int v = __shfl_up_sync(FULL_MASK, s, 8); s = s > v ? s : v; }
			{ const int v = __shfl_up_sync(FULL_MASK, s, 16); s = s > v ? s : v; }
			int f = __shfl_up_sync(FULL_MASK, s, 1) - le + e_ins;    /* F(i, j) = the scan value of the column on the left */
			if (lane0) f = carry_f;
			carry_f = __shfl_sync(FULL_MASK, s, 31) - 31 * e_ins;
			int d = m >= c.y ? 0 : 1, h = m >= c.y ? m : c.y;
			d = h >= f ? d : 2; h = h >= f ? h : f;
			if (!act) h = NEG_INF;
			int hp = __shfl_up_sync(FULL_MASK, h, 1);
			if (lane0) hp = carry_h;
			{
				int la = end - 1 - j0; la = la < 31 ? la : 31;
				carry_h = __shfl_sync(FULL_MASK, h, la);
			}
			const int te = m - oe_del, ed = c.y - e_del;
			d |= ed > te ? 1 << 2 : 0;
			d |= (f - e_ins) > tt ? 2 << 4 : 0;
			if (act) {
				A::st_he(he + 8 * j, hp, ed > te ? ed : te);
				if (zi) zi[j] = (uint8_t)d;
			}
		}
		if (lane0) A::st_he(he + 8 * end, carry_h, NEG_INF);
		__syncwarp();
	}
	return A::ld_he(he + 8 * qlen).x;
}

__device__ __forceinline__ int md_put_num(char *md, int l, int v)
{
	char buf[12];
	int n = 0;
	do { buf[n++] = (char)('0' + v % 10); v /= 10; } while (v);
	while (n) md[l++] = buf[--n];
	return l;
}

/* SM: H/E rows and the two sequences of the task in shared memory (short reads); the backtrack matrix, the CIGAR and
 * the MD staging stay in the warp's global scratch */
template <bool C, class X, class Y> struct SelG { typedef X type; };
template <class X, class Y> struct SelG<false, X, Y> { typedef Y type; };

template <bool SM, bool FAST>
__device__ __forceinline__ void global_body(const DevIndex &ix, const GlbArgs &a)
{
	const int lane = threadIdx.x & 31;
	const i64 wid = ((i64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	int *H, *E;
	uint8_t *rseq, *qseq, *z_glob = a.z + wid * a.cap_z, *z_sm = 0;
	if (SM) {
#ifdef BWAG_CUSIM
		unsigned char *dyn = cusim_dyn_smem;
#else
		extern __shared__ int4 k5_dyn[];
		unsigned char *dyn = reinterpret_cast<unsigned char *>(k5_dyn);
#endif
		unsigned char *mine = dyn + (size_t)(threadIdx.x >> 5) * a.smem_per_warp;
		H = reinterpret_cast<int *>(mine); E = H + a.cap_q + 2;
		rseq = reinterpret_cast<uint8_t *>(E + a.cap_q + 2);
		qseq = rseq + a.cap_r;
		if (a.z_sm_bytes) z_sm = mine + a.smem_per_warp - a.z_sm_bytes;   /* the warp's slice ends with its backtrack bytes */
	} else {
		H = a.eh + wid * (i64)(2 * (a.cap_q + 2)); E = H + a.cap_q + 2;
		rseq = a.rseq + wid * (i64)a.cap_r; qseq = a.qseq + wid * (i64)(a.cap_q + 2);
	}
	typedef typename SelG<SM, SmemAcc, PtrAcc>::type A;   /* how the lean sweep reaches H/E and the sequences; the matrix is always shared */
	typename A::addr he_a = A::make(H), rs_a = A::make(rseq), q_a = A::make(qseq);
	if constexpr (SM && FAST) { BWAG_KEEP(he_a); BWAG_KEEP(rs_a); BWAG_KEEP(q_a); }
	const bwag_sw_par_t &p = a.par;
	__shared__ int8_t s_mat[32];
	if (threadIdx.x < 25) s_mat[threadIdx.x] = p.mat[threadIdx.x];
	__syncthreads();
	typename SmemAcc::addr mat_a = SmemAcc::make(s_mat);
	if constexpr (FAST) BWAG_KEEP(mat_a);
	u64 cells = 0;
	int overflow = 0;

	for (;;) {
		int tix = 0;
		if (lane == 0) tix = atomicAdd(a.next_task, 1);
		tix = __shfl_sync(FULL_MASK, tix, 0);
		if (tix >= a.n_tasks) break;
		const bwag_gtask_t tk = a.tasks[tix];
		const int lq = tk.qe - tk.qb;
		const i64 rb = tk.rb, re = tk.re;
		u32 *cig = a.w_cig + wid * (i64)a.cap_wcig;   /* built in per-warp scratch, then appended to the compact pools */
		char *md = a.w_md + wid * (i64)a.cap_wmd;
		int score = 0, n_cigar = 0, NM = -1, l_md = 0;
		bool ok = !(lq <= 0 || rb >= re || (rb < ix.l_pac && re > ix.l_pac)) && rb >= 0 && re <= ix.l_pac << 1;
		const int rlen = (int)(re - rb);
		if (ok && (lq > a.cap_q || rlen > a.cap_r)) { ok = false; overflow |= 4; }
		if (ok) {
			const uint8_t *query = a.codes + a.off[tk.read] + tk.qb;
			const bool rev = rb >= ix.l_pac;   /* reverse both so that gaps are left-aligned on the forward strand (bwa.c:162-167) */
			__syncwarp();
			for (int x = lane; x < rlen; x += 32) rseq[rev ? rlen - 1 - x : x] = (uint8_t)bwag_ref_base(ix, rb + x);
			for (int x = lane; x < lq; x += 32) qseq[rev ? lq - 1 - x : x] = query[x];
			__syncwarp();
			const int want = tk.mode == BWAG_G_REG2ALN;
			int w2 = tk.w, it = 0, last_sc = -(1 << 30);
			const bool have_pre = a.pre_n && a.pre_n[tix] >= 0;   /* the lane-per-request kernel made score and CIGAR: only NM/MD are left */
			for (;;) {
				if (want) w2 = w2 < p.w << 2 ? w2 : p.w << 2;
				n_cigar = 0;
				if (have_pre) {
					score = a.pre_score[tix]; n_cigar = a.pre_n[tix];
					for (int x = lane; x < n_cigar; x += 32) cig[x] = a.pre_cig[(i64)tix * K5L_MAXCIG + x];
					__syncwarp();
				} else if (lq == rlen && w2 == 0) {    /* no gap possible: score the diagonal */
					int sc = 0;
					for (int x = lane; x < lq; x += 32) sc += s_mat[rseq[x] * 5 + qseq[x]];
					score = __reduce_add_sync(FULL_MASK, sc);
					if (want) { cig[0] = (u32)lq << 4; n_cigar = 1; }
				} else {
					int w, max_gap, max_ins, max_del, min_w, d = rlen - lq;
					d = d < 0 ? -d : d;
					max_ins = bwag_trunc_i32((double)(((lq + 1) >> 1) * s_mat[0] - p.o_ins) / p.e_ins + 1.);
					max_del = bwag_trunc_i32((double)(((lq + 1) >> 1) * s_mat[0] - p.o_del) / p.e_del + 1.);
					max_gap = max_ins > max_del ? max_ins : max_del;
					max_gap = max_gap > 1 ? max_gap : 1;
					w = (max_gap + d + 1) >> 1;
					w = w < w2 ? w : w2;
					min_w = d + 3;
					w = w > min_w ? w : min_w;
					const int n_col = lq < 2 * w + 1 ? lq : 2 * w + 1;
					if (want && (i64)n_col * rlen > a.cap_z) { overflow |= 4; score = 0; break; }
					/* the direction bytes of a typical task (band ~11, 150 rows: 3.5 KB) stay in shared memory: the sweep's byte stores and,
					 * above all, the serial backtrack walk (one dependent load per step) then never leave the SM */
					uint8_t *z = z_sm && (i64)n_col * rlen <= a.z_sm_bytes ? z_sm : z_glob;
					if constexpr (FAST) score = warp_ksw_global_fast<A, SmemAcc>(lane, lq, q_a, rlen, rs_a, mat_a, p.o_del, p.e_del, p.o_ins, p.e_ins, w, he_a, want ? z : 0, n_col, &cells);
					else score = warp_ksw_global(lane, lq, qseq, rlen, rseq, s_mat, p.o_del, p.e_del, p.o_ins, p.e_ins, w, H, E, want ? z : 0, n_col, &cells);
					if (want) {
						if (lane == 0) n_cigar = ksw_backtrack(z, n_col, rlen, lq, w, cig);   /* ksw.c:613-627 */
						n_cigar = __shfl_sync(FULL_MASK, n_cigar, 0);
						__syncwarp();
					}
				}
				if (want) {                     /* NM and MD (bwa.c:196-226) */
					const char *b2c = rev ? "TGCAN" : "ACGTN";
					int x = 0, y = 0, u = 0, n_mm = 0, n_gap = 0;
					l_md = 0;
					for (int k = 0; k < n_cigar; ++k) {
						const int op = cig[k] & 0xf, len = (int)(cig[k] >> 4);
						if (op == 0) {
							for (int b0 = 0; b0 < len; b0 += 32) {
								const int b = b0 + lane;
								const bool mm = b < len && qseq[x + b] != rseq[y + b];
								u32 bal = __ballot_sync(FULL_MASK, mm);
								n_mm += __popc(bal);
								if (lane == 0) {
									int done = 0;       /* positions of this 32-block already accounted in u */
									while (bal) {
										int pos = __ffs(bal) - 1;
										u += pos - done;
										l_md = md_put_num(md, l_md, u);
										md[l_md++] = b2c[rseq[y + b0 + pos]];
										u = 0; done = pos + 1;
										bal &= bal - 1;
									}
									int blk = len - b0 < 32 ? len - b0 : 32;
									u += blk - done;
								}
							}
							x += len; y += len;
						} else if (op == 2) {
							if (k > 0 && k < n_cigar - 1) {
								if (lane == 0) {
									l_md = md_put_num(md, l_md, u);
									md[l_md++] = '^';
									for (int b = 0; b < len; ++b) md[l_md++] = b2c[rseq[y + b]];
									u = 0;
								}
								n_gap += len;
							}
							y += len;
						} else if (op == 1) { x += len; n_gap += len; }
					}
					if (lane == 0) { l_md = md_put_num(md, l_md, u); md[l_md++] = 0; }
					l_md = __shfl_sync(FULL_MASK, l_md, 0);
					NM = n_mm + n_gap;
				}
				if (!want || have_pre) break;
				if (score == last_sc || w2 == p.w << 2) break;
				last_sc = score;
				w2 <<= 1;
				if (!(++it < 3 && score < tk.truesc - p.a)) break;
			}
		}
		i64 co = 0, mo = 0;
		if (n_cigar || l_md) {
			if (lane == 0) { co = (i64)atomicAdd(a.n_cig, (u64)n_cigar); mo = (i64)atomicAdd(a.n_md, (u64)((l_md + 3) & ~3)); }
			co = __shfl_sync(FULL_MASK, co, 0); mo = __shfl_sync(FULL_MASK, mo, 0);
			__syncwarp();
			if (co + n_cigar <= a.cap_cig && mo + l_md <= a.cap_md) {
				for (int x = lane; x < n_cigar; x += 32) a.cigar[co + x] = cig[x];
				for (int x = lane; x < l_md; x += 32) a.md[mo + x] = md[x];
			} else overflow |= 16;
			__syncwarp();
		}
		if (lane == 0) {
			bwag_gres_t r;
			r.score = score; r.n_cigar = n_cigar; r.NM = NM; r.l_md = l_md; r.cigar_off = co; r.md_off = mo;
			a.res[tix] = r;
		}
	}
	if (lane == 0 && cells) atomicAdd(a.cells, cells);
	if (overflow && lane == 0) atomicOr(a.flags, (u32)overflow);
}

#ifndef K5_MINB
#define K5_MINB 6
#endif
/* k_global*: the first formulation of the sweep (BWA_B200_K5_FAST=0); k_global*_fast: the lean one, the default */
__global__ void __launch_bounds__(K5_THREADS) k_global(DevIndex ix, GlbArgs a) { global_body<false, false>(ix, a); }
__global__ void __launch_bounds__(K5_THREADS) k_global_sm(DevIndex ix, GlbArgs a) { global_body<true, false>(ix, a); }
__global__ void __launch_bounds__(K5_THREADS, K5_MINB) k_global_fast(DevIndex ix, GlbArgs a) { global_body<false, true>(ix, a); }
__global__ void __launch_bounds__(K5_THREADS, K5_MINB) k_global_sm_fast(DevIndex ix, GlbArgs a) { global_body<true, true>(ix, a); }
