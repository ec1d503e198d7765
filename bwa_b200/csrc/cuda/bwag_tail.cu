/* bwag_tail.cu -- stage 4 kernels (K7a k_tail_regs, K7b k_tail_sam): what the reference does per read AFTER the
 * extension, on the device, for the reads whose post-processing is "simple" (the great majority of a sequencing run):
 *
 *   K7a  regions of a read -> mem_sort_dedup_patch (bwamem.c:463-515) -> one CIGAR request per surviving region
 *        (mem_reg2aln's starting band, bwamem.c:818-825,1138-1142) for the global-alignment kernel K5, and the
 *        read pair's insert-size candidate (the loop body of mem_pestat, bwamem_pair.c:88-101);
 *   K7b  mem_mark_primary_se (bwamem.c:547-584), mem_approx_mapq_se (982-1006), the decision whether mate rescue would
 *        align anything (bwamem_pair.c:137-170), mem_pair (208-269), the pair logic of mem_sam_pe (270-419),
 *        mem_reg2aln's coordinate / clipping work (1154-1189) and the SAM record itself (mem_aln2sam, 851-976).
 *
 * One LANE per read pair (single-end: per read): a few hundred instructions of branchy integer logic on a handful of
 * regions, all tie-breaks included (the unstable introsort of ksort.h restated for short arrays, hash_64).  A read whose
 * post-processing leaves the simple case -- more than TAIL_MAXR regions, ALT contigs, a region merge that needs a global
 * alignment (mem_patch_reg), a mate-rescue alignment that would have to run, XA/supplementary/secondary records, very
 * long reads -- is FLAGGED, produces no text, and is re-aligned by the host-side path of bb_process.c (same device
 * stages, host post-processing); the flag is a statement about the read, not an approximation of its result.
 *
 * Floating point: every double/float expression keeps the reference's operand types and order, this file is compiled
 * with -fmad=false (no contraction of a*b+c), and libm values (log, erfc) come from host-made tables, so the integer
 * decisions that hang on them are the host's.
 *
 * Text layout per record (the host adds what it has and the device does not: read name, quality string, comment):
 *   part A = "\t" FLAG "\t" RNAME ... "\t" SEQ "\t"      (QUAL follows, reversed iff rec.flags & 2)
 *   part B = "\tNM:i:" ... tags, no newline
 */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"

#define TAIL_MAXR 8      /* regions per read the simple path handles (one quicksort partition + insertion sort: n <= 17) */
#define TAIL_MAXC 20     /* CIGAR operations per record */
#define TAIL_LOGN 4096

/* ---------------------------------------------------------------- small helpers */
__device__ __forceinline__ u64 t_mix64(u64 k)   /* hash_64 (utils.h:98-109) */
{
	k += ~(k << 32); k ^= (k >> 22);
	k += ~(k << 13); k ^= (k >> 8);
	k += (k << 3);   k ^= (k >> 15);
	k += ~(k << 27); k ^= (k >> 31);
	return k;
}
__device__ __forceinline__ i64 t_depos(const TailCtg &c, i64 pos, int *is_rev) { *is_rev = pos >= c.l_pac; return *is_rev ? (c.l_pac << 1) - 1 - pos : pos; }
/* orientation class (0 FF, 1 FR, 2 RF, 3 RR) and distance of two hits (mem_infer_dir, bwamem_pair.c:48-56) */
__device__ __forceinline__ int t_infer_dir(i64 l_pac, i64 b1, i64 b2, i64 *dist)
{
	const int r1 = b1 >= l_pac, r2 = b2 >= l_pac;
	const i64 p2 = r1 == r2 ? b2 : (l_pac << 1) - 1 - b2;
	*dist = p2 > b1 ? p2 - b1 : b1 - p2;
	return (r1 == r2 ? 0 : 1) ^ (p2 > b1 ? 0 : 3);
}

struct LtEnd { __device__ bool operator()(const mem_alnreg_t &a, const mem_alnreg_t &b) const { return a.re < b.re; } };
struct LtScorePos { __device__ bool operator()(const mem_alnreg_t &a, const mem_alnreg_t &b) const { return a.score > b.score || (a.score == b.score && (a.rb < b.rb || (a.rb == b.rb && a.qb < b.qb))); } };
struct LtScoreHash { __device__ bool operator()(const mem_alnreg_t &a, const mem_alnreg_t &b) const { return a.score > b.score || (a.score == b.score && (a.is_alt < b.is_alt || (a.is_alt == b.is_alt && a.hash < b.hash))); } };
struct P64 { u64 x, y; };
struct LtP64 { __device__ bool operator()(const P64 &a, const P64 &b) const { return a.x < b.x || (a.x == b.x && a.y < b.y); } };

__device__ __forceinline__ int t_infer_bw(int l1, int l2, int score, int a, int q, int r)   /* bwamem.c:818-825 */
{
	int w;
	if (l1 == l2 && l1 * a - score < (q + r - a) << 1) return 0;
	w = (int)(((double)((l1 < l2 ? l1 : l2) * a - score - q) / r + 2.));
	const int d = l1 > l2 ? l1 - l2 : l2 - l1;
	if (w < d) w = d;
	return w;
}
__device__ __forceinline__ int t_reg2aln_band(const mem_opt_t &opt, const mem_alnreg_t &ar)   /* bwamem.c:1138-1142 */
{
	const int tmp = t_infer_bw(ar.qe - ar.qb, (int)(ar.re - ar.rb), ar.truesc, opt.a, opt.o_del, opt.e_del);
	int w2 = t_infer_bw(ar.qe - ar.qb, (int)(ar.re - ar.rb), ar.truesc, opt.a, opt.o_ins, opt.e_ins);
	w2 = w2 > tmp ? w2 : tmp;
	if (w2 > opt.w) w2 = w2 < ar.w ? w2 : ar.w;
	return w2;
}

/* ---------------------------------------------------------------- K7a */
/* mem_patch_reg up to the point where it would call the global alignment (bwamem.c:432-453): 0 = these two regions are
 * not merged, 1 = the decision needs the alignment score -> the read leaves the simple path */
__device__ int t_patch_needs_aln(const mem_opt_t &opt, i64 l_pac, const mem_alnreg_t &a, const mem_alnreg_t &b)
{
	int w;
	double r;
	if (a.rb < l_pac && b.rb >= l_pac) return 0;
	if (a.qb >= b.qb || a.qe >= b.qe || a.re >= b.re) return 0;
	w = (int)((a.re - b.rb) - (a.qe - b.qb));
	w = w > 0 ? w : -w;
	r = (double)(a.re - b.rb) / (b.re - a.rb) - (double)(a.qe - b.qb) / (b.qe - a.qb);
	r = r > 0. ? r : -r;
	if (a.re < b.rb || a.qe < b.qb) {
		if (w > opt.w << 1 || r >= 0.05f) return 0;
	} else if (w > opt.w << 2 || r >= 0.05f * 2) return 0;
	return 1;
}

/* mem_sort_dedup_patch (bwamem.c:463-515) on a[0..n); returns the new count or -1 (a merge needs an alignment) */
__device__ int t_dedup(const mem_opt_t &opt, i64 l_pac, int n, mem_alnreg_t *a)
{
	int m, i, j;
	if (n <= 1) return n;
	t_isort17(a, n, LtEnd());
	for (i = 0; i < n; ++i) a[i].n_comp = 1;
	for (i = 1; i < n; ++i) {
		mem_alnreg_t *p = &a[i];
		if (p->rid != a[i - 1].rid || p->rb >= a[i - 1].re + opt.max_chain_gap) continue;
		for (j = i - 1; j >= 0 && p->rid == a[j].rid && p->rb < a[j].re + opt.max_chain_gap; --j) {
			mem_alnreg_t *q = &a[j];
			i64 o_r, o_q, m_r, m_q;
			if (q->qe == q->qb) continue;
			o_r = q->re - p->rb;
			o_q = q->qb < p->qb ? q->qe - p->qb : p->qe - q->qb;
			m_r = q->re - q->rb < p->re - p->rb ? q->re - q->rb : p->re - p->rb;
			m_q = q->qe - q->qb < p->qe - p->qb ? q->qe - q->qb : p->qe - p->qb;
			if (o_r > opt.mask_level_redun * m_r && o_q > opt.mask_level_redun * m_q) {
				if (p->score < q->score) { p->qe = p->qb; break; }
				else q->qe = q->qb;
			} else if (q->rb < p->rb && t_patch_needs_aln(opt, l_pac, *q, *p)) return -1;
		}
	}
	for (i = 0, m = 0; i < n; ++i)
		if (a[i].qe > a[i].qb) { if (m != i) a[m] = a[i]; ++m; }
	n = m;
	t_isort17(a, n, LtScorePos());
	for (i = 1; i < n; ++i)
		if (a[i].score == a[i - 1].score && a[i].rb == a[i - 1].rb && a[i].qb == a[i - 1].qb) a[i].qe = a[i].qb;
	for (i = 1, m = 1; i < n; ++i)
		if (a[i].qe > a[i].qb) { if (m != i) a[m] = a[i]; ++m; }
	return n ? m : 0;
}

__device__ int t_best_overlapping_sub(const mem_opt_t &opt, int n, const mem_alnreg_t *a)   /* cal_sub, bwamem_pair.c:58-70 */
{
	int j;
	for (j = 1; j < n; ++j) {
		const int b_max = a[j].qb > a[0].qb ? a[j].qb : a[0].qb;
		const int e_min = a[j].qe < a[0].qe ? a[j].qe : a[0].qe;
		if (e_min > b_max) {
			const int lj = a[j].qe - a[j].qb, l0 = a[0].qe - a[0].qb;
			const int min_l = lj < l0 ? lj : l0;
			if (e_min - b_max >= min_l * opt.mask_level) break;
		}
	}
	return j < n ? a[j].score : opt.min_seed_len * opt.a;
}

__global__ void __launch_bounds__(128) k_tail_regs(TailRegsArgs a)
{
	const int unit = blockIdx.x * blockDim.x + threadIdx.x;
	const int n_units = a.pe ? a.n_reads >> 1 : a.n_reads;
	int max_lq = 0, max_rl = 0;
	u64 max_z = 0;
	if (unit < n_units) {
		const mem_opt_t &opt = a.opt;
		mem_alnreg_t regs[2][TAIL_MAXR];
		int cnt[2] = {0, 0}, bad[2] = {0, 0};
		const int n_ends = a.pe ? 2 : 1;
		for (int e = 0; e < n_ends; ++e) {
			const int r = a.pe ? (unit << 1 | e) : unit;
			const int n = a.n_raw[r];
			int flag = 0, m = 0;
			mem_alnreg_t *v = regs[e];
			if (n > TAIL_MAXR) flag = BWAG_CX_MANY;
			else {
				const bwag_xreg_t *x = a.xregs + a.reg_base[r];
				const i64 cb = a.chain_beg[r];
				for (int k = 0; k < n; ++k) {
					mem_alnreg_t t;
					memset(&t, 0, sizeof(t));
					t.rb = x[k].rb; t.re = x[k].re; t.qb = x[k].qb; t.qe = x[k].qe;
					t.score = x[k].score; t.truesc = x[k].truesc; t.w = x[k].w; t.seedcov = x[k].seedcov; t.seedlen0 = x[k].seedlen0;
					t.rid = a.chain_rid[cb + x[k].chain]; t.frac_rep = a.chain_frac[cb + x[k].chain];
					if (t.rid < 0 || a.ctg.alt[t.rid]) flag = BWAG_CX_ALT;
					v[k] = t;
				}
				if (!flag) { m = t_dedup(opt, a.ctg.l_pac, n, v); if (m < 0) { flag = BWAG_CX_PATCH; m = 0; } }
			}
			if (!flag) {
				const i64 base = (i64)atomicAdd(a.n_dregs, (u64)m);
				const i64 t0 = (i64)atomicAdd(a.n_tasks, (u64)m);
				a.dreg_beg[r] = base; a.task_beg[r] = t0; a.dreg_n[r] = m;
				if (base + m > a.cap_dregs || t0 + m > a.cap_tasks) flag = BWAG_CX_CAP;
				else for (int k = 0; k < m; ++k) {
					bwag_gtask_t t;
					mem_alnreg_t &p = v[k];
					p.n_comp = k;     /* from here on: which of the read's CIGAR requests belongs to this region (the reference never reads n_comp again) */
					t.rb = p.rb; t.re = p.re; t.read = r; t.qb = p.qb; t.qe = p.qe; t.w = t_reg2aln_band(opt, p); t.truesc = p.truesc; t.mode = BWAG_G_REG2ALN;
					a.tasks[t0 + k] = t;
					a.dregs[base + k] = p;
					{   /* scratch K5 needs for this task (as bwag_global sizes it from host-made tasks) */
						const i64 lq = p.qe - p.qb, rl = p.re - p.rb;
						i64 d = rl > lq ? rl - lq : lq - rl, wmax = (i64)opt.w << 2;
						if (d + 3 > wmax) wmax = d + 3;
						const i64 ncol = lq < 2 * wmax + 1 ? lq : 2 * wmax + 1;
						if (lq > max_lq) max_lq = (int)lq;
						if (rl > max_rl) max_rl = (int)rl;
						if ((u64)(ncol * rl) > max_z) max_z = (u64)(ncol * rl);
					}
				}
			} else { a.dreg_beg[r] = 0; a.task_beg[r] = 0; a.dreg_n[r] = 0; }
			a.cflag[r] = (uint8_t)flag;
			cnt[e] = m; bad[e] = flag;
		}
		if (a.pe) {   /* mem_pestat's per-pair candidate (bwamem_pair.c:88-101); pairs with a flagged end are filled in by the host path */
			u64 v = 0;
			if (!bad[0] && !bad[1] && cnt[0] && cnt[1]) {
				const mem_alnreg_t *r0 = regs[0], *r1 = regs[1];
				if (!(t_best_overlapping_sub(opt, cnt[0], r0) > 0.8 * r0[0].score) && !(t_best_overlapping_sub(opt, cnt[1], r1) > 0.8 * r1[0].score) && r0[0].rid == r1[0].rid) {
					i64 is;
					const int dir = t_infer_dir(a.ctg.l_pac, r0[0].rb, r1[0].rb, &is);
					if (is && is <= opt.max_ins) v = (u64)(dir + 1) << 48 | (u64)is;
				}
			}
			a.pe_is[unit] = v;
		}
	}
	max_lq = __reduce_max_sync(FULL_MASK, max_lq); max_rl = __reduce_max_sync(FULL_MASK, max_rl);
	for (int d = 16; d; d >>= 1) { const u64 o = __shfl_xor_sync(FULL_MASK, max_z, d); if (o > max_z) max_z = o; }
	if ((threadIdx.x & 31) == 0) {
		if (max_lq) atomicMax(a.max_lq, max_lq);
		if (max_rl) atomicMax(a.max_rl, max_rl);
		if (max_z) atomicMax(a.max_z, max_z);
	}
}

/* ---------------------------------------------------------------- K7b */
struct TAln {   /* mem_aln_t as far as one record needs it */
	i64 pos;
	int rid, flag, is_rev, mapq, NM, n_cigar, score, sub;
	int l_md;           /* without the NUL */
	const char *md;
	u32 cigar[TAIL_MAXC];
};

__device__ void t_mark_core(const mem_opt_t &opt, int n, mem_alnreg_t *a, int *z, int &zn)   /* mem_mark_primary_se_core, bwamem.c:519-545 */
{
	int tmp = opt.a + opt.b;
	if (opt.o_del + opt.e_del > tmp) tmp = opt.o_del + opt.e_del;
	if (opt.o_ins + opt.e_ins > tmp) tmp = opt.o_ins + opt.e_ins;
	zn = 0; z[zn++] = 0;
	for (int i = 1; i < n; ++i) {
		int k;
		for (k = 0; k < zn; ++k) {
			const int j = z[k];
			const int b_max = a[j].qb > a[i].qb ? a[j].qb : a[i].qb;
			const int e_min = a[j].qe < a[i].qe ? a[j].qe : a[i].qe;
			if (e_min > b_max) {
				const int min_l = a[i].qe - a[i].qb < a[j].qe - a[j].qb ? a[i].qe - a[i].qb : a[j].qe - a[j].qb;
				if (e_min - b_max >= min_l * opt.mask_level) {
					if (a[j].sub == 0) a[j].sub = a[i].score;
					if (a[j].score - a[i].score <= tmp && (a[j].is_alt || !a[i].is_alt)) ++a[j].sub_n;
					break;
				}
			}
		}
		if (k == zn) z[zn++] = i;
		else a[i].secondary = z[k];
	}
}
/* mem_mark_primary_se (bwamem.c:547-584) without ALT hits (the simple path has none): n_pri == n */
__device__ int t_mark_primary(const mem_opt_t &opt, int n, mem_alnreg_t *a, i64 id)
{
	int z[TAIL_MAXR], zn;
	if (n == 0) return 0;
	for (int i = 0; i < n; ++i) {
		a[i].sub = a[i].alt_sc = 0; a[i].secondary = a[i].secondary_all = -1;
		a[i].hash = t_mix64((u64)(id + i));
	}
	t_isort17(a, n, LtScoreHash());
	t_mark_core(opt, n, a, z, zn);
	for (int i = 0; i < n; ++i) a[i].secondary_all = a[i].secondary;
	return n;
}

/* mem_approx_mapq_se (bwamem.c:982-1006); logs of integers below TAIL_LOGN come from the host's libm table */
__device__ int t_mapq_se(const mem_opt_t &opt, const mem_alnreg_t &a, const double *logtab, int *cx)
{
	int mapq, l, sub = a.sub ? a.sub : opt.min_seed_len * opt.a;
	double identity;
	sub = a.csub > sub ? a.csub : sub;
	if (sub >= a.score) return 0;
	l = a.qe - a.qb > a.re - a.rb ? a.qe - a.qb : (int)(a.re - a.rb);
	identity = 1. - (double)(l * opt.a - a.score) / (opt.a + opt.b) / l;
	if (a.score == 0) mapq = 0;
	else if (opt.mapQ_coef_len > 0) {
		double tmp;
		if (l >= TAIL_LOGN) { *cx = BWAG_CX_LONG; return 0; }
		tmp = l < opt.mapQ_coef_len ? 1. : opt.mapQ_coef_fac / logtab[l];
		tmp *= identity * identity;
		mapq = (int)(6.02 * (a.score - sub) / opt.a * tmp * tmp + .499);
	} else {
		if (a.seedcov < 0 || a.seedcov >= TAIL_LOGN) { *cx = BWAG_CX_LONG; return 0; }
		mapq = (int)(30.0 * (1. - (double)sub / a.score) * logtab[a.seedcov] + .499);
		mapq = identity < 0.95 ? (int)(mapq * identity * identity + .499) : mapq;
	}
	if (a.sub_n > 0) mapq -= (int)(4.343 * logtab[a.sub_n + 1] + .499);
	if (mapq > 60) mapq = 60;
	if (mapq < 0) mapq = 0;
	mapq = (int)(mapq * (1. - a.frac_rep) + .499);
	return mapq;
}

/* would mem_matesw (bwamem_pair.c:137-206) run its local alignment for anchor `an` against the mate's hits ma[0..n_ma)? */
__device__ bool t_matesw_would_align(const TailSamArgs &g, const mem_alnreg_t &an, int n_ma, const mem_alnreg_t *ma, int l_ms)
{
	const i64 l_pac = g.ctg.l_pac;
	int skip[4], rid = -1;
	for (int r = 0; r < 4; ++r) skip[r] = g.pes[r].failed ? 1 : 0;
	for (int i = 0; i < n_ma; ++i) {
		i64 dist;
		const int r = t_infer_dir(l_pac, an.rb, ma[i].rb, &dist);
		if (dist >= g.pes[r].low && dist <= g.pes[r].high) skip[r] = 1;
	}
	if (skip[0] + skip[1] + skip[2] + skip[3] == 4) return false;
	for (int r = 0; r < 4; ++r) {
		if (skip[r]) continue;
		const int is_rev = (r >> 1 != (r & 1)), is_larger = !(r >> 1);
		i64 rb, re;
		if (!is_rev) {
			rb = is_larger ? an.rb + g.pes[r].low : an.rb - g.pes[r].high;
			re = (is_larger ? an.rb + g.pes[r].high : an.rb - g.pes[r].low) + l_ms;
		} else {
			rb = (is_larger ? an.rb + g.pes[r].low : an.rb - g.pes[r].high) - l_ms;
			re = is_larger ? an.rb + g.pes[r].high : an.rb - g.pes[r].low;
		}
		if (rb < 0) rb = 0;
		if (re > l_pac << 1) re = l_pac << 1;
		if (rb < re) {   /* bns_fetch_seq's clamp to the contig of the window's middle (bntseq.c:421-447) */
			int rev;
			const i64 mid = (rb + re) >> 1;
			rid = t_pos2rid(g.ctg, t_depos(g.ctg, mid, &rev));
			i64 far_beg = g.ctg.off[rid], far_end = far_beg + g.ctg.len[rid];
			if (rev) { const i64 t = far_beg; far_beg = (l_pac << 1) - far_end; far_end = (l_pac << 1) - t; }
			if (rb < far_beg) rb = far_beg;
			if (re > far_end) re = far_end;
		}
		if (an.rid == rid && re - rb >= g.opt.min_seed_len) return true;
	}
	return false;
}

/* mem_pair (bwamem_pair.c:208-269).  Returns the pair score o (0: none) or -1 when the simple path cannot decide. */
__device__ int t_pair(const TailSamArgs &g, const mem_alnreg_t *a0, int n0, const mem_alnreg_t *a1, int n1, int id, int *sub, int *n_sub, int z[2])
{
	const mem_opt_t &opt = g.opt;
	const i64 l_pac = g.ctg.l_pac;
	P64 v[2 * TAIL_MAXR], u[16];
	int nv = 0, nu = 0, y[4];
	for (int r = 0; r < 2; ++r) {
		const mem_alnreg_t *a = r ? a1 : a0;
		const int n = r ? n1 : n0;
		for (int i = 0; i < n; ++i) {
			const mem_alnreg_t &e = a[i];
			P64 key;
			key.x = e.rb < l_pac ? e.rb : (l_pac << 1) - 1 - e.rb;
			key.x = (u64)e.rid << 32 | (key.x - g.ctg.off[e.rid]);
			key.y = (u64)e.score << 32 | i << 2 | (e.rb >= l_pac) << 1 | r;
			v[nv++] = key;
		}
	}
	t_isort17(v, nv, LtP64());
	y[0] = y[1] = y[2] = y[3] = -1;
	for (int i = 0; i < nv; ++i) {
		for (int r = 0; r < 2; ++r) {
			const int dir = r << 1 | (int)(v[i].y >> 1 & 1);
			if (g.pes[dir].failed) continue;
			const int which = r << 1 | (int)((v[i].y & 1) ^ 1);
			if (y[which] < 0) continue;
			for (int k = y[which]; k >= 0; --k) {
				if ((v[k].y & 3) != (u64)which) continue;
				const i64 dist = (i64)v[i].x - (i64)v[k].x;
				if (dist > g.pes[dir].high) break;
				if (dist < g.pes[dir].low) continue;
				if (!g.ptab[dir]) return -1;
				int q = (int)((v[i].y >> 32) + (v[k].y >> 32) + g.ptab[dir][dist - g.pes[dir].low] + .499);
				if (q < 0) q = 0;
				if (nu == 16) return -1;
				P64 p;
				p.y = (u64)k << 32 | (u64)i;
				p.x = (u64)q << 32 | (t_mix64(p.y ^ (u64)(id << 8)) & 0xffffffffU);
				u[nu++] = p;
			}
		}
		y[v[i].y & 3] = i;
	}
	if (nu) {
		int tmp = opt.a + opt.b;
		if (opt.o_del + opt.e_del > tmp) tmp = opt.o_del + opt.e_del;
		if (opt.o_ins + opt.e_ins > tmp) tmp = opt.o_ins + opt.e_ins;
		t_isort17(u, nu, LtP64());
		const int i = (int)(u[nu - 1].y >> 32), k = (int)(u[nu - 1].y << 32 >> 32);
		z[v[i].y & 1] = (int)(v[i].y << 32 >> 34);
		z[v[k].y & 1] = (int)(v[k].y << 32 >> 34);
		const int ret = (int)(u[nu - 1].x >> 32);
		*sub = nu > 1 ? (int)(u[nu - 2].x >> 32) : 0;
		*n_sub = 0;
		for (int t = nu - 2; t >= 0; --t)
			if (*sub - (int)(u[t].x >> 32) <= tmp) ++*n_sub;
		return ret;
	}
	*sub = 0; *n_sub = 0;
	return 0;
}

/* does mem_gen_alt (bwamem_extra.c:124-172) list anything for this read? */
__device__ bool t_has_xa(const mem_opt_t &opt, int n, const mem_alnreg_t *a)
{
	if (n <= 1) return false;
	for (int i = 0; i < n; ++i) {
		const int k = a[i].secondary_all;
		if (k >= 0 && a[i].score >= a[k].score * (double)opt.XA_drop_ratio) return true;
	}
	return false;
}

/* mem_reg2aln (bwamem.c:1119-1189) with the CIGAR/NM/MD that K5 made for this region's request */
__device__ void t_reg2aln(const TailSamArgs &g, int read, int l_query, const mem_alnreg_t *ar, TAln *out, int *cx)
{
	TAln &a = *out;
	a.pos = 0; a.rid = 0; a.flag = 0; a.is_rev = 0; a.mapq = 0; a.NM = 0; a.n_cigar = 0; a.score = 0; a.sub = 0; a.l_md = 0; a.md = 0;
	if (ar == 0 || ar->rb < 0 || ar->re < 0) { a.rid = -1; a.pos = -1; a.flag |= 0x4; return; }
	const int qb = ar->qb, qe = ar->qe;
	const i64 rb = ar->rb, re = ar->re;
	a.mapq = ar->secondary < 0 ? t_mapq_se(g.opt, *ar, g.logtab, cx) : 0;
	if (ar->secondary >= 0) a.flag |= 0x100;
	int is_rev;
	i64 pos = t_depos(g.ctg, rb < g.ctg.l_pac ? rb : re - 1, &is_rev);
	a.is_rev = is_rev;
	const bwag_gres_t res = g.res[g.task_beg[read] + ar->n_comp];
	if (res.n_cigar <= 0 || res.n_cigar + 2 > TAIL_MAXC) { *cx = BWAG_CX_CIGAR; return; }
	const u32 *cg = g.cigar + res.cigar_off;
	int n = 0, first = 0, last = res.n_cigar;
	a.NM = res.NM; a.md = g.md + res.md_off; a.l_md = res.l_md > 0 ? res.l_md - 1 : 0;
	if ((cg[0] & 0xf) == 2) { pos += cg[0] >> 4; first = 1; }                 /* a leading or trailing deletion is dropped (bwamem.c:1157-1166) */
	else if ((cg[last - 1] & 0xf) == 2) --last;
	if (qb != 0 || qe != l_query) {
		const int clip5 = is_rev ? l_query - qe : qb, clip3 = is_rev ? qb : l_query - qe;
		if (clip5) a.cigar[n++] = (u32)clip5 << 4 | 3;
		for (int k = first; k < last; ++k) a.cigar[n++] = cg[k];
		if (clip3) a.cigar[n++] = (u32)clip3 << 4 | 3;
	} else for (int k = first; k < last; ++k) a.cigar[n++] = cg[k];
	a.n_cigar = n;
	a.rid = t_pos2rid(g.ctg, pos);
	if (a.rid != ar->rid) { *cx = BWAG_CX_CIGAR; return; }
	a.pos = pos - g.ctg.off[a.rid];
	a.score = ar->score; a.sub = ar->sub > ar->csub ? ar->sub : ar->csub;
}

struct TW { char *p; int n; };   /* text writer: p == 0 counts only */
__device__ __forceinline__ void tw_c(TW &w, char c) { if (w.p) w.p[w.n] = c; ++w.n; }
__device__ __forceinline__ void tw_s(TW &w, const char *s, int l) { if (w.p) for (int i = 0; i < l; ++i) w.p[w.n + i] = s[i]; w.n += l; }
__device__ void tw_l(TW &w, i64 v)   /* kputl's digits */
{
	char buf[24];
	int n = 0;
	u64 u = v < 0 ? (u64)(-(v + 1)) + 1u : (u64)v;
	do { buf[n++] = (char)('0' + u % 10); u /= 10; } while (u);
	if (v < 0) buf[n++] = '-';
	while (n) tw_c(w, buf[--n]);
}
__device__ void tw_cigar(TW &w, const TAln &al)
{
	if (al.n_cigar) for (int i = 0; i < al.n_cigar; ++i) { tw_l(w, al.cigar[i] >> 4); tw_c(w, "MIDSH"[al.cigar[i] & 0xf]); }   /* a single record: clips stay soft (which == 0) */
	else tw_c(w, '*');
}
__device__ int t_ref_len(const TAln &al)
{
	int l = 0;
	for (int k = 0; k < al.n_cigar; ++k) { const int op = al.cigar[k] & 0xf; if (op == 0 || op == 2) l += al.cigar[k] >> 4; }
	return l;
}

/* mem_aln2sam (bwamem.c:851-976) for a read with ONE record (n = 1, which = 0), mate m_ (0: single-end).  Writes part A
 * then part B through w; *len_a = bytes of part A; *qrev = strand the host must give the quality string. */
__device__ void t_aln2sam(const TailSamArgs &g, TW &w, const uint8_t *codes, int l_seq, const TAln &p_, const TAln *m_, int *len_a, int *qrev)
{
	TAln p = p_, m;
	const bool hm = m_ != 0;
	if (hm) m = *m_;
	p.flag |= hm ? 0x1 : 0;
	p.flag |= p.rid < 0 ? 0x4 : 0;
	p.flag |= hm && m.rid < 0 ? 0x8 : 0;
	if (p.rid < 0 && hm && m.rid >= 0) { p.rid = m.rid; p.pos = m.pos; p.is_rev = m.is_rev; p.n_cigar = 0; }
	if (hm && m.rid < 0 && p.rid >= 0) { m.rid = p.rid; m.pos = p.pos; m.is_rev = p.is_rev; m.n_cigar = 0; }
	p.flag |= p.is_rev ? 0x10 : 0;
	p.flag |= hm && m.is_rev ? 0x20 : 0;
	const int w0 = w.n;
	tw_c(w, '\t');
	tw_l(w, (p.flag & 0xffff) | (p.flag & 0x10000 ? 0x100 : 0)); tw_c(w, '\t');
	if (p.rid >= 0) {
		tw_s(w, g.ctg.names + g.ctg.name_off[p.rid], g.ctg.name_off[p.rid + 1] - g.ctg.name_off[p.rid]); tw_c(w, '\t');
		tw_l(w, p.pos + 1); tw_c(w, '\t');
		tw_l(w, p.mapq); tw_c(w, '\t');
		tw_cigar(w, p);
	} else tw_s(w, "*\t0\t0\t*", 7);
	tw_c(w, '\t');
	if (hm && m.rid >= 0) {
		if (p.rid == m.rid) tw_c(w, '=');
		else tw_s(w, g.ctg.names + g.ctg.name_off[m.rid], g.ctg.name_off[m.rid + 1] - g.ctg.name_off[m.rid]);
		tw_c(w, '\t');
		tw_l(w, m.pos + 1); tw_c(w, '\t');
		if (p.rid == m.rid) {
			const i64 p0 = p.pos + (p.is_rev ? t_ref_len(p) - 1 : 0);
			const i64 p1 = m.pos + (m.is_rev ? t_ref_len(m) - 1 : 0);
			if (m.n_cigar == 0 || p.n_cigar == 0) tw_c(w, '0');
			else tw_l(w, -(p0 - p1 + (p0 > p1 ? 1 : p0 < p1 ? -1 : 0)));
		} else tw_c(w, '0');
	} else tw_s(w, "*\t0\t0", 5);
	tw_c(w, '\t');
	if (w.p) {
		char *d = w.p + w.n;
		if (!p.is_rev) for (int i = 0; i < l_seq; ++i) { const int c = codes[i]; d[i] = "ACGTN"[c > 4 ? 4 : c]; }
		else for (int i = 0; i < l_seq; ++i) { const int c = codes[l_seq - 1 - i]; d[i] = "TGCAN"[c > 4 ? 4 : c]; }
	}
	w.n += l_seq;
	tw_c(w, '\t');
	*len_a = w.n - w0;
	*qrev = p.is_rev;
	if (p.n_cigar) {
		tw_s(w, "\tNM:i:", 6); tw_l(w, p.NM);
		tw_s(w, "\tMD:Z:", 6); tw_s(w, p.md, p.l_md);
	}
	if (hm && m.n_cigar) { tw_s(w, "\tMC:Z:", 6); tw_cigar(w, m); }
	if (hm) { tw_s(w, "\tMQ:i:", 6); tw_l(w, m.mapq); }
	if (p.score >= 0) { tw_s(w, "\tAS:i:", 6); tw_l(w, p.score); }
	if (p.sub >= 0) { tw_s(w, "\tXS:i:", 6); tw_l(w, p.sub); }
	if (g.l_rg) { tw_s(w, "\tRG:Z:", 6); tw_s(w, g.rg, g.l_rg); }
}

/* the record mem_reg2sam (bwamem.c:1033-1079) writes for a read, if it is exactly one: which region (or -1: the unmapped
 * record); more than one record, or an XA list, leaves the simple path */
__device__ int t_reg2sam_pick(const mem_opt_t &opt, int n, const mem_alnreg_t *a, int *cx)
{
	int l = 0, pick = -1;
	if (t_has_xa(opt, n, a)) { *cx = BWAG_CX_XA; return -1; }
	for (int k = 0; k < n; ++k) {
		const mem_alnreg_t &p = a[k];
		if (p.score < opt.T) continue;
		if (p.secondary >= 0) continue;             /* without MEM_F_ALL secondary hits are not printed */
		if (l++ == 0) pick = k;
	}
	if (l > 1) { *cx = BWAG_CX_MULTI; return -1; }
	return pick;
}

__global__ void __launch_bounds__(128) k_tail_sam(TailSamArgs g)
{
	const int unit = blockIdx.x * blockDim.x + threadIdx.x;
	const int n_units = g.pe ? g.n_reads >> 1 : g.n_reads;
	if (unit >= n_units) return;
	const mem_opt_t &opt = g.opt;
	const int n_ends = g.pe ? 2 : 1;
	mem_alnreg_t regs[2][TAIL_MAXR];
	int n[2] = {0, 0}, len[2] = {0, 0}, rd[2] = {0, 0}, cx = 0;
	for (int e = 0; e < n_ends; ++e) {
		const int r = g.pe ? (unit << 1 | e) : unit;
		rd[e] = r;
		len[e] = (int)(g.off[r + 1] - g.off[r]);
		if (g.cflag[r]) cx = g.cflag[r];
		else { n[e] = g.dreg_n[r]; for (int k = 0; k < n[e]; ++k) regs[e][k] = g.dregs[g.dreg_beg[r] + k]; }
	}
	TAln h[2], rec[2];
	bool have_rec[2] = {false, false};
	int extra_flag = 1;
	if (!cx && !g.pe) {   /* worker2, single-end (bwamem.c:1222-1226) */
		t_mark_primary(opt, n[0], regs[0], g.n_processed + unit);
		const int k = t_reg2sam_pick(opt, n[0], regs[0], &cx);
		if (!cx) t_reg2aln(g, rd[0], len[0], k >= 0 ? &regs[0][k] : 0, &rec[0], &cx);
	} else if (!cx) {     /* mem_sam_pe (bwamem_pair.c:270-419) */
		const u64 id = (u64)((g.n_processed >> 1) + unit);
		if (!(opt.flag & MEM_F_NO_RESCUE)) {   /* the rescue block: nothing may need aligning */
			for (int i = 0; i < 2 && !cx; ++i) {
				int nb = 0;
				for (int j = 0; j < n[i] && !cx; ++j) {
					if (!(regs[i][j].score >= regs[i][0].score - opt.pen_unpaired)) continue;
					if (nb++ >= opt.max_matesw) break;
					if (t_matesw_would_align(g, regs[i][j], n[!i], regs[!i], len[!i])) cx = BWAG_CX_RESCUE;
				}
			}
		}
		int n_pri[2], z[2] = {0, 0}, o = 0, subo = 0, n_sub = 0;
		bool paired = false;
		if (!cx) {
			n_pri[0] = t_mark_primary(opt, n[0], regs[0], (i64)(id << 1 | 0));
			n_pri[1] = t_mark_primary(opt, n[1], regs[1], (i64)(id << 1 | 1));
			if (!(opt.flag & MEM_F_NOPAIRING) && n_pri[0] && n_pri[1]) {
				o = t_pair(g, regs[0], n_pri[0], regs[1], n_pri[1], (int)id, &subo, &n_sub, z);
				if (o < 0) cx = BWAG_CX_PAIR;
			}
		}
		if (!cx && o > 0) {
			bool multi = false;
			for (int i = 0; i < 2; ++i)
				for (int j = 1; j < n_pri[i]; ++j)
					if (regs[i][j].secondary < 0 && regs[i][j].score >= opt.T) { multi = true; break; }
			paired = !multi;
		}
		if (!cx && paired) {
			int q_pe, q_se[2];
			const int score_un = regs[0][0].score + regs[1][0].score - opt.pen_unpaired;
			subo = subo > score_un ? subo : score_un;
			q_pe = (int)(6.02 * (o - subo) / opt.a + .499);
			if (n_sub > 0) { if (n_sub + 1 >= TAIL_LOGN) cx = BWAG_CX_PAIR; else q_pe -= (int)(4.343 * g.logtab[n_sub + 1] + .499); }
			if (q_pe < 0) q_pe = 0;
			if (q_pe > 60) q_pe = 60;
			q_pe = (int)(q_pe * (1. - .5 * (regs[0][0].frac_rep + regs[1][0].frac_rep)) + .499);
			if (o > score_un) {
				mem_alnreg_t *c[2] = { &regs[0][z[0]], &regs[1][z[1]] };
				for (int i = 0; i < 2; ++i) {
					if (c[i]->secondary >= 0) { c[i]->sub = regs[i][c[i]->secondary].score; c[i]->secondary = -2; }
					q_se[i] = t_mapq_se(opt, *c[i], g.logtab, &cx);
				}
				q_se[0] = q_se[0] > q_pe ? q_se[0] : q_pe < q_se[0] + 40 ? q_pe : q_se[0] + 40;
				q_se[1] = q_se[1] > q_pe ? q_se[1] : q_pe < q_se[1] + 40 ? q_pe : q_se[1] + 40;
				extra_flag |= 2;
				for (int i = 0; i < 2; ++i) {
					const int cap = (int)(6.02 * (c[i]->score - c[i]->csub) / opt.a + .499);
					q_se[i] = q_se[i] < cap ? q_se[i] : cap;
				}
			} else {
				z[0] = z[1] = 0;
				q_se[0] = t_mapq_se(opt, regs[0][0], g.logtab, &cx);
				q_se[1] = t_mapq_se(opt, regs[1][0], g.logtab, &cx);
			}
			for (int i = 0; i < 2; ++i) {
				const int k = regs[i][z[i]].secondary_all;
				if (k >= 0 && k < n_pri[i]) {
					for (int j = 0; j < n[i]; ++j)
						if (regs[i][j].secondary_all == k || j == k) regs[i][j].secondary_all = z[i];
					regs[i][z[i]].secondary_all = -1;
				}
			}
			if (!cx && (t_has_xa(opt, n[0], regs[0]) || t_has_xa(opt, n[1], regs[1]))) cx = BWAG_CX_XA;
			for (int i = 0; i < 2 && !cx; ++i) {
				t_reg2aln(g, rd[i], len[i], &regs[i][z[i]], &h[i], &cx);
				h[i].mapq = q_se[i];
				h[i].flag |= 0x40 << i | extra_flag;
				rec[i] = h[i];
			}
		} else if (!cx) {   /* no_pairing */
			for (int i = 0; i < 2 && !cx; ++i) {
				const int which = n[i] && regs[i][0].score >= opt.T ? 0 : -1;
				t_reg2aln(g, rd[i], len[i], which >= 0 ? &regs[i][which] : 0, &h[i], &cx);
			}
			if (!cx && !(opt.flag & MEM_F_NOPAIRING) && h[0].rid == h[1].rid && h[0].rid >= 0) {
				i64 dist;
				const int d = t_infer_dir(g.ctg.l_pac, regs[0][0].rb, regs[1][0].rb, &dist);
				if (!g.pes[d].failed && dist >= g.pes[d].low && dist <= g.pes[d].high) extra_flag |= 2;
			}
			for (int i = 0; i < 2 && !cx; ++i) {
				const int k = t_reg2sam_pick(opt, n[i], regs[i], &cx);
				if (cx) break;
				t_reg2aln(g, rd[i], len[i], k >= 0 ? &regs[i][k] : 0, &rec[i], &cx);
				rec[i].flag |= (i ? 0x81 : 0x41) | extra_flag;
			}
		}
		have_rec[0] = have_rec[1] = true;
	}
	if (!cx && !g.pe) have_rec[0] = true;
	for (int e = 0; e < n_ends; ++e) {
		bwag_samrec_t out;
		out.off = 0; out.len_a = out.len_b = 0; out.flags = 0; out.pad = 0;
		if (cx || !have_rec[e]) out.flags = BWAG_REC_COMPLEX | (u32)cx << 8;
		else {
			const uint8_t *codes = g.codes + g.off[rd[e]];
			const TAln *mate = g.pe ? &h[!e] : 0;
			TW w; w.p = 0; w.n = 0;
			int la = 0, qrev = 0;
			t_aln2sam(g, w, codes, len[e], rec[e], mate, &la, &qrev);
			const int total = w.n;
			const i64 o = (i64)atomicAdd(g.n_text, (u64)((total + 7) & ~7));
			out.off = o; out.len_a = la; out.len_b = total - la; out.flags = BWAG_REC_TEXT | (qrev ? BWAG_REC_QREV : 0);
			if (o + total <= g.cap_text) { w.p = g.text + o; w.n = 0; t_aln2sam(g, w, codes, len[e], rec[e], mate, &la, &qrev); }
		}
		g.rec[rd[e]] = out;
	}
	if (cx) atomicAdd(g.n_complex, (u64)n_ends);
}
