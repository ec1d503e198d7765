/* bwag_pemerge.cu -- the read-pair merging of `bwa pemerge` (bwa_pemerge and the printing loop, pemerge.c:59-215) on the device.
 *
 * A batch holds pairs: read 1 of pair i is read 2i, read 2 is read 2i + 1, as raw sequence bytes; their raw quality bytes sit at
 * the same offsets of a second buffer.
 *   M1 k_pem_encode  lane per pair: s0 = read 1, s1 = read 2 reversed and complemented, q0 / q1 their qualities minus 33 (uint8_t,
 *                    wrapping), and pair i's K6 task: query s1, target s0, KSW_XSTART | KSW_XSUBO with minsc 0 (16-bit kernel, the
 *                    reverse pass always runs).  s is K6's pool.  A pair with an empty read gets an empty task, which K6 skips.
 *   K6               bwag_localsw.cu, unchanged.
 *   M2/M3 k_pem_decide  warp per pair: the five early tests in the reference's order, then the tandem scan m(l) for l = 1 ..
 *                    min(l1, l2) - 1 with the lanes over l, the reference's top-two bookkeeping in l order, tests -6 and -7.
 *   M4 k_pem_text    lane per pair, twice around a scan: the merged read, sum_q and test -8, the outcome counts and the exact record
 *                    sizes; then the records (names uploaded with the batch) for -m, -u or both.
 * Every decision uses the reference's expressions: `(double)x / y >= 0.9f` (the float constant widened to double; a zero score
 * gives inf or NaN there as on the host) and uint8_t arithmetic for the qualities. */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"
#include "bwag_drv.h"

#define PEM_RATIO ((double)0.9f)   /* MAX_SCORE_RATIO (pemerge.c:19), a float compared with doubles */
#define PEM_A 5                     /* the reference's fixed scoring: bwa_fill_scmat(5, 4), N scores -1 */

/* nst_nt4_table (bntseq.c:46): ACGT in either case, everything else 4.  Its '-' (5) is taken as 4: see DESIGN.md 4.12 */
__device__ __forceinline__ int pem_nt4(int c)
{
	switch (c) {
	case 'A': case 'a': return 0;
	case 'C': case 'c': return 1;
	case 'G': case 'g': return 2;
	case 'T': case 't': return 3;
	default: return 4;
	}
}

__device__ __forceinline__ int pem_sc(int x, int y) { return x == 4 || y == 4 ? -1 : x == y ? PEM_A : -4; }

__global__ void k_pem_encode(PemArgs a)
{
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n_pairs; i += gridDim.x * blockDim.x) {
		const i64 o0 = a.off[2 * i], o1 = a.off[2 * i + 1], o2 = a.off[2 * i + 2];
		const int l0 = (int)(o1 - o0), l1 = (int)(o2 - o1), h0 = a.has_qual[2 * i], h1 = a.has_qual[2 * i + 1];
		for (int k = 0; k < l0; ++k) {   /* pemerge.c:67-71 */
			const int c = (signed char)a.raw[o0 + k];
			a.s[o0 + k] = (uint8_t)(c < 0 ? 4 : c <= 4 ? c : pem_nt4(c));
			a.q[o0 + k] = h0 ? (uint8_t)(a.qual[o0 + k] - 33) : (uint8_t)a.q_def;
		}
		for (int k = 0; k < l1; ++k) {   /* pemerge.c:72-77 */
			int c = (signed char)a.raw[o2 - 1 - k];
			c = c < 0 ? 4 : c < 4 ? c : pem_nt4(c);
			a.s[o1 + k] = (uint8_t)(c < 4 ? 3 - c : 4);
			a.q[o1 + k] = h1 ? (uint8_t)(a.qual[o2 - 1 - k] - 33) : (uint8_t)a.q_def;
		}
		bwag_swtask_t t;
		t.t_beg = o0; t.tlen = l0; t.q_beg = o1; t.qlen = l1;
		if (l0 == 0 || l1 == 0) t.tlen = t.qlen = 0;
		t.xtra = BWAG_SW_XSTART | BWAG_SW_XSUBO;   /* minsc 0 */
		t.flags = 0;
		a.tasks[i] = t;
		a.code[i] = 1;   /* not tried */
		a.ovl[i] = 0;
	}
}

__global__ void k_pem_decide(PemArgs a)
{
	const int lane = threadIdx.x & 31, nw = gridDim.x * (blockDim.x >> 5);
	for (int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < a.n_pairs; i += nw) {
		const i64 o0 = a.off[2 * i], o1 = a.off[2 * i + 1];
		const int l0 = (int)(o1 - o0), l1 = (int)(a.off[2 * i + 2] - o1);
		int score = 0, te = -1, qe = -1, score2 = -1, tb = 0, qb = 0;
		if (l0 > 0 && l1 > 0) {
			const bwag_swres_t r = a.res[i];
			score = r.score; te = r.te; qe = r.qe; score2 = r.score2; tb = r.tb; qb = r.qb;
		} else if (l0 > 0) score2 = 0;   /* empty query: ksw_i16 lists every row's maximum 0, so score2 = 0 (qe stays -1) */
		else if (l1 > 0) qe = 0;         /* empty target: the best query end of an all-zero row is 0 */
		++te; ++qe;
		int ret = 0;   /* pemerge.c:83-87; every lane decides the same */
		if (score < a.T) ret = -1;
		else if (tb < qb) ret = -2;
		else if (l0 - te > l1 - qe) ret = -3;
		else if ((double)score2 / score >= PEM_RATIO) ret = -4;
		else if (qe - qb != te - tb) ret = -5;
		if (ret == 0) {   /* pemerge.c:89-106 */
			const int min_l = l0 < l1 ? l0 : l1;
			const uint8_t *s0 = a.s + o0, *s1 = a.s + o1;
			int max_m = 0, max_m2 = 0, max_l = 0, max_l2 = 0;
			for (int base = 1; base < min_l; base += 32) {
				const int l = base + lane;
				int m = 0;
				if (l < min_l) {
					const uint8_t *s0o = s0 + (l0 - l);
					for (int k = 0; k < l; ++k) m += pem_sc(s1[k], s0o[k]);
				}
				const int nv = min_l - base < 32 ? min_l - base : 32;
				for (int j = 0; j < nv; ++j) {   /* in l order: strict >, the first maximum kept */
					const int mj = __shfl_sync(FULL_MASK, m, j), lj = base + j;
					if (mj > max_m) max_m2 = max_m, max_m = mj, max_l2 = max_l, max_l = lj;
					else if (mj > max_m2) max_m2 = mj, max_l2 = lj;
				}
			}
			if (max_m < a.T || max_l != l0 - (tb - qb)) ret = -6;
			else if (max_l2 < max_l && max_m2 >= a.T && (double)(max_m2 + (max_l - max_l2) * PEM_A) / max_m >= PEM_RATIO) ret = -7;
			else if (max_l2 > max_l && (double)max_m2 / max_m >= PEM_RATIO) ret = -7;
		}
		if (lane == 0) {
			a.code[i] = (int8_t)ret;
			a.ovl[i] = ret == 0 ? l0 - (tb - qb) : 0;
		}
	}
}

/* base k of the merged read (pemerge.c:108-128): its code and quality (before + 33) */
__device__ __forceinline__ void pem_merged(const PemArgs &a, i64 o0, i64 o1, int l0, int lm, int k, int &sc, int &qc)
{
	if (k >= l0) { sc = a.s[o1 + lm + k - l0]; qc = a.q[o1 + lm + k - l0]; return; }
	const int s0 = a.s[o0 + k], q0 = a.q[o0 + k];
	sc = s0; qc = q0;
	if (k < l0 - lm) return;
	const int i = k - (l0 - lm), s1 = a.s[o1 + i], q1 = a.q[o1 + i];
	if (s0 == 4) sc = s1, qc = q1;
	else if (s1 == 4) {}
	else if (s0 == s1) qc = q0 > q1 ? q0 : q1;
	else sc = q0 > q1 ? s0 : s1, qc = q0 > q1 ? q0 - q1 : q1 - q0;
}

__device__ __forceinline__ char *pem_put(char *p, const char *s, i64 n) { for (i64 k = 0; k < n; ++k) p[k] = s[k]; return p + n; }

/* one read as print_bseq prints it (pemerge.c:147-158): rn 1 or 2 -> "/1" "/2", 0 -> " merged"; returns its size */
__device__ i64 pem_read(const PemArgs &a, int r, int rn, char *p)
{
	const i64 o = a.off[r], l = a.off[r + 1] - o, nb = a.name_off[r], nl = a.name_off[r + 1] - nb;
	const int hq = a.has_qual[r];
	const i64 size = 1 + nl + (rn ? 3 : 8) + l + 1 + (hq ? 3 + l : 0);
	if (!p) return size;
	*p++ = hq ? '@' : '>';
	p = pem_put(p, a.names + nb, nl);
	if (rn) { *p++ = '/'; *p++ = (char)('0' + rn); *p++ = '\n'; }
	else p = pem_put(p, " merged\n", 8);
	p = pem_put(p, (const char *)a.raw + o, l);
	*p++ = '\n';
	if (hq) { *p++ = '+'; *p++ = '\n'; p = pem_put(p, (const char *)a.qual + o, l); *p++ = '\n'; }
	return size;
}

__global__ void k_pem_text(PemArgs a, int write)
{
	__shared__ unsigned cnt[9];
	if (!write && threadIdx.x < 9) cnt[threadIdx.x] = 0;
	__syncthreads();
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n_pairs; i += gridDim.x * blockDim.x) {
		const i64 o0 = a.off[2 * i], o1 = a.off[2 * i + 1];
		const int l0 = (int)(o1 - o0), l1 = (int)(a.off[2 * i + 2] - o1), lm = a.ovl[i];
		int code = a.code[i];
		i64 size = 0;
		char *p = write ? a.text + a.tbeg[i] : 0;
		if (!write && code == 0) {   /* sum_q over the overlap's mismatches, both bases called (pemerge.c:114-132) */
			int sum_q = 0;
			for (int k = 0; k < lm; ++k) {
				const int s0 = a.s[o0 + l0 - lm + k], s1 = a.s[o1 + k], q0 = a.q[o0 + l0 - lm + k], q1 = a.q[o1 + k];
				if (s0 == 4 || s1 == 4 || s0 == s1) continue;
				const int qq = q0 < q1 ? q0 : q1;
				sum_q += qq >= 3 ? qq << 1 : 1;
			}
			if (sum_q >> 1 > a.q_thres) code = -8;
			a.code[i] = (int8_t)code;
		}
		if (!write && code <= 0) atomicAdd(&cnt[-code], 1u);
		if (code == 0 || l1 == 0) {   /* the printing loop asks whether read 2 is empty (pemerge.c:203), which a merge makes it */
			if (a.flag & 1) {
				if (code == 0) {   /* "@name merged", the merged read; its quality string ends at a byte that wrapped to 0 */
					const int l_seq = l0 + l1 - lm;
					int nq = 0;
					while (nq < l_seq) { int sc, qc; pem_merged(a, o0, o1, l0, lm, nq, sc, qc); if ((uint8_t)(qc + 33) == 0) break; ++nq; }
					const i64 nb = a.name_off[2 * i], nl = a.name_off[2 * i + 1] - nb;
					size = 1 + nl + 8 + l_seq + 3 + nq + 1;
					if (p) {
						*p++ = '@';
						p = pem_put(p, a.names + nb, nl);
						p = pem_put(p, " merged\n", 8);
						for (int k = 0; k < l_seq; ++k) { int sc, qc; pem_merged(a, o0, o1, l0, lm, k, sc, qc); *p++ = "ACGTN"[sc]; }
						p = pem_put(p, "\n+\n", 3);
						for (int k = 0; k < nq; ++k) { int sc, qc; pem_merged(a, o0, o1, l0, lm, k, sc, qc); *p++ = (char)(uint8_t)(qc + 33); }
						*p++ = '\n';
					}
				} else size = pem_read(a, 2 * i, 0, p);   /* read 2 is empty: read 1 as it came, called merged */
			}
		} else if (a.flag & 2) {
			size = pem_read(a, 2 * i, 1, p);
			size += pem_read(a, 2 * i + 1, 2, p ? p + size : 0);
		}
		if (!write) a.tlen[i] = size;
	}
	if (!write) {
		__syncthreads();
		if (threadIdx.x < 9 && cnt[threadIdx.x]) atomicAdd(&a.cnt[threadIdx.x], (u64)cnt[threadIdx.x]);
	}
}

/* ------------------------------------------------------------------------------------------------ host driver */

/* M1, K6, M2/M3, then M4 around a scan */
extern "C" int bwag_pemerge(bwag_batch_t *b, const bwag_pemerge_par_t *par, bwag_pemerge_t *out)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	memset(out, 0, sizeof(*out));
	const int n = b->n;
	if (n & 1) return set_err("bwag_pemerge: a batch of %d reads is not a batch of pairs", n);
	const int np = n >> 1;
	const i64 nb = b->total_bases, nn = par->name_off[n];
	int max_q = 16, max_t = 16;
	for (int i = 0; i < np; ++i) {
		const int l0 = (int)(b->h_off[2 * i + 1] - b->h_off[2 * i]), l1 = (int)(b->h_off[2 * i + 2] - b->h_off[2 * i + 1]);
		if (l0 > max_t) max_t = l0;
		if (l1 > max_q) max_q = l1;
	}
	if (buf_reserve(&b->d_pm_qual, (size_t)nb + 16) || buf_reserve(&b->d_pm_hasq, (size_t)n + 16) || buf_reserve(&b->d_pm_names, (size_t)nn + 16) ||
	    buf_reserve(&b->d_pm_noff, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_swpool, (size_t)nb + 16) || buf_reserve(&b->d_pm_q, (size_t)nb + 16) ||
	    buf_reserve(&b->d_swtasks, sizeof(bwag_swtask_t) * ((size_t)np + 1)) || buf_reserve(&b->d_pm_code, (size_t)np + 16) || buf_reserve(&b->d_pm_ovl, 4 * ((size_t)np + 1)) ||
	    buf_reserve(&b->d_pm_tlen, 8 * ((size_t)np + 1)) || buf_reserve(&b->d_pm_tbeg, 8 * ((size_t)np + 1)) || buf_reserve(&b->d_pm_cnt, 8 * 9) ||
	    hbuf_reserve(&b->h_pm_cnt, 8 * 9)) return 1;
	PemArgs a;
	memset(&a, 0, sizeof(a));
	a.n_pairs = np; a.T = par->T; a.q_thres = par->q_thres; a.q_def = par->q_def; a.flag = par->flag;
	a.raw = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p;
	a.qual = (const uint8_t *)b->d_pm_qual.p; a.has_qual = (const uint8_t *)b->d_pm_hasq.p;
	a.names = (const char *)b->d_pm_names.p; a.name_off = (const i64 *)b->d_pm_noff.p;
	a.s = (uint8_t *)b->d_swpool.p; a.q = (uint8_t *)b->d_pm_q.p; a.tasks = (bwag_swtask_t *)b->d_swtasks.p;
	a.code = (int8_t *)b->d_pm_code.p; a.ovl = (int *)b->d_pm_ovl.p;
	a.tlen = (i64 *)b->d_pm_tlen.p; a.tbeg = (const i64 *)b->d_pm_tbeg.p; a.cnt = (u64 *)b->d_pm_cnt.p;
	if (reset_counters(c)) return 1;
	if (nb) H2D(c, b->d_pm_qual.p, par->qual, (size_t)nb);
	if (n) H2D(c, b->d_pm_hasq.p, par->has_qual, (size_t)n);
	if (nn) H2D(c, b->d_pm_names.p, par->names, (size_t)nn);
	H2D(c, b->d_pm_noff.p, par->name_off, 8 * ((size_t)n + 1));
	CK(cudaMemsetAsync(b->d_pm_cnt.p, 0, 8 * 9, c->stream));
	if (np) BWAG_LAUNCH(k_pem_encode, fm_grid(b->ctx, np), 128, 0, c->stream, a);
	CK(cudaGetLastError());
	++c->st.n_launch;
	if (par->merge && np) {
		bwag_sw_par_t sp;   /* ksw_align(l2, s1, l1, s0, 5, bwa_fill_scmat(5, 4), 2, 17, xtra): the same gaps for deletions and insertions */
		memset(&sp, 0, sizeof(sp));
		sp.a = 5; sp.b = 4; sp.o_del = sp.o_ins = 2; sp.e_del = sp.e_ins = 17;
		for (int i = 0; i < 5; ++i) for (int j = 0; j < 5; ++j) sp.mat[i * 5 + j] = (int8_t)(i < 4 && j < 4 ? (i == j ? 5 : -4) : -1);
		if (localsw_on_device(b, &sp, np, max_q, max_t)) return 1;
		a.res = (const bwag_swres_t *)b->d_swres.p;
		const i64 blocks = ((i64)np + 3) / 4, cap = (i64)b->ctx->n_sm * 16;
		BWAG_LAUNCH(k_pem_decide, (int)(blocks < cap ? blocks : cap), 128, 0, c->stream, a);
		CK(cudaGetLastError());
		if (fetch_counters(c)) return 1;
		c->st.ms_localsw += elapsed_at(c, "localsw", __FILE__, __LINE__); c->st.n_launch += 2; c->st.sw_tasks += (u64)np;
		if (c->h_cnt->flags & 32u) return set_err("pemerge: a local alignment exceeded the scratch capacity");
	}
	/* M4: sizes, their scan, then the text */
	if (np) BWAG_LAUNCH(k_pem_text, fm_grid(b->ctx, np), 128, 0, c->stream, a, 0);
	BWAG_LAUNCH(k_fm_scan64, 1, FM_SCAN_THREADS, 0, c->stream, (const i64 *)b->d_pm_tlen.p, (i64)np, (i64 *)b->d_pm_tbeg.p, &c->d_cnt->pm_total);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	c->st.n_launch += 2;
	const i64 n_text = (i64)c->h_cnt->pm_total;
	if (buf_reserve(&b->d_pm_text, (size_t)n_text + 16) || hbuf_reserve(&b->h_pm_text, (size_t)n_text + 16)) return 1;
	a.text = (char *)b->d_pm_text.p;
	if (np) BWAG_LAUNCH(k_pem_text, fm_grid(b->ctx, np), 128, 0, c->stream, a, 1);
	CK(cudaGetLastError());
	++c->st.n_launch;
	if (n_text) D2H(c, b->h_pm_text.p, b->d_pm_text.p, (size_t)n_text);
	D2H(c, b->h_pm_cnt.p, b->d_pm_cnt.p, 8 * 9);
	CK(stream_wait(c));
	out->text = (const char *)b->h_pm_text.p; out->n_text = n_text;
	memcpy(out->cnt, b->h_pm_cnt.p, 8 * 9);
	return 0;
}
