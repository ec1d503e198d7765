/* bwag_fastmap.cu -- `bwa-b200 fastmap` after K1 (k_smem_fm): the reference positions of each listed SMEM and the EM lines of
 * fastmap.c:457-473, as text, on the device.
 *
 * K1 leaves each read's matches as a slice of the batch-wide interval pool, in the reference's order; the slices lie in the pool in
 * the order the reads finished.  From there:
 *   F1  k_fm_lines    one lane per read: the read's matches move to read order (line L = one EM line), and each line asks for x[2]
 *                     suffix-array rows if x[2] <= w, none otherwise;
 *   F2  k_fm_rows     one lane per line: rows x[0], x[0]+1, ... at the line's offset (an exclusive scan of the requests), which K2
 *                     (k_sa) resolves to text positions in place;
 *   F3  k_fm_text     one lane per line, twice: first the exact byte length of the line (decimal widths, contig name lengths),
 *                     then, after a scan, the line itself.
 * One lane per LINE, not per read: a read whose matches list thousands of positions (-w -1 on a repeat) keeps one lane busy, not
 * a warp.  The scans are one block each (k_fm_scan); every buffer is sized from a scan's total, so nothing can overflow. */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"
#include "bwag_drv.h"

/* exclusive prefix sum of in[0..n) into out[0..n], out[n] = *total = the sum; one block of FM_SCAN_THREADS, tiles of 4 per lane */
template <typename T>
__device__ __forceinline__ void fm_scan(const T *in, i64 n, i64 *out, u64 *total)
{
	__shared__ i64 wsum[FM_SCAN_THREADS / 32];
	__shared__ i64 tile_sum;
	const int t = threadIdx.x, lane = t & 31, w = t >> 5;
	i64 carry = 0;
	for (i64 base = 0; base < n; base += 4 * FM_SCAN_THREADS) {
		i64 v[4], s = 0;
		for (int k = 0; k < 4; ++k) { const i64 idx = base + 4 * (i64)t + k; v[k] = idx < n ? (i64)in[idx] : 0; s += v[k]; }
		i64 inc = s;
		for (int d = 1; d < 32; d <<= 1) { const i64 y = __shfl_up_sync(FULL_MASK, inc, d); if (lane >= d) inc += y; }
		if (lane == 31) wsum[w] = inc;
		__syncthreads();
		if (w == 0) {
			const i64 ws = lane < FM_SCAN_THREADS / 32 ? wsum[lane] : 0;
			i64 wi = ws;
			for (int d = 1; d < 32; d <<= 1) { const i64 y = __shfl_up_sync(FULL_MASK, wi, d); if (lane >= d) wi += y; }
			if (lane < FM_SCAN_THREADS / 32) wsum[lane] = wi - ws;
			if (lane == 31) tile_sum = wi;
		}
		__syncthreads();
		i64 run = carry + wsum[w] + inc - s;
		for (int k = 0; k < 4; ++k) { const i64 idx = base + 4 * (i64)t + k; if (idx < n) out[idx] = run; run += v[k]; }
		carry += tile_sum;
		__syncthreads();
	}
	if (t == 0) { out[n] = carry; *total = (u64)carry; }
}
__global__ void __launch_bounds__(FM_SCAN_THREADS) k_fm_scan32(const int *in, i64 n, i64 *out, u64 *total) { fm_scan(in, n, out, total); }
__global__ void __launch_bounds__(FM_SCAN_THREADS) k_fm_scan64(const i64 *in, i64 n, i64 *out, u64 *total) { fm_scan(in, n, out, total); }

/* F1: read r's matches to lines lbeg[r] ..; rows wanted per line */
__global__ void k_fm_lines(FmArgs a)
{
	for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_reads; r += gridDim.x * blockDim.x) {
		const int n = a.intv_n[r];
		const bwtintv_t *src = a.intv + a.intv_beg[r];
		const i64 l0 = a.lbeg[r];
		for (int e = 0; e < n; ++e) {
			const bwtintv_t p = src[e];
			a.lines[l0 + e] = p;
			a.nrow[l0 + e] = (i64)(p.x[2] <= a.max_iwidth ? p.x[2] : 0);   /* fastmap.c:462: x[2] <= (uint64)w */
		}
	}
}

/* F2: the BWT rows of line L, for K2 */
__global__ void k_fm_rows(FmArgs a)
{
	for (i64 L = (i64)blockIdx.x * blockDim.x + threadIdx.x; L < a.n_lines; L += (i64)gridDim.x * blockDim.x) {
		const i64 o = a.rbeg[L], m = a.rbeg[L + 1] - o;
		const u64 x0 = a.lines[L].x[0];
		for (i64 k = 0; k < m; ++k) a.rows[o + k] = (i64)(x0 + (u64)k);
	}
}

__device__ __forceinline__ int fm_dec_len(u64 v) { int n = 1; while (v >= 10) { v /= 10; ++n; } return n; }
__device__ __forceinline__ char *fm_dec(char *p, u64 v)
{
	const int n = fm_dec_len(v);
	for (int k = n - 1; k >= 0; --k) { p[k] = (char)('0' + (int)(v % 10)); v /= 10; }
	return p + n;
}

/* position k of line L: contig, strand and 1-based coordinate as fastmap.c:466-469 prints them (bns_depos, pos -= len-1 on the
 * reverse strand, bns_pos2rid through bns_cnt_ambi) */
__device__ __forceinline__ void fm_pos(const FmArgs &a, i64 sa, int len, int &rid, int &rev, u64 &coord)
{
	rev = sa >= a.ctg.l_pac;
	i64 pos = rev ? (a.ctg.l_pac << 1) - 1 - sa : sa;
	if (rev) pos -= len - 1;
	rid = t_pos2rid(a.ctg, pos);
	coord = (u64)(pos - a.ctg.off[rid]) + 1;
}

/* F3: write = 0: tlen[L] = bytes of line L; write = 1: the line at tbeg[L] */
__global__ void k_fm_text(FmArgs a, int write)
{
	for (i64 L = (i64)blockIdx.x * blockDim.x + threadIdx.x; L < a.n_lines; L += (i64)gridDim.x * blockDim.x) {
		const bwtintv_t p = a.lines[L];
		const u32 beg = (u32)(p.info >> 32), end = (u32)p.info;
		const int len = (int)(end - beg);
		const i64 r0 = a.rbeg[L], m = a.rbeg[L + 1] - r0;
		const bool listed = p.x[2] <= a.max_iwidth;
		if (!write) {
			i64 b = 3 + fm_dec_len(beg) + 1 + fm_dec_len(end) + 1 + fm_dec_len(p.x[2]) + 1 + (listed ? 0 : 3);
			for (i64 k = 0; k < m; ++k) {
				int rid, rev; u64 coord;
				fm_pos(a, a.rows[r0 + k], len, rid, rev, coord);
				b += 1 + (a.ctg.name_off[rid + 1] - a.ctg.name_off[rid]) + 2 + fm_dec_len(coord);
			}
			a.tlen[L] = b;
		} else {
			char *q = a.text + a.tbeg[L];
			*q++ = 'E'; *q++ = 'M'; *q++ = '\t';
			q = fm_dec(q, beg); *q++ = '\t';
			q = fm_dec(q, end); *q++ = '\t';
			q = fm_dec(q, p.x[2]);
			for (i64 k = 0; k < m; ++k) {
				int rid, rev; u64 coord;
				fm_pos(a, a.rows[r0 + k], len, rid, rev, coord);
				*q++ = '\t';
				for (int c = a.ctg.name_off[rid]; c < a.ctg.name_off[rid + 1]; ++c) *q++ = a.ctg.names[c];
				*q++ = ':'; *q++ = rev ? '-' : '+';
				q = fm_dec(q, coord);
			}
			if (!listed) { *q++ = '\t'; *q++ = '*'; *q++ = '\n'; }   /* err_puts("\t*") brings its own newline */
			*q++ = '\n';
		}
	}
}

/* per read: its text starts where its first line does (lbeg[n_reads] = n_lines, so off[n_reads] = the total) */
__global__ void k_fm_readoff(FmArgs a)
{
	for (int r = blockIdx.x * blockDim.x + threadIdx.x; r <= a.n_reads; r += gridDim.x * blockDim.x) a.toff[r] = a.tbeg[a.lbeg[r]];
}

/* ------------------------------------------------------------------------------------------------ host driver */

/* K1 in its fastmap form, then F1-F3 with K2 between them; every buffer sized from a scan's total */
extern "C" int bwag_fastmap(bwag_batch_t *b, const bwag_fastmap_par_t *par, bwag_fastmap_t *out)
{
	Lane *c = &b->lane;
	const bwag_ctx_t *pc = b->ctx;
	CK(cudaSetDevice(pc->device));
	if (!pc->have_ctg) return set_err("bwag_fastmap needs the contig table (bwag_ctx_set_contigs)");
	const int n = b->n;
	for (int r = 0; r < n; ++r)
		if (b->h_off[r + 1] - b->h_off[r] >= (1 << 23)) return set_err("read %d of the batch has %lld bases; reads of 2^23 bases or more are not supported", r, (long long)(b->h_off[r + 1] - b->h_off[r]));
	bwag_seed_par_t sp;
	memset(&sp, 0, sizeof(sp));
	sp.min_seed_len = par->min_len;
	const FmK1 fm = { par->min_intv < 1 ? 1 : par->min_intv, par->max_intv };
	if (seed_impl(b, &sp, &fm, 0)) return 1;
	const i64 n_lines = b->n_intv;
	if (buf_reserve(&b->d_fm_lbeg, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_fm_toff, 8 * ((size_t)n + 1)) ||
	    buf_reserve(&b->d_fm_lines, sizeof(bwtintv_t) * ((size_t)n_lines + 1)) || buf_reserve(&b->d_fm_nrow, 8 * ((size_t)n_lines + 1)) ||
	    buf_reserve(&b->d_fm_rbeg, 8 * ((size_t)n_lines + 1)) || buf_reserve(&b->d_fm_tlen, 8 * ((size_t)n_lines + 1)) || buf_reserve(&b->d_fm_tbeg, 8 * ((size_t)n_lines + 1)) ||
	    hbuf_reserve(&b->h_fm_off, 8 * ((size_t)n + 1))) return 1;
	FmArgs f;
	memset(&f, 0, sizeof(f));
	f.n_reads = n; f.n_lines = n_lines; f.max_iwidth = (u64)(i64)par->max_iwidth; f.ctg = pc->tctg;
	f.intv_beg = (const i64 *)b->d_intv_beg.p; f.intv_n = (const int *)b->d_intv_n.p; f.intv = (const bwtintv_t *)b->d_intv.p;
	f.lbeg = (const i64 *)b->d_fm_lbeg.p; f.lines = (bwtintv_t *)b->d_fm_lines.p; f.nrow = (i64 *)b->d_fm_nrow.p; f.rbeg = (const i64 *)b->d_fm_rbeg.p;
	f.tlen = (i64 *)b->d_fm_tlen.p; f.tbeg = (const i64 *)b->d_fm_tbeg.p; f.toff = (i64 *)b->d_fm_toff.p;
	/* F1: read order, rows wanted per line, their scan */
	BWAG_LAUNCH(k_fm_scan32, 1, FM_SCAN_THREADS, 0, c->stream, (const int *)b->d_intv_n.p, (i64)n, (i64 *)b->d_fm_lbeg.p, &c->d_cnt->fm_total[0]);
	BWAG_LAUNCH(k_fm_lines, fm_grid(b->ctx, n), 128, 0, c->stream, f);
	BWAG_LAUNCH(k_fm_scan64, 1, FM_SCAN_THREADS, 0, c->stream, (const i64 *)b->d_fm_nrow.p, n_lines, (i64 *)b->d_fm_rbeg.p, &c->d_cnt->fm_total[1]);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	c->st.n_launch += 3;
	const i64 n_rows = (i64)c->h_cnt->fm_total[1];
	/* F2 + K2: the rows, resolved in place */
	if (buf_reserve(&b->d_fm_rows, 8 * ((size_t)n_rows + 1))) return 1;
	f.rows = (i64 *)b->d_fm_rows.p;
	if (n_rows > 0) {
		BWAG_LAUNCH(k_fm_rows, fm_grid(b->ctx, n_lines), 128, 0, c->stream, f);
		if (run_sa(b, f.rows, n_rows)) return 1;
		c->st.n_launch += 2;
	}
	/* F3: line sizes, their scan, the text, each read's range */
	BWAG_LAUNCH(k_fm_text, fm_grid(b->ctx, n_lines), 128, 0, c->stream, f, 0);
	BWAG_LAUNCH(k_fm_scan64, 1, FM_SCAN_THREADS, 0, c->stream, (const i64 *)b->d_fm_tlen.p, n_lines, (i64 *)b->d_fm_tbeg.p, &c->d_cnt->fm_total[2]);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	if (n_rows > 0) { c->st.ms_sa += elapsed_at(c, "sa", __FILE__, __LINE__); c->st.sa_touches += c->h_cnt->sa_touches; }
	c->st.n_launch += 2;
	const i64 n_text = (i64)c->h_cnt->fm_total[2];
	if (buf_reserve(&b->d_fm_text, (size_t)n_text + 1) || hbuf_reserve(&b->h_fm_text, (size_t)n_text + 1)) return 1;
	f.text = (char *)b->d_fm_text.p;
	BWAG_LAUNCH(k_fm_text, fm_grid(b->ctx, n_lines), 128, 0, c->stream, f, 1);
	BWAG_LAUNCH(k_fm_readoff, fm_grid(b->ctx, (i64)n + 1), 128, 0, c->stream, f);
	CK(cudaGetLastError());
	c->st.n_launch += 2;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_text) D2H(c, b->h_fm_text.p, b->d_fm_text.p, (size_t)n_text);
	D2H(c, b->h_fm_off.p, b->d_fm_toff.p, 8 * ((size_t)n + 1));
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	out->text = (const char *)b->h_fm_text.p; out->off = (const int64_t *)b->h_fm_off.p;
	return 0;
}
