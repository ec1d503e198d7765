/* bwag_index.cu -- construction of the FM-index files (`bwa-b200 index`) on the device: BWT, Occ checkpoints and the sampled
 * suffix array of T = forward + reverse complement of the reference (bwtindex.c:267-274), the same bytes `bwa index` writes.
 *
 * Method.  T (n = 2 l_pac bases) lives packed 16 bases per u32 word in HBM.  Suffixes are bucketed by their first
 * IX_HIST_BASES bases; consecutive buckets are grouped so that one group's (key, position) pairs fit in the free device memory.
 * Per group:
 *   1. k_ix_list   lists the positions of the group (warp-aggregated append; order arbitrary);
 *   2. LSD radix sort (k_rx_hist, scan, k_rx_scatter: 8-bit digits, per-block histograms, stable scatter) of the 64-bit keys
 *      = the first 32 bases (A beyond the end of T), skipping the leading bits that are constant within the group;
 *   3. runs of equal keys are ordered by a merge sort over global memory (k_ix_merge): per pass, every element of a run
 *      finds its place in the partner block by a binary search whose comparisons are made by a warp, 1024 bases per step,
 *      until the first difference or the end of T (a suffix that runs off the end sorts first, as with a terminal '$').
 *      A comparison costs LCP/1024 steps, and a run of any size finishes in log2(run) passes;
 *   4. k_ix_emit writes the group's BWT symbols T[pos-1] and its SA samples (every 32nd row) in place, and records primary.
 * Then the Occ checkpoints every 128 symbols are counted, scanned and interleaved with the symbols (bwt_bwtupdate_core,
 * bwtindex.c:150-172).  Device memory: the packed text (n/4 bytes), one byte per BWT row, the SA sample (n/4 bytes) and one
 * group's working set; nothing of 8 bytes per suffix over the whole text.
 *
 * The same group loop (ix_sort) serves `bwa-b200 pac2bwt`, which sorts a .pac text as it is (k_ix_pack_text) and returns the
 * raw '$'-less BWT of bwt_pac2bwt (k_bw_raw, bwtindex.c:83-145).  `bwa-b200 bwtupdate` adds the Occ checkpoints to such a raw
 * BWT: counts per block straight from the packed words (k_bw_count), scanned, then interleaved (k_bw_write). */
#include "bwag_drv.h"

#define IX_HIST_BASES 6          /* buckets of the planning histogram: 4^6, 16 KB of shared counters */
#define IX_THREADS 256
#define RX_ITEMS 16              /* radix sort: keys per thread and block tile */
#define RX_TILE (IX_THREADS * RX_ITEMS)
#define IX_GROUP_BYTES 56        /* working set per suffix of a group: keys and positions twice, tie lists, run table */
#define IX_SA_INTV 32

static int ix_clz64_host(u64 x) { return x ? __builtin_clzll(x) : 64; }
#define IXCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { rc = set_err("%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); goto done; } } while (0)

/* ------------------------------------------------------------------------------------------------ device helpers */

__device__ __forceinline__ int ix_clz64(u64 x) { return (x >> 32) ? __clz((int)(u32)(x >> 32)) : 32 + __clz((int)(u32)x); }

/* the 32 bases of T at q..q+31, first base in the top bits; words beyond the text are zero (A), so the key is A-padded */
__device__ __forceinline__ u64 ix_window(const u32 *W, u64 q)
{
	const u64 w0 = q >> 4;
	const int s = (int)(q & 15) << 1;
	u64 v = (u64)W[w0] << 32 | W[w0 + 1];
	if (s) v = v << s | W[w0 + 2] >> (32 - s);
	return v;
}
__device__ __forceinline__ int ix_base(const u32 *W, u64 q) { return W[q >> 4] >> ((15 - (int)(q & 15)) << 1) & 3; }

/* order of the suffixes at a != b: -1 if suffix a sorts first.  Lane l looks at bases [off + 32 l, off + 32 l + 32) of both,
 * so the warp advances 1024 bases per step; the first lane with a difference or an end of text decides.  Warp-uniform a, b. */
__device__ int ix_cmp_warp(const u32 *W, u64 n, u64 a, u64 b)
{
	const int lane = threadIdx.x & 31;
	for (u64 off = (u64)lane << 5;; off += 1024) {
		const u64 qa = a + off, qb = b + off;
		const u64 ra = qa < n ? n - qa : 0, rb = qb < n ? n - qb : 0;   /* bases left in each suffix */
		const u64 wa = ra ? ix_window(W, qa) : 0, wb = rb ? ix_window(W, qb) : 0;
		const int ea = ra < 32 ? (int)ra : 32, eb = rb < 32 ? (int)rb : 32;
		int ev = (wa ^ wb) ? ix_clz64(wa ^ wb) >> 1 : 32;
		ev = min(ev, min(ea, eb));
		const unsigned bal = __ballot_sync(FULL_MASK, ev < 32);
		if (bal) {
			int r;
			if (ea == ev) r = -1;              /* a ends first: the shorter suffix is the smaller one */
			else if (eb == ev) r = 1;
			else r = (int)(wa >> (62 - 2 * ev) & 3) < (int)(wb >> (62 - 2 * ev) & 3) ? -1 : 1;
			return __shfl_sync(FULL_MASK, r, __ffs((int)bal) - 1);
		}
	}
}

/* ------------------------------------------------------------------------------------------------ kernels */

/* T word w = bases 16w..16w+15: forward from the 2-bit pac, then the reverse complement, zero beyond n */
__global__ void k_ix_pack(const uint8_t *pac, i64 l_pac, u64 n, u32 *W, u64 nw)
{
	for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += (u64)gridDim.x * blockDim.x) {
		u32 v = 0;
		for (int j = 0; j < 16; ++j) {
			const u64 q = (w << 4) + j;
			int c = 0;
			if (q < (u64)l_pac) c = bwag_pac_base(pac, (i64)q);
			else if (q < n) c = 3 - bwag_pac_base(pac, (i64)(n - 1 - q));
			v |= (u32)c << ((15 - j) << 1);
		}
		W[w] = v;
	}
}

/* suffixes per bucket of the first kb bases (kb <= IX_HIST_BASES) */
__global__ void k_ix_hist(const u32 *W, u64 n, int kb, u64 *cnt)
{
	__shared__ u32 h[1 << (2 * IX_HIST_BASES)];
	const int nb = 1 << (2 * kb);
	for (int i = threadIdx.x; i < nb; i += blockDim.x) h[i] = 0;
	__syncthreads();
	for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (u64)gridDim.x * blockDim.x)
		atomicAdd(&h[ix_window(W, p) >> (64 - 2 * kb)], 1u);
	__syncthreads();
	for (int i = threadIdx.x; i < nb; i += blockDim.x) if (h[i]) atomicAdd(&cnt[i], (u64)h[i]);
}

/* the positions whose bucket lies in [lo, hi), with their keys */
__global__ void k_ix_list(const u32 *W, u64 n, int kb, u32 lo, u32 hi, u64 *keys, u64 *pos, u64 *counter)
{
	const int lane = threadIdx.x & 31;
	const u64 stride = (u64)gridDim.x * blockDim.x;
	for (u64 p0 = (u64)blockIdx.x * blockDim.x; p0 < n; p0 += stride) {   /* warp-uniform trip count */
		const u64 p = p0 + threadIdx.x;
		u64 key = 0;
		bool in = false;
		if (p < n) { key = ix_window(W, p); const u32 b = (u32)(key >> (64 - 2 * kb)); in = b >= lo && b < hi; }
		const unsigned bal = __ballot_sync(FULL_MASK, in);
		if (!bal) continue;
		u64 base = 0;
		const int leader = __ffs((int)bal) - 1;
		if (lane == leader) base = atomicAdd(counter, (u64)__popc(bal));
		base = __shfl_sync(FULL_MASK, base, leader);
		if (in) { const u64 slot = base + __popc(bal & ((1u << lane) - 1)); keys[slot] = key; pos[slot] = p; }
	}
}

/* LSD radix sort, one 8-bit digit per pass.  bh[d * nblk + b]: keys of tile b with digit d (then scanned to output offsets) */
__global__ void k_rx_hist(const u64 *keys, u64 m, int shift, u64 *bh, u64 nblk)
{
	__shared__ u32 h[256];
	h[threadIdx.x] = 0;
	__syncthreads();
	const u64 base = (u64)blockIdx.x * RX_TILE;
	for (int k = 0; k < RX_ITEMS; ++k) {
		const u64 i = base + (u64)k * IX_THREADS + threadIdx.x;
		if (i < m) atomicAdd(&h[keys[i] >> shift & 255], 1u);
	}
	__syncthreads();
	bh[(u64)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];
}

/* stable scatter of tile b: rounds of 256 keys in input order; inside a round, keys with equal digits are ranked by warp and
 * lane (8 ballots give each lane the lanes of its warp with the same digit), warps in order through a per-digit prefix */
__global__ void k_rx_scatter(const u64 *kin, const u64 *vin, u64 *kout, u64 *vout, u64 m, int shift, const u64 *bh, u64 nblk)
{
	__shared__ u32 wc[IX_THREADS / 32][256];
	__shared__ u64 dbase[256];
	const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
	dbase[t] = bh[(u64)t * nblk + blockIdx.x];
	const u64 base = (u64)blockIdx.x * RX_TILE;
	for (int k = 0; k < RX_ITEMS; ++k) {
		for (int w = 0; w < IX_THREADS / 32; ++w) wc[w][t] = 0;
		__syncthreads();
		const u64 i = base + (u64)k * IX_THREADS + t;
		const bool valid = i < m;
		u64 key = 0, val = 0;
		int d = 0;
		if (valid) { key = kin[i]; val = vin[i]; d = (int)(key >> shift & 255); }
		unsigned peers = __ballot_sync(FULL_MASK, valid);
		for (int bit = 0; bit < 8; ++bit) {
			const unsigned bb = __ballot_sync(FULL_MASK, d >> bit & 1);
			peers &= (d >> bit & 1) ? bb : ~bb;
		}
		const int rank = __popc(peers & ((1u << lane) - 1));
		if (valid && rank == 0) wc[warp][d] = (u32)__popc(peers);
		__syncthreads();
		u32 s = 0;
		for (int w = 0; w < IX_THREADS / 32; ++w) { const u32 c = wc[w][t]; wc[w][t] = s; s += c; }
		__syncthreads();
		if (valid) { const u64 o = dbase[d] + wc[warp][d] + rank; kout[o] = key; vout[o] = val; }
		__syncthreads();
		dbase[t] += s;
	}
}

/* exclusive scan of d[0..n) in segments of IX_THREADS; part[b] = total of segment b */
__global__ void k_scan_seg(u64 *d, u64 n, u64 *part)
{
	__shared__ u64 ws[IX_THREADS / 32];
	const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
	const u64 i = (u64)blockIdx.x * IX_THREADS + t;
	const u64 v = i < n ? d[i] : 0;
	u64 x = v;
	for (int o = 1; o < 32; o <<= 1) { const u64 y = __shfl_up_sync(FULL_MASK, x, o); if (lane >= o) x += y; }
	if (lane == 31) ws[warp] = x;
	__syncthreads();
	if (warp == 0) {
		u64 z = lane < IX_THREADS / 32 ? ws[lane] : 0;
		for (int o = 1; o < 32; o <<= 1) { const u64 y = __shfl_up_sync(FULL_MASK, z, o); if (lane >= o) z += y; }
		if (lane < IX_THREADS / 32) ws[lane] = z;
	}
	__syncthreads();
	const u64 before = (warp ? ws[warp - 1] : 0) + x - v;
	if (i < n) d[i] = before;
	if (t == IX_THREADS - 1) part[blockIdx.x] = ws[IX_THREADS / 32 - 1];
}
__global__ void k_scan_add(u64 *d, u64 n, const u64 *part)
{
	const u64 i = (u64)blockIdx.x * IX_THREADS + threadIdx.x;
	if (i < n) d[i] += part[blockIdx.x];
}

/* runs of equal keys of length >= 2: (start, length, first slot in the tie list) */
__global__ void k_ix_runs(const u64 *keys, u64 m, u64 *run_start, u64 *run_len, u64 *run_off, u64 *cnt /* n_runs, n_tied, max_len */)
{
	for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i + 1 < m; i += (u64)gridDim.x * blockDim.x) {
		const u64 k = keys[i];
		if ((i && keys[i - 1] == k) || keys[i + 1] != k) continue;
		u64 j = i + 2;
		while (j < m && keys[j] == k) ++j;
		const u64 r = atomicAdd(&cnt[0], 1ull);
		run_start[r] = i; run_len[r] = j - i;
		run_off[r] = atomicAdd(&cnt[1], j - i);
		atomicMax(&cnt[2], j - i);
	}
}
__global__ void k_ix_ties(const u64 *run_start, const u64 *run_len, const u64 *run_off, u64 n_runs, u64 *e_slot, u32 *e_run)
{
	for (u64 r = blockIdx.x; r < n_runs; r += gridDim.x)
		for (u64 x = threadIdx.x; x < run_len[r]; x += blockDim.x) { e_slot[run_off[r] + x] = run_start[r] + x; e_run[run_off[r] + x] = (u32)r; }
}

/* one merge pass of width w over every run: the element at rank `own` of its block goes to
 * (pair base) + own + (elements of the partner block that sort before it); one warp per element */
__global__ void k_ix_merge(const u32 *W, u64 n, const u64 *vin, u64 *vout, const u64 *e_slot, const u32 *e_run,
                           const u64 *run_start, const u64 *run_len, u64 n_tied, u64 w)
{
	const int lane = threadIdx.x & 31;
	const u64 n_warps = ((u64)gridDim.x * blockDim.x) >> 5;
	for (u64 t = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < n_tied; t += n_warps) {
		const u64 i = e_slot[t], s = run_start[e_run[t]], L = run_len[e_run[t]], r = i - s;
		const u64 bi = r / w, own = r - bi * w, ps = (bi ^ 1) * w;
		const u64 me = vin[i];
		u64 np = r;
		if (ps < L) {
			u64 lo = 0, hi = L - ps < w ? L - ps : w;
			while (lo < hi) {
				const u64 mid = (lo + hi) >> 1;
				if (ix_cmp_warp(W, n, vin[s + ps + mid], me) < 0) lo = mid + 1; else hi = mid;
			}
			np = (bi & ~(u64)1) * w + own + lo;
		}
		if (lane == 0) vout[s + np] = me;
	}
}

/* rows row0 .. row0+m-1 of the BWT matrix: their symbol T[pos-1] (the row of suffix 0 is primary) and SA samples */
__global__ void k_ix_emit(const u32 *W, const u64 *pos, u64 m, u64 row0, uint8_t *B, u64 *sa, u64 *primary)
{
	for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (u64)gridDim.x * blockDim.x) {
		const u64 p = pos[i], row = row0 + i;
		if (p == 0) { *primary = row; B[row] = 0; }
		else B[row] = (uint8_t)ix_base(W, p - 1);
		if (row % IX_SA_INTV == 0) sa[row / IX_SA_INTV] = p;
	}
}

/* symbols of each kind in each 128-symbol block of the '$'-less BWT (symbol j = row j, or j+1 from primary on) */
__global__ void k_occ_count(const uint8_t *B, u64 n, u64 primary, u64 *cnt, u64 n_blk)
{
	for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < n_blk; b += (u64)gridDim.x * blockDim.x) {
		u32 c[4] = { 0, 0, 0, 0 };
		const u64 e = (b + 1) * 128 < n ? (b + 1) * 128 : n;
		for (u64 j = b * 128; j < e; ++j) ++c[B[j + (j >= primary)]];
		for (int k = 0; k < 4; ++k) cnt[(u64)k * (n_blk + 1) + b] = c[k];
	}
}

/* the .bwt body: per block 4 x u64 counts before it, then 8 words of 16 symbols (first in the top bits); the last block
 * has only the words its symbols need, and the final counts follow it */
__global__ void k_occ_write(const uint8_t *B, u64 n, u64 primary, const u64 *occ, u64 n_blk, u32 *out)
{
	for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < n_blk; b += (u64)gridDim.x * blockDim.x) {
		u32 *o = out + b * 16;
		for (int k = 0; k < 4; ++k) { const u64 v = occ[(u64)k * (n_blk + 1) + b]; o[2 * k] = (u32)v; o[2 * k + 1] = (u32)(v >> 32); }
		int w;
		for (w = 0; w < 8 && b * 128 + (u64)w * 16 < n; ++w) {
			u32 v = 0;
			for (int s = 0; s < 16; ++s) {
				const u64 j = b * 128 + (u64)w * 16 + s;
				if (j < n) v |= (u32)B[j + (j >= primary)] << ((15 - s) << 1);
			}
			o[8 + w] = v;
		}
		if (b == n_blk - 1)
			for (int k = 0; k < 4; ++k) { const u64 v = occ[(u64)k * (n_blk + 1) + n_blk]; o[8 + w + 2 * k] = (u32)v; o[8 + w + 2 * k + 1] = (u32)(v >> 32); }
	}
}

/* T word w = bases 16w..16w+15 of a .pac text taken as it is (pac2bwt), zero beyond n */
__global__ void k_ix_pack_text(const uint8_t *pac, u64 n, u32 *W, u64 nw)
{
	for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += (u64)gridDim.x * blockDim.x) {
		u32 v = 0;
		for (int j = 0; j < 16; ++j) {
			const u64 q = (w << 4) + j;
			if (q < n) v |= (u32)bwag_pac_base(pac, (i64)q) << ((15 - j) << 1);
		}
		W[w] = v;
	}
}

/* the raw .bwt body of pac2bwt: the '$'-less BWT (symbol j = row j, or j+1 from primary on), 16 symbols per word, first in the
 * top bits, zero beyond n (bwt_pac2bwt, bwtindex.c:138-140) */
__global__ void k_bw_raw(const uint8_t *B, u64 n, u64 primary, u32 *out, u64 nw)
{
	for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += (u64)gridDim.x * blockDim.x) {
		u32 v = 0;
		for (int s = 0; s < 16; ++s) {
			const u64 j = (w << 4) + s;
			if (j < n) v |= (u32)B[j + (j >= primary)] << ((15 - s) << 1);
		}
		out[w] = v;
	}
}

/* symbols of each kind in each 128-symbol block of packed words (16 symbols per word, first in the top bits; symbols from n on
 * are not counted): per word, popcounts of the high bits, the low bits and both */
__global__ void k_bw_count(const u32 *words, u64 n, u64 *cnt, u64 n_blk)
{
	for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < n_blk; b += (u64)gridDim.x * blockDim.x) {
		u32 c[4] = { 0, 0, 0, 0 };
		for (int w = 0; w < 8 && b * 128 + (u64)w * 16 < n; ++w) {
			const u64 left = n - (b * 128 + (u64)w * 16);
			const int m = left < 16 ? (int)left : 16;
			const u32 v = words[b * 8 + w] & (m == 16 ? 0xffffffffu : ~(0xffffffffu >> (2 * m)));
			const u32 nH = __popc(v & 0xaaaaaaaau), nL = __popc(v & 0x55555555u), nT = __popc(v >> 1 & v & 0x55555555u);
			c[0] += m + nT - nH - nL; c[1] += nL - nT; c[2] += nH - nT; c[3] += nT;
		}
		for (int k = 0; k < 4; ++k) cnt[(u64)k * (n_blk + 1) + b] = c[k];
	}
}

/* the updated .bwt body from the raw words: k_occ_write's layout (bwt_bwtupdate_core, bwtindex.c:150-172), the words copied */
__global__ void k_bw_write(const u32 *words, u64 n, const u64 *occ, u64 n_blk, u32 *out)
{
	for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < n_blk; b += (u64)gridDim.x * blockDim.x) {
		u32 *o = out + b * 16;
		for (int k = 0; k < 4; ++k) { const u64 v = occ[(u64)k * (n_blk + 1) + b]; o[2 * k] = (u32)v; o[2 * k + 1] = (u32)(v >> 32); }
		int w;
		for (w = 0; w < 8 && b * 128 + (u64)w * 16 < n; ++w) o[8 + w] = words[b * 8 + w];
		if (b == n_blk - 1)
			for (int k = 0; k < 4; ++k) { const u64 v = occ[(u64)k * (n_blk + 1) + n_blk]; o[8 + w + 2 * k] = (u32)v; o[8 + w + 2 * k + 1] = (u32)(v >> 32); }
	}
}

/* ------------------------------------------------------------------------------------------------ host driver */

static size_t g_ix_cur, g_ix_peak;
static cudaError_t ix_malloc(void **p, size_t bytes)
{
	cudaError_t e = cudaMalloc(p, bytes + 64);
	if (e == cudaSuccess) { g_ix_cur += bytes + 64; if (g_ix_cur > g_ix_peak) g_ix_peak = g_ix_cur; }
	return e;
}
static void ix_free(void *p, size_t bytes) { if (p) { cudaFree(p); g_ix_cur -= bytes + 64; } }

static int ix_grid(u64 items, int n_sm)
{
	const u64 g = (items + IX_THREADS - 1) / IX_THREADS, cap = (u64)n_sm * 16;
	return (int)(g < 1 ? 1 : g < cap ? g : cap);
}

/* exclusive scan of d[0..n) in place (segments of IX_THREADS, recursively over the segment totals) */
static cudaError_t ix_scan(u64 *d, u64 n)
{
	const u64 nseg = (n + IX_THREADS - 1) / IX_THREADS;
	u64 *part = 0;
	cudaError_t e = ix_malloc((void **)&part, (nseg + 1) * 8);
	if (e != cudaSuccess) return e;
	BWAG_LAUNCH(k_scan_seg, (int)nseg, IX_THREADS, 0, 0, d, n, part);
	if (nseg > 1) {
		if ((e = ix_scan(part, nseg)) == cudaSuccess) BWAG_LAUNCH(k_scan_add, (int)nseg, IX_THREADS, 0, 0, d, n, part);
	}
	if (e == cudaSuccess) e = cudaGetLastError();
	ix_free(part, (nseg + 1) * 8);
	return e;
}

extern "C" void bwag_built_index_free(bwag_built_index_t *x)
{
	free(x->bwt); free(x->sa);
	x->bwt = 0; x->sa = 0;
}


/* BWA_B200_INDEX_BUCKET_BASES: the bucket depth of the planning histogram, forced (tests) */
static int ix_bucket_bases(int *kb, int *forced)
{
	const char *env = getenv("BWA_B200_INDEX_BUCKET_BASES");
	*kb = IX_HIST_BASES; *forced = 0;
	if (env && *env) {
		*kb = atoi(env); *forced = 1;
		if (*kb < 1 || *kb > IX_HIST_BASES) return set_err("BWA_B200_INDEX_BUCKET_BASES must lie in 1..%d", IX_HIST_BASES);
	}
	return 0;
}

/* the device that runs a build, made current; its SM count */
static int ix_device(int device, int *n_sm)
{
	int ndev = 0;
	*n_sm = 2;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return set_err("no CUDA device is visible: this library has no CPU path");
	if (device < 0) CK(cudaGetDevice(&device));
	CK(cudaSetDevice(device));
#ifndef BWAG_CUSIM
	{
		cudaDeviceProp prop;
		CK(cudaGetDeviceProperties(&prop, device));
		*n_sm = prop.multiProcessorCount;
	}
#endif
	return 0;
}

/* The group loop: sorts the n + 1 suffixes of the packed text W (n bases, zero words beyond it) and writes each row's BWT symbol
 * to B[row] (B[primary] = 0), every IX_SA_INTV-th row's suffix-array value to SA and the row of suffix 0 to *primary.  Holds
 * the working set of one group of buckets at a time. */
static int ix_sort(const u32 *W, u64 n, int n_sm, int kb, int forced, uint8_t *B, u64 *SA, u64 *primary, u64 *n_groups, u64 *max_group_out)
{
	int rc = 0;
	u64 *dcnt = 0, *hist = 0, *keys0 = 0, *keys1 = 0, *pos0 = 0, *pos1 = 0, *bh = 0, *run_start = 0, *run_len = 0, *run_off = 0, *e_slot = 0;
	u32 *e_run = 0;
	u64 cap = 0, h_hist[1 << (2 * IX_HIST_BASES)], h_cnt[4], row = 1, max_group = 0, nblk_cap = 0;
	size_t free_b = 0, total_b = 0;
	const char *genv = getenv("BWA_B200_INDEX_GROUP_SUFFIXES");
	*n_groups = 0;
	IXCK(ix_malloc((void **)&dcnt, 4 * 8));
	IXCK(cudaMemset(dcnt, 0, 4 * 8));

	/* planning histogram and groups of consecutive buckets */
	IXCK(ix_malloc((void **)&hist, ((u64)1 << (2 * kb)) * 8));
	IXCK(cudaMemset(hist, 0, ((u64)1 << (2 * kb)) * 8));
	BWAG_LAUNCH(k_ix_hist, ix_grid(n, n_sm), IX_THREADS, 0, 0, W, n, kb, hist);
	IXCK(cudaGetLastError());
	IXCK(cudaMemcpy(h_hist, hist, ((u64)1 << (2 * kb)) * 8, cudaMemcpyDeviceToHost));
	ix_free(hist, ((u64)1 << (2 * kb)) * 8); hist = 0;
	IXCK(cudaMemGetInfo(&free_b, &total_b));   /* again: others may have taken memory since the first look */
	if (0.9 * (double)free_b < (double)(64u << 20) + IX_GROUP_BYTES)
		{ rc = set_err("not enough free device memory: %.2f GB are free beside the text, BWT and SA sample", (double)free_b / 1e9); goto done; }
	cap = (u64)((0.9 * (double)free_b - (double)(64u << 20)) / IX_GROUP_BYTES);
	if (genv && *genv) {   /* tests: several groups of many buckets on a small reference */
		const long long g = atoll(genv);
		if (g < 1) { rc = set_err("BWA_B200_INDEX_GROUP_SUFFIXES must be positive"); goto done; }
		if ((u64)g < cap) cap = (u64)g;
	}
	{
		u64 acc = 0;
		for (u32 b = 0; b < (1u << (2 * kb)); ++b) {
			if (h_hist[b] > cap)
				{ rc = set_err("not enough free device memory: the %llu suffixes of one bucket need %.2f GB, %.2f GB are free (or more than BWA_B200_INDEX_GROUP_SUFFIXES)",
				              (unsigned long long)h_hist[b], (double)h_hist[b] * IX_GROUP_BYTES / 1e9, (double)free_b / 1e9); goto done; }
			if (forced || acc + h_hist[b] > cap) acc = 0;
			acc += h_hist[b];
			if (acc > max_group) max_group = acc;
		}
	}
	nblk_cap = (max_group + RX_TILE - 1) / RX_TILE;
	IXCK(ix_malloc((void **)&keys0, max_group * 8)); IXCK(ix_malloc((void **)&keys1, max_group * 8));
	IXCK(ix_malloc((void **)&pos0, max_group * 8)); IXCK(ix_malloc((void **)&pos1, max_group * 8));
	IXCK(ix_malloc((void **)&bh, nblk_cap * 256 * 8));
	IXCK(ix_malloc((void **)&run_start, max_group / 2 * 8)); IXCK(ix_malloc((void **)&run_len, max_group / 2 * 8));
	IXCK(ix_malloc((void **)&run_off, max_group / 2 * 8));
	IXCK(ix_malloc((void **)&e_slot, max_group * 8)); IXCK(ix_malloc((void **)&e_run, max_group * 4));

	/* row 0 is the empty suffix ('$'): its BWT symbol is the last base of T */
	{
		u32 last;
		uint8_t c;
		IXCK(cudaMemcpy(&last, W + (n - 1) / 16, 4, cudaMemcpyDeviceToHost));
		c = (uint8_t)(last >> ((15 - (int)((n - 1) & 15)) << 1) & 3);
		IXCK(cudaMemcpy(B, &c, 1, cudaMemcpyHostToDevice));
		const u64 nn = n;
		IXCK(cudaMemcpy(SA, &nn, 8, cudaMemcpyHostToDevice));
	}
	for (u32 lo = 0, nbk = 1u << (2 * kb); lo < nbk;) {
		u32 hi = lo;
		u64 m = 0;
		while (hi < nbk && (hi == lo || (!forced && m + h_hist[hi] <= cap))) m += h_hist[hi++];
		if (m == 0) { lo = hi; continue; }
		++*n_groups;
		/* 1. list */
		IXCK(cudaMemset(dcnt, 0, 3 * 8));   /* dcnt[3] holds primary */
		BWAG_LAUNCH(k_ix_list, ix_grid(n, n_sm), IX_THREADS, 0, 0, W, n, kb, lo, hi, keys0, pos0, dcnt);
		IXCK(cudaGetLastError());
		IXCK(cudaMemcpy(h_cnt, dcnt, 8, cudaMemcpyDeviceToHost));
		if (h_cnt[0] != m) { rc = set_err("bucket listing found %llu suffixes, expected %llu", (unsigned long long)h_cnt[0], (unsigned long long)m); goto done; }
		/* 2. radix sort on the bits that vary within the group */
		u64 *kin = keys0, *kout = keys1, *vin = pos0, *vout = pos1;
		{
			const u64 first = (u64)lo << (64 - 2 * kb), last = ((u64)(hi - 1) << (64 - 2 * kb)) | (((u64)1 << (64 - 2 * kb)) - 1);
			const int vary = 64 - ix_clz64_host(first ^ last);
			const u64 nblk = (m + RX_TILE - 1) / RX_TILE;
			for (int shift = 0; shift < vary; shift += 8) {
				BWAG_LAUNCH(k_rx_hist, (int)nblk, IX_THREADS, 0, 0, kin, m, shift, bh, nblk);
				IXCK(cudaGetLastError());
				IXCK(ix_scan(bh, nblk * 256));
				BWAG_LAUNCH(k_rx_scatter, (int)nblk, IX_THREADS, 0, 0, kin, vin, kout, vout, m, shift, bh, nblk);
				IXCK(cudaGetLastError());
				u64 *t = kin; kin = kout; kout = t;
				t = vin; vin = vout; vout = t;
			}
		}
		/* 3. runs of equal keys */
		IXCK(cudaMemset(dcnt, 0, 3 * 8));
		BWAG_LAUNCH(k_ix_runs, ix_grid(m, n_sm), IX_THREADS, 0, 0, kin, m, run_start, run_len, run_off, dcnt);
		IXCK(cudaGetLastError());
		IXCK(cudaMemcpy(h_cnt, dcnt, 3 * 8, cudaMemcpyDeviceToHost));
		if (h_cnt[0]) {
			const u64 n_runs = h_cnt[0], n_tied = h_cnt[1], max_len = h_cnt[2];
			BWAG_LAUNCH(k_ix_ties, (int)(n_runs < (u64)n_sm * 64 ? n_runs : (u64)n_sm * 64), IX_THREADS, 0, 0, run_start, run_len, run_off, n_runs, e_slot, e_run);
			IXCK(cudaGetLastError());
			IXCK(cudaMemcpy(vout, vin, m * 8, cudaMemcpyDeviceToDevice));
			for (u64 w = 1; w < max_len; w <<= 1) {
				const u64 warps = n_tied, blocks = (warps * 32 + IX_THREADS - 1) / IX_THREADS, cap_b = (u64)n_sm * 32;
				BWAG_LAUNCH(k_ix_merge, (int)(blocks < cap_b ? blocks : cap_b), IX_THREADS, 0, 0, W, n, vin, vout, e_slot, e_run, run_start, run_len, n_tied, w);
				IXCK(cudaGetLastError());
				u64 *t = vin; vin = vout; vout = t;
			}
		}
		/* 4. BWT symbols and SA samples of rows row .. row+m-1 */
		BWAG_LAUNCH(k_ix_emit, ix_grid(m, n_sm), IX_THREADS, 0, 0, W, vin, m, row, B, SA, dcnt + 3);
		IXCK(cudaGetLastError());
		IXCK(cudaDeviceSynchronize());
		row += m;
		lo = hi;
	}
	if (row != n + 1) { rc = set_err("sorted %llu rows, expected %llu", (unsigned long long)row, (unsigned long long)n + 1); goto done; }
	IXCK(cudaMemcpy(primary, dcnt + 3, 8, cudaMemcpyDeviceToHost));
	*max_group_out = max_group;
done:
	ix_free(dcnt, 32); ix_free(hist, ((u64)1 << (2 * kb)) * 8);
	ix_free(keys0, max_group * 8); ix_free(keys1, max_group * 8); ix_free(pos0, max_group * 8); ix_free(pos1, max_group * 8);
	ix_free(bh, nblk_cap * 256 * 8); ix_free(run_start, max_group / 2 * 8); ix_free(run_len, max_group / 2 * 8); ix_free(run_off, max_group / 2 * 8);
	ix_free(e_slot, max_group * 8); ix_free(e_run, max_group * 4);
	return rc;
}

/* the parts that live through the whole sort must fit with room for at least a small group */
static int ix_fixed_fits(u64 n, u64 nw, u64 n_sa, u64 pac_bytes)
{
	size_t free_b = 0, total_b = 0;
	CK(cudaMemGetInfo(&free_b, &total_b));
	const double fixed = (double)nw * 4 + (double)(n + 1) + (double)n_sa * 8 + (double)pac_bytes;
	if (fixed + (double)(64u << 20) > 0.9 * (double)free_b)
		return set_err("not enough free device memory: the text, BWT and SA sample of %llu bases need %.2f GB, %.2f GB are free",
		               (unsigned long long)n, fixed / 1e9, (double)free_b / 1e9);
	return 0;
}

extern "C" int bwag_index_build(int device, const uint8_t *pac, int64_t l_pac, bwag_built_index_t *out)
{
	int rc = 0, n_sm = 2, kb = IX_HIST_BASES, forced = 0;
	const u64 n = 2 * (u64)l_pac, nw = (n + 15) / 16 + 4, n_sa = (n + IX_SA_INTV) / IX_SA_INTV;
	const u64 n_blk = (n + 127) / 128, bwt_words = (n + 15) / 16 + (n_blk + 1) * 8;
	u32 *W = 0, *obwt = 0;
	uint8_t *dpac = 0, *B = 0;
	u64 *SA = 0, *occ = 0, h_cnt[4], primary = 0;
	g_ix_cur = g_ix_peak = 0;
	memset(out, 0, sizeof(*out));
	if (l_pac <= 0) return set_err("empty reference");
	if (n >= (u64)BWAG_MAX_SB << BWAG_SB_SHIFT) return set_err("reference too large: %llu bases", (unsigned long long)l_pac);
	if (ix_bucket_bases(&kb, &forced) || ix_device(device, &n_sm) || ix_fixed_fits(n, nw, n_sa, (u64)l_pac / 4 + 1)) return 1;
	IXCK(ix_malloc((void **)&W, nw * 4));
	IXCK(cudaMemset(W, 0, nw * 4));
	IXCK(ix_malloc((void **)&dpac, (size_t)l_pac / 4 + 1));
	IXCK(cudaMemcpy(dpac, pac, (size_t)l_pac / 4 + 1, cudaMemcpyHostToDevice));
	BWAG_LAUNCH(k_ix_pack, ix_grid(nw - 4, n_sm), IX_THREADS, 0, 0, dpac, (i64)l_pac, n, W, nw - 4);
	IXCK(cudaGetLastError());
	IXCK(cudaDeviceSynchronize());
	ix_free(dpac, (size_t)l_pac / 4 + 1); dpac = 0;
	IXCK(ix_malloc((void **)&B, n + 1));
	IXCK(ix_malloc((void **)&SA, n_sa * 8));
	if ((rc = ix_sort(W, n, n_sm, kb, forced, B, SA, &primary, (u64 *)&out->n_groups, (u64 *)&out->max_group)) != 0) goto done;
	ix_free(W, nw * 4); W = 0;

	/* Occ checkpoints: counts per block, scanned per symbol (entry n_blk = total), interleaved with the symbols */
	IXCK(ix_malloc((void **)&occ, 4 * (n_blk + 1) * 8));
	IXCK(cudaMemset(occ, 0, 4 * (n_blk + 1) * 8));
	BWAG_LAUNCH(k_occ_count, ix_grid(n_blk, n_sm), IX_THREADS, 0, 0, B, n, primary, occ, n_blk);
	IXCK(cudaGetLastError());
	for (int k = 0; k < 4; ++k) IXCK(ix_scan(occ + (u64)k * (n_blk + 1), n_blk + 1));
	IXCK(ix_malloc((void **)&obwt, bwt_words * 4));
	BWAG_LAUNCH(k_occ_write, ix_grid(n_blk, n_sm), IX_THREADS, 0, 0, B, n, primary, occ, n_blk, obwt);
	IXCK(cudaGetLastError());
	for (int k = 0; k < 4; ++k) IXCK(cudaMemcpy(&h_cnt[k], occ + (u64)k * (n_blk + 1) + n_blk, 8, cudaMemcpyDeviceToHost));
	out->bwt = (uint32_t *)malloc(bwt_words * 4);
	out->sa = (uint64_t *)malloc(n_sa * 8);
	if (!out->bwt || !out->sa) { rc = set_err("out of host memory"); goto done; }
	IXCK(cudaMemcpy(out->bwt, obwt, bwt_words * 4, cudaMemcpyDeviceToHost));
	IXCK(cudaMemcpy(out->sa, SA, n_sa * 8, cudaMemcpyDeviceToHost));
	out->primary = primary; out->seq_len = n; out->bwt_size = bwt_words; out->n_sa = n_sa;
	out->L2[0] = 0;
	for (int k = 0; k < 4; ++k) out->L2[k + 1] = out->L2[k] + h_cnt[k];
done:
	out->peak_device_bytes = g_ix_peak;
	ix_free(W, nw * 4); ix_free(dpac, (size_t)l_pac / 4 + 1); ix_free(B, n + 1); ix_free(SA, n_sa * 8);
	ix_free(occ, 4 * (n_blk + 1) * 8); ix_free(obwt, bwt_words * 4);
	if (rc) bwag_built_index_free(out);
	return rc;
}

/* symbol totals of n packed symbols (L2[1..4] cumulative), by k_bw_count and a scan; occ: 4 (n_blk + 1) words of scratch */
static int ix_totals(const u32 *words, u64 n, int n_sm, u64 *occ, u64 n_blk, u64 L2[5])
{
	u64 h[4];
	CK(cudaMemset(occ, 0, 4 * (n_blk + 1) * 8));
	BWAG_LAUNCH(k_bw_count, ix_grid(n_blk, n_sm), IX_THREADS, 0, 0, words, n, occ, n_blk);
	CK(cudaGetLastError());
	for (int k = 0; k < 4; ++k) CK(ix_scan(occ + (u64)k * (n_blk + 1), n_blk + 1));
	for (int k = 0; k < 4; ++k) CK(cudaMemcpy(&h[k], occ + (u64)k * (n_blk + 1) + n_blk, 8, cudaMemcpyDeviceToHost));
	L2[0] = 0;
	for (int k = 0; k < 4; ++k) L2[k + 1] = L2[k] + h[k];
	return 0;
}

extern "C" int bwag_pac2bwt(int device, const uint8_t *pac, uint64_t n, bwag_raw_bwt_t *out)
{
	int rc = 0, n_sm = 2, kb = IX_HIST_BASES, forced = 0;
	const u64 nw = (n + 15) / 16 + 4, n_sa = (n + IX_SA_INTV) / IX_SA_INTV, pac_bytes = (n + 3) / 4, n_blk = (n + 127) / 128;
	u32 *W = 0, *raw = 0;
	uint8_t *dpac = 0, *B = 0;
	u64 *SA = 0, *occ = 0, primary = 0, n_groups = 0, max_group = 0;
	g_ix_cur = g_ix_peak = 0;
	memset(out, 0, sizeof(*out));
	if (n == 0) return set_err("empty text");
	if (n >= (u64)BWAG_MAX_SB << BWAG_SB_SHIFT) return set_err("text too large: %llu bases, this build takes fewer than %llu", (unsigned long long)n, (unsigned long long)BWAG_MAX_SB << BWAG_SB_SHIFT);
	if (ix_bucket_bases(&kb, &forced) || ix_device(device, &n_sm) || ix_fixed_fits(n, nw, n_sa, pac_bytes + 4 * (n_blk + 1) * 8)) return 1;
	IXCK(ix_malloc((void **)&W, nw * 4));
	IXCK(cudaMemset(W, 0, nw * 4));
	IXCK(ix_malloc((void **)&dpac, pac_bytes));
	IXCK(cudaMemcpy(dpac, pac, pac_bytes, cudaMemcpyHostToDevice));
	BWAG_LAUNCH(k_ix_pack_text, ix_grid(nw - 4, n_sm), IX_THREADS, 0, 0, dpac, n, W, nw - 4);
	IXCK(cudaGetLastError());
	IXCK(cudaDeviceSynchronize());
	ix_free(dpac, pac_bytes); dpac = 0;
	IXCK(ix_malloc((void **)&occ, 4 * (n_blk + 1) * 8));
	if ((rc = ix_totals(W, n, n_sm, occ, n_blk, (u64 *)out->L2)) != 0) goto done;   /* the BWT holds the text's symbols */
	ix_free(occ, 4 * (n_blk + 1) * 8); occ = 0;
	IXCK(ix_malloc((void **)&B, n + 1));
	IXCK(ix_malloc((void **)&SA, n_sa * 8));
	if ((rc = ix_sort(W, n, n_sm, kb, forced, B, SA, &primary, &n_groups, &max_group)) != 0) goto done;
	ix_free(W, nw * 4); W = 0;
	ix_free(SA, n_sa * 8); SA = 0;
	IXCK(ix_malloc((void **)&raw, (n + 15) / 16 * 4));
	BWAG_LAUNCH(k_bw_raw, ix_grid((n + 15) / 16, n_sm), IX_THREADS, 0, 0, B, n, primary, raw, (n + 15) / 16);
	IXCK(cudaGetLastError());
	if ((out->bwt = (uint32_t *)malloc((n + 15) / 16 * 4)) == 0) { rc = set_err("out of host memory"); goto done; }
	IXCK(cudaMemcpy(out->bwt, raw, (n + 15) / 16 * 4, cudaMemcpyDeviceToHost));
	out->primary = primary; out->seq_len = n; out->bwt_size = (n + 15) / 16;
done:
	out->peak_device_bytes = g_ix_peak;
	ix_free(W, nw * 4); ix_free(dpac, pac_bytes); ix_free(B, n + 1); ix_free(SA, n_sa * 8); ix_free(occ, 4 * (n_blk + 1) * 8); ix_free(raw, (n + 15) / 16 * 4);
	if (rc) { free(out->bwt); out->bwt = 0; }
	return rc;
}

extern "C" int bwag_bwtupdate(int device, const uint32_t *raw, uint64_t n, uint32_t *out, uint64_t *peak_device_bytes)
{
	int rc = 0, n_sm = 2;
	const u64 nw = (n + 15) / 16, n_blk = (n + 127) / 128, out_words = nw + (n_blk + 1) * 8;
	u32 *dw = 0, *dout = 0;
	u64 *occ = 0;
	size_t free_b = 0, total_b = 0;
	g_ix_cur = g_ix_peak = 0;
	if (n == 0) return set_err("empty BWT");
	if (ix_device(device, &n_sm)) return 1;
	IXCK(cudaMemGetInfo(&free_b, &total_b));
	{
		const double need = (double)nw * 4 + (double)(n_blk + 1) * 32 + (double)out_words * 4;
		if (need + (double)(64u << 20) > 0.9 * (double)free_b)
			{ rc = set_err("not enough free device memory: the update of %llu symbols needs %.2f GB, %.2f GB are free", (unsigned long long)n, need / 1e9, (double)free_b / 1e9); goto done; }
	}
	IXCK(ix_malloc((void **)&dw, nw * 4));
	IXCK(cudaMemcpy(dw, raw, nw * 4, cudaMemcpyHostToDevice));
	IXCK(ix_malloc((void **)&occ, 4 * (n_blk + 1) * 8));
	{
		u64 L2[5];
		if ((rc = ix_totals(dw, n, n_sm, occ, n_blk, L2)) != 0) goto done;
	}
	IXCK(ix_malloc((void **)&dout, out_words * 4));
	BWAG_LAUNCH(k_bw_write, ix_grid(n_blk, n_sm), IX_THREADS, 0, 0, dw, n, occ, n_blk, dout);
	IXCK(cudaGetLastError());
	IXCK(cudaMemcpy(out, dout, out_words * 4, cudaMemcpyDeviceToHost));
done:
	if (peak_device_bytes) *peak_device_bytes = g_ix_peak;
	ix_free(dw, nw * 4); ix_free(occ, 4 * (n_blk + 1) * 8); ix_free(dout, out_words * 4);
	return rc;
}
