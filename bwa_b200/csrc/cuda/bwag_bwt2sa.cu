/* bwag_bwt2sa.cu -- the sampled suffix array of a BWT from the BWT alone (`bwa-b200 bwt2sa`; bwt_cal_sa, bwt.c:62-84).
 *
 * The reference walks the LF mapping from row 0 (SA = n) once around its cycle of n + 1 rows, one dependent step per row, and
 * notes SA at every intv-th row.  Here the cycle is ranked in parallel:
 *   rulers     row 0 and every row r = j S (S a power of two, a few million rulers in all);
 *   walk       persistent lanes take rulers from an atomic counter (as K2 does) and walk LF, one 32-byte Occ sector per step, from
 *              their ruler j to the next ruler.  They record that ruler and the distance, and leave (j, d) in the SA slot of every
 *              row r = 0 mod intv they pass at distance d (the ruler's own row at d = 0), packed as j << dbits | d;
 *   ranking    the host follows the rulers from row 0, where SA = n: SA(next) = SA(j) - dist(j).  The cycle must close after
 *              exactly n + 1 rows and visit every ruler, else LF is not one cycle and the input is not the BWT of any text;
 *   fix-up     a streaming pass turns each slot into SA(j) - d.
 * Every row lies on the one cycle, so each slot is written by exactly one walk; the total work is n + 1 LF steps.  dbits holds
 * any distance up to n and the ruler index takes the other bits (S is raised when a forced stride leaves too few), so a gap
 * of any length, up to a single ruler walking the whole cycle, encodes exactly.
 * Device memory: the Occ blocks (about 0.31 n bytes), the SA sample (8 (n / intv + 1) bytes) and 16 bytes per ruler. */
#include "bwag_drv.h"

#define B2S_THREADS 256
#define B2S_RULERS_LOG2 22       /* about 4 M rulers: a few per resident lane of an H100 */
#define B2S_BAD (~(u64)0)

/* walk from rulers to the next ruler (see above); a lane whose walk leaves the rows or outlasts the cycle marks its ruler bad */
__global__ void __launch_bounds__(B2S_THREADS)
k_b2s_walk(DevIndex ix, int s_shift, int i_shift, u64 n_rul, int dbits, u64 *slot, u64 *r_next, u64 *r_dist, u64 *counter)
{
	const int lane = threadIdx.x & 31;
	const u64 n = ix.seq_len, smask = ((u64)1 << s_shift) - 1, imask = ((u64)1 << i_shift) - 1;
	i64 j = -1;
	u64 k = 0, d = 0;
	for (;;) {
		const bool idle = j < 0;   /* refill idle lanes: one atomicAdd per warp for all of them */
		const u32 bal = __ballot_sync(FULL_MASK, idle);
		if (bal) {
			u64 base = 0;
			const int leader = __ffs(bal) - 1;
			if (lane == leader) base = atomicAdd(counter, (u64)__popc(bal));
			base = __shfl_sync(FULL_MASK, base, leader);
			if (idle) {
				const u64 mine = base + __popc(bal & ((1u << lane) - 1));
				if (mine < n_rul) { j = (i64)mine; k = mine << s_shift; d = 0; }
			}
		}
		if (__all_sync(FULL_MASK, j < 0)) break;
		if (j >= 0) {
			if ((k & imask) == 0) slot[k >> i_shift] = (u64)j << dbits | d;
			k = lf_step(ix, k);
			++d;
			if (k > n || ((k & smask) != 0 && d > n)) { r_next[j] = B2S_BAD; r_dist[j] = d; j = -1; }
			else if ((k & smask) == 0) { r_next[j] = k >> s_shift; r_dist[j] = d; j = -1; }
		}
	}
}

/* slot = (j, d) -> SA(ruler j) - d */
__global__ void k_b2s_fix(u64 *slot, u64 n_slot, const u64 *r_sa, int dbits)
{
	const u64 dmask = ((u64)1 << dbits) - 1;
	for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n_slot; i += (u64)gridDim.x * blockDim.x) {
		const u64 v = slot[i];
		slot[i] = r_sa[v >> dbits] - (v & dmask);
	}
}

static int log2_ceil(u64 x) { int s = 0; while (((u64)1 << s) < x) ++s; return s; }

extern "C" int bwag_bwt2sa(int device, const bwt_t *bwt, int intv, uint64_t *sa, bwag_bwt2sa_stats_t *st)
{
	const u64 n = bwt->seq_len;
	const int i_shift = log2_ceil((u64)(intv > 0 ? intv : 1));
	const u64 n_slot = (n + (u64)intv) / (u64)intv;
	const int dbits = 64 - __builtin_clzll(n | 1);   /* distances 0..n */
	int s_shift, n_sm = 2, ndev = 0, rc = 0;
	u64 n_rul, *slot = 0, *r_next = 0, *r_dist = 0, *counter = 0, *h_next = 0, *h_dist = 0;
	const size_t occ_bytes = (((size_t)bwt->bwt_size * 4 + 64) + 255) & ~(size_t)255;
	void *d_occ = 0;
	memset(st, 0, sizeof(*st));
	if (intv < 1 || (1 << i_shift) != intv) return set_err("the suffix-array interval %d is not a power of two >= 1", intv);
	if (n == 0) return set_err("empty BWT");
	if (n >= (u64)BWAG_MAX_SB << BWAG_SB_SHIFT) return set_err("BWT too large: %llu symbols", (unsigned long long)n);
	{
		const char *e = getenv("BWA_B200_BWT2SA_STRIDE");
		if (e && *e) {
			const long long f = atoll(e);
			if (f < 1 || (f & (f - 1))) return set_err("BWA_B200_BWT2SA_STRIDE must be a power of two >= 1");
			s_shift = log2_ceil((u64)f);
		} else {
			s_shift = log2_ceil(n >> B2S_RULERS_LOG2);
			if (s_shift < 6) s_shift = 6;
		}
		while (s_shift < 63 && (64 - __builtin_clzll((n >> s_shift) | 1)) + dbits > 64) ++s_shift;   /* (j, d) fits 64 bits */
	}
	n_rul = (n >> s_shift) + 1;
	st->stride = (u64)1 << s_shift; st->n_rulers = n_rul;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return set_err("no CUDA device is visible: this library has no CPU path");
	if (device < 0) CK(cudaGetDevice(&device));
	CK(cudaSetDevice(device));
#ifndef BWAG_CUSIM
	{
		cudaDeviceProp prop;
		CK(cudaGetDeviceProperties(&prop, device));
		n_sm = prop.multiProcessorCount;
	}
#endif
	{
		size_t free_b = 0, total_b = 0;
		CK(cudaMemGetInfo(&free_b, &total_b));
		const double need = (double)occ_bytes + (double)n_slot * 8 + (double)n_rul * 16 + 64;
		if (need + (double)(64u << 20) > 0.9 * (double)free_b)
			return set_err("not enough free device memory: the Occ blocks (%.2f GB), the suffix-array sample at interval %d (%.2f GB) and %llu rulers (%.2f GB) need %.2f GB, %.2f GB are free",
			               (double)occ_bytes / 1e9, intv, (double)n_slot * 8 / 1e9, (unsigned long long)n_rul, (double)n_rul * 16 / 1e9, need / 1e9, (double)free_b / 1e9);
		st->peak_device_bytes = (u64)need;
	}
#define B2CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { rc = set_err("%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); goto done; } } while (0)
	B2CK(cudaMalloc(&d_occ, occ_bytes));
	B2CK(cudaMalloc((void **)&slot, n_slot * 8));
	B2CK(cudaMalloc((void **)&r_next, n_rul * 8));
	B2CK(cudaMalloc((void **)&r_dist, n_rul * 8));
	B2CK(cudaMalloc((void **)&counter, 8));
	{
		DevIndex ix;
		memset(&ix, 0, sizeof(ix));
		if ((rc = occ_upload(d_occ, bwt, ix.sb)) != 0) goto done;
		ix.bwt = (const uint4 *)d_occ;
		ix.primary = bwt->primary; ix.seq_len = n;
		for (int c = 0; c < 5; ++c) ix.L2[c] = bwt->L2[c];
		B2CK(cudaMemset(counter, 0, 8));
		int grid = 0;
#ifdef BWAG_CUSIM
		grid = 2;
#else
		B2CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&grid, k_b2s_walk, B2S_THREADS, 0));
		grid = n_sm * (grid > 0 ? grid : 1);
#endif
		if ((u64)grid * B2S_THREADS > n_rul + B2S_THREADS) grid = (int)((n_rul + B2S_THREADS - 1) / B2S_THREADS);
		BWAG_LAUNCH(k_b2s_walk, grid, B2S_THREADS, 0, 0, ix, s_shift, i_shift, n_rul, dbits, slot, r_next, r_dist, counter);
		B2CK(cudaGetLastError());
		B2CK(cudaDeviceSynchronize());
	}
	/* ranking: from row 0 (SA = n) along the rulers; r_dist's host copy becomes SA(ruler) */
	h_next = (u64 *)malloc(n_rul * 8); h_dist = (u64 *)malloc(n_rul * 8);
	if (!h_next || !h_dist) { rc = set_err("out of host memory for %llu rulers", (unsigned long long)n_rul); goto done; }
	B2CK(cudaMemcpy(h_next, r_next, n_rul * 8, cudaMemcpyDeviceToHost));
	B2CK(cudaMemcpy(h_dist, r_dist, n_rul * 8, cudaMemcpyDeviceToHost));
	{
		u64 j = 0, walked = 0, seen = 0;
		do {
			const u64 nx = h_next[j], dist = h_dist[j];
			if (nx == B2S_BAD || dist == B2S_BAD || walked + dist > n + 1) break;
			h_dist[j] = B2S_BAD;   /* visited; its SA goes to h_next below */
			h_next[j] = n - walked;
			walked += dist; ++seen;
			j = nx;
		} while (j != 0 && h_dist[j] != B2S_BAD);
		if (j != 0 || walked != n + 1 || seen != n_rul)
			{ rc = set_err("not the BWT of any text: its LF mapping is not one cycle through all %llu rows (the cycle of row 0 has %llu%s)",
			               (unsigned long long)n + 1, (unsigned long long)walked, j != 0 || walked != n + 1 ? " or breaks off" : " but misses rulers"); goto done; }
	}
	B2CK(cudaMemcpy(r_dist, h_next, n_rul * 8, cudaMemcpyHostToDevice));
	{
		const u64 nb = (n_slot + B2S_THREADS - 1) / B2S_THREADS, cap = (u64)n_sm * 16;
		BWAG_LAUNCH(k_b2s_fix, (int)(nb < cap ? nb : cap), B2S_THREADS, 0, 0, slot, n_slot, r_dist, dbits);
		B2CK(cudaGetLastError());
	}
	B2CK(cudaMemcpy(sa, slot, n_slot * 8, cudaMemcpyDeviceToHost));
done:
#undef B2CK
	free(h_next); free(h_dist);
	if (d_occ) cudaFree(d_occ);
	if (slot) cudaFree(slot);
	if (r_next) cudaFree(r_next);
	if (r_dist) cudaFree(r_dist);
	if (counter) cudaFree(counter);
	return rc;
}
