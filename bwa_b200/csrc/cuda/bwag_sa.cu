/* bwag_sa.cu -- suffix-array lookup (K2) and the optional on-device densification of the SA sample.
 *
 * K2 replaces bwt_sa/bwt_invPsi/bwt_occ (bwt.c:53-59,86-129): one lane per seed walks LF-steps until it
 * hits a sampled row.  Walk lengths are geometric (mean = sampling interval - 1), so lanes that finish
 * pull new seeds (ballot + one atomicAdd per warp): a warp keeps 32 independent 64-byte requests in
 * flight regardless of the spread.  Each step reads ONE 32-byte sector (the block's counts and bit planes).
 */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"

/* ------------------------------------------------------------------------------------------------ K2 */

__global__ void __launch_bounds__(K2_THREADS)
k_sa(DevIndex ix, SaArgs a)
{
	const int lane = threadIdx.x & 31;
	const u64 mask = ((u64)1 << ix.sa_shift) - 1;
	i64 idx = -1;
	u64 k = 0, steps = 0, touches = 0;
	for (;;) {
		/* refill idle lanes: one atomicAdd per warp for all of them */
		bool idle = idx < 0;
		u32 bal = __ballot_sync(FULL_MASK, idle);
		if (bal) {
			i64 base = 0;
			int leader = __ffs(bal) - 1;
			if (lane == leader) base = (i64)atomicAdd(a.next, (u64)__popc(bal));
			base = __shfl_sync(FULL_MASK, base, leader);
			if (idle) {
				i64 mine = base + __popc(bal & ((1u << lane) - 1));
				if (mine < a.n) { idx = mine; k = (u64)a.rbeg[idx]; steps = 0; }
			}
		}
		if (__all_sync(FULL_MASK, idx < 0)) break;
		if (idx >= 0) {
			/* a lane either finishes (reads its sampled row) or takes one LF step (reads one Occ block): both are ONE
			 * 32-byte load, issued by the same instruction so that the two kinds of lane do not serialise their latencies */
			const bool fin = (k & mask) == 0;
			const u64 kp = k - (k > ix.primary), row = k >> ix.sa_shift;
			const uint4 *p = fin ? reinterpret_cast<const uint4 *>(ix.sa + (row & ~(u64)3)) : ix.bwt + ((kp >> 6) << 1);
			uint4 cn, pl;
			bwag_ld_block(p, cn, pl);
			if (fin) {
				const int e = (int)(row & 3);
				const u32 lo = e == 0 ? cn.x : e == 1 ? cn.z : e == 2 ? pl.x : pl.z, hi = e == 0 ? cn.y : e == 1 ? cn.w : e == 2 ? pl.y : pl.w;
				a.rbeg[idx] = (i64)(steps + ((u64)hi << 32 | lo));
				idx = -1;
			} else {
				u64 rank;
				const int c = bwag_block_symbol_rank(ix, cn, pl, kp, &rank);
				k = k == ix.primary ? 0 : ix.L2[c] + rank;     /* bwt.c:53-59 */
				++steps; ++touches;
			}
		}
	}
	if (touches) atomicAdd(a.sa_touches, touches);
}

/* densify the suffix-array sample: out[r] = SA[r << out_shift] for every r, walking from the existing sample */
__global__ void k_sa_densify(DevIndex ix, u64 *out, int out_shift, u64 n_out)
{
	const u64 mask = ((u64)1 << ix.sa_shift) - 1;
	for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < n_out; r += (u64)gridDim.x * blockDim.x) {
		u64 k = r << out_shift, steps = 0;
		while (k & mask) { k = lf_step(ix, k); ++steps; }
		out[r] = r == 0 ? (u64)-1 : steps + ix.sa[k >> ix.sa_shift];
	}
}

/* re-pack the Occ table in place from the file layout (64-byte block per 128 symbols: 4 x u64 counts, 8 words of
 * 16 2-bit symbols, first symbol in the top bits) to two 32-byte blocks of 64 symbols each (bwag_dev.cuh); one
 * lane per file block, which owns exactly the 64 bytes it rewrites */
__global__ void k_occ_pack(DevIndex ix, uint4 *bwt, u64 n_blocks)
{
	for (u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x; b < n_blocks; b += (u64)gridDim.x * blockDim.x) {
		const uint4 c0 = bwt[b * 4], c1 = bwt[b * 4 + 1], w0 = bwt[b * 4 + 2], w1 = bwt[b * 4 + 3];
		const u32 w[8] = { w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w };
		const int sbi = (int)((b << 7) >> BWAG_SB_SHIFT);
		u32 cnt[4] = { (u32)(((u64)c0.y << 32 | c0.x) - ix.sb[sbi][0]), (u32)(((u64)c0.w << 32 | c0.z) - ix.sb[sbi][1]),
		               (u32)(((u64)c1.y << 32 | c1.x) - ix.sb[sbi][2]), (u32)(((u64)c1.w << 32 | c1.z) - ix.sb[sbi][3]) };
		uint4 out[4];
#pragma unroll
		for (int half = 0; half < 2; ++half) {   /* 64 symbols = four file words -> two words of each plane */
			u32 hi[2], lo[2];
#pragma unroll
			for (int g = 0; g < 2; ++g) {
				u32 h = 0, l = 0;
#pragma unroll
				for (int t = 0; t < 2; ++t) {
					const u32 v = w[4 * half + 2 * g + t];
#pragma unroll
					for (int s = 0; s < 16; ++s) {
						const u32 sym = v >> ((15 - s) << 1) & 3;
						h |= (sym >> 1) << (16 * t + s); l |= (sym & 1) << (16 * t + s);
					}
				}
				hi[g] = h; lo[g] = l;
			}
			out[2 * half] = make_uint4(cnt[0], cnt[1], cnt[2], cnt[3]);
			out[2 * half + 1] = make_uint4(hi[0], hi[1], lo[0], lo[1]);
			const u32 nH = __popc(hi[0]) + __popc(hi[1]), nL = __popc(lo[0]) + __popc(lo[1]), nT = __popc(hi[0] & lo[0]) + __popc(hi[1] & lo[1]);
			cnt[0] += 64 + nT - nH - nL; cnt[1] += nL - nT; cnt[2] += nH - nT; cnt[3] += nT;
		}
		bwt[b * 4] = out[0]; bwt[b * 4 + 1] = out[1]; bwt[b * 4 + 2] = out[2]; bwt[b * 4 + 3] = out[3];
	}
}

/* ------------------------------------------------------------------------------------------------ index verification
 * Is the resident FM-index (Occ/BWT blocks + suffix-array sample) the index of the resident text (pac, forward + reverse
 * complement)?  For every checked row r with suffix-array value v = SA[r] (LF walk to the sample):
 *   (a) the BWT symbol of row r is the text base before position v            (BWT <-> text <-> SA, and through the LF walk the Occ counts), and
 *   (b) suffix v sorts strictly before the suffix of row r + 1                  (SA order; strictness also rules out a repeated position),
 * Over all rows this is a complete check of .bwt/.sa against .pac; it exists because indexes of benchmark size come from this
 * repository's own builder (bwa_b200/index_build.py) -- `bwa index` needs hours there -- and must not be trusted on faith. */
__device__ u64 verify_sa(const DevIndex &ix, u64 k)
{
	const u64 mask = ((u64)1 << ix.sa_shift) - 1;
	u64 steps = 0;
	while (k & mask) { k = lf_step(ix, k); ++steps; }
	return steps + ix.sa[k >> ix.sa_shift];      /* sa[0] = -1: the row of the empty suffix */
}
__global__ void k_index_verify(DevIndex ix, u64 first, u64 stride, u64 n_check, u64 *out)
{
	const u64 n = ix.seq_len;
	u64 bad_bwt = 0, bad_order = 0, unresolved = 0, done = 0;
	for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t < n_check; t += (u64)gridDim.x * blockDim.x) {
		const u64 r = first + t * stride;
		if (r > n) break;
		const u64 v = r == 0 ? n : verify_sa(ix, r);
		++done;
		if (v > n) { ++bad_bwt; continue; }
		if (r == ix.primary) { if (v != 0) ++bad_bwt; }
		else {   /* (a) */
			const u64 kp = r - (r > ix.primary);
			uint4 cn, pl;
			u64 rank;
			bwag_ld_block(ix.bwt + ((kp >> 6) << 1), cn, pl);
			const int c = bwag_block_symbol_rank(ix, cn, pl, kp, &rank);
			if (v == 0 || c != bwag_ref_base(ix, (i64)(v - 1))) ++bad_bwt;
		}
		if (r < n) {   /* (b) */
			const u64 v2 = verify_sa(ix, r + 1);
			if (v2 >= n) { ++bad_order; continue; }     /* only row 0 holds the empty suffix */
			int cmp = 0;
			u64 x;
			for (x = 0; x < 8192 && cmp == 0; ++x) {
				if (v + x >= n) { cmp = -1; break; }      /* the shorter suffix is the smaller one */
				if (v2 + x >= n) { cmp = 1; break; }
				const int a = bwag_ref_base(ix, (i64)(v + x)), b = bwag_ref_base(ix, (i64)(v2 + x));
				cmp = a < b ? -1 : a > b ? 1 : 0;
			}
			if (cmp == 0) ++unresolved; else if (cmp > 0) ++bad_order;
		}
	}
	if (done) atomicAdd(&out[0], done);
	if (bad_bwt) atomicAdd(&out[1], bad_bwt);
	if (bad_order) atomicAdd(&out[2], bad_order);
	if (unresolved) atomicAdd(&out[3], unresolved);
}
