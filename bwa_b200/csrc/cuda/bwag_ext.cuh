/* bwag_ext.cuh -- bwt_extend by one known symbol (bwt.c:262-275) on the 32-byte Occ blocks of bwag_dev.cuh, and the 16-byte
 * candidate-list entry: what the SMEM searches of K1 (bwag_smem.cu) and of `maxk` (bwag_maxk.cu) share. */
#ifndef BWAG_EXT_CUH
#define BWAG_EXT_CUH
#include "bwag_dev.cuh"

/* candidate-list entry, 16 bytes: a = x0[35] | x2.lo[29] ; b = x1[35] | x2.hi[6] | end[23] */
#define M35 ((u64)0x7ffffffffULL)
__device__ __forceinline__ ulonglong2 pack_ent(u64 x0, u64 x1, u64 x2, u32 end)
{
	ulonglong2 v;
	v.x = x0 | (x2 & 0x1fffffffULL) << 35;
	v.y = x1 | (x2 >> 29 & 0x3f) << 35 | (u64)end << 41;
	return v;
}
__device__ __forceinline__ void unpack_ent(ulonglong2 v, u64 &x0, u64 &x1, u64 &x2, u32 &end)
{
	x0 = v.x & M35; x1 = v.y & M35;
	x2 = v.x >> 35 | (v.y >> 35 & 0x3f) << 29;
	end = (u32)(v.y >> 41);
}

#define SEL4(c, a0, a1, a2, a3) ((c) == 0 ? (a0) : (c) == 1 ? (a1) : (c) == 2 ? (a2) : (a3))

/* the bi-interval of the one-base string c (bwt_set_intv, bwt.h:101-105) */
#define INIT_INTV(c, X0, X1, X2) do { int c_ = (c); X0 = SEL4(c_, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]) + 1; X2 = SEL4(c_, ix.L2[1], ix.L2[2], ix.L2[3], ix.L2[4]) - SEL4(c_, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]); X1 = SEL4(3 - c_, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]) + 1; } while (0)

/* within positions [0,p] of its 64-symbol block: occurrences of symbol c and of symbols greater than c, plus the block's counts of
 * both before it (relative to the superblock): all a bwt_extend by ONE known symbol needs -- 32-bit selects instead of four
 * 64-bit ranks per position */
__device__ __forceinline__ void block_eq_gt(const uint4 &cn, const uint4 &pl, u64 p, int c, u32 &eq, u32 &gt)
{
	const int n = (int)(p & 63) + 1;
	const u32 m0 = bwag_plane_mask(n), m1 = bwag_plane_mask(n - 32);
	const u32 h0 = pl.x & m0, h1 = pl.y & m1, l0 = pl.z & m0, l1 = pl.w & m1;
	const u32 nH = __popc(h0) + __popc(h1), nL = __popc(l0) + __popc(l1), nT = __popc(h0 & l0) + __popc(h1 & l1);
	const u32 s2 = cn.z + cn.w, s1 = cn.y + s2;
	eq = SEL4(c, cn.x + (u32)n + nT - nH - nL, cn.y + nL - nT, cn.z + nH - nT, cn.w + nT);
	gt = SEL4(c, s1 + nH + nL - nT, s2 + nH, cn.w + nT, 0u);
}

/* extend_step2 with the ranks of the one symbol that is asked for (same results): x[2] = occ_c(l) - occ_c(k), the extended
 * side = L2[c] + 1 + occ_c(k), the other side moves by the symbols greater than c inside the interval (bwt.c:262-275) */
__device__ __forceinline__ void extend_step3(const DevIndex &ix, u64 xs, u64 xo, u64 e2, int c, bool tab, u32 tidx, int back,
                                             int &t12, u64 &o_s, u64 &o_o, u64 &o_x2, u32 &ct)
{
	const u64 k = xs - 1, l = xs - 1 + e2;
	const bool kv = k != (u64)-1, lv = l != (u64)-1;
	const u64 kp = k - (k >= ix.primary), lp = l - (l >= ix.primary);
	const bool same = kv && lv && (kp >> 6) == (lp >> 6);
	uint4 b0, b1, c0, c1;
	b0 = b1 = c0 = c1 = make_uint4(0, 0, 0, 0);
	const uint4 *p1 = tab ? reinterpret_cast<const uint4 *>(ix.ktab + (tidx & ~1u)) : ix.bwt + ((lp >> 6) << 1);
	if (tab || lv) bwag_ld_block(p1, b0, b1);
	if (!tab && kv && !same) bwag_ld_block(ix.bwt + ((kp >> 6) << 1), c0, c1);
	if (same) { c0 = b0; c1 = b1; }   /* both ranks in one block: it was fetched once */
	u32 eq_l = 0, gt_l = 0, eq_k = 0, gt_k = 0;
	block_eq_gt(b0, b1, lp, c, eq_l, gt_l);            /* table lanes: computed on the entry's bits and discarded below */
	block_eq_gt(c0, c1, kp, c, eq_k, gt_k);
	t12 = (kv && lv && (kp >> 7) == (lp >> 7)) ? 1 : 2;   /* as the reference counts them: its blocks hold 128 symbols (bwt.c:194-197) */
	const int sl = lv ? (int)(lp >> BWAG_SB_SHIFT) : 0, sk = kv ? (int)(kp >> BWAG_SB_SHIFT) : 0;
	const u64 occ_l = lv ? ix.sb[sl][c] + eq_l : 0, occ_k = kv ? ix.sb[sk][c] + eq_k : 0;
	const u64 big_l = lv ? ix.sbgt[sl][c] + gt_l : 0, big_k = kv ? ix.sbgt[sk][c] + gt_k : 0;
	o_x2 = occ_l - occ_k;
	o_s = SEL4(c, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]) + 1 + occ_k;                                     /* new x[!is_back] */
	o_o = xo + ((xs <= ix.primary && xs + e2 - 1 >= ix.primary) ? 1 : 0) + (big_l - big_k);             /* new x[is_back]: bwt.c:271-274 */
	ct = 0;
	if (tab) {
		const uint4 ev = (tidx & 1u) ? b1 : b0;
		ulonglong2 v;
		u64 x0, x1, x2;
		v.x = (u64)ev.y << 32 | ev.x; v.y = (u64)ev.w << 32 | ev.z;
		unpack_ent(v, x0, x1, x2, ct);
		o_x2 = x2; o_s = back ? x0 : x1; o_o = back ? x1 : x0;
	}
}

#endif
