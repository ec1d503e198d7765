/* bwag_dev.cuh -- device-side view of the index, launch/portability macros, FM-index block arithmetic.
 *
 * Index layout in HBM (one blob, see bwag_api.cu):
 *   - Occ/BWT blocks.  The index files hold one 64-byte block per 128 BWT symbols: 4 x u64 cumulative counts +
 *     8 words of 16 2-bit symbols (bwt.h:74-82).  A rank query needs the counts AND the symbols, i.e. both
 *     32-byte HBM sectors of such a block.  Random sectors are the scarce resource here (see DESIGN.md), so
 *     k_occ_pack re-packs the table in place after upload into one 32-BYTE block per 64 symbols:
 *         bytes  0-15  four u32 counts of A,C,G,T before the block, relative to the block's 2^31-symbol superblock
 *         bytes 16-23  bit 1 of each of the 64 symbols (symbol p at bit p)
 *         bytes 24-31  bit 0 of each symbol
 *     plus a table of absolute u64 counts per superblock that travels in the kernel arguments.  Same 0.5 byte
 *     per symbol, but a rank now costs ONE sector, and the bit planes make the ranks of all four symbols six
 *     masked popcounts with no data-dependent branch: popc(hi), popc(lo), popc(hi&lo) give T = both,
 *     G = hi-only, C = lo-only, A = the rest;
 *   - the sampled suffix array bwt_t::sa (every sa_intv-th row, sa[0] = -1), re-sampled more densely on the
 *     device at load time;
 *   - the 2-bit forward reference pac (4 bases per byte, first base in the top bits).
 */
#ifndef BWAG_DEV_CUH
#define BWAG_DEV_CUH

#ifndef BWAG_CUSIM
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include "bwa_b200_dev.h"

#ifdef BWAG_CUSIM
#define BWAG_LAUNCH(kern, grid, block, smem, stream, ...) cusim_launch(dim3(grid), dim3(block), (smem), [&] { kern(__VA_ARGS__); })
#else
#define BWAG_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif

typedef unsigned long long u64;
typedef long long i64;
typedef unsigned int u32;

#ifndef BWAG_SB_SHIFT
#define BWAG_SB_SHIFT 31     /* symbols per superblock = 2^31: block counts fit u32 */
#endif
#ifndef BWAG_MAX_SB
#define BWAG_MAX_SB 8        /* tests build a variant with 2^16-symbol superblocks so that a 1 Mbp reference crosses dozens of them */
#endif

struct DevIndex {
	const uint4 *bwt;   /* 2 x uint4 per 64-symbol block: {counts}, {plane hi (2 words), plane lo (2 words)} */
	u64 sb[BWAG_MAX_SB][4];   /* counts of A,C,G,T before each superblock */
	u64 sbgt[BWAG_MAX_SB][4]; /* [s][c]: symbols greater than c before superblock s (sums of sb[s][c+1..3]) */
	const u64 *sa;
	const uint8_t *pac;
	u64 primary, seq_len;
	u64 L2[5];
	u64 n_sa;
	i64 l_pac;
	int sa_shift;       /* log2(sampling interval of sa[]) */
	/* bi-intervals of all strings of 1..ktab_k bases (bwag_smem.cu), 16 bytes each in 32-byte aligned pairs; 0 = none */
	const ulonglong2 *ktab;
	int ktab_k;
};

#define FULL_MASK 0xffffffffu
#ifdef BWAG_CUSIM
extern unsigned long long bwag_cusim_sector_loads, bwag_cusim_list_acc[5];
#endif

/* one 32-byte Occ block: sm_90 has no 256-bit global load, so the block is two adjacent 128-bit non-coherent loads
 * issued back to back.  The block is 32-byte aligned, so both halves lie in the same DRAM sector. */
__device__ __forceinline__ void bwag_ld_block(const uint4 *p, uint4 &cn, uint4 &pl)
{
#ifdef BWAG_CUSIM
	cn = p[0]; pl = p[1];
	__atomic_fetch_add(&bwag_cusim_sector_loads, 1ull, __ATOMIC_RELAXED);   /* emulator only: 32-byte requests of the seeding kernels */
#else
	asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
	             "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
	             : "=r"(cn.x), "=r"(cn.y), "=r"(cn.z), "=r"(cn.w), "=r"(pl.x), "=r"(pl.y), "=r"(pl.z), "=r"(pl.w) : "l"(p));
#endif
}

/* low t bits set, t clamped to [0,32]: which symbols of a 32-symbol plane word lie in [0,pos] */
__device__ __forceinline__ u32 bwag_plane_mask(int t) { return __funnelshift_lc(0xffffffffu, 0u, (u32)(t > 0 ? t : 0)); }

/* ranks of all four symbols over positions [0,p] of the '$'-less BWT (bwt_occ4, bwt.c:169-186), given the two
 * 16-byte halves of the block holding p: cn = relative counts, pl = {hi.lo32, hi.hi32, lo.lo32, lo.hi32} */
__device__ __forceinline__ void bwag_block_counts(const DevIndex &ix, const uint4 &cn, const uint4 &pl, u64 p, u64 out[4])
{
	const int n = (int)(p & 63) + 1;
	const int sbi = (int)(p >> BWAG_SB_SHIFT);
	const u32 m0 = bwag_plane_mask(n), m1 = bwag_plane_mask(n - 32);
	const u32 h0 = pl.x & m0, h1 = pl.y & m1, l0 = pl.z & m0, l1 = pl.w & m1;
	const u32 nH = __popc(h0) + __popc(h1), nL = __popc(l0) + __popc(l1), nT = __popc(h0 & l0) + __popc(h1 & l1);
	out[0] = ix.sb[sbi][0] + (u32)(cn.x + n + nT - nH - nL);
	out[1] = ix.sb[sbi][1] + (u32)(cn.y + nL - nT);
	out[2] = ix.sb[sbi][2] + (u32)(cn.z + nH - nT);
	out[3] = ix.sb[sbi][3] + (u32)(cn.w + nT);
}

/* symbol at position p and the number of its occurrences in [0,p], same inputs */
__device__ __forceinline__ int bwag_block_symbol_rank(const DevIndex &ix, const uint4 &cn, const uint4 &pl, u64 p, u64 *rank)
{
	const int pos = (int)(p & 63), n = pos + 1;
	const u32 hw = pos < 32 ? pl.x : pl.y, lw = pos < 32 ? pl.z : pl.w;
	const int c = (int)(hw >> (pos & 31) & 1) << 1 | (int)(lw >> (pos & 31) & 1);
	const u32 fh = (c & 2) ? 0u : 0xffffffffu, fl = (c & 1) ? 0u : 0xffffffffu;   /* flip a plane where the symbol's bit is 0 */
	const u32 r = __popc((pl.x ^ fh) & (pl.z ^ fl) & bwag_plane_mask(n)) + __popc((pl.y ^ fh) & (pl.w ^ fl) & bwag_plane_mask(n - 32));
	const u32 cc = c == 0 ? cn.x : c == 1 ? cn.y : c == 2 ? cn.z : cn.w;
	*rank = ix.sb[p >> BWAG_SB_SHIFT][c] + (u32)(cc + r);
	return c;
}

/* one LF step: row of the preceding text position (bwt.c:53-59 with bwt_occ bwt.c:107-129) */
__device__ __forceinline__ u64 lf_step(const DevIndex &ix, u64 k)
{
	if (k == ix.primary) return 0;
	u64 kp = k - (k > ix.primary);                 /* row in the '$'-less BWT == what bwt_occ uses since k != primary */
	const uint4 *blk = ix.bwt + ((kp >> 6) << 1);    /* one 32-byte sector: counts + bit planes of the 64 symbols around kp */
	u64 rank;
	uint4 cn, pl;
	bwag_ld_block(blk, cn, pl);
	const int c = bwag_block_symbol_rank(ix, cn, pl, kp, &rank);
	return ix.L2[c] + rank;
}

/* (int)x as the reference's x86-64 build computes it (cvttsd2si): x truncated toward zero when that fits an int, else INT_MIN --
 * for NaN, +-inf and every out-of-range value alike.  The device's own conversion (cvt.rzi.s32.f64) saturates instead (+inf and
 * large values give INT_MAX, NaN gives 0), which differs where the reference divides by a gap extension of 0 (-E 0): its band and
 * gap limits then come out as INT_MIN and are clamped to 1. */
__device__ __forceinline__ int bwag_trunc_i32(double x)
{
	return x > -2147483649.0 && x < 2147483648.0 ? (int)x : (-2147483647 - 1);
}

__device__ __forceinline__ int bwag_pac_base(const uint8_t *pac, i64 k) { return pac[k >> 2] >> ((~k & 3) << 1) & 3; }

/* base at position p of the doubled (forward + reverse-complement) coordinate system */
__device__ __forceinline__ int bwag_ref_base(const DevIndex &ix, i64 p)
{
	return p < ix.l_pac ? bwag_pac_base(ix.pac, p) : 3 - bwag_pac_base(ix.pac, (ix.l_pac << 1) - 1 - p);
}

/* Scratch accessors of the lean row sweeps (K4, K5).  Addresses are byte addresses.  PtrAcc: ordinary pointers (global scratch, and
 * every variant under the CPU emulator).  SmemAcc: 32-bit shared-window addresses with explicit ld/st.shared -- the
 * compiler otherwise re-derives the window base of every scratch array (S2UR CgaCtaId + 4 uniform ops) inside the row
 * loop.  All accesses are volatile asm, so they keep their program order among themselves and around __syncwarp(). */
struct PtrAcc {
	typedef unsigned char *addr;
	static __device__ __forceinline__ addr make(const void *p) { return (addr)const_cast<void *>(p); }
	static __device__ __forceinline__ int2 ld_he(addr a) { return *reinterpret_cast<const int2 *>(a); }
	static __device__ __forceinline__ void st_he(addr a, int h, int e) { *reinterpret_cast<int2 *>(a) = make_int2(h, e); }
	static __device__ __forceinline__ int ld_u8(addr a) { return *a; }
	static __device__ __forceinline__ int ld_s8(addr a) { return *reinterpret_cast<const int8_t *>(a); }
	static __device__ __forceinline__ void st_u8(addr a, int v) { *a = (unsigned char)v; }
};
#ifdef BWAG_CUSIM
typedef PtrAcc SmemAcc;
#define BWAG_KEEP(x) do { } while (0)
#else
struct SmemAcc {
	typedef u32 addr;
	static __device__ __forceinline__ addr make(const void *p) { return (u32)__cvta_generic_to_shared(p); }
	static __device__ __forceinline__ int2 ld_he(addr a) { int2 v; asm volatile("ld.shared.v2.s32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a)); return v; }
	static __device__ __forceinline__ void st_he(addr a, int h, int e) { asm volatile("st.shared.v2.s32 [%0], {%1, %2};" :: "r"(a), "r"(h), "r"(e)); }
	static __device__ __forceinline__ int ld_u8(addr a) { int v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
	static __device__ __forceinline__ int ld_s8(addr a) { int v; asm volatile("ld.shared.s8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
	static __device__ __forceinline__ void st_u8(addr a, int v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(a), "r"(v)); }
};
#define BWAG_KEEP(x) asm volatile("" : "+r"(x))   /* the value stays in its register: no re-derivation inside the loops */
#endif

/* ks_introsort (ksort.h:176-226) for n <= 17: the depth budget never runs out and neither side of the first partition
 * is deferred or iterated on (both have <= 16 gaps), so the procedure is ONE median-of-three partition followed by the
 * closing insertion sort -- move for move what the reference executes, hence the same order among equal keys.
 * A is anything indexable that yields an lvalue: a pointer, or a strided view of a shared-memory array (K3). */
template <class A, class LT>
__device__ void t_isort17(A a, int n, LT lt)
{
	if (n < 2) return;
	if (n == 2) { if (lt(a[1], a[0])) { auto x = a[0]; a[0] = a[1]; a[1] = x; } return; }
	{
		int i = 0, j = n - 1, k = ((n - 1) >> 1) + 1;
		const int hi = n - 1;
		if (lt(a[k], a[i])) { if (lt(a[k], a[j])) k = j; }
		else k = lt(a[j], a[i]) ? i : j;
		const auto piv = a[k];
		if (k != hi) { auto x = a[k]; a[k] = a[hi]; a[hi] = x; }
		for (;;) {
			do ++i; while (lt(a[i], piv));
			do --j; while (i <= j && lt(piv, a[j]));
			if (j <= i) break;
			{ auto x = a[i]; a[i] = a[j]; a[j] = x; }
		}
		{ auto x = a[i]; a[i] = a[hi]; a[hi] = x; }
	}
	for (int p = 1; p < n; ++p)
		for (int q = p; q > 0 && lt(a[q], a[q - 1]); --q) { auto x = a[q]; a[q] = a[q - 1]; a[q - 1] = x; }
}

#endif
