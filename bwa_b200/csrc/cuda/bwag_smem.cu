/* bwag_smem.cu -- stage 1 kernels: SMEM seeding (K1, K1f) and the per-read epilogue (K1b).
 *
 * K1/K1f replace mem_collect_intv (bwamem.c:140-188) and everything under it: bwt_smem1a (bwt.c:289-351),
 * bwt_seed_strategy1 (bwt.c:358-379), bwt_extend (bwt.c:262-275), bwt_2occ4/bwt_occ4 (bwt.c:169-220).
 *
 * Mapping to the machine.  Per read the work is a chain of ~800 dependent FM-index steps, each needing
 * one or two 64-byte Occ blocks at effectively random addresses of a multi-GB table.  Throughput =
 * (independent steps in flight) / (HBM latency + issue time of one step), so the design keeps as many
 * independent 64-byte requests in flight per SM as registers allow and spends as few issue slots per
 * step as possible:
 *   - ONE LANE PER READ.  A lane keeps the whole seeding state machine of its read in registers and
 *     fetches the blocks of its current bwt_extend itself (one 32-byte sector = one LDG.256 per rank
 *     position; positions that share a block fetch it once).  A warp thus has 32 independent
 *     extensions = up to 64 sectors in flight per iteration, and no shuffles are needed to combine
 *     partial counts;
 *   - LOCK-STEP STATE MACHINES.  The reads of a warp are in different phases, so each lane advances its
 *     own state machine (short, divergent) until it needs the next extension; then the whole warp meets
 *     at ONE converged, branch-free load/popcount/select sequence (bit-plane blocks, bwag_dev.cuh);
 *   - the third seeding pass (forward-only seeds, bwamem.c:170-185) does not depend on the first two, so
 *     it is its own kernel K1f with a tenth of the state, three times the occupancy and no lists; it
 *     leaves its intervals in a fixed-stride staging area that K1 appends to the read's list;
 *   - the read's bases and the first K1_SLOTS entries of both candidate lists live in SHARED memory
 *     (a lane's private slice, conflict-free stride); longer lists continue in a per-lane global array.
 *     Entries are 16 bytes (three 35-bit interval fields + a 23-bit end position);
 *   - PERSISTENT LANES pull the next read from an atomic counter, so a warp stays full until the batch
 *     is exhausted regardless of read length or repeat content;
 *   - a finished read appends its (unsorted) interval list to the batch-wide pool with one atomicAdd;
 *     K1b (one lane per read) sorts each list by (start,end) -- ties are identical intervals -- sizes
 *     the seed pool and writes the BWT rows whose suffix-array values K2 resolves.
 * The list above is k_smem, the first form (and the kernel of the table-less baseline).  The default since round 2 is k_smem_c
 * (below): the same lock-step design with the short candidates as bits of a mask, matches appended to the read's list at once,
 * and no byte copy of the read in shared memory -- half the L2 requests, none of the serial global round trips in the divergent part.
 * HBM-latency/bandwidth bound; algorithmic bytes = 64 B x Occ-block touches as the reference counts
 * them (bwt.c:194-197), accumulated per lane and summed into one counter.
 */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"
#include "bwag_ext.cuh"

enum { ST_IDLE = 0, ST_FWD, ST_BWD, ST_NONE };

struct Intv { u64 x0, x1, x2, info; };

__device__ __forceinline__ Intv ld_intv(const Intv *p)
{
	const ulonglong2 *q = reinterpret_cast<const ulonglong2 *>(p);
	ulonglong2 a = q[0], b = q[1];
	Intv r; r.x0 = a.x; r.x1 = a.y; r.x2 = b.x; r.info = b.y;
	return r;
}
__device__ __forceinline__ void st_intv(Intv *p, u64 x0, u64 x1, u64 x2, u64 info)
{
	ulonglong2 *q = reinterpret_cast<ulonglong2 *>(p);
	ulonglong2 a, b; a.x = x0; a.y = x1; b.x = x2; b.y = info;
	q[0] = a; q[1] = b;
}

/* bwt_extend (bwt.c:262-275) of the interval (xs = the side being extended, xo = the other side, size e2) by
 * symbol c: ranks of all four symbols at k = xs-1 and l = xs-1+e2, converged and branch-free across the warp */
__device__ __forceinline__ void extend_step(const DevIndex &ix, u64 xs, u64 xo, u64 e2, int c, u64 &touches, u64 &o_s, u64 &o_o, u64 &o_x2)
{
	const u64 k = xs - 1, l = xs - 1 + e2;
	u64 tk[4] = {0, 0, 0, 0}, tl[4] = {0, 0, 0, 0};
	const bool kv = k != (u64)-1, lv = l != (u64)-1;
	const u64 kp = k - (k >= ix.primary), lp = l - (l >= ix.primary);
	const bool same = kv && lv && (kp >> 6) == (lp >> 6);
	uint4 b0, b1, c0, c1;
	b0 = b1 = c0 = c1 = make_uint4(0, 0, 0, 0);
	if (lv) {
		bwag_ld_block(ix.bwt + ((lp >> 6) << 1), b0, b1);
	}
	if (kv && !same) {
		bwag_ld_block(ix.bwt + ((kp >> 6) << 1), c0, c1);
	}
	if (same) { c0 = b0; c1 = b1; }   /* both ranks in one block: it was fetched once */
	if (lv) bwag_block_counts(ix, b0, b1, lp, tl);
	if (kv) bwag_block_counts(ix, c0, c1, kp, tk);
	touches += (kv && lv && (kp >> 7) == (lp >> 7)) ? 1 : 2;   /* as the reference counts them: its blocks hold 128 symbols (bwt.c:194-197) */
	const u64 x2_1 = tl[1] - tk[1], x2_2 = tl[2] - tk[2], x2_3 = tl[3] - tk[3];
	o_x2 = SEL4(c, tl[0] - tk[0], x2_1, x2_2, x2_3);
	o_s = SEL4(c, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]) + 1 + SEL4(c, tk[0], tk[1], tk[2], tk[3]);   /* new x[!is_back] */
	o_o = xo + ((xs <= ix.primary && xs + e2 - 1 >= ix.primary) ? 1 : 0);                                 /* new x[is_back]: bwt.c:271-274 */
	if (c < 3) o_o += x2_3;
	if (c < 2) o_o += x2_2;
	if (c < 1) o_o += x2_1;
}

/* ------------------------------------------------------------------------------------------------ short-string table
 * Two thirds of all bwt_extend calls of a read produce a string of at most 12 bases (the first steps of every forward
 * sweep, and the many short candidates of the first steps of every backward sweep), each costing two Occ sectors because
 * such intervals are wide.  The bi-interval of a string does not depend on how it was reached, so the index keeps the
 * bi-intervals of ALL strings of 1..K bases in one table (K = 14 at 3 Gbp: 358 M entries, 5.7 GB), built once at
 * load time with the same extend_step; a step whose result is that short becomes ONE 16-byte lookup, fetched with the
 * same load sequence as an Occ block (bwag_ld_block) so that the warp stays converged.
 *   entry  = pack_ent(x0, x1, x2, t) with t = Occ-block touches of the forward chain that builds the string, as the
 *            reference counts them (bwt.c:194-197): the third pass jumps over that chain and adds t to its counter;
 *   index  = (4^len - 4)/3 + sum_t s[t] * 4^t   (all shorter strings first; first base in the low bits). */
__device__ __forceinline__ u32 ktab_off(int len) { return ((1u << (2 * len)) - 4u) / 3u; }
#define KTAB_BT_SHIFT 22                       /* count field of an entry: chain touches in the low bits, the backward-touch bit on top */
#define KTAB_CT_MASK ((1u << KTAB_BT_SHIFT) - 1u)

/* bwt_extend as extend_step, or -- for lanes with tab set -- the table entry tidx instead.  t12: the touches of this one
 * extension as the reference counts them (valid for every lane whose xs/e2 are the real input interval); ct: the entry's
 * chain count (table lanes only).  One converged instruction sequence for both kinds of lane. */
__device__ __forceinline__ void extend_step2(const DevIndex &ix, u64 xs, u64 xo, u64 e2, int c, bool tab, u32 tidx, int back,
                                             int &t12, u64 &o_s, u64 &o_o, u64 &o_x2, u32 &ct)
{
	const u64 k = xs - 1, l = xs - 1 + e2;
	u64 tk[4] = {0, 0, 0, 0}, tl[4] = {0, 0, 0, 0};
	const bool kv = k != (u64)-1, lv = l != (u64)-1;
	const u64 kp = k - (k >= ix.primary), lp = l - (l >= ix.primary);
	const bool same = kv && lv && (kp >> 6) == (lp >> 6);
	uint4 b0, b1, c0, c1;
	b0 = b1 = c0 = c1 = make_uint4(0, 0, 0, 0);
	const uint4 *p1 = tab ? reinterpret_cast<const uint4 *>(ix.ktab + (tidx & ~1u)) : ix.bwt + ((lp >> 6) << 1);
	if (tab || lv) bwag_ld_block(p1, b0, b1);
	if (!tab && kv && !same) bwag_ld_block(ix.bwt + ((kp >> 6) << 1), c0, c1);
	if (same) { c0 = b0; c1 = b1; }   /* both ranks in one block: it was fetched once */
	if (lv) bwag_block_counts(ix, b0, b1, lp, tl);   /* table lanes: computed on the entry's bits and discarded below */
	if (kv) bwag_block_counts(ix, c0, c1, kp, tk);
	t12 = (kv && lv && (kp >> 7) == (lp >> 7)) ? 1 : 2;   /* as the reference counts them: its blocks hold 128 symbols (bwt.c:194-197) */
	const u64 x2_1 = tl[1] - tk[1], x2_2 = tl[2] - tk[2], x2_3 = tl[3] - tk[3];
	o_x2 = SEL4(c, tl[0] - tk[0], x2_1, x2_2, x2_3);
	o_s = SEL4(c, ix.L2[0], ix.L2[1], ix.L2[2], ix.L2[3]) + 1 + SEL4(c, tk[0], tk[1], tk[2], tk[3]);   /* new x[!is_back] */
	o_o = xo + ((xs <= ix.primary && xs + e2 - 1 >= ix.primary) ? 1 : 0);                                 /* new x[is_back]: bwt.c:271-274 */
	if (c < 3) o_o += x2_3;
	if (c < 2) o_o += x2_2;
	if (c < 1) o_o += x2_1;
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

/* one lane per table entry: the string's bi-interval by forward extension from its first base, exactly as a sweep would */
__global__ void k_ktab_build(DevIndex ix, ulonglong2 *tab, int K)
{
	const u32 total = ktab_off(K + 1);
	for (u32 e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
		int len = 1;
		while (e >= ktab_off(len + 1)) ++len;
		const u32 key = e - ktab_off(len);
		u64 x0, x1, x2, touches = 0;
		INIT_INTV((int)(key & 3u), x0, x1, x2);
		for (int t = 1; t < len; ++t) {
			u64 o_s, o_o, o_x2;
			extend_step(ix, x1, x0, x2, 3 - (int)(key >> (2 * t) & 3u), touches, o_s, o_o, o_x2);
			x0 = o_o; x1 = o_s; x2 = o_x2;
		}
		/* bit 22 of the count field: the backward extension that produces this string from its suffix s[1..] touches two of the
		 * reference's 128-symbol blocks (bwt.c:194-197) rather than one.  k_smem_c keeps its short candidates as end positions
		 * only, so it cannot derive that from the input interval as k_smem does. */
		u32 bt = 0;
		if (len >= 2) {
			u64 y0, y1, y2, td = 0;
			INIT_INTV((int)(key >> 2 & 3u), y0, y1, y2);
			for (int t = 2; t < len; ++t) {
				u64 o_s, o_o, o_x2;
				extend_step(ix, y1, y0, y2, 3 - (int)(key >> (2 * t) & 3u), td, o_s, o_o, o_x2);
				y0 = o_o; y1 = o_s; y2 = o_x2;
			}
			const u64 k = y0 - 1, l = y0 - 1 + y2;
			const bool kv = k != (u64)-1, lv = l != (u64)-1;
			const u64 kp = k - (k >= ix.primary), lp = l - (l >= ix.primary);
			bt = (kv && lv && (kp >> 7) == (lp >> 7)) ? 0u : 1u;
		}
		tab[e] = pack_ent(x0, x1, x2, (u32)touches | bt << KTAB_BT_SHIFT);
	}
}

/* ------------------------------------------------------------------------------------------------ K1f
 * third pass (bwamem.c:170-185, bwt_seed_strategy1 bwt.c:358-379): from every start x extend forward until the
 * interval is smaller than max_mem_intv and at least min_seed_len long; continue after the seed's end */
__global__ void __launch_bounds__(K1F_THREADS)
k_smem_fwd(DevIndex ix, SeedArgs a)
{
	int rid = -1, len = 0, x = 0, i = 0, n_out = 0;
	bool in_seed = false, done = false;
	const uint8_t *q = 0;
	u64 ik0 = 0, ik1 = 0, ik2 = 0, touches = 0;
	u32 overflow = 0;
	Intv *out = 0;
	/* a seed cannot end before it is min_seed_len + 1 bases long, so its first kj bases are one table lookup */
	const int kj = ix.ktab_k < a.min_seed_len ? ix.ktab_k : a.min_seed_len;
	for (;;) {
		bool need = false, jump = false;
		u32 tidx = 0;
		for (;;) {
			if (!in_seed) {
				while (x < len && q[x] > 3) ++x;
				if (x >= len) {             /* read finished (or none yet): fetch the next one */
					if (done) break;
					if (rid >= 0) a.n3[rid] = n_out;
					rid = atomicAdd(a.next_read3, 1);
					if (rid >= a.n_reads) { rid = -1; len = 0; x = 0; done = true; break; }
					q = a.codes + a.off[rid]; len = (int)(a.off[rid + 1] - a.off[rid]);
					out = a.stage3 + (i64)rid * a.cap3;
					x = 0; n_out = 0;
					continue;
				}
				INIT_INTV(q[x], ik0, ik1, ik2);
				i = x + 1; in_seed = true;
				if (kj > 1 && x + kj <= len) {
					u32 key = q[x];
					bool ok = true;
					for (int t = 1; t < kj; ++t) { const int b = q[x + t]; ok = ok && b < 4; key |= (u32)(b & 3) << (2 * t); }
					if (ok) { jump = true; tidx = ktab_off(kj) + key; need = true; break; }   /* an N in range: step by step as before */
				}
			}
			if (i >= len) { x = len; in_seed = false; continue; }
			if (q[i] > 3) { x = i + 1; in_seed = false; continue; }
			need = true;
			break;
		}
		if (__all_sync(FULL_MASK, done)) break;
		if (!need) continue;
		u64 o_s, o_o, o_x2;
		u32 ct;
		int t12;
		extend_step3(ix, ik1, ik0, ik2, jump ? 0 : 3 - q[i], jump, tidx, 0, t12, o_s, o_o, o_x2, ct);
		if (jump) { ik0 = o_o; ik1 = o_s; ik2 = o_x2; i = x + kj; touches += ct & KTAB_CT_MASK; continue; }
		touches += (u64)t12;
		if (o_x2 < a.max_mem_intv && i - x >= a.min_seed_len) {     /* bwt.c:366-375 */
			if (o_x2 > 0) {
				if (n_out < a.cap3) { st_intv(out + n_out, o_o, o_s, o_x2, (u64)x << 32 | (u64)(i + 1)); ++n_out; } else overflow |= 8;
			}
			x = i + 1; in_seed = false;
		} else { ik0 = o_o; ik1 = o_s; ik2 = o_x2; ++i; }
	}
	for (int d = 16; d; d >>= 1) touches += __shfl_xor_sync(FULL_MASK, touches, d);
	if ((threadIdx.x & 31) == 0 && touches) atomicAdd(a.occ_touches, touches);
	overflow = __reduce_or_sync(FULL_MASK, overflow);
	if ((threadIdx.x & 31) == 0 && overflow) atomicOr(a.flags, overflow);
}

/* ------------------------------------------------------------------------------------------------ K0
 * 2-bit packed copy of every read (16 bases per word, first base in the low bits, one spare word; N packs as A and is never
 * looked up): the keys of the short-string table.  One lane per read, once per batch; K1 used to build this itself, one lane
 * at a time, with one active lane.  Read r's words start at
 * (off[r] >> 4) + 2 r. */
__global__ void __launch_bounds__(128) k_pack_reads(const uint8_t *codes, const i64 *off, int n_reads, u32 *packed, u32 *nmask, u32 *hasn)
{
	const int r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n_reads) return;
	const i64 o = off[r];
	const int len = (int)(off[r + 1] - o);
	const uint8_t *q = codes + o;
	u32 *dst = packed + (o >> 4) + 2 * (i64)r;
	const int nwp = ((len + 15) >> 4) + 1;
	u32 any_n = 0;
	for (int w = 0; w < nwp; ++w) {
		u32 pw = 0;
		for (int t = 0; t < 16; ++t) { const int idx = (w << 4) + t; if (idx < len) { pw |= (u32)(q[idx] & 3) << (2 * t); any_n |= (u32)(q[idx] > 3); } }
		dst[w] = pw;
	}
	if (hasn) hasn[r] = any_n;
	if (nmask) {   /* one bit per base: ambiguous (variant K1_PACKED8, which keeps no byte copy of the read); read r's words start at (off[r] >> 5) + 2 r */
		u32 *dn = nmask + (o >> 5) + 2 * (i64)r;
		const int nwn = (len + 31) >> 5;
		for (int w = 0; w < nwn; ++w) {
			u32 nb = 0;
			for (int t = 0; t < 32; ++t) { const int idx = (w << 5) + t; if (idx < len && q[idx] > 3) nb |= 1u << t; }
			dn[w] = nb;
		}
	}
}

/* ------------------------------------------------------------------------------------------------ K1
 * The body of k_smem, for two callers: `mem` (FM = false: the three seeding passes of mem_collect_intv) and `fastmap` (FM = true:
 * the SMEM listing of smem_next, bwamem_extra.c:86-96, one bwt_smem1a call after the other, bwt.c:289-351).  In the fastmap form
 *   - only the first pass runs, with min_intv = fm_min_intv (-i) instead of 1;
 *   - -I (fm_max_intv > 0) stops the forward sweep as soon as the current interval is smaller (bwt.c:305), and the backward sweep
 *     tests the size of bwt_smem1a's `ik` register, not the candidate's (bwt.c:330-331): ik2 keeps the last forward interval until a
 *     match is recorded and is the last recorded match from then on (bwt.c:334), short matches included;
 *   - the length filter is the reference's unsigned one (fastmap.c:460: -l < 0 keeps nothing);
 *   - the read's list is the calls' matches, each call's in ascending start (CALL_DONE), calls in the order made: nothing sorts it.
 * The FM = false instantiation (k_smem) keeps the registers, shared memory and SASS instruction count it had before. */
#ifndef K1_MIN_BLOCKS
#define K1_MIN_BLOCKS 5
#endif
template <bool FM>
__device__ __forceinline__ void smem_lane(const DevIndex &ix, const SeedArgs &a, int fm_min_intv, u64 fm_max_intv)
{
#ifdef BWAG_CUSIM
	ulonglong2 *sl = reinterpret_cast<ulonglong2 *>(cusim_dyn_smem);
#else
	extern __shared__ ulonglong2 k1_dyn[];
	ulonglong2 *sl = k1_dyn;
#endif
	/* shared: [2 lists][K1_SLOTS][K1_THREADS] entries, then K1_THREADS read slots of qstride bytes (odd word count) */
	const uint8_t *sq = reinterpret_cast<const uint8_t *>(sl + 2 * K1_SLOTS * K1_THREADS) + (size_t)threadIdx.x * a.qstride;
	/* then K1_THREADS packed copies of the reads (2 bits per base, pstride bytes each): the keys of the short-string table */
	u32 *sp = reinterpret_cast<u32 *>(const_cast<uint8_t *>(reinterpret_cast<const uint8_t *>(sl + 2 * K1_SLOTS * K1_THREADS) + (size_t)K1_THREADS * a.qstride + (size_t)threadIdx.x * a.pstride));
	const int ktk = a.pstride ? ix.ktab_k : 0;
#ifdef K1_PACKED8
	/* variant (not the default; tools/k1_variants.sh -DK1_PACKED8): the read lives in shared memory ONLY as the 2-bit packed
	 * copy plus one N bit per base (64 instead of 200 bytes per lane at 150 bp), which pays for K1_SLOTS = 8 list entries per
	 * list at the same footprint: 79 % instead of 47 % of the candidate-list accesses stay in shared memory */
	u32 *sn = reinterpret_cast<u32 *>(const_cast<uint8_t *>(reinterpret_cast<const uint8_t *>(sl + 2 * K1_SLOTS * K1_THREADS) + (size_t)K1_THREADS * (a.qstride + a.pstride) + (size_t)threadIdx.x * a.nstride));
#define QISN(i_) (a.pstride ? (int)(sn[(i_) >> 5] >> ((i_) & 31) & 1u) : (int)(q[i_] > 3))
#define QBASE(i_) (a.pstride ? (int)(sp[(i_) >> 4] >> (((i_) & 15) << 1) & 3u) : (int)q[i_])
#else
#define QISN(i_) (q[i_] > 3)
#define QBASE(i_) ((int)q[i_])
#endif
	sl += threadIdx.x;
	const i64 tid = (i64)blockIdx.x * blockDim.x + threadIdx.x;
	/* per-lane global scratch (units of 16 bytes): the tails of the two candidate lists (cap_list entries each),
	 * then the raw results of the current bwt_smem1 call (cap_list x 32 B) and the read's interval list (cap_mem x 32 B) */
	ulonglong2 *gl = reinterpret_cast<ulonglong2 *>(a.scratch) + tid * (i64)(4 * a.cap_list + 2 * a.cap_mem);
	Intv *m1 = reinterpret_cast<Intv *>(gl + 2 * a.cap_list), *mem = m1 + a.cap_list;

	int rid = -1, len = 0, pass = 2, st = ST_IDLE, x = 0, k2 = 0, old_n = 0;
	int sx = 0, min_intv = 1, i = 0, j = 0, n_prev = 0, n_curr = 0, rev_first = 0, mem_n = 0, m1_n = 0, last_start = 0, ret = 0;
	int pl = 0;                    /* which list is `prev`; the other is `curr` */
	const uint8_t *q = 0;
	u64 ik0 = 0, ik1 = 0, ik2 = 0, curr_last_x2 = 0;
	u32 ikend = 0, pend = 0;
	u64 e0 = 0, e1 = 0, e2 = 0;
	u64 touches = 0;
	u32 overflow = 0;

#define ENT_PTR(l, idx) ((idx) < K1_SLOTS ? sl + ((l) * K1_SLOTS + (idx)) * K1_THREADS : gl + (l) * a.cap_list + (idx))
#ifdef BWAG_CUSIM   /* emulator only: how much of the candidate-list traffic the K1_SLOTS shared entries per list catch */
#define ENT_COUNT(i_) __atomic_fetch_add(&bwag_cusim_list_acc[(i_) < 4 ? 0 : (i_) < 8 ? 1 : (i_) < 12 ? 2 : (i_) < 16 ? 3 : 4], 1ull, __ATOMIC_RELAXED)
#else
#define ENT_COUNT(i_) ((void)0)
#endif
#define ENT_ST(l, idx, X0, X1, X2, E) do { const int l_ = (l), i_ = (idx); const ulonglong2 v_ = pack_ent(X0, X1, X2, E); ENT_COUNT(i_); \
		if (i_ < K1_SLOTS) sl[(l_ * K1_SLOTS + i_) * K1_THREADS] = v_; else gl[l_ * a.cap_list + i_] = v_; } while (0)
#define ENT_LD(l, idx, X0, X1, X2, E) do { const int l_ = (l), i_ = (idx); ulonglong2 v_; ENT_COUNT(i_); \
		if (i_ < K1_SLOTS) v_ = sl[(l_ * K1_SLOTS + i_) * K1_THREADS]; else v_ = gl[l_ * a.cap_list + i_]; unpack_ent(v_, X0, X1, X2, E); } while (0)
	/* forward sweep over: candidates are visited longest match first; the call returns the end of the longest match */
#ifdef K1_PREFETCH
	ulonglong2 nxt; nxt.x = nxt.y = 0;
	bool have_nxt = false;
#define K1_PF_RESET() (have_nxt = false)
#else
#define K1_PF_RESET() ((void)0)
#endif
#define TURN_AROUND() do { ret = (int)ikend; pl ^= 1; n_prev = n_curr; n_curr = 0; rev_first = 1; i = sx - 1; j = 0; st = ST_BWD; K1_PF_RESET(); } while (0)
	/* bwt_smem1 returns (bwt.c:346-350 + bwamem.c:150-155): keep matches of at least min_seed_len, ascending start */
#define CALL_DONE() do { \
		for (int e_ = m1_n - 1; e_ >= 0; --e_) { \
			Intv p_ = ld_intv(m1 + e_); \
			if (FM ? (u64)((u32)p_.info - (u32)(p_.info >> 32)) >= (u64)(i64)a.min_seed_len : (int)((u32)p_.info - (u32)(p_.info >> 32)) >= a.min_seed_len) { \
				if (mem_n < a.cap_mem) { st_intv(mem + mem_n, p_.x0, p_.x1, p_.x2, p_.info); ++mem_n; } else overflow |= 8; \
			} \
		} \
		if (pass == 0) x = ret; \
		st = ST_IDLE; \
	} while (0)

	for (;;) {
		/* ---- advance this read's state machine until it needs a bwt_extend (or there is no read) ---- */
		bool need = false;
		int back = 0;
		for (;;) {
			if (st == ST_IDLE) {
				if (pass == 0) {            /* first pass: all SMEMs (bwamem.c:147-157) */
					while (x < len && QISN(x)) ++x;
					if (x >= len) { pass = FM ? 2 : 1; k2 = 0; old_n = mem_n; continue; }
					sx = x; min_intv = FM ? fm_min_intv : 1;
				} else if (pass == 1) {     /* second pass: re-seed inside long, rare SMEMs (bwamem.c:159-168) */
					bool found = false;
					while (k2 < old_n) {
						Intv p = ld_intv(mem + k2); ++k2;
						int s = (int)(p.info >> 32), e = (int)(u32)p.info;
						if (e - s < a.split_len || p.x2 > (u64)a.split_width) continue;
						sx = (s + e) >> 1; min_intv = (int)p.x2 + 1; found = true;
						break;
					}
					if (!found) { pass = 2; continue; }
				} else {                    /* read finished (or none yet): hand over its intervals, fetch the next read */
					if (rid >= 0) {
						const int n3 = a.n3 ? a.n3[rid] : 0;                    /* the third pass's seeds (K1f) join the list */
						const i64 base = (i64)atomicAdd(a.n_intv, (u64)(mem_n + n3));
						a.intv_beg[rid] = base; a.intv_n[rid] = mem_n + n3;
						if (base + mem_n + n3 > a.cap_intv) overflow |= 1;
						else {
							Intv *dst = reinterpret_cast<Intv *>(a.intv) + base;
							const Intv *s3 = a.stage3 + (i64)rid * a.cap3;
							for (int e = 0; e < mem_n; ++e) { Intv p = ld_intv(mem + e); st_intv(dst + e, p.x0, p.x1, p.x2, p.info); }
							for (int e = 0; e < n3; ++e) { Intv p = ld_intv(s3 + e); st_intv(dst + mem_n + e, p.x0, p.x1, p.x2, p.info); }
						}
					}
					rid = atomicAdd(a.next_read, 1);
					if (rid >= a.n_reads) { rid = -1; st = ST_NONE; break; }
					const i64 o = a.off[rid];
					len = (int)(a.off[rid + 1] - o);
					pass = 0; x = 0; mem_n = 0;
					if (len > a.cap_list || len >= (1 << 23)) { overflow |= 8; pass = 2; len = 0; }
#ifdef K1_PACKED8
					if (a.pstride) {            /* the packed copy and the N bitmap k_pack_reads made */
						q = a.codes + o;
						const int nwp = ((len + 15) >> 4) + 1, nwn = (len + 31) >> 5;
						const u32 *gp = a.packed + (o >> 4) + 2 * (i64)rid, *gn = a.nmask + (o >> 5) + 2 * (i64)rid;
						for (int w = 0; w < nwp; ++w) sp[w] = gp[w];
						for (int w = 0; w < nwn; ++w) sn[w] = gn[w];
					} else
#endif
					if (a.qstride) {            /* the read moves to this lane's shared slot (whole aligned words) */
						const u32 *g = reinterpret_cast<const u32 *>(a.codes + (o & ~(i64)3));
						u32 *d = reinterpret_cast<u32 *>(const_cast<uint8_t *>(sq));
						const int nw = ((int)(o & 3) + len + 3) >> 2;
						for (int w = 0; w < nw; ++w) d[w] = g[w];
						q = sq + (o & 3);
						if (ktk) {              /* the 2-bit packed copy k_pack_reads made */
							const int nwp = ((len + 15) >> 4) + 1;
							const u32 *gp = a.packed + (o >> 4) + 2 * (i64)rid;
							for (int w = 0; w < nwp; ++w) sp[w] = gp[w];
						}
					} else q = a.codes + o;
					continue;
				}
				/* start bwt_smem1(sx, min_intv) (bwt.c:289-303) */
				INIT_INTV(QBASE(sx), ik0, ik1, ik2);
				ikend = (u32)sx + 1;
				i = sx + 1; n_curr = 0; m1_n = 0; st = ST_FWD;
				continue;
			}
			if (st == ST_FWD) {
				if (i < len && !QISN(i) && !(FM && ik2 < fm_max_intv)) { e0 = ik0; e1 = ik1; e2 = ik2; need = true; back = 0; break; }
				/* end of read, ambiguous base, or (fastmap -I) an interval small enough: keep the current interval, then turn around (bwt.c:305-326) */
				ENT_ST(pl ^ 1, n_curr, ik0, ik1, ik2, ikend); ++n_curr;
				TURN_AROUND();
				continue;
			}
			if (st == ST_BWD) {
				const int c = i < 0 ? -1 : (QISN(i) ? -1 : QBASE(i));
				if (c < 0) {
					/* nothing extends: only the longest candidate (first in visiting order) can be an SMEM (bwt.c:332-338) */
					if (m1_n == 0 || i + 1 < last_start) {
						u64 p0, p1, p2; u32 pe;
						ENT_LD(pl, rev_first ? n_prev - 1 : 0, p0, p1, p2, pe);
						st_intv(m1 + m1_n, p0, p1, p2, (u64)(i + 1) << 32 | pe); ++m1_n; last_start = i + 1;
					}
					CALL_DONE();
					continue;
				}
				if (j < n_prev) {
					if (FM && ik2 < fm_max_intv) {   /* -I: no extension, the candidate is kept as if it died (bwt.c:330-336) */
						if (n_curr == 0 && (m1_n == 0 || i + 1 < last_start)) {
							u64 p0, p1, p2; u32 pe;
							ENT_LD(pl, rev_first ? n_prev - 1 - j : j, p0, p1, p2, pe);
							st_intv(m1 + m1_n, p0, p1, p2, (u64)(i + 1) << 32 | pe); ++m1_n; last_start = i + 1; ik2 = p2;
						}
						++j; K1_PF_RESET();
						continue;
					}
#ifdef K1_PREFETCH   /* variant: the next candidate's entry is requested one step ahead, so that a list tail in global memory is not a serial round trip before the Occ load */
					{
						ulonglong2 v_;
						if (have_nxt) v_ = nxt;
						else { const int i_ = rev_first ? n_prev - 1 - j : j; v_ = i_ < K1_SLOTS ? sl[(pl * K1_SLOTS + i_) * K1_THREADS] : gl[pl * a.cap_list + i_]; }
						unpack_ent(v_, e0, e1, e2, pend);
						have_nxt = j + 1 < n_prev;
						if (have_nxt) { const int i_ = rev_first ? n_prev - 2 - j : j + 1; nxt = i_ < K1_SLOTS ? sl[(pl * K1_SLOTS + i_) * K1_THREADS] : gl[pl * a.cap_list + i_]; }
					}
#else
					ENT_LD(pl, rev_first ? n_prev - 1 - j : j, e0, e1, e2, pend);
#endif
					need = true; back = 1;
					break;
				}
				if (n_curr == 0) { CALL_DONE(); continue; }
				pl ^= 1;
				n_prev = n_curr; n_curr = 0; rev_first = 0; --i; j = 0;
#ifdef K1_PREFETCH
				have_nxt = false;
#endif
				continue;
			}
			break; /* ST_NONE */
		}

		if (__all_sync(FULL_MASK, st == ST_NONE)) break;
		if (!need) continue;

		const int cq = QBASE(i);                           /* base to add: forward uses its complement (bwt.c:309), backward the base itself */
		u64 o_s, o_o, o_x2;
		{
			const int rlen = back ? (int)pend - i : i + 1 - sx;   /* the string this extension produces: q[i..pend) or q[sx..i] */
			const bool tab = rlen <= ktk;
			u32 tidx = 0, ct;
			int t12;
			if (tab) {
				const int pos = back ? i : sx;
				const u32 win = __funnelshift_r(sp[pos >> 4], sp[(pos >> 4) + 1], (u32)(pos & 15) << 1);
				tidx = ktab_off(rlen) + (win & ((1u << (2 * rlen)) - 1u));
			}
			extend_step3(ix, back ? e0 : e1, back ? e1 : e0, e2, back ? cq : 3 - cq, tab, tidx, back, t12, o_s, o_o, o_x2, ct);
			touches += (u64)t12;
		}

		/* ---- consume ---- */
		if (st == ST_FWD) {                 /* bwt.c:307-316 */
			bool stop = false;
			if (o_x2 != ik2) {
				if (n_curr < a.cap_list) { ENT_ST(pl ^ 1, n_curr, ik0, ik1, ik2, ikend); ++n_curr; } else overflow |= 8;
				if (o_x2 < (u64)min_intv) stop = true;
			}
			if (stop) TURN_AROUND();
			else {
				ik0 = o_o; ik1 = o_s; ik2 = o_x2; ikend = (u32)i + 1;
				++i;
				if (i == len) {             /* reached the end: the last interval is a candidate too (bwt.c:322) */
					if (n_curr < a.cap_list) { ENT_ST(pl ^ 1, n_curr, ik0, ik1, ik2, ikend); ++n_curr; } else overflow |= 8;
					TURN_AROUND();
				}
			}
		} else {                            /* ST_BWD, bwt.c:331-343 */
			if (o_x2 < (u64)min_intv) {
				if (n_curr == 0 && (m1_n == 0 || i + 1 < last_start)) {
					st_intv(m1 + m1_n, e0, e1, e2, (u64)(i + 1) << 32 | pend); ++m1_n; last_start = i + 1;
					if (FM) ik2 = e2;       /* bwt.c:334: ik = *p */
				}
			} else if (n_curr == 0 || o_x2 != curr_last_x2) {
				ENT_ST(pl ^ 1, n_curr, o_s, o_o, o_x2, pend); ++n_curr; curr_last_x2 = o_x2;
			}
			++j;
		}
	}
	/* warp-level sum of the touch counters, one atomic per warp */
	{
		u64 t = touches;
		for (int d = 16; d; d >>= 1) t += __shfl_xor_sync(FULL_MASK, t, d);
		if ((threadIdx.x & 31) == 0 && t) atomicAdd(a.occ_touches, t);
		u32 f = __reduce_or_sync(FULL_MASK, overflow);
		if ((threadIdx.x & 31) == 0 && f) atomicOr(a.flags, f);
	}
}

__global__ void __launch_bounds__(K1_THREADS, K1_MIN_BLOCKS)
k_smem(DevIndex ix, SeedArgs a)
{
	smem_lane<false>(ix, a, 1, 0);
}

/* fastmap: min_intv (-i, at least 1) and max_intv (-I, 0 = off); a.min_seed_len is -l */
__global__ void __launch_bounds__(K1_THREADS, K1_MIN_BLOCKS)
k_smem_fm(DevIndex ix, SeedArgs a, int min_intv, u64 max_intv)
{
	smem_lane<true>(ix, a, min_intv, max_intv);
}

#ifndef K1_PACKED8
/* ------------------------------------------------------------------------------------------------ K1, compact candidate lists
 * k_smem with two changes to what a lane keeps between extensions (same extensions, same results, same touch count):
 *
 *  - SHORT CANDIDATES ARE ONE BIT.  A backward sweep visits its candidates q[i+1..end) longest first and extends each by q[i].
 *    When the extended string q[i..end) is at most kc = min(table depth, min_seed_len) bases long, the extension is a table
 *    lookup keyed by the string alone: the candidate's interval is never read, and if the candidate dies it is shorter than
 *    min_seed_len, so bwt_smem1's caller drops it (bwamem.c:152).  Such a candidate is fully described by its end, and ends
 *    of short candidates lie within kc - 1 positions of the sweep's start sx: one bit (end - sx - 1) of a 32-bit mask per
 *    list.  Lists are ordered by decreasing end, so the candidates with an interval ("long", next string > kc bases) come
 *    first, in the shared/global slots as before, followed by the mask's bits from high to low.  A candidate whose next string
 *    outgrows kc is written out with the interval its table entry returned.  In k_smem 53 % of the list accesses went to the
 *    per-lane global tails (entries 4..); here a list rarely has more than 3 long candidates (a 3 Gbp text has few repeats of 15+
 *    bases), so the sweep's inner loop is register work between two table/Occ loads.
 *  - NO PER-CALL RESULT ARRAY.  A match that bwt_smem1 would return is appended to the read's list at once if it is long
 *    enough (k_smem parked it in a global array and copied it at the end of the call to restore ascending order; K1b sorts
 *    the read's list by (start, end) anyway, and equal keys are equal intervals).
 * The touch count of a short candidate's extension comes from the backward-touch bit of the table entry (k_ktab_build). */
#undef TURN_AROUND
#undef CALL_DONE
#define TURN_AROUND() do { ret = (int)ikend; pl ^= 1; n_prev = n_curr; n_curr = 0; rm = cm; cm = 0; rev_first = 1; i = sx - 1; j = 0; st = ST_BWD; } while (0)
#define CALL_DONE() do { if (pass == 0) x = ret; st = ST_IDLE; } while (0)
#define EMIT(X0, X1, X2, S, E) do { \
		if ((int)((E) - (u32)(S)) >= a.min_seed_len) { \
			if (mem_n < a.cap_mem) { st_intv(mem + mem_n, X0, X1, X2, (u64)(S) << 32 | (E)); ++mem_n; } else overflow |= 8; \
		} \
	} while (0)
/* a candidate for the next backward step (string of NEXT_LEN bases then): a mask bit or a list entry */
#define PUSH_CAND(NEXT_LEN, X0, X1, X2, E) do { \
		if ((NEXT_LEN) <= kc) cm |= 1u << ((int)(E) - sx - 1); \
		else if (n_curr < a.cap_list) { CENT_ST(pl ^ 1, n_curr, X0, X1, X2, E); ++n_curr; } else overflow |= 32; \
	} while (0)
#define CQISN(i_) (hn && q[i_] > 3)
#define SPW(w_) (a.pstride ? sp_sh[w_] : spg[w_])   /* a word of the packed copy: shared, or in place (uniform choice) */
#define CQBASE(i_) ((int)(SPW((i_) >> 4) >> (((i_) & 15) << 1) & 3u))
#define CENT_ST(l, idx, X0, X1, X2, E) do { const int l_ = (l), i_ = (idx); const ulonglong2 v_ = pack_ent(X0, X1, X2, E); ENT_COUNT(i_ < K1C_SLOTS ? 0 : i_); \
		if (i_ < K1C_SLOTS) sl[(l_ * K1C_SLOTS + i_) * nthr] = v_; else gl[l_ * a.cap_list + i_] = v_; } while (0)
#define CENT_LD(l, idx, X0, X1, X2, E) do { const int l_ = (l), i_ = (idx); ulonglong2 v_; ENT_COUNT(i_ < K1C_SLOTS ? 0 : i_); \
		if (i_ < K1C_SLOTS) v_ = sl[(l_ * K1C_SLOTS + i_) * nthr]; else v_ = gl[l_ * a.cap_list + i_]; unpack_ent(v_, X0, X1, X2, E); } while (0)

/* the second lookup of a pair: one 16-byte table entry */
__device__ __forceinline__ uint4 ld_ktab_ent(const ulonglong2 *p)
{
#ifdef BWAG_CUSIM
	__atomic_fetch_add(&bwag_cusim_sector_loads, 1ull, __ATOMIC_RELAXED);
#endif
	return __ldg(reinterpret_cast<const uint4 *>(p));
}
/* Occ-block touches of bwt_extend on the interval (xs, e2) as the reference counts them, with no load: extend_step3's t12 */
__device__ __forceinline__ int ref_touches(const DevIndex &ix, u64 xs, u64 e2)
{
	const u64 k = xs - 1, l = xs - 1 + e2;
	const bool kv = k != (u64)-1, lv = l != (u64)-1;
	const u64 kp = k - (k >= ix.primary), lp = l - (l >= ix.primary);
	return (kv && lv && (kp >> 7) == (lp >> 7)) ? 1 : 2;
}
#ifdef BWAG_K1_CLOCKS   /* tools/k1_bench.py: per-lane counts (the BWAG_K1CLK_* words) summed into a.k1clk; compiles to nothing otherwise */
#define K1CLK(w_, v_) (clk[w_] += (u64)(v_))
#ifdef BWAG_CUSIM
#define K1NOW() 0ull
#else
#define K1NOW() ((u64)clock64())
#endif
#else
#define K1CLK(w_, v_) ((void)0)
#endif

__global__ void __launch_bounds__(K1_THREADS, K1_MIN_BLOCKS)
k_smem_c(DevIndex ix, SeedArgs a)
{
#ifdef BWAG_CUSIM
	ulonglong2 *sl = reinterpret_cast<ulonglong2 *>(cusim_dyn_smem);
#else
	extern __shared__ ulonglong2 k1_dyn[];
	ulonglong2 *sl = k1_dyn;
#endif
	/* shared: [2 lists][K1C_SLOTS][threads] entries, then one 2-bit packed copy of pstride bytes per lane (pstride = 0: reads too long for
	 * that; the copy k_pack_reads left in global memory is read in place).  No byte copy of the read: bases come from the packed
	 * copy, and the bytes (global memory) are looked at only in reads that have an ambiguous base at all (hasn). */
	const int nthr = blockDim.x;
	u32 *sp_sh = reinterpret_cast<u32 *>(reinterpret_cast<uint8_t *>(sl + 2 * K1C_SLOTS * nthr) + (size_t)threadIdx.x * a.pstride);
	const u32 *spg = a.packed;
	bool hn = false;
	const int ktk = ix.ktab_k;                                           /* the host launches this kernel only with a table */
	const int kc = ktk < a.min_seed_len ? ktk : a.min_seed_len;
	sl += threadIdx.x;
	const i64 tid = (i64)blockIdx.x * blockDim.x + threadIdx.x;
	/* per-lane global scratch (units of 16 bytes): the tails of the two lists (cap_list entries each), then the read's interval list (cap_mem x 32 B) */
	ulonglong2 *gl = reinterpret_cast<ulonglong2 *>(a.scratch) + tid * (i64)(2 * a.cap_list + 2 * a.cap_mem);
	Intv *mem = reinterpret_cast<Intv *>(gl + 2 * a.cap_list);

	int rid = -1, len = 0, pass = 2, st = ST_IDLE, x = 0, k2 = 0, old_n = 0;
	int sx = 0, min_intv = 1, i = 0, j = 0, n_prev = 0, n_curr = 0, rev_first = 0, mem_n = 0, m1_n = 0, last_start = 0, ret = 0;
	int pl = 0;
	u32 cm = 0, rm = 0;            /* short candidates: of the list being built / still to visit in this step */
	bool cur_short = false;        /* the candidate being extended came from the mask: e0..e2 are stale */
	u32 pend2 = 0;                 /* a backward pair: the end of the second mask candidate */
#ifdef BWAG_K1_CLOCKS
	u64 clk[BWAG_K1CLK_LANE_WORDS] = {};
#endif
	const uint8_t *q = 0;
	u64 ik0 = 0, ik1 = 0, ik2 = 0, curr_last_x2 = 0;
	u32 ikend = 0, pend = 0;
	u64 e0 = 0, e1 = 0, e2 = 0;
	u64 touches = 0;
	u32 overflow = 0;

	for (;;) {
		bool need = false, two = false;   /* two: this extension and the lane's next one are both table lookups, issued together */
		int back = 0;
		K1CLK(BWAG_K1CLK_ITERS, 1);
		for (;;) {
			if (st == ST_IDLE) {
				if (pass == 0) {
					while (x < len && CQISN(x)) ++x;
					if (x >= len) { pass = 1; k2 = 0; old_n = mem_n; continue; }
					sx = x; min_intv = 1;
				} else if (pass == 1) {
					bool found = false;
					while (k2 < old_n) {
						Intv p = ld_intv(mem + k2); ++k2;
						int s = (int)(p.info >> 32), e = (int)(u32)p.info;
						if (e - s < a.split_len || p.x2 > (u64)a.split_width) continue;
						sx = (s + e) >> 1; min_intv = (int)p.x2 + 1; found = true;
						break;
					}
					if (!found) { pass = 2; continue; }
				} else {
#ifdef BWAG_K1_CLOCKS
					const u64 t_turn = K1NOW();
#endif
					if (rid >= 0) {
						const int n3 = a.n3 ? a.n3[rid] : 0;
						const i64 base = (i64)atomicAdd(a.n_intv, (u64)(mem_n + n3));
						a.intv_beg[rid] = base; a.intv_n[rid] = mem_n + n3;
						if (base + mem_n + n3 > a.cap_intv) overflow |= 1;
						else {
							/* this lane is alone here (the rest of its warp waits): two entries in flight per round trip (four spill); the third-pass
							 * seeds are appended by K1b, where every lane has a read */
							Intv *dst = reinterpret_cast<Intv *>(a.intv) + base;
							int e = 0;
							for (; e + 2 <= mem_n; e += 2) {
								const Intv p0 = ld_intv(mem + e), p1 = ld_intv(mem + e + 1);
								st_intv(dst + e, p0.x0, p0.x1, p0.x2, p0.info); st_intv(dst + e + 1, p1.x0, p1.x1, p1.x2, p1.info);
							}
							if (e < mem_n) { const Intv p0 = ld_intv(mem + e); st_intv(dst + e, p0.x0, p0.x1, p0.x2, p0.info); }
						}
					}
					rid = atomicAdd(a.next_read, 1);
					if (rid >= a.n_reads) { rid = -1; st = ST_NONE; K1CLK(BWAG_K1CLK_TURN_CYC, K1NOW() - t_turn); break; }
					const i64 o = a.off[rid];
					len = (int)(a.off[rid + 1] - o);
					pass = 0; x = 0; mem_n = 0;
					if (len >= (1 << 23)) { overflow |= 8; pass = 2; len = 0; }
					q = a.codes + o;
					hn = a.hasn[rid] != 0;
					{
						const u32 *gp = a.packed + (o >> 4) + 2 * (i64)rid;
						if (a.pstride) {
							const int nwp = ((len + 15) >> 4) + 1;
							for (int w = 0; w < nwp; ++w) sp_sh[w] = gp[w];
						} else spg = gp;
					}
					K1CLK(BWAG_K1CLK_TURN_CYC, K1NOW() - t_turn); K1CLK(BWAG_K1CLK_READS, 1);
					continue;
				}
				INIT_INTV(CQBASE(sx), ik0, ik1, ik2);
				ikend = (u32)sx + 1;
				i = sx + 1; n_curr = 0; cm = 0; m1_n = 0; st = ST_FWD;
				continue;
			}
			if (st == ST_FWD) {
				if (i < len && !CQISN(i)) {
					e0 = ik0; e1 = ik1; e2 = ik2; need = true; back = 0; cur_short = false;
					two = i + 2 - sx <= ktk && i + 1 < len && !CQISN(i + 1);   /* q[sx..i] and q[sx..i+1] */
					break;
				}
				PUSH_CAND((int)ikend - sx + 1, ik0, ik1, ik2, ikend);
				TURN_AROUND();
				continue;
			}
			if (st == ST_BWD) {
				const int c = i < 0 ? -1 : (CQISN(i) ? -1 : CQBASE(i));
				if (c < 0) {
					if (m1_n == 0 || i + 1 < last_start) {
						if (n_prev > 0) {   /* the longest candidate; one from the mask is shorter than min_seed_len */
							u64 p0, p1, p2; u32 pe;
							CENT_LD(pl, rev_first ? n_prev - 1 : 0, p0, p1, p2, pe);
							EMIT(p0, p1, p2, i + 1, pe);
						}
						++m1_n; last_start = i + 1;
					}
					CALL_DONE();
					continue;
				}
				if (j < n_prev) {
					CENT_LD(pl, rev_first ? n_prev - 1 - j : j, e0, e1, e2, pend);
					cur_short = false; need = true; back = 1;
					break;
				}
				if (rm) {
					const int b = 31 - __clz(rm);
					rm ^= 1u << b;
					pend = (u32)(sx + 1 + b);
					two = rm != 0;         /* the next candidate in visiting order is a mask bit too */
					if (two) { const int b2 = 31 - __clz(rm); rm ^= 1u << b2; pend2 = (u32)(sx + 1 + b2); }
					cur_short = true; need = true; back = 1;
					break;
				}
				if (n_curr == 0 && cm == 0) { CALL_DONE(); continue; }
				pl ^= 1;
				n_prev = n_curr; n_curr = 0; rm = cm; cm = 0; rev_first = 0; --i; j = 0;
				continue;
			}
			break; /* ST_NONE */
		}

		if (__all_sync(FULL_MASK, st == ST_NONE)) break;
		if (!need) continue;

		const int cq = CQBASE(i);
		u64 o_s, o_o, o_x2;
		uint4 ev2 = make_uint4(0, 0, 0, 0);
		{
			const int rlen = back ? (int)pend - i : i + 1 - sx;
			const bool tab = rlen <= ktk;
			u32 tidx = 0, ct;
			int t12;
			if (tab) {
				const int pos = back ? i : sx;
				const u32 win = __funnelshift_r(SPW(pos >> 4), SPW((pos >> 4) + 1), (u32)(pos & 15) << 1);
				tidx = ktab_off(rlen) + (win & ((1u << (2 * rlen)) - 1u));
				if (two) {                  /* same start: the forward string one base longer, or the next candidate's q[i..pend2) */
					const int rlen2 = back ? (int)pend2 - i : rlen + 1;
					ev2 = ld_ktab_ent(ix.ktab + ktab_off(rlen2) + (win & ((1u << (2 * rlen2)) - 1u)));
				}
			}
			/* a candidate from the mask passes stale (valid) interval registers; its lane is a table lane, which ignores them */
			extend_step3(ix, back ? e0 : e1, back ? e1 : e0, e2, back ? cq : 3 - cq, tab, tidx, back, t12, o_s, o_o, o_x2, ct);
			touches += cur_short ? (u64)(1u + (ct >> KTAB_BT_SHIFT)) : (u64)t12;
			K1CLK(back ? (cur_short ? BWAG_K1CLK_BWD_MASK : BWAG_K1CLK_BWD_LIST) : (tab ? BWAG_K1CLK_FWD_TAB : BWAG_K1CLK_FWD_OCC), 1);
			K1CLK(back ? BWAG_K1CLK_PAIR_BWD : BWAG_K1CLK_PAIR_FWD, two);
		}

		/* the result, then that of the pair's second lookup: the reference's bookkeeping sees them in visiting order */
		for (;;) {
			if (st == ST_FWD) {                 /* bwt.c:307-316 */
				bool stop = false;
				if (o_x2 != ik2) {
					PUSH_CAND((int)ikend - sx + 1, ik0, ik1, ik2, ikend);
					if (o_x2 < (u64)min_intv) stop = true;
				}
				if (stop) TURN_AROUND();
				else {
					ik0 = o_o; ik1 = o_s; ik2 = o_x2; ikend = (u32)i + 1;
					++i;
					if (i == len) {
						PUSH_CAND((int)ikend - sx + 1, ik0, ik1, ik2, ikend);
						TURN_AROUND();
					}
				}
			} else {                            /* ST_BWD, bwt.c:331-343 */
				const bool first = n_curr == 0 && cm == 0;
				if (o_x2 < (u64)min_intv) {
					if (first && (m1_n == 0 || i + 1 < last_start)) {
						if (!cur_short) EMIT(e0, e1, e2, i + 1, pend);
						++m1_n; last_start = i + 1;
					}
				} else if (first || o_x2 != curr_last_x2) {
					PUSH_CAND((int)pend - i + 1, o_s, o_o, o_x2, pend);
					curr_last_x2 = o_x2;
				}
				if (!cur_short) ++j;
			}
			if (!two) break;
			two = false;
			{
				ulonglong2 v;
				u64 x0, x1, x2;
				u32 ct2;
				v.x = (u64)ev2.y << 32 | ev2.x; v.y = (u64)ev2.w << 32 | ev2.z;
				unpack_ent(v, x0, x1, x2, ct2);
				if (back) { pend = pend2; touches += 1u + (ct2 >> KTAB_BT_SHIFT); o_s = x0; o_o = x1; }
				else {
					if (st != ST_FWD) break;    /* the first result ended the sweep: the longer string is never reached */
					touches += (u64)ref_touches(ix, ik1, ik2);   /* extending the first result */
					o_s = x1; o_o = x0;
				}
				o_x2 = x2;
			}
		}
	}
	{
		u64 t = touches;
		for (int d = 16; d; d >>= 1) t += __shfl_xor_sync(FULL_MASK, t, d);
		if ((threadIdx.x & 31) == 0 && t) atomicAdd(a.occ_touches, t);
		u32 f = __reduce_or_sync(FULL_MASK, overflow);
		if ((threadIdx.x & 31) == 0 && f) atomicOr(a.flags, f);
	}
#ifdef BWAG_K1_CLOCKS
	for (int w = 0; w < BWAG_K1CLK_LANE_WORDS; ++w) {
		u64 t = clk[w];
		for (int d = 16; d; d >>= 1) t += __shfl_xor_sync(FULL_MASK, t, d);
		if ((threadIdx.x & 31) == 0 && t) atomicAdd(a.k1clk + w, t);
	}
#endif
}
#endif /* !K1_PACKED8 */

/* K1b: one lane per read: sort the read's intervals by info, size and fill its share of the seed pool */
__global__ void __launch_bounds__(K1B_THREADS)
k_seed_post(SeedArgs a)
{
	const int rid = blockIdx.x * blockDim.x + threadIdx.x;
	if (rid >= a.n_reads) return;
	const int n = a.intv_n[rid];
	if (n == 0) return;
	if (a.intv_beg[rid] + n > a.cap_intv) return;   /* K1 ran out of pool space for this read (flag set, the stage is repeated with larger pools): its slice does not exist */
	Intv *v = reinterpret_cast<Intv *>(a.intv) + a.intv_beg[rid];
	if (a.post_copies3 && a.n3) {           /* k_smem_c left the tail of the slice for the third pass's seeds (K1f) */
		const int n3 = a.n3[rid];
		const Intv *s3 = a.stage3 + (i64)rid * a.cap3;
		for (int e = 0; e < n3; ++e) { Intv p = ld_intv(s3 + e); st_intv(v + (n - n3) + e, p.x0, p.x1, p.x2, p.info); }
	}
	for (int e = 1; e < n; ++e) {           /* insertion sort; lists are short (about 8 entries for 150-bp reads) */
		Intv p = ld_intv(v + e);
		int f = e - 1;
		while (f >= 0 && v[f].info > p.info) { Intv t = ld_intv(v + f); st_intv(v + f + 1, t.x0, t.x1, t.x2, t.info); --f; }
		st_intv(v + f + 1, p.x0, p.x1, p.x2, p.info);
	}
	i64 tot = 0;
	for (int e = 0; e < n; ++e) { u64 occ = v[e].x2; tot += (i64)(occ < (u64)a.max_occ ? occ : (u64)a.max_occ); }
	i64 sb = (i64)atomicAdd(a.n_seeds, (u64)tot);
	if (sb + tot > a.cap_seeds) { atomicOr(a.flags, 1u); return; }
	i64 *sbeg = a.seed_beg + a.intv_beg[rid];
	for (int e = 0; e < n; ++e) {           /* BWT rows whose SA value is wanted: x0 + c*step (bwamem.c:304-309) */
		const u64 occ = v[e].x2, x0 = v[e].x0;
		const i64 cnt = (i64)(occ < (u64)a.max_occ ? occ : (u64)a.max_occ);
		const u64 step = occ > (u64)a.max_occ ? occ / (u64)a.max_occ : 1;
		sbeg[e] = sb;
		for (i64 c = 0; c < cnt; ++c) a.rbeg[sb + c] = (i64)(x0 + (u64)c * step);
		sb += cnt;
	}
}
