/* bwag_chain.cu -- stage 2a kernel (K3): seeds -> chains -> filtered chains -> extension work, on the device.
 *
 * Replaces mem_chain's chaining loop (bwamem.c:299-334) with test_and_merge (216-237), mem_chain_weight
 * (239-258), mem_chain_flt (353-411) and the per-chain preparation of mem_chain2aln (reference window
 * bwamem.c:666-685, seed order 688-691).  Used for reads short enough that mem_flt_chained_seeds is inactive
 * (bwamem.c:626-628); longer reads take the host path (bb_chain.c) because that filter needs local SW.
 *
 * Mapping to the machine.  Chaining a read is a short, strictly sequential piece of pointer-light integer
 * logic (a handful of seeds, an ordered map with usually one node) whose outcome depends on exact tie-breaks:
 *   - which of several chains with the same position is found depends on the shape of klib's B-tree
 *     (kbtree.h, t = 5 for 40-byte keys in 512-byte nodes), and
 *   - the order of equal-weight chains depends on the moves of the unstable ks_introsort (ksort.h:176-226),
 * so both are re-implemented move for move, over chain indices.  One LANE per read.  The number of seeds tot bounds
 * the chains, tree nodes, list nodes and sort keys of a read, so its working arrays need no allocation:
 *   - k_chain_sm: a read with tot <= K3S_CAP (99.8 % of 150-bp reads) keeps them in shared memory (SWs below);
 *   - k_chain: the other reads, listed by k_chain_sm, and every read of a batch with the long-read seed filter, keep them
 *     in the slice [sb, sb+tot) of batch-wide scratch arrays in HBM (GWs).
 * Measured on the benchmark workload (DESIGN.md §7), the HBM form spent ~2.3 M lane cycles on every read whatever its
 * seed count, most likely because its dependent loads go to each lane's own slice of ~2 GB of scratch.
 */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"

#define BT_T 5
#define BT_MAXK (2 * BT_T - 1)

/* ---- where a read's working arrays live ----
 * The chaining code below is written once, over a workspace W that it indexes like arrays of records: w.sn[s].rbeg, w.ch[c].w,
 * w.bt[x].key[k], w.order[i], ...  Two forms exist:
 *   GWs     the read's slice [sb, sb+tot) of batch-wide scratch arrays in HBM, records as below (any number of seeds; the only form
 *           of the long-read seed filter, whose K3b reads the slice back);
 *   SWs<..> dynamic shared memory, for reads with at most K3S_CAP seeds: every field is its own array laid out [entry][lane], so
 *           the lanes of a warp touch consecutive elements (no bank conflicts) and a dependent chain of loads (key -> chain ->
 *           position) costs shared-memory latency instead of an L2 round trip.  Indices are bytes; a record keeps only what K3
 *           reads back.  No two fields share room, even where their lifetimes would allow it: the compiler may reorder accesses
 *           of different types to the same address (type-based alias analysis). */
struct BtNode { int n, internal; int key[BT_MAXK]; int child[BT_MAXK + 1]; };
struct SeedNode { i64 rbeg; int qbeg, len; int next, pad; };
struct ChainRec { i64 pos; int first, last, n, rid; int w, kept, is_alt, pad; };
struct KeptE { int qb, qe, w, fs, alt, pad; };

struct GWs {
	enum { CAP = 0x7fffffff, STACK = 24, LONG_READS = 1 };
	BtNode *bt; SeedNode *sn; ChainRec *ch; int *order; int *idx; u64 *keys; KeptE *kk;
	int n_bt, n_sn, n_ch, root, n_keys;
	int stk_node[STACK], stk_state[STACK];   /* bt_inorder's stack */
	__device__ __forceinline__ void init(const ChainArgs &a, i64 sb)
	{
		bt = reinterpret_cast<BtNode *>(a.s_bt) + sb; sn = reinterpret_cast<SeedNode *>(a.s_sn) + sb; ch = reinterpret_cast<ChainRec *>(a.s_ch) + sb;
		order = a.s_order + sb; idx = a.s_idx + sb; keys = a.s_keys + sb;
		kk = reinterpret_cast<KeptE *>(bt);     /* mem_chain_flt's kept list: the B-tree nodes are dead by then */
		n_bt = n_sn = n_ch = n_keys = 0;
	}
};

template <class T, int NT> struct SArr {   /* element i of a [entry][lane] array, seen from one lane */
	T *p;
	__device__ __forceinline__ T &operator[](int i) const { return p[i * NT]; }
};
template <int NT, int CAP_> struct SWs {
	enum { CAP = CAP_, NB = 1 + (CAP_ - 1) / (BT_T - 1), STACK = 2, LONG_READS = 0 };
	/* Every node but the root keeps >= BT_T-1 keys (insertions only), so CAP chains need at most NB nodes; a tree of height 2 needs
	 * 1 + 2(BT_T-1) + 2 BT_T (BT_T-1) = 49 keys, so below that bt_inorder's stack holds the root and one child. */
	static_assert(CAP_ >= 1 && CAP_ < 49 && CAP_ < 128, "K3S_CAP: byte indices and a B-tree of height <= 1");
	enum : u32 {   /* byte offsets of the fields in the block's shared memory, each [entry][NT] */
		O_RBEG = 0, O_POS = 8 * CAP * NT, O_KEYS = 16 * CAP * NT,                   /* 8-byte fields */
		O_KQB = 24 * CAP * NT, O_KQE = 28 * CAP * NT,                               /* 4-byte fields */
		O_QBEG = 32 * CAP * NT, O_LEN = 36 * CAP * NT, O_RID = 40 * CAP * NT, O_W = 44 * CAP * NT, O_KW = 48 * CAP * NT,
		O_NEXT = 52 * CAP * NT, O_FIRST = 53 * CAP * NT, O_LAST = 54 * CAP * NT, O_N = 55 * CAP * NT, O_KEPT = 56 * CAP * NT,   /* bytes */
		O_ALT = 57 * CAP * NT, O_KFS = 58 * CAP * NT, O_KALT = 59 * CAP * NT, O_ORD = 60 * CAP * NT, O_IDX = 61 * CAP * NT,
		O_BN = 62 * CAP * NT, O_BI = O_BN + NB * NT, O_BK = O_BI + NB * NT, O_BC = O_BK + BT_MAXK * NB * NT,
		O_SN = O_BC + (BT_MAXK + 1) * NB * NT, O_SI = O_SN + STACK * NT, BYTES = O_SI + STACK * NT
	};
	struct Base {   /* the block's shared memory and this lane: field arrays are found from these two */
		unsigned char *base; int lane;
		template <class T> __device__ __forceinline__ SArr<T, NT> f(u32 off) const { SArr<T, NT> r; r.p = reinterpret_cast<T *>(base + off) + lane; return r; }
	};
	struct SnRef { i64 &rbeg; int &qbeg, &len; int8_t &next; };
	struct ChRef { i64 &pos; int &rid, &w; uint8_t &first, &last, &n, &kept, &is_alt; };
	struct BtRef { uint8_t &n, &internal; SArr<uint8_t, NT> key, child; };
	struct KkRef {
		int &qb, &qe, &w; int8_t &fs; uint8_t &alt;
		__device__ __forceinline__ const KkRef &operator=(const KeptE &e) const { qb = e.qb; qe = e.qe; w = e.w; fs = (int8_t)e.fs; alt = (uint8_t)e.alt; return *this; }
	};
	struct SnArr : Base { __device__ __forceinline__ SnRef operator[](int i) const {
		return SnRef{ this->template f<i64>(O_RBEG)[i], this->template f<int>(O_QBEG)[i], this->template f<int>(O_LEN)[i], this->template f<int8_t>(O_NEXT)[i] }; } };
	struct ChArr : Base { __device__ __forceinline__ ChRef operator[](int i) const {
		return ChRef{ this->template f<i64>(O_POS)[i], this->template f<int>(O_RID)[i], this->template f<int>(O_W)[i], this->template f<uint8_t>(O_FIRST)[i],
		              this->template f<uint8_t>(O_LAST)[i], this->template f<uint8_t>(O_N)[i], this->template f<uint8_t>(O_KEPT)[i], this->template f<uint8_t>(O_ALT)[i] }; } };
	struct BtArr : Base { __device__ __forceinline__ BtRef operator[](int x) const {
		SArr<uint8_t, NT> k = this->template f<uint8_t>(O_BK), c = this->template f<uint8_t>(O_BC);
		k.p += x * BT_MAXK * NT; c.p += x * (BT_MAXK + 1) * NT;
		return BtRef{ this->template f<uint8_t>(O_BN)[x], this->template f<uint8_t>(O_BI)[x], k, c }; } };
	struct KkArr : Base { __device__ __forceinline__ KkRef operator[](int i) const {
		return KkRef{ this->template f<int>(O_KQB)[i], this->template f<int>(O_KQE)[i], this->template f<int>(O_KW)[i], this->template f<int8_t>(O_KFS)[i],
		              this->template f<uint8_t>(O_KALT)[i] }; } };

	SnArr sn; ChArr ch; BtArr bt; KkArr kk;
	SArr<uint8_t, NT> order, idx, stk_node, stk_state; SArr<u64, NT> keys;
	int n_bt, n_sn, n_ch, root, n_keys;
	__device__ __forceinline__ void init(unsigned char *smem, int l)
	{
		Base b; b.base = smem; b.lane = l;
		static_cast<Base &>(sn) = b; static_cast<Base &>(ch) = b; static_cast<Base &>(bt) = b; static_cast<Base &>(kk) = b;
		order = b.template f<uint8_t>(O_ORD); idx = b.template f<uint8_t>(O_IDX); stk_node = b.template f<uint8_t>(O_SN); stk_state = b.template f<uint8_t>(O_SI);
		keys = b.template f<u64>(O_KEYS);
		n_bt = n_sn = n_ch = n_keys = 0;
	}
};
static_assert(SWs<K3S_THREADS, K3S_CAP>::BYTES == K3S_SMEM, "K3S_SMEM (bwag_kernels.h) out of date");

__device__ __forceinline__ int dev_pos2rid(const ChainArgs &a, i64 pos_f) /* bntseq.c:354-368 */
{
	int lo = 0, hi = a.n_seqs, mid = 0;
	if (pos_f >= a.l_pac) return -1;
	while (lo < hi) {
		mid = (lo + hi) >> 1;
		if (pos_f < a.ctg_off[mid]) hi = mid;
		else if (mid == a.n_seqs - 1 || pos_f < a.ctg_off[mid + 1]) break;
		else lo = mid + 1;
	}
	return mid;
}
__device__ __forceinline__ i64 dev_depos(const ChainArgs &a, i64 pos) { return pos >= a.l_pac ? (a.l_pac << 1) - 1 - pos : pos; }
__device__ __forceinline__ int dev_intv2rid(const ChainArgs &a, i64 rb, i64 re) /* bntseq.c:370-378 */
{
	if (rb < a.l_pac && re > a.l_pac) return -2;
	int x = dev_pos2rid(a, dev_depos(a, rb));
	int y = rb < re ? dev_pos2rid(a, dev_depos(a, re - 1)) : x;
	return x == y ? x : -1;
}
__device__ __forceinline__ int dev_max_gap(const ChainArgs &p, int qlen) /* bwamem.c:647-654 */
{
	int l_del = bwag_trunc_i32((double)(qlen * p.a - p.o_del) / p.e_del + 1.);
	int l_ins = bwag_trunc_i32((double)(qlen * p.a - p.o_ins) / p.e_ins + 1.);
	int l = l_del > l_ins ? l_del : l_ins;
	l = l > 1 ? l : 1;
	return l < p.w << 1 ? l : p.w << 1;
}

/* ---- ordered multimap of chains keyed by pos: klib B-tree, same search/insert/split moves (kbtree.h) ---- */
template <class W> __device__ int bt_new(W &w, int internal)
{
	auto &&z = w.bt[w.n_bt];
	z.n = 0; z.internal = internal;
	return w.n_bt++;
}
template <class W, class N> __device__ int bt_locate(const W &w, const N &x, i64 pos, int *cmp)
{
	int lo = 0, hi = x.n;
	if (x.n == 0) return -1;
	while (lo < hi) {
		int mid = (lo + hi) >> 1;
		if (w.ch[x.key[mid]].pos < pos) lo = mid + 1; else hi = mid;
	}
	if (lo == x.n) { *cmp = 1; return x.n - 1; }
	i64 kp = w.ch[x.key[lo]].pos;
	*cmp = pos < kp ? -1 : pos > kp ? 1 : 0;
	if (*cmp < 0) --lo;
	return lo;
}
template <class W> __device__ int bt_floor(const W &w, i64 pos)
{
	int x = w.root, lower = -1;
	for (;;) {
		auto &&nd = w.bt[x];
		int cmp = 0, i = bt_locate(w, nd, pos, &cmp);
		if (i >= 0 && cmp == 0) return nd.key[i];
		if (i >= 0) lower = nd.key[i];
		if (!nd.internal) return lower;
		x = nd.child[i + 1];
	}
}
template <class W> __device__ void bt_split(W &w, int xi, int i, int yi)
{
	int zi = bt_new(w, w.bt[yi].internal);
	auto &&x = w.bt[xi];
	auto &&y = w.bt[yi];
	auto &&z = w.bt[zi];
	z.n = BT_T - 1;
	for (int k = 0; k < BT_T - 1; ++k) z.key[k] = y.key[BT_T + k];
	if (y.internal) for (int k = 0; k < BT_T; ++k) z.child[k] = y.child[BT_T + k];
	y.n = BT_T - 1;
	for (int k = x.n; k > i; --k) x.child[k + 1] = x.child[k];
	x.child[i + 1] = zi;
	for (int k = x.n - 1; k >= i; --k) x.key[k + 1] = x.key[k];
	x.key[i] = y.key[BT_T - 1];
	++x.n;
}
template <class W> __device__ void bt_insert(W &w, int chain)
{
	const i64 pos = w.ch[chain].pos;
	int cmp;
	++w.n_keys;
	if (w.bt[w.root].n == BT_MAXK) {
		int s = bt_new(w, 1);
		w.bt[s].child[0] = w.root;
		bt_split(w, s, 0, w.root);
		w.root = s;
	}
	int xi = w.root;
	for (;;) {
		auto &&x = w.bt[xi];
		int i = bt_locate(w, x, pos, &cmp);
		if (!x.internal) {
			for (int k = x.n - 1; k > i; --k) x.key[k + 1] = x.key[k];
			x.key[i + 1] = chain;
			++x.n;
			return;
		}
		++i;
		if (w.bt[x.child[i]].n == BT_MAXK) {
			bt_split(w, xi, i, x.child[i]);
			if (pos > w.ch[x.key[i]].pos) ++i;
		}
		xi = x.child[i];
	}
}
/* in-order traversal without recursion (kbtree.h __kb_traverse): explicit stack (W::STACK entries, in the workspace); an internal
 * node with n keys goes through states 0..2n: even = descend into child state/2, odd = emit key (state-1)/2 */
template <class W, class A> __device__ int bt_inorder(W &w, A out)
{
	auto sn = w.stk_node;
	auto si = w.stk_state;
	int sp = 0, n = 0;
	sn[0] = w.root; si[0] = 0;
	while (sp >= 0) {
		auto &&x = w.bt[sn[sp]];
		if (!x.internal) {
			for (int k = 0; k < x.n; ++k) out[n++] = x.key[k];
			--sp;
			continue;
		}
		const int i = si[sp];
		if (i > 2 * x.n) { --sp; continue; }
		si[sp] = i + 1;
		if ((i & 1) == 0) { ++sp; sn[sp] = x.child[i >> 1]; si[sp] = 0; }
		else out[n++] = x.key[(i - 1) >> 1];
	}
	return n;
}

/* ---- the unstable sort of chain indices by weight, move for move (ksort.h:176-226) ---- */
template <class W> struct WeightLt {   /* flt_lt: heavier first (bwamem.c:350) */
	const W *w;
	__device__ __forceinline__ bool operator()(int x, int y) const { return w->ch[x].w > w->ch[y].w; }
};
#define W_LT(x, y) (w.ch[x].w > w.ch[y].w)
template <class W, class A> __device__ void sort_ins(const W &w, A a, int lo, int hi)
{
	for (int p = lo + 1; p < hi; ++p)
		for (int q = p; q > lo && W_LT(a[q], a[q - 1]); --q) { auto t = a[q]; a[q] = a[q - 1]; a[q - 1] = t; }
}
template <class W, class A> __device__ void sort_comb(const W &w, A a, int lo, int n)   /* a[lo .. lo+n) */
{
	const double shrink = 1.2473309501039786540366528676643;
	int gap = n, moved;
	do {
		if (gap > 2) { gap = (int)(gap / shrink); if (gap == 9 || gap == 10) gap = 11; }   /* in range: 0 < gap / shrink < gap */
		moved = 0;
		for (int p = lo; p + gap < lo + n; ++p)
			if (W_LT(a[p + gap], a[p])) { auto t = a[p]; a[p] = a[p + gap]; a[p + gap] = t; moved = 1; }
	} while (moved || gap > 2);
	if (gap != 1) sort_ins(w, a, lo, lo + n);
}
template <class W, class A> __device__ void sort_by_weight(const W &w, int n, A a)
{
	if (W::CAP <= 17 || n <= 17) {   /* the whole of ks_introsort at this size (bwag_dev.cuh), with no stack */
		WeightLt<W> lt; lt.w = &w;
		t_isort17(a, n, lt);
		return;
	}
	if constexpr (W::CAP > 17) {
		int slo[72], shi[72], sd[72], top = 0, d, lo, hi;
		for (d = 2; (1u << d) < (unsigned)n; ++d) {}
		lo = 0; hi = n - 1; d <<= 1;
		for (;;) {
			if (lo < hi) {
				if (--d == 0) { sort_comb(w, a, lo, hi - lo + 1); hi = lo; continue; }
				int i = lo, j = hi, k = i + ((j - i) >> 1) + 1;
				if (W_LT(a[k], a[i])) { if (W_LT(a[k], a[j])) k = j; }
				else k = W_LT(a[j], a[i]) ? i : j;
				const int piv = a[k];
				if (k != hi) { auto t = a[k]; a[k] = a[hi]; a[hi] = t; }
				for (;;) {
					do ++i; while (W_LT(a[i], piv));
					do --j; while (i <= j && W_LT(piv, a[j]));
					if (j <= i) break;
					{ auto t = a[i]; a[i] = a[j]; a[j] = t; }
				}
				{ auto t = a[i]; a[i] = a[hi]; a[hi] = t; }
				if (i - lo > hi - i) {
					if (i - lo > 16) { slo[top] = lo; shi[top] = i - 1; sd[top] = d; ++top; }
					lo = hi - i > 16 ? i + 1 : hi;
				} else {
					if (hi - i > 16) { slo[top] = i + 1; shi[top] = hi; sd[top] = d; ++top; }
					hi = i - lo > 16 ? i - 1 : lo;
				}
			} else if (top == 0) { sort_ins(w, a, 0, n); return; }
			else { --top; lo = slo[top]; hi = shi[top]; d = sd[top]; }
		}
	}
}

/* heap sort of 64-bit keys (all distinct, so any correct sort gives ks_introsort_64's order, bwamem.c:688-691) */
template <class A> __device__ void sort_keys(A a, int n)
{
	for (int s = n / 2 - 1; s >= 0; --s) {
		int i = s; u64 v = a[i];
		for (;;) { int c = 2 * i + 1; if (c >= n) break; if (c + 1 < n && a[c + 1] > a[c]) ++c; if (a[c] <= v) break; a[i] = a[c]; i = c; }
		a[i] = v;
	}
	for (int e = n - 1; e > 0; --e) {
		u64 v = a[e]; a[e] = a[0];
		int i = 0;
		for (;;) { int c = 2 * i + 1; if (c >= e) break; if (c + 1 < e && a[c + 1] > a[c]) ++c; if (a[c] <= v) break; a[i] = a[c]; i = c; }
		a[i] = v;
	}
}

template <class W, class C> __device__ int chain_weight(const W &w, const C &c) /* bwamem.c:239-258 */
{
	i64 end = 0;
	int wq = 0, wr = 0;
	for (int s = c.first; s >= 0; s = w.sn[s].next) {
		auto &&e = w.sn[s];
		if (e.qbeg >= end) wq += e.len;
		else if (e.qbeg + e.len > end) wq += (int)(e.qbeg + e.len - end);
		if (e.qbeg + e.len > end) end = e.qbeg + e.len;
	}
	end = 0;
	for (int s = c.first; s >= 0; s = w.sn[s].next) {
		auto &&e = w.sn[s];
		if (e.rbeg >= end) wr += e.len;
		else if (e.rbeg + e.len > end) wr += (int)(e.rbeg + e.len - end);
		if (e.rbeg + e.len > end) end = e.rbeg + e.len;
	}
	if (wr < wq) wq = wr;
	return wq < 1 << 30 ? wq : (1 << 30) - 1;
}

#define SEEDSW_EXT 50          /* MEM_SHORT_EXT */
#define SEEDSW_SHORT_LEN 200   /* MEM_SHORT_LEN */

/* Per kept chain: reference window and seed order of mem_chain2aln (bwamem.c:666-691), written to the read's slice of the chain and
 * seed arrays K4 reads.  BY_SCORE: seeds carry the score of the seed-level filter in `pad` (else a seed's score is its length);
 * chains the filter emptied are skipped.  Returns the number of chains written; *rlen = the longest reference window among them. */
template <bool BY_SCORE, class W, class A>
__device__ int chain_emit(const ChainArgs &a, W &w, int l_query, int n_chn, A ord, float frac_rep, i64 sb, int *rlen)
{
	int n_out = 0;
	i64 s_out = 0;
	for (int i = 0; i < n_chn; ++i) {
		auto &&c = w.ch[ord[i]];
		if (c.kept == 0 || c.n == 0) continue;
		i64 rmax0 = a.l_pac << 1, rmax1 = 0;
		int k = 0;
		for (int s = c.first; s >= 0; s = w.sn[s].next, ++k) {
			auto &&t = w.sn[s];
			const i64 bb = t.rbeg - (t.qbeg + dev_max_gap(a, t.qbeg));
			const i64 ee = t.rbeg + t.len + ((l_query - t.qbeg - t.len) + dev_max_gap(a, l_query - t.qbeg - t.len));
			if (bb < rmax0) rmax0 = bb;
			if (ee > rmax1) rmax1 = ee;
			int score;
			if constexpr (BY_SCORE) score = t.pad; else score = t.len;   /* seed score == seed length unless the seed-level filter ran */
			w.keys[k] = (u64)score << 32 | (u32)k;
		}
		if (rmax0 < 0) rmax0 = 0;
		if (rmax1 > a.l_pac << 1) rmax1 = a.l_pac << 1;
		const i64 first_rbeg = w.sn[c.first].rbeg;
		if (rmax0 < a.l_pac && a.l_pac < rmax1) { if (first_rbeg < a.l_pac) rmax1 = a.l_pac; else rmax0 = a.l_pac; }
		{   /* bns_fetch_seq: clamp to the contig holding the first seed (bntseq.c:426-441) */
			const i64 mid = first_rbeg;
			const int crid = dev_pos2rid(a, dev_depos(a, mid));
			i64 far_beg = a.ctg_off[crid], far_end = far_beg + a.ctg_len[crid];
			if (mid >= a.l_pac) { const i64 t = far_beg; far_beg = (a.l_pac << 1) - far_end; far_end = (a.l_pac << 1) - t; }
			if (rmax0 < far_beg) rmax0 = far_beg;
			if (rmax1 > far_end) rmax1 = far_end;
		}
		sort_keys(w.keys, c.n);
		if ((int)(rmax1 - rmax0) > *rlen) *rlen = (int)(rmax1 - rmax0);
		bwag_xchain_t xc;
		xc.rmax0 = rmax0; xc.rmax1 = rmax1; xc.seed_off = (int32_t)(sb + s_out); xc.n_seeds = c.n;
		/* seeds of the chain in list order -> temporary order array, then emitted in key order */
		bwag_xseed_t *xs = a.xseeds + sb + s_out;
		{
			auto lst = w.idx;                          /* the kept list is dead by now: node ids in list order */
			int q = 0;
			for (int s = c.first; s >= 0; s = w.sn[s].next) lst[q++] = s;
			for (int q2 = 0; q2 < c.n; ++q2) {
				const u64 key = w.keys[q2];
				auto &&t = w.sn[lst[(u32)key]];
				bwag_xseed_t o;
				o.rbeg = t.rbeg; o.qbeg = t.qbeg; o.len = (u32)t.len | (key == 0 ? BWAG_XSEED_ZEROKEY : 0);
				xs[q2] = o;
			}
		}
		a.xchains[sb + n_out] = xc;
		a.chain_rid[sb + n_out] = c.rid;
		a.chain_frac[sb + n_out] = frac_rep;
		s_out += c.n;
		++n_out;
	}
	return n_out;
}

/* what K3 needs of a read before it knows where its workspace goes */
struct ReadPre { const bwtintv_t *iv; const i64 *sbeg; i64 sb, tot; int n_intv, l_query, l_rep; };

/* per-read defaults of the outputs, seed count and repeat length (bwamem.c:291-298); false: the read has nothing to chain */
__device__ __forceinline__ bool chain_prelude(const ChainArgs &a, int rid, ReadPre &p)
{
	p.n_intv = a.intv_n[rid];
	p.l_query = (int)(a.off[rid + 1] - a.off[rid]);
	a.n_chains[rid] = 0; a.reg_base[rid] = 0; a.chain_beg[rid] = 0;
	if (a.flt_nchn) a.flt_nchn[rid] = -1;
#ifdef BWAG_K3_CLOCKS
	{ u32 *clk = a.k3clk + 5 * (i64)rid; clk[0] = clk[1] = clk[2] = clk[3] = clk[4] = 0; }
#endif
	if (p.n_intv == 0 || p.l_query < a.min_seed_len) return false;
	p.iv = a.intv + a.intv_beg[rid];
	p.sbeg = a.seed_beg + a.intv_beg[rid];
	p.sb = p.sbeg[0];
	i64 tot = 0;
	int b = 0, e = 0, l_rep = 0;
	for (int i = 0; i < p.n_intv; ++i) {             /* seed count + bases covered by over-represented seeds */
		const u64 occ = p.iv[i].x[2];
		tot += (i64)(occ < (u64)a.max_occ ? occ : (u64)a.max_occ);
		const int s0 = (int)(p.iv[i].info >> 32), s1 = (int)(u32)p.iv[i].info;
		if (occ <= (u64)a.max_occ) continue;
		if (s0 > e) { l_rep += e - b; b = s0; e = s1; }
		else if (s1 > e) e = s1;
	}
	l_rep += e - b;
	p.tot = tot; p.l_rep = l_rep;
	a.reg_base[rid] = p.sb; a.chain_beg[rid] = p.sb;
	return tot > 0;
}

/* chaining, mem_chain_flt and chain emission of one read (bwamem.c:299-411, 666-691) in workspace w.  Returns the chains written
 * (0 if the read's chains were parked for K3b); *rlen grows to the longest reference window among them. */
template <class W>
__device__ int chain_read(const ChainArgs &a, int rid, const ReadPre &p, W &w, int *rlen)
{
	const int l_query = p.l_query;
	const i64 sb = p.sb;
#ifdef BWAG_K3_CLOCKS
	u32 *clk = a.k3clk + 5 * (i64)rid;
	const long long clk0 = clock64();
#endif
	w.root = bt_new(w, 0);

	/* ---- chaining (bwamem.c:299-327) ---- */
	for (int i = 0; i < p.n_intv; ++i) {
		const int qbeg = (int)(p.iv[i].info >> 32), slen = (int)((u32)p.iv[i].info - (u32)(p.iv[i].info >> 32));
		const u64 occ = p.iv[i].x[2];
		const i64 cnt = (i64)(occ < (u64)a.max_occ ? occ : (u64)a.max_occ);
		for (i64 j = 0; j < cnt; ++j) {
			const i64 rbeg = a.rbeg[p.sbeg[i] + j];
			const int srid = dev_intv2rid(a, rbeg, rbeg + slen);
			if (srid < 0) continue;
			bool merged = false;
			const int lower = w.n_keys ? bt_floor(w, rbeg) : -1;
			if (lower >= 0) {           /* test_and_merge (bwamem.c:216-237) */
				auto &&c = w.ch[lower];
				auto &&first = w.sn[c.first];
				auto &&last = w.sn[c.last];
				const i64 qend = last.qbeg + last.len, rend = last.rbeg + last.len;
				if (srid == c.rid) {
					if (qbeg >= first.qbeg && qbeg + slen <= qend && rbeg >= first.rbeg && rbeg + slen <= rend) merged = true;
					else if (!((last.rbeg < a.l_pac || first.rbeg < a.l_pac) && rbeg >= a.l_pac)) {
						const i64 x = qbeg - last.qbeg, y = rbeg - last.rbeg;
						if (y >= 0 && x - y <= a.w && y - x <= a.w && x - last.len < a.max_chain_gap && y - last.len < a.max_chain_gap) {
							auto &&nn = w.sn[w.n_sn];
							nn.rbeg = rbeg; nn.qbeg = qbeg; nn.len = slen; nn.next = -1;
							last.next = w.n_sn; c.last = w.n_sn; ++c.n; ++w.n_sn;
							merged = true;
						}
					}
				}
			}
			if (!merged) {
				auto &&nn = w.sn[w.n_sn];
				nn.rbeg = rbeg; nn.qbeg = qbeg; nn.len = slen; nn.next = -1;
				auto &&c = w.ch[w.n_ch];
				c.pos = rbeg; c.first = c.last = w.n_sn; c.n = 1; c.rid = srid; c.w = 0; c.kept = 0;
				c.is_alt = a.ctg_alt[srid] ? 1 : 0;
				++w.n_sn;
				bt_insert(w, w.n_ch);
				++w.n_ch;
			}
		}
	}
	int n_chn = bt_inorder(w, w.order);           /* chains ascending by pos, duplicates in tree order (bwamem.c:330-334) */
	const float frac_rep = (float)p.l_rep / l_query;
#ifdef BWAG_K3_CLOCKS
	const long long clk1 = clock64();
	clk[0] = (u32)p.tot; clk[1] = (u32)n_chn; clk[2] = (u32)(clk1 - clk0);
#endif

	/* ---- mem_chain_flt (bwamem.c:353-411) over the index array w.order ---- */
	auto ord = w.order;
	{
		int k = 0;
		for (int i = 0; i < n_chn; ++i) {
			auto &&c = w.ch[ord[i]];
			c.kept = 0;
			c.w = chain_weight(w, c) & 0x1fffffff;
			if (c.w >= a.min_chain_weight) ord[k++] = ord[i];
		}
		n_chn = k;
	}
	if (n_chn == 0) return 0;
	sort_by_weight(w, n_chn, ord);
	auto kept = w.idx;
	int n_kept = 0;
#define QBEG(c) (w.sn[(c).first].qbeg)
#define QEND(c) (w.sn[(c).last].qbeg + w.sn[(c).last].len)
	/* The kept chains are compared with every later chain (quadratic for a read from a repeat family: thousands of chains), so
	 * what the comparison reads -- query span, weight, ALT flag, first shadowed chain -- sits in one dense array in kept order:
	 * one sequential load per comparison instead of five dependent ones through the chain and seed records. */
	auto kk = w.kk;
	{
		auto &&c0 = w.ch[ord[0]];
		c0.kept = 3;
		KeptE e; e.qb = QBEG(c0); e.qe = QEND(c0); e.w = c0.w; e.fs = -1; e.alt = c0.is_alt; e.pad = 0;
		kk[0] = e;
		kept[n_kept++] = 0;
	}
	for (int i = 1; i < n_chn; ++i) {
		auto &&ci = w.ch[ord[i]];
		const int qb_i = QBEG(ci), qe_i = QEND(ci), w_i = ci.w, alt_i = ci.is_alt;
		int large_ovlp = 0, k;
		for (k = 0; k < n_kept; ++k) {
			const auto e = kk[k];
			const int b_max = e.qb > qb_i ? e.qb : qb_i;
			const int e_min = e.qe < qe_i ? e.qe : qe_i;
			if (e_min > b_max && (!e.alt || alt_i)) {
				const int li = qe_i - qb_i, lj = e.qe - e.qb;
				const int min_l = li < lj ? li : lj;
				if (e_min - b_max >= min_l * a.mask_level && min_l < a.max_chain_gap) {
					large_ovlp = 1;
					if (e.fs < 0) kk[k].fs = i;
					if (w_i < e.w * a.drop_ratio && e.w - w_i >= a.min_seed_len << 1) break;
				}
			}
		}
		if (k == n_kept) {
			KeptE e; e.qb = qb_i; e.qe = qe_i; e.w = w_i; e.fs = -1; e.alt = alt_i; e.pad = 0;
			kk[n_kept] = e;
			kept[n_kept++] = i; ci.kept = large_ovlp ? 2 : 3;
		}
	}
	for (int i = 0; i < n_kept; ++i)
		if (kk[i].fs >= 0) w.ch[ord[kk[i].fs]].kept = 1;
	{
		int i, k;
		for (i = k = 0; i < n_chn; ++i) {
			const int kp = w.ch[ord[i]].kept;
			if (kp == 0 || kp == 3) continue;
			if (++k >= a.max_chain_extend) break;
		}
		for (; i < n_chn; ++i) if (w.ch[ord[i]].kept < 3) w.ch[ord[i]].kept = 0;
	}

	if constexpr (W::LONG_READS) {
		if (a.hsp_tab && a.hsp_tab[l_query] >= 0) {
			/* Long read: the seeds of the kept chains first pass the seed-level filter (mem_flt_chained_seeds, bwamem.c:626-641): every
			 * seed shorter than 200 bp whose 50-bp-padded window is shorter than 200 bp on both axes is aligned locally (K6, next
			 * launch) and dropped if it scores below hsp_tab[l_query].  This launch lists the alignments; k_chain_emit applies the
			 * scores and writes the chains.  Chain records, seed lists and `ord` stay in the read's scratch slice meanwhile. */
			for (int i = 0; i < n_chn; ++i) {
				const ChainRec &c = w.ch[ord[i]];
				if (c.kept == 0) continue;
				for (int sx = c.first; sx >= 0; sx = w.sn[sx].next) {
					SeedNode &t = w.sn[sx];
					t.pad = -1;
					if (t.len >= SEEDSW_SHORT_LEN) continue;
					int qb = t.qbeg - SEEDSW_EXT, qe = t.qbeg + t.len + SEEDSW_EXT;
					i64 rb = t.rbeg - SEEDSW_EXT, re = t.rbeg + t.len + SEEDSW_EXT;
					const i64 mid = (t.rbeg + (t.rbeg + t.len)) >> 1;
					if (qb < 0) qb = 0;
					if (qe > l_query) qe = l_query;
					if (rb < 0) rb = 0;
					if (re > a.l_pac << 1) re = a.l_pac << 1;
					if (rb < a.l_pac && a.l_pac < re) { if (mid < a.l_pac) re = a.l_pac; else rb = a.l_pac; }
					if (qe - qb >= SEEDSW_SHORT_LEN || re - rb >= SEEDSW_SHORT_LEN) continue;
					{   /* bns_fetch_seq: clamp to the contig that holds the middle of the seed (bntseq.c:426-441) */
						const int crid = dev_pos2rid(a, dev_depos(a, mid));
						i64 far_beg = a.ctg_off[crid], far_end = far_beg + a.ctg_len[crid];
						if (mid >= a.l_pac) { const i64 x = far_beg; far_beg = (a.l_pac << 1) - far_end; far_end = (a.l_pac << 1) - x; }
						if (rb < far_beg) rb = far_beg;
						if (re > far_end) re = far_end;
					}
					const u32 slot = atomicAdd(a.n_swtasks, 1u);
					bwag_swtask_t k;
					k.t_beg = rb; k.q_beg = a.off[rid] + qb; k.tlen = (int)(re - rb); k.qlen = qe - qb;
					k.xtra = 0;                       /* 16-bit kernel, score only: the filter does not look at the start */
					k.flags = BWAG_SWF_QREAD | BWAG_SWF_TREF;
					a.sw_tasks[slot] = k;
					t.pad = (int)slot;
				}
			}
			a.flt_nchn[rid] = n_chn;
			a.chain_frac[sb] = frac_rep;          /* parked in the read's first output slot until k_chain_emit runs */
			return 0;
		}
	}
#ifdef BWAG_K3_CLOCKS
	const long long clk2 = clock64();
	clk[3] = (u32)(clk2 - clk1);
#endif
	const int n_out = chain_emit<false>(a, w, l_query, n_chn, ord, frac_rep, sb, rlen);
#ifdef BWAG_K3_CLOCKS
	clk[4] = (u32)(clock64() - clk2);
#endif
	return n_out;
}

/* one atomic per warp for the batch-wide results: the longest reference window, the reads with many chains.  Every lane of the
 * warp calls it. */
__device__ __forceinline__ void chain_flush(const ChainArgs &a, int rlen, int many)
{
	const int m = __reduce_max_sync(FULL_MASK, rlen);
	const int nm = (int)__reduce_add_sync(FULL_MASK, (unsigned)many);
	if ((threadIdx.x & 31) == 0) {
		if (m > 0) atomicMax(a.max_rlen, m);
		if (nm) atomicAdd(a.n_many, nm);
	}
}

/* K3, on-chip form: reads with at most K3S_CAP seeds are chained with their workspace in shared memory (K3S_SMEM bytes per block);
 * the others are listed in a.big for k_chain.  Not used when the long-read seed filter is on (K3b reads the HBM workspace back). */
__global__ void __launch_bounds__(K3S_THREADS)
k_chain_sm(ChainArgs a)
{
#ifdef BWAG_CUSIM
	unsigned char *dyn = cusim_dyn_smem;
#else
	extern __shared__ int4 k3s_dyn[];
	unsigned char *dyn = reinterpret_cast<unsigned char *>(k3s_dyn);
#endif
	const int rid = blockIdx.x * K3S_THREADS + threadIdx.x;
	int rlen = 0, many = 0;
	ReadPre p;
	if (rid < a.n_reads && chain_prelude(a, rid, p)) {
		if (p.tot > K3S_CAP) a.big[atomicAdd(a.n_big, 1)] = rid;
		else {
			SWs<K3S_THREADS, K3S_CAP> w;
			w.init(dyn, threadIdx.x);
			const int n_out = chain_read(a, rid, p, w, &rlen);
			a.n_chains[rid] = n_out;
			many = n_out > a.many;
		}
	}
	chain_flush(a, rlen, many);
}

/* K3, HBM form: the reads listed in a.big (count *a.n_big), or every read if a.big is NULL; grid-stride */
__global__ void __launch_bounds__(K3_THREADS)
k_chain(ChainArgs a)
{
	const int n = a.big ? *a.n_big : a.n_reads;
	int rlen = 0, many = 0;
	for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
		const int rid = a.big ? a.big[k] : k;
		ReadPre p;
		if (!chain_prelude(a, rid, p)) continue;
		GWs w;
		w.init(a, p.sb);
		const int n_out = chain_read(a, rid, p, w, &rlen);
		a.n_chains[rid] = n_out;
		many += n_out > a.many;
	}
	chain_flush(a, rlen, many);
}

/* K3b: the seed-level filter's verdicts are in (K6 ran on the tasks k_chain listed): drop the seeds that scored below the read's
 * threshold, give the others their score (bwamem.c:631-639), then write the chains as k_chain would have. */
__global__ void __launch_bounds__(K3_THREADS)
k_chain_emit(ChainArgs a)
{
	const int rid = blockIdx.x * blockDim.x + threadIdx.x;
	if (rid >= a.n_reads) return;
	const int n_chn = a.flt_nchn[rid];
	if (n_chn < 0) return;
	const int l_query = (int)(a.off[rid + 1] - a.off[rid]);
	const i64 sb = a.seed_beg[a.intv_beg[rid]];
	const int min_hsp = a.hsp_tab[l_query];
	GWs w;
	w.init(a, sb);
	const float frac_rep = a.chain_frac[sb];
	const int *ord = w.order;
	for (int i = 0; i < n_chn; ++i) {
		ChainRec &c = w.ch[ord[i]];
		if (c.kept == 0) continue;
		int prev = -1, kept = 0, first = -1;
		for (int sx = c.first; sx >= 0; sx = w.sn[sx].next) {
			SeedNode &t = w.sn[sx];
			int sc = t.pad >= 0 ? a.sw_res[t.pad].score : -1;
			if (sc >= 0 && sc < min_hsp) continue;             /* dropped: the list skips it */
			t.pad = sc < 0 ? t.len * a.a : sc;
			if (prev < 0) first = sx; else w.sn[prev].next = sx;
			prev = sx; ++kept;
		}
		if (prev >= 0) w.sn[prev].next = -1;
		c.first = first; c.last = prev; c.n = kept;
	}
	int rlen = 0;
	const int n_out = chain_emit<true>(a, w, l_query, n_chn, ord, frac_rep, sb, &rlen);
	a.n_chains[rid] = n_out;
	if (n_out) atomicMax(a.max_rlen, rlen);
	if (n_out > a.many) atomicAdd(a.n_many, 1);
}

/* compact the regions of all reads into one dense array for the download */
__global__ void k_regs_compact(RegCompactArgs a)
{
	const int rid = blockIdx.x * blockDim.x + threadIdx.x;
	if (rid >= a.n_reads) return;
	const int n = a.n_regs[rid];
	i64 base = 0;
	if (n > 0) base = (i64)atomicAdd(a.total, (u64)n);
	a.out_beg[rid] = base;
	const bwag_xreg_t *src = a.regs + a.reg_base[rid];
	const i64 cb = a.chain_beg[rid];
	for (int k = 0; k < n; ++k) {
		bwag_creg_t o;
		o.r = src[k];
		o.rid = a.chain_rid[cb + src[k].chain];
		o.frac_rep = a.chain_frac[cb + src[k].chain];
		a.out[base + k] = o;
	}
}

/* the same for a selection of reads (the reads stage 4 hands back): out_beg / out_n are indexed by position in sel[] */
__global__ void k_regs_compact_sel(RegCompactArgs a, const int *sel, int n_sel, int *out_n)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= n_sel) return;
	const int rid = sel[k];
	const int n = a.n_regs[rid];
	i64 base = 0;
	if (n > 0) base = (i64)atomicAdd(a.total, (u64)n);
	a.out_beg[k] = base; out_n[k] = n;
	const bwag_xreg_t *src = a.regs + a.reg_base[rid];
	const i64 cb = a.chain_beg[rid];
	for (int x = 0; x < n; ++x) {
		bwag_creg_t o;
		o.r = src[x];
		o.rid = a.chain_rid[cb + src[x].chain];
		o.frac_rep = a.chain_frac[cb + src[x].chain];
		a.out[base + x] = o;
	}
}
