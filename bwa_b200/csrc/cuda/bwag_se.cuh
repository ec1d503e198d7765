/* bwag_se.cuh -- the per-read pieces of `samse` and `sampe` (bwag_samse.cu, bwag_sampe.cu): bwa_sa2pos, the 16-bit bwa_cigar_t,
 * the record writer, bns_cnt_ambi, bwa_cal_md1 and bwa_correct_trimmed.  Force-inlined into each kernel that uses them. */
#ifndef BWAG_SE_CUH
#define BWAG_SE_CUH
#include "bwag_dev.cuh"
#include "bwag_kernels.h"

/* bwa_sa2pos (bwase.c:112-123) of a resolved row; -1: the hit spans the forward/reverse boundary */
__device__ __forceinline__ i64 se_sa2pos(i64 l_pac, i64 pos_f, int ref_len, uint8_t *strand)
{
	*strand = 0;
	if (pos_f < l_pac && l_pac < pos_f + ref_len) return -1;
	const int is_rev = pos_f >= l_pac;
	if (is_rev) pos_f = (l_pac << 1) - 1 - pos_f;
	*strand = !is_rev;
	if (is_rev) pos_f = pos_f + 1 < ref_len ? 0 : pos_f - ref_len + 1;
	return pos_f;
}

/* bwa_cigar_t (bwtaln.h:48-57): 16 bits, the op in the top two, a 14-bit length; __cigar_create ORs an unmasked length into it, so
 * a run of 16384 bases or more spills into the op bits, as in the reference (the CIGARs of the pool hold these 16-bit values) */
__device__ __forceinline__ u32 se_cigar16(u32 op, u32 len) { return (uint16_t)(op << 14 | len); }
__device__ __forceinline__ int se_op(u32 c) { return (int)(c >> 14 & 3); }
__device__ __forceinline__ int se_len(u32 c) { return (int)(c & 0x3fff); }

/* the record writer of both passes: p == NULL only counts */
struct SeOut {
	char *p; i64 n;
	__device__ __forceinline__ void c(char x) { if (p) p[n] = x; ++n; }
	__device__ __forceinline__ void s(const char *x) { while (*x) c(*x++); }
	__device__ __forceinline__ void s(const char *x, int l) { for (int k = 0; k < l; ++k) c(x[k]); }
	__device__ __forceinline__ void d(i64 v)
	{
		char buf[24];
		int k = 0;
		u64 u = v < 0 ? (u64)(-v) : (u64)v;
		do { buf[k++] = (char)('0' + (int)(u % 10)); u /= 10; } while (u);
		if (v < 0) c('-');
		while (k) c(buf[--k]);
	}
};

/* bns_cnt_ambi (bntseq.c:380-401): the N bases of the ONE hole the binary search lands on */
__device__ __forceinline__ int se_cnt_ambi(const SeArgs &a, i64 pos_f, int len, int *ref_id)
{
	int left = 0, right = a.n_holes, nn = 0;
	const int rid = t_pos2rid(a.ctg, pos_f);
	*ref_id = rid < 0 ? 0 : rid;
	while (left < right) {
		const int mid = (left + right) >> 1;
		const i64 ao = a.amb_off[mid], al = a.amb_len[mid];
		if (pos_f >= ao + al) left = mid + 1;
		else if (pos_f + len <= ao) right = mid;
		else {
			if (pos_f >= ao) nn += ao + al < pos_f + len ? (int)(ao + al - pos_f) : len;
			else nn += ao + al < pos_f + len ? (int)al : (int)(len - (ao - pos_f));
			break;
		}
	}
	return nn;
}

/* one read's bases as bwa_refine_gapped aligns them: seq (forward) or rseq (reversed, complemented under COMPREAD) */
struct SeRead {
	const uint8_t *r; int len; bool rev, comp;
	__device__ __forceinline__ int at(int y) const { if (!rev) return r[y]; const int c = r[len - 1 - y]; return comp && c < 4 ? 3 - c : c; }
};

/* bwa_cal_md1 (bwase.c:201-249) on the searched bases and the refined CIGAR (16-bit entries; NULL: ungapped): returns NM and
 * writes MD to o.  An N in the read is a mismatch; I and D count their lengths; the x+z < l_pac guards stay */
static __device__ int se_md(const DevIndex &ix, i64 l_pac, const u32 *cig, int n_cigar, const SeRead &q, i64 pos, SeOut *o)
{
	i64 x = pos, y = 0;
	int u = 0, nm = 0;
	if (cig) {
		for (int k = 0; k < n_cigar; ++k) {
			const int op = se_op(cig[k]), l = se_len(cig[k]);
			if (op == 0) {
				for (int z = 0; z < l && x + z < l_pac; ++z) {
					const int c = bwag_pac_base(ix.pac, x + z), b = q.at((int)(y + z));
					if (b > 3 || c != b) { o->d(u); o->c("ACGTN"[c]); ++nm; u = 0; } else ++u;
				}
				x += l; y += l;
			} else if (op == 1 || op == 3) {
				y += l;
				if (op == 1) nm += l;
			} else if (op == 2) {
				o->d(u); o->c('^');
				for (int z = 0; z < l && x + z < l_pac; ++z) o->c("ACGT"[bwag_pac_base(ix.pac, x + z)]);
				u = 0; x += l; nm += l;
			}
		}
	} else {
		for (int z = 0; z < q.len && x + z < l_pac; ++z) {
			const int c = bwag_pac_base(ix.pac, x + z), b = q.at(z);
			if (b > 3 || c != b) { o->d(u); o->c("ACGTN"[c]); ++nm; u = 0; } else ++u;
		}
	}
	o->d(u);
	return nm;
}

/* the chosen hit's CIGAR after bwa_correct_trimmed (bwase.c:251-285), in 16-bit entries: [lead] base[0, nb) [trail], base entry mi
 * replaced by mv (an S extended by the clipped length, with the reference's 16-bit wrap) */
struct SeCig {
	const u32 *b; int nb, n, mi; bool lead, trail; u32 lv, tv, mv;
	__device__ __forceinline__ u32 at(int k) const
	{
		if (lead) { if (k == 0) return lv; --k; }
		if (k < nb) return k == mi ? mv : b[k];
		return tv;
	}
};
__device__ __forceinline__ SeCig se_corrected(const u32 *cig, int n_cigar, int len, int full_len, int strand)
{
	SeCig e;
	e.b = cig; e.nb = cig ? n_cigar : 0; e.mi = -1; e.lead = e.trail = false; e.lv = e.tv = e.mv = 0;
	const u32 clip = (u32)(full_len - len);
	if (clip) {
		if (!strand) {
			if (cig && se_op(cig[n_cigar - 1]) == 3) { e.mi = n_cigar - 1; e.mv = (uint16_t)(cig[n_cigar - 1] + clip); }
			else {
				if (!cig) { e.lead = true; e.lv = se_cigar16(0, (u32)len); }
				e.trail = true; e.tv = se_cigar16(3, clip);
			}
		} else {
			if (cig && se_op(cig[0]) == 3) { e.mi = 0; e.mv = (uint16_t)(cig[0] + clip); }
			else {
				e.lead = true; e.lv = se_cigar16(3, clip);
				if (!cig) { e.trail = true; e.tv = se_cigar16(0, (u32)len); }
			}
		}
	}
	e.n = e.nb + e.lead + e.trail;
	return e;
}

#endif
