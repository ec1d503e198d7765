/* bwag_kernels.h -- argument blocks and launch constants shared by the kernels and their host drivers. */
#ifndef BWAG_KERNELS_H
#define BWAG_KERNELS_H
#include "bwag_dev.cuh"

#define K1_THREADS 128
#define K1F_THREADS 128
#ifndef K1_SLOTS
#ifdef K1_PACKED8
#define K1_SLOTS 8
#else
#define K1_SLOTS 4
#endif
#endif
//       /* candidate-list entries per list kept in shared memory */
#define K1C_SLOTS 8   /* the same for k_smem_c, which keeps no byte copy of the read in shared memory and has the room */
#define K1B_THREADS 128
#define K2_THREADS 128
#define K3_THREADS 128
/* K3 on chip (k_chain_sm): reads with at most K3S_CAP seeds keep their chaining workspace in K3S_SMEM bytes of shared memory per
 * block (62 bytes per seed, 21 per B-tree node, 4 of traversal stack, per lane; bwag_chain.cu) */
#ifndef K3S_CAP
#define K3S_CAP 16
#endif
#define K3S_THREADS 64
#define K3S_SMEM (K3S_THREADS * (62 * K3S_CAP + 21 * (1 + (K3S_CAP - 1) / 4) + 4))
#define K4_THREADS 128
#define K5_THREADS 128
#define K4L_THREADS 128   /* lane-per-read extension kernel (bwag_extend_lane.cu) */
#ifndef K4L_MINB
#define K4L_MINB 3
#endif

struct Intv;

struct SeedArgs {
	/* batch */
	const uint8_t *codes; const i64 *off; int n_reads;
	/* parameters (bwag_seed_par_t) */
	int min_seed_len, split_len, split_width, max_occ; u64 max_mem_intv;
	/* per-group scratch */
	Intv *scratch; int cap_list, cap_mem;
	int qstride;                                   /* bytes of a lane's shared read slot (0: read the bases from global memory) */
	int pstride;                                   /* bytes of a lane's 2-bit packed copy of the read (0: no short-string table lookups in K1) */
	int nstride;                                   /* variant K1_PACKED8 only: bytes of a lane's N bitmap (the byte copy of the read is dropped: qstride = 0) */
	Intv *stage3; int cap3; int *n3; int *next_read3;   /* third-pass seeds: cap3 slots per read, filled by K1f */
	int post_copies3;                              /* k_smem_c: K1 only reserves the room of the third-pass seeds in the read's slice, K1b (all lanes busy) copies them */
	const u32 *packed;                             /* k_pack_reads: 2-bit copy of every read, read r at word (off[r] >> 4) + 2 r */
	const u32 *nmask;                              /* k_pack_reads: one bit per base (ambiguous), read r at word (off[r] >> 5) + 2 r; variant K1_PACKED8 only */
	const u32 *hasn;                               /* k_pack_reads: per read, non-zero if it has an ambiguous base (k_smem_c looks at the bytes of such reads only) */
	/* outputs */
	i64 *intv_beg; int *intv_n; bwtintv_t *intv; i64 *seed_beg; i64 *rbeg;
	i64 cap_intv, cap_seeds;
	/* counters: [0] next read, n_intv, n_seeds, occ touches, flags */
	int *next_read; u64 *n_intv; u64 *n_seeds; u64 *occ_touches; u32 *flags;
#ifdef BWAG_K1_CLOCKS
	u64 *k1clk;   /* BWAG_K1CLK_LANE_WORDS counters of k_smem_c (include/bwa_b200_dev.h) */
#endif
};

struct SaArgs { i64 *rbeg; i64 n; u64 *next; u64 *sa_touches; };

/* one record per region for the download of the fused chain+extend path */
struct ChainArgs {
	const i64 *off; int n_reads;
	const i64 *intv_beg; const int *intv_n; const bwtintv_t *intv; const i64 *seed_beg; const i64 *rbeg;
	int w, max_chain_gap, max_occ, min_seed_len, min_chain_weight, max_chain_extend; float mask_level, drop_ratio;
	int a, o_del, e_del, o_ins, e_ins;
	i64 l_pac; int n_seqs; const i64 *ctg_off; const int *ctg_len; const uint8_t *ctg_alt;
	void *s_bt, *s_sn, *s_ch; int *s_order, *s_idx; u64 *s_keys;     /* scratch, indexed by seed slot */
	bwag_xchain_t *xchains; bwag_xseed_t *xseeds; int *chain_rid; float *chain_frac;   /* outputs, indexed by seed slot */
	i64 *chain_beg, *reg_base; int *n_chains;                          /* per read */
	int *max_rlen;                                                     /* longest reference window of any chain (sizes K4's scratch) */
	int *n_many; int many;                                             /* counts the reads with more than `many` chains (they go to the warp-per-read extension kernel) */
	/* seed-level filter of long reads (mem_flt_chained_seeds): threshold by read length (-1: inactive; NULL: no read of the chunk is
	 * long enough), the local alignments k_chain asks for, their results for k_chain_emit, per read the number of chains parked */
	const int *hsp_tab; bwag_swtask_t *sw_tasks; u32 *n_swtasks; const bwag_swres_t *sw_res; int *flt_nchn;
	int *big; int *n_big;                                              /* reads k_chain_sm leaves to k_chain (too many seeds), their count */
	u32 *k3clk;   /* builds with -DBWAG_K3_CLOCKS only: per read seeds, chains, cycles of chaining, mem_chain_flt, chain_emit */
};

struct RegCompactArgs {
	int n_reads; const int *n_regs; const bwag_xreg_t *regs; const i64 *reg_base, *chain_beg; const int *chain_rid; const float *chain_frac;
	i64 *out_beg; bwag_creg_t *out; u64 *total;
};

struct ExtArgs {
	const uint8_t *codes; const i64 *off; int n_reads;
	bwag_sw_par_t par;
	const i64 *chain_beg; const int *chain_cnt; const i64 *reg_base;   /* per read: its chains in chains[], where its regions go in regs[] */
	const bwag_xchain_t *chains; const bwag_xseed_t *seeds;
	bwag_xreg_t *regs; int32_t *n_regs;
	/* per-warp scratch: H, E (int32 each, cap_q+2), reference window (cap_r bytes) */
	int *eh; uint8_t *rseq; int cap_q, cap_r;
	int smem_per_warp;   /* k_extend_sm: bytes of shared scratch per warp = 8*(cap_q+2) + cap_r + cap_q, rounded up to 16 */
	int min_seed;        /* no seed is shorter than this (0 if unknown): an extension has at most cap_q - min_seed query columns */
	int chain_lo, chain_hi;   /* this launch takes the reads whose number of chains lies in [chain_lo, chain_hi]: reads with many chains go to the warp-per-read kernel */
	int *next_read; u64 *cells; u32 *flags;
};

struct GlbArgs {
	const uint8_t *codes; const i64 *off;
	bwag_sw_par_t par;
	const bwag_gtask_t *tasks; int n_tasks;
	bwag_gres_t *res; u32 *cigar; char *md;   /* compact output pools, filled with atomicAdd on n_cig / n_md */
	i64 cap_cig, cap_md; u64 *n_cig, *n_md;
	u32 *w_cig; char *w_md; int cap_wcig, cap_wmd;   /* per-warp staging of one task's CIGAR / MD */
	int *eh; uint8_t *rseq; uint8_t *qseq; uint8_t *z;   /* per-warp scratch: H/E rows, reference, query, backtrack matrix */
	int cap_q, cap_r; i64 cap_z;
	int smem_per_warp;   /* k_global_sm: 8*(cap_q+2) + cap_r + cap_q + 2, rounded up to 16, + z_sm_bytes */
	int z_sm_bytes;      /* backtrack bytes per warp kept in shared memory (tasks whose n_col x rows fit); 0: all in global memory */
	int *next_task; u64 *cells; u32 *flags;
	const int *pre_n, *pre_score; const u32 *pre_cig;   /* CIGARs the lane-per-request kernel made already (pre_n[t] < 0: none), K5L_MAXCIG words per request */
};

/* K5L (bwag_global_lane.cu): DP + backtrack of short-read CIGAR requests, one lane per request */
#define K5L_THREADS 128
#define K5L_RING 64      /* (h, e) slots per lane: bands up to 2w+2 = 64 */
#define K5L_QWORDS 64    /* query words per lane: reads up to 256 bases */
#define K5L_MAXCIG 16    /* CIGAR operations per request; longer ones are left to the warp kernel */
struct GlbLaneArgs {
	const uint8_t *codes; const i64 *off;
	bwag_sw_par_t par;
	const bwag_gtask_t *tasks; int n_tasks;
	int *pre_n, *pre_score; u32 *pre_cig;
	uint8_t *z; i64 cap_z;   /* direction bytes: cap_z cells per lane, byte-interleaved by lane within a warp's slice */
	int *next_task; u64 *cells; u32 *n_pre;
};

/* ---- stage 4 (device tail, bwag_tail.cu) ---- */
struct TailCtg { i64 l_pac; int n_seqs; const i64 *off; const int *len; const uint8_t *alt; const char *names; const int *name_off; };   /* bntann1_t columns; names back to back, name_off[n_seqs+1] */
__device__ __forceinline__ int t_pos2rid(const TailCtg &c, i64 pos_f)   /* bntseq.c:354-368 */
{
	int lo = 0, hi = c.n_seqs, mid = 0;
	if (pos_f >= c.l_pac) return -1;
	while (lo < hi) {
		mid = (lo + hi) >> 1;
		if (pos_f < c.off[mid]) hi = mid;
		else if (mid == c.n_seqs - 1 || pos_f < c.off[mid + 1]) break;
		else lo = mid + 1;
	}
	return mid;
}

struct TailRegsArgs {
	int n_reads, pe;
	mem_opt_t opt;
	TailCtg ctg;
	/* K4's output */
	const int *n_raw; const bwag_xreg_t *xregs; const i64 *reg_base, *chain_beg; const int *chain_rid; const float *chain_frac;
	/* per read: its de-duplicated regions in dregs[], its CIGAR requests in tasks[] (request k belongs to region k), why it left the simple path (0: it did not) */
	mem_alnreg_t *dregs; i64 *dreg_beg; int *dreg_n; i64 *task_beg; uint8_t *cflag; i64 cap_dregs;
	bwag_gtask_t *tasks; i64 cap_tasks;
	u64 *pe_is;                       /* per pair: mem_pestat's candidate ((orientation+1) << 48 | insert size, 0: none) */
	u64 *n_dregs, *n_tasks, *max_z; int *max_lq, *max_rl;
};

#ifndef TAIL_SLOT_MAX
#define TAIL_SLOT_MAX 512   /* bytes of shared memory per lane of k_tail_sam (at most 64 KB per 128-lane block) */
#endif
#define TAIL_SAM_SMEM_MAX (128 * TAIL_SLOT_MAX)
struct TailSamArgs {
	int n_reads, pe;
	mem_opt_t opt;
	TailCtg ctg;
	mem_pestat_t pes[4];
	const double *ptab[4];            /* per orientation: .721*log(2*erfc(|d-avg|/std/sqrt2))*a for d = low..high (host libm), or 0 */
	const double *logtab;             /* log(i), i < 4096 (host libm) */
	i64 n_processed;
	const uint8_t *codes; const i64 *off;
	const mem_alnreg_t *dregs; const i64 *dreg_beg; const int *dreg_n; const i64 *task_beg; const uint8_t *cflag;
	const bwag_gres_t *res; const u32 *cigar; const char *md;
	const char *rg; int l_rg;
	bwag_samrec_t *rec; char *text; i64 cap_text; u64 *n_text, *n_complex;
	int slot;                         /* bytes of shared memory per lane for its record (a multiple of 16) */
};

/* ---- K6 (bwag_localsw.cu) ---- */
struct SwArgs {
	const bwag_swtask_t *tasks; int n_tasks;
	bwag_sw_par_t par;
	const uint8_t *codes;            /* the batch's reads (BWAG_SWF_QREAD) */
	const uint8_t *pool;             /* caller bytes (queries / targets given explicitly) */
	bwag_swres_t *res;
	unsigned char *scratch; i64 per_thread; int cap_n, cap_q, cap_t;   /* per lane: 4 x short[cap_n], u64[cap_t], query[cap_q], target[cap_t] */
	int *next_task; u32 *flags;
};

/* ---- fastmap (bwag_fastmap.cu) ---- */
#define FM_SCAN_THREADS 1024
struct FmArgs {
	int n_reads; i64 n_lines;
	u64 max_iwidth;                                   /* -w as the reference compares it: (uint64_t)(int64_t)w */
	TailCtg ctg;
	const i64 *intv_beg; const int *intv_n; const bwtintv_t *intv;   /* K1's pool */
	const i64 *lbeg;                                  /* [n_reads+1] first line of each read (scan of intv_n) */
	bwtintv_t *lines; i64 *nrow;                      /* [n_lines] the matches in read order, rows each one wants */
	const i64 *rbeg; i64 *rows;                       /* [n_lines+1] first row of each line (scan of nrow); the rows, resolved by K2 */
	i64 *tlen; const i64 *tbeg; char *text;           /* [n_lines] bytes per line, [n_lines+1] their scan, the text */
	i64 *toff;                                        /* [n_reads+1] first byte of each read's text */
};
__global__ void k_fm_scan32(const int *in, i64 n, i64 *out, u64 *total);
__global__ void k_fm_scan64(const i64 *in, i64 n, i64 *out, u64 *total);
__global__ void k_fm_lines(FmArgs a);
__global__ void k_fm_rows(FmArgs a);
__global__ void k_fm_text(FmArgs a, int write);
__global__ void k_fm_readoff(FmArgs a);
__global__ void k_smem_fm(DevIndex ix, SeedArgs a, int min_intv, u64 max_intv);   /* K1 listing SMEMs as `bwa fastmap` does (bwag_smem.cu) */

/* ---- aln (bwag_aln.cu) ---- */
#define ALN_THREADS 128
struct AlnNode { u64 k, l; u32 pos, cnt, id; int next; };   /* a queue entry, 32 bytes: see bwag_aln.cu */
/* a lane's arena: bucket heads, bucket bitmap, widths of the read and of its seed (w, bid), then the nodes */
struct AlnLayout { i64 heads, mask, ww, wb, sw, sb, nodes, bytes; };
__host__ __device__ __forceinline__ AlnLayout aln_layout(int n_buckets, int max_len, int seed_cap, i64 cap_nodes)
{
	AlnLayout L;
	i64 o = 0;
	L.heads = o; o += (4 * (i64)n_buckets + 15) & ~(i64)15;
	L.mask = o;  o += (8 * (i64)((n_buckets + 63) / 64) + 15) & ~(i64)15;
	L.ww = o;    o += (8 * (i64)(max_len + 1) + 15) & ~(i64)15;
	L.wb = o;    o += (4 * (i64)(max_len + 1) + 15) & ~(i64)15;
	L.sw = o;    o += (8 * (i64)(seed_cap + 1) + 15) & ~(i64)15;
	L.sb = o;    o += (4 * (i64)(seed_cap + 1) + 15) & ~(i64)15;
	L.nodes = o; o += (i64)sizeof(AlnNode) * cap_nodes;
	L.bytes = o;
	return L;
}
struct AlnArgs {
	const uint8_t *codes; const i64 *off;
	bwag_aln_par_t par;
	int n_buckets;                                    /* queue scores 0 .. n_buckets-1 */
	const int *work; int n_work;                      /* the reads to search (NULL: 0 .. n_work-1) */
	unsigned char *arena; i64 lane_bytes;             /* per lane: bucket heads and bitmap, widths, cap_nodes 32-byte nodes */
	int cap_nodes, max_len, seed_cap, n_lanes;
	int *n_aln; i64 *hit_beg;                         /* [n_reads] */
	bwag_aln1_t *pool; i64 cap_pool; u64 *n_pool;     /* every read's hits, at hit_beg[r] */
	int *redo; u32 *n_redo; u32 *flags;               /* reads to search again: 1 = their arena overflowed, 2 = the pool did */
	int *next;
};
__global__ void k_aln(DevIndex ix, AlnArgs a);
__global__ void k_aln_gather(int n_reads, const int *n_aln, const i64 *hit_beg, const bwag_aln1_t *pool, const i64 *off, bwag_aln1_t *out);

/* ---- samse (bwag_samse.cu) ---- */
#define SE_THREADS 128
struct SeTask { int read, slot; i64 cig_off; };   /* a gapped hit: slot -1 = the read's chosen hit, else its XA candidate multi[slot] */
struct SeArgs {
	int n_reads; i64 n_multi; int n_tasks;
	int mode, max_top2; const char *rg; int l_rg;
	TailCtg ctg; int n_holes; const i64 *amb_off; const int *amb_len;
	const uint8_t *codes; const i64 *off;            /* the whole reads */
	const bwag_se_read_t *reads; const bwag_se_hit_t *multi; const char *bc;
	i64 *rows;                                        /* [n_reads + n_multi]: SA rows, resolved in place by K2 */
	i64 *pos; uint8_t *strand, *mapped;               /* [n_reads]: bwa_sa2pos of the chosen hit (before refinement) */
	i64 *mpos; uint8_t *mstrand, *mkeep;              /* [n_multi]: the candidates' positions; kept in XA */
	const SeTask *tasks; const int *main_task, *multi_task;   /* the gapped hits; per read / candidate its task or -1 */
	u32 *cig; int *ncig; int *tshift;                 /* per task: CIGAR at cig_off, its length (0: not run), the start's shift */
	int *eh; uint8_t *rseq, *qseq, *z; int cap_q, cap_r; i64 cap_z;   /* per-warp scratch of the refinement */
	int *next_task; int *past_end; u64 *n_run, *cells;
	i64 *tlen; const i64 *tbeg; char *text; bwag_samrec_t *rec;   /* the records: bytes per read, their scan, the text */
	int *nm;                                          /* [n_reads] NM of each mapped read, from pass 0 of S4 for pass 1 */
};
__global__ void k_se_rows(SeArgs a);
__global__ void k_se_pos(SeArgs a);
__global__ void k_se_refine(DevIndex ix, SeArgs a);
__global__ void k_se_text(DevIndex ix, SeArgs a, int write);

/* ---- sampe (bwag_sampe.cu) ---- */
struct PePosArgs { i64 n, l_pac; const i64 *rows; const int *ref_len; i64 *pos; uint8_t *strand; };   /* [n] rows, [2n] the rest */
struct PeGlbArgs {
	int n_tasks; const bwag_pe_gtask_t *tasks; bwag_pe_gres_t *res; u32 *cig; const uint8_t *pool;
	int *eh; uint8_t *rseq, *z; int cap_q, cap_r; i64 cap_z;   /* per-warp scratch */
	int *next_task; u64 *cells;
};
__global__ void k_pe_pos(PePosArgs a);
__global__ void k_pe_global(DevIndex ix, PeGlbArgs a);
__global__ void k_pe_text(DevIndex ix, SeArgs a, const bwag_pe_read_t *pe, int write);

/* ---- pemerge (bwag_pemerge.cu) ---- */
struct PemArgs {
	int n_pairs, T, q_thres, q_def, flag;
	const uint8_t *raw; const i64 *off;              /* the batch: raw sequence bytes; read 1 of pair i is read 2i, read 2 is read 2i + 1 */
	const uint8_t *qual; const uint8_t *has_qual;    /* raw quality bytes at the reads' offsets; per read: it has a quality string */
	const char *names; const i64 *name_off;          /* [2 n_pairs + 1] */
	uint8_t *s, *q;                                  /* codes (K6's pool) and qualities - 33: s0 / q0 at read 1's offset, s1 / q1 at read 2's */
	bwag_swtask_t *tasks; const bwag_swres_t *res;   /* K6: task i is pair i */
	int8_t *code; int *ovl;                          /* [n_pairs] 0 merged, -1 .. -8 why not, 1 not tried; the overlap of a merge */
	i64 *tlen; const i64 *tbeg; char *text;          /* the records: bytes per pair, their scan, the text */
	u64 *cnt;                                        /* [9] pairs per outcome */
};
__global__ void k_pem_encode(PemArgs a);
__global__ void k_pem_decide(PemArgs a);
__global__ void k_pem_text(PemArgs a, int write);

__global__ void k_chain_emit(ChainArgs a);
__global__ void k_global_lane(DevIndex ix, GlbLaneArgs a);
__global__ void k_localsw(DevIndex ix, SwArgs a);
__global__ void k_localsw_warp(DevIndex ix, SwArgs a);
__global__ void k_occ_pack(DevIndex ix, uint4 *bwt, u64 n_blocks);
__global__ void k_ktab_build(DevIndex ix, ulonglong2 *tab, int K);
__global__ void k_pack_reads(const uint8_t *codes, const i64 *off, int n_reads, u32 *packed, u32 *nmask, u32 *hasn);
__global__ void k_smem(DevIndex ix, SeedArgs a);
#ifndef K1_PACKED8
__global__ void k_smem_c(DevIndex ix, SeedArgs a);   /* short candidates as mask bits, matches appended at once (bwag_smem.cu) */
#endif
__global__ void k_smem_fwd(DevIndex ix, SeedArgs a);
__global__ void k_seed_post(SeedArgs a);
__global__ void k_sa(DevIndex ix, SaArgs a);
__global__ void k_sa_densify(DevIndex ix, u64 *out, int out_shift, u64 n_out);
__global__ void k_index_verify(DevIndex ix, u64 first, u64 stride, u64 n_check, u64 *out);
__global__ void k_chain(ChainArgs a);
__global__ void k_chain_sm(ChainArgs a);
__global__ void k_regs_compact(RegCompactArgs a);
__global__ void k_regs_compact_sel(RegCompactArgs a, const int *sel, int n_sel, int *out_n);
__global__ void k_extend(DevIndex ix, ExtArgs a);
__global__ void k_extend_sm(DevIndex ix, ExtArgs a);
__global__ void k_extend_fast(DevIndex ix, ExtArgs a);
__global__ void k_extend_sm_fast(DevIndex ix, ExtArgs a);
__global__ void k_extend_lane(DevIndex ix, ExtArgs a);
__global__ void k_global(DevIndex ix, GlbArgs a);
__global__ void k_global_sm(DevIndex ix, GlbArgs a);
__global__ void k_global_fast(DevIndex ix, GlbArgs a);
__global__ void k_global_sm_fast(DevIndex ix, GlbArgs a);
__global__ void k_tail_regs(TailRegsArgs a);
__global__ void k_tail_sam(TailSamArgs g);

#endif
