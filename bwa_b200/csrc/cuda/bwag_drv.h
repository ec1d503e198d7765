/* bwag_drv.h -- what the host drivers of the device-batch C ABI share (internal, not installed): error reporting, the buffers,
 * the context, the batch and its lane.  bwag_api.cu holds the context, the index blob, residency, batch lifetime, stats and the
 * helpers declared here; each command's driver sits beside its kernels (bwag_fastmap.cu, bwag_aln.cu, bwag_samse.cu,
 * bwag_sampe.cu, bwag_pemerge.cu) and mem's stages 1-4 in bwag_mem.cu. */
#ifndef BWAG_DRV_H
#define BWAG_DRV_H
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include "bwag_dev.cuh"
#include "bwag_kernels.h"

#ifdef BWAG_CUSIM
/* emulator build only: the device blocks the drivers hold (bwag_cusim_live_dev_blocks), so that tests can check that a context
 * and its batches give back every one of them */
extern long bwag_cusim_dev_blocks;
static inline cudaError_t bwag_cusim_malloc(void **p, size_t n) { cudaError_t e = cudaMalloc(p, n); if (e == cudaSuccess) __atomic_add_fetch(&bwag_cusim_dev_blocks, 1, __ATOMIC_RELAXED); return e; }
static inline cudaError_t bwag_cusim_free(void *p) { if (p) __atomic_sub_fetch(&bwag_cusim_dev_blocks, 1, __ATOMIC_RELAXED); return cudaFree(p); }
#define cudaMalloc bwag_cusim_malloc
#define cudaFree bwag_cusim_free
#endif

int set_err(const char *fmt, ...);   /* sets what bwag_last_error() returns; returns 1 */
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return set_err("%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); } while (0)
#define CKP(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_err("%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); return 0; } } while (0)

#define K1_SMEM_MAX (200 * 1024)
#define K4_SMEM_MAX (96 * 1024)
#define K4L_SMEM_MAX (200 * 1024)

/* device counters, mirrored in pinned host memory */
struct Counters {
	int next_read, next_task, max_rlen, next_read3;
	u64 next_seed;
	u64 n_intv, n_seeds;
	u64 occ_touches, sa_touches, ext_cells, glb_cells;
	u64 n_cig, n_md;
	u32 flags, n_pre;   /* n_pre: CIGARs made by the lane-per-request kernel (K5L) */
	/* stage 4 */
	u64 t_dregs, t_tasks, t_max_z, t_text, t_complex;
	int t_max_lq, t_max_rl;
	int n_many;      /* reads with more chains than the lane kernel takes (K3) */
	int n_big;       /* reads with more seeds than the on-chip form of K3 takes */
	u32 n_swtasks;   /* local alignments the seed-level filter of long reads asks for (K3) */
	u64 fm_total[3]; /* fastmap: lines, suffix-array rows and text bytes of the batch (totals of the scans) */
	int aln_next;    /* aln: next read of the work list, reads listed for another run, why (1 arena, 2 pool), hits reserved in the pool, hits in all */
	u32 aln_redo, aln_flags;
	u64 aln_pool, aln_total;
	u64 se_total, se_run, se_cells;   /* samse: text bytes of the batch (scan total), global alignments run and their cells */
	int se_next, se_past;             /* samse: next refinement task; n_reads - the first read whose window runs past the forward strand (0: none) */
	u64 pm_total;                     /* pemerge: text bytes of the batch (scan total) */
};

/* device and pinned host buffers that only grow (buf_reserve, hbuf_reserve) and free themselves */
struct DevBuf {
	void *p = 0; size_t cap = 0;
	DevBuf() = default;
	DevBuf(const DevBuf &) = delete;
	DevBuf &operator=(const DevBuf &) = delete;
	~DevBuf() { if (p) cudaFree(p); }
};
struct HostBuf {
	void *p = 0; size_t cap = 0;
	HostBuf() = default;
	HostBuf(const HostBuf &) = delete;
	HostBuf &operator=(const HostBuf &) = delete;
	~HostBuf() { if (p) cudaFreeHost(p); }
};

/* what a sequence of launches needs: a stream, its events and counters, the index view and the scratch of K1/K4/K5/K5L.  The
 * context has one (densify, the table build, verify, the table uploads; its stats are the context's totals), each batch has
 * its own, so that batches can overlap. */
struct Lane {
	cudaStream_t stream = 0;
	cudaEvent_t ev0 = 0, ev1 = 0, ev_wait = 0;
	Counters *d_cnt = 0, *h_cnt = 0;
	bwag_stats_t st = {};
	DevIndex ix = {};            /* a batch's: without the short-string table if the batch began under baseline */
	int baseline = 0;            /* bwag_ctx_baseline(): first row sweeps in K4/K5 and no table lookups */
	DevBuf s_k1, s_k1f, s_n3, s_eh, s_rseq, s_qseq, s_z, s_wcig, s_wmd, s_pack, s_zl;
	~Lane();
};
int lane_init(Lane *l);

struct bwag_ctx {
	int device, own_blob, n_sm;
	int imported;                /* blob, dense SA and table belong to another process (bwag_ctx_import): closed, not freed */
	size_t map_bytes[3];         /* (emulator build) sizes of the three shared mappings */
	void *blob;
	u64 *dense_sa;
	ulonglong2 *ktab;            /* short-string table (bwag_ctx_build_ktab) */
	Lane lane;
	int grid_k1f, grid_k2, grid_k4, grid_k5;
	int k3s_blocks;   /* resident blocks per SM of k_chain_sm (occupancy API) */
#define N_SPARE 12
	struct bwag_batch *spare[N_SPARE]; /* batch objects (lane, device and pinned buffers) kept for later batches */
	pthread_mutex_t mu;
	/* stage 4: contig table (offsets, lengths, ALT flags, names) and log(i) table, resident once per context */
	DevBuf tail; TailCtg tctg; const double *d_logtab; int have_ctg;
	/* samse: the reference's holes (bns->ambs), for bns_cnt_ambi */
	DevBuf ambs; int n_holes, have_ambs;
};

struct bwag_batch {
	bwag_ctx_t *ctx;
	Lane lane;
	int n;
	i64 total_bases;
	int max_len;
	const i64 *h_off;
	DevBuf d_codes, d_off;
	/* stage 1 */
	DevBuf d_intv_beg, d_intv_n, d_intv, d_seed_beg, d_rbeg;
	HostBuf h_intv_beg, h_intv_n, h_intv, h_seed_beg, h_rbeg;
	/* stage 2 */
	DevBuf d_chain_off, d_chains, d_seeds, d_regs, d_nregs;
	DevBuf d_chain_beg, d_chain_cnt, d_reg_base, d_chain_rid, d_chain_frac, d_cregs, d_creg_beg, d_ctg;
	DevBuf s_bt, s_sn, s_ch, s_order, s_idx, s_keys;
	HostBuf h_regs, h_nregs, h_cregs, h_creg_beg, h_tmp;
	i64 n_intv, n_seeds;         /* pool sizes left in HBM by the last bwag_seed */
	int seeded;
	/* stage 3 */
	DevBuf d_tasks, d_res, d_cig, d_md;
	HostBuf h_res, h_cig, h_md;
	/* stage 4 */
	DevBuf d_dregs, d_dreg_beg, d_dreg_n, d_task_beg, d_cflag, d_pe_is, d_rec, d_text, d_ptab;
	DevBuf d_swtasks, d_swres, d_swpool, d_swscratch; HostBuf h_swres;   /* K6 */
	DevBuf d_hsp, d_flt_nchn; HostBuf h_hsp;   /* seed-level filter of long reads (K3/K3b) */
	DevBuf d_k3big;                            /* reads k_chain_sm leaves to k_chain */
	DevBuf d_pre_n, d_pre_score, d_pre_cig;    /* K5L results for the warp kernel */
	DevBuf d_sel;
	HostBuf h_pe_is, h_cflag, h_rec, h_text, h_ptab;
	/* fastmap (bwag_fastmap.cu) */
	DevBuf d_fm_lbeg, d_fm_lines, d_fm_nrow, d_fm_rbeg, d_fm_rows, d_fm_tlen, d_fm_tbeg, d_fm_text, d_fm_toff;
	HostBuf h_fm_text, h_fm_off;
	/* aln (bwag_aln.cu) */
	DevBuf d_aln_md, d_aln_n, d_aln_beg, d_aln_pool, d_aln_redo[2], d_aln_off, d_aln_out, d_aln_arena;
	HostBuf h_aln_n, h_aln_off, h_aln_out;
	/* samse (bwag_samse.cu) */
	DevBuf d_se_reads, d_se_multi, d_se_bc, d_se_rows, d_se_pos, d_se_mpos, d_se_flags, d_se_tasks, d_se_mtask, d_se_cig, d_se_ncig, d_se_scratch, d_se_tlen, d_se_tbeg, d_se_rec, d_se_text, d_se_nm;
	HostBuf h_se_tasks, h_se_mtask, h_se_rec, h_se_text;
	/* sampe (bwag_sampe.cu; the rest of its buffers are samse's) */
	DevBuf d_pe_rlen, d_pe_reads, d_pe_gtasks, d_pe_gres, d_pe_gcig, d_pe_pool;
	HostBuf h_pe_pos, h_pe_gres, h_pe_gcig;
	/* pemerge (bwag_pemerge.cu; K6's buffers hold its tasks, codes and alignments) */
	DevBuf d_pm_qual, d_pm_hasq, d_pm_names, d_pm_noff, d_pm_q, d_pm_code, d_pm_ovl, d_pm_tlen, d_pm_tbeg, d_pm_text, d_pm_cnt;
	HostBuf h_pm_text, h_pm_cnt;
	/* maxk (bwag_maxk.cu) */
	DevBuf d_mk_woff, d_mk_cnt, d_mk_ctr, d_mk_scratch;
	HostBuf h_mk_woff, h_mk_ctr;
	int tail_ready;             /* bwag_tail_regs ran on this batch */
	int regs_on_device;          /* bwag_chain_extend left the regions in HBM */
};

/* bwag_api.cu */
int buf_reserve(DevBuf *b, size_t bytes);
int hbuf_reserve(HostBuf *b, size_t bytes);
int buf_grow_keep(Lane *c, DevBuf *b, size_t keep, size_t bytes);   /* grows and keeps the first `keep` bytes */
int reset_counters(Lane *c);
int fetch_counters(Lane *c);
cudaError_t stream_wait(Lane *c);
double elapsed_at(Lane *c, const char *stage, const char *file, int line);   /* ms from ev0 to ev1 */
int fm_grid(const bwag_ctx_t *c, i64 n_items);   /* blocks of 128 for one lane per item, at most 16 per SM */
int run_sa(bwag_batch_t *b, i64 *rows, i64 n);
int occ_upload(void *d, const bwt_t *bwt, u64 sb[BWAG_MAX_SB][4]);   /* a .bwt's words, re-packed into 32-byte blocks on the device */
#define H2D(c, dst, src, bytes) do { CK(cudaMemcpyAsync((dst), (src), (bytes), cudaMemcpyHostToDevice, (c)->stream)); (c)->st.h2d_bytes += (u64)(bytes); } while (0)
#define D2H(c, dst, src, bytes) do { CK(cudaMemcpyAsync((dst), (src), (bytes), cudaMemcpyDeviceToHost, (c)->stream)); (c)->st.d2h_bytes += (u64)(bytes); } while (0)

/* bwag_mem.cu */
int localsw_on_device(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, int max_q, int max_t);
int run_global(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, int cap_q, int cap_r, i64 cap_z, i64 n_aln, i64 *nc_out, i64 *nm_out);
struct FmK1 { int min_intv; u64 max_intv; };   /* fastmap's form of K1 (k_smem_fm): -i and -I */
int seed_impl(bwag_batch_t *b, const bwag_seed_par_t *par, const FmK1 *fm, bwag_seeds_t *out);

/* bwag_samse.cu: what sampe's P6/P7 share with samse's S3/S4 */
struct SeList { SeTask *tasks; int n_tasks = 0, cap_q = 1, cap_r = 1; i64 n_cig = 0, cap_z = 1; };
int se_list_read(SeList &L, const bwag_se_read_t &p, const bwag_se_hit_t *multi, int r, bool gapped, int *mtask, int n);
void se_args(bwag_batch_t *b, SeArgs &a, int n_tasks, i64 nm, int mode, int max_top2, i64 l_bc, int l_rg);
i64 se_scratch(bwag_batch_t *b, int n_tasks, int cap_q, int cap_r, i64 cap_z, int **eh, uint8_t **rseq, uint8_t **qseq, uint8_t **z);
#endif
