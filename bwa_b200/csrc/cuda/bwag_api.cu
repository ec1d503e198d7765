/* bwag_api.cu -- host side of the device-batch C ABI (include/bwa_b200_dev.h): index residency in HBM,
 * batch upload, kernel launches on the context's stream, result download into pinned buffers, and
 * the work/time counters the roofline is computed from.
 *
 * HBM layout of the index blob (all offsets 256-byte aligned):
 *   [ header | Occ/BWT blocks (bwt_size*4 B, re-packed: 32 B per 64 symbols) | sampled SA (n_sa*8 B) | pac (l_pac/4+1 B) ]
 * The blob is position independent (the header holds sizes, not pointers) so that it can be filled
 * on one GPU and broadcast to the others with a single collective.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdarg.h>
#include <pthread.h>
#include <time.h>
#include <math.h>
#include <sched.h>
#include "bwag_dev.cuh"
#include "bwag_kernels.h"

struct BlobHeader {
	u64 magic, primary, seq_len, bwt_size, n_sa, l_pac;
	u64 L2[5];
	u64 sa_shift;
	u64 off_bwt, off_sa, off_pac, total;
	u64 sb[BWAG_MAX_SB][4];   /* counts before each 2^31-symbol superblock of the re-packed Occ table */
};
#define BLOB_MAGIC 0x3142574142323030ull
#define ALIGN256(x) (((x) + 255) & ~(size_t)255)

static __thread char g_err[512];
extern "C" const char *bwag_last_error(void) { return g_err[0] ? g_err : "no error"; }
static int set_err(const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof(g_err), fmt, ap);
	va_end(ap);
	return 1;
}
int bwag_set_error(const char *msg) { return set_err("%s", msg); }   /* for the other host drivers of the library (bwag_index.cu) */
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return set_err("%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); } while (0)
#define CKP(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_err("%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); return 0; } } while (0)

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
};

struct DevBuf { void *p; size_t cap; };
static int buf_reserve(DevBuf *b, size_t bytes)
{
	if (bytes <= b->cap) return 0;
	if (b->p) cudaFree(b->p);
	b->p = 0; b->cap = 0;
	size_t want = bytes + bytes / 4 + 256;
	CK(cudaMalloc(&b->p, want));
	b->cap = want;
	return 0;
}
struct HostBuf { void *p; size_t cap; };
static int hbuf_reserve(HostBuf *b, size_t bytes)
{
	if (bytes <= b->cap) return 0;
	if (b->p) cudaFreeHost(b->p);
	b->p = 0; b->cap = 0;
	size_t want = bytes + bytes / 4 + 256;
	CK(cudaMallocHost(&b->p, want));
	b->cap = want;
	return 0;
}

struct bwag_ctx {
	int device, own_blob, n_sm;
	int imported;                /* blob, dense SA and table belong to another process (bwag_ctx_import): closed, not freed */
	size_t map_bytes[3];         /* (emulator build) sizes of the three shared mappings */
	void *blob;
	DevIndex ix;
	u64 *dense_sa;
	ulonglong2 *ktab;            /* short-string table (bwag_ctx_build_ktab) */
	int baseline;                /* bwag_ctx_baseline(): first row sweeps in K4/K5 and no table lookups */
	cudaStream_t stream;
	cudaEvent_t ev0, ev1, ev_wait;
	Counters *d_cnt, *h_cnt;
	bwag_stats_t st;
	int sa_intv_disk;
	/* scratch reused across batches */
	DevBuf s_k1, s_k1f, s_n3, s_eh, s_rseq, s_qseq, s_z, s_wcig, s_wmd, s_pack, s_zl;
	int grid_k1, grid_k1f, grid_k2, grid_k4, grid_k5;
	int k3s_blocks;   /* resident blocks per SM of k_chain_sm (occupancy API) */
#define N_SPARE 12
	struct bwag_batch *spare[N_SPARE]; /* batch objects (stream, counters, scratch, device and pinned buffers) kept for later batches */
	pthread_mutex_t mu;
	struct bwag_ctx *parent;     /* set in the per-batch view of the context */
	/* stage 4: contig table (offsets, lengths, ALT flags, names) and log(i) table, resident once per context */
	void *d_tail; TailCtg tctg; const double *d_logtab; int have_ctg;
	/* samse: the reference's holes (bns->ambs), for bns_cnt_ambi */
	void *d_ambs; int n_holes, have_ambs;
};

struct bwag_batch {
	bwag_ctx_t *ctx;
	bwag_ctx_t lc;               /* per-batch view of the context: own stream, events, counters, scratch, stats -> batches can overlap */
	int lc_ready;
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
	int tail_ready;             /* bwag_tail_regs ran on this batch */
	int regs_on_device;          /* bwag_chain_extend left the regions in HBM */
};

static void batch_free(bwag_batch_t *b);
static void free_dev(DevBuf *b) { if (b->p) cudaFree(b->p); b->p = 0; b->cap = 0; }
static void free_host(HostBuf *b) { if (b->p) cudaFreeHost(b->p); b->p = 0; b->cap = 0; }

#ifndef BWAG_L2_FETCH_DEFAULT
#define BWAG_L2_FETCH_DEFAULT 0   /* 0: leave the device's setting */
#endif
#define K1_SMEM_MAX (200 * 1024)
#ifndef K1_COMPACT_DEFAULT
#define K1_COMPACT_DEFAULT 1   /* k_smem_c unless BWA_B200_K1_COMPACT=0 */
#endif
#ifdef BWAG_CUSIM
#define BWAG_KTAB_MAX_AUTO 5     /* the emulator builds the table one fiber per entry: keep it small */
#else
#define BWAG_KTAB_MAX_AUTO 14
#endif
#define K4_SMEM_MAX (96 * 1024)
#define K4L_SMEM_MAX (200 * 1024)
#define SEEDSW_MAXLEN 200   /* the seed-level filter aligns windows shorter than this on both axes (bwamem.c:591,612) */

#ifdef BWAG_CUSIM
unsigned long long bwag_cusim_sector_loads, bwag_cusim_list_acc[5];
#endif

/* ------------------------------------------------------------------------------------------------ index */

extern "C" size_t bwag_blob_bytes(const bwt_t *bwt, int64_t l_pac)
{
	return ALIGN256(sizeof(BlobHeader)) + ALIGN256((size_t)bwt->bwt_size * 4 + 64) + ALIGN256((size_t)bwt->n_sa * 8 + 32) + ALIGN256((size_t)l_pac / 4 + 1 + 64);
}

extern "C" int bwag_blob_fill(int device, void *d_blob, const bwt_t *bwt, int64_t l_pac, const uint8_t *pac)
{
	BlobHeader h;
	if (device >= 0) CK(cudaSetDevice(device));
	memset(&h, 0, sizeof(h));
	h.magic = BLOB_MAGIC; h.primary = bwt->primary; h.seq_len = bwt->seq_len; h.bwt_size = bwt->bwt_size; h.n_sa = bwt->n_sa; h.l_pac = (u64)l_pac;
	for (int i = 0; i < 5; ++i) h.L2[i] = bwt->L2[i];
	{
		int s = 0;
		while ((1 << s) < bwt->sa_intv) ++s;
		if ((1 << s) != bwt->sa_intv) return set_err("suffix-array interval %d is not a power of two", bwt->sa_intv);
		h.sa_shift = (u64)s;
	}
	if (bwt->seq_len >= (u64)BWAG_MAX_SB << BWAG_SB_SHIFT) return set_err("index too large: %llu BWT symbols", (unsigned long long)bwt->seq_len);
	for (u64 s = 0; s << BWAG_SB_SHIFT < bwt->seq_len; ++s) {   /* counts before symbol s*2^31 = the count words of that file block */
		const u64 *cnt = (const u64 *)(bwt->bwt + ((s << BWAG_SB_SHIFT) >> 7) * 16);
		for (int k = 0; k < 4; ++k) h.sb[s][k] = cnt[k];
	}
	h.off_bwt = ALIGN256(sizeof(BlobHeader));
	h.off_sa = h.off_bwt + ALIGN256((size_t)bwt->bwt_size * 4 + 64);
	h.off_pac = h.off_sa + ALIGN256((size_t)bwt->n_sa * 8 + 32);
	h.total = h.off_pac + ALIGN256((size_t)l_pac / 4 + 1 + 64);
	char *d = (char *)d_blob;
	CK(cudaMemcpy(d, &h, sizeof(h), cudaMemcpyHostToDevice));
	CK(cudaMemset(d + h.off_bwt, 0, ALIGN256((size_t)bwt->bwt_size * 4 + 64)));
	CK(cudaMemcpy(d + h.off_bwt, bwt->bwt, (size_t)bwt->bwt_size * 4, cudaMemcpyHostToDevice));
	{   /* file layout -> 32-byte blocks, in place (bwag_dev.cuh) */
		const u64 n_blocks = ((u64)bwt->bwt_size * 4 + 63) / 64;
		DevIndex tmp;
		memset(&tmp, 0, sizeof(tmp));
		for (int s = 0; s < BWAG_MAX_SB; ++s)
			for (int k = 0; k < 4; ++k) tmp.sb[s][k] = h.sb[s][k];
		BWAG_LAUNCH(k_occ_pack, (int)((n_blocks + 255) / 256 < 65535 ? (n_blocks + 255) / 256 : 65535), 256, 0, 0, tmp, (uint4 *)(d + h.off_bwt), n_blocks);
		CK(cudaGetLastError());
		CK(cudaDeviceSynchronize());
	}
	CK(cudaMemcpy(d + h.off_sa, bwt->sa, (size_t)bwt->n_sa * 8, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(d + h.off_pac, pac, (size_t)l_pac / 4 + 1, cudaMemcpyHostToDevice));
	return 0;
}

static int pick_grid(bwag_ctx_t *c)
{
#ifdef BWAG_CUSIM
	c->n_sm = 2;
	c->grid_k1 = c->grid_k1f = c->grid_k2 = c->grid_k4 = c->grid_k5 = 2;
	c->k3s_blocks = 1;
#else
	cudaDeviceProp prop;
	int nb;
	CK(cudaGetDeviceProperties(&prop, c->device));
	c->n_sm = prop.multiProcessorCount;
	CK(cudaFuncSetAttribute(k_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, K1_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_smem_fm, cudaFuncAttributeMaxDynamicSharedMemorySize, K1_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_chain_sm, cudaFuncAttributeMaxDynamicSharedMemorySize, K3S_SMEM));
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c->k3s_blocks, k_chain_sm, K3S_THREADS, K3S_SMEM));
#ifndef K1_PACKED8
	CK(cudaFuncSetAttribute(k_smem_c, cudaFuncAttributeMaxDynamicSharedMemorySize, K1_SMEM_MAX));
#endif
	c->grid_k1 = 0;   /* depends on the shared read slots: chosen per launch */
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_smem_fwd, K1F_THREADS, 0)); c->grid_k1f = c->n_sm * (nb > 0 ? nb : 1);
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_sa, K2_THREADS, 0)); c->grid_k2 = c->n_sm * (nb > 0 ? nb : 1);
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_extend, K4_THREADS, 0)); c->grid_k4 = c->n_sm * (nb > 0 ? nb : 1);
	CK(cudaFuncSetAttribute(k_extend_sm, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_extend_sm_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_extend_lane, cudaFuncAttributeMaxDynamicSharedMemorySize, K4L_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_global_sm, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_global_sm_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_global, K5_THREADS, 0)); c->grid_k5 = c->n_sm * (nb > 0 ? nb : 1);
#endif
	return 0;
}

static cudaEvent_t g_trace_ref;   /* BWA_B200_GPUTRACE: origin of the device-clock timeline (see elapsed_at) */
static int g_gputrace = -1;

extern "C" bwag_ctx_t *bwag_ctx_from_blob(int device, void *d_blob, int own_blob)
{
	BlobHeader h;
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_err("no CUDA device is visible: this library has no CPU path"); return 0; }
	if (device < 0) CKP(cudaGetDevice(&device));
	CKP(cudaSetDevice(device));
	CKP(cudaMemcpy(&h, d_blob, sizeof(h), cudaMemcpyDeviceToHost));
	if (h.magic != BLOB_MAGIC) { set_err("index blob has a bad magic number"); return 0; }
	{   /* the hot tables are read one random 32-byte sector at a time: ask L2 not to fetch the neighbouring sector as well
	     * (BWA_B200_L2_FETCH=32|64|128; a hint the hardware may ignore) */
		const char *e = getenv("BWA_B200_L2_FETCH");
		int g = e ? atoi(e) : BWAG_L2_FETCH_DEFAULT;
		if (g == 32 || g == 64 || g == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)g);
	}
	bwag_ctx_t *c = (bwag_ctx_t *)calloc(1, sizeof(*c));
	c->device = device; c->own_blob = own_blob; c->blob = d_blob;
	char *d = (char *)d_blob;
	c->ix.bwt = (const uint4 *)(d + h.off_bwt);
	c->ix.sa = (const u64 *)(d + h.off_sa);
	c->ix.pac = (const uint8_t *)(d + h.off_pac);
	c->ix.primary = h.primary; c->ix.seq_len = h.seq_len; c->ix.n_sa = h.n_sa; c->ix.l_pac = (i64)h.l_pac; c->ix.sa_shift = (int)h.sa_shift;
	for (int i = 0; i < 5; ++i) c->ix.L2[i] = h.L2[i];
	for (int s = 0; s < BWAG_MAX_SB; ++s)
		for (int k = 0; k < 4; ++k) { c->ix.sb[s][k] = h.sb[s][k]; c->ix.sbgt[s][k] = 0; for (int t = k + 1; t < 4; ++t) c->ix.sbgt[s][k] += h.sb[s][t]; }
	c->sa_intv_disk = 1 << h.sa_shift;
	CKP(cudaStreamCreate(&c->stream));
	CKP(cudaEventCreate(&c->ev0)); CKP(cudaEventCreate(&c->ev1));
	if (g_gputrace < 0) {
		const char *e = getenv("BWA_B200_GPUTRACE");
		g_gputrace = e && atoi(e) > 0;
		if (g_gputrace) { CKP(cudaEventCreate(&g_trace_ref)); CKP(cudaEventRecord(g_trace_ref, c->stream)); CKP(cudaEventSynchronize(g_trace_ref)); }
	}
	CKP(cudaEventCreateWithFlags(&c->ev_wait, cudaEventBlockingSync | cudaEventDisableTiming));
	CKP(cudaMalloc((void **)&c->d_cnt, sizeof(Counters)));
	CKP(cudaMallocHost((void **)&c->h_cnt, sizeof(Counters)));
	pthread_mutex_init(&c->mu, 0);
	if (pick_grid(c)) { free(c); return 0; }
	return c;
}

extern "C" bwag_ctx_t *bwag_ctx_create(int device, const bwt_t *bwt, int64_t l_pac, const uint8_t *pac)
{
	int ndev = 0;
	void *blob = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_err("no CUDA device is visible: this library has no CPU path"); return 0; }
	if (device < 0) CKP(cudaGetDevice(&device));
	CKP(cudaSetDevice(device));
	CKP(cudaMalloc(&blob, bwag_blob_bytes(bwt, l_pac)));
	if (bwag_blob_fill(device, blob, bwt, l_pac, pac)) { cudaFree(blob); return 0; }
	bwag_ctx_t *c = bwag_ctx_from_blob(device, blob, 1);
	if (!c) cudaFree(blob);
	return c;
}

/* ------------------------------------------------------------------------------------------------ residency across processes */
#include <sys/mman.h>
#include <sys/stat.h>
#include <fcntl.h>
#include <signal.h>
#include <errno.h>
#include <unistd.h>
struct ShareFile {
	char magic[8];
	int32_t version, device, pid, dense_shift, ktab_k, pad;
	u64 l_pac, blob_bytes, dense_bytes, dense_n, ktab_bytes;
#ifndef BWAG_CUSIM
	cudaIpcMemHandle_t h[3];     /* blob, dense SA sample, short-string table */
#else
	char name[3][64];            /* emulator build: "device memory" is host memory, the three regions travel as POSIX shared memory */
#endif
};
#define SHARE_MAGIC "BWAB2SHR"

static void shared_close(bwag_ctx_t *c)
{
	void *p[3] = { c->blob, (void *)c->dense_sa, (void *)c->ktab };
	for (int i = 0; i < 3; ++i) {
		if (!p[i]) continue;
#ifndef BWAG_CUSIM
		cudaIpcCloseMemHandle(p[i]);
#else
		munmap(p[i], c->map_bytes[i]);
#endif
	}
}

extern "C" void bwag_ctx_unexport(const char *path)
{
#ifdef BWAG_CUSIM
	ShareFile f;
	FILE *fp = fopen(path, "rb");
	if (fp) { if (fread(&f, sizeof(f), 1, fp) == 1 && memcmp(f.magic, SHARE_MAGIC, 8) == 0) for (int i = 0; i < 3; ++i) if (f.name[i][0]) shm_unlink(f.name[i]); fclose(fp); }
#endif
	unlink(path);
}

extern "C" int bwag_ctx_export(bwag_ctx_t *c, const char *path)
{
	ShareFile f;
	BlobHeader h;
	CK(cudaSetDevice(c->device));
	CK(cudaStreamSynchronize(c->stream));
	CK(cudaMemcpy(&h, c->blob, sizeof(h), cudaMemcpyDeviceToHost));
	memset(&f, 0, sizeof(f));
	memcpy(f.magic, SHARE_MAGIC, 8);
	f.version = 2; f.device = c->device; f.pid = (int32_t)getpid(); f.l_pac = h.l_pac; f.blob_bytes = h.total;
	f.dense_shift = c->dense_sa ? c->ix.sa_shift : -1; f.dense_n = c->dense_sa ? c->ix.n_sa : 0; f.dense_bytes = c->dense_sa ? c->ix.n_sa * 8 + 32 : 0;
	f.ktab_k = c->ktab ? c->ix.ktab_k : 0; f.ktab_bytes = c->ktab ? (((((u64)1 << (2 * (c->ix.ktab_k + 1))) - 4) / 3) + 2) * 16 : 0;
	{
		void *p[3] = { c->blob, (void *)c->dense_sa, (void *)c->ktab };
		const u64 bytes[3] = { f.blob_bytes, f.dense_bytes, f.ktab_bytes };
		for (int i = 0; i < 3; ++i) {
			if (!p[i]) continue;
#ifndef BWAG_CUSIM
			(void)bytes;
			CK(cudaIpcGetMemHandle(&f.h[i], p[i]));
#else
			snprintf(f.name[i], sizeof(f.name[i]), "/bwa_b200.%d.%d", (int)getpid(), i);
			int fd = shm_open(f.name[i], O_CREAT | O_RDWR | O_TRUNC, 0600);
			if (fd < 0 || ftruncate(fd, (off_t)bytes[i]) != 0) return set_err("cannot create shared memory %s: %s", f.name[i], strerror(errno));
			void *m = mmap(0, bytes[i], PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
			close(fd);
			if (m == MAP_FAILED) return set_err("cannot map shared memory %s: %s", f.name[i], strerror(errno));
			memcpy(m, p[i], bytes[i]);
			munmap(m, bytes[i]);
#endif
		}
	}
	{   /* the file appears complete or not at all */
		char tmp[4096];
		snprintf(tmp, sizeof(tmp), "%s.tmp%d", path, (int)getpid());
		FILE *fp = fopen(tmp, "wb");
		if (!fp || fwrite(&f, sizeof(f), 1, fp) != 1 || fclose(fp) != 0 || rename(tmp, path) != 0) return set_err("cannot write %s: %s", path, strerror(errno));
	}
	return 0;
}

extern "C" bwag_ctx_t *bwag_ctx_import(const char *path, int64_t l_pac)
{
	ShareFile f;
	FILE *fp = fopen(path, "rb");
	if (!fp) { set_err("no resident index at %s", path); return 0; }
	const size_t got = fread(&f, sizeof(f), 1, fp);
	fclose(fp);
	if (got != 1 || memcmp(f.magic, SHARE_MAGIC, 8) != 0 || f.version != 2) { set_err("%s is not a resident-index descriptor of this version", path); return 0; }
	if (kill((pid_t)f.pid, 0) != 0 && errno == ESRCH) { set_err("the process that kept the index resident (pid %d) is gone", f.pid); return 0; }
	if (l_pac >= 0 && (u64)l_pac != f.l_pac) { set_err("the resident index is not this index (l_pac %llu, expected %lld)", (unsigned long long)f.l_pac, (long long)l_pac); return 0; }
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_err("no CUDA device is visible: this library has no CPU path"); return 0; }
	if (f.device >= ndev) { set_err("the resident index lives on device %d, which this process does not see", f.device); return 0; }
	CKP(cudaSetDevice(f.device));
	void *p[3] = { 0, 0, 0 };
	const u64 bytes[3] = { f.blob_bytes, f.dense_bytes, f.ktab_bytes };
	for (int i = 0; i < 3; ++i) {
		if (!bytes[i]) continue;
#ifndef BWAG_CUSIM
		if (cudaIpcOpenMemHandle(&p[i], f.h[i], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
			set_err("cannot open the resident index of pid %d: %s", f.pid, cudaGetErrorString(cudaGetLastError()));
			for (int k = 0; k < i; ++k) if (p[k]) cudaIpcCloseMemHandle(p[k]);
			return 0;
		}
#else
		int fd = shm_open(f.name[i], O_RDONLY, 0);
		void *m = fd >= 0 ? mmap(0, bytes[i], PROT_READ, MAP_SHARED, fd, 0) : MAP_FAILED;
		if (fd >= 0) close(fd);
		if (m == MAP_FAILED) { set_err("cannot map the resident index of pid %d (%s): %s", f.pid, f.name[i], strerror(errno)); for (int k = 0; k < i; ++k) if (p[k]) munmap(p[k], bytes[k]); return 0; }
		p[i] = m;
#endif
	}
	bwag_ctx_t *c = bwag_ctx_from_blob(f.device, p[0], 0);
	if (!c) return 0;
	c->imported = 1;
	for (int i = 0; i < 3; ++i) c->map_bytes[i] = bytes[i];
	if (p[1]) { c->dense_sa = (u64 *)p[1]; c->ix.sa = c->dense_sa; c->ix.sa_shift = f.dense_shift; c->ix.n_sa = f.dense_n; }
	if (p[2]) { c->ktab = (ulonglong2 *)p[2]; c->ix.ktab = c->ktab; c->ix.ktab_k = f.ktab_k; }
	return c;
}

extern "C" void bwag_ctx_destroy(bwag_ctx_t *c)
{
	if (!c) return;
	cudaSetDevice(c->device);
	cudaStreamSynchronize(c->stream);
	free_dev(&c->s_pack); free_dev(&c->s_k1); free_dev(&c->s_k1f); free_dev(&c->s_n3); free_dev(&c->s_eh); free_dev(&c->s_rseq); free_dev(&c->s_qseq); free_dev(&c->s_z); free_dev(&c->s_wcig); free_dev(&c->s_wmd); free_dev(&c->s_zl);
	for (int i = 0; i < N_SPARE; ++i) if (c->spare[i]) { batch_free(c->spare[i]); c->spare[i] = 0; }
	if (c->imported) shared_close(c);
	else {
		if (c->dense_sa) cudaFree(c->dense_sa);
		if (c->ktab) cudaFree(c->ktab);
		if (c->own_blob && c->blob) cudaFree(c->blob);
	}
	if (c->d_tail) cudaFree(c->d_tail);
	if (c->d_ambs) cudaFree(c->d_ambs);
	cudaFree(c->d_cnt); cudaFreeHost(c->h_cnt);
	cudaEventDestroy(c->ev0); cudaEventDestroy(c->ev1); cudaEventDestroy(c->ev_wait);
	cudaStreamDestroy(c->stream);
	free(c);
}

extern "C" int bwag_ctx_densify_sa(bwag_ctx_t *c, int intv)
{
	if (intv == 0) {   /* the densest interval >= 2 whose sample takes at most an eighth of the device's memory; the rest holds the
	                    * index, the short-string table and the batches of the calls in flight (3 Gbp on an 80 GB H100: every 8th row, 6 GB) */
		size_t free_b = 0, total_b = 0;
		CK(cudaSetDevice(c->device));
		CK(cudaMemGetInfo(&free_b, &total_b));
		intv = 2;
		while (intv < 32 && (double)(c->ix.seq_len / (u64)intv + 1) * 8 > (double)total_b / 8) intv <<= 1;
		if (intv < 8 && bwag_ctx_densify_sa(c, 8)) return 1;   /* in two stages (32 -> 8 -> intv): each walks only a few LF steps per row */
	}
	int s = 0;
	while ((1 << s) < intv) ++s;
	if ((1 << s) != intv || s > c->ix.sa_shift) return set_err("dense suffix-array interval must be a power of two not above the current %d", 1 << c->ix.sa_shift);
	if (s == c->ix.sa_shift || c->imported) return 0;   /* an imported context keeps the sample of the process that owns the memory */
	CK(cudaSetDevice(c->device));
	u64 n_out = (c->ix.seq_len + (u64)intv) / (u64)intv, *out = 0;
	{   /* leave room for the batch buffers */
		size_t free_b = 0, total_b = 0;
		CK(cudaMemGetInfo(&free_b, &total_b));
		if ((double)n_out * 8 > 0.5 * (double)free_b) return set_err("not enough free device memory for a suffix-array sample of interval %d", intv);
	}
	CK(cudaMalloc((void **)&out, n_out * 8 + 32));   /* K2 reads the sample in aligned groups of four rows */
	BWAG_LAUNCH(k_sa_densify, c->n_sm * 8, 256, 0, c->stream, c->ix, out, s, n_out);
	CK(cudaGetLastError());
	CK(cudaStreamSynchronize(c->stream));
	if (c->dense_sa) cudaFree(c->dense_sa);
	c->dense_sa = out;
	c->ix.sa = out; c->ix.sa_shift = s; c->ix.n_sa = n_out;
	++c->st.n_launch;
	return 0;
}

/* bi-intervals of all strings of 1..K bases (bwag_smem.cu); K = 0 picks a depth from the index size, K < 0 removes the table */
extern "C" int bwag_ctx_build_ktab(bwag_ctx_t *c, int K)
{
	CK(cudaSetDevice(c->device));
	if (c->imported) return 0;   /* the table, or its absence, is the owner's */
	if (K == 0) {   /* as deep as strings still have a few dozen occurrences (their intervals span two Occ blocks): 14 at 3 Gbp = 5.7 GB */
		int lg = 0;
		while (lg < 31 && ((u64)1 << (2 * (lg + 1))) <= c->ix.seq_len) ++lg;   /* floor(log4(seq_len)) */
		K = lg - 2;
		if (K > BWAG_KTAB_MAX_AUTO) K = BWAG_KTAB_MAX_AUTO;
	}
	if (K > 14) K = 14;
	if (K < 2) {
		CK(cudaStreamSynchronize(c->stream));
		if (c->ktab) { cudaFree(c->ktab); c->ktab = 0; }
		c->ix.ktab = 0; c->ix.ktab_k = 0;
		return 0;
	}
	if (c->ktab && c->ix.ktab_k == K) return 0;
	const u64 total = (((u64)1 << (2 * (K + 1))) - 4) / 3;
	ulonglong2 *tab = 0;
	{
		size_t free_b = 0, total_b = 0;
		CK(cudaMemGetInfo(&free_b, &total_b));
		if ((double)total * 16 > 0.25 * (double)free_b) return set_err("not enough free device memory for a short-string table of depth %d", K);
	}
	CK(cudaMalloc((void **)&tab, (total + 2) * 16));
	CK(cudaMemsetAsync(tab, 0, (total + 2) * 16, c->stream));
	DevIndex plain = c->ix;
	plain.ktab = 0; plain.ktab_k = 0;
	{
		u64 nb = (total + 255) / 256;
		BWAG_LAUNCH(k_ktab_build, (int)(nb < (u64)c->n_sm * 32 ? nb : (u64)c->n_sm * 32), 256, 0, c->stream, plain, tab, K);
	}
	CK(cudaGetLastError());
	CK(cudaStreamSynchronize(c->stream));
	if (c->ktab) cudaFree(c->ktab);
	c->ktab = tab;
	c->ix.ktab = tab; c->ix.ktab_k = K;
#ifdef BWAG_CUSIM
	bwag_cusim_sector_loads = 0;   /* the emulator's request counter reports the alignment work only */
#endif
	++c->st.n_launch;
	return 0;
}

/* Check the resident index against the resident text on rows first, first + stride, ... (stride 1 = every row, a complete check;
 * see k_index_verify).  out: rows checked, BWT/text/SA mismatches, order violations, pairs of suffixes equal over 8192 bases. */
extern "C" int bwag_ctx_verify(bwag_ctx_t *c, uint64_t first, uint64_t stride, uint64_t out[4])
{
	CK(cudaSetDevice(c->device));
	if (stride == 0) stride = 1;
	const u64 n_check = first > c->ix.seq_len ? 0 : (c->ix.seq_len - first) / stride + 1;
	u64 *d = 0;
	CK(cudaMalloc((void **)&d, 4 * sizeof(u64)));
	CK(cudaMemsetAsync(d, 0, 4 * sizeof(u64), c->stream));
	if (n_check) {
		const u64 nb = (n_check + 255) / 256;
		BWAG_LAUNCH(k_index_verify, (int)(nb < (u64)c->n_sm * 64 ? nb : (u64)c->n_sm * 64), 256, 0, c->stream, c->ix, (u64)first, (u64)stride, n_check, d);
		CK(cudaGetLastError());
	}
	CK(cudaMemcpyAsync(out, d, 4 * sizeof(u64), cudaMemcpyDeviceToHost, c->stream));
	CK(cudaStreamSynchronize(c->stream));
	cudaFree(d);
	++c->st.n_launch;
	return 0;
}

/* on = 1: batches begun from now on use the first formulation of the K4/K5 row sweeps and no short-string table (the
 * configuration measured in round 1); on = 0: back to the defaults.  Used by the host's start-up self-check. */
extern "C" void bwag_ctx_baseline(bwag_ctx_t *c, int on) { pthread_mutex_lock(&c->mu); c->baseline = on != 0; pthread_mutex_unlock(&c->mu); }
extern "C" int bwag_is_emulator(void)
{
#ifdef BWAG_CUSIM
	return 1;
#else
	return 0;
#endif
}

extern "C" void bwag_stats_get(bwag_ctx_t *c, bwag_stats_t *s) { pthread_mutex_lock(&c->mu); *s = c->st; pthread_mutex_unlock(&c->mu); }
extern "C" void bwag_stats_reset(bwag_ctx_t *c) { pthread_mutex_lock(&c->mu); memset(&c->st, 0, sizeof(c->st)); pthread_mutex_unlock(&c->mu); }

/* K3 cycle histograms of a build with -DBWAG_K3_CLOCKS (tools/chain_bench.py): by seeds per read (0..64, then > 64) the reads and the
 * clock64() cycles of their chaining loop, mem_chain_flt and chain_emit, then the reads by chains per read (0..32, then > 32) */
#ifdef BWAG_K3_CLOCKS
static pthread_mutex_t g_k3clk_mu = PTHREAD_MUTEX_INITIALIZER;
static u64 g_k3clk[BWAG_K3CLK_WORDS];
#endif
extern "C" int bwag_k3_clocks(uint64_t *out, int reset)
{
#ifdef BWAG_K3_CLOCKS
	pthread_mutex_lock(&g_k3clk_mu);
	if (out) memcpy(out, g_k3clk, sizeof(g_k3clk));
	if (reset) memset(g_k3clk, 0, sizeof(g_k3clk));
	pthread_mutex_unlock(&g_k3clk_mu);
	return 0;
#else
	(void)out; (void)reset;
	return -1;
#endif
}
#ifdef BWAG_K3_CLOCKS
static void k3clk_add(const u32 *rec, int n)
{
	pthread_mutex_lock(&g_k3clk_mu);
	for (int r = 0; r < n; ++r, rec += 5) {
		const int t = rec[0] > 64 ? 65 : (int)rec[0], ch = rec[1] > 32 ? 33 : (int)rec[1];
		u64 *h = g_k3clk + 4 * t;
		h[0] += 1; h[1] += rec[2]; h[2] += rec[3]; h[3] += rec[4];
		g_k3clk[4 * 66 + ch] += 1;
	}
	pthread_mutex_unlock(&g_k3clk_mu);
}
#endif

extern "C" void *bwag_host_alloc(size_t bytes)
{
	void *p = 0;
	if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) { cudaGetLastError(); return 0; }
	return p;
}
extern "C" void bwag_host_free(void *p) { if (p) cudaFreeHost(p); }

/* ------------------------------------------------------------------------------------------------ batch */

extern "C" bwag_batch_t *bwag_batch_begin(bwag_ctx_t *c, int n, const uint8_t *codes, const int64_t *off)
{
	bwag_batch_t *b = 0;   /* buffers only grow: cudaMalloc/cudaMallocHost per batch would cost more than the kernels */
	pthread_mutex_lock(&c->mu);
	for (int i = 0; i < N_SPARE; ++i) if (c->spare[i]) { b = c->spare[i]; c->spare[i] = 0; break; }
	pthread_mutex_unlock(&c->mu);
	if (!b) b = (bwag_batch_t *)calloc(1, sizeof(*b));
	CKP(cudaSetDevice(c->device));
	if (!b->lc_ready) {    /* first use of this batch object: its own stream, events and counters */
		memset(&b->lc, 0, sizeof(b->lc));
		CKP(cudaStreamCreate(&b->lc.stream));
		CKP(cudaEventCreate(&b->lc.ev0)); CKP(cudaEventCreate(&b->lc.ev1));
		CKP(cudaEventCreateWithFlags(&b->lc.ev_wait, cudaEventBlockingSync | cudaEventDisableTiming));
		CKP(cudaMalloc((void **)&b->lc.d_cnt, sizeof(Counters)));
		CKP(cudaMallocHost((void **)&b->lc.h_cnt, sizeof(Counters)));
		b->lc_ready = 1;
	}
	b->lc.device = c->device; b->lc.n_sm = c->n_sm; b->lc.ix = c->ix; b->lc.parent = c;
	b->lc.baseline = c->baseline;
	if (c->baseline) { b->lc.ix.ktab = 0; b->lc.ix.ktab_k = 0; }
	b->lc.grid_k1 = c->grid_k1; b->lc.grid_k1f = c->grid_k1f; b->lc.grid_k2 = c->grid_k2; b->lc.grid_k4 = c->grid_k4; b->lc.grid_k5 = c->grid_k5;
	b->lc.k3s_blocks = c->k3s_blocks;
	memset(&b->lc.st, 0, sizeof(b->lc.st));
	b->max_len = 0; b->seeded = 0; b->tail_ready = 0; b->regs_on_device = 0;
	b->ctx = c; b->n = n; b->h_off = (const i64 *)off; b->total_bases = off[n];
	for (int i = 0; i < n; ++i) { int l = (int)(off[i + 1] - off[i]); if (l > b->max_len) b->max_len = l; }
	if (buf_reserve(&b->d_codes, (size_t)b->total_bases + 16) || buf_reserve(&b->d_off, sizeof(i64) * ((size_t)n + 1))) { batch_free(b); return 0; }
	c = &b->lc;
	CKP(cudaEventRecord(c->ev0, c->stream));
	CKP(cudaMemcpyAsync(b->d_codes.p, codes, (size_t)b->total_bases, cudaMemcpyHostToDevice, c->stream));
	CKP(cudaMemcpyAsync(b->d_off.p, off, sizeof(i64) * ((size_t)n + 1), cudaMemcpyHostToDevice, c->stream));
	c->st.h2d_bytes += (u64)b->total_bases + sizeof(i64) * ((u64)n + 1);
	CKP(cudaEventRecord(c->ev1, c->stream));
	CKP(cudaStreamSynchronize(c->stream));
	{ float ms = 0; cudaEventElapsedTime(&ms, c->ev0, c->ev1); c->st.ms_h2d += ms; }
	return b;
}

extern "C" void bwag_batch_end(bwag_batch_t *b)
{
	if (!b) return;
	bwag_ctx_t *c = b->ctx;
	cudaSetDevice(c->device);
	cudaStreamSynchronize(b->lc.stream);
	pthread_mutex_lock(&c->mu);
	{   /* fold this batch's counters into the context */
		bwag_stats_t *d = &c->st, *x = &b->lc.st;
		d->occ_touches += x->occ_touches; d->sa_touches += x->sa_touches; d->sa_touches_algo += x->sa_touches_algo;
		d->ext_cells += x->ext_cells; d->glb_cells += x->glb_cells;
		d->ms_smem += x->ms_smem; d->ms_sa += x->ms_sa; d->ms_chain += x->ms_chain; d->ms_extend += x->ms_extend; d->ms_global += x->ms_global;
		d->ms_h2d += x->ms_h2d; d->ms_d2h += x->ms_d2h; d->n_launch += x->n_launch; d->h2d_bytes += x->h2d_bytes; d->d2h_bytes += x->d2h_bytes;
		d->ms_tail += x->ms_tail; d->tail_reads += x->tail_reads; d->tail_complex += x->tail_complex; d->ms_localsw += x->ms_localsw; d->sw_tasks += x->sw_tasks;
	}
#ifdef BWAG_CUSIM
	if (getenv("BWA_B200_PROFILE")) fprintf(stderr, "[prof] emulator: %llu 32-byte block/table loads so far (K1, K1f, K2, table build); K1 candidate-list accesses by entry index 0-3: %llu, 4-7: %llu, 8-11: %llu, 12-15: %llu, 16+: %llu (the first K1_SLOTS of a list live in shared memory)\n", bwag_cusim_sector_loads, bwag_cusim_list_acc[0], bwag_cusim_list_acc[1], bwag_cusim_list_acc[2], bwag_cusim_list_acc[3], bwag_cusim_list_acc[4]);
#endif
	if (getenv("BWA_B200_PROFILE"))   /* with the host's phase timer: the work counters of this batch */
		fprintf(stderr, "[prof] batch counters: %d reads, occ_touches %llu, sa_touches %llu, ext_cells %llu, glb_cells %llu; stage 4: %llu reads, %llu handed back to the host-side post-processing; K6: %llu local alignments\n", b->n,
		        (unsigned long long)b->lc.st.occ_touches, (unsigned long long)b->lc.st.sa_touches, (unsigned long long)b->lc.st.ext_cells, (unsigned long long)b->lc.st.glb_cells,
		        (unsigned long long)b->lc.st.tail_reads, (unsigned long long)b->lc.st.tail_complex, (unsigned long long)b->lc.st.sw_tasks);
	for (int i = 0; i < N_SPARE; ++i) if (!c->spare[i]) { c->spare[i] = b; b = 0; break; }
	pthread_mutex_unlock(&c->mu);
	if (b) batch_free(b);
}

static void batch_free(bwag_batch_t *b)
{
	if (b->lc_ready) {
		free_dev(&b->lc.s_pack); free_dev(&b->lc.s_k1); free_dev(&b->lc.s_k1f); free_dev(&b->lc.s_n3); free_dev(&b->lc.s_eh); free_dev(&b->lc.s_rseq); free_dev(&b->lc.s_qseq); free_dev(&b->lc.s_z); free_dev(&b->lc.s_wcig); free_dev(&b->lc.s_wmd);
		cudaFree(b->lc.d_cnt); cudaFreeHost(b->lc.h_cnt);
		cudaEventDestroy(b->lc.ev0); cudaEventDestroy(b->lc.ev1); cudaEventDestroy(b->lc.ev_wait); cudaStreamDestroy(b->lc.stream);
	}
	free_dev(&b->d_codes); free_dev(&b->d_off);
	free_dev(&b->d_intv_beg); free_dev(&b->d_intv_n); free_dev(&b->d_intv); free_dev(&b->d_seed_beg); free_dev(&b->d_rbeg);
	free_host(&b->h_intv_beg); free_host(&b->h_intv_n); free_host(&b->h_intv); free_host(&b->h_seed_beg); free_host(&b->h_rbeg);
	free_dev(&b->d_chain_off); free_dev(&b->d_chains); free_dev(&b->d_seeds); free_dev(&b->d_regs); free_dev(&b->d_nregs);
	free_dev(&b->d_chain_beg); free_dev(&b->d_chain_cnt); free_dev(&b->d_reg_base); free_dev(&b->d_chain_rid); free_dev(&b->d_chain_frac); free_dev(&b->d_cregs); free_dev(&b->d_creg_beg); free_dev(&b->d_ctg);
	free_dev(&b->s_bt); free_dev(&b->s_sn); free_dev(&b->s_ch); free_dev(&b->s_order); free_dev(&b->s_idx); free_dev(&b->s_keys);
	free_host(&b->h_regs); free_host(&b->h_nregs); free_host(&b->h_cregs); free_host(&b->h_creg_beg); free_host(&b->h_tmp);
	free_dev(&b->d_tasks); free_dev(&b->d_res); free_dev(&b->d_cig); free_dev(&b->d_md);
	free_host(&b->h_res); free_host(&b->h_cig); free_host(&b->h_md);
	free_dev(&b->d_sel); free_dev(&b->d_swtasks); free_dev(&b->d_swres); free_dev(&b->d_swpool); free_dev(&b->d_swscratch); free_host(&b->h_swres);
	free_dev(&b->d_hsp); free_dev(&b->d_flt_nchn); free_host(&b->h_hsp); free_dev(&b->d_k3big);
	free_dev(&b->d_pre_n); free_dev(&b->d_pre_score); free_dev(&b->d_pre_cig);
	free_dev(&b->d_dregs); free_dev(&b->d_dreg_beg); free_dev(&b->d_dreg_n); free_dev(&b->d_task_beg); free_dev(&b->d_cflag); free_dev(&b->d_pe_is); free_dev(&b->d_rec); free_dev(&b->d_text); free_dev(&b->d_ptab);
	free_host(&b->h_pe_is); free_host(&b->h_cflag); free_host(&b->h_rec); free_host(&b->h_text); free_host(&b->h_ptab);
	free_dev(&b->d_fm_lbeg); free_dev(&b->d_fm_lines); free_dev(&b->d_fm_nrow); free_dev(&b->d_fm_rbeg); free_dev(&b->d_fm_rows);
	free_dev(&b->d_fm_tlen); free_dev(&b->d_fm_tbeg); free_dev(&b->d_fm_text); free_dev(&b->d_fm_toff); free_host(&b->h_fm_text); free_host(&b->h_fm_off);
	free_dev(&b->d_aln_md); free_dev(&b->d_aln_n); free_dev(&b->d_aln_beg); free_dev(&b->d_aln_pool); free_dev(&b->d_aln_redo[0]); free_dev(&b->d_aln_redo[1]);
	free_dev(&b->d_aln_off); free_dev(&b->d_aln_out); free_dev(&b->d_aln_arena); free_host(&b->h_aln_n); free_host(&b->h_aln_off); free_host(&b->h_aln_out);
	free_dev(&b->d_se_reads); free_dev(&b->d_se_multi); free_dev(&b->d_se_bc); free_dev(&b->d_se_rows); free_dev(&b->d_se_pos); free_dev(&b->d_se_mpos); free_dev(&b->d_se_flags);
	free_dev(&b->d_se_tasks); free_dev(&b->d_se_mtask); free_dev(&b->d_se_cig); free_dev(&b->d_se_ncig); free_dev(&b->d_se_scratch); free_dev(&b->d_se_tlen); free_dev(&b->d_se_tbeg);
	free_dev(&b->d_se_rec); free_dev(&b->d_se_text); free_dev(&b->d_se_nm); free_host(&b->h_se_tasks); free_host(&b->h_se_mtask); free_host(&b->h_se_rec); free_host(&b->h_se_text);
	free(b);
}

static int reset_counters(bwag_ctx_t *c)
{
	CK(cudaMemsetAsync(c->d_cnt, 0, sizeof(Counters), c->stream));
	return 0;
}
/* wait for the context's stream.  Default: poll with short sleeps (a waiting lane costs no core; with the post-processing on the
 * device the host threads are few); BWA_B200_SYNC=spin: cudaStreamSynchronize, =yield / =block: see below */
static cudaError_t stream_wait(bwag_ctx_t *c)
{
	static int mode = -1;   /* BWA_B200_SYNC=block: sleep on a blocking event (saves the cores of waiting lanes, adds wake-up latency to every
	                         * stage); =yield: poll the stream and give the core away between polls (for boxes with fewer CPUs than threads) */
	if (mode < 0) { const char *e = getenv("BWA_B200_SYNC"); mode = !e ? 3 : strcmp(e, "spin") == 0 ? 0 : strcmp(e, "block") == 0 ? 1 : strcmp(e, "yield") == 0 ? 2 : 3; }   /* default: sleep-poll */
	if (mode == 0) return cudaStreamSynchronize(c->stream);
	if (mode == 3) {   /* =sleep: poll, sleeping 5..80 us between polls: under a CPU quota a spinning lane eats the host workers' budget */
		long ns = 5000;
		for (;;) {
			cudaError_t q = cudaStreamQuery(c->stream);
			if (q != cudaErrorNotReady) return q;
			struct timespec ts = { 0, ns };
			nanosleep(&ts, 0);
			if (ns < 80000) ns <<= 1;
		}
	}
	if (mode == 2) {
		for (;;) {
			cudaError_t q = cudaStreamQuery(c->stream);
			if (q != cudaErrorNotReady) return q;
			sched_yield();
		}
	}
	cudaError_t e = cudaEventRecord(c->ev_wait, c->stream);
	if (e != cudaSuccess) return e;
	return cudaEventSynchronize(c->ev_wait);
}

static int fetch_counters(bwag_ctx_t *c)
{
	CK(cudaMemcpyAsync(c->h_cnt, c->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, c->stream));
	CK(stream_wait(c));
	return 0;
}
#define H2D(c, dst, src, bytes) do { CK(cudaMemcpyAsync((dst), (src), (bytes), cudaMemcpyHostToDevice, (c)->stream)); (c)->st.h2d_bytes += (u64)(bytes); } while (0)
#define D2H(c, dst, src, bytes) do { CK(cudaMemcpyAsync((dst), (src), (bytes), cudaMemcpyDeviceToHost, (c)->stream)); (c)->st.d2h_bytes += (u64)(bytes); } while (0)
/* BWA_B200_GPUTRACE=1: every timed stage also prints its start and end on the device clock (ms since the first context was made),
 * one line per stage and lane, so that tools/gpu_timeline.py can tell how much of a run the GPU sat idle and between which stages */
static double elapsed_at(bwag_ctx_t *c, const char *stage, int line)
{
	float ms = 0;
	cudaEventElapsedTime(&ms, c->ev0, c->ev1);
	if (g_gputrace > 0) {
		float t0 = 0, t1 = 0;
		cudaEventElapsedTime(&t0, g_trace_ref, c->ev0); cudaEventElapsedTime(&t1, g_trace_ref, c->ev1);
		fprintf(stderr, "[gputrace] %p %s:%d %.3f %.3f\n", (void *)c, stage, line, t0, t1);
	}
	return ms;
}

/* ------------------------------------------------------------------------------------------------ stage 1 */

/* fastmap's form of K1 (k_smem_fm): -i and -I; NULL = the seeding of `mem` */
struct FmK1 { int min_intv; u64 max_intv; };

/* K1 (+ K1f, K1b, K2 for `mem`).  fm != NULL: K1 alone, in its fastmap form, with the same scratch sizing and repeats; the read's
 * matches stay in HBM (b->n_intv of them in the pool) */
static int seed_impl(bwag_batch_t *b, const bwag_seed_par_t *par, const FmK1 *fm, bwag_seeds_t *out)
{
	bwag_ctx_t *c = &b->lc;
	CK(cudaSetDevice(c->device));
	const int n = b->n;
	/* pools: typical short reads need ~8 intervals / ~10 seeds each; long noisy reads against a large index pick up chance matches of
	 * their minimum seed length all along (measured: 10-kbp reads at 10 % error against 3 Gbp), hence the per-base terms */
	i64 cap_intv = (i64)n * 16 + b->total_bases / 4 + 1024, cap_seeds = (i64)n * 32 + b->total_bases / 2 + 4096;
	if (getenv("BWA_B200_TEST_SMALL_POOLS")) { cap_intv = n / 2 + 8; cap_seeds = n / 2 + 8; }   /* test hook: start with pools that overflow, so that the repeat-with-reported-sizes path runs */
	int cap_list = b->max_len + 1, cap_mem = 2 * b->max_len + 64;
	/* k_smem_c (compact candidate lists, bwag_smem.cu) needs the short-string table; BWA_B200_K1_COMPACT=0 selects k_smem */
	bool k1c = false;
#ifndef K1_PACKED8
	{
		const char *e = getenv("BWA_B200_K1_COMPACT");
		k1c = (e ? atoi(e) != 0 : K1_COMPACT_DEFAULT) && c->ix.ktab_k > 0 && !fm;   /* fastmap needs every match's interval (-I): k_smem */
	}
	/* k_smem_c checks every list and result append, so long reads start with scratch for what they typically need (a few
	 * candidates with an interval per list, a result per ~4 bases) instead of the worst case: more lanes fit the scratch budget.
	 * A lane that runs out sets a flag and the stage is repeated with the worst-case sizes. */
	if (k1c && b->max_len > 2048) { cap_list = 1024; cap_mem = b->max_len / 4 + 256; }
	if (k1c && getenv("BWA_B200_TEST_SMALL_K1")) { cap_list = 9; cap_mem = 3; }   /* test hook: the repeat-with-larger-scratch path (9: the shared slots + one entry of global tail) */
#endif
	SeedArgs a;
	memset(&a, 0, sizeof(a));
	for (int attempt = 0;; ++attempt) {
		const int groups_per_block = K1_THREADS;   /* one lane per read */
		/* shared memory of a block: the heads of both candidate lists + one read slot per lane (odd number of words) */
		int qstride = (((b->max_len + 6) >> 2) | 1) << 2;
		/* + a 2-bit packed copy of each read (the keys of the short-string table): 16 bases per word, one spare word, odd word count */
		int pstride = c->ix.ktab_k ? ((((b->max_len + 15) >> 4) + 1) | 1) << 2 : 0;
		int nstride = 0;
#ifdef K1_PACKED8   /* variant: packed read + N bitmap only, eight list entries per list in shared memory (bwag_smem.cu) */
		pstride = ((((b->max_len + 15) >> 4) + 1) | 1) << 2;
		nstride = (((b->max_len + 31) >> 5) | 1) << 2;
		qstride = 0;
#endif
		size_t smem = (size_t)2 * K1_SLOTS * K1_THREADS * 16 + (size_t)K1_THREADS * (qstride + pstride + nstride);
#ifdef K1_NO_QSMEM
		qstride = 0; pstride = 0; smem = (size_t)2 * K1_SLOTS * K1_THREADS * 16;
#endif
		bool want_pack = pstride != 0;
		if (k1c) {   /* list heads + the packed copy; reads too long for that are read in place (pstride = 0) */
			qstride = 0;
			smem = (size_t)2 * K1C_SLOTS * K1_THREADS * 16 + (size_t)K1_THREADS * pstride;
			if (smem > 44 * 1024) { pstride = 0; smem = (size_t)2 * K1C_SLOTS * K1_THREADS * 16; }   /* the shared copy must not cost a resident block (registers allow 5 per SM): reads up to ~350 bases */
		} else
		if (smem > K1_SMEM_MAX) { qstride = 0; pstride = 0; nstride = 0; want_pack = false; smem = (size_t)2 * K1_SLOTS * K1_THREADS * 16; }   /* very long reads stay in global memory */
		int grid;
#ifdef BWAG_CUSIM
		grid = 2;
#else
		{
			/* BWA_B200_K1_BLOCKS: resident blocks per SM K1 may take.  K1 waits on DRAM, K4/K5 on shared memory and the integer
			 * pipes: leaving room lets another lane's K4/K5 run beside it (chunks travel on independent streams) */
			static int cap = -1;
			int nb;
			if (cap < 0) { const char *e = getenv("BWA_B200_K1_BLOCKS"); cap = e ? atoi(e) : 0; }
#ifndef K1_PACKED8
			if (k1c) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_smem_c, K1_THREADS, smem));
			else
#endif
			if (fm) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_smem_fm, K1_THREADS, smem));
			else
			CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_smem, K1_THREADS, smem));
			if (cap > 0 && nb > cap) nb = cap;
			grid = c->n_sm * (nb > 0 ? nb : 1);
		}
#endif
		const int cap3 = fm ? 1 : b->max_len / (par->min_seed_len + 1) + 2;   /* fastmap: no third pass (and -l may be -1) */
		size_t per_group = (size_t)((k1c ? 2 : 4) * cap_list + 2 * cap_mem) * 16;   /* k_smem_c has no per-call result array */
		{   /* keep the per-group scratch within ~6 GB: very long reads get fewer groups */
			size_t budget = (size_t)6 << 30;
			i64 max_groups = (i64)(budget / per_group);
			if (max_groups < groups_per_block) max_groups = groups_per_block;
			if ((i64)grid * groups_per_block > max_groups) grid = (int)(max_groups / groups_per_block);
			i64 need_groups = ((i64)n + groups_per_block - 1) / groups_per_block;
			if (grid > need_groups) grid = (int)(need_groups > 0 ? need_groups : 1);
		}
		if (buf_reserve(&c->s_k1, per_group * (size_t)grid * groups_per_block)) return 1;
		if (buf_reserve(&c->s_k1f, 32 * (size_t)cap3 * (size_t)n + 64) || buf_reserve(&c->s_n3, sizeof(int) * (size_t)(n + 1))) return 1;
		const size_t pack_words = (size_t)(b->total_bases >> 4) + 2 * (size_t)n + 8, nmask_words = nstride ? (size_t)(b->total_bases >> 5) + 2 * (size_t)n + 8 : 0;
		if (want_pack && buf_reserve(&c->s_pack, 4 * (pack_words + nmask_words + (size_t)n + 8))) return 1;
		if (buf_reserve(&b->d_intv_beg, sizeof(i64) * (size_t)(n + 1)) || buf_reserve(&b->d_intv_n, sizeof(int) * (size_t)(n + 1)) ||
		    buf_reserve(&b->d_intv, 32 * (size_t)cap_intv) || buf_reserve(&b->d_seed_beg, 8 * (size_t)cap_intv) || buf_reserve(&b->d_rbeg, 8 * (size_t)cap_seeds)) return 1;
		a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p; a.n_reads = n;
		a.min_seed_len = par->min_seed_len; a.split_len = par->split_len; a.split_width = par->split_width; a.max_occ = par->max_occ; a.max_mem_intv = par->max_mem_intv;
		a.scratch = (Intv *)c->s_k1.p; a.cap_list = cap_list; a.cap_mem = cap_mem; a.qstride = qstride; a.pstride = pstride; a.nstride = nstride;
		a.post_copies3 = k1c ? 1 : 0;
		a.stage3 = (Intv *)c->s_k1f.p; a.cap3 = cap3; a.n3 = par->max_mem_intv ? (int *)c->s_n3.p : 0; a.next_read3 = &c->d_cnt->next_read3;
		a.intv_beg = (i64 *)b->d_intv_beg.p; a.intv_n = (int *)b->d_intv_n.p; a.intv = (bwtintv_t *)b->d_intv.p; a.seed_beg = (i64 *)b->d_seed_beg.p; a.rbeg = (i64 *)b->d_rbeg.p;
		a.cap_intv = cap_intv; a.cap_seeds = cap_seeds;
		a.next_read = &c->d_cnt->next_read; a.n_intv = &c->d_cnt->n_intv; a.n_seeds = &c->d_cnt->n_seeds; a.occ_touches = &c->d_cnt->occ_touches; a.flags = &c->d_cnt->flags;
		if (reset_counters(c)) return 1;
		CK(cudaEventRecord(c->ev0, c->stream));
		if (want_pack) {   /* the packed copies K1's table lookups key on, and which reads have an ambiguous base */
			a.packed = (const u32 *)c->s_pack.p; a.nmask = nstride ? (const u32 *)c->s_pack.p + pack_words : 0; a.hasn = (const u32 *)c->s_pack.p + pack_words + nmask_words;
			BWAG_LAUNCH(k_pack_reads, (n + 127) / 128, 128, 0, c->stream, a.codes, a.off, n, (u32 *)c->s_pack.p, nstride ? (u32 *)c->s_pack.p + pack_words : (u32 *)0, (u32 *)c->s_pack.p + pack_words + nmask_words);
			CK(cudaGetLastError());
			++c->st.n_launch;
		}
		if (a.n3) {   /* third pass first: K1 appends its seeds to the read's list */
			int g3 = c->grid_k1f;
			if (g3 > (n + K1F_THREADS - 1) / K1F_THREADS) g3 = (n + K1F_THREADS - 1) / K1F_THREADS;
			BWAG_LAUNCH(k_smem_fwd, g3, K1F_THREADS, 0, c->stream, c->ix, a);
			CK(cudaGetLastError());
			++c->st.n_launch;
		}
#ifndef K1_PACKED8
		if (k1c) BWAG_LAUNCH(k_smem_c, grid, K1_THREADS, smem, c->stream, c->ix, a);
		else
#endif
		if (fm) BWAG_LAUNCH(k_smem_fm, grid, K1_THREADS, smem, c->stream, c->ix, a, fm->min_intv, fm->max_intv);
		else
		BWAG_LAUNCH(k_smem, grid, K1_THREADS, smem, c->stream, c->ix, a);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		if (!fm) {
			BWAG_LAUNCH(k_seed_post, (n + K1B_THREADS - 1) / K1B_THREADS, K1B_THREADS, 0, c->stream, a);   /* harmless if K1 overflowed: the run is repeated */
			CK(cudaGetLastError());
		}
		if (fetch_counters(c)) return 1;
		c->st.ms_smem += elapsed_at(c, "smem", __LINE__); c->st.n_launch += 2;
		if (!(c->h_cnt->flags & 41u)) break;
		if (attempt >= 6) return set_err("seeding: output pools keep overflowing (intervals %llu, seeds %llu)", (unsigned long long)c->h_cnt->n_intv, (unsigned long long)c->h_cnt->n_seeds);
		if (c->h_cnt->flags & 1u) { /* pools too small: the counters say how much is needed */
			if ((i64)c->h_cnt->n_intv > cap_intv) cap_intv = (i64)c->h_cnt->n_intv + 1024;
			if ((i64)c->h_cnt->n_seeds > cap_seeds) cap_seeds = (i64)c->h_cnt->n_seeds + 4096;
		}
		if (c->h_cnt->flags & 8u) cap_mem = cap_mem * 4 < 2 * b->max_len + 64 || !k1c ? cap_mem * 4 : 2 * b->max_len + 64;
		if (c->h_cnt->flags & 32u) cap_list = b->max_len + 1;
		if (getenv("BWA_B200_PROFILE")) fprintf(stderr, "[prof] seeding repeated (flags %u): pools %lld intervals / %lld seeds, per-lane scratch %d list entries / %d results\n", c->h_cnt->flags, (long long)cap_intv, (long long)cap_seeds, cap_list, cap_mem);
	}
	c->st.occ_touches += c->h_cnt->occ_touches;
	const i64 n_intv = (i64)c->h_cnt->n_intv, n_seeds = (i64)c->h_cnt->n_seeds;
	if (fm) { b->n_intv = n_intv; b->n_seeds = 0; b->seeded = 0; return 0; }
	/* K2: resolve the BWT rows left in rbeg[] to suffix-array positions, in place */
	if (n_seeds > 0) {
		SaArgs s;
		s.rbeg = (i64 *)b->d_rbeg.p; s.n = n_seeds; s.next = &c->d_cnt->next_seed; s.sa_touches = &c->d_cnt->sa_touches;
		int grid = c->grid_k2;
		i64 need = (n_seeds + K2_THREADS - 1) / K2_THREADS;
		if (grid > need) grid = (int)need;
		CK(cudaEventRecord(c->ev0, c->stream));
		BWAG_LAUNCH(k_sa, grid, K2_THREADS, 0, c->stream, c->ix, s);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		if (fetch_counters(c)) return 1;
		c->st.ms_sa += elapsed_at(c, "sa", __LINE__); ++c->st.n_launch;
		c->st.sa_touches += c->h_cnt->sa_touches;
	}
	b->n_intv = n_intv; b->n_seeds = n_seeds; b->seeded = 1;
	if (!out) return 0;      /* results stay in HBM for bwag_chain_extend */
	if (hbuf_reserve(&b->h_intv_beg, sizeof(i64) * (size_t)(n + 1)) || hbuf_reserve(&b->h_intv_n, sizeof(int) * (size_t)(n + 1)) ||
	    hbuf_reserve(&b->h_intv, 32 * (size_t)(n_intv + 1)) || hbuf_reserve(&b->h_seed_beg, 8 * (size_t)(n_intv + 1)) || hbuf_reserve(&b->h_rbeg, 8 * (size_t)(n_seeds + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	D2H(c, b->h_intv_beg.p, b->d_intv_beg.p, sizeof(i64) * (size_t)n);
	D2H(c, b->h_intv_n.p, b->d_intv_n.p, sizeof(int) * (size_t)n);
	if (n_intv) D2H(c, b->h_intv.p, b->d_intv.p, 32 * (size_t)n_intv);
	if (n_intv) D2H(c, b->h_seed_beg.p, b->d_seed_beg.p, 8 * (size_t)n_intv);
	if (n_seeds) D2H(c, b->h_rbeg.p, b->d_rbeg.p, 8 * (size_t)n_seeds);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __LINE__);
	out->intv_beg = (const int64_t *)b->h_intv_beg.p; out->intv_n = (const int32_t *)b->h_intv_n.p; out->intv = (const bwtintv_t *)b->h_intv.p;
	out->seed_beg = (const int64_t *)b->h_seed_beg.p; out->rbeg = (const int64_t *)b->h_rbeg.p; out->n_intv = n_intv; out->n_seeds = n_seeds;
	return 0;
}

extern "C" int bwag_seed(bwag_batch_t *b, const bwag_seed_par_t *par, bwag_seeds_t *out) { return seed_impl(b, par, 0, out); }

/* ------------------------------------------------------------------------------------------------ fastmap */

static int fm_grid(const bwag_ctx_t *c, i64 n_items)
{
	const i64 g = (n_items + 127) / 128, cap = (i64)c->n_sm * 16;
	return (int)(g < 1 ? 1 : g < cap ? g : cap);
}

/* K1 in its fastmap form, then F1-F3 (bwag_fastmap.cu) with K2 between them; every buffer sized from a scan's total */
extern "C" int bwag_fastmap(bwag_batch_t *b, const bwag_fastmap_par_t *par, bwag_fastmap_t *out)
{
	bwag_ctx_t *c = &b->lc, *pc = b->ctx;
	CK(cudaSetDevice(c->device));
	if (!pc->have_ctg) return set_err("bwag_fastmap needs the contig table (bwag_ctx_set_contigs)");
	const int n = b->n;
	for (int r = 0; r < n; ++r)
		if (b->h_off[r + 1] - b->h_off[r] >= (1 << 23)) return set_err("read %d of the batch has %lld bases; reads of 2^23 bases or more are not supported", r, (long long)(b->h_off[r + 1] - b->h_off[r]));
	bwag_seed_par_t sp;
	memset(&sp, 0, sizeof(sp));
	sp.min_seed_len = par->min_len;
	const FmK1 fm = { par->min_intv < 1 ? 1 : par->min_intv, par->max_intv };
	if (seed_impl(b, &sp, &fm, 0)) return 1;
	const i64 n_lines = b->n_intv;
	if (buf_reserve(&b->d_fm_lbeg, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_fm_toff, 8 * ((size_t)n + 1)) ||
	    buf_reserve(&b->d_fm_lines, sizeof(bwtintv_t) * ((size_t)n_lines + 1)) || buf_reserve(&b->d_fm_nrow, 8 * ((size_t)n_lines + 1)) ||
	    buf_reserve(&b->d_fm_rbeg, 8 * ((size_t)n_lines + 1)) || buf_reserve(&b->d_fm_tlen, 8 * ((size_t)n_lines + 1)) || buf_reserve(&b->d_fm_tbeg, 8 * ((size_t)n_lines + 1)) ||
	    hbuf_reserve(&b->h_fm_off, 8 * ((size_t)n + 1))) return 1;
	FmArgs f;
	memset(&f, 0, sizeof(f));
	f.n_reads = n; f.n_lines = n_lines; f.max_iwidth = (u64)(i64)par->max_iwidth; f.ctg = pc->tctg;
	f.intv_beg = (const i64 *)b->d_intv_beg.p; f.intv_n = (const int *)b->d_intv_n.p; f.intv = (const bwtintv_t *)b->d_intv.p;
	f.lbeg = (const i64 *)b->d_fm_lbeg.p; f.lines = (bwtintv_t *)b->d_fm_lines.p; f.nrow = (i64 *)b->d_fm_nrow.p; f.rbeg = (const i64 *)b->d_fm_rbeg.p;
	f.tlen = (i64 *)b->d_fm_tlen.p; f.tbeg = (const i64 *)b->d_fm_tbeg.p; f.toff = (i64 *)b->d_fm_toff.p;
	/* F1: read order, rows wanted per line, their scan */
	BWAG_LAUNCH(k_fm_scan32, 1, FM_SCAN_THREADS, 0, c->stream, (const int *)b->d_intv_n.p, (i64)n, (i64 *)b->d_fm_lbeg.p, &c->d_cnt->fm_total[0]);
	BWAG_LAUNCH(k_fm_lines, fm_grid(c, n), 128, 0, c->stream, f);
	BWAG_LAUNCH(k_fm_scan64, 1, FM_SCAN_THREADS, 0, c->stream, (const i64 *)b->d_fm_nrow.p, n_lines, (i64 *)b->d_fm_rbeg.p, &c->d_cnt->fm_total[1]);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	c->st.n_launch += 3;
	const i64 n_rows = (i64)c->h_cnt->fm_total[1];
	/* F2 + K2: the rows, resolved in place */
	if (buf_reserve(&b->d_fm_rows, 8 * ((size_t)n_rows + 1))) return 1;
	f.rows = (i64 *)b->d_fm_rows.p;
	if (n_rows > 0) {
		BWAG_LAUNCH(k_fm_rows, fm_grid(c, n_lines), 128, 0, c->stream, f);
		SaArgs s;
		s.rbeg = f.rows; s.n = n_rows; s.next = &c->d_cnt->next_seed; s.sa_touches = &c->d_cnt->sa_touches;
		int grid = c->grid_k2;
		const i64 need = (n_rows + K2_THREADS - 1) / K2_THREADS;
		if (grid > need) grid = (int)need;
		CK(cudaEventRecord(c->ev0, c->stream));
		BWAG_LAUNCH(k_sa, grid, K2_THREADS, 0, c->stream, c->ix, s);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		c->st.n_launch += 2;
	}
	/* F3: line sizes, their scan, the text, each read's range */
	BWAG_LAUNCH(k_fm_text, fm_grid(c, n_lines), 128, 0, c->stream, f, 0);
	BWAG_LAUNCH(k_fm_scan64, 1, FM_SCAN_THREADS, 0, c->stream, (const i64 *)b->d_fm_tlen.p, n_lines, (i64 *)b->d_fm_tbeg.p, &c->d_cnt->fm_total[2]);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	if (n_rows > 0) { c->st.ms_sa += elapsed_at(c, "sa", __LINE__); c->st.sa_touches += c->h_cnt->sa_touches; }
	c->st.n_launch += 2;
	const i64 n_text = (i64)c->h_cnt->fm_total[2];
	if (buf_reserve(&b->d_fm_text, (size_t)n_text + 1) || hbuf_reserve(&b->h_fm_text, (size_t)n_text + 1)) return 1;
	f.text = (char *)b->d_fm_text.p;
	BWAG_LAUNCH(k_fm_text, fm_grid(c, n_lines), 128, 0, c->stream, f, 1);
	BWAG_LAUNCH(k_fm_readoff, fm_grid(c, (i64)n + 1), 128, 0, c->stream, f);
	CK(cudaGetLastError());
	c->st.n_launch += 2;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_text) D2H(c, b->h_fm_text.p, b->d_fm_text.p, (size_t)n_text);
	D2H(c, b->h_fm_off.p, b->d_fm_toff.p, 8 * ((size_t)n + 1));
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __LINE__);
	out->text = (const char *)b->h_fm_text.p; out->off = (const int64_t *)b->h_fm_off.p;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ aln */

#ifdef BWAG_CUSIM
#define ALN_BUDGET ((i64)256 << 20)   /* the emulator's device memory is the host's */
#else
#define ALN_BUDGET ((i64)6 << 30)     /* the lanes' arenas, next to the index (K1 takes as much) */
#endif
#define ALN_T1_NODES 4096             /* queue nodes per lane in tier 1 (fewer if the lanes do not fit the budget) */
#define ALN_T2_HITS 1024              /* tier 2: room for this many hits beyond max_entries + 9 queue entries, x4 per repeat at full size */

/* a device buffer that grows and keeps its first `keep` bytes */
static int buf_grow_keep(bwag_ctx_t *c, DevBuf *b, size_t keep, size_t bytes)
{
	if (bytes <= b->cap) return 0;
	void *p = 0;
	const size_t want = bytes + bytes / 4 + 256;
	CK(cudaMalloc(&p, want));
	if (keep) CK(cudaMemcpyAsync(p, b->p, keep, cudaMemcpyDeviceToDevice, c->stream));
	CK(cudaStreamSynchronize(c->stream));
	if (b->p) cudaFree(b->p);
	b->p = p; b->cap = want;
	return 0;
}

/* A1 over all reads with small arenas (tier 1), then over the reads it listed with larger arenas (tier 2, fewer lanes: 16 times
 * the nodes per round, up to max_entries + 9 entries and room for their hits), repeated while reads are listed (a full pool grows,
 * a full-size arena too small for the hits gets more room); then the scan of the counts and A2 */
extern "C" int bwag_aln(bwag_batch_t *b, const bwag_aln_par_t *par, bwag_aln_t *out)
{
	bwag_ctx_t *c = &b->lc;
	CK(cudaSetDevice(c->device));
	const int n = b->n;
	memset(out, 0, sizeof(*out));
	for (int r = 0; r < n; ++r)
		if (b->h_off[r + 1] - b->h_off[r] >= 65536) return set_err("read %d of the batch has %lld bases; reads of 65536 bases or more are not supported", r, (long long)(b->h_off[r + 1] - b->h_off[r]));
	if (par->s_mm < 0 || par->s_gapo < 0 || par->s_gape < 0) return set_err("negative penalties are not supported");
	if (par->seed_len < 0) return set_err("the seed length must not be negative");
	int md_max = 0;
	for (int r = 0; r < n; ++r) if (par->max_diff[r] > md_max) md_max = par->max_diff[r];
	/* every score pushed is below aln_score(max_diff+1, max_gapo+1, max_gape+1), the reference's number of stacks */
	const i64 n_buckets = (i64)(md_max + 1) * par->s_mm + (i64)((par->max_gapo > 0 ? par->max_gapo : 0) + 1) * par->s_gapo + (i64)((par->max_gape > 0 ? par->max_gape : 0) + 1) * par->s_gape + 1;
	if (n_buckets > (1 << 20)) return set_err("penalties too large: %lld queue scores", (long long)n_buckets);
	const int seed_cap = par->seed_len < b->max_len ? par->seed_len : b->max_len;
	const bool small = getenv("BWA_B200_TEST_SMALL_POOLS") != 0;   /* test hook: tier 1 and the pool too small for nearly every read */
	i64 cap_pool = small ? n / 8 + 1 : 2 * (i64)n + 1024;
	if (buf_reserve(&b->d_aln_md, (size_t)n + 16) || buf_reserve(&b->d_aln_n, 4 * ((size_t)n + 1)) || buf_reserve(&b->d_aln_beg, 8 * ((size_t)n + 1)) ||
	    buf_reserve(&b->d_aln_redo[0], 4 * ((size_t)n + 1)) || buf_reserve(&b->d_aln_redo[1], 4 * ((size_t)n + 1)) || buf_reserve(&b->d_aln_off, 8 * ((size_t)n + 1)) ||
	    buf_reserve(&b->d_aln_pool, sizeof(bwag_aln1_t) * (size_t)cap_pool) ||
	    hbuf_reserve(&b->h_aln_n, 4 * ((size_t)n + 1)) || hbuf_reserve(&b->h_aln_off, 8 * ((size_t)n + 1))) return 1;
	cap_pool = (i64)(b->d_aln_pool.cap / sizeof(bwag_aln1_t));
	if (n) H2D(c, b->d_aln_md.p, par->max_diff, (size_t)n);
	if (reset_counters(c)) return 1;
	int grid_lanes = 2 * ALN_THREADS;
#ifndef BWAG_CUSIM
	{
		int nb = 0;
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_aln, ALN_THREADS, 0));
		grid_lanes = c->n_sm * (nb > 0 ? nb : 1) * ALN_THREADS;
	}
#endif
	AlnArgs a;
	memset(&a, 0, sizeof(a));
	a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p;
	a.par = *par; a.par.max_diff = (const int8_t *)b->d_aln_md.p;
	a.n_buckets = (int)n_buckets; a.max_len = b->max_len; a.seed_cap = seed_cap;
	a.n_aln = (int *)b->d_aln_n.p; a.hit_beg = (i64 *)b->d_aln_beg.p;
	a.n_pool = &c->d_cnt->aln_pool; a.n_redo = &c->d_cnt->aln_redo; a.flags = &c->d_cnt->aln_flags; a.next = &c->d_cnt->aln_next;
	i64 cap_nodes = small ? 8 : ALN_T1_NODES, hit_room = ALN_T2_HITS;
	int lanes = n < grid_lanes ? (n > 0 ? n : 1) : grid_lanes;
	while (cap_nodes > 64 && lanes * aln_layout(a.n_buckets, a.max_len, seed_cap, cap_nodes).bytes > ALN_BUDGET) cap_nodes >>= 1;
	const int *work = 0;
	int n_work = n;
	for (int round = 0;; ++round) {
		const i64 lane_bytes = aln_layout(a.n_buckets, a.max_len, seed_cap, cap_nodes).bytes;
		if (lanes > ALN_BUDGET / lane_bytes) lanes = (int)(ALN_BUDGET / lane_bytes);
		if (lanes < 1) {
			int r = 0;
			if (work) CK(cudaMemcpy(&r, work, sizeof(int), cudaMemcpyDeviceToHost));
			return set_err("read %d of the batch needs a search queue of %lld entries, more than the device can give", r, (long long)cap_nodes);
		}
		if (buf_reserve(&b->d_aln_arena, (size_t)(lanes * lane_bytes))) return 1;
		a.work = work; a.n_work = n_work; a.arena = (unsigned char *)b->d_aln_arena.p; a.lane_bytes = lane_bytes;
		a.cap_nodes = (int)cap_nodes; a.n_lanes = lanes;
		a.pool = (bwag_aln1_t *)b->d_aln_pool.p; a.cap_pool = cap_pool;
		a.redo = (int *)b->d_aln_redo[round & 1].p;
		CK(cudaMemsetAsync(&c->d_cnt->aln_next, 0, sizeof(int), c->stream));
		CK(cudaMemsetAsync(&c->d_cnt->aln_redo, 0, 2 * sizeof(u32), c->stream));
		BWAG_LAUNCH(k_aln, (lanes + ALN_THREADS - 1) / ALN_THREADS, ALN_THREADS, 0, c->stream, c->ix, a);
		CK(cudaGetLastError());
		if (fetch_counters(c)) return 1;
		++c->st.n_launch;
		const u32 n_redo = c->h_cnt->aln_redo, flags = c->h_cnt->aln_flags;
		if (round == 0) out->n_tier2 = n_redo;
		if (n_redo == 0) break;
		if (flags & 2) {   /* the pool is full: it grows, the hits already in it stay */
			const i64 want = 2 * (i64)c->h_cnt->aln_pool + 1024;
			if (buf_grow_keep(c, &b->d_aln_pool, sizeof(bwag_aln1_t) * (size_t)cap_pool, sizeof(bwag_aln1_t) * (size_t)want)) return 1;
			cap_pool = (i64)(b->d_aln_pool.cap / sizeof(bwag_aln1_t));
		}
		/* tier 2 grows the arena 16-fold per round up to max_entries + 9 entries and the hit room: most listed reads need far
		 * less than the full size, and smaller arenas leave room for more lanes */
		const i64 queue_max = (i64)(par->max_entries > 0 ? par->max_entries : 0) + 9 + 1;
		if (round > 0 && (flags & 1) && cap_nodes >= queue_max + hit_room) hit_room *= 4;   /* a full-size arena overflowed: only its hits can have done that */
		cap_nodes = cap_nodes * 16 < queue_max + hit_room ? cap_nodes * 16 : queue_max + hit_room;
		if (cap_nodes > 0x7fffffff) cap_nodes = 0x7fffffff;
		work = (const int *)b->d_aln_redo[round & 1].p; n_work = (int)n_redo;
		lanes = n_work < grid_lanes ? n_work : grid_lanes;
	}
	/* A2 */
	BWAG_LAUNCH(k_fm_scan32, 1, FM_SCAN_THREADS, 0, c->stream, (const int *)b->d_aln_n.p, (i64)n, (i64 *)b->d_aln_off.p, &c->d_cnt->aln_total);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	const i64 total = (i64)c->h_cnt->aln_total;
	if (buf_reserve(&b->d_aln_out, sizeof(bwag_aln1_t) * ((size_t)total + 1)) || hbuf_reserve(&b->h_aln_out, sizeof(bwag_aln1_t) * ((size_t)total + 1))) return 1;
	if (n) BWAG_LAUNCH(k_aln_gather, fm_grid(c, n), 128, 0, c->stream, n, (const int *)b->d_aln_n.p, (const i64 *)b->d_aln_beg.p, (const bwag_aln1_t *)b->d_aln_pool.p,
	                   (const i64 *)b->d_aln_off.p, (bwag_aln1_t *)b->d_aln_out.p);
	CK(cudaGetLastError());
	c->st.n_launch += 2;
	if (n) D2H(c, b->h_aln_n.p, b->d_aln_n.p, 4 * (size_t)n);
	D2H(c, b->h_aln_off.p, b->d_aln_off.p, 8 * ((size_t)n + 1));
	if (total) D2H(c, b->h_aln_out.p, b->d_aln_out.p, sizeof(bwag_aln1_t) * (size_t)total);
	CK(stream_wait(c));
	out->n_aln = (const int32_t *)b->h_aln_n.p; out->off = (const int64_t *)b->h_aln_off.p; out->aln = (const bwag_aln1_t *)b->h_aln_out.p;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ samse */

extern "C" int bwag_ctx_set_ambs(bwag_ctx_t *c, int n_holes, const int64_t *offset, const int32_t *len)
{
	CK(cudaSetDevice(c->device));
	const size_t bytes = 12 * (size_t)(n_holes > 0 ? n_holes : 0) + 16;   /* offsets | lengths */
	char *h = (char *)calloc(1, bytes);
	if (!h) return set_err("out of memory");
	if (n_holes > 0) { memcpy(h, offset, 8 * (size_t)n_holes); memcpy(h + 8 * (size_t)n_holes, len, 4 * (size_t)n_holes); }
	pthread_mutex_lock(&c->mu);
	if (c->d_ambs) { cudaStreamSynchronize(c->stream); cudaFree(c->d_ambs); c->d_ambs = 0; c->have_ambs = 0; }
	cudaError_t e = cudaMalloc(&c->d_ambs, bytes);
	if (e == cudaSuccess) e = cudaMemcpy(c->d_ambs, h, bytes, cudaMemcpyHostToDevice);
	free(h);
	if (e != cudaSuccess) { pthread_mutex_unlock(&c->mu); return set_err("upload of the holes failed: %s", cudaGetErrorString(e)); }
	c->n_holes = n_holes > 0 ? n_holes : 0; c->have_ambs = 1;
	pthread_mutex_unlock(&c->mu);
	return 0;
}

#ifdef BWAG_CUSIM
#define SE_BUDGET ((i64)256 << 20)
#define SE_WARPS_PER_SM 1
#else
#define SE_BUDGET ((i64)4 << 30)     /* per-warp scratch of the refinement (backtrack bytes above all) */
#define SE_WARPS_PER_SM 32
#endif

/* S1, K2, S2 and S3 (bwag_samse.cu), then S4 twice around a scan: every buffer is sized from the parameters or a scan's total.
 * The gapped hits and the room of their CIGARs are listed here, from what the caller gives (len + rlen + 2 words each: a global
 * alignment has at most len + rlen operations); the device skips those whose hit turns out unmapped or leaves XA. */
extern "C" int bwag_samse(bwag_batch_t *b, const bwag_samse_par_t *par, bwag_sam_t *out, int *past_end, int64_t *n_sa, int64_t *n_glb)
{
	bwag_ctx_t *c = &b->lc, *pc = b->ctx;
	CK(cudaSetDevice(c->device));
	memset(out, 0, sizeof(*out));
	*past_end = -1; *n_sa = 0; *n_glb = 0;
	if (!pc->have_ctg || !pc->have_ambs) return set_err("bwag_samse needs the contig table and the holes (bwag_ctx_set_contigs, bwag_ctx_set_ambs)");
	const int n = b->n;
	const i64 nm = par->n_multi, n_rows = (i64)n + nm;
	if (hbuf_reserve(&b->h_se_tasks, sizeof(SeTask) * ((size_t)n_rows + 1)) || hbuf_reserve(&b->h_se_mtask, 4 * ((size_t)n_rows + 1))) return 1;
	SeTask *tasks = (SeTask *)b->h_se_tasks.p;
	int *mtask = (int *)b->h_se_mtask.p;   /* [n] the chosen hit's task, then [nm] each candidate's */
	int n_tasks = 0, cap_q = 1, cap_r = 1;
	i64 n_cig = 0, cap_z = 1, n_mapped = 0;
	for (int r = 0; r < n; ++r) {
		const bwag_se_read_t &p = par->reads[r];
		if (p.len < 1 || p.len > (int)(b->h_off[r + 1] - b->h_off[r])) return set_err("read %d of the batch: %d bases searched of %lld", r, p.len, (long long)(b->h_off[r + 1] - b->h_off[r]));
		n_mapped += p.type != 0;
		for (int k = -1; k < p.n_multi; ++k) {
			const i64 slot = k < 0 ? -1 : p.multi_beg + k;
			int &mt = k < 0 ? mtask[r] : mtask[n + slot];
			mt = -1;
			if (k < 0 ? !(p.type && p.n_gapo) : !par->multi[slot].gap) continue;
			const int rlen = p.len + (k < 0 ? p.ref_shift : par->multi[slot].ref_shift);
			if (rlen < 0) return set_err("read %d of the batch: a gapped hit with %d reference bases", r, rlen);
			int w = (int)(abs(rlen - p.len) * 1.5);
			w = w > 50 ? w : 50;
			const i64 n_col = p.len < 2 * w + 1 ? p.len : 2 * w + 1;
			mt = n_tasks;
			tasks[n_tasks].read = r; tasks[n_tasks].slot = (int)slot; tasks[n_tasks].cig_off = n_cig;
			++n_tasks;
			n_cig += (i64)p.len + rlen + 2;
			if (p.len > cap_q) cap_q = p.len;
			if (rlen > cap_r) cap_r = rlen;
			if (n_col * rlen > cap_z) cap_z = n_col * rlen;
		}
	}
	*n_sa = n_mapped + nm;
	const size_t l_rg = par->rg_id ? strlen(par->rg_id) : 0;
	if (buf_reserve(&b->d_se_reads, sizeof(bwag_se_read_t) * ((size_t)n + 1)) || buf_reserve(&b->d_se_multi, sizeof(bwag_se_hit_t) * ((size_t)nm + 1)) ||
	    buf_reserve(&b->d_se_bc, (size_t)par->l_bc + l_rg + 16) || buf_reserve(&b->d_se_rows, 8 * ((size_t)n_rows + 1)) ||
	    buf_reserve(&b->d_se_pos, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_se_mpos, 8 * ((size_t)nm + 1)) || buf_reserve(&b->d_se_flags, 2 * (size_t)n_rows + 16) ||
	    buf_reserve(&b->d_se_tasks, sizeof(SeTask) * ((size_t)n_tasks + 1)) || buf_reserve(&b->d_se_mtask, 4 * ((size_t)n_rows + 1)) ||
	    buf_reserve(&b->d_se_cig, 4 * ((size_t)n_cig + 1)) || buf_reserve(&b->d_se_ncig, 8 * ((size_t)n_tasks + 1)) ||
	    buf_reserve(&b->d_se_tlen, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_se_tbeg, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_se_nm, 4 * ((size_t)n + 1)) || buf_reserve(&b->d_se_rec, sizeof(bwag_samrec_t) * ((size_t)n + 1)) ||
	    hbuf_reserve(&b->h_se_rec, sizeof(bwag_samrec_t) * ((size_t)n + 1))) return 1;
	SeArgs a;
	memset(&a, 0, sizeof(a));
	a.n_reads = n; a.n_multi = nm; a.n_tasks = n_tasks; a.mode = par->mode; a.max_top2 = par->max_top2;
	a.ctg = pc->tctg; a.n_holes = pc->n_holes; a.amb_off = (const i64 *)pc->d_ambs; a.amb_len = (const int *)((const char *)pc->d_ambs + 8 * (size_t)pc->n_holes);
	a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p;
	a.reads = (const bwag_se_read_t *)b->d_se_reads.p; a.multi = (const bwag_se_hit_t *)b->d_se_multi.p;
	a.bc = (const char *)b->d_se_bc.p; a.rg = (const char *)b->d_se_bc.p + par->l_bc; a.l_rg = (int)l_rg;
	a.rows = (i64 *)b->d_se_rows.p; a.pos = (i64 *)b->d_se_pos.p; a.mpos = (i64 *)b->d_se_mpos.p;
	a.strand = (uint8_t *)b->d_se_flags.p; a.mapped = a.strand + n; a.mstrand = a.mapped + n; a.mkeep = a.mstrand + nm;
	a.tasks = (const SeTask *)b->d_se_tasks.p; a.main_task = (const int *)b->d_se_mtask.p; a.multi_task = a.main_task + n;
	a.cig = (u32 *)b->d_se_cig.p; a.ncig = (int *)b->d_se_ncig.p; a.tshift = a.ncig + n_tasks;
	a.next_task = &c->d_cnt->se_next; a.past_end = &c->d_cnt->se_past; a.n_run = &c->d_cnt->se_run; a.cells = &c->d_cnt->se_cells;
	a.tlen = (i64 *)b->d_se_tlen.p; a.tbeg = (const i64 *)b->d_se_tbeg.p; a.rec = (bwag_samrec_t *)b->d_se_rec.p; a.nm = (int *)b->d_se_nm.p;
	if (reset_counters(c)) return 1;
	if (n) H2D(c, b->d_se_reads.p, par->reads, sizeof(bwag_se_read_t) * (size_t)n);
	if (nm) H2D(c, b->d_se_multi.p, par->multi, sizeof(bwag_se_hit_t) * (size_t)nm);
	if (par->l_bc) H2D(c, b->d_se_bc.p, par->bc, (size_t)par->l_bc);
	if (l_rg) H2D(c, (char *)b->d_se_bc.p + par->l_bc, par->rg_id, l_rg);
	if (n_tasks) H2D(c, b->d_se_tasks.p, tasks, sizeof(SeTask) * (size_t)n_tasks);
	if (n_rows) H2D(c, b->d_se_mtask.p, mtask, 4 * (size_t)n_rows);
	/* S1 + K2: the rows, resolved in place; S2 */
	if (n_rows) {
		BWAG_LAUNCH(k_se_rows, fm_grid(c, n_rows), 128, 0, c->stream, a);
		SaArgs sa;
		sa.rbeg = a.rows; sa.n = n_rows; sa.next = &c->d_cnt->next_seed; sa.sa_touches = &c->d_cnt->sa_touches;
		int grid = c->grid_k2;
		const i64 need = (n_rows + K2_THREADS - 1) / K2_THREADS;
		if (grid > need) grid = (int)need;
		CK(cudaEventRecord(c->ev0, c->stream));
		BWAG_LAUNCH(k_sa, grid, K2_THREADS, 0, c->stream, c->ix, sa);
		CK(cudaEventRecord(c->ev1, c->stream));
		BWAG_LAUNCH(k_se_pos, fm_grid(c, n), 128, 0, c->stream, a);
		CK(cudaGetLastError());
		c->st.n_launch += 3;
	}
	/* S3: persistent warps over the gapped hits, as many as the scratch budget allows */
	if (n_tasks) {
		const i64 per_warp = (8 * ((i64)cap_q + 2) + cap_r + cap_q + cap_z + 15) & ~(i64)15;
		i64 warps = (i64)c->n_sm * SE_WARPS_PER_SM;
		if (warps > n_tasks) warps = n_tasks;
		if (warps > SE_BUDGET / per_warp) warps = SE_BUDGET / per_warp;
		if (warps < 1) warps = 1;
		warps = (warps + 3) & ~(i64)3;   /* whole blocks of SE_THREADS */
		if (buf_reserve(&b->d_se_scratch, (size_t)(warps * per_warp))) return 1;
		unsigned char *sc = (unsigned char *)b->d_se_scratch.p;
		a.eh = (int *)sc; sc += warps * 8 * ((i64)cap_q + 2);
		a.rseq = sc; sc += warps * (i64)cap_r;
		a.qseq = sc; sc += warps * (i64)cap_q;
		a.z = sc;
		a.cap_q = cap_q; a.cap_r = cap_r; a.cap_z = cap_z;
		CK(cudaMemsetAsync(b->d_se_ncig.p, 0, 8 * (size_t)n_tasks, c->stream));
		BWAG_LAUNCH(k_se_refine, (int)(warps * 32 / SE_THREADS), SE_THREADS, 0, c->stream, c->ix, a);
		CK(cudaGetLastError());
		++c->st.n_launch;
	}
	/* S4: sizes, their scan, then the text */
	if (n) BWAG_LAUNCH(k_se_text, fm_grid(c, n), 128, 0, c->stream, c->ix, a, 0);
	BWAG_LAUNCH(k_fm_scan64, 1, FM_SCAN_THREADS, 0, c->stream, (const i64 *)b->d_se_tlen.p, (i64)n, (i64 *)b->d_se_tbeg.p, &c->d_cnt->se_total);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	c->st.n_launch += 2;
	if (n_rows) { c->st.ms_sa += elapsed_at(c, "sa", __LINE__); c->st.sa_touches += c->h_cnt->sa_touches; }
	c->st.glb_cells += c->h_cnt->se_cells;
	*n_glb = (int64_t)c->h_cnt->se_run;
	if (c->h_cnt->se_past) {
		*past_end = n - c->h_cnt->se_past;
		return set_err("read %d of the batch: its gapped alignment window runs past the end of the forward strand", *past_end);
	}
	const i64 n_text = (i64)c->h_cnt->se_total;
	if (buf_reserve(&b->d_se_text, (size_t)n_text + 1) || hbuf_reserve(&b->h_se_text, (size_t)n_text + 1)) return 1;
	a.text = (char *)b->d_se_text.p;
	if (n) BWAG_LAUNCH(k_se_text, fm_grid(c, n), 128, 0, c->stream, c->ix, a, 1);
	CK(cudaGetLastError());
	++c->st.n_launch;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_text) D2H(c, b->h_se_text.p, b->d_se_text.p, (size_t)n_text);
	if (n) D2H(c, b->h_se_rec.p, b->d_se_rec.p, sizeof(bwag_samrec_t) * (size_t)n);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __LINE__);
	out->rec = (const bwag_samrec_t *)b->h_se_rec.p; out->text = (const char *)b->h_se_text.p; out->n_text = n_text;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ stage 2 */

/* K4 with its per-warp scratch in shared memory when that fits, else in global memory; n_units = reads to process */
static int k4_lane_maxchains(void) { const char *e = getenv("BWA_B200_K4_LANE_MAXCHAINS"); return e ? atoi(e) : 8; }

/* n_many: reads with more chains than the lane kernel takes, if the caller knows (K3 counts them), else -1 */
static int launch_extend(bwag_ctx_t *c, ExtArgs &a, int n_units, int n_many = -1)
{
	const int wpb = K4_THREADS / 32;
	a.chain_lo = 0; a.chain_hi = 0x7fffffff;
	int per_warp = (8 * (a.cap_q + 2) + a.cap_r + a.cap_q + 15) & ~15;
	size_t smem = (size_t)per_warp * wpb;
	int grid = c->grid_k4, use_sm = smem <= K4_SMEM_MAX && !(getenv("BWA_B200_K4_SM") && atoi(getenv("BWA_B200_K4_SM")) == 0);
	/* the leaner row sweep (and its row cut-off) needs non-negative gap penalties (every real scoring scheme); BWA_B200_K4_FAST=0 forces the general one */
	const int fast = a.par.e_ins >= 0 && a.par.o_ins + a.par.e_ins >= 0 && a.par.e_del >= 0 && a.par.o_del + a.par.e_del >= 0 &&
	                 !c->baseline && !(getenv("BWA_B200_K4_FAST") && atoi(getenv("BWA_B200_K4_FAST")) == 0);
	{   /* short reads: one lane per read (bwag_extend_lane.cu) when every score fits its 13-bit cells and a block's columns fit shared memory */
		int maxsc = 0;
		for (int k = 0; k < 25; ++k) maxsc = maxsc > a.par.mat[k] ? maxsc : a.par.mat[k];
		const int lcols = a.cap_q - (a.min_seed > 0 && a.min_seed < a.cap_q ? a.min_seed - 3 : 0) + 2 + 8;   /* longest extension (read minus its shortest possible seed; cap_q rounds the read length up by <= 3) + column `end` + the chunk's spare columns (K4L_CH) */
		const size_t lsm = (size_t)lcols * K4L_THREADS * 4;
		const int lane_ok = fast && (i64)a.cap_q * maxsc < 8192 && a.par.a <= maxsc && lsm <= K4L_SMEM_MAX && !(getenv("BWA_B200_K4_LANE") && atoi(getenv("BWA_B200_K4_LANE")) == 0);
		if (lane_ok) {
			int lgrid = c->n_sm;
#ifndef BWAG_CUSIM
			{ int nb = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_extend_lane, K4L_THREADS, lsm)); lgrid = c->n_sm * (nb > 0 ? nb : 1); }
#else
			lgrid = 2;
#endif
			const i64 lneed = ((i64)n_units + K4L_THREADS - 1) / K4L_THREADS;
			if (lgrid > lneed) lgrid = (int)(lneed > 0 ? lneed : 1);
			/* a lane works through its read's chains one after the other, which is right for the usual one or two chains and hopeless for a
			 * read from a repeat family with hundreds (measured on the repeat-rich workload): those go to the warp-per-read kernel below */
			const int many = k4_lane_maxchains();
			ExtArgs la = a;
			la.eh = 0; la.rseq = 0; la.smem_per_warp = lcols;   /* here: the number of columns of a lane's row */
			la.chain_lo = 0; la.chain_hi = many;
			if (getenv("BWA_B200_PROFILE")) fprintf(stderr, "[prof] extension: lane-per-read kernel, grid %d x %d, %zu bytes of shared memory per block\n", lgrid, K4L_THREADS, lsm);
			BWAG_LAUNCH(k_extend_lane, lgrid, K4L_THREADS, lsm, c->stream, c->ix, la);
			CK(cudaGetLastError());
			++c->st.n_launch;
			if (n_many == 0) return 0;                 /* no read is left for the warp-per-read kernel */
			CK(cudaMemsetAsync(a.next_read, 0, sizeof(int), c->stream));
			a.chain_lo = many + 1; a.chain_hi = 0x7fffffff;
		}
	}
#ifndef BWAG_CUSIM
	if (use_sm) { int nb = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fast ? k_extend_sm_fast : k_extend_sm, K4_THREADS, smem)); if (nb < 2) use_sm = 0; else grid = c->n_sm * nb; }
#endif
	i64 need = ((i64)n_units + wpb - 1) / wpb;
	if (grid > need) grid = (int)(need > 0 ? need : 1);
	if (!use_sm) {
		const size_t n_warps = (size_t)grid * wpb;
		if (buf_reserve(&c->s_eh, n_warps * 2 * (size_t)(a.cap_q + 2) * 4) || buf_reserve(&c->s_rseq, n_warps * (size_t)a.cap_r)) return 1;
		a.eh = (int *)c->s_eh.p; a.rseq = (uint8_t *)c->s_rseq.p; a.smem_per_warp = 0;
		if (fast) BWAG_LAUNCH(k_extend_fast, grid, K4_THREADS, 0, c->stream, c->ix, a);
		else BWAG_LAUNCH(k_extend, grid, K4_THREADS, 0, c->stream, c->ix, a);
	} else {
		a.eh = 0; a.rseq = 0; a.smem_per_warp = per_warp;
		if (fast) BWAG_LAUNCH(k_extend_sm_fast, grid, K4_THREADS, smem, c->stream, c->ix, a);
		else BWAG_LAUNCH(k_extend_sm, grid, K4_THREADS, smem, c->stream, c->ix, a);
	}
	CK(cudaGetLastError());
	return 0;
}


extern "C" int bwag_extend(bwag_batch_t *b, const bwag_sw_par_t *par, const int32_t *chain_off, const bwag_xchain_t *chains,
                           int64_t n_seeds, const bwag_xseed_t *seeds, bwag_regs_t *out)
{
	bwag_ctx_t *c = &b->lc;
	CK(cudaSetDevice(c->device));
	const int n = b->n;
	const i64 n_chains = chain_off[n];
	int cap_r = 16;
	for (i64 i = 0; i < n_chains; ++i) { i64 l = chains[i].rmax1 - chains[i].rmax0; if (l > cap_r) cap_r = (int)l; }
	cap_r = (cap_r + 15) & ~15;
	const int cap_q = (b->max_len + 3) & ~3;
	int grid = c->grid_k4;
	{
		i64 need = ((i64)n + (K4_THREADS / 32) - 1) / (K4_THREADS / 32);
		if (grid > need) grid = (int)(need > 0 ? need : 1);
	}
	if (buf_reserve(&b->d_chain_off, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_chains, sizeof(bwag_xchain_t) * (size_t)(n_chains + 1)) ||
	    buf_reserve(&b->d_seeds, sizeof(bwag_xseed_t) * (size_t)(n_seeds + 1)) || buf_reserve(&b->d_regs, sizeof(bwag_xreg_t) * (size_t)(n_seeds + 1)) ||
	    buf_reserve(&b->d_nregs, 4 * (size_t)(n + 1))) return 1;
	if (buf_reserve(&b->d_chain_beg, 8 * (size_t)(n + 1)) || buf_reserve(&b->d_chain_cnt, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_reg_base, 8 * (size_t)(n + 1)) ||
	    hbuf_reserve(&b->h_tmp, 20 * (size_t)(n + 1))) return 1;
	i64 *h_cbeg = (i64 *)b->h_tmp.p, *h_rbase = h_cbeg + n + 1;
	int *h_ccnt = (int *)(h_rbase + n + 1);
	for (int r = 0; r < n; ++r) {   /* per read: its chains, and where its regions go (the slot range of its seeds) */
		h_cbeg[r] = chain_off[r]; h_ccnt[r] = chain_off[r + 1] - chain_off[r];
		h_rbase[r] = h_ccnt[r] ? chains[chain_off[r]].seed_off : 0;
	}
	if (reset_counters(c)) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	H2D(c, b->d_chain_beg.p, h_cbeg, 8 * (size_t)n);
	H2D(c, b->d_reg_base.p, h_rbase, 8 * (size_t)n);
	H2D(c, b->d_chain_cnt.p, h_ccnt, 4 * (size_t)n);
	if (n_chains) H2D(c, b->d_chains.p, chains, sizeof(bwag_xchain_t) * (size_t)n_chains);
	if (n_seeds) H2D(c, b->d_seeds.p, seeds, sizeof(bwag_xseed_t) * (size_t)n_seeds);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_h2d += elapsed_at(c, "h2d", __LINE__);
	ExtArgs a;
	memset(&a, 0, sizeof(a));
	a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p; a.n_reads = n; a.par = *par;
	a.chain_beg = (const i64 *)b->d_chain_beg.p; a.chain_cnt = (const int *)b->d_chain_cnt.p; a.reg_base = (const i64 *)b->d_reg_base.p;
	a.chains = (const bwag_xchain_t *)b->d_chains.p; a.seeds = (const bwag_xseed_t *)b->d_seeds.p;
	a.regs = (bwag_xreg_t *)b->d_regs.p; a.n_regs = (int32_t *)b->d_nregs.p;
	a.cap_q = cap_q; a.cap_r = cap_r;
	a.next_read = &c->d_cnt->next_read; a.cells = &c->d_cnt->ext_cells; a.flags = &c->d_cnt->flags;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (launch_extend(c, a, n)) return 1;
	CK(cudaEventRecord(c->ev1, c->stream));
	if (fetch_counters(c)) return 1;
	c->st.ms_extend += elapsed_at(c, "extend", __LINE__); ++c->st.n_launch;
	if (c->h_cnt->flags & 2u) return set_err("extension: a read or reference window exceeded the scratch capacity");
	c->st.ext_cells += c->h_cnt->ext_cells;
	if (hbuf_reserve(&b->h_regs, sizeof(bwag_xreg_t) * (size_t)(n_seeds + 1)) || hbuf_reserve(&b->h_nregs, 4 * (size_t)(n + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_seeds) D2H(c, b->h_regs.p, b->d_regs.p, sizeof(bwag_xreg_t) * (size_t)n_seeds);
	D2H(c, b->h_nregs.p, b->d_nregs.p, 4 * (size_t)n);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __LINE__);
	out->n_regs = (const int32_t *)b->h_nregs.p; out->regs = (const bwag_xreg_t *)b->h_regs.p;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ stages 2a+2 fused */

/* K6 over n_tasks tasks that are in b->d_swtasks already (queries/targets: the batch's reads, the reference, or b->d_swpool);
 * results to b->d_swres.  max_q / max_t: no task is longer.  Records ev0/ev1 around the kernel; the caller fetches the counters. */
static int localsw_on_device(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, int max_q, int max_t)
{
	bwag_ctx_t *c = &b->lc;
	const int cap_q = ((max_q > 16 ? max_q : 16) + 15) & ~15, cap_t = ((max_t > 16 ? max_t : 16) + 15) & ~15;
	const int cap_n = cap_q + 16;                                       /* query length rounded up to a whole number of vectors */
	/* warp per task (vectors in shared memory) when a block's share fits, else lane per task (everything in a global scratch slice) */
	const size_t w_smem = (size_t)(8 * cap_n + cap_q) * 4;
	const int warp_ok = w_smem <= K4_SMEM_MAX && !(getenv("BWA_B200_K6_WARP") && atoi(getenv("BWA_B200_K6_WARP")) == 0);
	const i64 per_thread = warp_ok ? (((i64)cap_t * 8 + cap_t + 63) & ~(i64)63) : (((i64)cap_n * 8 + (i64)cap_t * 8 + cap_q + cap_t + 63) & ~(i64)63);   /* per warp / per lane */
	int grid = c->n_sm * 16;
	if (warp_ok) {
#ifndef BWAG_CUSIM
		int nb = 0;
		CK(cudaFuncSetAttribute(k_localsw_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_localsw_warp, 128, w_smem));
		grid = c->n_sm * (nb > 0 ? nb : 1);
#else
		grid = 2;
#endif
		const i64 need = ((i64)n_tasks + 3) / 4;
		if (grid > need) grid = (int)need;
	} else {
		const i64 need = ((i64)n_tasks + 63) / 64;
		if (grid > need) grid = (int)need;
		const i64 max_threads = ((i64)4 << 30) / per_thread;            /* bound the scratch to ~4 GB */
		if ((i64)grid * 64 > max_threads) grid = (int)(max_threads / 64 > 0 ? max_threads / 64 : 1);
	}
	if (buf_reserve(&b->d_swres, sizeof(bwag_swres_t) * (size_t)n_tasks) || buf_reserve(&b->d_swscratch, (size_t)per_thread * (size_t)grid * (warp_ok ? 4 : 64)) ||
	    buf_reserve(&b->d_swpool, 16)) return 1;
	SwArgs a;
	memset(&a, 0, sizeof(a));
	a.tasks = (const bwag_swtask_t *)b->d_swtasks.p; a.n_tasks = n_tasks; a.par = *par;
	a.codes = (const uint8_t *)b->d_codes.p; a.pool = (const uint8_t *)b->d_swpool.p; a.res = (bwag_swres_t *)b->d_swres.p;
	a.scratch = (unsigned char *)b->d_swscratch.p; a.per_thread = per_thread; a.cap_n = cap_n; a.cap_q = cap_q; a.cap_t = cap_t;
	a.next_task = &c->d_cnt->next_task; a.flags = &c->d_cnt->flags;
	CK(cudaMemsetAsync(&c->d_cnt->next_task, 0, sizeof(int), c->stream));
	CK(cudaEventRecord(c->ev0, c->stream));
	if (warp_ok) BWAG_LAUNCH(k_localsw_warp, grid, 128, w_smem, c->stream, c->ix, a);
	else BWAG_LAUNCH(k_localsw, grid, 64, 0, c->stream, c->ix, a);
	CK(cudaGetLastError());
	CK(cudaEventRecord(c->ev1, c->stream));
	return 0;
}

extern "C" int bwag_localsw(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, const bwag_swtask_t *tasks, const uint8_t *pool, size_t pool_bytes, const bwag_swres_t **out)
{
	bwag_ctx_t *c = &b->lc;
	CK(cudaSetDevice(c->device));
	*out = 0;
	if (n_tasks <= 0) return 0;
	int max_q = 16, max_t = 16;
	for (int t = 0; t < n_tasks; ++t) { if (tasks[t].qlen > max_q) max_q = tasks[t].qlen; if (tasks[t].tlen > max_t) max_t = tasks[t].tlen; }
	if (buf_reserve(&b->d_swtasks, sizeof(bwag_swtask_t) * (size_t)n_tasks) || buf_reserve(&b->d_swpool, pool_bytes + 16) ||
	    hbuf_reserve(&b->h_swres, sizeof(bwag_swres_t) * (size_t)n_tasks)) return 1;
	if (reset_counters(c)) return 1;
	H2D(c, b->d_swtasks.p, tasks, sizeof(bwag_swtask_t) * (size_t)n_tasks);
	if (pool && pool_bytes) H2D(c, b->d_swpool.p, pool, pool_bytes);
	if (localsw_on_device(b, par, n_tasks, max_q, max_t)) return 1;
	D2H(c, b->h_swres.p, b->d_swres.p, sizeof(bwag_swres_t) * (size_t)n_tasks);
	if (fetch_counters(c)) return 1;
	c->st.ms_localsw += elapsed_at(c, "localsw", __LINE__); ++c->st.n_launch; c->st.sw_tasks += (u64)n_tasks;
	if (c->h_cnt->flags & 32u) return set_err("local alignment: a task exceeded the scratch capacity");
	*out = (const bwag_swres_t *)b->h_swres.p;
	return 0;
}

extern "C" int bwag_chain_extend(bwag_batch_t *b, const bwag_chain_par_t *cp, const bwag_sw_par_t *par, const bwag_contigs_t *ctg, bwag_cregs_t *out)
{
	bwag_ctx_t *c = &b->lc;
	CK(cudaSetDevice(c->device));
	if (!b->seeded) return set_err("bwag_chain_extend needs a preceding bwag_seed on the same batch");
	const int n = b->n;
	const i64 ns = b->n_seeds;
	if (ns >= ((i64)1 << 31)) return set_err("too many seeds in one batch for the 32-bit seed offsets; use smaller chunks");
	/* contig table: offsets (i64), lengths (int), ALT flags (byte) in one device buffer */
	const size_t ctg_bytes = (size_t)ctg->n_seqs * 13 + 64;
	if (buf_reserve(&b->d_ctg, ctg_bytes) || hbuf_reserve(&b->h_tmp, ctg_bytes)) return 1;
	{
		char *h = (char *)b->h_tmp.p;
		memcpy(h, ctg->offset, 8 * (size_t)ctg->n_seqs);
		memcpy(h + 8 * (size_t)ctg->n_seqs, ctg->len, 4 * (size_t)ctg->n_seqs);
		memcpy(h + 12 * (size_t)ctg->n_seqs, ctg->is_alt, (size_t)ctg->n_seqs);
	}
	if (buf_reserve(&b->s_bt, 88 * (size_t)(ns + 1)) || buf_reserve(&b->s_sn, 32 * (size_t)(ns + 1)) || buf_reserve(&b->s_ch, 48 * (size_t)(ns + 1)) ||
	    buf_reserve(&b->s_order, 4 * (size_t)(ns + 1)) || buf_reserve(&b->s_idx, 4 * (size_t)(ns + 1)) || buf_reserve(&b->s_keys, 8 * (size_t)(ns + 1)) ||
	    buf_reserve(&b->d_chains, sizeof(bwag_xchain_t) * (size_t)(ns + 1)) || buf_reserve(&b->d_seeds, sizeof(bwag_xseed_t) * (size_t)(ns + 1)) ||
	    buf_reserve(&b->d_regs, sizeof(bwag_xreg_t) * (size_t)(ns + 1)) || buf_reserve(&b->d_chain_rid, 4 * (size_t)(ns + 1)) || buf_reserve(&b->d_chain_frac, 4 * (size_t)(ns + 1)) ||
	    buf_reserve(&b->d_chain_beg, 8 * (size_t)(n + 1)) || buf_reserve(&b->d_chain_cnt, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_reg_base, 8 * (size_t)(n + 1)) ||
	    buf_reserve(&b->d_nregs, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_creg_beg, 8 * (size_t)(n + 1)) || buf_reserve(&b->d_k3big, 4 * (size_t)(n + 1))) return 1;
	if (reset_counters(c)) return 1;
	H2D(c, b->d_ctg.p, b->h_tmp.p, 13 * (size_t)ctg->n_seqs);
	ChainArgs k;
	memset(&k, 0, sizeof(k));
	k.off = (const i64 *)b->d_off.p; k.n_reads = n;
	k.intv_beg = (const i64 *)b->d_intv_beg.p; k.intv_n = (const int *)b->d_intv_n.p; k.intv = (const bwtintv_t *)b->d_intv.p;
	k.seed_beg = (const i64 *)b->d_seed_beg.p; k.rbeg = (const i64 *)b->d_rbeg.p;
	k.w = cp->w; k.max_chain_gap = cp->max_chain_gap; k.max_occ = cp->max_occ; k.min_seed_len = cp->min_seed_len; k.min_chain_weight = cp->min_chain_weight;
	k.max_chain_extend = cp->max_chain_extend; k.mask_level = cp->mask_level; k.drop_ratio = cp->drop_ratio;
	k.a = par->a; k.o_del = par->o_del; k.e_del = par->e_del; k.o_ins = par->o_ins; k.e_ins = par->e_ins;
	k.l_pac = c->ix.l_pac; k.n_seqs = ctg->n_seqs;
	k.ctg_off = (const i64 *)b->d_ctg.p; k.ctg_len = (const int *)((char *)b->d_ctg.p + 8 * (size_t)ctg->n_seqs); k.ctg_alt = (const uint8_t *)b->d_ctg.p + 12 * (size_t)ctg->n_seqs;
	k.s_bt = b->s_bt.p; k.s_sn = b->s_sn.p; k.s_ch = b->s_ch.p; k.s_order = (int *)b->s_order.p; k.s_idx = (int *)b->s_idx.p; k.s_keys = (u64 *)b->s_keys.p;
	k.xchains = (bwag_xchain_t *)b->d_chains.p; k.xseeds = (bwag_xseed_t *)b->d_seeds.p; k.chain_rid = (int *)b->d_chain_rid.p; k.chain_frac = (float *)b->d_chain_frac.p;
	k.chain_beg = (i64 *)b->d_chain_beg.p; k.reg_base = (i64 *)b->d_reg_base.p; k.n_chains = (int *)b->d_chain_cnt.p;
	k.max_rlen = &c->d_cnt->max_rlen; k.n_many = &c->d_cnt->n_many; k.many = k4_lane_maxchains();
	{   /* seed-level filter of long reads (mem_flt_chained_seeds, bwamem.c:626-641): threshold by read length, from the host's libm
	     * (the value is truncated to an int: bwamem.c:628); no table if no read of the chunk can be long enough */
		const int L = b->max_len;
		int any = 0;
		if (hbuf_reserve(&b->h_hsp, sizeof(int) * (size_t)(L + 2))) return 1;
		int *tab = (int *)b->h_hsp.p;
		for (int l = 0; l <= L; ++l) {
			const double min_l = cp->min_chain_weight ? 1.1f * cp->min_chain_weight : 5.5f * log((double)l);
			tab[l] = min_l > 0.05f * l ? -1 : (int)(par->a * min_l + .499);
			if (tab[l] >= 0 && l >= cp->min_seed_len) any = 1;
		}
		if (any && !(getenv("BWA_B200_DEVICE_SEEDSW") && atoi(getenv("BWA_B200_DEVICE_SEEDSW")) == 0)) {
			if (buf_reserve(&b->d_hsp, sizeof(int) * (size_t)(L + 2)) || buf_reserve(&b->d_flt_nchn, sizeof(int) * (size_t)(n + 1)) ||
			    buf_reserve(&b->d_swtasks, sizeof(bwag_swtask_t) * (size_t)(ns + 1))) return 1;
			H2D(c, b->d_hsp.p, tab, sizeof(int) * (size_t)(L + 1));
			k.hsp_tab = (const int *)b->d_hsp.p; k.flt_nchn = (int *)b->d_flt_nchn.p;
			k.sw_tasks = (bwag_swtask_t *)b->d_swtasks.p; k.n_swtasks = &c->d_cnt->n_swtasks;
		} else if (any) return BWAG_DECLINED;   /* switched off: the caller chains these reads on the host */
	}
#ifdef BWAG_K3_CLOCKS
	CK(cudaMalloc((void **)&k.k3clk, 20 * (size_t)(n + 1)));
#endif
	/* Without the long-read filter, k_chain_sm chains the reads with few seeds in shared memory and lists the others, which
	 * k_chain then takes with their workspace in HBM (grid-stride over the list, whose length only the device knows).  With the
	 * filter every read takes k_chain: K3b reads the HBM workspace back. */
	const int on_chip = !k.hsp_tab;
	int k3_grid = (n + K3_THREADS - 1) / K3_THREADS;
	if (on_chip) {
		k.big = (int *)b->d_k3big.p; k.n_big = &c->d_cnt->n_big;
		if (k3_grid > c->n_sm * 16) k3_grid = c->n_sm * 16;
	}
	CK(cudaEventRecord(c->ev0, c->stream));
	if (on_chip) {
		BWAG_LAUNCH(k_chain_sm, (n + K3S_THREADS - 1) / K3S_THREADS, K3S_THREADS, K3S_SMEM, c->stream, k);
		CK(cudaGetLastError());
	}
	BWAG_LAUNCH(k_chain, k3_grid > 0 ? k3_grid : 1, K3_THREADS, 0, c->stream, k);
	CK(cudaGetLastError());
	CK(cudaEventRecord(c->ev1, c->stream));
	if (fetch_counters(c)) return 1;
	c->st.ms_chain += elapsed_at(c, "chain", __LINE__); c->st.n_launch += 1 + on_chip;
	if (getenv("BWA_B200_PROFILE"))
		fprintf(stderr, "[prof] chain: %d reads on chip, %d in HBM, CAP %d seeds, %d blocks of %d threads per SM on chip\n",
		        on_chip ? n - c->h_cnt->n_big : 0, on_chip ? c->h_cnt->n_big : n, K3S_CAP, c->k3s_blocks, K3S_THREADS);
#ifdef BWAG_K3_CLOCKS
	{
		u32 *h = (u32 *)malloc(20 * (size_t)(n + 1));
		CK(cudaMemcpy(h, k.k3clk, 20 * (size_t)n, cudaMemcpyDeviceToHost));
		CK(cudaFree(k.k3clk));
		k.k3clk = 0;
		k3clk_add(h, n);
		free(h);
	}
#endif
	if (k.hsp_tab) {
		const int n_sw = (int)c->h_cnt->n_swtasks;
		if (n_sw > 0) {
			if (localsw_on_device(b, par, n_sw, SEEDSW_MAXLEN, SEEDSW_MAXLEN)) return 1;
			if (fetch_counters(c)) return 1;
			c->st.ms_localsw += elapsed_at(c, "localsw", __LINE__); ++c->st.n_launch; c->st.sw_tasks += (u64)n_sw;
			if (c->h_cnt->flags & 32u) return set_err("seed filter: a local alignment exceeded the scratch capacity");
		}
		k.sw_res = (const bwag_swres_t *)b->d_swres.p;
		CK(cudaEventRecord(c->ev0, c->stream));
		BWAG_LAUNCH(k_chain_emit, (n + K3_THREADS - 1) / K3_THREADS, K3_THREADS, 0, c->stream, k);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		if (fetch_counters(c)) return 1;
		c->st.ms_chain += elapsed_at(c, "chain", __LINE__); ++c->st.n_launch;
	}

	/* extension over the chains that K3 left in HBM; K3 reported the longest reference window */
	const int cap_q = (b->max_len + 3) & ~3;
	const int cap_r = (c->h_cnt->max_rlen + 16 + 15) & ~15;
	CK(cudaMemsetAsync(&c->d_cnt->next_read, 0, sizeof(int), c->stream));
	int grid = c->grid_k4;
	{
		i64 need = ((i64)n + (K4_THREADS / 32) - 1) / (K4_THREADS / 32);
		if (grid > need) grid = (int)(need > 0 ? need : 1);
	}
	ExtArgs a;
	memset(&a, 0, sizeof(a));
	a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p; a.n_reads = n; a.par = *par;
	a.chain_beg = (const i64 *)b->d_chain_beg.p; a.chain_cnt = (const int *)b->d_chain_cnt.p; a.reg_base = (const i64 *)b->d_reg_base.p;
	a.chains = (const bwag_xchain_t *)b->d_chains.p; a.seeds = (const bwag_xseed_t *)b->d_seeds.p;
	a.regs = (bwag_xreg_t *)b->d_regs.p; a.n_regs = (int32_t *)b->d_nregs.p;
	a.cap_q = cap_q; a.cap_r = cap_r; a.min_seed = cp->min_seed_len;
	a.next_read = &c->d_cnt->next_read; a.cells = &c->d_cnt->ext_cells; a.flags = &c->d_cnt->flags;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (launch_extend(c, a, n, c->h_cnt->n_many)) return 1;
	CK(cudaEventRecord(c->ev1, c->stream));
	if (!out) {   /* the regions stay in HBM for bwag_tail_regs */
		if (fetch_counters(c)) return 1;
		c->st.ms_extend += elapsed_at(c, "extend", __LINE__); ++c->st.n_launch;
		if (c->h_cnt->flags & 2u) return set_err("extension: a read or reference window exceeded the scratch capacity");
		c->st.ext_cells += c->h_cnt->ext_cells;
		b->regs_on_device = 1;
		return 0;
	}
	/* dense copy of the regions (with contig id and repeat fraction of their chain) for the download */
	RegCompactArgs rc;
	rc.n_reads = n; rc.n_regs = (const int *)b->d_nregs.p; rc.regs = (const bwag_xreg_t *)b->d_regs.p; rc.reg_base = (const i64 *)b->d_reg_base.p;
	rc.chain_beg = (const i64 *)b->d_chain_beg.p; rc.chain_rid = (const int *)b->d_chain_rid.p; rc.chain_frac = (const float *)b->d_chain_frac.p;
	rc.out_beg = (i64 *)b->d_creg_beg.p; rc.total = &c->d_cnt->n_cig;
	/* the number of regions is not known before K4 ran: size the dense array by the number of seeds (upper bound) */
	if (buf_reserve(&b->d_cregs, sizeof(bwag_creg_t) * (size_t)(ns + 1))) return 1;
	rc.out = (bwag_creg_t *)b->d_cregs.p;
	BWAG_LAUNCH(k_regs_compact, (n + 127) / 128, 128, 0, c->stream, rc);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	c->st.ms_extend += elapsed_at(c, "extend", __LINE__); c->st.n_launch += 2;
	if (c->h_cnt->flags & 2u) return set_err("extension: a read or reference window exceeded the scratch capacity");
	c->st.ext_cells += c->h_cnt->ext_cells;
	const i64 n_regs = (i64)c->h_cnt->n_cig;
	if (hbuf_reserve(&b->h_cregs, sizeof(bwag_creg_t) * (size_t)(n_regs + 1)) || hbuf_reserve(&b->h_creg_beg, 8 * (size_t)(n + 1)) || hbuf_reserve(&b->h_nregs, 4 * (size_t)(n + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_regs) D2H(c, b->h_cregs.p, b->d_cregs.p, sizeof(bwag_creg_t) * (size_t)n_regs);
	D2H(c, b->h_creg_beg.p, b->d_creg_beg.p, 8 * (size_t)n);
	D2H(c, b->h_nregs.p, b->d_nregs.p, 4 * (size_t)n);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __LINE__);
	out->n_regs = (const int32_t *)b->h_nregs.p; out->reg_beg = (const int64_t *)b->h_creg_beg.p; out->regs = (const bwag_creg_t *)b->h_cregs.p;
	return 0;
}

extern "C" int bwag_fetch_cregs(bwag_batch_t *b, int n_sel, const int32_t *sel, bwag_cregs_t *out)
{
	bwag_ctx_t *c = &b->lc;
	CK(cudaSetDevice(c->device));
	if (!b->regs_on_device) return set_err("bwag_fetch_cregs needs a preceding bwag_chain_extend(..., NULL) on the same batch");
	out->n_regs = 0; out->reg_beg = 0; out->regs = 0;
	if (n_sel <= 0) return 0;
	const i64 ns = b->n_seeds;
	if (buf_reserve(&b->d_cregs, sizeof(bwag_creg_t) * (size_t)(ns + 1)) || buf_reserve(&b->d_creg_beg, 8 * (size_t)(b->n + 1)) || buf_reserve(&b->d_sel, 8 * (size_t)(n_sel + 1))) return 1;
	if (reset_counters(c)) return 1;
	H2D(c, b->d_sel.p, sel, 4 * (size_t)n_sel);
	RegCompactArgs rc;
	rc.n_reads = b->n; rc.n_regs = (const int *)b->d_nregs.p; rc.regs = (const bwag_xreg_t *)b->d_regs.p; rc.reg_base = (const i64 *)b->d_reg_base.p;
	rc.chain_beg = (const i64 *)b->d_chain_beg.p; rc.chain_rid = (const int *)b->d_chain_rid.p; rc.chain_frac = (const float *)b->d_chain_frac.p;
	rc.out_beg = (i64 *)b->d_creg_beg.p; rc.total = &c->d_cnt->n_cig; rc.out = (bwag_creg_t *)b->d_cregs.p;
	int *d_out_n = (int *)b->d_sel.p + n_sel;
	BWAG_LAUNCH(k_regs_compact_sel, (n_sel + 127) / 128, 128, 0, c->stream, rc, (const int *)b->d_sel.p, n_sel, d_out_n);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	++c->st.n_launch;
	const i64 n_regs = (i64)c->h_cnt->n_cig;
	if (hbuf_reserve(&b->h_cregs, sizeof(bwag_creg_t) * (size_t)(n_regs + 1)) || hbuf_reserve(&b->h_creg_beg, 8 * (size_t)(n_sel + 1)) || hbuf_reserve(&b->h_nregs, 4 * (size_t)(n_sel + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_regs) D2H(c, b->h_cregs.p, b->d_cregs.p, sizeof(bwag_creg_t) * (size_t)n_regs);
	D2H(c, b->h_creg_beg.p, b->d_creg_beg.p, 8 * (size_t)n_sel);
	D2H(c, b->h_nregs.p, d_out_n, 4 * (size_t)n_sel);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __LINE__);
	out->n_regs = (const int32_t *)b->h_nregs.p; out->reg_beg = (const int64_t *)b->h_creg_beg.p; out->regs = (const bwag_creg_t *)b->h_cregs.p;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ stage 3 */

/* K5 over n_tasks requests that already sit in b->d_tasks; results stay in b->d_res / d_cig / d_md, their pool sizes in *nc, *nm */
static int run_global(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, int cap_q, int cap_r, i64 cap_z, i64 n_aln, i64 *nc_out, i64 *nm_out)
{
	bwag_ctx_t *c = &b->lc;
	cap_q = (cap_q + 3) & ~3; cap_r = (cap_r + 15) & ~15; cap_z = (cap_z + 15) & ~(i64)15;
	if (cap_q < 4) cap_q = 4;
	if (cap_r < 16) cap_r = 16;
	if (cap_z < 64) cap_z = 64;
	/* one task's CIGAR has at most lq+rlen ops, its MD at most 3 characters per reference base */
	const int cap_wcig = cap_q + cap_r + 4, cap_wmd = 3 * cap_r + cap_q + 16;
	int grid = c->grid_k5;
	/* H/E rows and the sequences in shared memory when a block's share fits (BWA_B200_K5_SM=0 keeps them in global memory) */
	const int k5_zsm = getenv("BWA_B200_K5_ZSM") ? atoi(getenv("BWA_B200_K5_ZSM")) & ~15 : 6144;   /* backtrack bytes per warp in shared memory */
	const int k5_per_warp = ((8 * (cap_q + 2) + cap_r + cap_q + 2 + 15) & ~15) + k5_zsm;
	const size_t k5_smem = (size_t)k5_per_warp * (K5_THREADS / 32);
	int k5_sm = k5_smem <= K4_SMEM_MAX && !(getenv("BWA_B200_K5_SM") && atoi(getenv("BWA_B200_K5_SM")) == 0);
	const int k5_fast = !c->baseline && !(getenv("BWA_B200_K5_FAST") && atoi(getenv("BWA_B200_K5_FAST")) == 0);   /* 0: the first formulation of the row sweep */
#ifndef BWAG_CUSIM
	if (k5_sm) { int nb = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k5_fast ? k_global_sm_fast : k_global_sm, K5_THREADS, k5_smem)); if (nb < 2) k5_sm = 0; else grid = c->n_sm * nb; }
#endif
	{
		i64 need = ((i64)n_tasks + (K5_THREADS / 32) - 1) / (K5_THREADS / 32);
		if (grid > need) grid = (int)(need > 0 ? need : 1);
		i64 max_warps = ((i64)8 << 30) / cap_z;    /* bound the per-warp backtrack scratch to ~8 GB */
		if (max_warps < K5_THREADS / 32) max_warps = K5_THREADS / 32;
		if ((i64)grid * (K5_THREADS / 32) > max_warps) grid = (int)(max_warps / (K5_THREADS / 32));
	}
	const size_t n_warps = (size_t)grid * (K5_THREADS / 32);
	if (buf_reserve(&c->s_eh, n_warps * 2 * (size_t)(cap_q + 2) * 4) || buf_reserve(&c->s_rseq, n_warps * (size_t)cap_r) ||
	    buf_reserve(&c->s_qseq, n_warps * (size_t)(cap_q + 2)) || buf_reserve(&c->s_z, n_warps * (size_t)cap_z) ||
	    buf_reserve(&c->s_wcig, n_warps * (size_t)cap_wcig * 4) || buf_reserve(&c->s_wmd, n_warps * (size_t)cap_wmd)) return 1;
	if (buf_reserve(&b->d_res, sizeof(bwag_gres_t) * (size_t)n_tasks)) return 1;
	/* K5L for batches of short reads (the requests it cannot take fall through to the warp kernel one by one).  Off by default: in
	 * its first form it takes 32 consecutive requests per warp, of which only the quarter that needs a DP is live, and it was slower
	 * than the warp kernel; it needs the requests compacted and bucketed by
	 * band first.  BWA_B200_K5_LANE=1 switches it on (exact: tests/test_tail.py runs both). */
	int k5_lane = !c->baseline && cap_q <= K5L_QWORDS * 4 && n_tasks >= 64 && getenv("BWA_B200_K5_LANE") && atoi(getenv("BWA_B200_K5_LANE")) != 0;
	const size_t k5l_smem = (size_t)K5L_RING * K5L_THREADS * 8 + (size_t)K5L_QWORDS * K5L_THREADS * 4;
	const i64 k5l_cap_z = (i64)(K5L_RING - 1) * (cap_r < 1024 ? cap_r : 1024);   /* cells per lane: the widest band it takes x the longest window */
	int k5l_grid = 0;
	if (k5_lane) {
#ifndef BWAG_CUSIM
		int nb = 0;
		CK(cudaFuncSetAttribute(k_global_lane, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k5l_smem));
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_global_lane, K5L_THREADS, k5l_smem));
		k5l_grid = c->n_sm * (nb > 0 ? nb : 1);
#else
		k5l_grid = 2;
#endif
		const i64 need = ((i64)n_tasks + K5L_THREADS - 1) / K5L_THREADS;
		if (k5l_grid > need) k5l_grid = (int)need;
		if (buf_reserve(&b->d_pre_n, 4 * (size_t)n_tasks) || buf_reserve(&b->d_pre_score, 4 * (size_t)n_tasks) || buf_reserve(&b->d_pre_cig, 4 * (size_t)K5L_MAXCIG * (size_t)n_tasks) ||
		    buf_reserve(&c->s_zl, (size_t)k5l_cap_z * (size_t)k5l_grid * K5L_THREADS)) return 1;
	}
	i64 cap_cig = n_aln * 6 + 1024, cap_md = n_aln * 24 + 4096;   /* typical short-read sizes; grown on demand */
	for (int attempt = 0;; ++attempt) {
		if (buf_reserve(&b->d_cig, 4 * (size_t)cap_cig) || buf_reserve(&b->d_md, (size_t)cap_md)) return 1;
		GlbArgs a;
		memset(&a, 0, sizeof(a));
		a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p; a.par = *par;
		a.tasks = (const bwag_gtask_t *)b->d_tasks.p; a.n_tasks = n_tasks;
		a.res = (bwag_gres_t *)b->d_res.p; a.cigar = (u32 *)b->d_cig.p; a.md = (char *)b->d_md.p;
		a.cap_cig = cap_cig; a.cap_md = cap_md; a.n_cig = &c->d_cnt->n_cig; a.n_md = &c->d_cnt->n_md;
		a.w_cig = (u32 *)c->s_wcig.p; a.w_md = (char *)c->s_wmd.p; a.cap_wcig = cap_wcig; a.cap_wmd = cap_wmd;
		a.eh = (int *)c->s_eh.p; a.rseq = (uint8_t *)c->s_rseq.p; a.qseq = (uint8_t *)c->s_qseq.p; a.z = (uint8_t *)c->s_z.p;
		a.cap_q = cap_q; a.cap_r = cap_r; a.cap_z = cap_z;
		a.next_task = &c->d_cnt->next_task; a.cells = &c->d_cnt->glb_cells; a.flags = &c->d_cnt->flags;
		if (reset_counters(c)) return 1;
		CK(cudaEventRecord(c->ev0, c->stream));
		if (k5_lane) {   /* DP + backtrack of the short-read CIGAR requests, one lane per request; the warp kernel then adds NM/MD and takes the rest */
			GlbLaneArgs la;
			memset(&la, 0, sizeof(la));
			la.codes = a.codes; la.off = a.off; la.par = *par; la.tasks = a.tasks; la.n_tasks = n_tasks;
			la.pre_n = (int *)b->d_pre_n.p; la.pre_score = (int *)b->d_pre_score.p; la.pre_cig = (u32 *)b->d_pre_cig.p;
			la.z = (uint8_t *)c->s_zl.p; la.cap_z = k5l_cap_z; la.next_task = &c->d_cnt->next_task; la.cells = &c->d_cnt->glb_cells; la.n_pre = &c->d_cnt->n_pre;
			BWAG_LAUNCH(k_global_lane, k5l_grid, K5L_THREADS, k5l_smem, c->stream, c->ix, la);
			CK(cudaGetLastError());
			CK(cudaMemsetAsync(&c->d_cnt->next_task, 0, sizeof(int), c->stream));
			a.pre_n = la.pre_n; a.pre_score = la.pre_score; a.pre_cig = la.pre_cig;
			++c->st.n_launch;
		}
		a.smem_per_warp = k5_sm ? k5_per_warp : 0; a.z_sm_bytes = k5_sm ? k5_zsm : 0;
		if (k5_sm && k5_fast) BWAG_LAUNCH(k_global_sm_fast, grid, K5_THREADS, k5_smem, c->stream, c->ix, a);
		else if (k5_sm) BWAG_LAUNCH(k_global_sm, grid, K5_THREADS, k5_smem, c->stream, c->ix, a);
		else if (k5_fast) BWAG_LAUNCH(k_global_fast, grid, K5_THREADS, 0, c->stream, c->ix, a);
		else BWAG_LAUNCH(k_global, grid, K5_THREADS, 0, c->stream, c->ix, a);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		if (fetch_counters(c)) return 1;
		c->st.ms_global += elapsed_at(c, "global", __LINE__); ++c->st.n_launch;
		if (k5_lane && getenv("BWA_B200_PROFILE")) fprintf(stderr, "[prof] global alignment: lane-per-request kernel made %u of %d CIGARs, grid %d x %d\n", c->h_cnt->n_pre, n_tasks, k5l_grid, K5L_THREADS);
		if (c->h_cnt->flags & 4u) return set_err("global alignment: a task exceeded the scratch capacity");
		if (!(c->h_cnt->flags & 16u)) break;
		if (attempt >= 3) return set_err("global alignment: output pools keep overflowing");
		cap_cig = (i64)c->h_cnt->n_cig + 1024; cap_md = (i64)c->h_cnt->n_md + 4096;
	}
	c->st.glb_cells += c->h_cnt->glb_cells;
	*nc_out = (i64)c->h_cnt->n_cig; *nm_out = (i64)c->h_cnt->n_md;
	return 0;
}

extern "C" int bwag_global(bwag_batch_t *b, const bwag_sw_par_t *par, int n_tasks, const bwag_gtask_t *tasks, bwag_galn_t *out)
{
	bwag_ctx_t *c = &b->lc;
	CK(cudaSetDevice(c->device));
	if (n_tasks <= 0) { out->res = 0; out->cigar = 0; out->md = 0; return 0; }
	i64 cap_z = 64, n_aln = 0, nc = 0, nm = 0;
	int cap_q = 4, cap_r = 16;
	for (int t = 0; t < n_tasks; ++t) {
		i64 lq = tasks[t].qe - tasks[t].qb, rl = tasks[t].re - tasks[t].rb;
		if (lq > cap_q) cap_q = (int)lq;
		if (rl > cap_r) cap_r = (int)rl;
		if (tasks[t].mode == BWAG_G_REG2ALN) { /* backtrack bytes of the widest band this task can reach */
			i64 d = rl > lq ? rl - lq : lq - rl, wmax = (i64)par->w << 2;
			if (d + 3 > wmax) wmax = d + 3;
			i64 ncol = lq < 2 * wmax + 1 ? lq : 2 * wmax + 1;
			if (ncol * rl > cap_z) cap_z = ncol * rl;
			++n_aln;
		}
	}
	if (buf_reserve(&b->d_tasks, sizeof(bwag_gtask_t) * (size_t)n_tasks)) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	H2D(c, b->d_tasks.p, tasks, sizeof(bwag_gtask_t) * (size_t)n_tasks);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_h2d += elapsed_at(c, "h2d", __LINE__);
	b->tail_ready = 0;   /* the request pool of a preceding bwag_tail_regs is gone */
	if (run_global(b, par, n_tasks, cap_q, cap_r, cap_z, n_aln, &nc, &nm)) return 1;
	if (hbuf_reserve(&b->h_res, sizeof(bwag_gres_t) * (size_t)n_tasks) || hbuf_reserve(&b->h_cig, 4 * (size_t)(nc + 1)) || hbuf_reserve(&b->h_md, (size_t)nm + 16)) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	D2H(c, b->h_res.p, b->d_res.p, sizeof(bwag_gres_t) * (size_t)n_tasks);
	if (nc) D2H(c, b->h_cig.p, b->d_cig.p, 4 * (size_t)nc);
	if (nm) D2H(c, b->h_md.p, b->d_md.p, (size_t)nm);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __LINE__);
	out->res = (const bwag_gres_t *)b->h_res.p; out->cigar = (const uint32_t *)b->h_cig.p; out->md = (const char *)b->h_md.p;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ stage 4 */

#define TAIL_LOGN 4096
extern "C" int bwag_ctx_set_contigs(bwag_ctx_t *c, int n_seqs, const int64_t *offset, const int32_t *len, const uint8_t *is_alt, const char *const *names)
{
	CK(cudaSetDevice(c->device));
	size_t l_names = 0;
	for (int i = 0; i < n_seqs; ++i) l_names += strlen(names[i]);
	/* one block: offsets | lengths | name offsets | ALT flags | names | log table (8-byte aligned first) */
	const size_t o_off = 0, o_log = o_off + 8 * (size_t)n_seqs, o_len = o_log + 8 * TAIL_LOGN, o_noff = o_len + 4 * (size_t)n_seqs, o_alt = o_noff + 4 * ((size_t)n_seqs + 1), o_names = o_alt + (size_t)n_seqs, total = o_names + l_names + 16;
	char *h = (char *)malloc(total);
	if (!h) return set_err("out of memory");
	memset(h, 0, total);
	memcpy(h + o_off, offset, 8 * (size_t)n_seqs);
	memcpy(h + o_len, len, 4 * (size_t)n_seqs);
	memcpy(h + o_alt, is_alt, (size_t)n_seqs);
	{
		int *no = (int *)(h + o_noff), at = 0;
		for (int i = 0; i < n_seqs; ++i) { const size_t l = strlen(names[i]); no[i] = at; memcpy(h + o_names + at, names[i], l); at += (int)l; }
		no[n_seqs] = at;
		double *lt = (double *)(h + o_log);
		for (int i = 0; i < TAIL_LOGN; ++i) lt[i] = log((double)i);   /* the host's libm: log(0) = -inf included */
	}
	pthread_mutex_lock(&c->mu);
	if (c->d_tail) { cudaStreamSynchronize(c->stream); cudaFree(c->d_tail); c->d_tail = 0; c->have_ctg = 0; }
	cudaError_t e = cudaMalloc(&c->d_tail, total);
	if (e == cudaSuccess) e = cudaMemcpy(c->d_tail, h, total, cudaMemcpyHostToDevice);
	free(h);
	if (e != cudaSuccess) { pthread_mutex_unlock(&c->mu); return set_err("contig table upload failed: %s", cudaGetErrorString(e)); }
	char *d = (char *)c->d_tail;
	c->tctg.l_pac = c->ix.l_pac; c->tctg.n_seqs = n_seqs;
	c->tctg.off = (const i64 *)(d + o_off); c->tctg.len = (const int *)(d + o_len); c->tctg.alt = (const uint8_t *)(d + o_alt);
	c->tctg.names = d + o_names; c->tctg.name_off = (const int *)(d + o_noff);
	c->d_logtab = (const double *)(d + o_log);
	c->have_ctg = 1;
	pthread_mutex_unlock(&c->mu);
	return 0;
}

extern "C" int bwag_tail_regs(bwag_batch_t *b, const mem_opt_t *opt, const bwag_sw_par_t *sp, const uint64_t **pe_is, const uint8_t **cflag)
{
	bwag_ctx_t *c = &b->lc, *pc = b->ctx;
	CK(cudaSetDevice(c->device));
	if (!pc->have_ctg) return BWAG_UNSUPPORTED;
	if (c->baseline) return BWAG_DECLINED;   /* the baseline of the start-up self-check is the host-side post-processing */
	if (!b->regs_on_device) return set_err("bwag_tail_regs needs a preceding bwag_chain_extend(..., NULL) on the same batch");
	const int n = b->n, pe = !!(opt->flag & MEM_F_PE);
	if (pe && (n & 1)) return set_err("paired-end batch with an odd number of reads");
	const i64 cap = b->n_seeds + 1;   /* regions <= seeds */
	if (buf_reserve(&b->d_dregs, sizeof(mem_alnreg_t) * (size_t)cap) || buf_reserve(&b->d_tasks, sizeof(bwag_gtask_t) * (size_t)cap) ||
	    buf_reserve(&b->d_dreg_beg, 8 * (size_t)(n + 1)) || buf_reserve(&b->d_dreg_n, 4 * (size_t)(n + 1)) || buf_reserve(&b->d_task_beg, 8 * (size_t)(n + 1)) ||
	    buf_reserve(&b->d_cflag, (size_t)n + 16) || buf_reserve(&b->d_pe_is, 8 * (size_t)(n / 2 + 1))) return 1;
	TailRegsArgs a;
	memset(&a, 0, sizeof(a));
	a.n_reads = n; a.pe = pe; a.opt = *opt; a.ctg = pc->tctg;
	a.n_raw = (const int *)b->d_nregs.p; a.xregs = (const bwag_xreg_t *)b->d_regs.p; a.reg_base = (const i64 *)b->d_reg_base.p; a.chain_beg = (const i64 *)b->d_chain_beg.p;
	a.chain_rid = (const int *)b->d_chain_rid.p; a.chain_frac = (const float *)b->d_chain_frac.p;
	a.dregs = (mem_alnreg_t *)b->d_dregs.p; a.dreg_beg = (i64 *)b->d_dreg_beg.p; a.dreg_n = (int *)b->d_dreg_n.p; a.task_beg = (i64 *)b->d_task_beg.p; a.cflag = (uint8_t *)b->d_cflag.p;
	a.cap_dregs = cap; a.tasks = (bwag_gtask_t *)b->d_tasks.p; a.cap_tasks = cap; a.pe_is = (u64 *)b->d_pe_is.p;
	a.n_dregs = &c->d_cnt->t_dregs; a.n_tasks = &c->d_cnt->t_tasks; a.max_z = &c->d_cnt->t_max_z; a.max_lq = &c->d_cnt->t_max_lq; a.max_rl = &c->d_cnt->t_max_rl;
	if (reset_counters(c)) return 1;
	const int n_units = pe ? n >> 1 : n;
	CK(cudaEventRecord(c->ev0, c->stream));
	BWAG_LAUNCH(k_tail_regs, (n_units + 127) / 128, 128, 0, c->stream, a);
	CK(cudaGetLastError());
	CK(cudaEventRecord(c->ev1, c->stream));
	if (fetch_counters(c)) return 1;
	c->st.ms_tail += elapsed_at(c, "tail", __LINE__); ++c->st.n_launch;
	const i64 n_tasks = (i64)c->h_cnt->t_tasks;
	if (n_tasks > cap || (i64)c->h_cnt->t_dregs > cap) return set_err("stage 4: more regions than seeds?");
	if (n_tasks >= ((i64)1 << 31)) return set_err("stage 4: too many alignment requests in one batch; use smaller chunks");
	const int cap_q = c->h_cnt->t_max_lq, cap_r = c->h_cnt->t_max_rl;
	const i64 cap_z = (i64)c->h_cnt->t_max_z;
	if (n_tasks > 0) {
		i64 nc = 0, nm = 0;
		if (run_global(b, sp, (int)n_tasks, cap_q, cap_r, cap_z, n_tasks, &nc, &nm)) return 1;
	}
	if (hbuf_reserve(&b->h_cflag, (size_t)n + 16) || hbuf_reserve(&b->h_pe_is, 8 * (size_t)(n / 2 + 1))) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	D2H(c, b->h_cflag.p, b->d_cflag.p, (size_t)n);
	if (pe) D2H(c, b->h_pe_is.p, b->d_pe_is.p, 8 * (size_t)(n / 2));
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __LINE__);
	b->tail_ready = 1;
	if (pe_is) *pe_is = pe ? (const uint64_t *)b->h_pe_is.p : 0;
	if (cflag) *cflag = (const uint8_t *)b->h_cflag.p;
	return 0;
}

extern "C" int bwag_tail_sam(bwag_batch_t *b, const mem_opt_t *opt, const mem_pestat_t pes[4], const double *const pair_tab[4], const double *log_tab,
                             int64_t n_processed, const char *rg_id, bwag_sam_t *out)
{
	bwag_ctx_t *c = &b->lc, *pc = b->ctx;
	(void)log_tab;   /* the context keeps its own copy (bwag_ctx_set_contigs computes it with the same libm) */
	CK(cudaSetDevice(c->device));
	if (!pc->have_ctg) return BWAG_UNSUPPORTED;
	if (!b->tail_ready) return set_err("bwag_tail_sam needs a preceding bwag_tail_regs on the same batch");
	const int n = b->n, pe = !!(opt->flag & MEM_F_PE);
	TailSamArgs g;
	memset(&g, 0, sizeof(g));
	g.n_reads = n; g.pe = pe; g.opt = *opt; g.ctg = pc->tctg; g.logtab = pc->d_logtab; g.n_processed = n_processed;
	size_t tab_bytes = 256;   /* read-group id first */
	if (pe) {
		memcpy(g.pes, pes, 4 * sizeof(mem_pestat_t));
		for (int d = 0; d < 4; ++d) if (pair_tab && pair_tab[d] && !pes[d].failed && pes[d].high >= pes[d].low) tab_bytes += 8 * ((size_t)pes[d].high - pes[d].low + 1);
	}
	if (buf_reserve(&b->d_ptab, tab_bytes) || hbuf_reserve(&b->h_ptab, tab_bytes)) return 1;
	{
		char *h = (char *)b->h_ptab.p;
		size_t at = 256;
		const size_t l_rg = rg_id ? strlen(rg_id) : 0;
		memset(h, 0, 256);
		if (l_rg > 255) return set_err("read-group id too long");
		if (l_rg) memcpy(h, rg_id, l_rg);
		g.rg = (const char *)b->d_ptab.p; g.l_rg = (int)l_rg;
		if (pe) for (int d = 0; d < 4; ++d) if (pair_tab && pair_tab[d] && !pes[d].failed && pes[d].high >= pes[d].low) {
			const size_t bytes = 8 * ((size_t)pes[d].high - pes[d].low + 1);
			memcpy(h + at, pair_tab[d], bytes);
			g.ptab[d] = (const double *)((char *)b->d_ptab.p + at);
			at += bytes;
		}
		H2D(c, b->d_ptab.p, h, tab_bytes);
	}
	g.codes = (const uint8_t *)b->d_codes.p; g.off = (const i64 *)b->d_off.p;
	g.dregs = (const mem_alnreg_t *)b->d_dregs.p; g.dreg_beg = (const i64 *)b->d_dreg_beg.p; g.dreg_n = (const int *)b->d_dreg_n.p; g.task_beg = (const i64 *)b->d_task_beg.p; g.cflag = (const uint8_t *)b->d_cflag.p;
	g.res = (const bwag_gres_t *)b->d_res.p; g.cigar = (const u32 *)b->d_cig.p; g.md = (const char *)b->d_md.p;
	if (buf_reserve(&b->d_rec, sizeof(bwag_samrec_t) * (size_t)(n + 1))) return 1;
	g.rec = (bwag_samrec_t *)b->d_rec.p;
	g.n_text = &c->d_cnt->t_text; g.n_complex = &c->d_cnt->t_complex;
	i64 cap_text = b->total_bases + 176 * (i64)n + 4096;
	const int n_units = pe ? n >> 1 : n;
	for (int attempt = 0;; ++attempt) {
		if (buf_reserve(&b->d_text, (size_t)cap_text)) return 1;
		g.text = (char *)b->d_text.p; g.cap_text = cap_text;
		if (reset_counters(c)) return 1;
		CK(cudaEventRecord(c->ev0, c->stream));
		BWAG_LAUNCH(k_tail_sam, (n_units + 127) / 128, 128, 0, c->stream, g);
		CK(cudaGetLastError());
		CK(cudaEventRecord(c->ev1, c->stream));
		if (fetch_counters(c)) return 1;
		c->st.ms_tail += elapsed_at(c, "tail", __LINE__); ++c->st.n_launch;
		if ((i64)c->h_cnt->t_text <= cap_text) break;
		if (attempt >= 2) return set_err("stage 4: the text pool keeps overflowing");
		cap_text = (i64)c->h_cnt->t_text + 4096;
	}
	const i64 n_text = (i64)c->h_cnt->t_text;
	if (hbuf_reserve(&b->h_rec, sizeof(bwag_samrec_t) * (size_t)(n + 1)) || hbuf_reserve(&b->h_text, (size_t)n_text + 16)) return 1;
	CK(cudaEventRecord(c->ev0, c->stream));
	D2H(c, b->h_rec.p, b->d_rec.p, sizeof(bwag_samrec_t) * (size_t)n);
	if (n_text) D2H(c, b->h_text.p, b->d_text.p, (size_t)n_text);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __LINE__);
	c->st.tail_reads += (u64)n; c->st.tail_complex += c->h_cnt->t_complex;
	out->rec = (const bwag_samrec_t *)b->h_rec.p; out->text = (const char *)b->h_text.p; out->n_text = n_text; out->n_complex = (int64_t)c->h_cnt->t_complex;
	return 0;
}

/* ------------------------------------------------------------------------------------------------ K6 */


