/* bwag_api.cu -- host side of the device-batch C ABI (include/bwa_b200_dev.h): errors, the context and its index residency
 * in HBM, batch upload and lifetime, the work/time counters the roofline is computed from, and the helpers the drivers of
 * the stages share (bwag_drv.h).  The drivers themselves sit beside their kernels.
 *
 * HBM layout of the index blob (all offsets 256-byte aligned):
 *   [ header | Occ/BWT blocks (bwt_size*4 B, re-packed: 32 B per 64 symbols) | sampled SA (n_sa*8 B) | pac (l_pac/4+1 B) ]
 * The blob is position independent (the header holds sizes, not pointers) so that it can be filled
 * on one GPU and broadcast to the others with a single collective.
 */
#include <stdarg.h>
#include <time.h>
#include <sched.h>
#include "bwag_drv.h"

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
int set_err(const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof(g_err), fmt, ap);
	va_end(ap);
	return 1;
}

int buf_reserve(DevBuf *b, size_t bytes)
{
	if (bytes <= b->cap) return 0;
	if (b->p) cudaFree(b->p);
	b->p = 0; b->cap = 0;
	size_t want = bytes + bytes / 4 + 256;
	CK(cudaMalloc(&b->p, want));
	b->cap = want;
	return 0;
}
int hbuf_reserve(HostBuf *b, size_t bytes)
{
	if (bytes <= b->cap) return 0;
	if (b->p) cudaFreeHost(b->p);
	b->p = 0; b->cap = 0;
	size_t want = bytes + bytes / 4 + 256;
	CK(cudaMallocHost(&b->p, want));
	b->cap = want;
	return 0;
}

#ifndef BWAG_L2_FETCH_DEFAULT
#define BWAG_L2_FETCH_DEFAULT 0   /* 0: leave the device's setting */
#endif
#ifdef BWAG_CUSIM
#define BWAG_KTAB_MAX_AUTO 5     /* the emulator builds the table one fiber per entry: keep it small */
#else
#define BWAG_KTAB_MAX_AUTO 14
#endif

#ifdef BWAG_CUSIM
unsigned long long bwag_cusim_sector_loads, bwag_cusim_list_acc[5];
long bwag_cusim_dev_blocks;
extern "C" long bwag_cusim_live_dev_blocks(void) { return __atomic_load_n(&bwag_cusim_dev_blocks, __ATOMIC_RELAXED); }
#endif

/* ------------------------------------------------------------------------------------------------ index */

extern "C" size_t bwag_blob_bytes(const bwt_t *bwt, int64_t l_pac)
{
	return ALIGN256(sizeof(BlobHeader)) + ALIGN256((size_t)bwt->bwt_size * 4 + 64) + ALIGN256((size_t)bwt->n_sa * 8 + 32) + ALIGN256((size_t)l_pac / 4 + 1 + 64);
}

/* The Occ/BWT words of an updated .bwt uploaded to d (at least bwt_size * 4 + 64 bytes) and re-packed there, in place, into
 * 32-byte blocks of 64 symbols (bwag_dev.cuh); sb[s]: the counts before superblock s.  The blob holds this beside the SA and
 * the pac; `bwa-b200 bwt2sa` needs it alone. */
int occ_upload(void *d, const bwt_t *bwt, u64 sb[BWAG_MAX_SB][4])
{
	if (bwt->seq_len >= (u64)BWAG_MAX_SB << BWAG_SB_SHIFT) return set_err("index too large: %llu BWT symbols", (unsigned long long)bwt->seq_len);
	memset(sb, 0, sizeof(u64) * BWAG_MAX_SB * 4);
	for (u64 s = 0; s << BWAG_SB_SHIFT < bwt->seq_len; ++s) {   /* counts before symbol s*2^31 = the count words of that file block */
		const u64 *cnt = (const u64 *)(bwt->bwt + ((s << BWAG_SB_SHIFT) >> 7) * 16);
		for (int k = 0; k < 4; ++k) sb[s][k] = cnt[k];
	}
	CK(cudaMemset(d, 0, ALIGN256((size_t)bwt->bwt_size * 4 + 64)));
	CK(cudaMemcpy(d, bwt->bwt, (size_t)bwt->bwt_size * 4, cudaMemcpyHostToDevice));
	{   /* file layout -> 32-byte blocks, in place (bwag_dev.cuh) */
		const u64 n_blocks = ((u64)bwt->bwt_size * 4 + 63) / 64;
		DevIndex tmp;
		memset(&tmp, 0, sizeof(tmp));
		for (int s = 0; s < BWAG_MAX_SB; ++s)
			for (int k = 0; k < 4; ++k) tmp.sb[s][k] = sb[s][k];
		BWAG_LAUNCH(k_occ_pack, (int)((n_blocks + 255) / 256 < 65535 ? (n_blocks + 255) / 256 : 65535), 256, 0, 0, tmp, (uint4 *)d, n_blocks);
		CK(cudaGetLastError());
		CK(cudaDeviceSynchronize());
	}
	return 0;
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
	h.off_bwt = ALIGN256(sizeof(BlobHeader));
	h.off_sa = h.off_bwt + ALIGN256((size_t)bwt->bwt_size * 4 + 64);
	h.off_pac = h.off_sa + ALIGN256((size_t)bwt->n_sa * 8 + 32);
	h.total = h.off_pac + ALIGN256((size_t)l_pac / 4 + 1 + 64);
	char *d = (char *)d_blob;
	if (occ_upload(d + h.off_bwt, bwt, h.sb)) return 1;
	CK(cudaMemcpy(d, &h, sizeof(h), cudaMemcpyHostToDevice));
	CK(cudaMemcpy(d + h.off_sa, bwt->sa, (size_t)bwt->n_sa * 8, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(d + h.off_pac, pac, (size_t)l_pac / 4 + 1, cudaMemcpyHostToDevice));
	return 0;
}

static int pick_grid(bwag_ctx_t *c)
{
#ifdef BWAG_CUSIM
	c->n_sm = 2;
	c->grid_k1f = c->grid_k2 = c->grid_k4 = c->grid_k5 = 2;
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
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_smem_fwd, K1F_THREADS, 0)); c->grid_k1f = c->n_sm * (nb > 0 ? nb : 1);
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_sa, K2_THREADS, 0)); c->grid_k2 = c->n_sm * (nb > 0 ? nb : 1);
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_extend, K4_THREADS, 0)); c->grid_k4 = c->n_sm * (nb > 0 ? nb : 1);
	CK(cudaFuncSetAttribute(k_extend_sm, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_extend_sm_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_extend_lane, cudaFuncAttributeMaxDynamicSharedMemorySize, K4L_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_global_sm, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_global_sm_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, K4_SMEM_MAX));
	CK(cudaFuncSetAttribute(k_tail_sam, cudaFuncAttributeMaxDynamicSharedMemorySize, TAIL_SAM_SMEM_MAX));   /* one limit for every batch: lanes launch it concurrently */
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_global, K5_THREADS, 0)); c->grid_k5 = c->n_sm * (nb > 0 ? nb : 1);
#endif
	return 0;
}

static cudaEvent_t g_trace_ref;   /* BWA_B200_GPUTRACE: origin of the device-clock timeline (see elapsed_at) */
static int g_gputrace = -1;

/* the first lane made (the first context's) starts the device-clock timeline of BWA_B200_GPUTRACE */
int lane_init(Lane *l)
{
	CK(cudaStreamCreate(&l->stream));
	CK(cudaEventCreate(&l->ev0)); CK(cudaEventCreate(&l->ev1));
	if (g_gputrace < 0) {
		const char *e = getenv("BWA_B200_GPUTRACE");
		g_gputrace = e && atoi(e) > 0;
		if (g_gputrace) { CK(cudaEventCreate(&g_trace_ref)); CK(cudaEventRecord(g_trace_ref, l->stream)); CK(cudaEventSynchronize(g_trace_ref)); }
	}
	CK(cudaEventCreateWithFlags(&l->ev_wait, cudaEventBlockingSync | cudaEventDisableTiming));
	CK(cudaMalloc((void **)&l->d_cnt, sizeof(Counters)));
	CK(cudaMallocHost((void **)&l->h_cnt, sizeof(Counters)));
	return 0;
}

/* the owner has made the device current and synchronised the stream; the scratch frees itself */
Lane::~Lane()
{
	if (d_cnt) cudaFree(d_cnt);
	if (h_cnt) cudaFreeHost(h_cnt);
	if (ev0) cudaEventDestroy(ev0);
	if (ev1) cudaEventDestroy(ev1);
	if (ev_wait) cudaEventDestroy(ev_wait);
	if (stream) cudaStreamDestroy(stream);
}

/* what every context owns besides its index: its lane and the launch grids */
static int ctx_init(bwag_ctx_t *c)
{
	if (lane_init(&c->lane)) return 1;
	pthread_mutex_init(&c->mu, 0);
	return pick_grid(c);
}

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
	bwag_ctx_t *c = new bwag_ctx();
	c->device = device; c->own_blob = own_blob; c->blob = d_blob;
	if (ctx_init(c)) { delete c; return 0; }
	char *d = (char *)d_blob;
	c->lane.ix.bwt = (const uint4 *)(d + h.off_bwt);
	c->lane.ix.sa = (const u64 *)(d + h.off_sa);
	c->lane.ix.pac = (const uint8_t *)(d + h.off_pac);
	c->lane.ix.primary = h.primary; c->lane.ix.seq_len = h.seq_len; c->lane.ix.n_sa = h.n_sa; c->lane.ix.l_pac = (i64)h.l_pac; c->lane.ix.sa_shift = (int)h.sa_shift;
	for (int i = 0; i < 5; ++i) c->lane.ix.L2[i] = h.L2[i];
	for (int s = 0; s < BWAG_MAX_SB; ++s)
		for (int k = 0; k < 4; ++k) { c->lane.ix.sb[s][k] = h.sb[s][k]; c->lane.ix.sbgt[s][k] = 0; for (int t = k + 1; t < 4; ++t) c->lane.ix.sbgt[s][k] += h.sb[s][t]; }
	return c;
}

/* a context without an index (pemerge): the index view stays zeroed, which K6 reads only for targets on the reference */
extern "C" bwag_ctx_t *bwag_ctx_create_bare(int device)
{
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_err("no CUDA device is visible: this library has no CPU path"); return 0; }
	if (device < 0) CKP(cudaGetDevice(&device));
	CKP(cudaSetDevice(device));
	bwag_ctx_t *c = new bwag_ctx();
	c->device = device;
	if (ctx_init(c)) { delete c; return 0; }
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
	CK(cudaStreamSynchronize(c->lane.stream));
	CK(cudaMemcpy(&h, c->blob, sizeof(h), cudaMemcpyDeviceToHost));
	memset(&f, 0, sizeof(f));
	memcpy(f.magic, SHARE_MAGIC, 8);
	f.version = 2; f.device = c->device; f.pid = (int32_t)getpid(); f.l_pac = h.l_pac; f.blob_bytes = h.total;
	f.dense_shift = c->dense_sa ? c->lane.ix.sa_shift : -1; f.dense_n = c->dense_sa ? c->lane.ix.n_sa : 0; f.dense_bytes = c->dense_sa ? c->lane.ix.n_sa * 8 + 32 : 0;
	f.ktab_k = c->ktab ? c->lane.ix.ktab_k : 0; f.ktab_bytes = c->ktab ? (((((u64)1 << (2 * (c->lane.ix.ktab_k + 1))) - 4) / 3) + 2) * 16 : 0;
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
	if (p[1]) { c->dense_sa = (u64 *)p[1]; c->lane.ix.sa = c->dense_sa; c->lane.ix.sa_shift = f.dense_shift; c->lane.ix.n_sa = f.dense_n; }
	if (p[2]) { c->ktab = (ulonglong2 *)p[2]; c->lane.ix.ktab = c->ktab; c->lane.ix.ktab_k = f.ktab_k; }
	return c;
}

extern "C" void bwag_ctx_destroy(bwag_ctx_t *c)
{
	if (!c) return;
	cudaSetDevice(c->device);
	cudaStreamSynchronize(c->lane.stream);
	for (int i = 0; i < N_SPARE; ++i) delete c->spare[i];
	if (c->imported) shared_close(c);
	else {
		if (c->dense_sa) cudaFree(c->dense_sa);
		if (c->ktab) cudaFree(c->ktab);
		if (c->own_blob && c->blob) cudaFree(c->blob);
	}
	delete c;
}

extern "C" int bwag_ctx_densify_sa(bwag_ctx_t *c, int intv)
{
	if (intv == 0) {   /* the densest interval >= 2 whose sample takes at most an eighth of the device's memory; the rest holds the
	                    * index, the short-string table and the batches of the calls in flight (3 Gbp on an 80 GB H100: every 8th row, 6 GB) */
		size_t free_b = 0, total_b = 0;
		CK(cudaSetDevice(c->device));
		CK(cudaMemGetInfo(&free_b, &total_b));
		intv = 2;
		while (intv < 32 && (double)(c->lane.ix.seq_len / (u64)intv + 1) * 8 > (double)total_b / 8) intv <<= 1;
		if (intv < 8 && bwag_ctx_densify_sa(c, 8)) return 1;   /* in two stages (32 -> 8 -> intv): each walks only a few LF steps per row */
	}
	int s = 0;
	while ((1 << s) < intv) ++s;
	if ((1 << s) != intv || s > c->lane.ix.sa_shift) return set_err("dense suffix-array interval must be a power of two not above the current %d", 1 << c->lane.ix.sa_shift);
	if (s == c->lane.ix.sa_shift || c->imported) return 0;   /* an imported context keeps the sample of the process that owns the memory */
	CK(cudaSetDevice(c->device));
	u64 n_out = (c->lane.ix.seq_len + (u64)intv) / (u64)intv, *out = 0;
	{   /* leave room for the batch buffers */
		size_t free_b = 0, total_b = 0;
		CK(cudaMemGetInfo(&free_b, &total_b));
		if ((double)n_out * 8 > 0.5 * (double)free_b) return set_err("not enough free device memory for a suffix-array sample of interval %d", intv);
	}
	CK(cudaMalloc((void **)&out, n_out * 8 + 32));   /* K2 reads the sample in aligned groups of four rows */
	BWAG_LAUNCH(k_sa_densify, c->n_sm * 8, 256, 0, c->lane.stream, c->lane.ix, out, s, n_out);
	CK(cudaGetLastError());
	CK(cudaStreamSynchronize(c->lane.stream));
	if (c->dense_sa) cudaFree(c->dense_sa);
	c->dense_sa = out;
	c->lane.ix.sa = out; c->lane.ix.sa_shift = s; c->lane.ix.n_sa = n_out;
	++c->lane.st.n_launch;
	return 0;
}

/* bi-intervals of all strings of 1..K bases (bwag_smem.cu); K = 0 picks a depth from the index size, K < 0 removes the table */
extern "C" int bwag_ctx_build_ktab(bwag_ctx_t *c, int K)
{
	CK(cudaSetDevice(c->device));
	if (c->imported) return 0;   /* the table, or its absence, is the owner's */
	if (K == 0) {   /* as deep as strings still have a few dozen occurrences (their intervals span two Occ blocks): 14 at 3 Gbp = 5.7 GB */
		int lg = 0;
		while (lg < 31 && ((u64)1 << (2 * (lg + 1))) <= c->lane.ix.seq_len) ++lg;   /* floor(log4(seq_len)) */
		K = lg - 2;
		if (K > BWAG_KTAB_MAX_AUTO) K = BWAG_KTAB_MAX_AUTO;
	}
	if (K > 14) K = 14;
	if (K < 2) {
		CK(cudaStreamSynchronize(c->lane.stream));
		if (c->ktab) { cudaFree(c->ktab); c->ktab = 0; }
		c->lane.ix.ktab = 0; c->lane.ix.ktab_k = 0;
		return 0;
	}
	if (c->ktab && c->lane.ix.ktab_k == K) return 0;
	const u64 total = (((u64)1 << (2 * (K + 1))) - 4) / 3;
	ulonglong2 *tab = 0;
	{
		size_t free_b = 0, total_b = 0;
		CK(cudaMemGetInfo(&free_b, &total_b));
		if ((double)total * 16 > 0.25 * (double)free_b) return set_err("not enough free device memory for a short-string table of depth %d", K);
	}
	CK(cudaMalloc((void **)&tab, (total + 2) * 16));
	CK(cudaMemsetAsync(tab, 0, (total + 2) * 16, c->lane.stream));
	DevIndex plain = c->lane.ix;
	plain.ktab = 0; plain.ktab_k = 0;
	{
		u64 nb = (total + 255) / 256;
		BWAG_LAUNCH(k_ktab_build, (int)(nb < (u64)c->n_sm * 32 ? nb : (u64)c->n_sm * 32), 256, 0, c->lane.stream, plain, tab, K);
	}
	CK(cudaGetLastError());
	CK(cudaStreamSynchronize(c->lane.stream));
	if (c->ktab) cudaFree(c->ktab);
	c->ktab = tab;
	c->lane.ix.ktab = tab; c->lane.ix.ktab_k = K;
#ifdef BWAG_CUSIM
	bwag_cusim_sector_loads = 0;   /* the emulator's request counter reports the alignment work only */
#endif
	++c->lane.st.n_launch;
	return 0;
}

/* Check the resident index against the resident text on rows first, first + stride, ... (stride 1 = every row, a complete check;
 * see k_index_verify).  out: rows checked, BWT/text/SA mismatches, order violations, pairs of suffixes equal over 8192 bases. */
extern "C" int bwag_ctx_verify(bwag_ctx_t *c, uint64_t first, uint64_t stride, uint64_t out[4])
{
	CK(cudaSetDevice(c->device));
	if (stride == 0) stride = 1;
	const u64 n_check = first > c->lane.ix.seq_len ? 0 : (c->lane.ix.seq_len - first) / stride + 1;
	u64 *d = 0;
	CK(cudaMalloc((void **)&d, 4 * sizeof(u64)));
	CK(cudaMemsetAsync(d, 0, 4 * sizeof(u64), c->lane.stream));
	if (n_check) {
		const u64 nb = (n_check + 255) / 256;
		BWAG_LAUNCH(k_index_verify, (int)(nb < (u64)c->n_sm * 64 ? nb : (u64)c->n_sm * 64), 256, 0, c->lane.stream, c->lane.ix, (u64)first, (u64)stride, n_check, d);
		CK(cudaGetLastError());
	}
	CK(cudaMemcpyAsync(out, d, 4 * sizeof(u64), cudaMemcpyDeviceToHost, c->lane.stream));
	CK(cudaStreamSynchronize(c->lane.stream));
	cudaFree(d);
	++c->lane.st.n_launch;
	return 0;
}

/* on = 1: batches begun from now on use the first formulation of the K4/K5 row sweeps and no short-string table (the
 * configuration measured in round 1); on = 0: back to the defaults.  Used by the host's start-up self-check. */
extern "C" void bwag_ctx_baseline(bwag_ctx_t *c, int on) { pthread_mutex_lock(&c->mu); c->lane.baseline = on != 0; pthread_mutex_unlock(&c->mu); }
extern "C" int bwag_is_emulator(void)
{
#ifdef BWAG_CUSIM
	return 1;
#else
	return 0;
#endif
}

extern "C" void bwag_stats_get(bwag_ctx_t *c, bwag_stats_t *s) { pthread_mutex_lock(&c->mu); *s = c->lane.st; pthread_mutex_unlock(&c->mu); }
extern "C" void bwag_stats_reset(bwag_ctx_t *c) { pthread_mutex_lock(&c->mu); memset(&c->lane.st, 0, sizeof(c->lane.st)); pthread_mutex_unlock(&c->mu); }


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
	CKP(cudaSetDevice(c->device));
	bwag_batch_t *b = 0;   /* buffers only grow: cudaMalloc/cudaMallocHost per batch would cost more than the kernels */
	pthread_mutex_lock(&c->mu);
	for (int i = 0; i < N_SPARE; ++i) if (c->spare[i]) { b = c->spare[i]; c->spare[i] = 0; break; }
	pthread_mutex_unlock(&c->mu);
	if (!b) {
		b = new bwag_batch();
		if (lane_init(&b->lane)) { delete b; return 0; }
	}
	Lane *l = &b->lane;
	l->ix = c->lane.ix;
	l->baseline = c->lane.baseline;
	if (l->baseline) { l->ix.ktab = 0; l->ix.ktab_k = 0; }
	memset(&l->st, 0, sizeof(l->st));
	b->max_len = 0; b->seeded = 0; b->tail_ready = 0; b->regs_on_device = 0;
	b->ctx = c; b->n = n; b->h_off = (const i64 *)off; b->total_bases = off[n];
	for (int i = 0; i < n; ++i) { int len = (int)(off[i + 1] - off[i]); if (len > b->max_len) b->max_len = len; }
	if (buf_reserve(&b->d_codes, (size_t)b->total_bases + 16) || buf_reserve(&b->d_off, sizeof(i64) * ((size_t)n + 1))) { delete b; return 0; }
	CKP(cudaEventRecord(l->ev0, l->stream));
	CKP(cudaMemcpyAsync(b->d_codes.p, codes, (size_t)b->total_bases, cudaMemcpyHostToDevice, l->stream));
	CKP(cudaMemcpyAsync(b->d_off.p, off, sizeof(i64) * ((size_t)n + 1), cudaMemcpyHostToDevice, l->stream));
	l->st.h2d_bytes += (u64)b->total_bases + sizeof(i64) * ((u64)n + 1);
	CKP(cudaEventRecord(l->ev1, l->stream));
	CKP(cudaStreamSynchronize(l->stream));
	{ float ms = 0; cudaEventElapsedTime(&ms, l->ev0, l->ev1); l->st.ms_h2d += ms; }
	return b;
}

extern "C" void bwag_batch_end(bwag_batch_t *b)
{
	if (!b) return;
	bwag_ctx_t *c = b->ctx;
	const bwag_stats_t *x = &b->lane.st;
	cudaSetDevice(c->device);
	cudaStreamSynchronize(b->lane.stream);
	pthread_mutex_lock(&c->mu);
	{   /* fold this batch's counters into the context */
		bwag_stats_t *d = &c->lane.st;
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
		        (unsigned long long)x->occ_touches, (unsigned long long)x->sa_touches, (unsigned long long)x->ext_cells, (unsigned long long)x->glb_cells,
		        (unsigned long long)x->tail_reads, (unsigned long long)x->tail_complex, (unsigned long long)x->sw_tasks);
	for (int i = 0; i < N_SPARE; ++i) if (!c->spare[i]) { c->spare[i] = b; b = 0; break; }
	pthread_mutex_unlock(&c->mu);
	delete b;
}

int reset_counters(Lane *c)
{
	CK(cudaMemsetAsync(c->d_cnt, 0, sizeof(Counters), c->stream));
	return 0;
}
/* wait for the lane's stream.  Default: poll with short sleeps (a waiting lane costs no core; with the post-processing on the
 * device the host threads are few); BWA_B200_SYNC=spin: cudaStreamSynchronize, =yield / =block: see below */
cudaError_t stream_wait(Lane *c)
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

int fetch_counters(Lane *c)
{
	CK(cudaMemcpyAsync(c->h_cnt, c->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, c->stream));
	CK(stream_wait(c));
	return 0;
}
/* BWA_B200_GPUTRACE=1: every timed stage also prints its start and end on the device clock (ms since the first context was made),
 * one line per stage and lane, so that tools/gpu_timeline.py can tell how much of a run the GPU sat idle and between which stages */
double elapsed_at(Lane *c, const char *stage, const char *file, int line)
{
	float ms = 0;
	cudaEventElapsedTime(&ms, c->ev0, c->ev1);
	if (g_gputrace > 0) {
		float t0 = 0, t1 = 0;
		const char *f = strrchr(file, '/');
		cudaEventElapsedTime(&t0, g_trace_ref, c->ev0); cudaEventElapsedTime(&t1, g_trace_ref, c->ev1);
		fprintf(stderr, "[gputrace] %p %s:%s:%d %.3f %.3f\n", (void *)c, stage, f ? f + 1 : file, line, t0, t1);
	}
	return ms;
}

int fm_grid(const bwag_ctx_t *c, i64 n_items)
{
	const i64 g = (n_items + 127) / 128, cap = (i64)c->n_sm * 16;
	return (int)(g < 1 ? 1 : g < cap ? g : cap);
}

int buf_grow_keep(Lane *c, DevBuf *b, size_t keep, size_t bytes)
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

/* K2: the BWT rows rows[0..n) become suffix-array positions in place, between ev0 and ev1 */
int run_sa(bwag_batch_t *b, i64 *rows, i64 n)
{
	Lane *c = &b->lane;
	SaArgs s;
	s.rbeg = rows; s.n = n; s.next = &c->d_cnt->next_seed; s.sa_touches = &c->d_cnt->sa_touches;
	int grid = b->ctx->grid_k2;
	const i64 need = (n + K2_THREADS - 1) / K2_THREADS;
	if (grid > need) grid = (int)need;
	CK(cudaEventRecord(c->ev0, c->stream));
	BWAG_LAUNCH(k_sa, grid, K2_THREADS, 0, c->stream, c->ix, s);
	CK(cudaGetLastError());
	CK(cudaEventRecord(c->ev1, c->stream));
	return 0;
}
