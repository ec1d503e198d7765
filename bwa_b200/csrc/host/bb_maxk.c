/* bb_maxk.c -- `bwa-b200 maxk`: for each base of each input sequence the longest SMEM that covers it (capped at 255), as a
 * 256-bin histogram, byte for byte what the reference's `bwa maxk` prints (maxk.c:11-66), with the SMEM search on the GPU
 * (bwag_maxk, bwag_maxk.cu).  `maxk -s <ref>.bwt <ref>.fa` counts, for each k, the bases of a genome that lie in exact repeats
 * of length k.
 *
 * The index is the updated .bwt file alone (bwt_restore_bwt).  The reader parses batches of whole sequences up to
 * BWA_B200_MAXK_CHUNK bases (kseq grammar: FASTA/FASTQ, plain or gzip, '-' for stdin); a longer sequence is a batch of its own,
 * since its search needs the whole sequence.  The device cuts each sequence into windows of BWA_B200_MAXK_WINDOW bases that run in
 * parallel when every base occurs at least min_intv times in the BWT (DESIGN.md §4.14), and runs one window per sequence
 * otherwise.  The histogram is printed once, after the last sequence.  Where the reference crashes or prints garbage (a .bwt
 * without Occ checkpoints, a file that is no .bwt at all) the command says why and exits 1 with nothing on stdout.
 * BWA_B200_PROFILE=1 names the path taken and reports the device's times. */
#include <unistd.h>
#include <errno.h>
#include "bb_host.h"

#define MAXK_WINDOW_DEFAULT 1024   /* fastest of 1024, 4096 and 16384 on a 3 Gbp self-run (DESIGN.md §7) */

typedef struct mk_batch {
	int n;
	int64_t *off;              /* [n+1] first base of each sequence in codes[] */
	uint8_t *codes;            /* 0..4 */
	uint64_t hist[256];
	bwag_maxk_stats_t st;
} mk_batch_t;

typedef struct {
	bb_fq_t *fq;
	int64_t chunk, window;     /* window 0: one per sequence */
	int min_intv;
	bwag_ctx_t *ctx;
	uint64_t hist[256];
	int64_t n_windows, n_bases;
	int n_repeat, list_cap;
	double ms_kernel, ms_hist, max_window_ms;
} mk_run_t;

static void batch_free(mk_batch_t *b)
{
	free(b->off); free(b->codes); free(b);
}

/* the next batch: whole sequences until chunk bases are reached (at least one sequence), NULL at the end of the input */
static mk_batch_t *read_batch(mk_run_t *r)
{
	const bb_str_t *name, *comment, *seq;
	mk_batch_t *b = 0;
	int64_t m = 0, bases = 0, m_bases = 0;
	while (bases < r->chunk || !b) {
		int len, i;
		if ((len = bb_fq_read1(r->fq, &name, &comment, &seq)) < 0) break;   /* kseq_read < 0 ends the reference's loop too */
		if (!b) { b = bb_calloc(1, sizeof(*b)); m = 1024; b->off = bb_malloc(8 * (size_t)(m + 1)); b->off[0] = 0; }
		if (b->n == m) { m <<= 1; b->off = bb_realloc(b->off, 8 * (size_t)(m + 1)); }
		if (bases + len > m_bases) {
			m_bases = m_bases ? m_bases : 1 << 16;
			while (m_bases < bases + len) m_bases <<= 1;
			b->codes = bb_realloc(b->codes, (size_t)m_bases);
		}
		for (i = 0; i < len; ++i) { const int c = bb_nt4_table[(unsigned char)seq->s[i]]; b->codes[bases + i] = (uint8_t)(c > 4 ? 4 : c); }
		bases += len;
		b->off[++b->n] = bases;
	}
	if (b && !b->codes) b->codes = bb_malloc(16);   /* a batch of empty sequences */
	return b;
}

static void read_all(bb_pipe_t *p, void *run)
{
	mk_batch_t *b;
	while ((b = read_batch(run)) != 0) bb_pipe_to_device(p, b);
}

static void run_device(bb_pipe_t *p, void *run, void *item)
{
	mk_run_t *r = run;
	mk_batch_t *b = item;
	bwag_batch_t *d;
	int rc;
	if ((d = bwag_batch_begin(r->ctx, b->n, b->codes, b->off)) == 0) bb_fatal("main_maxk", "cannot start a device batch: %s", bwag_last_error());
	rc = bwag_maxk(d, r->min_intv, r->window, b->hist, &b->st);
	if (rc == BWAG_UNSUPPORTED) { fprintf(stderr, "[E::%s] this build has no device SMEM search\n", "main_maxk"); exit(1); }
	if (rc != 0) bb_fatal("main_maxk", "device SMEM search failed: %s", bwag_last_error());
	bwag_batch_end(d);
	bb_pipe_to_writer(p, b);
}

/* the batch's counts join the total; nothing is printed before the last batch */
static void write_batch(void *run, void *item)
{
	mk_run_t *r = run;
	mk_batch_t *b = item;
	int k;
	for (k = 0; k < 256; ++k) r->hist[k] += b->hist[k];
	r->n_windows += b->st.n_windows; r->n_bases += b->off[b->n];
	r->n_repeat += b->st.n_repeat;
	if (b->st.list_cap > r->list_cap) r->list_cap = b->st.list_cap;
	r->ms_kernel += b->st.ms_kernel; r->ms_hist += b->st.ms_hist;
	if (b->st.max_window_ms > r->max_window_ms) r->max_window_ms = b->st.max_window_ms;
	batch_free(b);
}

static const bb_pipe_ops_t ops = { read_all, run_device, write_batch };

int bb_maxk_main(int argc, char *argv[])
{
	int c, k, self = 0, fails = 0;
	bwt_t *bwt;
	mk_run_t run;
	bb_pipe_busy_t busy;
	double t0 = bb_realtime(), t_load;
	const char *e;
	bb_str_t s = {0, 0, 0};

	while ((c = getopt(argc, argv, "s")) >= 0)   /* maxk.c:22-24: other options are reported by getopt and ignored */
		if (c == 's') self = 1;
	if (optind + 2 > argc) { fprintf(stderr, "Usage: bwa-b200 maxk [-s] <in.bwt> <seq.fa>\n"); return 1; }

	memset(&run, 0, sizeof(run));
	run.min_intv = self ? 2 : 1;   /* smem_config(itr, 2, INT_MAX, 0) under -s; the iterator's defaults otherwise */
	run.chunk = (e = getenv("BWA_B200_MAXK_CHUNK")) != 0 && atol(e) > 0 ? atol(e) : 64000000;   /* bases per batch */
	if ((run.fq = bb_fq_open(argv[optind + 1])) == 0) { fprintf(stderr, "[E::%s] fail to open file '%s' : %s\n", "main_maxk", argv[optind + 1], strerror(errno)); return 1; }
	if ((bwt = bb_read_bwt(argv[optind], 1, "main_maxk")) == 0) { bb_fq_close(run.fq); return 1; }
	/* windows give the reference's counts only if every base occurs at least min_intv times in the BWT (DESIGN.md §4.14) */
	for (k = 0; k < 4; ++k) if (bwt->L2[k + 1] - bwt->L2[k] < (uint64_t)run.min_intv) fails = 1;
	run.window = fails ? 0 : (e = getenv("BWA_B200_MAXK_WINDOW")) != 0 && atol(e) > 0 ? atol(e) : MAXK_WINDOW_DEFAULT;
	if ((run.ctx = bwag_ctx_create_occ(-1, bwt)) == 0) { fprintf(stderr, "[E::%s] %s\n", "main_maxk", bwag_last_error()); bb_fq_close(run.fq); free(bwt->bwt); free(bwt); return 1; }
	free(bwt->bwt); free(bwt);
	t_load = bb_realtime() - t0;
	bb_pipe_run(&ops, &run, &busy);
	for (k = 0; k < 256; ++k) {
		bb_putl(&s, k); bb_putc(&s, '\t'); bb_putl(&s, (int64_t)run.hist[k]); bb_putc(&s, '\n');
	}
	bb_str_write(&s, 0, "main_maxk");
	if (fflush(stdout) != 0 || ferror(stdout)) bb_fatal("main_maxk", "fail to write the output");
	if (getenv("BWA_B200_PROFILE")) {
		if (run.window > 0) fprintf(stderr, "[prof] maxk: path: windows of %lld bases (%lld windows)\n", (long long)run.window, (long long)run.n_windows);
		else fprintf(stderr, "[prof] maxk: path: one window per sequence (a base occurs fewer than %d times in the BWT)\n", run.min_intv);
		fprintf(stderr, "[prof] maxk: %lld bases; index load %.3f s; search kernel %.3f ms, longest window %.3f ms, binning %.3f ms; list capacity %d, runs repeated %d; busy time of the reader %.3f s, the device %.3f s, the writer %.3f s; total %.3f s\n",
		        (long long)run.n_bases, t_load, run.ms_kernel, run.max_window_ms, run.ms_hist, run.list_cap, run.n_repeat, busy.read, busy.device, busy.write, bb_realtime() - t0);
	}
	bb_fq_close(run.fq);
	bwag_ctx_destroy(run.ctx);
	return 0;
}
