/* bb_pemerge.c -- `bwa-b200 pemerge`: the merged and unmerged read pairs of the reference's `bwa pemerge` (pemerge.c:217-291) byte for
 * byte, with the alignment, the tests, the merge and the records on the GPU (bwag_pemerge, bwag_pemerge.cu).
 *
 * It runs on the pipeline of bb_util.h: the reader takes the pairs with bseq_read (two files, or one interleaved file; trim_readno,
 * gzip, "-" for stdin and the two "fewer sequences" warnings come with it), drops an odd last read as process_seqs does, and copies
 * each batch of BWA_B200_PEMERGE_CHUNK pairs into page-locked buffers: sequences, qualities and names, one copy per byte; the writer
 * prints the records the device wrote and returns the batch, buffers kept, to a free list for the reader.  Pairs are independent
 * and the reference only breaks its batches at an even read count, so our batch size shows in no byte; the reader still calls
 * bseq_read with the reference's size, because a call that reads no base probes file 2 and so consumes one of its records.  The
 * nine counts go to stderr after the output.  BWA_B200_PROFILE=1 reports the busy time of the three threads. */
#include <unistd.h>
#include <errno.h>
#include "bb_host.h"

#define PM_GROUP_BASES (1 << 26)   /* bases per group of pairs the reader gathers; no byte depends on it */
#define PM_CHUNK       (1 << 18)   /* pairs per device batch unless BWA_B200_PEMERGE_CHUNK says otherwise */
#define WHO "main_pemerge"

static const char *err_msg[9] = {   /* pemerge.c:22-32 */
	"successful merges",
	"low-scoring pairs",
	"pairs where the best SW alignment is not an overlap (long left end)",
	"pairs where the best SW alignment is not an overlap (long right end)",
	"pairs with large 2nd best SW score",
	"pairs with gapped overlap",
	"pairs where the end-to-end alignment is inconsistent with SW",
	"pairs potentially with tandem overlaps",
	"pairs with high sum of errors"
};

typedef struct { void *p; size_t cap; } pm_buf_t;   /* page-locked, grown as needed */

typedef struct pm_batch {
	struct pm_batch *next;        /* the free list */
	int n;                        /* pairs */
	pm_buf_t seq, qual, hasq, names, off, noff;
	bwag_batch_t *dev;
	bwag_pemerge_t res;
} pm_batch_t;

typedef struct {
	bb_fq_t *fq[2];
	int chunk;
	int ref_chunk;                /* the reference's bseq_read size, n_threads * 10000000 as an int */
	pthread_mutex_t mu; pm_batch_t *free_list;   /* batches the writer is done with, buffers kept */
	bwag_ctx_t *ctx;
	bwag_pemerge_par_t par;
	int64_t cnt[9];               /* writer */
	int eof;
	long long n_pairs;
} pm_run_t;

static void *buf_need(pm_buf_t *b, size_t bytes)
{
	if (bytes > b->cap) {
		bwag_host_free(b->p);
		b->cap = bytes + bytes / 4 + 4096;
		if ((b->p = bwag_host_alloc(b->cap)) == 0) bb_fatal(WHO, "cannot allocate %zu bytes of page-locked memory", b->cap);
	}
	return b->p;
}

static pm_batch_t *batch_get(pm_run_t *r)
{
	pm_batch_t *b;
	pthread_mutex_lock(&r->mu);
	if ((b = r->free_list) != 0) r->free_list = b->next;
	pthread_mutex_unlock(&r->mu);
	return b ? b : bb_calloc(1, sizeof(pm_batch_t));
}

static void batch_put(pm_run_t *r, pm_batch_t *b)
{
	if (b->dev) bwag_batch_end(b->dev);
	b->dev = 0;
	pthread_mutex_lock(&r->mu);
	b->next = r->free_list; r->free_list = b;
	pthread_mutex_unlock(&r->mu);
}

static void batch_destroy(pm_batch_t *b)
{
	bwag_host_free(b->seq.p); bwag_host_free(b->qual.p); bwag_host_free(b->hasq.p); bwag_host_free(b->names.p); bwag_host_free(b->off.p); bwag_host_free(b->noff.p);
	free(b);
}

/* pairs [beg, end) of a group, copied into a batch's page-locked buffers */
static pm_batch_t *fill(pm_run_t *r, const bseq1_t *seqs, int beg, int end)
{
	pm_batch_t *b = batch_get(r);
	const int nr = 2 * (end - beg);
	int64_t nb = 0, nn = 0, *off, *noff;
	uint8_t *hasq;
	char *seq, *qual, *names;
	int i;
	b->n = end - beg;
	for (i = 0; i < nr; ++i) { const bseq1_t *s = &seqs[2 * beg + i]; nb += s->l_seq; nn += (int64_t)strlen(s->name); }
	seq = buf_need(&b->seq, (size_t)nb + 1); qual = buf_need(&b->qual, (size_t)nb + 1); names = buf_need(&b->names, (size_t)nn + 1);
	hasq = buf_need(&b->hasq, (size_t)nr + 1);
	off = buf_need(&b->off, 8 * ((size_t)nr + 1)); noff = buf_need(&b->noff, 8 * ((size_t)nr + 1));
	off[0] = noff[0] = 0;
	for (i = 0; i < nr; ++i) {
		const bseq1_t *s = &seqs[2 * beg + i];
		const size_t ln = strlen(s->name);
		memcpy(seq + off[i], s->seq, (size_t)s->l_seq);
		if ((hasq[i] = s->qual != 0) != 0) memcpy(qual + off[i], s->qual, (size_t)s->l_seq);
		memcpy(names + noff[i], s->name, ln);
		off[i + 1] = off[i] + s->l_seq; noff[i + 1] = noff[i] + (int64_t)ln;
	}
	return b;
}

/* the next group of pairs: the reference's bseq_read calls (their sizes matter: a call whose reads hold no base reads one more
 * record of file 2, see DESIGN.md 4.12), gathered until the group holds PM_GROUP_BASES bases; an odd last read of a call is dropped
 * (pemerge.c:178).  NULL at the end of the input. */
static bseq1_t *read_group(pm_run_t *r, int *n_)
{
	bseq1_t *g = 0;
	int n = 0, m = 0;
	int64_t bases = 0;
	for (;;) {
		int k, i;
		bseq1_t *seqs = bseq_read(r->ref_chunk, &k, r->fq[0], r->fq[1]);
		if (!seqs) { r->eof = 1; break; }
		if (k & 1) { --k; free(seqs[k].name); free(seqs[k].comment); free(seqs[k].seq); free(seqs[k].qual); }
		if (n + k > m) { m = (n + k) * 2; g = bb_realloc(g, sizeof(*g) * (size_t)m); }
		for (i = 0; i < k; ++i) bases += seqs[i].l_seq;
		memcpy(g + n, seqs, sizeof(*g) * (size_t)k);
		n += k;
		free(seqs);
		if (bases >= PM_GROUP_BASES || n >= (1 << 24)) break;
	}
	*n_ = n;
	return n ? g : (free(g), (bseq1_t *)0);
}

static void read_all(bb_pipe_t *p, void *run)
{
	pm_run_t *r = run;
	while (!r->eof) {
		int n, i, beg;
		bseq1_t *seqs = read_group(r, &n);
		if (!seqs) break;
		const int np = n >> 1;
		for (beg = 0; beg < np; beg += r->chunk) bb_pipe_to_device(p, fill(r, seqs, beg, beg + r->chunk < np ? beg + r->chunk : np));
		for (i = 0; i < n; ++i) { free(seqs[i].name); free(seqs[i].comment); free(seqs[i].seq); free(seqs[i].qual); }
		free(seqs);
	}
}

static void run_device(bb_pipe_t *p, void *run, void *item)
{
	pm_run_t *r = run;
	pm_batch_t *b = item;
	if ((b->dev = bwag_batch_begin(r->ctx, 2 * b->n, b->seq.p, b->off.p)) == 0) bb_fatal(WHO, "cannot start a device batch: %s", bwag_last_error());
	r->par.qual = b->qual.p; r->par.has_qual = b->hasq.p; r->par.names = b->names.p; r->par.name_off = b->noff.p;
	if (bwag_pemerge(b->dev, &r->par, &b->res) != 0) bb_fatal(WHO, "device pemerge failed: %s", bwag_last_error());
	bb_pipe_to_writer(p, b);
}

static void write_batch(void *run, void *item)
{
	pm_run_t *r = run;
	pm_batch_t *b = item;
	int k;
	if (b->res.n_text && fwrite(b->res.text, 1, (size_t)b->res.n_text, stdout) != (size_t)b->res.n_text) bb_fatal(WHO, "fail to write the output");
	for (k = 0; k < 9; ++k) r->cnt[k] += b->res.cnt[k];
	r->n_pairs += b->n;
	batch_put(r, b);
}

static const bb_pipe_ops_t ops = { read_all, run_device, write_batch };

static bb_fq_t *open_reads(const char *fn)
{
	bb_fq_t *f;
	errno = 0;
	if ((f = bb_fq_open(fn)) == 0) {   /* pemerge.c:252-258 */
		fprintf(stderr, "Couldn't open %s : %s\n", strcmp(fn, "-") ? fn : "stdin", errno ? strerror(errno) : "Out of memory");
		exit(EXIT_FAILURE);
	}
	return f;
}

int bb_pemerge_main(int argc, char *argv[])
{
	int c, flag = 0, min_ovlp = 10, q_thres = 70, n_threads = 1, i;
	pm_run_t run;
	bwag_pemerge_par_t *par = &run.par;
	bb_pipe_busy_t busy;
	double t0 = bb_realtime();
	const char *e;
	while ((c = getopt(argc, argv, "muQ:t:T:")) >= 0) {   /* pemerge.c:227-234 */
		if (c == 'm') flag |= 1;
		else if (c == 'u') flag |= 2;
		else if (c == 'Q') q_thres = atoi(optarg);
		else if (c == 't') n_threads = atoi(optarg);
		else if (c == 'T') min_ovlp = atoi(optarg);
		else return 1;
	}
	if (flag == 0) flag = 3;
	if (optind == argc) {
		fprintf(stderr, "\n");
		fprintf(stderr, "Usage:   bwa-b200 pemerge [-mu] <read1.fq> [read2.fq]\n\n");
		fprintf(stderr, "Options: -m       output merged reads only\n");
		fprintf(stderr, "         -u       output unmerged reads only\n");
		fprintf(stderr, "         -t INT   number of threads [%d]\n", n_threads);
		fprintf(stderr, "         -T INT   minimum end overlap [%d]\n", min_ovlp);
		fprintf(stderr, "         -Q INT   max sum of errors [%d]\n", q_thres);
		fprintf(stderr, "\n");
		return 1;
	}
	if (n_threads < 0) { fprintf(stderr, "[E::%s] the number of threads (-t) must not be negative\n", WHO); return 1; }
	memset(&run, 0, sizeof(run));
	run.fq[0] = open_reads(argv[optind]);
	if (optind + 1 < argc) {
		if (strcmp(argv[optind + 1], "-") && access(argv[optind + 1], R_OK) != 0) {   /* the reference tests the wrong handle here and crashes */
			fprintf(stderr, "Couldn't open %s : %s\n", argv[optind + 1], strerror(errno));
			exit(EXIT_FAILURE);
		}
		run.fq[1] = open_reads(argv[optind + 1]);
	}
	if ((run.ctx = bwag_ctx_create_bare(-1)) == 0) bb_fatal(WHO, "cannot use the GPU: %s", bwag_last_error());   /* before any output */
	par->T = 5 * min_ovlp; par->q_thres = q_thres; par->q_def = 20; par->flag = flag;
	par->merge = n_threads > 0;   /* -t 0: the reference starts no worker, so no pair is tried */
	{   /* a batch of no pairs: does this build have the device stage at all? */
		static const uint8_t none[1] = {0};
		static const int64_t zero[1] = {0};
		bwag_pemerge_t res;
		bwag_batch_t *b = bwag_batch_begin(run.ctx, 0, none, zero);
		int rc;
		if (!b) bb_fatal(WHO, "cannot start a device batch: %s", bwag_last_error());
		par->qual = none; par->has_qual = none; par->names = (const char *)none; par->name_off = zero;
		rc = bwag_pemerge(b, par, &res);
		bwag_batch_end(b);
		if (rc == BWAG_UNSUPPORTED) { fprintf(stderr, "[E::%s] this build has no device pemerge\n", WHO); exit(1); }
		if (rc != 0) bb_fatal(WHO, "device pemerge failed: %s", bwag_last_error());
	}
	run.ref_chunk = (int)((uint32_t)n_threads * 10000000u);   /* pemerge.c:52,272: wraps above -t 214 */
	run.chunk = (e = getenv("BWA_B200_PEMERGE_CHUNK")) != 0 && atoi(e) > 0 ? atoi(e) : PM_CHUNK;
	pthread_mutex_init(&run.mu, 0);
	bb_pipe_run(&ops, &run, &busy);
	if (fflush(stdout) != 0 || ferror(stdout)) bb_fatal(WHO, "fail to write the output");
	for (i = 0; i <= 8; ++i) fprintf(stderr, "%12ld %s\n", (long)run.cnt[i], err_msg[i]);   /* pemerge.c:277-279 */
	if (getenv("BWA_B200_PROFILE"))
		fprintf(stderr, "[prof] pemerge: busy time of the reader %.3f s, the device %.3f s, the writer %.3f s; %lld pairs; total %.3f s\n",
		        busy.read, busy.device, busy.write, run.n_pairs, bb_realtime() - t0);
	while (run.free_list) { pm_batch_t *b = run.free_list; run.free_list = b->next; batch_destroy(b); }
	bb_fq_close(run.fq[0]); bb_fq_close(run.fq[1]);
	bwag_ctx_destroy(run.ctx);
	return 0;
}
