/* bb_fastmap.c -- `bwa-b200 fastmap`: every SMEM of each read with its occurrence count and reference positions, byte for byte
 * what the reference's `bwa fastmap` prints (fastmap.c:408-483), with the SMEM search, the suffix-array lookups and the EM lines
 * on the GPU (bwag_fastmap: K1 in its fastmap form, K2, bwag_fastmap.cu).
 *
 * It runs on the pipeline of bb_util.h: the reader parses batches of BWA_B200_FASTMAP_CHUNK bases (kseq grammar: FASTA/FASTQ, plain
 * or gzip, '-' for stdin), and the writer prints per read its SQ line, the device's EM lines and "//".  At most four batches exist
 * at a time.  BWA_B200_PROFILE=1 reports the busy time of the three threads and the index load. */
#include <unistd.h>
#include "bb_host.h"

#define FM_MAX_LEN (1 << 23)   /* K1 keeps match ends in 23 bits (bwag_smem.cu) */

typedef struct fm_batch {
	int n;
	int64_t *off;              /* [n+1] first base of each read in codes[] (and raw[]) */
	uint8_t *codes;            /* 0..4 */
	char *raw;                 /* the letters as read (-p only) */
	bb_str_t names;            /* NUL-terminated, back to back */
	int64_t *name_off;         /* [n] */
	bwag_batch_t *dev;
	bwag_fastmap_t res;
} fm_batch_t;

typedef struct {
	bb_fq_t *fq;
	int64_t chunk;
	int print_seq;
	bwag_ctx_t *ctx;
	bwag_fastmap_par_t par;
} fm_run_t;

static void batch_free(fm_batch_t *b)
{
	if (!b) return;
	if (b->dev) bwag_batch_end(b->dev);
	free(b->off); free(b->codes); free(b->raw); free(b->names.s); free(b->name_off);
	free(b);
}

/* the next batch: reads until chunk bases are reached (at least one read), NULL at the end of the input */
static fm_batch_t *read_batch(fm_run_t *r)
{
	const bb_str_t *name, *comment, *seq;
	fm_batch_t *b = 0;
	int64_t m = 0, bases = 0, m_bases = 0;
	while (bases < r->chunk || !b) {
		int len = bb_fq_read1(r->fq, &name, &comment, &seq), i;
		if (len < 0) break;   /* end of input, or a truncated quality string: kseq_read < 0 ends the reference's loop too */
		if (len >= FM_MAX_LEN) bb_fatal("main_fastmap", "read '%s' has %d bases; reads of 2^23 (%d) bases or more are not supported", name->s, len, FM_MAX_LEN);
		if (!b) { b = bb_calloc(1, sizeof(*b)); m = 1024; b->off = bb_malloc(8 * (size_t)(m + 1)); b->name_off = bb_malloc(8 * (size_t)m); b->off[0] = 0; }
		if (b->n == m) { m <<= 1; b->off = bb_realloc(b->off, 8 * (size_t)(m + 1)); b->name_off = bb_realloc(b->name_off, 8 * (size_t)m); }
		if (bases + len > m_bases) {
			m_bases = m_bases ? m_bases : 1 << 16;
			while (m_bases < bases + len) m_bases <<= 1;
			b->codes = bb_realloc(b->codes, (size_t)m_bases);
			if (r->print_seq) b->raw = bb_realloc(b->raw, (size_t)m_bases);
		}
		for (i = 0; i < len; ++i) { const int c = bb_nt4_table[(unsigned char)seq->s[i]]; b->codes[bases + i] = (uint8_t)(c > 4 ? 4 : c); }
		if (r->print_seq && len) memcpy(b->raw + bases, seq->s, (size_t)len);
		b->name_off[b->n] = (int64_t)b->names.l;
		bb_putsn(&b->names, name->s, name->l);
		bb_putc(&b->names, 0);   /* a NUL inside the text, after the name */
		bases += len;
		b->off[++b->n] = bases;
	}
	if (b && !b->codes) b->codes = bb_malloc(16);   /* a batch of empty reads */
	return b;
}

static void read_all(bb_pipe_t *p, void *run)
{
	fm_batch_t *b;
	while ((b = read_batch(run)) != 0) bb_pipe_to_device(p, b);
}

static void run_device(bb_pipe_t *p, void *run, void *item)
{
	fm_run_t *r = run;
	fm_batch_t *b = item;
	int rc;
	if ((b->dev = bwag_batch_begin(r->ctx, b->n, b->codes, b->off)) == 0) bb_fatal("main_fastmap", "cannot start a device batch: %s", bwag_last_error());
	rc = bwag_fastmap(b->dev, &r->par, &b->res);
	if (rc == BWAG_UNSUPPORTED) { fprintf(stderr, "[E::%s] this build has no device SMEM lister\n", "main_fastmap"); exit(1); }
	if (rc != 0) bb_fatal("main_fastmap", "device SMEM listing failed: %s", bwag_last_error());
	bb_pipe_to_writer(p, b);
}

static void write_batch(void *run, void *item)
{
	const fm_run_t *r = run;
	fm_batch_t *b = item;
	bb_str_t s = {0, 0, 0};
	int i;
	for (i = 0; i < b->n; ++i) {
		const int64_t len = b->off[i + 1] - b->off[i], t0 = b->res.off[i], t1 = b->res.off[i + 1];
		bb_puts(&s, "SQ\t");
		bb_puts(&s, b->names.s + b->name_off[i]);
		bb_putc(&s, '\t');
		bb_putl(&s, len);
		if (r->print_seq) { bb_putc(&s, '\t'); bb_putsn(&s, b->raw + b->off[i], (size_t)len); }   /* err_puts: the letters as read, then a newline */
		bb_putc(&s, '\n');
		bb_putsn(&s, b->res.text + t0, (size_t)(t1 - t0));
		bb_puts(&s, "//\n");
		bb_str_write(&s, 1 << 20, "main_fastmap");
	}
	bb_str_write(&s, 0, "main_fastmap");
	batch_free(b);   /* the device batch too: its pinned text buffer held the EM lines until now */
}

static const bb_pipe_ops_t ops = { read_all, run_device, write_batch };

static void usage(int min_len, int w, int min_intv, int max_len, uint64_t max_intv)
{
	fprintf(stderr, "\n");
	fprintf(stderr, "Usage:   bwa-b200 fastmap [options] <idxbase> <in.fq>\n\n");
	fprintf(stderr, "Options: -l INT    min SMEM length to output [%d]\n", min_len);
	fprintf(stderr, "         -w INT    max interval size to find coordinates [%d]\n", w);
	fprintf(stderr, "         -i INT    min SMEM interval size [%d]\n", min_intv);
	fprintf(stderr, "         -L INT    max MEM length [%d] (accepted; no effect, as in bwa fastmap)\n", max_len);
	fprintf(stderr, "         -I INT    stop if MEM is longer than -l with a size less than INT [%ld]\n", (long)max_intv);
	fprintf(stderr, "         -p        print the read's sequence on its SQ line\n");
	fprintf(stderr, "\n");
}

int bb_fastmap_main(int argc, char *argv[])
{
	int c, min_iwidth = 20, min_len = 17, print_seq = 0, min_intv = 1, max_len = 0x7fffffff;
	uint64_t max_intv = 0;
	bwaidx_t *idx;
	fm_run_t run;
	bb_pipe_busy_t busy;
	double t0, t_load;
	const char *e;

	while ((c = getopt(argc, argv, "w:l:pi:I:L:")) >= 0) {   /* fastmap.c:419-429 */
		switch (c) {
		case 'p': print_seq = 1; break;
		case 'w': min_iwidth = atoi(optarg); break;
		case 'l': min_len = atoi(optarg); break;
		case 'i': min_intv = atoi(optarg); break;
		case 'I': max_intv = (uint64_t)atol(optarg); break;
		case 'L': max_len = atoi(optarg); break;   /* smem_next never reads it */
		default: return 1;
		}
	}
	if (optind + 1 >= argc) { usage(min_len, min_iwidth, min_intv, max_len, max_intv); return 1; }

	memset(&run, 0, sizeof(run));
	run.print_seq = print_seq;
	run.chunk = (e = getenv("BWA_B200_FASTMAP_CHUNK")) != 0 && atol(e) > 0 ? atol(e) : 40000000;   /* bases per batch */
	if ((run.fq = bb_fq_open(argv[optind + 1])) == 0) bb_fatal("main_fastmap", "fail to open file '%s'", argv[optind + 1]);
	t0 = bb_realtime();
	if ((idx = bb_idx_from_resident(argv[optind])) == 0 && (idx = bwa_idx_load(argv[optind], BWA_IDX_ALL)) == 0) { bb_fq_close(run.fq); return 1; }
	run.ctx = bb_device_attach(idx->bwt, idx->bns, idx->pac);   /* fails here, before any output, if there is no GPU */
	t_load = bb_realtime() - t0;
	run.par.min_len = min_len; run.par.min_intv = min_intv; run.par.max_intv = max_intv; run.par.max_iwidth = min_iwidth;
	bb_pipe_run(&ops, &run, &busy);
	if (fflush(stdout) != 0 || ferror(stdout)) bb_fatal("main_fastmap", "fail to write the output");
	if (getenv("BWA_B200_PROFILE"))
		fprintf(stderr, "[prof] fastmap: index load %.3f s; busy time of the reader %.3f s, the device %.3f s, the writer %.3f s; total %.3f s\n",
		        t_load, busy.read, busy.device, busy.write, bb_realtime() - t0);
	bb_fq_close(run.fq);
	bwa_idx_destroy(idx);
	return 0;
}
