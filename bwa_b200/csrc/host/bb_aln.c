/* bb_aln.c -- `bwa-b200 aln`: BWA-backtrack, the .sai stream of the reference's `bwa aln` (bwtaln.c:159-321) byte for byte, with the
 * search on the GPU (bwag_aln, bwag_aln.cu).  `bwa samse` / `bwa sampe` read what it writes.
 *
 * It runs on the pipeline of bb_util.h: the reader parses the reads as bwa_read_seq does (bb_read_group, bb_seqio.c) in the
 * reference's groups of 262144 reads and cuts each group into device batches of BWA_B200_ALN_CHUNK reads.  The group matters: the
 * reference clamps max_gapo to the max_diff of the group's longest read (bwtaln.c:91-94), and that value enters every search of the
 * group.  max_diff itself (bwa_cal_maxdiff, a libm expression) is computed here, per read, and handed
 * to the device.  BWA_B200_PROFILE=1 reports the index load, the busy time of the three threads and the reads of tier 2. */
#include <unistd.h>
#include <math.h>
#include <stddef.h>
#include "bb_host.h"

#define ALN_MAX_LEN   65536      /* the reference keeps a read's remaining length in 16 bits of its queue entries (bwtgap.c:61,142) */
#define ALN_GROUP     0x40000    /* reads per bwa_read_seq call (bwtaln.c:180) */
#define ALN_AVG_ERR   0.02       /* BWA_AVG_ERR */
#define ALN_MODE_GAPE    0x01    /* the mode bits of gap_opt_t (bwtaln.h:94-103) */
#define ALN_MODE_COMPREAD 0x02
#define ALN_MODE_LOGGAP  0x04
#define ALN_MODE_CFY     0x08
#define ALN_MODE_NONSTOP 0x10
#define ALN_MODE_BAM_SE  0x40
#define ALN_MODE_BAM_READ1 0x80
#define ALN_MODE_BAM_READ2 0x100
#define ALN_MODE_IL13    0x200

/* bwt_aln1_t (bwtaln.h:43-46) on x86-64 GCC: the bit-field word, then k and l */
_Static_assert(sizeof(bwag_aln1_t) == 24 && offsetof(bwag_aln1_t, k) == 8 && offsetof(bwag_aln1_t, l) == 16, "bwt_aln1_t layout");

typedef struct aln_batch {
	int n;
	int64_t *off;              /* [n+1] first base of each read in codes[] */
	uint8_t *codes;            /* the searched bases, 0..4 */
	int8_t *md;                /* [n] max_diff of each read */
	int max_gapo;              /* -o clamped for the read's group */
	bwag_batch_t *dev;
	bwag_aln_t res;
} aln_batch_t;

typedef struct {
	bb_fq_t *fq;
	const aln_opt_t *opt;
	int chunk;
	int *md_of_len;            /* [ALN_MAX_LEN] max_diff by read length (-1: not computed yet) */
	bwag_ctx_t *ctx;
	bwag_aln_par_t par;
	long long n_tier2;
	int header_out;            /* writer: the .sai header is out */
} aln_run_t;

static int read_maxdiff(aln_run_t *r, int len)
{
	if (r->opt->fnr <= 0.0) return r->opt->max_diff;
	if (r->md_of_len[len] < 0) r->md_of_len[len] = bb_cal_maxdiff(len, ALN_AVG_ERR, r->opt->fnr);
	return r->md_of_len[len];
}

static void batch_free(aln_batch_t *b)
{
	if (!b) return;
	if (b->dev) bwag_batch_end(b->dev);
	free(b->off); free(b->codes); free(b->md);
	free(b);
}

/* the next group of the reference: up to ALN_GROUP reads that bwa_read_seq keeps (bb_read_group), with their max_diff and the
 * group's max_gapo; NULL at the end of the input */
static aln_batch_t *read_group(aln_run_t *r)
{
	const aln_opt_t *opt = r->opt;
	bb_reads_t *rd = bb_read_group(r->fq, opt->mode, opt->trim_qual, ALN_GROUP, 0, ALN_MAX_LEN, "bwa_aln");
	aln_batch_t *g;
	int i;
	if (!rd) return 0;
	g = bb_calloc(1, sizeof(*g));
	g->n = rd->n; g->off = rd->off; g->codes = rd->codes;   /* the searched bases */
	rd->off = 0; rd->codes = 0;
	{
		const int md_group = read_maxdiff(r, rd->max_len);
		g->max_gapo = md_group < opt->max_gapo ? md_group : opt->max_gapo;
	}
	g->md = bb_malloc((size_t)g->n + 1);
	for (i = 0; i < g->n; ++i) {
		const int md = read_maxdiff(r, rd->len[i]);
		if (md < -128 || md > 127) bb_fatal("bwa_aln", "max_diff %d is not supported (at most 127 differences)", md);
		g->md[i] = (int8_t)md;
	}
	bb_reads_free(rd);
	return g;
}

/* reads [beg, end) of a group as a batch of their own */
static aln_batch_t *slice(const aln_batch_t *g, int beg, int end)
{
	aln_batch_t *b = bb_calloc(1, sizeof(*b));
	const int64_t b0 = g->off[beg], nb = g->off[end] - b0;
	int i;
	b->n = end - beg;
	b->max_gapo = g->max_gapo;
	b->off = bb_malloc(8 * (size_t)(b->n + 1));
	for (i = 0; i <= b->n; ++i) b->off[i] = g->off[beg + i] - b0;
	b->codes = bb_malloc((size_t)nb + 16);
	if (nb) memcpy(b->codes, g->codes + b0, (size_t)nb);
	b->md = bb_malloc((size_t)b->n + 1);
	memcpy(b->md, g->md + beg, (size_t)b->n);
	return b;
}

static void read_all(bb_pipe_t *p, void *run)
{
	aln_run_t *r = run;
	aln_batch_t *g;
	while ((g = read_group(r)) != 0) {
		if (g->n <= r->chunk) { bb_pipe_to_device(p, g); continue; }
		for (int beg = 0; beg < g->n; beg += r->chunk) bb_pipe_to_device(p, slice(g, beg, beg + r->chunk < g->n ? beg + r->chunk : g->n));
		batch_free(g);
	}
}

static void run_device(bb_pipe_t *p, void *run, void *item)
{
	aln_run_t *r = run;
	aln_batch_t *b = item;
	int rc;
	if ((b->dev = bwag_batch_begin(r->ctx, b->n, b->codes, b->off)) == 0) bb_fatal("bwa_aln", "cannot start a device batch: %s", bwag_last_error());
	r->par.max_gapo = b->max_gapo; r->par.max_diff = b->md;
	rc = bwag_aln(b->dev, &r->par, &b->res);
	if (rc == BWAG_UNSUPPORTED) { fprintf(stderr, "[E::%s] this build has no device backtracking search\n", "bwa_aln"); exit(1); }
	if (rc != 0) bb_fatal("bwa_aln", "device search failed: %s", bwag_last_error());
	r->n_tier2 += b->res.n_tier2;
	bb_pipe_to_writer(p, b);
}

/* the header goes out once the first batch has been searched (or the input turned out empty): a build without the device search
 * leaves stdout empty */
static void write_header(aln_run_t *r)
{
	if (fwrite("SAI\1", 1, 4, stdout) != 4 || fwrite(r->opt, sizeof(*r->opt), 1, stdout) != 1) bb_fatal("bwa_aln", "fail to write the output");
	r->header_out = 1;
}

/* per read: int32 n_aln, then its n_aln 24-byte records (bwtaln.c:214-218) */
static void write_batch(void *run, void *item)
{
	aln_run_t *r = run;
	aln_batch_t *b = item;
	bb_str_t s = {0, 0, 0};
	int i;
	if (!r->header_out) write_header(r);
	for (i = 0; i < b->n; ++i) {
		const int32_t n = b->res.n_aln[i];
		bb_putsn(&s, (const char *)&n, 4);
		if (n) bb_putsn(&s, (const char *)(b->res.aln + b->res.off[i]), sizeof(bwag_aln1_t) * (size_t)n);
		bb_str_write(&s, 1 << 20, "bwa_aln");
	}
	bb_str_write(&s, 0, "bwa_aln");
	batch_free(b);   /* the device batch too: its pinned buffers held the hits until now */
}

static const bb_pipe_ops_t ops = { read_all, run_device, write_batch };

static void usage(const aln_opt_t *opt)
{
	fprintf(stderr, "\n");
	fprintf(stderr, "Usage:   bwa-b200 aln [options] <prefix> <in.fq>\n\n");
	fprintf(stderr, "Options: -n NUM    max #diff (int) or missing prob under %.2f err rate (float) [%.2f]\n", ALN_AVG_ERR, opt->fnr);
	fprintf(stderr, "         -o INT    maximum number or fraction of gap opens [%d]\n", opt->max_gapo);
	fprintf(stderr, "         -e INT    maximum number of gap extensions, -1 for disabling long gaps [-1]\n");
	fprintf(stderr, "         -i INT    do not put an indel within INT bp towards the ends [%d]\n", opt->indel_end_skip);
	fprintf(stderr, "         -d INT    maximum occurrences for extending a long deletion [%d]\n", opt->max_del_occ);
	fprintf(stderr, "         -l INT    seed length [%d]\n", opt->seed_len);
	fprintf(stderr, "         -k INT    maximum differences in the seed [%d]\n", opt->max_seed_diff);
	fprintf(stderr, "         -m INT    maximum entries in the queue [%d]\n", opt->max_entries);
	fprintf(stderr, "         -t INT    number of threads [%d] (written to the .sai header; the search runs on the GPU)\n", opt->n_threads);
	fprintf(stderr, "         -M INT    mismatch penalty [%d]\n", opt->s_mm);
	fprintf(stderr, "         -O INT    gap open penalty [%d]\n", opt->s_gapo);
	fprintf(stderr, "         -E INT    gap extension penalty [%d]\n", opt->s_gape);
	fprintf(stderr, "         -R INT    stop searching when there are >INT equally best hits [%d]\n", opt->max_top2);
	fprintf(stderr, "         -q INT    quality threshold for read trimming down to %dbp [%d]\n", BB_MIN_RDLEN, opt->trim_qual);
	fprintf(stderr, "         -f FILE   file to write output to instead of stdout\n");
	fprintf(stderr, "         -B INT    length of barcode\n");
	fprintf(stderr, "         -L        log-scaled gap penalty for long deletions\n");
	fprintf(stderr, "         -N        non-iterative mode: search for all n-difference hits (slooow)\n");
	fprintf(stderr, "         -I        the input is in the Illumina 1.3+ FASTQ-like format\n");
	fprintf(stderr, "         -b        BAM input: not supported (convert the reads to FASTQ)\n");
	fprintf(stderr, "         -0 -1 -2  accepted and recorded in the header (they select reads of BAM input)\n");
	fprintf(stderr, "         -Y        filter Casava-filtered sequences\n");
	fprintf(stderr, "\n");
}

int bb_aln_main(int argc, char *argv[])
{
	int c, opte = -1;
	aln_opt_t opt;
	bwaidx_t *idx;
	aln_run_t run;
	bwag_aln_par_t *par = &run.par;
	bb_pipe_busy_t busy;
	double t0, t_load;
	const char *e;

	memset(&opt, 0, sizeof(opt));   /* gap_init_opt (bwtaln.c:24-40) */
	opt.s_mm = 3; opt.s_gapo = 11; opt.s_gape = 4;
	opt.max_diff = -1; opt.max_gapo = 1; opt.max_gape = 6;
	opt.indel_end_skip = 5; opt.max_del_occ = 10; opt.max_entries = 2000000;
	opt.mode = ALN_MODE_GAPE | ALN_MODE_COMPREAD;
	opt.seed_len = 32; opt.max_seed_diff = 2;
	opt.fnr = 0.04f;
	opt.n_threads = 1;
	opt.max_top2 = 30;
	opt.trim_qual = 0;
	while ((c = getopt(argc, argv, "n:o:e:i:d:l:k:LR:m:t:NM:O:E:q:f:b012IYB:")) >= 0) {   /* bwtaln.c:237-268 */
		switch (c) {
		case 'n':
			if (strstr(optarg, ".")) opt.fnr = (float)atof(optarg), opt.max_diff = -1;
			else opt.max_diff = atoi(optarg), opt.fnr = -1.0f;
			break;
		case 'o': opt.max_gapo = atoi(optarg); break;
		case 'e': opte = atoi(optarg); break;
		case 'M': opt.s_mm = atoi(optarg); break;
		case 'O': opt.s_gapo = atoi(optarg); break;
		case 'E': opt.s_gape = atoi(optarg); break;
		case 'd': opt.max_del_occ = atoi(optarg); break;
		case 'i': opt.indel_end_skip = atoi(optarg); break;
		case 'l': opt.seed_len = atoi(optarg); break;
		case 'k': opt.max_seed_diff = atoi(optarg); break;
		case 'm': opt.max_entries = atoi(optarg); break;
		case 't': opt.n_threads = atoi(optarg); break;
		case 'L': opt.mode |= ALN_MODE_LOGGAP; break;
		case 'R': opt.max_top2 = atoi(optarg); break;
		case 'q': opt.trim_qual = atoi(optarg); break;
		case 'N': opt.mode |= ALN_MODE_NONSTOP; opt.max_top2 = 0x7fffffff; break;
		case 'f': if (freopen(optarg, "wb", stdout) == 0) bb_fatal("bwa_aln", "fail to open file '%s'", optarg); break;
		case 'b': fprintf(stderr, "[bwa_aln] BAM input (-b) is not supported: convert the reads to FASTQ\n"); return 1;
		case '0': opt.mode |= ALN_MODE_BAM_SE; break;
		case '1': opt.mode |= ALN_MODE_BAM_READ1; break;
		case '2': opt.mode |= ALN_MODE_BAM_READ2; break;
		case 'I': opt.mode |= ALN_MODE_IL13; break;
		case 'Y': opt.mode |= ALN_MODE_CFY; break;
		case 'B': opt.mode |= (int)((unsigned)atoi(optarg) << 24); break;
		default: return 1;
		}
	}
	if (opte > 0) {
		opt.max_gape = opte;
		opt.mode &= ~ALN_MODE_GAPE;
	}
	if (optind + 2 > argc) { usage(&opt); return 1; }
	if (opt.fnr > 0.0) {   /* bwtaln.c:305-312 */
		int i, k;
		for (i = 17, k = 0; i <= 250; ++i) {
			const int l = bb_cal_maxdiff(i, ALN_AVG_ERR, opt.fnr);
			if (l != k) fprintf(stderr, "[bwa_aln] %dbp reads: max_diff = %d\n", i, l);
			k = l;
		}
	}
	if (opt.s_mm < 0 || opt.s_gapo < 0 || opt.s_gape < 0) bb_fatal("bwa_aln", "the penalties -M, -O and -E must not be negative");
	if (opt.seed_len < 0) bb_fatal("bwa_aln", "the seed length -l must not be negative");

	memset(&run, 0, sizeof(run));
	run.opt = &opt;
	run.chunk = (e = getenv("BWA_B200_ALN_CHUNK")) != 0 && atoi(e) > 0 ? atoi(e) : ALN_GROUP;   /* reads per device batch */
	run.md_of_len = bb_malloc(sizeof(int) * ALN_MAX_LEN);
	memset(run.md_of_len, 0xff, sizeof(int) * ALN_MAX_LEN);
	if ((run.fq = bb_fq_open(argv[optind + 1])) == 0) bb_fatal("bwa_aln", "fail to open file '%s'", argv[optind + 1]);
	t0 = bb_realtime();
	if ((idx = bb_idx_from_resident(argv[optind])) == 0 && (idx = bwa_idx_load(argv[optind], BWA_IDX_ALL)) == 0) {
		fprintf(stderr, "[bwa_aln] fail to locate the index\n");
		bb_fq_close(run.fq); free(run.md_of_len);
		return 1;
	}
	run.ctx = bb_device_attach(idx->bwt, idx->bns, idx->pac);   /* fails here, before any output, if there is no GPU */
	t_load = bb_realtime() - t0;
	par->s_mm = opt.s_mm; par->s_gapo = opt.s_gapo; par->s_gape = opt.s_gape;
	par->mode = opt.mode & (BWAG_ALN_GAPE | BWAG_ALN_LOGGAP | BWAG_ALN_NONSTOP);
	par->indel_end_skip = opt.indel_end_skip; par->max_del_occ = opt.max_del_occ; par->max_entries = opt.max_entries;
	par->max_gape = opt.max_gape; par->max_seed_diff = opt.max_seed_diff; par->seed_len = opt.seed_len; par->max_top2 = opt.max_top2;
	bb_pipe_run(&ops, &run, &busy);
	if (!run.header_out) write_header(&run);   /* an empty input */
	if (fflush(stdout) != 0 || ferror(stdout)) bb_fatal("bwa_aln", "fail to write the output");
	if (getenv("BWA_B200_PROFILE"))
		fprintf(stderr, "[prof] aln: index load %.3f s; busy time of the reader %.3f s, the device %.3f s, the writer %.3f s; %lld reads in tier 2; total %.3f s\n",
		        t_load, busy.read, busy.device, busy.write, run.n_tier2, bb_realtime() - t0);
	bb_fq_close(run.fq);
	free(run.md_of_len);
	bwa_idx_destroy(idx);
	return 0;
}
