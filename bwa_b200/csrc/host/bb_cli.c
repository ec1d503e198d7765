/* bb_cli.c -- the `bwa mem` command line over the H100 path (reference fastmap.c:141-406, main.c:87-130).
 *
 * Same options, presets and -A scaling rules as the reference.  I/O runs beside the GPU work on its
 * own threads: a reader thread parses the next batch while the current one is aligned, and a writer
 * thread prints the previous one; batches are handed over through depth-1 mailboxes so output order
 * equals input order (the reference gets the same overlap from its 2-thread kt_pipeline).
 */
#include <unistd.h>
#include <ctype.h>
#include <math.h>
#include <pthread.h>
#include <assert.h>
#include "bb_host.h"

#define BB_VERSION "0.7.19-r1273-b200"

typedef struct { int n; bseq1_t *seqs; int last; int skip; long no, seq_no; int64_t n_before; } batch_t;   /* skip: another rank's batch (multi-GPU runs); no: number in the whole run; seq_no: number in this process (the writer's order) */

/* finished batches wait here until it is their turn to be written (several batches are aligned at a time) */
#define RO_SLOTS 8
typedef struct {
	pthread_mutex_t mu;
	pthread_cond_t cv;
	batch_t *slot[RO_SLOTS];
	long next_write, total;   /* total < 0 until the reader has seen the end of the input */
} reorder_t;
static void ro_init(reorder_t *o) { pthread_mutex_init(&o->mu, 0); pthread_cond_init(&o->cv, 0); memset(o->slot, 0, sizeof(o->slot)); o->next_write = 0; o->total = -1; }
static void ro_post(reorder_t *o, batch_t *b)
{
	pthread_mutex_lock(&o->mu);
	while (b->seq_no - o->next_write >= RO_SLOTS) pthread_cond_wait(&o->cv, &o->mu);
	o->slot[b->seq_no % RO_SLOTS] = b;
	pthread_cond_broadcast(&o->cv);
	pthread_mutex_unlock(&o->mu);
}
static void ro_finish(reorder_t *o, long total) { pthread_mutex_lock(&o->mu); o->total = total; pthread_cond_broadcast(&o->cv); pthread_mutex_unlock(&o->mu); }
static batch_t *ro_next(reorder_t *o)   /* the batch with the next number, or NULL when all have been written */
{
	batch_t *b;
	pthread_mutex_lock(&o->mu);
	while (!o->slot[o->next_write % RO_SLOTS] && !(o->total >= 0 && o->next_write >= o->total)) pthread_cond_wait(&o->cv, &o->mu);
	b = o->slot[o->next_write % RO_SLOTS];
	o->slot[o->next_write % RO_SLOTS] = 0;
	if (b) { ++o->next_write; pthread_cond_broadcast(&o->cv); }
	pthread_mutex_unlock(&o->mu);
	return b;
}

typedef struct {
	bb_fq_t *f1, *f2;
	mem_opt_t *opt;
	mem_pestat_t *pes0;
	bwaidx_t *idx;
	int copy_comment, chunk;
	int64_t n_processed;
	bb_mbox_t to_align;   /* closed at the end of the input: every aligner thread then stops */
	reorder_t done;
	/* multi-GPU runs (bwa_b200/multi.py): batches are dealt round-robin, batch b belongs to rank b % world; every rank
	 * parses the whole input so that batch boundaries -- and with them the per-batch insert-size model -- are those of
	 * a single-GPU run.  shard_idx records "batch bytes" per written batch so that rank 0 can merge the parts in order */
	int rank, world;
	long n_batches;
	FILE *shard_idx;
	const char *fn1, *fn2;    /* input paths (planned batches reopen them by byte range) */
} run_t;

static bwaidx_t *g_cli_idx;   /* an index the caller already holds (and has made resident): used instead of loading */
void bb_cli_set_index(bwaidx_t *idx) { g_cli_idx = idx; }

/* striped ingest (include/bwa_b200.h): the batches of this process as byte ranges of the input files, set by the launcher */
static const bb_planned_batch_t *g_plan;
static int64_t g_plan_n = -1, g_plan_total;
void bb_cli_set_plan(const bb_planned_batch_t *mine, int64_t n_mine, int64_t n_batches_total) { g_plan = mine; g_plan_n = mine ? n_mine : -1; g_plan_total = n_batches_total; }

/* a planned batch: everything in its byte range(s), read the way bseq_read reads (pairs interleaved, warnings included) */
static bseq1_t *read_planned(const run_t *r, const bb_planned_batch_t *p, int *n)
{
	bb_fq_t *f1 = bb_fq_open_range(r->fn1, p->beg1, p->end1), *f2 = r->fn2 ? bb_fq_open_range(r->fn2, p->beg2, p->end2) : 0;
	bseq1_t *seqs;
	if (!f1 || (r->fn2 && !f2)) bb_fatal("main_mem", "fail to reopen the input for batch %ld", (long)p->no);
	seqs = bseq_read(0x7fffffff, n, f1, f2);
	bb_fq_close(f1); bb_fq_close(f2);
	return seqs;
}

static void w_free_reads(void *d, long c, int tid)   /* 1024 reads per item */
{
	batch_t *b = d;
	long i, e = (c + 1) * 1024 < b->n ? (c + 1) * 1024 : b->n;
	(void)tid;
	for (i = c * 1024; i < e; ++i) { bseq1_t *s = &b->seqs[i]; free(s->name); free(s->comment); free(s->seq); free(s->qual); free(s->sam); }
}
static void free_reads(batch_t *b)   /* five strings per read, allocated by many threads: released by several threads as well */
{
	if (b->seqs) bb_parallel_for(b->n >= 8192 ? 4 : 1, w_free_reads, b, ((long)b->n + 1023) / 1024);
	free(b->seqs); b->seqs = 0;
}

static void write_batch(run_t *r, batch_t *b)
{
	long bytes = 0;
	int i;
	for (i = 0; i < b->n; ++i) {
		bseq1_t *s = &b->seqs[i];
		if (!s->sam) continue;
		if (fputs(s->sam, stdout) == EOF) bb_fatal("main_mem", "fail to write the SAM output");
		if (r->shard_idx) bytes += (long)strlen(s->sam);
	}
	if (r->shard_idx) fprintf(r->shard_idx, "%ld %ld\n", b->no, bytes);
}

static void *reader_main(void *a)
{
	run_t *r = a;
	int64_t k = 0;
	for (;;) {
		batch_t *b = bb_calloc(1, sizeof(*b));
		int i;
		int64_t size = 0;
		if (g_plan_n >= 0) {   /* only this process's batches, each from its byte range; the writer sees just those */
			if (k >= g_plan_n) { free(b); ro_finish(&r->done, k); bb_mbox_put(&r->to_align, 0); return 0; }
			b->seqs = read_planned(r, &g_plan[k], &b->n);
			b->no = g_plan[k].no; b->n_before = g_plan[k].n_before; b->seq_no = k++;
			if (!b->seqs) bb_fatal("main_mem", "planned batch %ld is empty", b->no);
		} else {
			b->seqs = bseq_read(r->chunk, &b->n, r->f1, r->f2);
			if (!b->seqs) { free(b); ro_finish(&r->done, r->n_batches); bb_mbox_put(&r->to_align, 0); return 0; }
			b->no = b->seq_no = r->n_batches++;
			b->n_before = r->n_processed; r->n_processed += b->n;
		}
		if (g_plan_n < 0 && b->no % r->world != r->rank) { b->skip = 1; free_reads(b); bb_mbox_put(&r->to_align, b); continue; }
		if (!r->copy_comment)
			for (i = 0; i < b->n; ++i) { free(b->seqs[i].comment); b->seqs[i].comment = 0; }
		for (i = 0; i < b->n; ++i) size += b->seqs[i].l_seq;
		if (bwa_verbose >= 3) fprintf(stderr, "[M::%s] read %d sequences (%ld bp)...\n", "process", b->n, (long)size);
		bb_mbox_put(&r->to_align, b);
	}
}

static void *writer_main(void *a)
{
	run_t *r = a;
	batch_t *b;
	while ((b = ro_next(&r->done)) != 0) {
		if (!b->skip) { write_batch(r, b); free_reads(b); }
		free(b);
	}
	return 0;
}

static void align_batch(run_t *r, batch_t *b)
{
	const mem_opt_t *opt = r->opt;
	const bwaidx_t *idx = r->idx;
	if (b->skip) return;
	if (opt->flag & MEM_F_SMARTPE) { /* -p: split the batch into single-end and paired reads (fastmap.c:90-109) */
		bseq1_t *sep[2];
		int n_sep[2], i;
		mem_opt_t tmp = *opt;
		bseq_classify(b->n, b->seqs, n_sep, sep);
		if (bwa_verbose >= 3) fprintf(stderr, "[M::%s] %d single-end sequences; %d paired-end sequences\n", "process", n_sep[0], n_sep[1]);
		if (n_sep[0]) {
			tmp.flag &= ~MEM_F_PE;
			mem_process_seqs(&tmp, idx->bwt, idx->bns, idx->pac, b->n_before, n_sep[0], sep[0], 0);
			for (i = 0; i < n_sep[0]; ++i) b->seqs[sep[0][i].id].sam = sep[0][i].sam;
		}
		if (n_sep[1]) {
			tmp.flag |= MEM_F_PE;
			mem_process_seqs(&tmp, idx->bwt, idx->bns, idx->pac, b->n_before + n_sep[0], n_sep[1], sep[1], r->pes0);
			for (i = 0; i < n_sep[1]; ++i) b->seqs[sep[1][i].id].sam = sep[1][i].sam;
		}
		free(sep[0]); free(sep[1]);
	} else mem_process_seqs(opt, idx->bwt, idx->bns, idx->pac, b->n_before, b->n, b->seqs, r->pes0);
}

static void *aligner_main(void *a)
{
	run_t *r = a;
	batch_t *b;
	while ((b = bb_mbox_get(&r->to_align)) != 0) {
		align_batch(r, b);
		ro_post(&r->done, b);
	}
	return 0;
}

static void scale_by_match_score(mem_opt_t *opt, const mem_opt_t *set) /* -A scales what the user left alone (fastmap.c:125-139) */
{
	if (!set->a) return;
	if (!set->b) opt->b *= opt->a;
	if (!set->T) opt->T *= opt->a;
	if (!set->o_del) opt->o_del *= opt->a;
	if (!set->e_del) opt->e_del *= opt->a;
	if (!set->o_ins) opt->o_ins *= opt->a;
	if (!set->e_ins) opt->e_ins *= opt->a;
	if (!set->zdrop) opt->zdrop *= opt->a;
	if (!set->pen_clip5) opt->pen_clip5 *= opt->a;
	if (!set->pen_clip3) opt->pen_clip3 *= opt->a;
	if (!set->pen_unpaired) opt->pen_unpaired *= opt->a;
}

static int two_ints(const char *arg, int *first, int *second) /* "INT[,INT]" */
{
	char *p;
	*first = *second = (int)strtol(arg, &p, 10);
	if (*p != 0 && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) *second = (int)strtol(p + 1, &p, 10);
	return 0;
}

static void usage(const mem_opt_t *opt)
{
	fprintf(stderr, "\nUsage: bwa-b200 mem [options] <idxbase> <in1.fq> [in2.fq]\n\n");
	fprintf(stderr, "Options are those of `bwa mem` (lh3/bwa 0.7.19), e.g.:\n");
	fprintf(stderr, "  -t INT  host threads [%d]     -k INT  min seed length [%d]   -w INT  band width [%d]\n", opt->n_threads, opt->min_seed_len, opt->w);
	fprintf(stderr, "  -d INT  Z-dropoff [%d]        -r FLOAT re-seed factor [%g]   -y INT  3rd-round seed occ [%ld]\n", opt->zdrop, opt->split_factor, (long)opt->max_mem_intv);
	fprintf(stderr, "  -c INT  max occ [%d]          -D FLOAT chain drop ratio [%.2f] -W INT min chain weight [0]\n", opt->max_occ, opt->drop_ratio);
	fprintf(stderr, "  -m INT  mate-rescue rounds [%d] -S skip rescue  -P skip pairing\n", opt->max_matesw);
	fprintf(stderr, "  -A -B -O -E -L -U  scoring [%d,%d,%d/%d,%d/%d,%d/%d,%d]   -x pacbio|ont2d|intractg|pbref\n", opt->a, opt->b, opt->o_del, opt->o_ins, opt->e_del, opt->e_ins, opt->pen_clip5, opt->pen_clip3, opt->pen_unpaired);
	fprintf(stderr, "  -p smart pairing  -R STR read group  -H STR/FILE header  -o FILE output  -j ignore ALT\n");
	fprintf(stderr, "  -5 -q -K INT -v INT -T INT -h INT[,INT] -z FLOAT -a -C -V -Y -M -I FLOAT[,FLOAT[,INT[,INT]]] -u\n\n");
}

int main_mem(int argc, char *argv[])
{
	mem_opt_t *opt, set;
	int c, i, ignore_alt = 0, no_mt_io = 0, fixed_chunk = -1, t_given = 0;
	char *p, *rg_line = 0, *hdr_line = 0;
	const char *mode = 0;
	mem_pestat_t pes[4];
	run_t run;
	pthread_t th_r, th_w;

	memset(&run, 0, sizeof(run));
	memset(pes, 0, sizeof(pes));
	for (i = 0; i < 4; ++i) pes[i].failed = 1;
	run.opt = opt = mem_opt_init();
	memset(&set, 0, sizeof(set)); /* which options the user set explicitly */
	while ((c = getopt(argc, argv, "51qpaMCSPVYjuk:c:v:s:r:t:R:A:B:O:E:U:w:L:d:T:Q:D:m:I:N:o:f:W:x:G:h:y:K:X:H:F:z:")) >= 0) {
		switch (c) {
		case 'k': opt->min_seed_len = atoi(optarg); set.min_seed_len = 1; break;
		case '1': no_mt_io = 1; break;
		case 'x': mode = optarg; break;
		case 'w': opt->w = atoi(optarg); set.w = 1; break;
		case 'A': opt->a = atoi(optarg); set.a = 1; break;
		case 'B': opt->b = atoi(optarg); set.b = 1; break;
		case 'T': opt->T = atoi(optarg); set.T = 1; break;
		case 'U': opt->pen_unpaired = atoi(optarg); set.pen_unpaired = 1; break;
		case 't': opt->n_threads = atoi(optarg); if (opt->n_threads < 1) opt->n_threads = 1; t_given = 1; break;
		case 'P': opt->flag |= MEM_F_NOPAIRING; break;
		case 'a': opt->flag |= MEM_F_ALL; break;
		case 'p': opt->flag |= MEM_F_PE | MEM_F_SMARTPE; break;
		case 'M': opt->flag |= MEM_F_NO_MULTI; break;
		case 'S': opt->flag |= MEM_F_NO_RESCUE; break;
		case 'Y': opt->flag |= MEM_F_SOFTCLIP; break;
		case 'V': opt->flag |= MEM_F_REF_HDR; break;
		case '5': opt->flag |= MEM_F_PRIMARY5 | MEM_F_KEEP_SUPP_MAPQ; break;
		case 'q': opt->flag |= MEM_F_KEEP_SUPP_MAPQ; break;
		case 'u': opt->flag |= MEM_F_XB; break;
		case 'c': opt->max_occ = atoi(optarg); set.max_occ = 1; break;
		case 'd': opt->zdrop = atoi(optarg); set.zdrop = 1; break;
		case 'v': bwa_verbose = atoi(optarg); break;
		case 'j': ignore_alt = 1; break;
		case 'r': opt->split_factor = atof(optarg); set.split_factor = 1.; break;
		case 'D': opt->drop_ratio = atof(optarg); set.drop_ratio = 1.; break;
		case 'm': opt->max_matesw = atoi(optarg); set.max_matesw = 1; break;
		case 's': opt->split_width = atoi(optarg); set.split_width = 1; break;
		case 'G': opt->max_chain_gap = atoi(optarg); set.max_chain_gap = 1; break;
		case 'N': opt->max_chain_extend = atoi(optarg); set.max_chain_extend = 1; break;
		case 'o': case 'f': if (!freopen(optarg, "wb", stdout)) bb_fatal("main_mem", "fail to open '%s' for writing", optarg); break;
		case 'W': opt->min_chain_weight = atoi(optarg); set.min_chain_weight = 1; break;
		case 'y': opt->max_mem_intv = atol(optarg); set.max_mem_intv = 1; break;
		case 'C': run.copy_comment = 1; break;
		case 'K': fixed_chunk = atoi(optarg); break;
		case 'X': opt->mask_level = atof(optarg); break;
		case 'F': break; /* debug flags of the reference: accepted, unused */
		case 'h': set.max_XA_hits = set.max_XA_hits_alt = 1; two_ints(optarg, &opt->max_XA_hits, &opt->max_XA_hits_alt); break;
		case 'z': opt->XA_drop_ratio = atof(optarg); break;
		case 'Q': set.mapQ_coef_len = 1; opt->mapQ_coef_len = atoi(optarg); opt->mapQ_coef_fac = opt->mapQ_coef_len > 0 ? log(opt->mapQ_coef_len) : 0; break;
		case 'O': set.o_del = set.o_ins = 1; two_ints(optarg, &opt->o_del, &opt->o_ins); break;
		case 'E': set.e_del = set.e_ins = 1; two_ints(optarg, &opt->e_del, &opt->e_ins); break;
		case 'L': set.pen_clip5 = set.pen_clip3 = 1; two_ints(optarg, &opt->pen_clip5, &opt->pen_clip3); break;
		case 'R': if ((rg_line = bwa_set_rg(optarg)) == 0) return 1; break;
		case 'H':
			if (optarg[0] != '@') {
				FILE *fp = fopen(optarg, "r");
				if (fp) {
					char *buf = bb_calloc(1, 0x10000);
					while (fgets(buf, 0xffff, fp)) {
						size_t l = strlen(buf);
						if (l && buf[l - 1] == '\n') buf[l - 1] = 0;
						hdr_line = bwa_insert_header(buf, hdr_line);
					}
					free(buf); fclose(fp);
				}
			} else hdr_line = bwa_insert_header(optarg, hdr_line);
			break;
		case 'I':
			run.pes0 = pes;
			pes[1].failed = 0;
			pes[1].avg = strtod(optarg, &p);
			pes[1].std = pes[1].avg * .1;
			if (*p != 0 && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) pes[1].std = strtod(p + 1, &p);
			pes[1].high = (int)(pes[1].avg + 4. * pes[1].std + .499);
			pes[1].low = (int)(pes[1].avg - 4. * pes[1].std + .499);
			if (pes[1].low < 1) pes[1].low = 1;
			if (*p != 0 && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) pes[1].high = (int)(strtod(p + 1, &p) + .499);
			if (*p != 0 && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) pes[1].low = (int)(strtod(p + 1, &p) + .499);
			if (bwa_verbose >= 3) fprintf(stderr, "[M::%s] mean insert size: %.3f, stddev: %.3f, max: %d, min: %d\n", __func__, pes[1].avg, pes[1].std, pes[1].high, pes[1].low);
			break;
		default: return 1;
		}
	}
	if (rg_line) { hdr_line = bwa_insert_header(rg_line, hdr_line); free(rg_line); }
	if (opt->n_threads < 1) opt->n_threads = 1;
	if (optind + 1 >= argc || optind + 3 < argc) { usage(opt); free(opt); return 1; }

	if (mode) { /* presets only touch what the user did not set (fastmap.c:330-358) */
		if (strcmp(mode, "intractg") == 0) {
			if (!set.o_del) opt->o_del = 16;
			if (!set.o_ins) opt->o_ins = 16;
			if (!set.b) opt->b = 9;
			if (!set.pen_clip5) opt->pen_clip5 = 5;
			if (!set.pen_clip3) opt->pen_clip3 = 5;
		} else if (strcmp(mode, "pacbio") == 0 || strcmp(mode, "pbref") == 0 || strcmp(mode, "ont2d") == 0) {
			int ont = strcmp(mode, "ont2d") == 0;
			if (!set.o_del) opt->o_del = 1;
			if (!set.e_del) opt->e_del = 1;
			if (!set.o_ins) opt->o_ins = 1;
			if (!set.e_ins) opt->e_ins = 1;
			if (!set.b) opt->b = 1;
			if (set.split_factor == 0.) opt->split_factor = 10.;
			if (!set.min_chain_weight) opt->min_chain_weight = ont ? 20 : 40;
			if (!set.min_seed_len) opt->min_seed_len = ont ? 14 : 17;
			if (!set.pen_clip5) opt->pen_clip5 = 0;
			if (!set.pen_clip3) opt->pen_clip3 = 0;
		} else {
			fprintf(stderr, "[E::%s] unknown read type '%s'\n", __func__, mode);
			return 1;
		}
	} else scale_by_match_score(opt, &set);
	bwa_fill_scmat(opt->a, opt->b, opt->mat);

	{   /* rank/world of a multi-GPU run, set by the launcher */
		const char *e;
		run.rank = (e = getenv("BWA_B200_RANK")) ? atoi(e) : 0;
		run.world = (e = getenv("BWA_B200_WORLD")) ? atoi(e) : 1;
		if (run.world < 1 || run.rank < 0 || run.rank >= run.world) bb_fatal("main_mem", "bad BWA_B200_RANK/BWA_B200_WORLD");
		if ((e = getenv("BWA_B200_SHARD_IDX")) != 0 && (run.shard_idx = fopen(e, "w")) == 0) bb_fatal("main_mem", "fail to open '%s' for writing", e);
	}
	if (g_cli_idx) run.idx = g_cli_idx;
	else if ((run.idx = bb_idx_from_resident(argv[optind])) != 0) {}   /* kept on the GPU by `bwa-b200 shm` */
	else if ((run.idx = bwa_idx_load(argv[optind], BWA_IDX_ALL)) == 0) return 1;
	if (ignore_alt) for (i = 0; i < run.idx->bns->n_seqs; ++i) run.idx->bns->anns[i].is_alt = 0;
	run.fn1 = argv[optind + 1];
	if ((run.f1 = bb_fq_open(argv[optind + 1])) == 0) {
		if (bwa_verbose >= 1) fprintf(stderr, "[E::%s] fail to open file `%s'.\n", __func__, argv[optind + 1]);
		return 1;
	}
	if (optind + 2 < argc) {
		if (opt->flag & MEM_F_PE) {
			if (bwa_verbose >= 2) fprintf(stderr, "[W::%s] when '-p' is in use, the second query file is ignored.\n", __func__);
		} else {
			if ((run.f2 = bb_fq_open(argv[optind + 2])) == 0) {
				if (bwa_verbose >= 1) fprintf(stderr, "[E::%s] fail to open file `%s'.\n", __func__, argv[optind + 2]);
				return 1;
			}
			run.fn2 = argv[optind + 2];
			opt->flag |= MEM_F_PE;
		}
	}
	bb_device_attach(run.idx->bwt, run.idx->bns, run.idx->pac); /* fail early, before any output, if there is no GPU */
	if (run.rank == 0) bwa_print_sam_hdr(run.idx->bns, hdr_line);
	if (run.shard_idx) { fflush(stdout); fprintf(run.shard_idx, "-1 %ld\n", ftell(stdout)); }
	run.chunk = fixed_chunk > 0 ? fixed_chunk : opt->chunk_size * opt->n_threads;
	/* Without -t the reference runs one thread and forms batches of chunk_size bases; the batches stay exactly those (so
	 * the output is `bwa mem`'s), but the host phases between the GPU stages use the CPUs the process is allowed. */
	if (!t_given) opt->n_threads = bb_effective_cpus();

	bb_mbox_init(&run.to_align); ro_init(&run.done);
	if (no_mt_io) {
		int64_t k = 0;
		for (;;) {
			batch_t bb;
			memset(&bb, 0, sizeof(bb));
			if (g_plan_n >= 0) {
				if (k >= g_plan_n) break;
				bb.seqs = read_planned(&run, &g_plan[k], &bb.n);
				bb.no = g_plan[k].no; bb.n_before = g_plan[k].n_before; ++k;
				if (!bb.seqs) bb_fatal("main_mem", "planned batch %ld is empty", bb.no);
			} else {
				bb.seqs = bseq_read(run.chunk, &bb.n, run.f1, run.f2);
				if (!bb.seqs) break;
				bb.no = run.n_batches++;
				bb.n_before = run.n_processed; run.n_processed += bb.n;
				bb.skip = bb.no % run.world != run.rank;
			}
			if (!bb.skip && !run.copy_comment) for (i = 0; i < bb.n; ++i) { free(bb.seqs[i].comment); bb.seqs[i].comment = 0; }
			align_batch(&run, &bb);
			if (!bb.skip) write_batch(&run, &bb);
			free_reads(&bb);
		}
	} else {
		pthread_create(&th_r, 0, reader_main, &run);
		pthread_create(&th_w, 0, writer_main, &run);
		/* BWA_B200_INFLIGHT batches are aligned at a time (default 3): while one
		 * waits for a device stage or splices its text, the GPU works on another; the writer restores the input order */
		{
			const char *e = getenv("BWA_B200_INFLIGHT");
			int n_al = e ? atoi(e) : 3, t;
			pthread_t th_a[4];
			if (n_al < 1) n_al = 1;
			if (n_al > 4) n_al = 4;
			for (t = 1; t < n_al; ++t) pthread_create(&th_a[t], 0, aligner_main, &run);
			aligner_main(&run);
			for (t = 1; t < n_al; ++t) pthread_join(th_a[t], 0);
		}
		pthread_join(th_r, 0);
		pthread_join(th_w, 0);
	}
	fflush(stdout);
	if (run.shard_idx) fclose(run.shard_idx);
	free(hdr_line);
	if (run.idx != g_cli_idx) bwa_idx_destroy(run.idx);
	bb_fq_close(run.f1);
	bb_fq_close(run.f2);
	free(opt);
	return 0;
}

#ifdef BB_MAIN
int main(int argc, char *argv[])
{
	double t0 = bb_realtime();
	bb_str_t pg = {0, 0, 0};
	int i, ret;
	bb_puts(&pg, "@PG\tID:bwa\tPN:bwa\tVN:" BB_VERSION "\tCL:");
	for (i = 0; i < argc; ++i) { if (i) bb_putc(&pg, ' '); bb_puts(&pg, argv[i]); }
	bwa_pg = pg.s;
	if (argc >= 2 && strcmp(argv[1], "shm") == 0) { free(pg.s); return bb_shm_main(argc - 1, argv + 1); }
	if (argc >= 2 && strcmp(argv[1], "index") == 0) { free(pg.s); return bb_index_main(argc - 1, argv + 1); }
	if (argc >= 2 && strcmp(argv[1], "fa2pac") == 0) { free(pg.s); return bb_fa2pac_main(argc - 1, argv + 1); }
	if (argc >= 2 && strcmp(argv[1], "pac2bwt") == 0) { free(pg.s); return bb_pac2bwt_main(argc - 1, argv + 1); }
	if (argc >= 2 && strcmp(argv[1], "pac2bwtgen") == 0) { free(pg.s); return bb_pac2bwtgen_main(argc - 1, argv + 1); }
	if (argc >= 2 && strcmp(argv[1], "bwtupdate") == 0) { free(pg.s); return bb_bwtupdate_main(argc - 1, argv + 1); }
	if (argc >= 2 && strcmp(argv[1], "bwt2sa") == 0) { free(pg.s); return bb_bwt2sa_main(argc - 1, argv + 1); }
	if (argc >= 2 && strcmp(argv[1], "maxk") == 0) { free(pg.s); ret = bb_maxk_main(argc - 1, argv + 1); fflush(stdout); return ret; }
	if (argc >= 2 && strcmp(argv[1], "fastmap") == 0) { free(pg.s); ret = bb_fastmap_main(argc - 1, argv + 1); fflush(stdout); return ret; }
	if (argc >= 2 && strcmp(argv[1], "aln") == 0) { free(pg.s); ret = bb_aln_main(argc - 1, argv + 1); fflush(stdout); return ret; }
	if (argc >= 2 && strcmp(argv[1], "samse") == 0) { ret = bb_samse_main(argc - 1, argv + 1); fflush(stdout); free(pg.s); return ret; }
	if (argc >= 2 && strcmp(argv[1], "sampe") == 0) { ret = bb_sampe_main(argc - 1, argv + 1); fflush(stdout); free(pg.s); return ret; }
	if (argc >= 2 && strcmp(argv[1], "pemerge") == 0) { free(pg.s); ret = bb_pemerge_main(argc - 1, argv + 1); fflush(stdout); return ret; }
	if (argc < 2 || strcmp(argv[1], "mem") != 0) {
		fprintf(stderr, "\nProgram: bwa-b200 (BWA-MEM seed-and-extend on NVIDIA H100)\nVersion: %s\n\nUsage:   bwa-b200 index [-p prefix] <in.fasta[.gz]>   build the index files on the GPU\n", BB_VERSION);
		fprintf(stderr, "         bwa-b200 mem [options] <idxbase> <in1.fq> [in2.fq]\n");
		fprintf(stderr, "         bwa-b200 fastmap [options] <idxbase> <in.fq>   list each read's SMEMs and their positions\n");
		fprintf(stderr, "         bwa-b200 maxk [-s] <in.bwt> <seq.fa>            histogram of each base's longest SMEM (-s: against its own index)\n");
		fprintf(stderr, "         bwa-b200 aln [options] <idxbase> <in.fq>       BWA-backtrack: the .sai file of `bwa aln`\n");
		fprintf(stderr, "         bwa-b200 samse [-n max_occ] [-f out.sam] [-r RG_line] <idxbase> <in.sai> <in.fq>   single-end SAM from a .sai file\n");
		fprintf(stderr, "         bwa-b200 sampe [-a maxins] [-o maxocc] [-n INT] [-N INT] [-c FLOAT] [-f out.sam] [-r RG_line] [-P] [-s] [-A]\n"
		                "                        <idxbase> <in1.sai> <in2.sai> <in1.fq> <in2.fq>   paired-end SAM from two .sai files\n");
		fprintf(stderr, "         bwa-b200 pemerge [-mu] [-t INT] [-T INT] [-Q INT] <read1.fq> [read2.fq]   merge overlapping read pairs\n");
		fprintf(stderr, "         bwa-b200 shm [-d|-l] [idxbase]      keep an index resident on the GPU between runs\n\n");
		fprintf(stderr, "The steps of `index` on their own:\n");
		fprintf(stderr, "         bwa-b200 fa2pac [-f] <in.fasta> [<out.prefix>]   .pac .ann .amb (without -f: with the reverse complement)\n");
		fprintf(stderr, "         bwa-b200 pac2bwt [-d] <in.pac> <out.bwt>         the BWT of the .pac text, without Occ (-d: ignored)\n");
		fprintf(stderr, "         bwa-b200 pac2bwtgen <in.pac> <out.bwt>           the same file\n");
		fprintf(stderr, "         bwa-b200 bwtupdate <the.bwt>                     add the Occ checkpoints, in place\n");
		fprintf(stderr, "         bwa-b200 bwt2sa [-i 32] <in.bwt> <out.sa>        the suffix array, every INT-th row, from the .bwt alone\n\n");
		fprintf(stderr, "The index is the one `bwa index` writes; `bwa-b200 index` writes the same files.\n\n");
		return 1;
	}
	ret = main_mem(argc - 1, argv + 1);
	fflush(stdout);
	if (ret == 0 && bwa_verbose >= 3) {
		fprintf(stderr, "[%s] Version: %s\n[%s] CMD:", __func__, BB_VERSION, __func__);
		for (i = 0; i < argc; ++i) fprintf(stderr, " %s", argv[i]);
		fprintf(stderr, "\n[%s] Real time: %.3f sec; CPU: %.3f sec\n", __func__, bb_realtime() - t0, bb_cputime());
	}
	free(pg.s);
	return ret;
}
#endif
