/* bb_samse.c -- `bwa-b200 samse`: the single-end SAM of the reference's `bwa samse` (bwase.c:507-606) byte for byte, from a .sai
 * file of `bwa aln` or `bwa-b200 aln`, with the suffix-array lookups, the gapped refinement, MD/NM and the SAM text on the GPU
 * (bwag_samse, bwag_samse.cu).
 *
 * Three threads overlap: a reader parses the reads as bwa_read_seq does (bb_read_group) in the reference's groups of 262144 reads,
 * reads the group's .sai records, chooses each read's hit and its XA candidates (bwa_aln2seq_core) and its mapping quality
 * (bwa_approx_mapQ), and cuts the group into device batches of BWA_B200_SAMSE_CHUNK reads; the calling thread runs the current
 * batch on the device; a writer prints the previous one.  The hit choice draws random numbers in read order over the whole input,
 * so it stays on the one reader thread, with a private erand48 state seeded as the reference's srand48(bns->seed) seeds drand48:
 * the same sequence, which nothing else in the process can disturb, and the batch size cannot change a byte.  A group's .sai records
 * are read before any of its batches reaches the writer: when the .sai ends early, the earlier groups are out, as in the
 * reference, and the command fails with its message.  BWA_B200_PROFILE=1 reports the index load, the busy time of the three
 * threads, the hits sent to the suffix array and the global alignments. */
#include <unistd.h>
#include <math.h>
#include <pthread.h>
#include "bb_host.h"

#define SE_GROUP   0x40000     /* reads per bwa_read_seq call (bwase.c:538) */
#define SE_MAX_LEN (1 << 20)   /* bwa_seq_t keeps len and full_len in 20 bits (its 14-bit CIGAR lengths wrap as they do there, bwag_samse.cu) */
#define SE_AVG_ERR 0.02        /* BWA_AVG_ERR */

typedef struct se_group {     /* one group of the reference: its reads and what the host chose for them */
	bb_reads_t *rd;
	bwag_se_read_t *reads;
	bwag_se_hit_t *multi; int64_t n_multi;
} se_group_t;

typedef struct se_batch {
	int n, last, sai_eof;          /* last: the group's final batch (the writer frees the group); sai_eof: the .sai ended in this group */
	se_group_t *g; int beg;        /* reads [beg, beg + n) of the group */
	int64_t *off;                  /* [n+1] the reads' codes, from 0 */
	bwag_se_read_t *reads;         /* multi_beg and bc_off relative to this batch */
	char *bc; int64_t l_bc;
	bwag_batch_t *dev;
	bwag_sam_t res;
} se_batch_t;

typedef struct {
	bb_fq_t *fq;
	FILE *fp_sa;
	const aln_opt_t *opt;
	int n_occ, chunk;
	unsigned short rng[3];         /* erand48 state: the drand48 sequence after srand48(bns->seed) */
	int log_n[256];                /* g_log_n (bwase_initialize) */
	bwag_aln1_t *aln; int m_aln;
	bb_mbox_t to_dev, to_write;
	int sai_eof;
	double t_read, t_write;
} se_run_t;

static void group_free(se_group_t *g)
{
	if (!g) return;
	bb_reads_free(g->rd); free(g->reads); free(g->multi);
	free(g);
}

static void batch_free(se_batch_t *b)
{
	if (!b) return;
	if (b->dev) bwag_batch_end(b->dev);
	free(b->off); free(b->reads); free(b->bc);
	if (b->last) group_free(b->g);
	free(b);
}

/* bwa_aln2seq_core(n_aln, aln, p, 1, n_occ) (bwase.c:22-94) with the reference's integer widths: int counts, 28-bit c1/c2 */
static void choose_hit(se_run_t *r, int n_aln, const bwag_aln1_t *aln, bwag_se_read_t *p, se_group_t *g, int64_t *m_multi)
{
	int i, cnt, best;
	if (n_aln == 0) { p->type = 0; p->c1 = p->c2 = 0; return; }
	best = (int)(aln[0].bits >> 24 & 0xfffff);
	for (i = cnt = 0; i < n_aln; ++i) {
		const bwag_aln1_t *q = aln + i;
		const uint64_t w = q->l - q->k + 1;
		if ((int)(q->bits >> 24 & 0xfffff) > best) break;
		if (erand48(r->rng) * (double)(w + (uint64_t)(int64_t)cnt) > (double)cnt) {
			p->n_mm = (uint8_t)(q->bits & 0xff); p->n_gapo = (uint8_t)(q->bits >> 8 & 0xff); p->n_gape = (uint8_t)(q->bits >> 16 & 0xff);
			p->ref_shift = (int)(q->bits >> 54 & 0x3ff) - (int)(q->bits >> 44 & 0x3ff);
			p->sa = q->k + (uint64_t)((double)w * erand48(r->rng));
		}
		cnt = (int)((uint64_t)(int64_t)cnt + w);
	}
	p->c1 = (uint32_t)((uint64_t)(int64_t)cnt & 0xfffffff);
	for (; i < n_aln; ++i) cnt = (int)((uint64_t)(int64_t)cnt + (aln[i].l - aln[i].k + 1));
	p->c2 = (uint32_t)(((uint64_t)(int64_t)cnt - p->c1) & 0xfffffff);
	p->type = p->c1 > 1 ? 2 : 1;
	if (r->n_occ) {
		int k, n_occ;
		for (k = n_occ = 0; k < n_aln; ++k) n_occ = (int)((uint64_t)(int64_t)n_occ + (aln[k].l - aln[k].k + 1));
		if (n_occ > r->n_occ + 1) return;   /* too many hits: none listed */
		/* all n_occ <= n_multi + 1 hits fit, so the reference's random sampling of a partly listed interval (bwase.c:78-89) is
		 * never reached: every interval is listed whole, in order */
		for (k = 0; k < n_aln; ++k) {
			const bwag_aln1_t *q = aln + k;
			uint64_t l;
			for (l = q->k; l <= q->l; ++l) {
				bwag_se_hit_t *h;
				if (g->n_multi == *m_multi) { *m_multi = *m_multi ? *m_multi << 1 : 1024; g->multi = bb_realloc(g->multi, sizeof(*g->multi) * (size_t)*m_multi); }
				h = &g->multi[g->n_multi++];
				memset(h, 0, sizeof(*h));
				h->sa = l;
				h->gap = (uint8_t)((q->bits >> 8 & 0xff) + (q->bits >> 16 & 0xff));
				h->ref_shift = (int)(q->bits >> 54 & 0x3ff) - (int)(q->bits >> 44 & 0x3ff);
				h->mm = (uint8_t)(q->bits & 0xff);
			}
			if (p->n_multi == 0) p->multi_beg = g->n_multi - (int64_t)(q->l - q->k + 1);
			p->n_multi += (int32_t)(q->l - q->k + 1);
		}
	}
}

/* bwa_approx_mapQ (bwase.c:101-110) with bwa_cal_pac_pos_core's max_diff (bwase.c:135) */
static int approx_mapq(const se_run_t *r, const bwag_se_read_t *p)
{
	const int mm = r->opt->fnr > 0.0 ? bb_cal_maxdiff(p->len, SE_AVG_ERR, r->opt->fnr) : r->opt->max_diff;
	int n;
	if (p->c1 == 0) return 23;
	if (p->c1 > 1) return 0;
	if (p->n_mm == mm) return 25;
	if (p->c2 == 0) return 37;
	n = p->c2 >= 255 ? 255 : (int)p->c2;
	return 23 < r->log_n[n] ? 0 : 23 - r->log_n[n];
}

/* the next group with its hits chosen; NULL at the end of the reads.  *eof: the .sai ended inside the group */
static se_group_t *read_group(se_run_t *r, int *eof)
{
	bb_reads_t *rd = bb_read_group(r->fq, r->opt->mode, r->opt->trim_qual, SE_GROUP, 1, SE_MAX_LEN, "bwa_sai2sam_se_core");
	se_group_t *g;
	int64_t m_multi = 0;
	int i;
	*eof = 0;
	if (!rd) return 0;
	g = bb_calloc(1, sizeof(*g));
	g->rd = rd;
	g->reads = bb_calloc((size_t)rd->n, sizeof(*g->reads));
	for (i = 0; i < rd->n; ++i) {
		bwag_se_read_t *p = &g->reads[i];
		int32_t n_aln;
		if (fread(&n_aln, 4, 1, r->fp_sa) != 1 || n_aln < 0) { *eof = 1; return g; }   /* a negative count is a huge size_t to the reference's fread */
		if (n_aln > r->m_aln) { r->m_aln = n_aln; r->aln = bb_realloc(r->aln, sizeof(*r->aln) * (size_t)n_aln); }
		if (n_aln > 0 && fread(r->aln, sizeof(*r->aln), (size_t)n_aln, r->fp_sa) != (size_t)n_aln) { *eof = 1; return g; }
		p->len = rd->len[i];
		p->clip_len = rd->len[i];
		p->l_bc = rd->bc[i] >= 0 ? (uint8_t)strlen(rd->text.s + rd->bc[i]) : 0;
		choose_hit(r, n_aln, r->aln, p, g, &m_multi);
		if (p->type) p->mapq = (uint8_t)approx_mapq(r, p);
	}
	return g;
}

/* reads [beg, end) of a group as a device batch */
static se_batch_t *slice(se_group_t *g, int beg, int end)
{
	se_batch_t *b = bb_calloc(1, sizeof(*b));
	const bb_reads_t *rd = g->rd;
	const int64_t b0 = rd->off[beg];
	int64_t m0 = -1, l_bc = 0;
	int i;
	b->g = g; b->beg = beg; b->n = end - beg;
	b->off = bb_malloc(8 * (size_t)(b->n + 1));
	for (i = 0; i <= b->n; ++i) b->off[i] = rd->off[beg + i] - b0;
	b->reads = bb_malloc(sizeof(*b->reads) * (size_t)(b->n + 1));
	memcpy(b->reads, g->reads + beg, sizeof(*b->reads) * (size_t)b->n);
	for (i = 0; i < b->n; ++i) {
		if (b->reads[i].n_multi && m0 < 0) m0 = b->reads[i].multi_beg;
		l_bc += b->reads[i].l_bc;
	}
	b->bc = bb_malloc((size_t)l_bc + 1);
	for (i = 0; i < b->n; ++i) {
		bwag_se_read_t *p = &b->reads[i];
		if (p->n_multi) p->multi_beg -= m0;
		p->bc_off = b->l_bc;
		if (p->l_bc) memcpy(b->bc + b->l_bc, rd->text.s + rd->bc[beg + i], p->l_bc);
		b->l_bc += p->l_bc;
	}
	return b;
}

static void *reader_main(void *arg)
{
	se_run_t *r = arg;
	for (;;) {
		int eof;
		double t0 = bb_realtime();
		se_group_t *g = read_group(r, &eof);
		r->t_read += bb_realtime() - t0;
		if (!g) break;
		if (eof) {   /* nothing of this group is printed */
			se_batch_t *b = bb_calloc(1, sizeof(*b));
			group_free(g);
			b->sai_eof = 1;
			bb_mbox_put(&r->to_dev, b);
			break;
		}
		/* the writer frees the group with its last batch: nothing of g may be touched once that batch is handed over */
		const int n = g->rd->n;
		for (int beg = 0; beg < n; beg += r->chunk) {
			const int end = beg + r->chunk < n ? beg + r->chunk : n;
			t0 = bb_realtime();
			se_batch_t *b = slice(g, beg, end);
			b->last = end == n;
			r->t_read += bb_realtime() - t0;
			bb_mbox_put(&r->to_dev, b);
		}
	}
	bb_mbox_put(&r->to_dev, 0);
	return 0;
}

/* per read: name + part A + QUAL (reversed on the reverse strand) + part B + "\n" */
static void write_batch(const se_batch_t *b)
{
	const bb_reads_t *rd = b->g->rd;
	bb_str_t s = {0, 0, 0};
	int i;
	for (i = 0; i < b->n; ++i) {
		const bwag_samrec_t *rec = &b->res.rec[i];
		const char *t = b->res.text + rec->off;
		const int r = b->beg + i;
		bb_puts(&s, rd->text.s + rd->name[r]);
		bb_putsn(&s, t, (size_t)rec->len_a);
		if (rd->qual[r] >= 0) {
			const int full_len = (int)(rd->off[r + 1] - rd->off[r]);
			const char *q = rd->text.s + rd->qual[r];
			bb_str_need(&s, (size_t)full_len);
			bb_copy_text(s.s + s.l, q, full_len, (rec->flags & BWAG_REC_QREV) != 0);
			s.l += full_len; s.s[s.l] = 0;
		} else bb_putc(&s, '*');
		bb_putsn(&s, t + rec->len_a, (size_t)rec->len_b);
		bb_putc(&s, '\n');
		if (s.l >= (1 << 20)) {
			if (fwrite(s.s, 1, s.l, stdout) != s.l) bb_fatal("bwa_sai2sam_se_core", "fail to write the output");
			s.l = 0;
		}
	}
	if (s.l && fwrite(s.s, 1, s.l, stdout) != s.l) bb_fatal("bwa_sai2sam_se_core", "fail to write the output");
	free(s.s);
}

static void *writer_main(void *arg)
{
	se_run_t *r = arg;
	se_batch_t *b;
	while ((b = bb_mbox_get(&r->to_write)) != 0) {
		double t0 = bb_realtime();
		if (b->sai_eof) r->sai_eof = 1;
		else if (!r->sai_eof) write_batch(b);
		batch_free(b);
		r->t_write += bb_realtime() - t0;
	}
	return 0;
}

int bb_samse_main(int argc, char *argv[])
{
	int c, n_occ = 3, i;
	char *rg_line = 0, magic[4];
	aln_opt_t opt;
	bwaidx_t *idx;
	bwag_ctx_t *ctx;
	se_run_t run;
	bwag_samse_par_t par;
	pthread_t th_r, th_w;
	double t0, t_load, t_dev = 0;
	long long n_sa = 0, n_glb = 0;
	const char *e;
	while ((c = getopt(argc, argv, "hn:f:r:")) >= 0) {   /* bwase.c:583-593 */
		switch (c) {
		case 'h': break;
		case 'r': if ((rg_line = bwa_set_rg(optarg)) == 0) return 1; break;
		case 'n': n_occ = atoi(optarg); break;
		case 'f': if (freopen(optarg, "w", stdout) == 0) bb_fatal("xreopen", "fail to open file '%s'", optarg); break;
		default: return 1;
		}
	}
	if (optind + 3 > argc) {
		fprintf(stderr, "Usage: bwa-b200 samse [-n max_occ] [-f out.sam] [-r RG_line] <prefix> <in.sai> <in.fq>\n");
		return 1;
	}
	memset(&run, 0, sizeof(run));
	t0 = bb_realtime();
	if ((idx = bb_idx_from_resident(argv[optind])) == 0 && (idx = bwa_idx_load(argv[optind], BWA_IDX_ALL)) == 0) {
		fprintf(stderr, "[bwa_sai2sam_se] fail to locate the index\n");
		free(rg_line);
		return 1;
	}
	ctx = bb_device_attach(idx->bwt, idx->bns, idx->pac);   /* fails here, before any output, if there is no GPU */
	{
		const bntseq_t *bns = idx->bns;
		int64_t *ao = bb_malloc(8 * (size_t)(bns->n_holes + 1));
		int32_t *al = bb_malloc(4 * (size_t)(bns->n_holes + 1));
		for (i = 0; i < bns->n_holes; ++i) ao[i] = bns->ambs[i].offset, al[i] = bns->ambs[i].len;
		if (bwag_ctx_set_ambs(ctx, bns->n_holes, ao, al) != 0) bb_fatal("bwa_sai2sam_se_core", "cannot place the reference's holes on the GPU: %s", bwag_last_error());
		free(ao); free(al);
	}
	t_load = bb_realtime() - t0;
	{   /* srand48(bns->seed) */
		const uint32_t seed = idx->bns->seed;
		run.rng[0] = 0x330e; run.rng[1] = (unsigned short)(seed & 0xffff); run.rng[2] = (unsigned short)(seed >> 16);
	}
	for (i = 1; i != 256; ++i) run.log_n[i] = (int)(4.343 * log(i) + 0.5);
	if (strcmp(argv[optind + 1], "-") == 0) run.fp_sa = stdin;
	else if ((run.fp_sa = fopen(argv[optind + 1], "r")) == 0) bb_fatal("xopen", "fail to open file '%s'", argv[optind + 1]);
	if (fread(magic, 1, 4, run.fp_sa) != 4) bb_fatal("fread", "Unexpected end of file");
	if (strncmp(magic, "SAI\1", 4) != 0) {
		fprintf(stderr, "[E::%s] Unmatched SAI magic. Please re-run `aln' with the same version of bwa.\n", "bwa_sai2sam_se_core");
		exit(1);
	}
	if (fread(&opt, sizeof(opt), 1, run.fp_sa) != 1) bb_fatal("fread", "Unexpected end of file");
	if (opt.mode & BB_MODE_BAM) bb_fatal("bwa_sai2sam_se_core", "the .sai file was made from BAM input (`aln -b`), which is not supported: convert the reads to FASTQ");
	bwa_print_sam_hdr(idx->bns, rg_line);
	if ((run.fq = bb_fq_open(argv[optind + 2])) == 0) bb_fatal("xzopen", "fail to open file '%s'", argv[optind + 2]);
	run.opt = &opt;
	run.n_occ = n_occ;
	run.chunk = (e = getenv("BWA_B200_SAMSE_CHUNK")) != 0 && atoi(e) > 0 ? atoi(e) : SE_GROUP;   /* reads per device batch */
	memset(&par, 0, sizeof(par));
	par.mode = opt.mode & BWAG_SE_COMPREAD;
	par.max_top2 = opt.max_top2;
	par.rg_id = bwa_rg_id[0] ? bwa_rg_id : 0;

	bb_mbox_init(&run.to_dev); bb_mbox_init(&run.to_write);
	pthread_create(&th_r, 0, reader_main, &run);
	pthread_create(&th_w, 0, writer_main, &run);
	for (;;) {
		se_batch_t *b = bb_mbox_get(&run.to_dev);
		double t1 = bb_realtime();
		int rc, past_end;
		int64_t ns, ng;
		if (!b) break;
		if (!b->sai_eof) {
			if ((b->dev = bwag_batch_begin(ctx, b->n, b->g->rd->codes + b->g->rd->off[b->beg], b->off)) == 0) bb_fatal("bwa_sai2sam_se_core", "cannot start a device batch: %s", bwag_last_error());
			par.reads = b->reads;
			{   /* the batch's candidates: those of its reads, contiguous in the group's list */
				int64_t m0 = -1, m1 = 0;
				for (i = 0; i < b->n; ++i) {
					const bwag_se_read_t *p = &b->g->reads[b->beg + i];
					if (p->n_multi) { if (m0 < 0) m0 = p->multi_beg; m1 = p->multi_beg + p->n_multi; }
				}
				par.multi = m0 >= 0 ? b->g->multi + m0 : 0;
				par.n_multi = m0 >= 0 ? m1 - m0 : 0;
			}
			par.bc = b->bc; par.l_bc = b->l_bc;
			rc = bwag_samse(b->dev, &par, &b->res, &past_end, &ns, &ng);
			if (rc == BWAG_UNSUPPORTED) { fprintf(stderr, "[E::%s] this build has no device samse\n", "bwa_sai2sam_se_core"); exit(1); }
			if (past_end >= 0)
				bb_fatal("bwa_sai2sam_se_core", "read '%s': its gapped alignment runs past the end of the reference (the reference's `bwa samse` aborts here)",
				         b->g->rd->text.s + b->g->rd->name[b->beg + past_end]);
			if (rc != 0) bb_fatal("bwa_sai2sam_se_core", "device samse failed: %s", bwag_last_error());
			n_sa += ns; n_glb += ng;
		}
		t_dev += bb_realtime() - t1;
		bb_mbox_put(&run.to_write, b);
	}
	bb_mbox_put(&run.to_write, 0);
	pthread_join(th_r, 0);
	pthread_join(th_w, 0);
	if (fflush(stdout) != 0 || ferror(stdout)) bb_fatal("bwa_sai2sam_se_core", "fail to write the output");
	if (getenv("BWA_B200_PROFILE"))
		fprintf(stderr, "[prof] samse: index load %.3f s; busy time of the reader %.3f s, the device %.3f s, the writer %.3f s; %lld hits sent to bwt_sa; %lld global alignments; total %.3f s\n",
		        t_load, run.t_read, t_dev, run.t_write, n_sa, n_glb, bb_realtime() - t0);
	if (run.sai_eof) { fprintf(stderr, "[fread] Unexpected end of file\n"); exit(1); }   /* err_fread_noeof, the earlier groups printed */
	bb_fq_close(run.fq);
	if (run.fp_sa != stdin) fclose(run.fp_sa);
	free(run.aln); free(rg_line);
	bwa_idx_destroy(idx);
	return 0;
}
