/* bb_samse.c -- `bwa-b200 samse`: the single-end SAM of the reference's `bwa samse` (bwase.c:507-606) byte for byte, from a .sai
 * file of `bwa aln` or `bwa-b200 aln`, with the suffix-array lookups, the gapped refinement, MD/NM and the SAM text on the GPU
 * (bwag_samse, bwag_samse.cu).
 *
 * It runs on the pipeline of bb_util.h: the reader parses the reads as bwa_read_seq does (bb_read_group) in the reference's groups
 * of 262144 reads, reads the group's .sai records, chooses each read's hit and its XA candidates (bwa_aln2seq_core) and its mapping
 * quality (bwa_approx_mapQ), and cuts the group into device batches of BWA_B200_SAMSE_CHUNK reads.  The hit choice draws random
 * numbers in read order over the whole input, so it stays on the one reader thread, with the private erand48 state of
 * bb_aln2seq_t, and the batch size cannot change a byte.  A group's .sai records are read before any of its batches reaches the
 * writer: when the .sai ends early, the earlier groups are out, as in the reference, and the command fails with its message.
 * BWA_B200_PROFILE=1 reports the index load, the busy time of the three threads, the hits sent to the suffix array and the global
 * alignments.
 *
 * The parts of bwase.c that bwape.c calls too are here, as in the reference, and `sampe` uses them: the hit draw, the mapping
 * quality, their set-up, the upload of the reference's holes and the SAM splice. */
#include <unistd.h>
#include <math.h>
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
	int n, last;                   /* last: the group's final batch (the writer frees the group) */
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
	bb_aln2seq_t se;
	bwag_aln1_t *aln; int m_aln;
	int sai_eof;                   /* reader: the .sai ended inside a group, whose reads were not handed on */
	bwag_ctx_t *ctx;
	bwag_samse_par_t par;
	long long n_sa, n_glb;
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

/* ---- the parts of bwase.c that sampe uses too ---- */

void bb_aln2seq_init(bb_aln2seq_t *s, const bntseq_t *bns)
{
	const uint32_t seed = bns->seed;   /* srand48(bns->seed) */
	int i;
	s->rng[0] = 0x330e; s->rng[1] = (unsigned short)(seed & 0xffff); s->rng[2] = (unsigned short)(seed >> 16);
	s->log_n[0] = 0;
	for (i = 1; i != 256; ++i) s->log_n[i] = (int)(4.343 * log(i) + 0.5);
}

/* with the reference's integer widths: int counts, 28-bit c1/c2 */
void bb_choose_hit(bb_aln2seq_t *s, int n_aln, const bwag_aln1_t *aln, bb_hit_t *h)
{
	int i, cnt, best;
	if (n_aln == 0) { h->type = 0; h->c1 = h->c2 = 0; return; }
	best = (int)(aln[0].bits >> 24 & 0xfffff);
	for (i = cnt = 0; i < n_aln; ++i) {
		const bwag_aln1_t *q = aln + i;
		const uint64_t w = q->l - q->k + 1;
		if ((int)(q->bits >> 24 & 0xfffff) > best) break;
		if (erand48(s->rng) * (double)(w + (uint64_t)(int64_t)cnt) > (double)cnt) {
			h->n_mm = (uint8_t)(q->bits & 0xff); h->n_gapo = (uint8_t)(q->bits >> 8 & 0xff); h->n_gape = (uint8_t)(q->bits >> 16 & 0xff);
			h->ref_shift = (int)(q->bits >> 54 & 0x3ff) - (int)(q->bits >> 44 & 0x3ff);
			h->score = (int)(q->bits >> 24 & 0xfffff);
			h->sa = q->k + (uint64_t)((double)w * erand48(s->rng));
		}
		cnt = (int)((uint64_t)(int64_t)cnt + w);
	}
	h->c1 = (uint32_t)((uint64_t)(int64_t)cnt & 0xfffffff);
	for (; i < n_aln; ++i) cnt = (int)((uint64_t)(int64_t)cnt + (aln[i].l - aln[i].k + 1));
	h->c2 = (uint32_t)(((uint64_t)(int64_t)cnt - h->c1) & 0xfffffff);
	h->type = h->c1 > 1 ? 2 : 1;
}

/* with bwa_cal_pac_pos_core's max_diff (bwase.c:135) */
int bb_approx_mapq(const bb_aln2seq_t *s, const aln_opt_t *opt, int len, const bb_hit_t *h)
{
	const int mm = opt->fnr > 0.0 ? bb_cal_maxdiff(len, SE_AVG_ERR, opt->fnr) : opt->max_diff;
	int n;
	if (h->c1 == 0) return 23;
	if (h->c1 > 1) return 0;
	if (h->n_mm == mm) return 25;
	if (h->c2 == 0) return 37;
	n = h->c2 >= 255 ? 255 : (int)h->c2;
	return 23 < s->log_n[n] ? 0 : 23 - s->log_n[n];
}

void bb_upload_holes(bwag_ctx_t *ctx, const bntseq_t *bns, const char *who)
{
	int64_t *ao = bb_malloc(8 * (size_t)(bns->n_holes + 1));
	int32_t *al = bb_malloc(4 * (size_t)(bns->n_holes + 1));
	int i;
	for (i = 0; i < bns->n_holes; ++i) ao[i] = bns->ambs[i].offset, al[i] = bns->ambs[i].len;
	if (bwag_ctx_set_ambs(ctx, bns->n_holes, ao, al) != 0) bb_fatal(who, "cannot place the reference's holes on the GPU: %s", bwag_last_error());
	free(ao); free(al);
}

void bb_splice_sam(bb_str_t *s, const bb_reads_t *rd, int r, const bwag_samrec_t *rec, const char *text)
{
	const char *t = text + rec->off;
	bb_puts(s, rd->text.s + rd->name[r]);
	bb_putsn(s, t, (size_t)rec->len_a);
	if (rd->qual[r] >= 0) {
		const int full_len = (int)(rd->off[r + 1] - rd->off[r]);
		bb_str_need(s, (size_t)full_len);
		bb_copy_text(s->s + s->l, rd->text.s + rd->qual[r], full_len, (rec->flags & BWAG_REC_QREV) != 0);
		s->l += full_len; s->s[s->l] = 0;
	} else bb_putc(s, '*');
	bb_putsn(s, t + rec->len_a, (size_t)rec->len_b);
	bb_putc(s, '\n');
}

/* ---- samse ---- */

/* the XA candidates of bwa_aln2seq_core(n_aln, aln, p, 1, n_occ) (bwase.c:49-94): every hit, or none when there are too many */
static void list_multi(const se_run_t *r, int n_aln, const bwag_aln1_t *aln, bwag_se_read_t *p, se_group_t *g, int64_t *m_multi)
{
	int k, n_occ;
	for (k = n_occ = 0; k < n_aln; ++k) n_occ = (int)((uint64_t)(int64_t)n_occ + (aln[k].l - aln[k].k + 1));
	if (n_occ > r->n_occ + 1) return;
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

/* the next group with its hits chosen; NULL at the end of the reads.  r->sai_eof: the .sai ended inside the group */
static se_group_t *read_group(se_run_t *r)
{
	bb_reads_t *rd = bb_read_group(r->fq, r->opt->mode, r->opt->trim_qual, SE_GROUP, 1, SE_MAX_LEN, "bwa_sai2sam_se_core");
	se_group_t *g;
	int64_t m_multi = 0;
	int i;
	if (!rd) return 0;
	g = bb_calloc(1, sizeof(*g));
	g->rd = rd;
	g->reads = bb_calloc((size_t)rd->n, sizeof(*g->reads));
	for (i = 0; i < rd->n; ++i) {
		bwag_se_read_t *p = &g->reads[i];
		bb_hit_t h = {0};
		int32_t n_aln;
		if (fread(&n_aln, 4, 1, r->fp_sa) != 1 || n_aln < 0) { r->sai_eof = 1; return g; }   /* a negative count is a huge size_t to the reference's fread */
		if (n_aln > r->m_aln) { r->m_aln = n_aln; r->aln = bb_realloc(r->aln, sizeof(*r->aln) * (size_t)n_aln); }
		if (n_aln > 0 && fread(r->aln, sizeof(*r->aln), (size_t)n_aln, r->fp_sa) != (size_t)n_aln) { r->sai_eof = 1; return g; }
		p->len = rd->len[i];
		p->clip_len = rd->len[i];
		p->l_bc = rd->bc[i] >= 0 ? (uint8_t)strlen(rd->text.s + rd->bc[i]) : 0;
		bb_choose_hit(&r->se, n_aln, r->aln, &h);
		p->sa = h.sa; p->ref_shift = h.ref_shift; p->type = h.type; p->n_mm = h.n_mm; p->n_gapo = h.n_gapo; p->n_gape = h.n_gape;
		p->c1 = h.c1; p->c2 = h.c2;
		if (r->n_occ && n_aln) list_multi(r, n_aln, r->aln, p, g, &m_multi);
		if (p->type) p->mapq = (uint8_t)bb_approx_mapq(&r->se, r->opt, p->len, &h);
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

static void read_all(bb_pipe_t *p, void *run)
{
	se_run_t *r = run;
	se_group_t *g;
	while ((g = read_group(r)) != 0) {
		if (r->sai_eof) { group_free(g); return; }   /* nothing of this group is printed */
		/* the writer frees the group with its last batch: nothing of g may be touched once that batch is handed over */
		const int n = g->rd->n;
		for (int beg = 0; beg < n; beg += r->chunk) {
			const int end = beg + r->chunk < n ? beg + r->chunk : n;
			se_batch_t *b = slice(g, beg, end);
			b->last = end == n;
			bb_pipe_to_device(p, b);
		}
	}
}

static void run_device(bb_pipe_t *p, void *run, void *item)
{
	se_run_t *r = run;
	se_batch_t *b = item;
	bwag_samse_par_t *par = &r->par;
	int rc, past_end, i;
	int64_t ns, ng, m0 = -1, m1 = 0;
	if ((b->dev = bwag_batch_begin(r->ctx, b->n, b->g->rd->codes + b->g->rd->off[b->beg], b->off)) == 0) bb_fatal("bwa_sai2sam_se_core", "cannot start a device batch: %s", bwag_last_error());
	par->reads = b->reads;
	for (i = 0; i < b->n; ++i) {   /* the batch's candidates: those of its reads, contiguous in the group's list */
		const bwag_se_read_t *q = &b->g->reads[b->beg + i];
		if (q->n_multi) { if (m0 < 0) m0 = q->multi_beg; m1 = q->multi_beg + q->n_multi; }
	}
	par->multi = m0 >= 0 ? b->g->multi + m0 : 0;
	par->n_multi = m0 >= 0 ? m1 - m0 : 0;
	par->bc = b->bc; par->l_bc = b->l_bc;
	rc = bwag_samse(b->dev, par, &b->res, &past_end, &ns, &ng);
	if (rc == BWAG_UNSUPPORTED) { fprintf(stderr, "[E::%s] this build has no device samse\n", "bwa_sai2sam_se_core"); exit(1); }
	if (past_end >= 0)
		bb_fatal("bwa_sai2sam_se_core", "read '%s': its gapped alignment runs past the end of the reference (the reference's `bwa samse` aborts here)",
		         b->g->rd->text.s + b->g->rd->name[b->beg + past_end]);
	if (rc != 0) bb_fatal("bwa_sai2sam_se_core", "device samse failed: %s", bwag_last_error());
	r->n_sa += ns; r->n_glb += ng;
	bb_pipe_to_writer(p, b);
}

static void write_batch(void *run, void *item)
{
	se_batch_t *b = item;
	bb_str_t s = {0, 0, 0};
	int i;
	(void)run;
	for (i = 0; i < b->n; ++i) {
		bb_splice_sam(&s, b->g->rd, b->beg + i, &b->res.rec[i], b->res.text);
		bb_str_write(&s, 1 << 20, "bwa_sai2sam_se_core");
	}
	bb_str_write(&s, 0, "bwa_sai2sam_se_core");
	batch_free(b);
}

static const bb_pipe_ops_t ops = { read_all, run_device, write_batch };

int bb_samse_main(int argc, char *argv[])
{
	int c, n_occ = 3;
	char *rg_line = 0, magic[4];
	aln_opt_t opt;
	bwaidx_t *idx;
	se_run_t run;
	bb_pipe_busy_t busy;
	double t0, t_load;
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
	run.ctx = bb_device_attach(idx->bwt, idx->bns, idx->pac);   /* fails here, before any output, if there is no GPU */
	bb_upload_holes(run.ctx, idx->bns, "bwa_sai2sam_se_core");
	t_load = bb_realtime() - t0;
	bb_aln2seq_init(&run.se, idx->bns);
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
	run.par.mode = opt.mode & BWAG_SE_COMPREAD;
	run.par.max_top2 = opt.max_top2;
	run.par.rg_id = bwa_rg_id[0] ? bwa_rg_id : 0;
	bb_pipe_run(&ops, &run, &busy);
	if (fflush(stdout) != 0 || ferror(stdout)) bb_fatal("bwa_sai2sam_se_core", "fail to write the output");
	if (getenv("BWA_B200_PROFILE"))
		fprintf(stderr, "[prof] samse: index load %.3f s; busy time of the reader %.3f s, the device %.3f s, the writer %.3f s; %lld hits sent to bwt_sa; %lld global alignments; total %.3f s\n",
		        t_load, busy.read, busy.device, busy.write, run.n_sa, run.n_glb, bb_realtime() - t0);
	if (run.sai_eof) { fprintf(stderr, "[fread] Unexpected end of file\n"); exit(1); }   /* err_fread_noeof, the earlier groups printed */
	bb_fq_close(run.fq);
	if (run.fp_sa != stdin) fclose(run.fp_sa);
	free(run.aln); free(rg_line);
	bwa_idx_destroy(idx);
	return 0;
}
