/* bb_sampe.c -- `bwa-b200 sampe`: the paired-end SAM of the reference's `bwa sampe` (bwape.c:260-784) byte for byte, from the two
 * .sai files of `bwa aln` or `bwa-b200 aln`, with the suffix-array lookups, the mate rescue's alignments, the gapped refinement,
 * MD/NM and the SAM text on the GPU (bwag_pe_sa2pos, bwag_localsw, bwag_pe_global, bwag_sampe; bwag_sampe.cu).
 *
 * It runs on the pipeline of bb_util.h: the reader parses the two read files (bb_read_group, file 1 with the mode and trimming of
 * .sai 1, file 2 with those of .sai 2) in the reference's groups of 262144 pairs, reads the two .sai files pair by pair and chooses
 * each read's hit and single-end mapping quality with samse's bwa_aln2seq_core and bwa_approx_mapQ (bb_samse.c); the device stage
 * runs a group and cuts it into writer batches.  Per group:
 *   P1  the chosen hits' positions (bwag_pe_sa2pos), then the insert-size model (infer_isize, host libm, with last_ii and -A);
 *   P2  per batch of BWA_B200_SAMPE_CHUNK pairs, cut further by a budget of rows: every row of every interval the pairing or XA can
 *       need, resolved once, with bwa_sa2pos for both reference lengths; the pairing (pairing(), bwape.c:156-254) and the XA
 *       choice (bwape.c:370-388) on the host;
 *   P5  the mate rescue (bwa_paired_sw, bwape.c:496-622): windows and early-outs here, the local alignments on K6 and the global
 *       ones on the device, the acceptance tests here;
 *   P6  refinement, MD/NM, the trimming correction and the records on the device (bwag_sampe); the writer splices name and QUAL.
 * Everything from .sai 2's gap_opt_t except the reading of file 1, because the reference overwrites its opt (bwape.c:661).
 * BWA_B200_PROFILE=1 reports the index load, the busy time of the three threads and the work of each step. */
#include <unistd.h>
#include <math.h>
#include "bb_host.h"

#define PE_GROUP    0x40000       /* pairs per bwa_read_seq call (bwape.c:675) */
#define PE_MAX_LEN  (1 << 20)
#define PE_ROWS     ((int64_t)1 << 22)   /* rows resolved per device call (P2): 34 bytes each on the device */
#define SW_MIN_MATCH_LEN 20
#define SW_MIN_MAPQ 17
#define F_PD  1                   /* SAM_FPD, SAM_FPP, SAM_FR1, SAM_FR2 */
#define F_PP  2
#define F_R1  0x40
#define F_R2  0x80
#define WHO "bwa_sai2sam_pe_core"

typedef struct { double avg, std, ap_prior; uint64_t low, high, high_bayesian; } isize_info_t;
typedef struct { long long n_rows, n_sorted, n_local, n_global, n_refine; double t_pair, t_sw, t_dev_calls; } pe_work_t;

typedef struct {                  /* one end as bwa_seq_t keeps it */
	uint64_t sa, pos;
	int len, ref_shift, score;
	uint32_t c1, c2;
	uint8_t type, strand, n_mm, n_gapo, n_gape, mapq, seq_q, flag;
	int64_t aln_beg; int n_aln;   /* its .sai records in the group's pool */
	int n_multi; int64_t multi_beg;   /* XA: the batch's lists */
	int64_t cig_off; int n_cig;   /* mate rescue: its CIGAR in the batch's list */
} pe_end_t;

typedef struct {
	bb_reads_t *rd[2];
	int n;                        /* pairs */
	pe_end_t *e;                  /* [2n]: pair i = e[2i], e[2i + 1] */
	bwag_aln1_t *aln; int64_t n_aln, m_aln;
	char *bc; int64_t *bc_off; int *l_bc;   /* each pair's barcode: both reads' barcodes concatenated (bwape.c:703-706) */
	int last;                     /* file 2 ended inside this group: the reference prints nothing after it */
} pe_group_t;

typedef struct {
	pe_group_t *g; int beg, n, last_of_group;
	bwag_batch_t *dev;
	bwag_sam_t res;
} pe_batch_t;

typedef struct {
	bb_fq_t *fq[2];
	FILE *fp_sa[2];
	aln_opt_t opt[2];
	int max_isize, max_occ, n_multi, N_multi, is_sw, force_isize, chunk;
	double ap_prior;
	bb_aln2seq_t se;
	/* reader: a .sai file ended inside a group, or a group cannot be printed (the message); the reader stops there and the command
	 * fails once the earlier groups are out */
	int sai_eof; char *err;
	char *bad_names;              /* writer: the message of the first pair with different names; nothing is printed after it */
	int no_device;                /* device stage: this build has no device sampe; the groups the reader still hands on are dropped */
	bwag_ctx_t *ctx;
	const bwaidx_t *idx;
	isize_info_t last_ii;
	pe_work_t work;
} pe_run_t;

static void group_free(pe_group_t *g)
{
	if (!g) return;
	bb_reads_free(g->rd[0]); bb_reads_free(g->rd[1]);
	free(g->e); free(g->aln); free(g->bc); free(g->bc_off); free(g->l_bc);
	free(g);
}

static char *xstrdup_printf(const char *fmt, const char *a, const char *b)
{
	const size_t l = strlen(fmt) + strlen(a) + (b ? strlen(b) : 0) + 1;
	char *s = bb_malloc(l);
	snprintf(s, l, fmt, a, b ? b : "");
	return s;
}

/* the next group with its hits chosen; NULL at the end of file 1.  r->sai_eof or r->err: the group cannot be printed */
static pe_group_t *read_group(pe_run_t *r)
{
	bb_reads_t *rd0 = bb_read_group(r->fq[0], r->opt[0].mode, r->opt[0].trim_qual, PE_GROUP, 1, PE_MAX_LEN, WHO), *rd1;
	pe_group_t *g;
	int i;
	if (!rd0) return 0;
	rd1 = bb_read_group(r->fq[1], r->opt[1].mode, r->opt[1].trim_qual, PE_GROUP, 1, PE_MAX_LEN, WHO);
	g = bb_calloc(1, sizeof(*g));
	g->rd[0] = rd0; g->rd[1] = rd1;
	g->n = rd1 ? rd1->n : 0;   /* the reference's n_seqs is file 2's count (bwape.c:680) */
	if (g->n > rd0->n) {       /* the reference reads past its array of file-1 reads here */
		char a[32];
		snprintf(a, sizeof(a), "%d", rd0->n);
		r->err = xstrdup_printf("the first read file has fewer reads than the second (%s pairs in its last group)%s", a, 0);
		return g;
	}
	if (g->n < rd0->n) g->last = 1;
	g->e = bb_calloc((size_t)2 * g->n + 1, sizeof(*g->e));
	g->bc_off = bb_calloc((size_t)g->n + 1, 8); g->l_bc = bb_calloc((size_t)g->n + 1, sizeof(int));
	{
		bb_str_t bc = {0, 0, 0};
		for (i = 0; i < g->n; ++i) {
			const char *b0 = rd0->bc[i] >= 0 ? rd0->text.s + rd0->bc[i] : "", *b1 = rd1->bc[i] >= 0 ? rd1->text.s + rd1->bc[i] : "";
			const int l = (int)(strlen(b0) + strlen(b1));
			if (l > BB_MAX_BCLEN) {
				r->err = xstrdup_printf("pair '%s': its two barcodes together are longer than 63 bases%s", rd0->text.s + rd0->name[i], 0);
				free(bc.s);
				return g;
			}
			g->bc_off[i] = (int64_t)bc.l; g->l_bc[i] = l;
			bb_puts(&bc, b0); bb_puts(&bc, b1);
		}
		g->bc = bc.s;
	}
	for (i = 0; i < g->n; ++i) {
		int j;
		for (j = 0; j < 2; ++j) {
			pe_end_t *p = &g->e[2 * i + j];
			bb_hit_t h = {0};
			int32_t n_aln;
			if (fread(&n_aln, 4, 1, r->fp_sa[j]) != 1 || n_aln < 0) { r->sai_eof = 1; return g; }
			if (g->n_aln + n_aln > g->m_aln) {
				while (g->n_aln + n_aln > g->m_aln) g->m_aln = g->m_aln ? g->m_aln << 1 : 4096;
				g->aln = bb_realloc(g->aln, sizeof(*g->aln) * (size_t)g->m_aln);
			}
			if (n_aln > 0 && fread(g->aln + g->n_aln, sizeof(*g->aln), (size_t)n_aln, r->fp_sa[j]) != (size_t)n_aln) { r->sai_eof = 1; return g; }
			p->aln_beg = g->n_aln; p->n_aln = n_aln; g->n_aln += n_aln;
			p->len = g->rd[j]->len[i];
			p->flag = F_PD | (j == 0 ? F_R1 : F_R2);
			bb_choose_hit(&r->se, n_aln, g->aln + p->aln_beg, &h);
			p->sa = h.sa; p->ref_shift = h.ref_shift; p->score = h.score; p->c1 = h.c1; p->c2 = h.c2;
			p->type = h.type; p->n_mm = h.n_mm; p->n_gapo = h.n_gapo; p->n_gape = h.n_gape;
			if (p->type) p->seq_q = p->mapq = (uint8_t)bb_approx_mapq(&r->se, &r->opt[1], p->len, &h);
		}
	}
	return g;
}

static void read_all(bb_pipe_t *p, void *run)
{
	pe_run_t *r = run;
	pe_group_t *g;
	while ((g = read_group(r)) != 0) {
		if (r->sai_eof || r->err) { group_free(g); return; }   /* nothing of this group is printed */
		const int last = g->last;   /* read before the hand-over: the other threads may free g at once */
		bb_pipe_to_device(p, g);
		if (last) return;
	}
}

/* ---------------------------------------------------------------- insert size (infer_isize, bwape.c:81-154) */

static int cmp_u64(const void *a, const void *b) { const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b; return x < y ? -1 : x > y; }

static int infer_isize(const pe_group_t *g, isize_info_t *ii, double ap_prior, int64_t L)
{
	uint64_t x, *isizes, n_ap = 0;
	int n, i, tot, p25, p75, p50, max_len = 1, tmp;
	double skewness = 0.0, kurtosis = 0.0, y;
	ii->avg = ii->std = -1.0;
	ii->low = ii->high = ii->high_bayesian = 0;
	isizes = bb_calloc((size_t)g->n + 1, 8);
	for (i = 0, tot = 0; i != g->n; ++i) {
		const pe_end_t *p0 = &g->e[2 * i], *p1 = &g->e[2 * i + 1];
		if (p0->mapq >= 20 && p1->mapq >= 20) {
			x = p0->pos < p1->pos ? p1->pos + (uint64_t)(int64_t)p1->len - p0->pos : p0->pos + (uint64_t)(int64_t)p0->len - p1->pos;
			if (x < 100000) isizes[tot++] = x;
		}
		if (p0->len > max_len) max_len = p0->len;
		if (p1->len > max_len) max_len = p1->len;
	}
	if (tot < 20) {
		fprintf(stderr, "[infer_isize] fail to infer insert size: too few good pairs\n");
		free(isizes);
		return -1;
	}
	qsort(isizes, (size_t)tot, 8, cmp_u64);
	p25 = (int)isizes[(int)(tot * 0.25 + 0.5)];
	p50 = (int)isizes[(int)(tot * 0.50 + 0.5)];
	p75 = (int)isizes[(int)(tot * 0.75 + 0.5)];
	tmp = (int)(p25 - 2.0 * (p75 - p25) + .499);
	ii->low = (uint64_t)(int64_t)(tmp > max_len ? tmp : max_len);
	ii->high = (uint64_t)(int64_t)(int)(p75 + 2.0 * (p75 - p25) + .499);
	if (ii->low > ii->high) {
		fprintf(stderr, "[infer_isize] fail to infer insert size: upper bound is smaller than read length\n");
		free(isizes);
		return -1;
	}
	for (i = 0, x = n = 0; i < tot; ++i)
		if (isizes[i] >= ii->low && isizes[i] <= ii->high) ++n, x += isizes[i];
	ii->avg = (double)x / n;
	for (i = 0; i < tot; ++i) {
		if (isizes[i] >= ii->low && isizes[i] <= ii->high) {
			double t = (isizes[i] - ii->avg) * (isizes[i] - ii->avg);
			ii->std += t;
			skewness += t * (isizes[i] - ii->avg);
			kurtosis += t * t;
		}
	}
	kurtosis = kurtosis / n / (ii->std / n * ii->std / n) - 3;
	ii->std = sqrt(ii->std / n);
	skewness = skewness / n / (ii->std * ii->std * ii->std);
	for (y = 1.0; y < 10.0; y += 0.01)
		if (.5 * erfc(y / M_SQRT2) < ap_prior / L * (y * ii->std + ii->avg)) break;
	ii->high_bayesian = (uint64_t)(y * ii->std + ii->avg + .499);
	for (i = 0; i < tot; ++i)
		if (isizes[i] > ii->high_bayesian) ++n_ap;
	ii->ap_prior = .01 * (n_ap + .01) / tot;
	if (ii->ap_prior < ap_prior) ii->ap_prior = ap_prior;
	free(isizes);
	fprintf(stderr, "[infer_isize] (25, 50, 75) percentile: (%d, %d, %d)\n", p25, p50, p75);
	if (isnan(ii->std) || p75 > 100000) {
		ii->low = ii->high = ii->high_bayesian = 0; ii->avg = ii->std = -1.0;
		fprintf(stderr, "[infer_isize] fail to infer insert size: weird pairing\n");
		return -1;
	}
	for (y = 1.0; y < 10.0; y += 0.01)
		if (.5 * erfc(y / M_SQRT2) < ap_prior / L * (y * ii->std + ii->avg)) break;
	ii->high_bayesian = (uint64_t)(y * ii->std + ii->avg + .499);
	fprintf(stderr, "[infer_isize] low and high boundaries: %ld and %ld for estimating avg and std\n", (long)ii->low, (long)ii->high);
	fprintf(stderr, "[infer_isize] inferred external isize from %d pairs: %.3lf +/- %.3lf\n", n, ii->avg, ii->std);
	fprintf(stderr, "[infer_isize] skewness: %.3lf; kurtosis: %.3lf; ap_prior: %.2e\n", skewness, kurtosis, ii->ap_prior);
	fprintf(stderr, "[infer_isize] inferred maximum insert size: %ld (%.2lf sigma)\n", (long)ii->high_bayesian, y);
	return 0;
}

/* ---------------------------------------------------------------- pairing (bwape.c:156-254) */

typedef struct { uint64_t x, y; } pair64_t;

static int cmp_pair64(const void *a, const void *b)
{
	const pair64_t *u = a, *v = b;
	if (u->x != v->x) return u->x < v->x ? -1 : 1;
	return u->y < v->y ? -1 : u->y > v->y;
}

static inline uint64_t hash_64(uint64_t key)
{
	key += ~(key << 32); key ^= (key >> 22); key += ~(key << 13); key ^= (key >> 8);
	key += (key << 3); key ^= (key >> 15); key += ~(key << 27); key ^= (key >> 31);
	return key;
}

typedef struct {                  /* one call of pairing() */
	pe_end_t *p[2];
	const bwag_aln1_t *aln[2];
	const pe_run_t *r;
	const isize_info_t *ii;
	int max_len, o_n, subo_n;
	uint64_t o_score, subo_score;
	pair64_t o_pos[2];
} pairing_t;

static inline int aln_score(const bwag_aln1_t *a) { return (int)(a->bits >> 24 & 0xfffff); }

static void pairing_aux(pairing_t *s, pair64_t u, pair64_t v)
{
	const uint64_t l = v.x + (uint64_t)(int64_t)s->p[v.y & 1]->len - u.x;
	const isize_info_t *ii = s->ii;
	if (u.x != (uint64_t)-1 && v.x > u.x && l >= (uint64_t)(int64_t)s->max_len
	    && ((ii->high && l <= ii->high_bayesian) || (ii->high == 0 && l <= (uint64_t)(int64_t)s->r->max_isize))) {
		uint64_t sc = (uint64_t)(int64_t)aln_score(s->aln[v.y & 1] + (v.y >> 2)) + (uint64_t)(int64_t)aln_score(s->aln[u.y & 1] + (u.y >> 2));
		sc *= 10;
		if (ii->high) sc += (uint64_t)(int64_t)(int)(-4.343 * log(.5 * erfc(M_SQRT1_2 * fabs(l - ii->avg) / ii->std)) + .499);
		sc = sc << 32 | (uint32_t)hash_64(u.x << 32 | v.x);
		if (sc >> 32 == s->o_score >> 32) ++s->o_n;
		else if (sc >> 32 < s->o_score >> 32) { s->subo_n += s->o_n; s->o_n = 1; }
		else ++s->subo_n;
		if (sc < s->o_score) s->subo_score = s->o_score, s->o_score = sc, s->o_pos[u.y & 1] = u, s->o_pos[v.y & 1] = v;
		else if (sc < s->subo_score) s->subo_score = sc;
	}
}

static int pairing_aux2(pe_end_t *q, const bwag_aln1_t *aln, pair64_t w)
{
	const bwag_aln1_t *a = aln + (w.y >> 2);
	q->flag |= F_PP;
	if (q->pos != w.x || q->strand != (w.y >> 1 & 1)) {
		q->n_mm = (uint8_t)(a->bits & 0xff); q->n_gapo = (uint8_t)(a->bits >> 8 & 0xff); q->n_gape = (uint8_t)(a->bits >> 16 & 0xff);
		q->strand = (uint8_t)(w.y >> 1 & 1);
		q->score = aln_score(a);
		q->pos = w.x;
		return q->mapq > 0;
	}
	return 0;
}

/* arr: the pairing candidates of both ends (sorted here); returns the ends that moved with a non-zero mapping quality */
static int pairing(const pe_run_t *r, pe_end_t *p[2], const int full_len[2], const bwag_aln1_t *aln[2], pair64_t *arr, int64_t n_arr, const isize_info_t *ii)
{
	pairing_t s;
	pair64_t last_pos[2][2];
	int64_t i;
	int j, cnt_chg = 0;
	memset(&s, 0, sizeof(s));
	s.p[0] = p[0]; s.p[1] = p[1]; s.aln[0] = aln[0]; s.aln[1] = aln[1]; s.r = r; s.ii = ii;
	s.max_len = full_len[0] > full_len[1] ? full_len[0] : full_len[1];
	s.o_score = s.subo_score = (uint64_t)-1;
	qsort(arr, (size_t)n_arr, sizeof(*arr), cmp_pair64);   /* equal records are identical: any correct sort gives the reference's order */
	for (j = 0; j < 2; ++j) last_pos[j][0].x = last_pos[j][0].y = last_pos[j][1].x = last_pos[j][1].y = (uint64_t)-1;
	for (i = 0; i < n_arr; ++i) {
		const pair64_t x = arr[i];
		if (x.y >> 1 & 1) {   /* reverse strand: check */
			const int y = 1 - (int)(x.y & 1);
			pairing_aux(&s, last_pos[y][1], x);
			pairing_aux(&s, last_pos[y][0], x);
		} else {              /* forward strand: push */
			last_pos[x.y & 1][0] = last_pos[x.y & 1][1];
			last_pos[x.y & 1][1] = x;
		}
	}
	if (s.o_score != (uint64_t)-1) {
		int mapq_p = 0;
		const int same0 = p[0]->pos == s.o_pos[0].x && p[0]->strand == (s.o_pos[0].y >> 1 & 1);
		const int same1 = p[1]->pos == s.o_pos[1].x && p[1]->strand == (s.o_pos[1].y >> 1 & 1);
		if (s.o_n == 1) {
			if (s.subo_score == (uint64_t)-1) mapq_p = 29;
			else if ((s.subo_score >> 32) - (s.o_score >> 32) > (uint64_t)(int64_t)(r->opt[1].s_mm * 10)) mapq_p = 23;
			else {
				const int n = s.subo_n > 255 ? 255 : s.subo_n;
				mapq_p = (int)(((s.subo_score >> 32) - (s.o_score >> 32)) / 2 - (uint64_t)(int64_t)r->se.log_n[n]);
				if (mapq_p < 0) mapq_p = 0;
			}
		}
		if (same0 && same1) {
			if (p[0]->mapq > 0 && p[1]->mapq > 0) {
				int q = p[0]->mapq + p[1]->mapq;
				if (q > 60) q = 60;
				p[0]->mapq = p[1]->mapq = (uint8_t)q;
			} else {
				if (p[0]->mapq == 0) p[0]->mapq = (uint8_t)(mapq_p + 7 < p[1]->mapq ? mapq_p + 7 : p[1]->mapq);
				if (p[1]->mapq == 0) p[1]->mapq = (uint8_t)(mapq_p + 7 < p[0]->mapq ? mapq_p + 7 : p[0]->mapq);
			}
		} else if (same0) {
			p[1]->seq_q = 0; p[1]->mapq = p[0]->mapq;
			if (p[1]->mapq > mapq_p) p[1]->mapq = (uint8_t)mapq_p;
		} else if (same1) {
			p[0]->seq_q = 0; p[0]->mapq = p[1]->mapq;
			if (p[0]->mapq > mapq_p) p[0]->mapq = (uint8_t)mapq_p;
		} else {
			p[0]->seq_q = p[1]->seq_q = 0;
			mapq_p -= 20;
			if (mapq_p < 0) mapq_p = 0;
			p[0]->mapq = p[1]->mapq = (uint8_t)mapq_p;
		}
		cnt_chg += pairing_aux2(p[0], aln[s.o_pos[0].y & 1], s.o_pos[0]);
		cnt_chg += pairing_aux2(p[1], aln[s.o_pos[1].y & 1], s.o_pos[1]);
	}
	return cnt_chg;
}

/* ---------------------------------------------------------------- one device batch */

typedef struct {                  /* what a batch builds for bwag_sampe */
	bwag_se_hit_t *multi; int64_t *mpos; uint8_t *mstrand; int64_t n_multi, m_multi;
	uint32_t *cig; int64_t n_cig, m_cig;
} pe_lists_t;


static void push_multi(pe_lists_t *L, const bwag_aln1_t *q, int64_t pos, int strand)
{
	if (L->n_multi == L->m_multi) {
		L->m_multi = L->m_multi ? L->m_multi << 1 : 1024;
		L->multi = bb_realloc(L->multi, sizeof(*L->multi) * (size_t)L->m_multi);
		L->mpos = bb_realloc(L->mpos, 8 * (size_t)L->m_multi);
		L->mstrand = bb_realloc(L->mstrand, (size_t)L->m_multi);
	}
	bwag_se_hit_t *h = &L->multi[L->n_multi];
	memset(h, 0, sizeof(*h));
	h->gap = (uint8_t)((q->bits >> 8 & 0xff) + (q->bits >> 16 & 0xff));
	h->mm = (uint8_t)(q->bits & 0xff);
	h->ref_shift = (int)(q->bits >> 54 & 0x3ff) - (int)(q->bits >> 44 & 0x3ff);
	L->mpos[L->n_multi] = pos; L->mstrand[L->n_multi] = (uint8_t)strand;
	++L->n_multi;
}

static int64_t n_occ_of(const pe_group_t *g, const pe_end_t *e)
{
	int64_t n = 0;
	for (int k = 0; k < e->n_aln; ++k) n += (int64_t)(g->aln[e->aln_beg + k].l - g->aln[e->aln_beg + k].k + 1);
	return n;
}

static inline int mapped_type(const pe_end_t *e) { return e->type == 1 || e->type == 2; }

/* P2: pairing and XA of pairs [beg, end) of the group */
static void pair_and_xa(pe_run_t *r, bwag_batch_t *b, pe_group_t *g, int beg, int end, const isize_info_t *ii, pe_lists_t *L, pe_work_t *w)
{
	const int xa = r->N_multi || r->n_multi, xa_max = r->n_multi > r->N_multi ? r->n_multi : r->N_multi;
	uint64_t *rows = 0; int32_t *rlen = 0; int64_t *pos = 0; uint8_t *str = 0; pair64_t *arr = 0;
	int64_t m_rows = 0, m_arr = 0;
	int s0 = beg;
	while (s0 < end) {   /* a slice of pairs whose rows fit the budget */
		int s1 = s0;
		int64_t n_rows = 0;
		for (; s1 < end; ++s1) {
			pe_end_t *e0 = &g->e[2 * s1], *e1 = e0 + 1;
			const int64_t o0 = n_occ_of(g, e0), o1 = n_occ_of(g, e1);
			const int both = mapped_type(e0) && mapped_type(e1), skip = both && (o0 > r->max_occ || o1 > r->max_occ);
			int64_t need = 0;
			if (!skip) for (int j = 0; j < 2; ++j) {
				const pe_end_t *e = e0 + j;
				const int64_t o = j ? o1 : o0;
				if (both || (e->type && xa && o <= (int64_t)xa_max + 1)) need += o;
			}
			if (s1 > s0 && n_rows + need > PE_ROWS) break;
			n_rows += need;
		}
		if (n_rows > m_rows) {
			m_rows = n_rows;
			rows = bb_realloc(rows, 8 * (size_t)m_rows); rlen = bb_realloc(rlen, 8 * (size_t)m_rows);
			pos = bb_realloc(pos, 16 * (size_t)m_rows); str = bb_realloc(str, 2 * (size_t)m_rows);
		}
		{   /* the rows, pair by pair, end by end, interval by interval */
			int64_t x = 0;
			for (int i = s0; i < s1; ++i) {
				pe_end_t *e0 = &g->e[2 * i], *e1 = e0 + 1;
				const int64_t o0 = n_occ_of(g, e0), o1 = n_occ_of(g, e1);
				const int both = mapped_type(e0) && mapped_type(e1), skip = both && (o0 > r->max_occ || o1 > r->max_occ);
				if (skip) continue;
				for (int j = 0; j < 2; ++j) {
					const pe_end_t *e = e0 + j;
					if (!(both || (e->type && xa && (j ? o1 : o0) <= (int64_t)xa_max + 1))) continue;
					for (int k = 0; k < e->n_aln; ++k) {
						const bwag_aln1_t *q = &g->aln[e->aln_beg + k];
						for (uint64_t l = q->k; l <= q->l; ++l) {
							rows[x] = l;
							rlen[2 * x] = e->len + e->ref_shift;
							rlen[2 * x + 1] = e->len + ((int)(q->bits >> 54 & 0x3ff) - (int)(q->bits >> 44 & 0x3ff));
							++x;
						}
					}
				}
			}
		}
		{
			const double t0 = bb_realtime();
			if (n_rows && bwag_pe_sa2pos(b, n_rows, rows, rlen, pos, str) != 0) bb_fatal(WHO, "device suffix-array lookup failed: %s", bwag_last_error());
			w->t_dev_calls += bb_realtime() - t0;
		}
		w->n_rows += n_rows;
		{   /* pairing, then XA, in pair order */
			int64_t x = 0;
			for (int i = s0; i < s1; ++i) {
				pe_end_t *p[2] = { &g->e[2 * i], &g->e[2 * i + 1] };
				const int64_t o[2] = { n_occ_of(g, p[0]), n_occ_of(g, p[1]) };
				const int both = mapped_type(p[0]) && mapped_type(p[1]), skip = both && (o[0] > r->max_occ || o[1] > r->max_occ);
				int64_t row0[2] = { -1, -1 };
				if (skip) continue;   /* bwape.c:331: no pairing and no XA for either end */
				for (int j = 0; j < 2; ++j)
					if (both || (p[j]->type && xa && o[j] <= (int64_t)xa_max + 1)) { row0[j] = x; x += o[j]; }
				if (both) {
					const bwag_aln1_t *aln[2] = { g->aln + p[0]->aln_beg, g->aln + p[1]->aln_beg };
					const int full_len[2] = { (int)(g->rd[0]->off[i + 1] - g->rd[0]->off[i]), (int)(g->rd[1]->off[i + 1] - g->rd[1]->off[i]) };
					int64_t n_arr = 0;
					if (o[0] + o[1] > m_arr) { m_arr = o[0] + o[1]; arr = bb_realloc(arr, sizeof(*arr) * (size_t)m_arr); }
					for (int j = 0; j < 2; ++j) {
						int64_t y = row0[j];
						for (int k = 0; k < p[j]->n_aln; ++k)
							for (uint64_t l = aln[j][k].k; l <= aln[j][k].l; ++l, ++y) {
								arr[n_arr].x = (uint64_t)pos[2 * y];
								arr[n_arr].y = (uint64_t)k << 2 | (uint64_t)str[2 * y] << 1 | (uint64_t)j;
								++n_arr;
							}
					}
					w->n_sorted += n_arr;
					pairing(r, p, full_len, aln, arr, n_arr, ii);
				}
				if (!xa) continue;
				for (int j = 0; j < 2; ++j) {
					int nm;
					if (p[j]->type == 0) continue;
					if (!(p[j]->flag & F_PP) && p[1 - j]->type != 0) nm = (int)(p[j]->c1 + p[j]->c2) - 1 > r->N_multi ? r->n_multi : r->N_multi;
					else nm = r->n_multi;
					if (!nm || o[j] > (int64_t)nm + 1) continue;   /* bwa_aln2seq_core(set_main = 0): all hits, or none */
					int64_t y = row0[j];
					p[j]->multi_beg = L->n_multi;
					for (int k = 0; k < p[j]->n_aln; ++k) {
						const bwag_aln1_t *q = g->aln + p[j]->aln_beg + k;
						for (uint64_t l = q->k; l <= q->l; ++l, ++y) {
							const int64_t qp = pos[2 * y + 1];
							if ((uint64_t)qp != p[j]->pos && qp != -1) push_multi(L, q, qp, str[2 * y + 1]);
						}
					}
					p[j]->n_multi = (int)(L->n_multi - p[j]->multi_beg);
				}
			}
		}
		s0 = s1;
	}
	free(rows); free(rlen); free(pos); free(str); free(arr);
}

/* P5: bwa_paired_sw (bwape.c:496-622) over pairs [beg, end) */
static void mate_sw(pe_run_t *r, bwag_batch_t *b, pe_group_t *g, int beg, int end, const isize_info_t *ii, int64_t l_pac, const uint8_t *pac, pe_lists_t *L, pe_work_t *w)
{
	typedef struct { int pair, k; int64_t beg, end; } sw_job_t;
	sw_job_t *jobs = 0; bwag_swtask_t *tasks = 0; bb_str_t pool = {0, 0, 0};
	int n_jobs = 0, m_jobs = 0, i, k;
	if (!r->is_sw || ii->avg < 0.0) return;
	for (i = beg; i < end; ++i) {
		pe_end_t *p[2] = { &g->e[2 * i], &g->e[2 * i + 1] };
		if (!((p[0]->mapq >= SW_MIN_MAPQ || p[1]->mapq >= SW_MIN_MAPQ) && (p[0]->flag & F_PP) == 0)) continue;
		for (k = 0; k < 2; ++k) {
			const pe_end_t *pref = p[1 - k], *pm = p[k];
			const bb_reads_t *rd = g->rd[k];
			const uint8_t *read = rd->codes + rd->off[i];
			const int comp = (r->opt[k].mode & BB_MODE_COMPREAD) != 0;   /* file k was read with .sai k's mode */
			int64_t a, bb;
			if (pref->type == 0) continue;
			if (pref->strand == 0) {   /* __set_rght_coor */
				a = (int64_t)((double)(int64_t)pref->pos + ii->avg - 3 * ii->std - pm->len * 1.5);
				bb = (int64_t)(a + 6 * ii->std + 2 * pm->len);
				if (a < (int64_t)pref->pos + pref->len) a = (int64_t)pref->pos + pref->len;
				if (bb > l_pac) bb = l_pac;
			} else {                   /* __set_left_coor */
				a = (int64_t)((double)((int64_t)pref->pos + pref->len) - ii->avg - 3 * ii->std - pm->len * 0.5);
				bb = (int64_t)(a + 6 * ii->std + 2 * pm->len);
				if (a < 0) a = 0;
				if ((uint64_t)bb > pref->pos) bb = (int64_t)pref->pos;
			}
			{   /* bwa_sw_core's early-outs (bwape.c:421-424) */
				const int reglen = (int)(bb - a), len = pm->len;
				int nn = 0;
				if (reglen < SW_MIN_MATCH_LEN || l_pac - a < len) continue;
				for (int x = 0; x < len; ++x) if (read[x] >= 4) ++nn;
				if ((float)nn / len >= 0.25 || len - nn < SW_MIN_MATCH_LEN) continue;
				if (n_jobs == m_jobs) { m_jobs = m_jobs ? m_jobs << 1 : 256; jobs = bb_realloc(jobs, sizeof(*jobs) * (size_t)m_jobs); tasks = bb_realloc(tasks, sizeof(*tasks) * (size_t)m_jobs); }
				jobs[n_jobs].pair = i; jobs[n_jobs].k = k; jobs[n_jobs].beg = a; jobs[n_jobs].end = bb;
				tasks[n_jobs].t_beg = a; tasks[n_jobs].tlen = reglen; tasks[n_jobs].q_beg = (int64_t)pool.l; tasks[n_jobs].qlen = len;
				tasks[n_jobs].xtra = BWAG_SW_XSUBO | BWAG_SW_XSTART | (len < 250 ? BWAG_SW_XBYTE : 0);
				tasks[n_jobs].flags = BWAG_SWF_TREF;
				bb_str_need(&pool, (size_t)len + 1);
				for (int x = 0; x < len; ++x) {   /* the anchor on the forward strand: rseq (reversed, complemented under COMPREAD); else seq */
					int c = pref->strand == 0 ? read[len - 1 - x] : read[x];
					if (c > 4) c = 4;
					if (pref->strand == 0 && comp && c < 4) c = 3 - c;
					pool.s[pool.l + x] = (char)c;
				}
				pool.l += (size_t)len;
				++n_jobs;
			}
		}
	}
	{
		const bwag_swres_t *sr = 0;
		bwag_pe_gtask_t *gt = bb_calloc((size_t)n_jobs + 1, sizeof(*gt));
		int *gi = bb_malloc(sizeof(int) * ((size_t)n_jobs + 1)), n_gt = 0;
		const bwag_pe_gres_t *gr = 0; const uint32_t *gc = 0;
		uint32_t *cnt = bb_calloc((size_t)n_jobs + 1, 4);
		int64_t *cig_of = bb_malloc(8 * ((size_t)n_jobs + 1)); int *ncig_of = bb_calloc((size_t)n_jobs + 1, sizeof(int));
		if (n_jobs) {
			bwag_sw_par_t sp;
			memset(&sp, 0, sizeof(sp));
			sp.a = 1; sp.b = 3; sp.o_del = sp.o_ins = 5; sp.e_del = sp.e_ins = 1;
			for (i = 0; i < 25; ++i) sp.mat[i] = (int8_t)(i >= 20 || i % 5 == 4 ? -1 : i / 5 == i % 5 ? 1 : -3);   /* bwa_fill_scmat(1, 3) */
			const double t0 = bb_realtime();
			if (bwag_localsw(b, &sp, n_jobs, tasks, (const uint8_t *)pool.s, pool.l, &sr) != 0) bb_fatal(WHO, "device local alignment failed: %s", bwag_last_error());
			w->t_dev_calls += bb_realtime() - t0;
			w->n_local += n_jobs;
		}
		for (i = 0; i < n_jobs; ++i) {
			gi[i] = -1;
			if (sr[i].score < SW_MIN_MATCH_LEN || sr[i].score2 == sr[i].score) continue;
			if (sr[i].qb < 0 || sr[i].tb < 0) {   /* the reference runs ksw_global from before its buffers here */
				const bb_reads_t *rd = g->rd[jobs[i].k];
				bb_fatal(WHO, "read '%s': the start of its mate-rescue alignment cannot be recovered (the reference's `bwa sampe` reads before its buffers here)", rd->text.s + rd->name[jobs[i].pair]);
			}
			gi[i] = n_gt;
			gt[n_gt].q_beg = tasks[i].q_beg + sr[i].qb; gt[n_gt].qlen = sr[i].qe - sr[i].qb + 1;
			gt[n_gt].t_beg = jobs[i].beg + sr[i].tb; gt[n_gt].tlen = sr[i].te - sr[i].tb + 1;
			++n_gt;
		}
		{
			const double t0 = bb_realtime();
			if (n_gt && bwag_pe_global(b, n_gt, gt, (const uint8_t *)pool.s, pool.l, &gr, &gc) != 0) bb_fatal(WHO, "device global alignment failed: %s", bwag_last_error());
			w->t_dev_calls += bb_realtime() - t0;
		}
		w->n_global += n_gt;
		/* bwa_sw_core's checks and CIGAR (bwape.c:439-490) */
		for (i = 0; i < n_jobs; ++i) {
			const int t = gi[i], len = tasks[i].qlen;
			const uint8_t *seq = (const uint8_t *)pool.s + tasks[i].q_beg;
			uint64_t x, y;
			int n_cigar, n_mm = 0, n_gapo = 0, n_gape = 0;
			cig_of[i] = -1;
			if (t < 0 || gr[t].score != sr[i].score) continue;
			const uint32_t *c32 = gc + gr[t].cig_off;
			n_cigar = gr[t].n_cigar;
			for (k = 0, x = y = 0; k < n_cigar; ++k) {
				const int op = (int)(c32[k] & 0xf), l = (int)((uint16_t)(op << 14 | (c32[k] >> 4)) & 0x3fff);
				const int op16 = (int)((uint16_t)(op << 14 | (c32[k] >> 4)) >> 14 & 3);
				if (op16 == 0) x += (uint64_t)l, y += (uint64_t)l;
				else if (op16 == 2) x += (uint64_t)l;
				else y += (uint64_t)l;
			}
			if (x < SW_MIN_MATCH_LEN || y < SW_MIN_MATCH_LEN) continue;
			if (L->n_cig + n_cigar + 2 > L->m_cig) {
				while (L->n_cig + n_cigar + 2 > L->m_cig) L->m_cig = L->m_cig ? L->m_cig << 1 : 1024;
				L->cig = bb_realloc(L->cig, 4 * (size_t)L->m_cig);
			}
			{
				uint32_t *c = L->cig + L->n_cig;
				int n = 0;
				const int start = sr[i].qb, e1 = sr[i].qe + 1;
				if (start) c[n++] = (uint16_t)(3 << 14 | start);
				for (k = 0; k < n_cigar; ++k) c[n++] = (uint16_t)((c32[k] & 0xf) << 14 | (c32[k] >> 4));
				if (e1 < len) c[n++] = (uint16_t)(3 << 14 | (len - e1));
				cig_of[i] = L->n_cig; ncig_of[i] = n; L->n_cig += n;
				/* cnt: n_mm only where both bases are < 4, n_gapo and n_gape over I and D */
				{
					uint64_t rx = (uint64_t)sr[i].tb, qy = (uint64_t)sr[i].qb;
					const int64_t t0 = jobs[i].beg;
					for (k = 0; k < n; ++k) {
						const int op = (int)(c[k] >> 14 & 3), l = (int)(c[k] & 0x3fff);
						if (op == 0) {
							for (int z = 0; z < l; ++z) {
								const int64_t rp = t0 + (int64_t)(rx + z);
								const int rb = rp < l_pac ? pac[rp >> 2] >> ((~rp & 3) << 1) & 3 : 0, qb = seq[qy + z];
								if (rb < 4 && qb < 4 && rb != qb) ++n_mm;
							}
							rx += l, qy += l;
						} else if (op == 2) rx += l, ++n_gapo, n_gape += l - 1;
						else if (op == 1) qy += l, ++n_gapo, n_gape += l - 1;
					}
					cnt[i] = (uint32_t)n_mm << 16 | (uint32_t)(n_gapo << 8 | n_gape);
				}
			}
		}
		/* the acceptance, pair by pair (bwape.c:571-613) */
		{
			const int s_new0 = (int)(-4.343 * log(.5 * erfc(M_SQRT1_2 * 1.5) + .499));
			const double s_old0 = -4.343 * log(ii->ap_prior / l_pac);
			int jx = 0;
			while (jx < n_jobs) {
				const int pair = jobs[jx].pair;
				int ix[2] = { -1, -1 }, kk, mapq = 0, madj[2] = { 255, 255 };
				pe_end_t *p[2] = { &g->e[2 * pair], &g->e[2 * pair + 1] };
				for (; jx < n_jobs && jobs[jx].pair == pair; ++jx) ix[jobs[jx].k] = jx;
				for (kk = 0; kk < 2; ++kk) {
					const int q = ix[kk];
					if (q < 0 || cig_of[q] < 0 || p[kk]->type == 0) continue;
					{
						const uint32_t *c = L->cig + cig_of[q];
						const int n = ncig_of[q];
						int clip = 0, s_old, s_new;
						if ((c[0] >> 14 & 3) == 3) clip += (int)(c[0] & 0x3fff);
						if ((c[n - 1] >> 14 & 3) == 3) clip += (int)(c[n - 1] & 0x3fff);
						s_old = (int)((p[kk]->n_mm * 9 + p[kk]->n_gapo * 13 + p[kk]->n_gape * 2) / 3. * 8. + .499);
						s_new = (int)(((cnt[q] >> 16) * 9 + (cnt[q] >> 8 & 0xff) * 13 + (cnt[q] & 0xff) * 2 + (uint32_t)clip * 3) / 3. * 8. + .499);
						s_old = (int)(s_old + s_old0);
						s_new += s_new0;
						if (s_old < s_new) { madj[kk] = s_new - s_old; cig_of[q] = -1; }
						else madj[kk] = s_old - s_new;
					}
				}
				{
					const int h0 = ix[0] >= 0 && cig_of[ix[0]] >= 0, h1 = ix[1] >= 0 && cig_of[ix[1]] >= 0;
					int kf = -1;
					if (h0 && h1) { kf = p[0]->mapq < p[1]->mapq ? 0 : 1; mapq = abs((int)p[1]->mapq - (int)p[0]->mapq); }
					else if (h0) kf = 0, mapq = p[1]->mapq;
					else if (h1) kf = 1, mapq = p[0]->mapq;
					if (kf >= 0) {
						const int q = ix[kf];
						const int64_t nb = jobs[q].beg + sr[q].tb;
						if (p[kf]->pos != (uint64_t)nb) {
							pe_end_t *pk = p[kf], *pr = p[1 - kf];
							int tmp = (int)pr->mapq - pk->mapq / 2 - 8;
							if (tmp <= 0) tmp = 1;
							if (mapq > tmp) mapq = tmp;
							pk->mapq = pr->mapq = (uint8_t)mapq;
							pk->seq_q = pr->seq_q = (uint8_t)(pr->seq_q < mapq ? pr->seq_q : mapq);
							if (pk->mapq > madj[kf]) pk->mapq = (uint8_t)madj[kf];
							if (pk->seq_q > madj[kf]) pk->seq_q = (uint8_t)madj[kf];
							pk->cig_off = cig_of[q]; pk->n_cig = ncig_of[q];
							pk->type = 3; pk->pos = (uint64_t)nb; pk->seq_q = pr->seq_q;
							pk->strand = (uint8_t)(1 - pr->strand);
							pk->n_mm = (uint8_t)(cnt[q] >> 16); pk->n_gapo = (uint8_t)(cnt[q] >> 8 & 0xff); pk->n_gape = (uint8_t)(cnt[q] & 0xff);
							pk->flag |= F_PP; pr->flag |= F_PP;
						}
					}
				}
			}
		}
		free(gt); free(gi); free(cnt); free(cig_of); free(ncig_of);
	}
	free(jobs); free(tasks); free(pool.s);
}

/* pairs [beg, end) of a group: P2, P5 and the records (P6) */
static pe_batch_t *run_batch(pe_run_t *r, bwag_ctx_t *ctx, const bwaidx_t *idx, pe_group_t *g, int beg, int end, const isize_info_t *ii, pe_work_t *w)
{
	pe_batch_t *bt = bb_calloc(1, sizeof(*bt));
	const int n = end - beg, nr = 2 * n;
	int64_t *off = bb_malloc(8 * ((size_t)nr + 1)), tot = 0;
	uint8_t *codes;
	pe_lists_t L;
	int i, j, past_end = -1;
	memset(&L, 0, sizeof(L));
	bt->g = g; bt->beg = beg; bt->n = n;
	for (i = 0; i < n; ++i) for (j = 0; j < 2; ++j) { off[2 * i + j] = tot; tot += g->rd[j]->off[beg + i + 1] - g->rd[j]->off[beg + i]; }
	off[nr] = tot;
	codes = bb_malloc((size_t)tot + 1);
	for (i = 0; i < n; ++i) for (j = 0; j < 2; ++j) memcpy(codes + off[2 * i + j], g->rd[j]->codes + g->rd[j]->off[beg + i], (size_t)(off[2 * i + j + 1] - off[2 * i + j]));
	if ((bt->dev = bwag_batch_begin(ctx, nr, codes, off)) == 0) bb_fatal(WHO, "cannot start a device batch: %s", bwag_last_error());
	{   /* host time of the pairing, XA and rescue decisions: the steps' wall time less that of their device calls */
		double t0 = bb_realtime(), d0 = w->t_dev_calls;
		pair_and_xa(r, bt->dev, g, beg, end, ii, &L, w);
		w->t_pair += bb_realtime() - t0 - (w->t_dev_calls - d0);
		t0 = bb_realtime(); d0 = w->t_dev_calls;
		mate_sw(r, bt->dev, g, beg, end, ii, idx->bns->l_pac, idx->pac, &L, w);
		w->t_sw += bb_realtime() - t0 - (w->t_dev_calls - d0);
	}
	{   /* the records */
		bwag_se_read_t *rd = bb_calloc((size_t)nr + 1, sizeof(*rd));
		bwag_pe_read_t *pe = bb_calloc((size_t)nr + 1, sizeof(*pe));
		int64_t *pos = bb_calloc((size_t)nr + 1, 8);
		uint8_t *str = bb_calloc((size_t)nr + 1, 1);
		bwag_sampe_par_t par;
		int64_t ng = 0;
		for (i = 0; i < n; ++i) for (j = 0; j < 2; ++j) {
			const pe_end_t *e = &g->e[2 * (beg + i) + j];
			bwag_se_read_t *p = &rd[2 * i + j];
			p->len = e->len; p->clip_len = e->len;   /* bwa_trim_read sets both */
			p->ref_shift = e->ref_shift; p->type = e->type; p->n_mm = e->n_mm; p->n_gapo = e->n_gapo; p->n_gape = e->n_gape;
			p->c1 = e->c1; p->c2 = e->c2; p->mapq = e->mapq;
			p->l_bc = (uint8_t)g->l_bc[beg + i]; p->bc_off = g->bc_off[beg + i] - g->bc_off[beg];
			p->n_multi = e->n_multi; p->multi_beg = e->multi_beg;
			pe[2 * i + j].flag = e->flag; pe[2 * i + j].seq_q = e->seq_q;
			pe[2 * i + j].comp = (r->opt[j].mode & BB_MODE_COMPREAD) != 0;
			pe[2 * i + j].cig_off = e->type == 3 ? e->cig_off : 0; pe[2 * i + j].n_cig = e->type == 3 ? e->n_cig : 0;
			pos[2 * i + j] = e->type ? (int64_t)e->pos : 0;
			str[2 * i + j] = e->type ? e->strand : 0;   /* an unmapped read is corrected on the forward strand */
		}
		memset(&par, 0, sizeof(par));
		par.mode = r->opt[1].mode & BWAG_SE_COMPREAD; par.max_top2 = r->opt[1].max_top2;
		par.comp[0] = (r->opt[0].mode & BB_MODE_COMPREAD) != 0; par.comp[1] = (r->opt[1].mode & BB_MODE_COMPREAD) != 0; par.rg_id = bwa_rg_id[0] ? bwa_rg_id : 0;
		par.reads = rd; par.pe = pe; par.pos = pos; par.strand = str;
		par.multi = L.multi; par.mpos = L.mpos; par.mstrand = L.mstrand; par.n_multi = L.n_multi;
		par.cig = L.cig; par.n_cig = L.n_cig;
		{   /* both reads of a pair carry the pair's barcode */
			const int64_t b0 = g->bc_off[beg], b1 = end < g->n ? g->bc_off[end] : (int64_t)(g->bc ? strlen(g->bc) : 0);
			par.bc = g->bc ? g->bc + b0 : 0; par.l_bc = b1 - b0;
		}
		const int rc = bwag_sampe(bt->dev, &par, &bt->res, &past_end, &ng);
		if (rc == BWAG_UNSUPPORTED) {   /* the caller drops the rest of the input and fails */
			bwag_batch_end(bt->dev);
			free(rd); free(pe); free(pos); free(str); free(L.multi); free(L.mpos); free(L.mstrand); free(L.cig); free(off); free(codes); free(bt);
			return 0;
		}
		if (past_end >= 0) {
			const int pr = beg + past_end / 2;
			bb_fatal(WHO, "read '%s': its gapped alignment runs past the end of the reference (the reference's `bwa sampe` aborts here)", g->rd[past_end & 1]->text.s + g->rd[past_end & 1]->name[pr]);
		}
		if (rc != 0) bb_fatal(WHO, "device sampe failed: %s", bwag_last_error());
		w->n_refine += ng;
		free(rd); free(pe); free(pos); free(str);
	}
	free(L.multi); free(L.mpos); free(L.mstrand); free(L.cig);
	free(off); free(codes);
	return bt;
}

/* P1 and the insert-size model of a group */
static void group_model(pe_run_t *r, bwag_ctx_t *ctx, const bwaidx_t *idx, pe_group_t *g, isize_info_t *ii, isize_info_t *last_ii, pe_work_t *w)
{
	int64_t n = 0, x;
	uint64_t *rows = bb_malloc(8 * ((size_t)2 * g->n + 1));
	int32_t *rlen = bb_malloc(8 * ((size_t)2 * g->n + 1));
	int64_t *pos = bb_malloc(16 * ((size_t)2 * g->n + 1));
	uint8_t *str = bb_malloc(2 * ((size_t)2 * g->n + 1));
	static const int64_t zero = 0;
	const uint8_t none = 0;
	int i;
	for (i = 0; i < 2 * g->n; ++i)
		if (g->e[i].type) { rows[n] = g->e[i].sa; rlen[2 * n] = rlen[2 * n + 1] = g->e[i].len + g->e[i].ref_shift; ++n; }
	if (n) {
		bwag_batch_t *b = bwag_batch_begin(ctx, 0, &none, &zero);   /* rows only: no reads */
		if (!b) bb_fatal(WHO, "cannot start a device batch: %s", bwag_last_error());
		if (bwag_pe_sa2pos(b, n, rows, rlen, pos, str) != 0) bb_fatal(WHO, "device suffix-array lookup failed: %s", bwag_last_error());
		bwag_batch_end(b);
	}
	w->n_rows += n;
	for (i = 0, x = 0; i < 2 * g->n; ++i) {
		pe_end_t *e = &g->e[i];
		if (!e->type) continue;
		e->pos = (uint64_t)pos[2 * x]; e->strand = str[2 * x]; ++x;
		if (e->pos == (uint64_t)-1) e->type = 0;   /* NO_MATCH, with its mapping quality and position kept */
	}
	free(rows); free(rlen); free(pos); free(str);
	infer_isize(g, ii, r->ap_prior, idx->bns->l_pac);
	if (ii->avg < 0.0 && last_ii->avg > 0.0) *ii = *last_ii;
	if (r->force_isize) {
		fprintf(stderr, "[%s] discard insert size estimate as user's request.\n", "bwa_cal_pac_pos_pe");
		ii->low = ii->high = 0; ii->avg = ii->std = -1.0;
	}
	*last_ii = *ii;
}

static void run_device(bb_pipe_t *p, void *run, void *item)
{
	pe_run_t *r = run;
	pe_group_t *g = item;
	const int n = g->n;
	isize_info_t ii;
	if (r->no_device) { group_free(g); return; }
	group_model(r, r->ctx, r->idx, g, &ii, &r->last_ii, &r->work);
	if (n == 0) { group_free(g); return; }
	/* the writer frees g with the group's last batch: nothing of g is touched once that batch is handed over */
	for (int beg = 0; beg < n; beg += r->chunk) {
		const int end = beg + r->chunk < n ? beg + r->chunk : n;
		pe_batch_t *b = run_batch(r, r->ctx, r->idx, g, beg, end, &ii, &r->work);
		if (!b) {
			r->no_device = 1;
			if (beg == 0) group_free(g);   /* no batch of g went out */
			return;
		}
		b->last_of_group = end == n;
		bb_pipe_to_writer(p, b);
	}
}

/* per read: name + part A + QUAL + part B + "\n"; after each pair the names are compared (bwape.c:709).  Nothing is printed after
 * a mismatch: the command fails with the reference's message once the other threads have stopped. */
static void write_batch(void *run, void *item)
{
	pe_run_t *r = run;
	pe_batch_t *b = item;
	const pe_group_t *g = b->g;
	bb_str_t s = {0, 0, 0};
	int i, j, bad = -1;
	for (i = 0; i < b->n && bad < 0 && !r->bad_names; ++i) {
		const int gi = b->beg + i;
		for (j = 0; j < 2; ++j) bb_splice_sam(&s, g->rd[j], gi, &b->res.rec[2 * i + j], b->res.text);
		if (strcmp(g->rd[0]->text.s + g->rd[0]->name[gi], g->rd[1]->text.s + g->rd[1]->name[gi]) != 0) bad = gi;
		bb_str_write(&s, 1 << 20, WHO);
	}
	bb_str_write(&s, 0, WHO);
	if (bad >= 0)
		r->bad_names = xstrdup_printf("paired reads have different names: \"%s\", \"%s\"\n", g->rd[0]->text.s + g->rd[0]->name[bad], g->rd[1]->text.s + g->rd[1]->name[bad]);
	bwag_batch_end(b->dev);
	if (b->last_of_group) group_free(b->g);
	free(b);
}

static const bb_pipe_ops_t ops = { read_all, run_device, write_batch };

int bb_sampe_main(int argc, char *argv[])
{
	int c, i;
	char *rg_line = 0, magic[2][4];
	bwaidx_t *idx;
	pe_run_t run;
	bb_pipe_busy_t busy;
	double t0, t_load;
	const char *e;
	memset(&run, 0, sizeof(run));
	run.max_isize = 500; run.max_occ = 100000; run.n_multi = 3; run.N_multi = 10; run.is_sw = 1; run.ap_prior = 1e-5;   /* bwa_init_pe_opt */
	while ((c = getopt(argc, argv, "a:o:sPn:N:c:f:Ar:")) >= 0) {   /* bwape.c:740-756 */
		switch (c) {
		case 'r': if ((rg_line = bwa_set_rg(optarg)) == 0) return 1; break;
		case 'a': run.max_isize = atoi(optarg); break;
		case 'o': run.max_occ = atoi(optarg); break;
		case 's': run.is_sw = 0; break;
		case 'P': break;   /* the index is resident on the device anyway */
		case 'n': run.n_multi = atoi(optarg); break;
		case 'N': run.N_multi = atoi(optarg); break;
		case 'c': run.ap_prior = atof(optarg); break;
		case 'f': if (freopen(optarg, "w", stdout) == 0) bb_fatal("xreopen", "fail to open file '%s'", optarg); break;
		case 'A': run.force_isize = 1; break;
		default: return 1;
		}
	}
	if (optind + 5 > argc) {
		fprintf(stderr, "Usage: bwa-b200 sampe [-a maxins] [-o maxocc] [-n maxhits] [-N maxdisc] [-c prior] [-f out.sam] [-r RG_line] [-P] [-s] [-A]\n"
		                "                      <idxbase> <in1.sai> <in2.sai> <in1.fq> <in2.fq>\n");
		return 1;
	}
	t0 = bb_realtime();
	if ((idx = bb_idx_from_resident(argv[optind])) == 0 && (idx = bwa_idx_load(argv[optind], BWA_IDX_ALL)) == 0) {
		fprintf(stderr, "[bwa_sai2sam_pe] fail to locate the index\n");
		free(rg_line);
		return 1;
	}
	run.idx = idx;
	run.ctx = bb_device_attach(idx->bwt, idx->bns, idx->pac);   /* fails here, before any output, if there is no GPU */
	bb_upload_holes(run.ctx, idx->bns, WHO);
	t_load = bb_realtime() - t0;
	bb_aln2seq_init(&run.se, idx->bns);
	for (i = 0; i < 2; ++i)
		if ((run.fp_sa[i] = fopen(argv[optind + 1 + i], "r")) == 0) bb_fatal("xopen", "fail to open file '%s'", argv[optind + 1 + i]);
	for (i = 0; i < 2; ++i) if (fread(magic[i], 1, 4, run.fp_sa[i]) != 4) bb_fatal("fread", "Unexpected end of file");
	if (strncmp(magic[0], "SAI\1", 4) != 0 || strncmp(magic[1], "SAI\1", 4) != 0) {
		fprintf(stderr, "[E::%s] Unmatched SAI magic. Please re-run `aln' with the same version of bwa.\n", WHO);
		exit(1);
	}
	for (i = 0; i < 2; ++i) {
		if (fread(&run.opt[i], sizeof(run.opt[i]), 1, run.fp_sa[i]) != 1) bb_fatal("fread", "Unexpected end of file");
		if (run.opt[i].mode & BB_MODE_BAM) bb_fatal(WHO, "the .sai file '%s' was made from BAM input (`aln -b`), which is not supported: convert the reads to FASTQ", argv[optind + 1 + i]);
		if ((run.fq[i] = bb_fq_open(argv[optind + 3 + i])) == 0) bb_fatal("xzopen", "fail to open file '%s'", argv[optind + 3 + i]);
	}
	bwa_print_sam_hdr(idx->bns, rg_line);
	run.chunk = (e = getenv("BWA_B200_SAMPE_CHUNK")) != 0 && atoi(e) > 0 ? atoi(e) : PE_GROUP;   /* pairs per device batch */
	run.last_ii.avg = -1.0; run.last_ii.std = -1.0;
	bb_pipe_run(&ops, &run, &busy);
	if (fflush(stdout) != 0 || ferror(stdout)) bb_fatal(WHO, "fail to write the output");
	if (getenv("BWA_B200_PROFILE"))
		fprintf(stderr, "[prof] sampe: index load %.3f s; busy time of the reader %.3f s, the device %.3f s, the writer %.3f s; %lld rows sent to bwt_sa; %lld pairing candidates sorted; "
		        "%lld mate local alignments, %lld mate global alignments; %lld gapped refinements; host part of the device thread: pairing and XA %.3f s, mate-rescue decisions %.3f s; total %.3f s\n",
		        t_load, busy.read, busy.device, busy.write, run.work.n_rows, run.work.n_sorted, run.work.n_local, run.work.n_global, run.work.n_refine,
		        run.work.t_pair, run.work.t_sw, bb_realtime() - t0);
	if (run.no_device) { fprintf(stderr, "[E::%s] this build has no device sampe\n", WHO); exit(1); }
	if (run.bad_names) { fprintf(stderr, "[%s] %s\n", WHO, run.bad_names); exit(1); }   /* it comes before any group the reader refused */
	if (run.sai_eof) { fprintf(stderr, "[fread] Unexpected end of file\n"); exit(1); }   /* err_fread_noeof, the earlier groups printed */
	if (run.err) { fprintf(stderr, "[%s] %s\n", WHO, run.err); exit(1); }
	for (i = 0; i < 2; ++i) { bb_fq_close(run.fq[i]); fclose(run.fp_sa[i]); }
	free(rg_line);
	bwa_idx_destroy(idx);
	return 0;
}
