#define _GNU_SOURCE
/* bb_index.c -- load the index files written by the reference's own `bwa index`, unchanged.
 *
 * On-disk formats (SURVEY.md appendix D):
 *   .bwt  u64 primary, u64 L2[1..4], then u32 words of interleaved Occ/BWT blocks   (bwt.c:385-394 / 443-462)
 *   .sa   u64 primary, u64 L2[1..4], u64 sa_intv, u64 seq_len, u64 sa[1..n_sa-1]     (bwt.c:396-407 / 421-441)
 *   .pac  forward strand, 4 bases per byte MSB first, l_pac/4+1 bytes read            (bwa.c:308-309)
 *   .ann / .amb text, .alt optional                                                   (bntseq.c:97-211)
 * The in-memory structs are the reference's (include/bwa_b200.h).
 */
#include <stdio.h>
#include <errno.h>
#include <ctype.h>
#include "bwa_b200.h"
#include "bb_host.h"

int bwa_verbose = 3;
char bwa_rg_id[256];
char *bwa_pg = 0;

/* ASCII -> 2-bit code; everything that is not ACGT/acgt is 4 ('-' is 5 in the reference table,
 * bntseq.c:46-63, and is kept so that pre-coded input behaves the same). */
unsigned char bb_nt4_table[256];
static void nt4_init(void)
{
	static int done = 0;
	if (done) return;
	memset(bb_nt4_table, 4, 256);
	bb_nt4_table['A'] = bb_nt4_table['a'] = 0;
	bb_nt4_table['C'] = bb_nt4_table['c'] = 1;
	bb_nt4_table['G'] = bb_nt4_table['g'] = 2;
	bb_nt4_table['T'] = bb_nt4_table['t'] = 3;
	bb_nt4_table['-'] = 5;
	done = 1;
}
__attribute__((constructor)) static void bb_index_ctor(void) { nt4_init(); }

static FILE *open_or_die(const char *fn, const char *mode)
{
	FILE *fp = fopen(fn, mode);
	if (!fp) bb_fatal("bwa_idx_load", "fail to open file '%s' : %s", fn, strerror(errno));
	return fp;
}

static void read_exact(FILE *fp, void *dst, size_t bytes, const char *fn)
{
	size_t got = 0;
	while (got < bytes) { /* chunked so that >2 GB reads work everywhere */
		size_t want = bytes - got < (64u << 20) ? bytes - got : (64u << 20);
		size_t r = fread((char *)dst + got, 1, want, fp);
		if (r == 0) bb_fatal("bwa_idx_load", "unexpected end of file in '%s'", fn);
		got += r;
	}
}

static char *infer_prefix(const char *hint)
{
	size_t l = strlen(hint);
	char *p = bb_malloc(l + 16);
	FILE *fp;
	sprintf(p, "%s.64.bwt", hint);
	if ((fp = fopen(p, "rb")) != 0) { fclose(fp); p[l + 3] = 0; return p; }
	sprintf(p, "%s.bwt", hint);
	if ((fp = fopen(p, "rb")) != 0) { fclose(fp); p[l] = 0; return p; }
	free(p);
	return 0;
}

bwt_t *bb_bwt_restore(const char *fn)
{
	bwt_t *bwt = bb_calloc(1, sizeof(bwt_t));
	FILE *fp;
	long fsz;
	int i, j;
	fp = open_or_die(fn, "rb");
	fseek(fp, 0, SEEK_END); fsz = ftell(fp); fseek(fp, 0, SEEK_SET);
	bwt->bwt_size = (uint64_t)(fsz - 40) >> 2;
	/* 64-byte alignment: one Occ block = one aligned 64-byte line for the device upload */
	if (posix_memalign((void **)&bwt->bwt, 64, (bwt->bwt_size << 2) + 64) != 0) bb_fatal("bwa_idx_load", "out of memory");
	read_exact(fp, &bwt->primary, 8, fn);
	read_exact(fp, bwt->L2 + 1, 32, fn);
	read_exact(fp, bwt->bwt, bwt->bwt_size << 2, fn);
	bwt->seq_len = bwt->L2[4];
	fclose(fp);
	for (i = 0; i < 256; ++i) { /* per-byte symbol counts packed 4x8 bit (bwt.c:42-51); kept for ABI completeness */
		uint32_t x = 0;
		for (j = 0; j < 4; ++j)
			x |= (uint32_t)(((i & 3) == j) + ((i >> 2 & 3) == j) + ((i >> 4 & 3) == j) + ((i >> 6) == j)) << (j << 3);
		bwt->cnt_table[i] = x;
	}
	return bwt;
}

static bwt_t *load_bwt(const char *prefix)
{
	char *fn = bb_malloc(strlen(prefix) + 8);
	bwt_t *bwt;
	FILE *fp;
	uint64_t hdr[2];
	sprintf(fn, "%s.bwt", prefix);
	bwt = bb_bwt_restore(fn);
	sprintf(fn, "%s.sa", prefix);
	fp = open_or_die(fn, "rb");
	read_exact(fp, hdr, 8, fn);
	if (hdr[0] != bwt->primary) bb_fatal("bwa_idx_load", "SA-BWT inconsistency: primary is not the same.");
	read_exact(fp, hdr, 8, fn); read_exact(fp, hdr, 8, fn); read_exact(fp, hdr, 8, fn); read_exact(fp, hdr, 8, fn); /* L2 copy */
	read_exact(fp, hdr, 16, fn);
	bwt->sa_intv = (int)hdr[0];
	if (hdr[1] != bwt->seq_len) bb_fatal("bwa_idx_load", "SA-BWT inconsistency: seq_len is not the same.");
	bwt->n_sa = (bwt->seq_len + bwt->sa_intv) / bwt->sa_intv;
	bwt->sa = bb_calloc(bwt->n_sa, 8);
	bwt->sa[0] = (bwtint_t)-1;
	read_exact(fp, bwt->sa + 1, 8 * (bwt->n_sa - 1), fn);
	fclose(fp);
	free(fn);
	return bwt;
}

/* next line of a text file into a growable buffer, newline stripped; returns 0 at EOF */
static int next_line(FILE *fp, bb_str_t *ln)
{
	int c, any = 0;
	ln->l = 0;
	bb_str_need(ln, 1); ln->s[0] = 0;
	while ((c = fgetc(fp)) != EOF) {
		any = 1;
		if (c == '\n') break;
		bb_putc(ln, c);
	}
	return any;
}

static int cmp_ann_name(const void *a, const void *b, void *anns_)
{
	const bntann1_t *anns = anns_;
	const int x = *(const int *)a, y = *(const int *)b;
	const int c = strcmp(anns[x].name, anns[y].name);
	return c ? c : (x > y) - (x < y);   /* equal names: by index, so that the last one is found last */
}

static bntseq_t *load_bns(const char *prefix)
{
	bntseq_t *bns = bb_calloc(1, sizeof(bntseq_t));
	char *fn = bb_malloc(strlen(prefix) + 8);
	bb_str_t ln = {0, 0, 0};
	FILE *fp;
	long long xx;
	int i;

	sprintf(fn, "%s.ann", prefix);
	fp = open_or_die(fn, "r");
	if (!next_line(fp, &ln) || sscanf(ln.s, "%lld%d%u", &xx, &bns->n_seqs, &bns->seed) != 3) bb_fatal("bns_restore", "Parse error reading %s", fn);
	bns->l_pac = xx;
	bns->anns = bb_calloc(bns->n_seqs, sizeof(bntann1_t));
	for (i = 0; i < bns->n_seqs; ++i) {
		bntann1_t *p = &bns->anns[i];
		char *s, *name_end;
		if (!next_line(fp, &ln)) bb_fatal("bns_restore", "Error reading %s : Unexpected end of file", fn);
		s = ln.s;
		p->gi = (uint32_t)strtoul(s, &s, 10);
		while (*s == ' ' || *s == '\t') ++s;
		name_end = s;
		while (*name_end && !isspace((unsigned char)*name_end)) ++name_end;
		p->name = bb_malloc(name_end - s + 1);
		memcpy(p->name, s, name_end - s); p->name[name_end - s] = 0;
		/* rest of the line = " <anno>"; " (null)" and empty mean no annotation (bntseq.c:124-131) */
		if (strlen(name_end) > 1 && strcmp(name_end, " (null)") != 0) p->anno = bb_strdup(name_end + 1);
		else p->anno = bb_strdup("");
		if (!next_line(fp, &ln) || sscanf(ln.s, "%lld%d%d", &xx, &p->len, &p->n_ambs) != 3) bb_fatal("bns_restore", "Parse error reading %s", fn);
		p->offset = xx;
	}
	fclose(fp);

	sprintf(fn, "%s.amb", prefix);
	fp = open_or_die(fn, "r");
	{
		int n_seqs;
		if (!next_line(fp, &ln) || sscanf(ln.s, "%lld%d%d", &xx, &n_seqs, &bns->n_holes) != 3) bb_fatal("bns_restore", "Parse error reading %s", fn);
		if (xx != bns->l_pac || n_seqs != bns->n_seqs) bb_fatal("bns_restore", "inconsistent .ann and .amb files.");
		bns->ambs = bns->n_holes ? bb_calloc(bns->n_holes, sizeof(bntamb1_t)) : 0;
		for (i = 0; i < bns->n_holes; ++i) {
			char c[64];
			if (!next_line(fp, &ln) || sscanf(ln.s, "%lld%d%63s", &xx, &bns->ambs[i].len, c) != 3) bb_fatal("bns_restore", "Parse error reading %s", fn);
			bns->ambs[i].offset = xx;
			bns->ambs[i].amb = c[0];
		}
	}
	fclose(fp);

	sprintf(fn, "%s.alt", prefix);
	if ((fp = fopen(fn, "r")) != 0) {
		/* The first field of every line that does not start with '@' names an ALT contig (bntseq.c:178-209).  As there: a name
		 * counts only once a tab / newline / carriage return ends it (a last line without one is ignored), it is cut at 1022
		 * characters, and of several contigs with the same name the LAST one is marked.  Names are looked up in a sorted copy. */
		int *order = bb_malloc(sizeof(int) * ((size_t)bns->n_seqs + 1)), c, l = 0;
		char str[1024];
		for (i = 0; i < bns->n_seqs; ++i) order[i] = i;
		qsort_r(order, (size_t)bns->n_seqs, sizeof(int), cmp_ann_name, bns->anns);
		while ((c = fgetc(fp)) != EOF) {
			if (c == '\t' || c == '\n' || c == '\r') {
				str[l] = 0;
				if (str[0] != '@') {
					int lo = 0, hi = bns->n_seqs;   /* first entry whose name is greater: the one before it is the last with this name */
					while (lo < hi) { int mid = (lo + hi) >> 1; if (strcmp(bns->anns[order[mid]].name, str) <= 0) lo = mid + 1; else hi = mid; }
					if (lo > 0 && strcmp(bns->anns[order[lo - 1]].name, str) == 0) bns->anns[order[lo - 1]].is_alt = 1;
				}
				while (c != '\n' && c != EOF) c = fgetc(fp);
				l = 0;
			} else {
				if (l >= 1022) bb_fatal("bns_restore_core", "sequence name longer than 1023 characters. Abort!");
				str[l++] = (char)c;
			}
		}
		free(order);
		fclose(fp);
	}
	free(ln.s); free(fn);
	return bns;
}

bwaidx_t *bwa_idx_load(const char *hint, int which)
{
	char *prefix = infer_prefix(hint);
	bwaidx_t *idx;
	if (!prefix) {
		if (bwa_verbose >= 1) fprintf(stderr, "[E::%s] fail to locate the index files\n", __func__);
		return 0;
	}
	idx = bb_calloc(1, sizeof(bwaidx_t));
	if (which & BWA_IDX_BWT) idx->bwt = load_bwt(prefix);
	if (which & BWA_IDX_BNS) {
		int i, c = 0;
		idx->bns = load_bns(prefix);
		for (i = 0; i < idx->bns->n_seqs; ++i) c += idx->bns->anns[i].is_alt ? 1 : 0;
		if (bwa_verbose >= 3) fprintf(stderr, "[M::%s] read %d ALT contigs\n", "bwa_idx_load_from_disk", c);
		if (which & BWA_IDX_PAC) {
			char *fn = bb_malloc(strlen(prefix) + 8);
			FILE *fp;
			sprintf(fn, "%s.pac", prefix);
			fp = open_or_die(fn, "rb");
			idx->pac = bb_calloc(idx->bns->l_pac / 4 + 1, 1);
			read_exact(fp, idx->pac, idx->bns->l_pac / 4 + 1, fn);
			fclose(fp);
			free(fn);
		}
	}
	free(prefix);
	return idx;
}

void bwa_idx_destroy(bwaidx_t *idx)
{
	int i;
	if (!idx) return;
	bb_device_release(idx->bwt); /* drop the HBM copy keyed by this index, if any */
	if (idx->bwt) { free(idx->bwt->sa); free(idx->bwt->bwt); free(idx->bwt); }
	if (idx->bns) {
		for (i = 0; i < idx->bns->n_seqs; ++i) { free(idx->bns->anns[i].name); free(idx->bns->anns[i].anno); }
		free(idx->bns->anns); free(idx->bns->ambs); free(idx->bns);
	}
	free(idx->pac);
	free(idx);
}

/* ---------------------------------------------------------------- coordinate helpers */

int bb_pos2rid(const bntseq_t *bns, int64_t pos_f) /* contig holding forward position pos_f (bntseq.c:354-368) */
{
	int lo = 0, hi = bns->n_seqs, mid = 0;
	if (pos_f >= bns->l_pac) return -1;
	while (lo < hi) {
		mid = (lo + hi) >> 1;
		if (pos_f < bns->anns[mid].offset) hi = mid;
		else if (mid == bns->n_seqs - 1 || pos_f < bns->anns[mid + 1].offset) break;
		else lo = mid + 1;
	}
	return mid;
}

int bb_intv2rid(const bntseq_t *bns, int64_t rb, int64_t re) /* bntseq.c:370-378 */
{
	int rev, a, b;
	if (rb < bns->l_pac && re > bns->l_pac) return -2;
	a = bb_pos2rid(bns, bb_depos(bns, rb, &rev));
	b = rb < re ? bb_pos2rid(bns, bb_depos(bns, re - 1, &rev)) : a;
	return a == b ? a : -1;
}

/* bases [beg,end) of the doubled (fwd + revcomp) coordinate system, one code per byte (bntseq.c:403-424) */
uint8_t *bb_get_seq(int64_t l_pac, const uint8_t *pac, int64_t beg, int64_t end, int64_t *len)
{
	uint8_t *seq = 0;
	if (end < beg) { int64_t t = beg; beg = end; end = t; }
	if (end > l_pac << 1) end = l_pac << 1;
	if (beg < 0) beg = 0;
	*len = 0;
	if (beg >= l_pac || end <= l_pac) {
		int64_t k, l = 0;
		*len = end - beg;
		seq = bb_malloc(end - beg);
		if (beg >= l_pac) {
			int64_t lo = (l_pac << 1) - 1 - end, hi = (l_pac << 1) - 1 - beg;
			for (k = hi; k > lo; --k) seq[l++] = 3 - bb_pac_get(pac, k);
		} else for (k = beg; k < end; ++k) seq[l++] = bb_pac_get(pac, k);
	}
	return seq;
}

/* clamp [*beg,*end) to the contig holding mid, then fetch (bntseq.c:426-451) */
uint8_t *bb_fetch_seq(const bntseq_t *bns, const uint8_t *pac, int64_t *beg, int64_t mid, int64_t *end, int *rid)
{
	int64_t len;
	uint8_t *seq;
	bb_clamp_to_contig(bns, beg, mid, end, rid);
	seq = bb_get_seq(bns->l_pac, pac, *beg, *end, &len);
	if (!seq || *end - *beg != len) bb_fatal("bb_fetch_seq", "begin=%ld, mid=%ld, end=%ld, len=%ld, rid=%d", (long)*beg, (long)mid, (long)*end, (long)len, *rid);
	return seq;
}

void bb_clamp_to_contig(const bntseq_t *bns, int64_t *beg, int64_t mid, int64_t *end, int *rid)
{
	int64_t far_beg, far_end;
	int rev;
	if (*end < *beg) { int64_t t = *beg; *beg = *end; *end = t; }
	if (!(*beg <= mid && mid < *end)) bb_fatal("bb_clamp_to_contig", "mid outside [beg,end)");
	*rid = bb_pos2rid(bns, bb_depos(bns, mid, &rev));
	far_beg = bns->anns[*rid].offset;
	far_end = far_beg + bns->anns[*rid].len;
	if (rev) {
		int64_t t = far_beg;
		far_beg = (bns->l_pac << 1) - far_end;
		far_end = (bns->l_pac << 1) - t;
	}
	if (*beg < far_beg) *beg = far_beg;
	if (*end > far_end) *end = far_end;
}
