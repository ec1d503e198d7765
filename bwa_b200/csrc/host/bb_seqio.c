/* bb_seqio.c -- the reads of `bwa-b200 aln` and `bwa-b200 samse` as the reference's bwa_read_seq gives them (bwaseqio.c:151-221):
 * Casava filtering (-Y), Illumina 1.3+ qualities (-I: every quality byte minus 31), barcode removal (-B, the barcode's bases
 * lowercase where their quality is below 13), quality trimming (bwa_trim_read: down to 35 bases at most) and, for SAM, the name
 * without a trailing /1 or /2.  kseq grammar: FASTA/FASTQ, plain or gzip, '-' for stdin. */
#include <ctype.h>
#include "bb_host.h"

#define BARCODE_LOW_QUAL 13

void bb_reads_free(bb_reads_t *g)
{
	if (!g) return;
	free(g->off); free(g->codes); free(g->len);
	free(g->name); free(g->qual); free(g->bc); free(g->text.s);
	free(g);
}

static void put_text(bb_reads_t *g, int64_t *at, const char *s, size_t l)
{
	*at = (int64_t)g->text.l;
	bb_putsn(&g->text, s, l);
	bb_putc(&g->text, 0);
}

bb_reads_t *bb_read_group(bb_fq_t *fq, int mode, int trim_qual, int n_max, int keep, int max_len, const char *who)
{
	const int l_bc = mode >> 24, is_64 = (mode & BB_MODE_IL13) != 0;
	const bb_str_t *name, *comment, *seq;
	bb_reads_t *g = 0;
	int64_t bases = 0, m_bases = 0;
	int m = 0, i;
	char bcbuf[BB_MAX_BCLEN + 1];
	if (l_bc > BB_MAX_BCLEN) {   /* bwaseqio.c:158-161: no reads at all */
		fprintf(stderr, "[%s] the maximum barcode length is %d.\n", "bwa_read_seq", BB_MAX_BCLEN);
		return 0;
	}
	while (!g || g->n < n_max) {
		int len = bb_fq_read1(fq, &name, &comment, &seq), full_len, n_store;
		const bb_str_t *qual;
		if (len < 0) break;   /* end of input, or a truncated quality string: kseq_read < 0 ends the reference's loop too */
		qual = bb_fq_qual(fq);
		if ((mode & BB_MODE_CFY) && comment->l != 0) {   /* Casava-filtered: the comment has 'Y' right after its first ':' */
			const char *s = strchr(comment->s, ':');
			if (s && s[1] == 'Y') continue;
		}
		if ((int)seq->l <= l_bc) continue;   /* no longer than the barcode: no record */
		full_len = len = (int)seq->l - l_bc;
		if (qual->l && trim_qual >= 1) {   /* bwa_trim_read (bwaseqio.c:80-91) on the qualities after -I and the barcode */
			int s = 0, best = 0, best_l = len, t;
			for (t = len - 1; t >= BB_MIN_RDLEN; --t) {
				const uint8_t q = (uint8_t)(qual->s[l_bc + t] - (is_64 ? 31 : 0));
				s += trim_qual - (q - 33);
				if (s < 0) break;
				if (s > best) best = s, best_l = t;
			}
			len = best_l;
		}
		if (len >= max_len) bb_fatal(who, "read '%s' has %d bases to search; reads of %d bases or more are not supported", name->s, len, max_len);
		if (!g) {
			g = bb_calloc(1, sizeof(*g)); m = 1024;
			g->off = bb_malloc(8 * (size_t)(m + 1)); g->off[0] = 0;
			g->len = bb_malloc(4 * (size_t)m);
			if (keep) { g->name = bb_malloc(8 * (size_t)m); g->qual = bb_malloc(8 * (size_t)m); g->bc = bb_malloc(8 * (size_t)m); }
		}
		if (g->n == m) {
			m <<= 1;
			g->off = bb_realloc(g->off, 8 * (size_t)(m + 1));
			g->len = bb_realloc(g->len, 4 * (size_t)m);
			if (keep) { g->name = bb_realloc(g->name, 8 * (size_t)m); g->qual = bb_realloc(g->qual, 8 * (size_t)m); g->bc = bb_realloc(g->bc, 8 * (size_t)m); }
		}
		n_store = keep ? full_len : len;
		if (bases + n_store > m_bases) {
			m_bases = m_bases ? m_bases : 1 << 16;
			while (m_bases < bases + n_store) m_bases <<= 1;
			g->codes = bb_realloc(g->codes, (size_t)m_bases);
		}
		if (keep) {   /* nst_nt4_table codes of the whole read ('-' stays 5) */
			for (i = 0; i < n_store; ++i) g->codes[bases + i] = bb_nt4_table[(unsigned char)seq->s[l_bc + i]];
		} else {
			for (i = 0; i < n_store; ++i) { const int c = bb_nt4_table[(unsigned char)seq->s[l_bc + i]]; g->codes[bases + i] = (uint8_t)(c > 4 ? 4 : c); }   /* '-' (5) acts as N */
		}
		if (keep) {
			const int r = g->n;
			size_t l_name = name->l;
			if (l_name > 2 && name->s[l_name - 2] == '/' && (name->s[l_name - 1] == '1' || name->s[l_name - 1] == '2')) l_name -= 2;
			put_text(g, &g->name[r], name->s, l_name);
			if (qual->l) {
				int64_t q0;
				put_text(g, &q0, qual->s + l_bc, (size_t)full_len);
				if (is_64) for (i = 0; i < full_len; ++i) g->text.s[q0 + i] -= 31;
				g->qual[r] = q0;
			} else g->qual[r] = -1;
			if (l_bc) {
				for (i = 0; i < l_bc; ++i) {
					const int q = qual->l ? (char)(qual->s[i] - (is_64 ? 31 : 0)) : 0;
					bcbuf[i] = (char)(qual->l && q - 33 < BARCODE_LOW_QUAL ? tolower((unsigned char)seq->s[i]) : toupper((unsigned char)seq->s[i]));
				}
				put_text(g, &g->bc[r], bcbuf, (size_t)l_bc);
			} else g->bc[r] = -1;
		}
		if (len > g->max_len) g->max_len = len;
		g->len[g->n] = len;
		bases += n_store;
		g->off[++g->n] = bases;
	}
	if (g && !g->codes) g->codes = bb_malloc(16);
	return g;
}
