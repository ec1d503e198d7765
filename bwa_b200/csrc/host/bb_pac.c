/* bb_pac.c -- the .pac, .ann and .amb files of a FASTA reference, as bns_fasta2bntseq + bns_dump write them (bntseq.c:65-95,
 * 232-353), for `bwa-b200 index` and `bwa-b200 fa2pac`; and whole-file writes that appear complete or not at all.
 *
 * Records as kseq reads them, holes = runs of the same non-ACGT character, those bases drawn by lrand48()&3 (the caller seeds
 * srand48(11) as the reference does), "(null)" for an empty comment, .pac padded to l_pac/4+1(+1) bytes with l_pac%4 last. */
#include <unistd.h>
#include <errno.h>
#include "bb_host.h"

void bb_pack_add(bb_packed_t *P, const bb_str_t *name, const bb_str_t *comment, const bb_str_t *seq)   /* add1, bntseq.c:232-278 */
{
	bntann1_t a;
	size_t i;
	int lasts = 0;
	memset(&a, 0, sizeof(a));
	a.name = bb_strdup(name->l ? name->s : "");
	a.anno = bb_strdup(comment->l > 0 ? comment->s : "(null)");
	a.len = (int32_t)seq->l;
	a.offset = P->l_pac;
	if ((size_t)(P->l_pac + seq->l) / 4 + 1 > P->m_pac) {
		size_t m = P->m_pac ? P->m_pac : 1 << 16;
		while (m < (size_t)(P->l_pac + seq->l) / 4 + 1) m <<= 1;
		P->pac = bb_realloc(P->pac, m);
		memset(P->pac + P->m_pac, 0, m - P->m_pac);
		P->m_pac = m;
	}
	for (i = 0; i < seq->l; ++i) {
		const int ch = seq->s[i];
		int c = bb_nt4_table[(unsigned char)ch];
		if (c >= 4) {
			if (lasts == ch) ++P->ambs.a[P->ambs.n - 1].len;   /* the same character as the one before: the hole goes on */
			else {
				bntamb1_t h;
				h.offset = a.offset + (int64_t)i; h.len = 1; h.amb = (char)ch;
				bb_vec_push(P->ambs, h);
				++a.n_ambs;
			}
			c = (int)(lrand48() & 3);
		}
		lasts = ch;
		P->pac[P->l_pac >> 2] |= (uint8_t)(c << ((~P->l_pac & 3) << 1));
		++P->l_pac;
	}
	bb_vec_push(P->anns, a);
}

/* append the reverse complement of the text, doubling l_pac (bntseq.c:306-312); records and holes stay those of the forward strand */
void bb_pack_add_revcomp(bb_packed_t *P)
{
	const int64_t l = P->l_pac;
	int64_t k;
	if ((size_t)(2 * l) / 4 + 1 > P->m_pac) {
		const size_t m = (size_t)(2 * l) / 4 + 1;
		P->pac = bb_realloc(P->pac, m);
		memset(P->pac + P->m_pac, 0, m - P->m_pac);
		P->m_pac = m;
	}
	for (k = l - 1; k >= 0; --k, ++P->l_pac)
		P->pac[P->l_pac >> 2] |= (uint8_t)((3 - bb_pac_get(P->pac, k)) << ((~P->l_pac & 3) << 1));
}

void bb_pack_free(bb_packed_t *P)
{
	size_t i;
	for (i = 0; i < P->anns.n; ++i) { free(P->anns.a[i].name); free(P->anns.a[i].anno); }
	bb_vec_free(P->anns); bb_vec_free(P->ambs); free(P->pac);
	memset(P, 0, sizeof(*P));
}

/* fn gets a then b: written to a temporary file beside it, then renamed into place, so that a failed write leaves whatever was
 * at fn before and no partial file */
int bb_write_whole(const char *fn, const void *a, size_t bytes, const void *b, size_t b_bytes, const char *where)
{
	char *tmp = bb_malloc(strlen(fn) + 32);
	FILE *fp;
	int ok;
	sprintf(tmp, "%s.tmp%ld", fn, (long)getpid());
	if ((fp = fopen(tmp, "wb")) == 0) { fprintf(stderr, "[E::%s] fail to open '%s' for writing: %s\n", where, tmp, strerror(errno)); free(tmp); return 1; }
	ok = fwrite(a, 1, bytes, fp) == bytes && (!b_bytes || fwrite(b, 1, b_bytes, fp) == b_bytes);
	ok = fclose(fp) == 0 && ok;
	ok = ok && rename(tmp, fn) == 0;
	if (!ok) { fprintf(stderr, "[E::%s] fail to write '%s': %s\n", where, fn, strerror(errno)); unlink(tmp); }
	free(tmp);
	return !ok;
}

int bb_write_index_file(const char *prefix, const char *ext, const void *a, size_t bytes, const void *b, size_t b_bytes, const char *where)
{
	char *fn = bb_malloc(strlen(prefix) + strlen(ext) + 1);
	int rc;
	sprintf(fn, "%s%s", prefix, ext);
	rc = bb_write_whole(fn, a, bytes, b, b_bytes, where);
	free(fn);
	return rc;
}

int bb_pack_dump(const bb_packed_t *P, const char *prefix, const char *where)   /* .pac (bntseq.c:314-327), .ann and .amb (bns_dump) */
{
	bb_str_t s = {0, 0, 0};
	size_t i, n_pac = (size_t)(P->l_pac >> 2) + ((P->l_pac & 3) ? 1 : 0);
	uint8_t tail[2] = {0, 0};
	int rc;
	tail[P->l_pac % 4 == 0] = (uint8_t)(P->l_pac % 4);
	rc = bb_write_index_file(prefix, ".pac", P->pac, n_pac, tail, P->l_pac % 4 == 0 ? 2 : 1, where);
	if (rc) return rc;
	bb_putl(&s, P->l_pac); bb_putc(&s, ' '); bb_putl(&s, (int64_t)P->anns.n); bb_puts(&s, " 11\n");
	for (i = 0; i < P->anns.n; ++i) {
		const bntann1_t *a = &P->anns.a[i];
		bb_puts(&s, "0 "); bb_puts(&s, a->name);
		if (a->anno[0]) { bb_putc(&s, ' '); bb_puts(&s, a->anno); }
		bb_putc(&s, '\n');
		bb_putl(&s, a->offset); bb_putc(&s, ' '); bb_putl(&s, a->len); bb_putc(&s, ' '); bb_putl(&s, a->n_ambs); bb_putc(&s, '\n');
	}
	rc = bb_write_index_file(prefix, ".ann", s.s, s.l, 0, 0, where);
	s.l = 0;
	bb_putl(&s, P->l_pac); bb_putc(&s, ' '); bb_putl(&s, (int64_t)P->anns.n); bb_putc(&s, ' '); bb_putl(&s, (int64_t)P->ambs.n); bb_putc(&s, '\n');
	for (i = 0; i < P->ambs.n; ++i) {
		const bntamb1_t *h = &P->ambs.a[i];
		bb_putl(&s, h->offset); bb_putc(&s, ' '); bb_putl(&s, h->len); bb_putc(&s, ' '); bb_putc(&s, h->amb); bb_putc(&s, '\n');
	}
	rc = rc || bb_write_index_file(prefix, ".amb", s.s, s.l, 0, 0, where);
	free(s.s);
	return rc;
}
