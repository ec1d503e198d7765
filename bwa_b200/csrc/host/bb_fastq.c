/* bb_fastq.c -- FASTA/FASTQ (optionally gzip'd) batch reader behind bseq_read (reference bwa.c:79-112,
 * grammar of kseq.h:175-215): header '>'/'@', name up to the first white space, rest of the line is the
 * comment, sequence may span lines, '+' line, quality may span lines and must match the sequence length.
 */
#include <zlib.h>
#include <ctype.h>
#include <pthread.h>
#include <fcntl.h>
#include <unistd.h>
#include <sys/stat.h>
#include "bb_host.h"

/* Parsing runs ahead of the consumer in one background thread per file (started by the first bseq_read on the
 * file): the two files of a paired-end run are parsed concurrently, and both overlap whatever the caller does
 * between two bseq_read calls.  Records travel in blocks through a small bounded queue. */
#define BLK_RECS 512
#define MAX_BLOCKS 64            /* at most this many parsed blocks wait per file */
typedef struct { char *name, *comment, *seq, *qual; int l_seq; } fq_rec_t;
typedef struct fq_blk { struct fq_blk *next; int n, status; fq_rec_t r[BLK_RECS]; } fq_blk_t;   /* status: 0, or the parser's end code (-1 EOF, -2 truncated) after the n records */

struct bb_fq {
	gzFile fp;
	unsigned char *buf;
	int beg, end, eof;
	int64_t left;             /* bytes the reader may still take from the file (a byte range of it), or -1: up to its end */
	int pending_hdr;          /* header character already consumed ('>' or '@'), or 0 */
	bb_str_t name, comment, seq, qual;
	/* producer/consumer state */
	pthread_t th;
	int started, stop, n_queued;
	pthread_mutex_t mu;
	pthread_cond_t cv;
	fq_blk_t *head, *tail;    /* parsed blocks not yet taken by the consumer */
	fq_blk_t *cur;            /* block the consumer is reading */
	int cur_pos, end_status;  /* end_status != 0: the stream has ended with that code */
};

#define FQ_BUFSZ (1 << 20)

bb_fq_t *bb_fq_open(const char *fn)
{
	bb_fq_t *f = bb_calloc(1, sizeof(*f));
	f->fp = strcmp(fn, "-") == 0 ? gzdopen(0, "r") : gzopen(fn, "r");
	if (!f->fp) { free(f); return 0; }
	gzbuffer(f->fp, 1 << 18);
	f->buf = bb_malloc(FQ_BUFSZ);
	f->left = -1;
	return f;
}

/* reader over the bytes [beg, end) of an uncompressed file; beg is the first byte of a record (bb_fq_scan_stripe finds such offsets) */
bb_fq_t *bb_fq_open_range(const char *fn, int64_t beg, int64_t end)
{
	bb_fq_t *f;
	int fd = open(fn, O_RDONLY);
	if (fd < 0) return 0;
	if (lseek(fd, (off_t)beg, SEEK_SET) < 0) { close(fd); return 0; }
	f = bb_calloc(1, sizeof(*f));
	f->fp = gzdopen(fd, "r");
	if (!f->fp) { close(fd); free(f); return 0; }
	gzbuffer(f->fp, 1 << 18);
	f->buf = bb_malloc(FQ_BUFSZ);
	f->left = end > beg ? end - beg : 0;
	return f;
}

static void blk_free(fq_blk_t *b, int from)
{
	int i;
	for (i = from; i < b->n; ++i) { free(b->r[i].name); free(b->r[i].comment); free(b->r[i].seq); free(b->r[i].qual); }
	free(b);
}

void bb_fq_close(bb_fq_t *f)
{
	if (!f) return;
	if (f->started) {
		pthread_mutex_lock(&f->mu);
		f->stop = 1;
		pthread_cond_broadcast(&f->cv);
		pthread_mutex_unlock(&f->mu);
		pthread_join(f->th, 0);
		while (f->head) { fq_blk_t *b = f->head; f->head = b->next; blk_free(b, 0); }
		if (f->cur) blk_free(f->cur, f->cur_pos);
		pthread_mutex_destroy(&f->mu); pthread_cond_destroy(&f->cv);
	}
	gzclose(f->fp);
	free(f->buf); free(f->name.s); free(f->comment.s); free(f->seq.s); free(f->qual.s);
	free(f);
}

static inline int fq_fill(bb_fq_t *f)
{
	if (f->eof) return 0;
	f->beg = 0;
	if (f->left == 0) { f->end = 0; f->eof = 1; return 0; }
	f->end = gzread(f->fp, f->buf, f->left >= 0 && f->left < FQ_BUFSZ ? (unsigned)f->left : FQ_BUFSZ);
	if (f->end <= 0) { f->end = 0; f->eof = 1; return 0; }
	if (f->left > 0) f->left -= f->end;
	return 1;
}

static inline int fq_getc(bb_fq_t *f)
{
	if (f->beg >= f->end && !fq_fill(f)) return -1;
	return f->buf[f->beg++];
}

/* append bytes up to (not including) the delimiter: '\n' when line!=0, else any white space.
 * Returns -1 if nothing could be read at EOF, else the new length; *dret = delimiter met (0 at EOF). */
static int fq_until(bb_fq_t *f, int line, bb_str_t *s, int *dret, int append)
{
	int any = 0;
	if (dret) *dret = 0;
	if (!append) s->l = 0;
	for (;;) {
		int i;
		if (f->beg >= f->end && !fq_fill(f)) break;
		if (line) { unsigned char *p = memchr(f->buf + f->beg, '\n', f->end - f->beg); i = p ? (int)(p - f->buf) : f->end; }
		else for (i = f->beg; i < f->end && !isspace(f->buf[i]); ++i) {}
		any = 1;
		bb_putsn(s, (char *)f->buf + f->beg, (size_t)(i - f->beg));
		f->beg = i + 1;
		if (i < f->end) { if (dret) *dret = f->buf[i]; break; }
	}
	if (!any && f->eof) return -1;
	bb_str_need(s, 1);
	if (line && s->l > 1 && s->s[s->l - 1] == '\r') --s->l;
	s->s[s->l] = 0;
	return (int)s->l;
}

/* >=0 sequence length; -1 end of file; -2 truncated quality */
static int fq_next(bb_fq_t *f)
{
	int c;
	if (f->pending_hdr == 0) {
		while ((c = fq_getc(f)) != -1 && c != '>' && c != '@') {}
		if (c == -1) return -1;
		f->pending_hdr = c;
	}
	f->comment.l = f->seq.l = f->qual.l = 0;
	if (fq_until(f, 0, &f->name, &c, 0) < 0) return -1;
	if (c != '\n') fq_until(f, 1, &f->comment, 0, 0);
	bb_str_need(&f->seq, 256);
	while ((c = fq_getc(f)) != -1 && c != '>' && c != '+' && c != '@') {
		if (c == '\n') continue;
		bb_putc(&f->seq, c);
		fq_until(f, 1, &f->seq, 0, 1);
	}
	if (c == '>' || c == '@') f->pending_hdr = c;
	f->seq.s[f->seq.l] = 0;
	if (c != '+') return (int)f->seq.l;
	while ((c = fq_getc(f)) != -1 && c != '\n') {}
	if (c == -1) return -2;
	while (fq_until(f, 1, &f->qual, 0, 1) >= 0 && f->qual.l < f->seq.l) {}
	f->pending_hdr = 0;
	if (f->seq.l != f->qual.l) return -2;
	return (int)f->seq.l;
}

/* one record exactly as kseq_read returns it, for readers of a reference (no read-name trimming, no parser thread):
 * >= 0 its length, -1 end of file, -2 truncated quality.  The strings stay valid until the next call. */
int bb_fq_read1(bb_fq_t *f, const bb_str_t **name, const bb_str_t **comment, const bb_str_t **seq)
{
	int r = fq_next(f);
	*name = &f->name; *comment = &f->comment; *seq = &f->seq;
	return r;
}
const bb_str_t *bb_fq_qual(const bb_fq_t *f) { return &f->qual; }   /* the quality string of the record bb_fq_read1 returned last (empty for FASTA) */

static char *dup_str(const bb_str_t *s, int dup_empty)
{
	char *p;
	if (s->l == 0 && !dup_empty) return 0;
	p = bb_malloc(s->l + 1);
	if (s->l) memcpy(p, s->s, s->l);
	p[s->l] = 0;
	return p;
}

static void take_record(bb_fq_t *f, fq_rec_t *s)
{
	if (f->name.l > 2 && f->name.s[f->name.l - 2] == '/' && isdigit((unsigned char)f->name.s[f->name.l - 1])) { f->name.l -= 2; f->name.s[f->name.l] = 0; }
	s->name = dup_str(&f->name, 1);
	s->comment = dup_str(&f->comment, 0);
	s->seq = dup_str(&f->seq, 1);
	s->qual = dup_str(&f->qual, 0);
	s->l_seq = (int)f->seq.l;
}

static void *producer_main(void *a)
{
	bb_fq_t *f = a;
	for (;;) {
		fq_blk_t *b = bb_malloc(sizeof(*b));
		int st = 0;
		b->next = 0; b->n = 0; b->status = 0;
		while (b->n < BLK_RECS) {
			st = fq_next(f);
			if (st < 0) break;
			take_record(f, &b->r[b->n++]);
		}
		if (st < 0) b->status = st;
		pthread_mutex_lock(&f->mu);
		while (f->n_queued >= MAX_BLOCKS && !f->stop) pthread_cond_wait(&f->cv, &f->mu);
		if (f->stop) { pthread_mutex_unlock(&f->mu); blk_free(b, 0); return 0; }
		if (f->tail) f->tail->next = b; else f->head = b;
		f->tail = b; ++f->n_queued;
		pthread_cond_broadcast(&f->cv);
		pthread_mutex_unlock(&f->mu);
		if (st < 0) return 0;
	}
}

/* next parsed record of the file: 1 and *r filled (ownership of the strings moves to the caller), or the parser's end code */
static int next_record(bb_fq_t *f, fq_rec_t *r)
{
	if (f->end_status) return f->end_status;
	if (!f->started) {
		pthread_mutex_init(&f->mu, 0); pthread_cond_init(&f->cv, 0);
		f->started = 1;
		if (pthread_create(&f->th, 0, producer_main, f) != 0) bb_fatal("bseq_read", "pthread_create failed");
	}
	for (;;) {
		fq_blk_t *b = f->cur;
		if (b && f->cur_pos < b->n) { *r = b->r[f->cur_pos++]; return 1; }
		if (b) {
			int st = b->status;
			free(b); f->cur = 0;
			if (st) { f->end_status = st; return st; }
		}
		pthread_mutex_lock(&f->mu);
		while (!f->head) pthread_cond_wait(&f->cv, &f->mu);
		b = f->head; f->head = b->next;
		if (!f->head) f->tail = 0;
		--f->n_queued;
		pthread_cond_broadcast(&f->cv);
		pthread_mutex_unlock(&f->mu);
		f->cur = b; f->cur_pos = 0;
	}
}

static void put_record(bseq1_t *s, const fq_rec_t *r, int id)
{
	s->name = r->name; s->comment = r->comment; s->seq = r->seq; s->qual = r->qual;
	s->l_seq = r->l_seq; s->sam = 0; s->id = id;
}

bseq1_t *bseq_read(int chunk_size, int *n_, void *ks1_, void *ks2_)
{
	bb_fq_t *f1 = ks1_, *f2 = ks2_;
	int size = 0, m = 0, n = 0;
	bseq1_t *seqs = 0;
	fq_rec_t r1, r2;
	while (next_record(f1, &r1) >= 0) {
		if (f2 && next_record(f2, &r2) < 0) {
			fprintf(stderr, "[W::%s] the 2nd file has fewer sequences.\n", __func__);
			free(r1.name); free(r1.comment); free(r1.seq); free(r1.qual);
			break;
		}
		if (n + 2 > m) { m = m ? m << 1 : 256; seqs = bb_realloc(seqs, (size_t)m * sizeof(bseq1_t)); }
		put_record(&seqs[n], &r1, n); size += seqs[n++].l_seq;
		if (f2) { put_record(&seqs[n], &r2, n); size += seqs[n++].l_seq; }
		if (size >= chunk_size && (n & 1) == 0) break;
	}
	if (size == 0 && f2 && next_record(f2, &r2) >= 0) {
		fprintf(stderr, "[W::%s] the 1st file has fewer sequences.\n", __func__);
		free(r2.name); free(r2.comment); free(r2.seq); free(r2.qual);
	}
	*n_ = n;
	return seqs;
}

/* ---------------------------------------------------------------------------------------------------------------- striped ingest
 * A multi-GPU run (bwa_b200/multi.py) must form the batches a single process would (fastmap.c:64-123: records until >= chunk bases
 * and an even count), yet no rank should parse more than its share.  Each rank scans ONE byte stripe of the file with the line
 * scanner below (record lengths and offsets only, no strings), the ranks exchange the lengths, compute the same batch boundaries,
 * and then parse just the byte ranges of their own batches (bb_fq_open_range).  Only strictly laid out uncompressed files qualify:
 * four-line FASTQ ('@' line, one sequence line, '+' line, one quality line of the same length) or two-line FASTA; anything else
 * (gzip, wrapped lines, stdin) makes the scan return BB_SCAN_UNFIT and the launcher falls back to every rank parsing everything. */
typedef struct { int fd; unsigned char *buf; int64_t base, size; int64_t n, i; int eof; } lines_t;   /* buf holds bytes [base, base + n) of the file; i = cursor */
#define LN_BUFSZ (8 << 20)

static int ln_fill(lines_t *l)   /* keep the unread tail, append fresh bytes; 0 when nothing was added */
{
	int64_t keep = l->n - l->i;
	ssize_t got;
	if (l->eof) return 0;
	if (keep > 0 && l->i > 0) memmove(l->buf, l->buf + l->i, (size_t)keep);
	l->base += l->i; l->i = 0; l->n = keep;
	if (l->n >= LN_BUFSZ) return 0;   /* a line longer than the buffer: not the kind of file this path is for */
	got = pread(l->fd, l->buf + l->n, (size_t)(LN_BUFSZ - l->n), (off_t)(l->base + l->n));
	if (got <= 0) { l->eof = 1; return 0; }
	l->n += got;
	return 1;
}
/* next line: its offset in the file, its length without the line terminator(s), its first byte (0 if empty); 0 at the end of the file */
static int ln_next(lines_t *l, int64_t *off, int *len, int *c0)
{
	unsigned char *nl;
	for (;;) {
		nl = l->i < l->n ? memchr(l->buf + l->i, '\n', (size_t)(l->n - l->i)) : 0;
		if (nl) break;
		if (!ln_fill(l)) {
			if (l->n >= LN_BUFSZ) return -1;
			if (l->i >= l->n) return 0;
			nl = l->buf + l->n;          /* last line without a terminator */
			break;
		}
	}
	{
		int64_t e = nl - l->buf, n = e - l->i;
		*off = l->base + l->i;
		*c0 = n > 0 ? l->buf[l->i] : 0;
		if (n > 1 && l->buf[e - 1] == '\r') --n;   /* as the record reader does (a lone CR stays) */
		if (n > 0x7fffffff) return -1;
		*len = (int)n;
		l->i = e < l->n ? e + 1 : e;
	}
	return 1;
}
static void ln_seek(lines_t *l, int64_t off) { l->base = off; l->n = l->i = 0; l->eof = 0; }

void bb_fq_stripe_free(bb_fqstripe_t *s) { if (s) { free(s->len); free(s->off); memset(s, 0, sizeof(*s)); } }

int64_t bb_fq_plain_size(const char *fn)   /* size of a regular uncompressed FASTA/FASTQ file, else -1 */
{
	struct stat st;
	unsigned char m[2];
	int fd = open(fn, O_RDONLY);
	int64_t size = -1;
	if (fd < 0) return -1;
	if (fstat(fd, &st) == 0 && S_ISREG(st.st_mode) && st.st_size >= 2 && pread(fd, m, 2, 0) == 2 && (m[0] == '@' || m[0] == '>')) size = (int64_t)st.st_size;
	close(fd);
	return size;
}

int bb_fq_scan_stripe(const char *fn, int64_t beg, int64_t end, bb_fqstripe_t *out)
{
	lines_t l;
	int64_t off[4], m = 0, size = bb_fq_plain_size(fn);
	int len[4], c[4], rc = BB_SCAN_UNFIT, st, kind;
	unsigned char first;
	memset(out, 0, sizeof(*out));
	if (size < 0) return BB_SCAN_UNFIT;
	memset(&l, 0, sizeof(l));
	if ((l.fd = open(fn, O_RDONLY)) < 0) return BB_SCAN_UNFIT;
	if (pread(l.fd, &first, 1, 0) != 1) { close(l.fd); return BB_SCAN_UNFIT; }
	kind = first;   /* '@': FASTQ, '>': FASTA */
	l.buf = bb_malloc(LN_BUFSZ);
	l.size = size;
	if (end > size) end = size;
	/* the first record whose header starts at or after beg: for FASTQ a line starting with '@' whose second successor starts with
	 * '+' (a quality line may start with '@', but then the line two below it is a sequence); for FASTA any line starting with '>' */
	if (beg <= 0) ln_seek(&l, 0);
	else {
		ln_seek(&l, beg - 1);
		if ((st = ln_next(&l, &off[0], &len[0], &c[0])) <= 0) { rc = st < 0 ? BB_SCAN_UNFIT : 0; goto done; }   /* the (rest of the) line that holds byte beg-1 */
	}
	if (kind == '@' && beg > 0) {
		int have = 0;
		int64_t start = -1;
		while (start < 0) {
			while (have < 3) { if ((st = ln_next(&l, &off[have], &len[have], &c[have])) <= 0) break; ++have; }
			if (have < 3) { rc = st < 0 ? BB_SCAN_UNFIT : 0; goto done; }   /* fewer than three lines left: no record starts here */
			if (off[0] >= end) { rc = 0; goto done; }
			if (c[0] == '@' && c[2] == '+') start = off[0];
			else { off[0] = off[1]; off[1] = off[2]; len[0] = len[1]; len[1] = len[2]; c[0] = c[1]; c[1] = c[2]; have = 2; }
		}
		ln_seek(&l, start);
	} else if (kind == '>' && beg > 0) {
		int64_t start = -1;
		while (start < 0) {
			if ((st = ln_next(&l, &off[0], &len[0], &c[0])) <= 0) { rc = st < 0 ? BB_SCAN_UNFIT : 0; goto done; }
			if (off[0] >= end) { rc = 0; goto done; }
			if (c[0] == '>') start = off[0];
		}
		ln_seek(&l, start);
	}
	for (;;) {
		const int want = kind == '@' ? 4 : 2;
		int k;
		if ((st = ln_next(&l, &off[0], &len[0], &c[0])) < 0) goto done;
		if (st == 0 || off[0] >= end) break;
		if (len[0] == 0) {   /* blank lines are legal after the last record only (the record grammar skips them there) */
			while ((st = ln_next(&l, &off[0], &len[0], &c[0])) > 0) if (len[0] != 0) goto done;
			if (st < 0) goto done;
			break;
		}
		for (k = 1; k < want; ++k) if (ln_next(&l, &off[k], &len[k], &c[k]) <= 0) goto done;   /* truncated record */
		if (c[0] != kind || c[1] == '@' || c[1] == '>' || c[1] == '+') goto done;
		if (kind == '@' && (c[2] != '+' || len[3] != len[1])) goto done;
		if (out->n == m) { m = m ? m << 1 : 1 << 16; out->len = bb_realloc(out->len, (size_t)m * sizeof(int32_t)); out->off = bb_realloc(out->off, (size_t)m * sizeof(int64_t)); }
		out->len[out->n] = len[1]; out->off[out->n] = off[0]; ++out->n;
	}
	rc = 0;
done:
	if (rc != 0) bb_fq_stripe_free(out);
	free(l.buf); close(l.fd);
	return rc;
}
