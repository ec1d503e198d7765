/* bb_index_steps.c -- the steps of `bwa index` as commands of their own (main.c:98-102), with the same files as the reference's:
 *
 *   fa2pac [-f] <in.fasta> [<out.prefix>]   .pac .ann .amb; without -f the reverse complement is appended and l_pac doubled
 *                                           (bns_fasta2bntseq, bntseq.c:280-353).  Host only.
 *   pac2bwt [-d] <in.pac> <out.bwt>         the raw .bwt (primary, L2[1..4], (n+15)/16 words, no Occ) of the .pac text as it is
 *   pac2bwtgen <in.pac> <out.bwt>           (bwtindex.c:64-145, bwt_gen.c:1560-1613): one file, whichever algorithm; sorted on the GPU
 *   bwtupdate <the.bwt>                     the Occ checkpoints interleaved, in place (bwtindex.c:147-187), on the GPU
 *   bwt2sa [-i 32] <in.bwt> <out.sa>        the suffix-array sample from the updated .bwt alone (bwt_cal_sa, bwt.c:62-84), on the GPU
 *
 * Every output is written to a temporary file beside it and renamed into place.  Where the reference aborts or crashes (an
 * interval that is not a power of two >= 1, bwt2sa on a raw .bwt, bwtupdate on an updated one, an empty or too large text) the
 * command says why, exits 1 and writes nothing.  bwt2sa also refuses a .bwt whose LF mapping is not one cycle, i.e. that is
 * not the BWT of any text; the reference writes an arbitrary .sa for it. */
#include <unistd.h>
#include <errno.h>
#include <sys/stat.h>
#include "bb_host.h"

static int file_size(const char *fn, int64_t *size, const char *where)
{
	struct stat st;
	if (stat(fn, &st) != 0) { fprintf(stderr, "[E::%s] fail to open file '%s' : %s\n", where, fn, strerror(errno)); return 1; }
	*size = (int64_t)st.st_size;
	return 0;
}

static int device_failed(int rc, const char *where, const char *what)
{
	if (rc == BWAG_UNSUPPORTED) fprintf(stderr, "[E::%s] this build has no device %s\n", where, what);
	else fprintf(stderr, "[E::%s] %s\n", where, bwag_last_error());
	return 1;
}

/* ------------------------------------------------------------------------------------------------ fa2pac */

int bb_fa2pac_main(int argc, char *argv[])
{
	int c, for_only = 0, rc;
	bb_packed_t P;
	bb_fq_t *fp;
	const bb_str_t *name, *comment, *seq;
	while ((c = getopt(argc, argv, "f")) >= 0)
		if (c == 'f') for_only = 1;   /* the reference ignores other options */
	if (argc == optind) { fprintf(stderr, "Usage: bwa-b200 fa2pac [-f] <in.fasta> [<out.prefix>]\n"); return 1; }
	if ((fp = bb_fq_open(argv[optind])) == 0) { fprintf(stderr, "[E::%s] fail to open file '%s' : %s\n", "bwa_fa2pac", argv[optind], strerror(errno)); return 1; }
	memset(&P, 0, sizeof(P));
	srand48(11);
	while (bb_fq_read1(fp, &name, &comment, &seq) >= 0) bb_pack_add(&P, name, comment, seq);
	bb_fq_close(fp);
	if (!for_only) bb_pack_add_revcomp(&P);
	rc = bb_pack_dump(&P, optind + 1 < argc ? argv[optind + 1] : argv[optind], "bwa_fa2pac");
	bb_pack_free(&P);
	return rc ? 1 : 0;
}

/* ------------------------------------------------------------------------------------------------ pac2bwt, pac2bwtgen */

/* the text of a .pac file as bwa_seq_len reads it (bwtindex.c:52-62): (size - 2) * 4 + the last byte bases */
static uint8_t *read_pac(const char *fn, uint64_t *n, const char *where)
{
	int64_t size;
	uint8_t last, *pac;
	FILE *fp;
	if (file_size(fn, &size, where)) return 0;
	if (size < 2) { fprintf(stderr, "[E::%s] '%s' is not a .pac file: %lld bytes\n", where, fn, (long long)size); return 0; }
	if ((fp = fopen(fn, "rb")) == 0) { fprintf(stderr, "[E::%s] fail to open file '%s' : %s\n", where, fn, strerror(errno)); return 0; }
	if (fseek(fp, (long)(size - 1), SEEK_SET) != 0 || fread(&last, 1, 1, fp) != 1 || last > 3) {
		fprintf(stderr, "[E::%s] '%s' is not a .pac file: its last byte is not the length of the text modulo 4\n", where, fn);
		fclose(fp);
		return 0;
	}
	*n = (uint64_t)(size - 2) * 4 + last;
	if (*n == 0) { fprintf(stderr, "[E::%s] '%s' holds an empty text\n", where, fn); fclose(fp); return 0; }
	pac = bb_malloc((size_t)(*n + 3) / 4);
	rewind(fp);
	if (fread(pac, 1, (size_t)(*n + 3) / 4, fp) != (size_t)(*n + 3) / 4) {
		fprintf(stderr, "[E::%s] fail to read '%s'\n", where, fn);
		free(pac); fclose(fp);
		return 0;
	}
	fclose(fp);
	return pac;
}

static int pac2bwt(const char *fn_pac, const char *fn_bwt, const char *where)
{
	uint64_t n, hdr[5];
	uint8_t *pac = read_pac(fn_pac, &n, where);
	bwag_raw_bwt_t x;
	double t = bb_realtime();
	int rc;
	if (!pac) return 1;
	rc = bwag_pac2bwt(-1, pac, n, &x);
	free(pac);
	if (rc) return device_failed(rc, where, "BWT builder");
	if (bwa_verbose >= 3)
		fprintf(stderr, "[M::%s] BWT of %llu symbols on the GPU in %.2f sec (peak device memory %.2f GB)\n", where,
		        (unsigned long long)x.seq_len, bb_realtime() - t, (double)x.peak_device_bytes / 1e9);
	hdr[0] = x.primary;
	memcpy(hdr + 1, x.L2 + 1, 4 * sizeof(uint64_t));
	rc = bb_write_whole(fn_bwt, hdr, 5 * 8, x.bwt, (size_t)x.bwt_size * 4, where);
	free(x.bwt);
	return rc;
}

int bb_pac2bwt_main(int argc, char *argv[])
{
	int c;
	while ((c = getopt(argc, argv, "d")) >= 0) {
		switch (c) {
		case 'd': break;   /* the reference's other construction algorithm: the BWT is the same */
		default: return 1;
		}
	}
	if (optind + 2 > argc) { fprintf(stderr, "Usage: bwa-b200 pac2bwt [-d] <in.pac> <out.bwt>\n"); return 1; }
	return pac2bwt(argv[optind], argv[optind + 1], "bwa_pac2bwt");
}

int bb_pac2bwtgen_main(int argc, char *argv[])
{
	if (argc < 3) { fprintf(stderr, "Usage: bwa-b200 pac2bwtgen <in.pac> <out.bwt>\n"); return 1; }
	return pac2bwt(argv[1], argv[2], "bwt_bwtgen");
}

/* ------------------------------------------------------------------------------------------------ bwtupdate, bwt2sa */

static uint64_t raw_words(uint64_t n) { return (n + 15) / 16; }
static uint64_t updated_words(uint64_t n) { return (n + 15) / 16 + ((n + 127) / 128 + 1) * 8; }

bwt_t *bb_read_bwt(const char *fn, int updated, const char *where)
{
	int64_t size;
	bwt_t *bwt;
	if (file_size(fn, &size, where)) return 0;
	if (size < 40 || (size - 40) % 4) { fprintf(stderr, "[E::%s] '%s' is not a .bwt file: %lld bytes\n", where, fn, (long long)size); return 0; }
	bwt = bb_bwt_restore(fn);
	if (bwt->seq_len == 0) fprintf(stderr, "[E::%s] '%s' holds an empty BWT\n", where, fn);
	else if (bwt->bwt_size == (updated ? updated_words : raw_words)(bwt->seq_len)) return bwt;
	else if (!updated && bwt->bwt_size == updated_words(bwt->seq_len))
		fprintf(stderr, "[E::%s] '%s' already holds its Occ checkpoints\n", where, fn);
	else if (updated && bwt->bwt_size == raw_words(bwt->seq_len))
		fprintf(stderr, "[E::%s] '%s' has no Occ checkpoints: run `bwa-b200 bwtupdate` on it first\n", where, fn);
	else
		fprintf(stderr, "[E::%s] '%s' is not a %s .bwt of %llu symbols: %llu words, expected %llu\n", where, fn, updated ? "updated" : "raw",
		        (unsigned long long)bwt->seq_len, (unsigned long long)bwt->bwt_size, (unsigned long long)(updated ? updated_words : raw_words)(bwt->seq_len));
	free(bwt->bwt); free(bwt);
	return 0;
}

int bb_bwtupdate_main(int argc, char *argv[])
{
	const char *where = "bwt_bwtupdate_core";
	bwt_t *bwt;
	uint32_t *out;
	uint64_t hdr[5], peak = 0;
	double t = bb_realtime();
	int rc;
	if (argc != 2) { fprintf(stderr, "Usage: bwa-b200 bwtupdate <the.bwt>\n"); return 1; }
	if ((bwt = bb_read_bwt(argv[1], 0, where)) == 0) return 1;
	out = bb_malloc((size_t)updated_words(bwt->seq_len) * 4);
	if ((rc = bwag_bwtupdate(-1, bwt->bwt, bwt->seq_len, out, &peak)) != 0) rc = device_failed(rc, where, "Occ builder");
	else {
		if (bwa_verbose >= 3)
			fprintf(stderr, "[M::%s] Occ checkpoints of %llu symbols on the GPU in %.2f sec (peak device memory %.2f GB)\n", where,
			        (unsigned long long)bwt->seq_len, bb_realtime() - t, (double)peak / 1e9);
		hdr[0] = bwt->primary;
		memcpy(hdr + 1, bwt->L2 + 1, 4 * sizeof(uint64_t));
		rc = bb_write_whole(argv[1], hdr, 5 * 8, out, (size_t)updated_words(bwt->seq_len) * 4, where);
	}
	free(out); free(bwt->bwt); free(bwt);
	return rc ? 1 : 0;
}

int bb_bwt2sa_main(int argc, char *argv[])
{
	const char *where = "bwt_cal_sa";
	int c, intv = 32, rc;
	bwt_t *bwt;
	uint64_t *sa, hdr[7], n_sa;
	bwag_bwt2sa_stats_t st;
	double t = bb_realtime();
	while ((c = getopt(argc, argv, "i:")) >= 0) {
		switch (c) {
		case 'i': intv = atoi(optarg); break;
		default: return 1;
		}
	}
	if (optind + 2 > argc) { fprintf(stderr, "Usage: bwa-b200 bwt2sa [-i %d] <in.bwt> <out.sa>\n", intv); return 1; }
	if (intv < 1 || (intv & (intv - 1))) { fprintf(stderr, "[E::%s] the SA sample interval %d is not a power of two >= 1\n", where, intv); return 1; }
	if ((bwt = bb_read_bwt(argv[optind], 1, where)) == 0) return 1;
	n_sa = (bwt->seq_len + (uint64_t)intv) / (uint64_t)intv;
	sa = malloc((size_t)n_sa * 8);
	if (!sa) { fprintf(stderr, "[E::%s] out of host memory for %llu suffix-array entries\n", where, (unsigned long long)n_sa); free(bwt->bwt); free(bwt); return 1; }
	if ((rc = bwag_bwt2sa(-1, bwt, intv, sa, &st)) != 0) rc = device_failed(rc, where, "suffix-array builder");
	else {
		if (bwa_verbose >= 3)
			fprintf(stderr, "[M::%s] suffix array of %llu rows, every %d-th, on the GPU in %.2f sec: %llu rulers %llu rows apart (peak device memory %.2f GB)\n", where,
			        (unsigned long long)bwt->seq_len + 1, intv, bb_realtime() - t, (unsigned long long)st.n_rulers, (unsigned long long)st.stride, (double)st.peak_device_bytes / 1e9);
		hdr[0] = bwt->primary;
		memcpy(hdr + 1, bwt->L2 + 1, 4 * sizeof(uint64_t));
		hdr[5] = (uint64_t)intv; hdr[6] = bwt->seq_len;
		rc = bb_write_whole(argv[optind + 1], hdr, 7 * 8, sa + 1, (size_t)(n_sa - 1) * 8, where);
	}
	free(sa); free(bwt->bwt); free(bwt);
	return rc ? 1 : 0;
}
