/* bb_index_build.c -- `bwa-b200 index`: the five index files of a FASTA reference, byte for byte those of the reference's
 * `bwa index` (bwtindex.c:213-330), with the suffix sorting on the GPU (bwag_index_build, bwag_index.cu).
 *
 *   .pac .ann .amb   packed as bns_fasta2bntseq(..., for_only=1) + bns_dump do (bb_pac.c, shared with `fa2pac`), after srand48(11)
 *   .bwt .sa         from the device, written in the layout of bwt_dump_bwt / bwt_dump_sa (bwt.c:385-407)
 *
 * Before it reports success the command loads the new index onto the device and checks every row of it against the text
 * (bwag_ctx_verify, stride 1). */
#include <unistd.h>
#include <errno.h>
#include "bb_host.h"

static int dump_bwt_sa(const bwag_built_index_t *x, const char *prefix)   /* bwt_dump_bwt, bwt_dump_sa */
{
	uint64_t hdr[7];
	hdr[0] = x->primary;
	memcpy(hdr + 1, x->L2 + 1, 4 * sizeof(uint64_t));
	hdr[5] = 32; hdr[6] = x->seq_len;
	return bb_write_index_file(prefix, ".bwt", hdr, 5 * 8, x->bwt, (size_t)x->bwt_size * 4, "bwa_index") ||
	       bb_write_index_file(prefix, ".sa", hdr, 7 * 8, x->sa + 1, (size_t)(x->n_sa - 1) * 8, "bwa_index");
}

/* every row of the new index against the text, on the device: BWT/text/SA mismatches and order violations are fatal; pairs of
 * suffixes equal over the verifier's 8192-base window are reported (long exact repeats produce them legitimately) */
static int self_check(const char *prefix)
{
	bwaidx_t *idx = bwa_idx_load(prefix, BWA_IDX_ALL);
	bwag_ctx_t *ctx;
	uint64_t out[4] = {0, 0, 0, 0};
	int rc;
	if (!idx) { fprintf(stderr, "[E::%s] cannot load the new index '%s'\n", "bwa_index", prefix); return 1; }
	if ((ctx = bwag_ctx_create(-1, idx->bwt, idx->bns->l_pac, idx->pac)) == 0) {
		fprintf(stderr, "[E::%s] cannot place the new index on the device: %s\n", "bwa_index", bwag_last_error());
		bwa_idx_destroy(idx);
		return 1;
	}
	rc = bwag_ctx_verify(ctx, 0, 1, out);
	if (rc) fprintf(stderr, "[E::%s] verification failed to run: %s\n", "bwa_index", bwag_last_error());
	else if (out[0] != idx->bwt->seq_len + 1 || out[1] || out[2]) {
		fprintf(stderr, "[E::%s] the new index is wrong: %llu rows checked of %llu, %llu BWT/text/SA mismatches, %llu order violations\n", "bwa_index",
		        (unsigned long long)out[0], (unsigned long long)idx->bwt->seq_len + 1, (unsigned long long)out[1], (unsigned long long)out[2]);
		rc = 1;
	} else if (bwa_verbose >= 3)
		fprintf(stderr, "[M::%s] verified all %llu rows on the device; %llu adjacent suffix pairs agree over 8192 bases (long exact repeats)\n",
		        "bwa_index", (unsigned long long)out[0], (unsigned long long)out[3]);
	bwag_ctx_destroy(ctx);
	bwa_idx_destroy(idx);
	return rc;
}

static int usage(void)
{
	fprintf(stderr, "\nUsage:   bwa-b200 index [options] <in.fasta[.gz]>\n\n");
	fprintf(stderr, "Options: -p STR    prefix of the index [same as fasta name]\n");
	fprintf(stderr, "         -6        index files named as <in.fasta>.64.* instead of <in.fasta>.*\n");
	fprintf(stderr, "         -a STR    accepted for compatibility (bwtsw, is or rb2) and ignored\n");
	fprintf(stderr, "         -b INT    accepted for compatibility and ignored\n\n");
	fprintf(stderr, "Writes .pac .ann .amb .bwt .sa identical to those of `bwa index`: the BWT and suffix array of a text are\n");
	fprintf(stderr, "unique, so the construction algorithm cannot change them.  The suffixes are sorted on the GPU.\n\n");
	return 1;
}

int bb_index_main(int argc, char *argv[])
{
	int c, is_64 = 0, rc = 0, packed = 0;
	char *prefix = 0;
	bb_packed_t P;
	bb_fq_t *fp;
	const bb_str_t *name, *comment, *seq;
	bwag_built_index_t x;
	double t0 = bb_realtime(), t;
	while ((c = getopt(argc, argv, "6a:p:b:")) >= 0) {
		switch (c) {
		case 'a':
			if (strcmp(optarg, "rb2") && strcmp(optarg, "bwtsw") && strcmp(optarg, "is")) { fprintf(stderr, "[E::%s] unknown algorithm: '%s'.\n", "bwa_index", optarg); return 1; }
			break;
		case 'p': free(prefix); prefix = bb_strdup(optarg); break;
		case '6': is_64 = 1; break;
		case 'b': break;
		default: return 1;
		}
	}
	if (optind + 1 > argc) { free(prefix); return usage(); }
	if (prefix == 0) {
		prefix = bb_malloc(strlen(argv[optind]) + 4);
		strcpy(prefix, argv[optind]);
		if (is_64) strcat(prefix, ".64");
	}
	if ((fp = bb_fq_open(argv[optind])) == 0) { fprintf(stderr, "[E::%s] fail to open file '%s' : %s\n", "bwa_index", argv[optind], strerror(errno)); free(prefix); return 1; }

	memset(&P, 0, sizeof(P));
	srand48(11);
	while (bb_fq_read1(fp, &name, &comment, &seq) >= 0) bb_pack_add(&P, name, comment, seq);
	bb_fq_close(fp);
	if (P.l_pac == 0) { fprintf(stderr, "[E::%s] no sequence in '%s'\n", "bwa_index", argv[optind]); rc = 1; goto end; }
	if (bb_pack_dump(&P, prefix, "bwa_index")) { rc = 1; goto end; }
	packed = 1;
	if (bwa_verbose >= 3) fprintf(stderr, "[M::%s] packed %ld sequences (%lld bp, %ld holes) in %.2f sec\n", "bwa_index", (long)P.anns.n, (long long)P.l_pac, (long)P.ambs.n, bb_realtime() - t0);

	t = bb_realtime();
	if ((rc = bwag_index_build(-1, P.pac, P.l_pac, &x)) != 0) {
		if (rc == BWAG_UNSUPPORTED) fprintf(stderr, "[E::%s] this build has no device index builder\n", "bwa_index");
		else fprintf(stderr, "[E::%s] %s\n", "bwa_index", bwag_last_error());
		goto end;
	}
	if (bwa_verbose >= 3) {
		fprintf(stderr, "[M::%s] BWT and suffix array of %llu symbols on the GPU in %.2f sec (peak device memory %.2f GB)\n", "bwa_index",
		        (unsigned long long)x.seq_len, bb_realtime() - t, (double)x.peak_device_bytes / 1e9);
		fprintf(stderr, "[M::%s] %llu suffix groups, at most %llu suffixes each\n", "bwa_index", (unsigned long long)x.n_groups, (unsigned long long)x.max_group);
	}
	rc = dump_bwt_sa(&x, prefix);
	bwag_built_index_free(&x);
	if (rc) goto end;
	t = bb_realtime();
	if ((rc = self_check(prefix)) != 0) goto end;
	if (bwa_verbose >= 3) fprintf(stderr, "[M::%s] self-check %.2f sec; index '%s' written in %.2f sec\n", "bwa_index", bb_realtime() - t, prefix, bb_realtime() - t0);
end:
	if (rc && packed) {   /* no .bwt/.sa, earlier or partial, may stay beside the new .pac: `mem` would load a mismatched index */
		char *fn = bb_malloc(strlen(prefix) + 8);
		sprintf(fn, "%s.bwt", prefix); unlink(fn);
		sprintf(fn, "%s.sa", prefix); unlink(fn);
		fprintf(stderr, "[E::%s] index '%s' is incomplete: only .pac .ann .amb were written\n", "bwa_index", prefix);
		free(fn);
	}
	bb_pack_free(&P);
	free(prefix);
	return rc ? 1 : 0;
}
