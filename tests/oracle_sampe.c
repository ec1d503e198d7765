/* TEST INFRASTRUCTURE ONLY.
 *
 * oracle_sampe.c -- the device half of `sampe` (bwag_pe_sa2pos, bwag_pe_global, bwag_sampe; include/bwa_b200_dev.h) as the CPU
 * oracle stages answer the device-only entry points: BWAG_UNSUPPORTED.  Linked next to oracle/oracle_*.c and the other
 * tests/oracle_*.c stubs into the test binaries of the host pipeline (make testbin, make tsan), whose `sampe` command then says it
 * has no device sampe. */
#include <string.h>
#include "bwa_b200_dev.h"

int bwag_pe_sa2pos(bwag_batch_t *b, int64_t n_rows, const uint64_t *rows, const int32_t *ref_len, int64_t *pos, uint8_t *strand)
{   /* every row across the strand boundary: all reads unmapped, so the command reaches bwag_sampe */
	(void)b; (void)rows; (void)ref_len;
	for (int64_t i = 0; i < 2 * n_rows; ++i) pos[i] = -1, strand[i] = 0;
	return 0;
}

int bwag_pe_global(bwag_batch_t *b, int n_tasks, const bwag_pe_gtask_t *tasks, const uint8_t *pool, size_t pool_bytes, const bwag_pe_gres_t **res, const uint32_t **cig)
{
	(void)b; (void)n_tasks; (void)tasks; (void)pool; (void)pool_bytes;
	*res = 0; *cig = 0;
	return BWAG_UNSUPPORTED;
}

int bwag_sampe(bwag_batch_t *b, const bwag_sampe_par_t *par, bwag_sam_t *out, int *past_end, int64_t *n_glb)
{
	(void)b; (void)par;
	memset(out, 0, sizeof(*out));
	*past_end = -1; *n_glb = 0;
	return BWAG_UNSUPPORTED;
}
