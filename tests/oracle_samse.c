/* TEST INFRASTRUCTURE ONLY.
 *
 * oracle_samse.c -- the device half of `samse` (bwag_samse, bwag_ctx_set_ambs; include/bwa_b200_dev.h) as the CPU oracle stages
 * answer the device-only entry points: BWAG_UNSUPPORTED.  Linked next to oracle/oracle_*.c and the other tests/oracle_*.c stubs into
 * the test binaries of the host pipeline (make testbin, make tsan), whose `samse` command then says it has no device samse. */
#include <string.h>
#include "bwa_b200_dev.h"

int bwag_ctx_set_ambs(bwag_ctx_t *ctx, int n_holes, const int64_t *offset, const int32_t *len)
{
	(void)ctx; (void)n_holes; (void)offset; (void)len;
	return 0;
}

int bwag_samse(bwag_batch_t *b, const bwag_samse_par_t *par, bwag_sam_t *out, int *past_end, int64_t *n_sa, int64_t *n_glb)
{
	(void)b; (void)par;
	memset(out, 0, sizeof(*out));
	*past_end = -1; *n_sa = 0; *n_glb = 0;
	return BWAG_UNSUPPORTED;
}
