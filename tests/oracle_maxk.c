/* TEST INFRASTRUCTURE ONLY.
 *
 * oracle_maxk.c -- the device half of `maxk` (bwag_ctx_create_occ, bwag_maxk; include/bwa_b200_dev.h) as the CPU oracle stages
 * answer the device-only entry points: a context without a device, and BWAG_UNSUPPORTED.  Linked next to oracle/oracle_*.c into the
 * test binaries of the host pipeline (make testbin, make tsan), whose `maxk` command then says it has no device SMEM search. */
#include <string.h>
#include "bwa_b200_dev.h"

bwag_ctx_t *bwag_ctx_create_occ(int device, const bwt_t *bwt) { return bwag_ctx_create(device, bwt, 0, 0); }
int bwag_maxk(bwag_batch_t *b, int min_intv, int64_t window, uint64_t hist[256], bwag_maxk_stats_t *st)
{
	(void)b; (void)min_intv; (void)window; (void)hist;
	memset(st, 0, sizeof(*st));
	return BWAG_UNSUPPORTED;
}
