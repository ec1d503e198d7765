/* TEST INFRASTRUCTURE ONLY.
 *
 * oracle_fastmap.c -- the device SMEM lister (bwag_fastmap, include/bwa_b200_dev.h) as the CPU oracle stages answer the
 * device-only entry points: BWAG_UNSUPPORTED.  Linked next to oracle/oracle_*.c and tests/oracle_index.c into the test binaries
 * of the host pipeline (make testbin, make tsan), whose `fastmap` command then says it has no device SMEM lister. */
#include <string.h>
#include "bwa_b200_dev.h"

int bwag_fastmap(bwag_batch_t *b, const bwag_fastmap_par_t *par, bwag_fastmap_t *out)
{
	(void)b; (void)par;
	memset(out, 0, sizeof(*out));
	return BWAG_UNSUPPORTED;
}
