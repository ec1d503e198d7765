/* TEST INFRASTRUCTURE ONLY.
 *
 * oracle_pemerge.c -- the device half of `pemerge` (bwag_ctx_create_bare, bwag_pemerge; include/bwa_b200_dev.h) as the CPU oracle
 * stages answer the device-only entry points: BWAG_UNSUPPORTED.  Linked next to oracle/oracle_*.c and the other tests/oracle_*.c stubs
 * into the test binaries of the host pipeline (make testbin, make tsan), whose `pemerge` command then says it has no device pemerge. */
#include <string.h>
#include "bwa_b200_dev.h"

bwag_ctx_t *bwag_ctx_create_bare(int device) { return bwag_ctx_create(device, 0, 0, 0); }

int bwag_pemerge(bwag_batch_t *b, const bwag_pemerge_par_t *par, bwag_pemerge_t *out)
{
	(void)b; (void)par;
	memset(out, 0, sizeof(*out));
	return BWAG_UNSUPPORTED;
}
