/* TEST INFRASTRUCTURE ONLY.
 *
 * oracle_aln.c -- the device backtracking search (bwag_aln, include/bwa_b200_dev.h) as the CPU oracle stages answer the device-only
 * entry points: BWAG_UNSUPPORTED.  Linked next to oracle/oracle_*.c, tests/oracle_index.c and tests/oracle_fastmap.c into the test
 * binaries of the host pipeline (make testbin, make tsan), whose `aln` command then says it has no device backtracking search. */
#include <string.h>
#include "bwa_b200_dev.h"

int bwag_aln(bwag_batch_t *b, const bwag_aln_par_t *par, bwag_aln_t *out)
{
	(void)b; (void)par;
	memset(out, 0, sizeof(*out));
	return BWAG_UNSUPPORTED;
}
