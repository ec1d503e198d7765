/* TEST INFRASTRUCTURE ONLY.
 *
 * oracle_index_steps.c -- the device entry points of the index steps (bwag_pac2bwt, bwag_bwtupdate, bwag_bwt2sa,
 * include/bwa_b200_dev.h) as the CPU oracle stages answer the device-only entry points: BWAG_UNSUPPORTED.  Linked next to
 * oracle/oracle_*.c into the test binaries of the host pipeline (make testbin, make tsan), whose `pac2bwt`, `pac2bwtgen`,
 * `bwtupdate` and `bwt2sa` commands then say they have no device builder. */
#include <string.h>
#include "bwa_b200_dev.h"

int bwag_pac2bwt(int device, const uint8_t *pac, uint64_t seq_len, bwag_raw_bwt_t *out)
{
	(void)device; (void)pac; (void)seq_len;
	memset(out, 0, sizeof(*out));
	return BWAG_UNSUPPORTED;
}
int bwag_bwtupdate(int device, const uint32_t *raw, uint64_t seq_len, uint32_t *out, uint64_t *peak_device_bytes)
{
	(void)device; (void)raw; (void)seq_len; (void)out; (void)peak_device_bytes;
	return BWAG_UNSUPPORTED;
}
int bwag_bwt2sa(int device, const bwt_t *bwt, int intv, uint64_t *sa, bwag_bwt2sa_stats_t *st)
{
	(void)device; (void)bwt; (void)intv; (void)sa;
	memset(st, 0, sizeof(*st));
	return BWAG_UNSUPPORTED;
}
