/* bb_util.h -- small host-side utilities: fatal errors, checked allocation, growable arrays, timers,
 * the 64-bit mixer used for tie-breaks.  Internal to libbwa_b200. */
#ifndef BB_UTIL_H
#define BB_UTIL_H
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <pthread.h>

#ifdef __cplusplus
extern "C" {
#endif

void bb_fatal(const char *where, const char *fmt, ...) __attribute__((noreturn, format(printf, 2, 3)));
void *bb_malloc(size_t n);
void *bb_calloc(size_t n, size_t sz);
void *bb_realloc(void *p, size_t n);
char *bb_strdup(const char *s);
double bb_cputime(void);
double bb_realtime(void);

/* growable array: struct { size_t n, m; T *a; } */
#define BB_VEC(T) struct { size_t n, m; T *a; }
#define bb_vec_reserve(v, need) do { size_t need_ = (need); if ((v).m < need_) { size_t m_ = (v).m ? (v).m : 4; \
		while (m_ < need_) { m_ <<= 1; } \
		(v).a = bb_realloc((v).a, m_ * sizeof(*(v).a)); (v).m = m_; } } while (0)
#define bb_vec_push(v, x) do { bb_vec_reserve(v, (v).n + 1); (v).a[(v).n++] = (x); } while (0)
#define bb_vec_free(v) do { free((v).a); (v).a = 0; (v).n = (v).m = 0; } while (0)
typedef BB_VEC(int) bb_int_v;

/* Thomas Wang style 64-bit mixer; must equal the reference's hash_64 (utils.h:98-109) bit for bit
 * because it decides ties between equal-score hits (bwamem.c:553) and pairs (bwamem_pair.c:249). */
static inline uint64_t bb_mix64(uint64_t k)
{
	k += ~(k << 32); k ^= (k >> 22);
	k += ~(k << 13); k ^= (k >> 8);
	k += (k << 3);   k ^= (k >> 15);
	k += ~(k << 27); k ^= (k >> 31);
	return k;
}

/* parallel-for over [0,n) on nt threads; fn(data, i, tid).  Same contract as kt_for (kthread.c:49-61). */
void bb_parallel_for(int nt, void (*fn)(void *, long, int), void *data, long n);
void bb_parallel_for_lane(int lane, int nt, void (*fn)(void *, long, int), void *data, long n);
int bb_effective_cpus(void);   /* affinity mask capped by a cgroup CPU quota */
int bb_parallel_ids(void);
void bb_parallel_name(void (*fn)(void *, long, int), const char *name);   /* label a loop body for BWA_B200_PROFILE */
void bb_parallel_report(void);   /* upper bound (exclusive) of the thread ids passed to loop bodies */

/* single-slot mailbox between two threads: put waits while the slot is full, get while it is empty; the item NULL is a valid
 * message (the commands use it for the end of the input).  Stages connected by such mailboxes keep their order and at most one
 * item waits between two of them. */
typedef struct { pthread_mutex_t mu; pthread_cond_t cv; void *slot; int full; } bb_mbox_t;
void bb_mbox_init(bb_mbox_t *m);
void bb_mbox_put(bb_mbox_t *m, void *item);
void *bb_mbox_get(bb_mbox_t *m);

/* bwa_cal_maxdiff (bwtaln.c:42-54): the most differences `bwa aln` allows in a read of l bases (-n as a fraction) */
int bb_cal_maxdiff(int l, double err, double thres);

typedef struct { uint64_t x, y; } bb_pair64_t;
void bb_sort_u64(size_t n, uint64_t *a);         /* == ks_introsort_64 */
void bb_sort_pair64(size_t n, bb_pair64_t *a);   /* == ks_introsort_128 (by x, then y) */

#ifdef __cplusplus
}
#endif
#endif
