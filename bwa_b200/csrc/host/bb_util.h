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

/* single-slot mailbox: put waits while the slot is full, get while it is empty.  Putting NULL closes the box: once the item before
 * it is taken, every get returns NULL, so any number of consumers see the end.  Stages connected by such mailboxes keep their order
 * and at most one item waits between two of them. */
typedef struct { pthread_mutex_t mu; pthread_cond_t cv; void *slot; int closed; } bb_mbox_t;
void bb_mbox_init(bb_mbox_t *m);
void bb_mbox_put(bb_mbox_t *m, void *item);
void *bb_mbox_get(bb_mbox_t *m);

/* The pipeline of fastmap, aln, samse, sampe and pemerge: three threads overlap.  A reader thread parses the input and hands items
 * to the device stage; the device stage runs on the calling thread and hands its results to a writer thread, which prints and
 * frees them.  Single-slot mailboxes join the stages, so output order is input order and at most one item waits between two
 * stages.  A stage may hand on any number of items per call: aln, samse and pemerge cut a reader group into several device
 * batches, sampe cuts a device group into several writer batches.  Items are never NULL.  bb_pipe_run returns once the reader
 * has returned and every item is written; a stage that wants to stop early returns (reader) or drops what it gets (device).
 * The busy time of a stage is its thread's wall time less the time it spent blocked in a hand-off (BWA_B200_PROFILE). */
typedef struct bb_pipe bb_pipe_t;
typedef struct {
	void (*read)(bb_pipe_t *p, void *run);               /* reader thread: bb_pipe_to_device() per batch; returns at the end of the input */
	void (*device)(bb_pipe_t *p, void *run, void *item);  /* calling thread: zero or more bb_pipe_to_writer() per item */
	void (*write)(void *run, void *item);                 /* writer thread: prints the item and frees it */
} bb_pipe_ops_t;
typedef struct { double read, device, write; } bb_pipe_busy_t;
void bb_pipe_run(const bb_pipe_ops_t *ops, void *run, bb_pipe_busy_t *busy);
void bb_pipe_to_device(bb_pipe_t *p, void *item);
void bb_pipe_to_writer(bb_pipe_t *p, void *item);

/* bwa_cal_maxdiff (bwtaln.c:42-54): the most differences `bwa aln` allows in a read of l bases (-n as a fraction) */
int bb_cal_maxdiff(int l, double err, double thres);

typedef struct { uint64_t x, y; } bb_pair64_t;
void bb_sort_u64(size_t n, uint64_t *a);         /* == ks_introsort_64 */
void bb_sort_pair64(size_t n, bb_pair64_t *a);   /* == ks_introsort_128 (by x, then y) */

#ifdef __cplusplus
}
#endif
#endif
