#define _GNU_SOURCE
/* bb_util.c -- fatal errors, checked allocation, timers, thread helpers, plain-key sorts. */
#include <stdarg.h>
#include <pthread.h>
#include <sched.h>
#include <unistd.h>
#include <time.h>
#include <sys/time.h>
#include <sys/resource.h>
#include <limits.h>
#include <math.h>
#include "bb_util.h"
#include "bb_sort.h"

void bb_fatal(const char *where, const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	fprintf(stderr, "[%s] ", where);
	vfprintf(stderr, fmt, ap);
	fprintf(stderr, "\n");
	va_end(ap);
	exit(EXIT_FAILURE); /* reference: err_fatal -> exit(EXIT_FAILURE), utils.c:90-99 */
}

void *bb_malloc(size_t n)
{
	void *p = malloc(n ? n : 1);
	if (!p) bb_fatal("bb_malloc", "out of memory allocating %zu bytes", n);
	return p;
}
void *bb_calloc(size_t n, size_t sz)
{
	void *p = calloc(n ? n : 1, sz ? sz : 1);
	if (!p) bb_fatal("bb_calloc", "out of memory allocating %zu x %zu bytes", n, sz);
	return p;
}
void *bb_realloc(void *q, size_t n)
{
	void *p = realloc(q, n ? n : 1);
	if (!p) bb_fatal("bb_realloc", "out of memory allocating %zu bytes", n);
	return p;
}
char *bb_strdup(const char *s)
{
	size_t l = strlen(s);
	char *p = bb_malloc(l + 1);
	memcpy(p, s, l + 1);
	return p;
}

double bb_cputime(void)
{
	struct rusage r;
	getrusage(RUSAGE_SELF, &r);
	return r.ru_utime.tv_sec + r.ru_stime.tv_sec + 1e-6 * (r.ru_utime.tv_usec + r.ru_stime.tv_usec);
}
double bb_realtime(void)
{
	struct timeval tp;
	gettimeofday(&tp, 0);
	return tp.tv_sec + tp.tv_usec * 1e-6;
}

/* ---- sorts on plain keys ---- */
#define u64_lt(a, b) ((a) < (b))
BB_SORT_DEFINE(, bb_sort_u64, uint64_t, u64_lt)
#define p64_lt(a, b) ((a).x < (b).x || ((a).x == (b).x && (a).y < (b).y))
BB_SORT_DEFINE(, bb_sort_pair64, bb_pair64_t, p64_lt)

/* ---- parallel loops on ONE shared pool of worker threads ----
 * Several batches (lanes) are in flight at once and each issues parallel loops; if every lane had its own
 * threads the process would oversubscribe the CPUs it is allowed to use (containers with a CFS quota then
 * throttle ALL threads for the rest of the period).  So there is one pool of `nt` workers; a loop is a job
 * record on a shared list, workers take chunks from any active job, and the caller works on its own job and
 * waits for it.  Worker ids are 0..nt-1, the caller of lane L uses id BB_MAX_WORKERS+L (per-id scratch arrays
 * are sized with bb_parallel_ids()). */
#define BB_MAX_WORKERS 256
#define BB_MAX_LANES 8
typedef struct pjob {
	void (*fn)(void *, long, int);
	void *data;
	long n, chunk, n_chunks;
	volatile long next, done;
	volatile int refs;            /* workers currently holding this record */
	struct pjob *link;
} pjob_t;

static struct {
	pthread_mutex_t mu;
	pthread_cond_t cv_work, cv_done;
	pjob_t *jobs;
	int n_workers;
	pthread_t th[BB_MAX_WORKERS];
} g_pool = { PTHREAD_MUTEX_INITIALIZER, PTHREAD_COND_INITIALIZER, PTHREAD_COND_INITIALIZER, 0, 0, {0} };

/* CPUs this process may really use: the affinity mask, capped by a cgroup CPU quota (containers) */
int bb_effective_cpus(void)
{
	int n = 0;
	FILE *f;
	cpu_set_t set;
	if (sched_getaffinity(0, sizeof(set), &set) == 0) n = CPU_COUNT(&set);
	if (n < 1) n = (int)sysconf(_SC_NPROCESSORS_ONLN);
	if (n < 1) n = 1;
	if ((f = fopen("/sys/fs/cgroup/cpu.max", "r")) != 0) {          /* cgroup v2: "<quota|max> <period>" */
		char q[32]; long period = 0;
		if (fscanf(f, "%31s %ld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) { long c = (atol(q) + period - 1) / period; if (c >= 1 && c < n) n = (int)c; }
		fclose(f);
	} else if ((f = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) != 0) {   /* cgroup v1 */
		long quota = -1, period = 0;
		FILE *g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r");
		if (fscanf(f, "%ld", &quota) != 1) quota = -1;
		if (g) { if (fscanf(g, "%ld", &period) != 1) period = 0; fclose(g); }
		if (quota > 0 && period > 0) { long c = (quota + period - 1) / period; if (c >= 1 && c < n) n = (int)c; }
		fclose(f);
	}
	return n;
}

int bb_parallel_ids(void) { return BB_MAX_WORKERS + BB_MAX_LANES; }

/* BWA_B200_PROFILE: thread-CPU seconds per loop body, printed by bb_parallel_report() */
static struct { void (*fn)(void *, long, int); const char *name; double cpu; long calls; } g_pstat[32];
static int g_pstat_on = -1;
static pthread_mutex_t g_pstat_mu = PTHREAD_MUTEX_INITIALIZER;
static double thread_cpu(void) { struct timespec ts; clock_gettime(CLOCK_THREAD_CPUTIME_ID, &ts); return ts.tv_sec + 1e-9 * ts.tv_nsec; }
static void pstat_add(void (*fn)(void *, long, int), double dt, long items)
{
	int i;
	pthread_mutex_lock(&g_pstat_mu);
	for (i = 0; i < 32 && g_pstat[i].fn && g_pstat[i].fn != fn; ++i) {}
	if (i < 32) { g_pstat[i].fn = fn; g_pstat[i].cpu += dt; g_pstat[i].calls += items; }
	pthread_mutex_unlock(&g_pstat_mu);
}
void bb_parallel_name(void (*fn)(void *, long, int), const char *name)
{
	int i;
	pthread_mutex_lock(&g_pstat_mu);
	for (i = 0; i < 32 && g_pstat[i].fn && g_pstat[i].fn != fn; ++i) {}
	if (i < 32) { g_pstat[i].fn = fn; g_pstat[i].name = name; }
	pthread_mutex_unlock(&g_pstat_mu);
}
void bb_parallel_report(void)
{
	int i;
	if (__atomic_load_n(&g_pstat_on, __ATOMIC_RELAXED) <= 0) return;
	for (i = 0; i < 32 && g_pstat[i].fn; ++i) {
		fprintf(stderr, "[prof] loop %-14s %8.3f CPU-s %10ld items\n", g_pstat[i].name ? g_pstat[i].name : "?", g_pstat[i].cpu, g_pstat[i].calls);
		g_pstat[i].cpu = 0; g_pstat[i].calls = 0;
	}
}

static long job_run(pjob_t *j, int tid)   /* returns the number of chunks executed */
{
	long c = 0, items = 0;
	double t0 = 0;
	int prof = __atomic_load_n(&g_pstat_on, __ATOMIC_RELAXED);
	if (prof < 0) { prof = getenv("BWA_B200_PROFILE") != 0; __atomic_store_n(&g_pstat_on, prof, __ATOMIC_RELAXED); }
	if (prof) t0 = thread_cpu();
	for (;;) {
		long b = __sync_fetch_and_add(&j->next, j->chunk), e, i;
		if (b >= j->n) break;
		e = b + j->chunk < j->n ? b + j->chunk : j->n;
		for (i = b; i < e; ++i) j->fn(j->data, i, tid);
		++c; items += e - b;
	}
	if (prof && items) pstat_add(j->fn, thread_cpu() - t0, items);
	return c;
}

static void *pool_worker(void *a_)
{
	int tid = (int)(long)a_;
	pthread_mutex_lock(&g_pool.mu);
	for (;;) {
		pjob_t *j;
		long c;
		for (j = g_pool.jobs; j; j = j->link) if (__atomic_load_n(&j->next, __ATOMIC_RELAXED) < j->n) break;
		if (!j) { pthread_cond_wait(&g_pool.cv_work, &g_pool.mu); continue; }
		++j->refs;
		pthread_mutex_unlock(&g_pool.mu);
		c = job_run(j, tid);
		pthread_mutex_lock(&g_pool.mu);
		j->done += c; --j->refs;
		if (j->done == j->n_chunks && j->refs == 0) pthread_cond_broadcast(&g_pool.cv_done);
	}
	return 0;
}

void bb_parallel_for(int nt, void (*fn)(void *, long, int), void *data, long n) { bb_parallel_for_lane(0, nt, fn, data, n); }

void bb_parallel_for_lane(int lane, int nt, void (*fn)(void *, long, int), void *data, long n)
{
	pjob_t job, **pp;
	long c;
	if (n <= 0) return;
	if (nt < 1) nt = 1;
	if (nt > BB_MAX_WORKERS) nt = BB_MAX_WORKERS;
	if (lane < 0 || lane >= BB_MAX_LANES) lane = 0;
	if (nt == 1 || n == 1) { long i; for (i = 0; i < n; ++i) fn(data, i, BB_MAX_WORKERS + lane); return; }
	job.fn = fn; job.data = data; job.n = n; job.next = 0; job.done = 0; job.refs = 0;
	job.chunk = n / (nt * 8L); if (job.chunk < 1) job.chunk = 1; if (job.chunk > 512) job.chunk = 512;
	job.n_chunks = (n + job.chunk - 1) / job.chunk;
	pthread_mutex_lock(&g_pool.mu);
	while (g_pool.n_workers < nt - 1) {   /* the caller is the nt-th participant */
		int t = g_pool.n_workers;
		if (pthread_create(&g_pool.th[t], 0, pool_worker, (void *)(long)t) != 0) bb_fatal("bb_parallel_for", "pthread_create failed");
		pthread_detach(g_pool.th[t]);
		++g_pool.n_workers;
	}
	job.link = g_pool.jobs; g_pool.jobs = &job;
	pthread_cond_broadcast(&g_pool.cv_work);
	pthread_mutex_unlock(&g_pool.mu);
	c = job_run(&job, BB_MAX_WORKERS + lane);
	pthread_mutex_lock(&g_pool.mu);
	job.done += c;
	while (job.done < job.n_chunks || job.refs > 0) pthread_cond_wait(&g_pool.cv_done, &g_pool.mu);
	for (pp = &g_pool.jobs; *pp; pp = &(*pp)->link) if (*pp == &job) { *pp = job.link; break; }
	pthread_mutex_unlock(&g_pool.mu);
}

void bb_mbox_init(bb_mbox_t *m) { pthread_mutex_init(&m->mu, 0); pthread_cond_init(&m->cv, 0); m->slot = 0; m->closed = 0; }
void bb_mbox_put(bb_mbox_t *m, void *item)
{
	pthread_mutex_lock(&m->mu);
	while (m->slot) pthread_cond_wait(&m->cv, &m->mu);
	m->slot = item;
	if (!item) m->closed = 1;
	pthread_cond_broadcast(&m->cv);
	pthread_mutex_unlock(&m->mu);
}
void *bb_mbox_get(bb_mbox_t *m)
{
	void *item;
	pthread_mutex_lock(&m->mu);
	while (!m->slot && !m->closed) pthread_cond_wait(&m->cv, &m->mu);
	item = m->slot; m->slot = 0;
	pthread_cond_broadcast(&m->cv);
	pthread_mutex_unlock(&m->mu);
	return item;
}

struct bb_pipe {
	const bb_pipe_ops_t *ops;
	void *run;
	bb_mbox_t to_dev, to_write;
	double wait_read, wait_dev;   /* time the reader and the device stage spent blocked in a hand-off */
	bb_pipe_busy_t busy;
};

static void pipe_put(bb_mbox_t *m, void *item, double *wait)
{
	const double t0 = bb_realtime();
	bb_mbox_put(m, item);
	*wait += bb_realtime() - t0;
}
static void *pipe_get(bb_mbox_t *m, double *wait)
{
	const double t0 = bb_realtime();
	void *item = bb_mbox_get(m);
	*wait += bb_realtime() - t0;
	return item;
}
void bb_pipe_to_device(bb_pipe_t *p, void *item) { pipe_put(&p->to_dev, item, &p->wait_read); }
void bb_pipe_to_writer(bb_pipe_t *p, void *item) { pipe_put(&p->to_write, item, &p->wait_dev); }

static void *pipe_reader(void *arg)
{
	bb_pipe_t *p = arg;
	const double t0 = bb_realtime();
	p->ops->read(p, p->run);
	p->busy.read = bb_realtime() - t0 - p->wait_read;
	bb_mbox_put(&p->to_dev, 0);
	return 0;
}

static void *pipe_writer(void *arg)
{
	bb_pipe_t *p = arg;
	const double t0 = bb_realtime();
	double wait = 0;
	void *item;
	while ((item = pipe_get(&p->to_write, &wait)) != 0) p->ops->write(p->run, item);
	p->busy.write = bb_realtime() - t0 - wait;
	return 0;
}

void bb_pipe_run(const bb_pipe_ops_t *ops, void *run, bb_pipe_busy_t *busy)
{
	bb_pipe_t p;
	pthread_t th_r, th_w;
	double t0;
	void *item;
	memset(&p, 0, sizeof(p));
	p.ops = ops; p.run = run;
	bb_mbox_init(&p.to_dev); bb_mbox_init(&p.to_write);
	if (pthread_create(&th_r, 0, pipe_reader, &p) != 0 || pthread_create(&th_w, 0, pipe_writer, &p) != 0) bb_fatal("bb_pipe_run", "pthread_create failed");
	t0 = bb_realtime();
	while ((item = pipe_get(&p.to_dev, &p.wait_dev)) != 0) ops->device(&p, run, item);
	p.busy.device = bb_realtime() - t0 - p.wait_dev;
	bb_mbox_put(&p.to_write, 0);
	pthread_join(th_r, 0);
	pthread_join(th_w, 0);
	*busy = p.busy;
}

/* bwa_cal_maxdiff (bwtaln.c:42-54): the smallest k with P(more than k errors in l bases) < thres for Poisson(l*err) errors, in the
 * reference's double expression order and with its int factorial, which wraps past 12! (then k comes out of the wrapped values,
 * as in the reference binary) */
int bb_cal_maxdiff(int l, double err, double thres)
{
	const double elambda = exp(-l * err);
	double sum = elambda, y = 1.0;
	int k, x = 1;
	for (k = 1; k < 1000; ++k) {
		y *= l * err;
		x = (int)((unsigned)x * (unsigned)k);
		sum += elambda * y / x;
		if (1.0 - sum < thres) return k;
	}
	return 2;
}
