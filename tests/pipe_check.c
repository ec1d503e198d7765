/* pipe_check.c -- drives the reader/device/writer pipeline and the closing mailbox of bb_util.c with batches flowing, for
 * tests/test_pipe.py, which builds it under ThreadSanitizer.  Exit 0: every check held.
 *
 *   pipe    the reader hands on numbered ranges, cutting some into single numbers; the device stage hands on 0, 1 or 3 ranges per
 *           input; the writer checks that the numbers arrive in strictly increasing order and that none is lost
 *   mbox    one producer, several consumers of one mailbox that the producer closes (the way `mem`'s aligner threads share it) */
#include <stdio.h>
#include <stdlib.h>
#include <pthread.h>
#include "bb_util.h"

#define N_NUMBERS 5000
#define N_CONSUMERS 4

typedef struct { int beg, end; long sum; } range_t;   /* the numbers [beg, end); sum: the device stage's checksum of them */

typedef struct {
	unsigned rng;
	int n_dropped;       /* device stage */
	int next, n_written; /* writer: the smallest number that may come next, numbers seen */
	int bad;
} pipe_run_t;

static range_t *range_new(int beg, int end)
{
	range_t *x = malloc(sizeof(*x));
	x->beg = beg; x->end = end; x->sum = -1;
	return x;
}

static void read_all(bb_pipe_t *p, void *run)
{
	pipe_run_t *r = run;
	int beg = 0;
	while (beg < N_NUMBERS) {
		int len = 1 + (int)((r->rng = r->rng * 1103515245u + 12345u) >> 16) % 9, end = beg + len < N_NUMBERS ? beg + len : N_NUMBERS;
		if (beg % 4 == 0) for (int i = beg; i < end; ++i) bb_pipe_to_device(p, range_new(i, i + 1));   /* a group cut into batches */
		else bb_pipe_to_device(p, range_new(beg, end));
		beg = end;
	}
}

static void run_device(bb_pipe_t *p, void *run, void *item)
{
	pipe_run_t *r = run;
	range_t *x = item;
	const int mode = x->beg % 3;   /* 0: drop, 1: hand on, 2: hand on in three parts (some may be empty) */
	if (mode == 0) { r->n_dropped += x->end - x->beg; free(x); return; }
	if (mode == 1) {
		x->sum = 0;
		for (int i = x->beg; i < x->end; ++i) x->sum += i;
		bb_pipe_to_writer(p, x);
		return;
	}
	const int a = x->beg + (x->end - x->beg) / 3, b = x->beg + 2 * (x->end - x->beg) / 3;
	const int cut[4] = { x->beg, a, b, x->end };
	for (int k = 0; k < 3; ++k) {
		range_t *y = range_new(cut[k], cut[k + 1]);
		y->sum = 0;
		for (int i = y->beg; i < y->end; ++i) y->sum += i;
		bb_pipe_to_writer(p, y);
	}
	free(x);
}

static void write_range(void *run, void *item)
{
	pipe_run_t *r = run;
	range_t *x = item;
	long sum = 0;
	for (int i = x->beg; i < x->end; ++i) {
		if (i < r->next) { fprintf(stderr, "FAIL: number %d after %d\n", i, r->next - 1); r->bad = 1; }
		r->next = i + 1;
		sum += i;
		++r->n_written;
	}
	if (sum != x->sum) { fprintf(stderr, "FAIL: range [%d, %d) has checksum %ld, not %ld\n", x->beg, x->end, x->sum, sum); r->bad = 1; }
	free(x);
}

static int check_pipe(void)
{
	static const bb_pipe_ops_t ops = { read_all, run_device, write_range };
	pipe_run_t r = { 7u, 0, 0, 0, 0 };
	bb_pipe_busy_t busy;
	const double t0 = bb_realtime();
	double wall;
	bb_pipe_run(&ops, &r, &busy);
	wall = bb_realtime() - t0;
	if (r.n_written + r.n_dropped != N_NUMBERS) { fprintf(stderr, "FAIL: %d numbers written, %d dropped, of %d\n", r.n_written, r.n_dropped, N_NUMBERS); r.bad = 1; }
	if (r.n_written == 0 || r.n_dropped == 0) { fprintf(stderr, "FAIL: every number written or every number dropped\n"); r.bad = 1; }
	if (busy.read < 0 || busy.device < 0 || busy.write < 0 || busy.read > wall || busy.device > wall || busy.write > wall) {
		fprintf(stderr, "FAIL: busy times %.6f %.6f %.6f s outside [0, %.6f]\n", busy.read, busy.device, busy.write, wall);
		r.bad = 1;
	}
	printf("pipe: %d numbers written, %d dropped\n", r.n_written, r.n_dropped);
	return r.bad;
}

typedef struct { bb_mbox_t *box; long sum; int n; } consumer_t;

static void *consume(void *arg)
{
	consumer_t *c = arg;
	int *v;
	while ((v = bb_mbox_get(c->box)) != 0) { c->sum += *v; ++c->n; free(v); }
	return 0;
}

static int check_mbox(void)
{
	bb_mbox_t box;
	pthread_t th[N_CONSUMERS];
	consumer_t c[N_CONSUMERS];
	long sum = 0;
	int i, n = 0;
	bb_mbox_init(&box);
	for (i = 0; i < N_CONSUMERS; ++i) { c[i].box = &box; c[i].sum = 0; c[i].n = 0; pthread_create(&th[i], 0, consume, &c[i]); }
	for (i = 1; i <= N_NUMBERS; ++i) { int *v = malloc(sizeof(*v)); *v = i; bb_mbox_put(&box, v); }
	bb_mbox_put(&box, 0);   /* closes the box: every consumer stops */
	for (i = 0; i < N_CONSUMERS; ++i) { pthread_join(th[i], 0); sum += c[i].sum; n += c[i].n; }
	if (bb_mbox_get(&box) != 0) { fprintf(stderr, "FAIL: a get after the close returned an item\n"); return 1; }
	if (n != N_NUMBERS || sum != (long)N_NUMBERS * (N_NUMBERS + 1) / 2) { fprintf(stderr, "FAIL: consumers took %d items summing to %ld\n", n, sum); return 1; }
	printf("mbox: %d items over %d consumers\n", n, N_CONSUMERS);
	return 0;
}

int main(void)
{
	int bad = check_pipe();
	bad |= check_mbox();
	return bad;
}
