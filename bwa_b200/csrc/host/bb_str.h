/* bb_str.h -- append-only text buffer used by the SAM emitter. */
#ifndef BB_STR_H
#define BB_STR_H
#include <stdint.h>
#include <string.h>
#include "bb_util.h"

typedef struct { size_t l, m; char *s; } bb_str_t;

static inline void bb_str_need(bb_str_t *s, size_t extra)
{
	size_t need = s->l + extra + 1;
	if (need > s->m) {
		size_t m = s->m ? s->m : 64;
		if (s->m == 0 && need > 64) m = (need + 31) & ~(size_t)31;   /* a caller's up-front estimate is taken as it is */
		while (m < need) m <<= 1;
		s->s = bb_realloc(s->s, m);
		s->m = m;
	}
}
static inline void bb_putc(bb_str_t *s, int c) { bb_str_need(s, 1); s->s[s->l++] = (char)c; s->s[s->l] = 0; }
static inline void bb_putsn(bb_str_t *s, const char *p, size_t n) { bb_str_need(s, n); memcpy(s->s + s->l, p, n); s->l += n; s->s[s->l] = 0; }
static inline void bb_puts(bb_str_t *s, const char *p) { bb_putsn(s, p, strlen(p)); }
/* a writer's output: once s holds at_least bytes, write them to stdout and empty s; at_least 0 writes the rest and frees s.  A short
 * write is fatal (`who` names the command). */
static inline void bb_str_write(bb_str_t *s, size_t at_least, const char *who)
{
	if (s->l && s->l >= at_least) {
		if (fwrite(s->s, 1, s->l, stdout) != s->l) bb_fatal(who, "fail to write the output");
		s->l = 0;
	}
	if (at_least == 0) { free(s->s); s->s = 0; s->m = 0; }
}
/* decimal text of a signed 64-bit value; identical digits to kputw/kputl (kstring.h:63-112) */
static inline void bb_putl(bb_str_t *s, int64_t v)
{
	char buf[24];
	int n = 0;
	uint64_t u = v < 0 ? (uint64_t)(-(v + 1)) + 1u : (uint64_t)v;
	do { buf[n++] = (char)('0' + u % 10); u /= 10; } while (u);
	if (v < 0) buf[n++] = '-';
	bb_str_need(s, (size_t)n);
	while (n) s->s[s->l++] = buf[--n];
	s->s[s->l] = 0;
}
/* the same digits at a raw write position with room for 21 characters; returns the position after them */
static inline char *bb_fmt_l(char *w, int64_t v)
{
	char buf[24];
	int n = 0;
	uint64_t u = v < 0 ? (uint64_t)(-(v + 1)) + 1u : (uint64_t)v;
	if (v >= 0 && u < 10) { *w++ = (char)('0' + u); return w; }
	do { buf[n++] = (char)('0' + u % 10); u /= 10; } while (u);
	if (v < 0) buf[n++] = '-';
	while (n) *w++ = buf[--n];
	return w;
}
#endif