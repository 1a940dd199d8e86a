/*
 * rollup_oracle.c -- TEST INFRASTRUCTURE (CPU oracle), never linked into or called by the
 * product library.  Built by __graft_entry__.build() into tests/libm3tsz_rollup_oracle.so and
 * bound by tests/rollup_oracle_lib.py; self-contained (it shares no code with oracle/ or the
 * other test oracles).
 *
 * Restates the fold of m3tsz_aggregate_tiles_rollup: one window of a rollup element, which
 * receives the forwarded values of the group's members in listed order, all at one timestamp,
 * through GenericElem.AddUnique (src/aggregator/aggregator/generic_elem.go:246-281) ->
 * Gauge.Update / Counter.Update (src/aggregator/aggregation/{gauge,counter}.go).  NaN payloads
 * are the x86-64 SSE ones, as in Go on amd64.  Build with -ffp-contract=off.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

static double ro_bits(uint64_t b) {
  double d;
  memcpy(&d, &b, 8);
  return d;
}

/* int64(float64) on amd64 (CVTTSD2SQ): truncation, MinInt64 for NaN and out of range */
static int64_t ro_go_int64(double v) {
  if (!(v >= -9223372036854775808.0 && v < 9223372036854775808.0)) return INT64_MIN;
  return (int64_t)v;
}

/* Gauge: NewGauge (gauge.go:45-51), then updateTotals (gauge.go:74-101) with one timestamp for every value: the first
 * value sets lastAt / last (lastAt.IsZero()), the others are not After it.  out: sum, min, max, last, sumSq; count. */
void m3o_rollup_gauge(const double *v, size_t n, double *out5, int64_t *count) {
  double sum = 0, mn = ro_bits(0x7ff8000000000001ULL), mx = ro_bits(0x7ff8000000000001ULL), last = 0, sq = 0;
  int64_t cnt = 0;
  for (size_t i = 0; i < n; i++) {
    const double x = v[i];
    if (i == 0) last = x;
    cnt++;
    if (isnan(x)) continue;
    sum += x;
    if (isnan(mx) || mx < x) mx = x;
    if (isnan(mn) || mn > x) mn = x;
    sq += x * x;
  }
  out5[0] = sum;
  out5[1] = mn;
  out5[2] = mx;
  out5[3] = last;
  out5[4] = sq;
  *count = cnt;
}

/* Counter: NewCounter (counter.go:44-50), then Update(int64(value)) (counter.go:52-78): int64 arithmetic that wraps.
 * out: sum, count, min, max, sumSq. */
void m3o_rollup_counter(const double *v, size_t n, int64_t *out5) {
  uint64_t sum = 0, sq = 0;
  int64_t mn = INT64_MAX, mx = INT64_MIN, cnt = 0;
  for (size_t i = 0; i < n; i++) {
    const int64_t x = ro_go_int64(v[i]);
    sum += (uint64_t)x;
    cnt++;
    if (mx < x) mx = x;
    if (mn > x) mn = x;
    sq += (uint64_t)x * (uint64_t)x;
  }
  out5[0] = (int64_t)sum;
  out5[1] = cnt;
  out5[2] = mn;
  out5[3] = mx;
  out5[4] = (int64_t)sq;
}
