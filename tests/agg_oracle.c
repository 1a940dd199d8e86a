/*
 * agg_oracle.c -- TEST INFRASTRUCTURE (CPU oracle), never linked into or called by the
 * product library.  Built by __graft_entry__.build() into tests/libm3tsz_agg_oracle.so and
 * bound by tests/agg_oracle_lib.py; self-contained (it shares no code with oracle/).
 *
 * Restates what the fused downsample modes 4 / 5 and the tile aggregation of
 * m3tsz_aggregate_tiles_ex compute, from src/aggregator/aggregation in the reference:
 * gauge.go:74-165 (with HasExpensiveAggregations), counter.go:44-134, common.go:29-37.
 * Pinned by the reference's test tables in tests/golden/m3tsz_agg_goldens.json.
 * Build with -ffp-contract=off: every multiply and add is rounded on its own, as in Go on amd64.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------- */
/* The rest of src/aggregator/aggregation that the fused downsample and the   */
/* tile aggregation cover: the Gauge with expensive aggregations (sumSq,      */
/* gauge.go:74-103), the Counter (counter.go:44-78) and stdev (common.go:29-37).*/
/* Windows as m3o_downsample_series: w = floor((ts - range_start) / window),  */
/* datapoints outside [0, n_windows) ignored, stream order kept.              */
/* ------------------------------------------------------------------------- */

static double f64_from_bits_q(uint64_t b) {
  double d;
  memcpy(&d, &b, 8);
  return d;
}

/* int64(v) as Go compiles it on amd64 (CVTTSD2SQ): truncation toward zero, and
 * NaN / +-Inf / anything outside [-2^63, 2^63) is the "integer indefinite"
 * 0x8000000000000000. */
int64_t m3o_go_int64(double v) {
  if (!(v >= -9223372036854775808.0 && v < 9223372036854775808.0)) return INT64_MIN;
  return (int64_t)v;
}

/* common.go:29-37.  div in int64 (wrapping); num and the quotient rounded per
 * operation (-ffp-contract=off); sqrt of a negative num is NaN, as math.Sqrt. */
double m3o_stdev(int64_t count, double sum_sq, double sum) {
  int64_t div = (int64_t)((uint64_t)count * (uint64_t)(count - 1));
  if (div == 0) return 0.0;
  double num = (double)count * sum_sq - sum * sum;
  return sqrt(num / (double)div);
}

/* Gauge with HasExpensiveAggregations: the outputs of m3o_downsample_series plus
 * lastAt (0 for an empty window) and sumSq (0 for an empty window). */
void m3o_downsample_gauge_ex(const int64_t *ts, const double *vals, size_t n, int64_t range_start_ns,
                             int64_t window_ns, size_t n_windows, double *sum, int64_t *count, double *min,
                             double *max, double *last, int64_t *last_at, double *sum_sq) {
  const double nan = f64_from_bits_q(0x7ff8000000000001ULL); /* Go math.NaN() */
  uint8_t *has_last = (uint8_t *)calloc(n_windows ? n_windows : 1, 1);
  for (size_t w = 0; w < n_windows; w++) {
    sum[w] = 0;
    count[w] = 0;
    min[w] = nan;
    max[w] = nan;
    last[w] = 0;
    last_at[w] = 0;
    sum_sq[w] = 0;
  }
  for (size_t i = 0; i < n; i++) {
    int64_t rel = ts[i] - range_start_ns;
    int64_t w = rel / window_ns;
    if (rel % window_ns != 0 && rel < 0) w--;
    if (w < 0 || (uint64_t)w >= (uint64_t)n_windows) continue;
    double v = vals[i];
    if (!has_last[w] || ts[i] > last_at[w]) { /* lastAt.IsZero() || timestamp.After(lastAt) */
      has_last[w] = 1;
      last_at[w] = ts[i];
      last[w] = v;
    }
    count[w]++;
    if (isnan(v)) continue;
    sum[w] += v;
    if (isnan(max[w]) || max[w] < v) max[w] = v;
    if (isnan(min[w]) || min[w] > v) min[w] = v;
    sum_sq[w] += v * v;
  }
  free(has_last);
}

/* Counter fed int64(value): int64 sum / count / min / max / sumSq, wrapping like Go.
 * Empty window: sum 0, count 0, min MaxInt64, max MinInt64, sumSq 0. */
void m3o_downsample_counter(const int64_t *ts, const double *vals, size_t n, int64_t range_start_ns,
                            int64_t window_ns, size_t n_windows, int64_t *sum, int64_t *count, int64_t *min,
                            int64_t *max, int64_t *sum_sq) {
  for (size_t w = 0; w < n_windows; w++) {
    sum[w] = 0;
    count[w] = 0;
    min[w] = INT64_MAX;
    max[w] = INT64_MIN;
    sum_sq[w] = 0;
  }
  for (size_t i = 0; i < n; i++) {
    int64_t rel = ts[i] - range_start_ns;
    int64_t w = rel / window_ns;
    if (rel % window_ns != 0 && rel < 0) w--;
    if (w < 0 || (uint64_t)w >= (uint64_t)n_windows) continue;
    int64_t x = m3o_go_int64(vals[i]);
    sum[w] = (int64_t)((uint64_t)sum[w] + (uint64_t)x);
    count[w]++;
    if (max[w] < x) max[w] = x;
    if (min[w] > x) min[w] = x;
    sum_sq[w] = (int64_t)((uint64_t)sum_sq[w] + (uint64_t)x * (uint64_t)x);
  }
}

/* Gauge.ValueOf, gauge.go:144-165, every type (8 SumSq, 9 Stdev included) */
double m3o_gauge_value_of_ex(int agg_type, double sum, int64_t count, double min, double max, double last,
                             double sum_sq) {
  switch (agg_type) {
    case 8: return sum_sq;
    case 9: return m3o_stdev(count, sum_sq, sum);
    case 1: return last;
    case 2: return min;
    case 3: return max;
    case 4: return count == 0 ? 0.0 : sum / (double)count; /* Mean, gauge.go:117-122 */
    case 6: return (double)count;
    case 7: return sum;
    default: return 0.0;
  }
}

/* Counter.ValueOf, counter.go:112-134 */
double m3o_counter_value_of(int agg_type, int64_t sum, int64_t count, int64_t min, int64_t max, int64_t sum_sq) {
  switch (agg_type) {
    case 2: return (double)min;
    case 3: return (double)max;
    case 4: return count == 0 ? 0.0 : (double)sum / (double)count;
    case 6: return (double)count;
    case 7: return (double)sum;
    case 8: return (double)sum_sq;
    case 9: return m3o_stdev(count, (double)sum_sq, (double)sum);
    default: return 0.0;
  }
}

/* m3o_aggregate_tiles_series for metric_type 3 (Gauge, with sumSq) or 1 (Counter) */
size_t m3o_aggregate_tiles_series_ex(const int64_t *ts, const double *vals, size_t n, int64_t start_ns,
                                     int64_t step_ns, size_t n_windows, int metric_type, int agg_type,
                                     int64_t *ts_out, double *val_out) {
  const size_t nw = n_windows ? n_windows : 1;
  double *f = (double *)malloc(sizeof(double) * 5 * nw);
  int64_t *g = (int64_t *)malloc(sizeof(int64_t) * 6 * nw);
  int64_t *count = g;
  if (metric_type == 1)
    m3o_downsample_counter(ts, vals, n, start_ns, step_ns, n_windows, g + nw, count, g + 2 * nw, g + 3 * nw,
                           g + 4 * nw);
  else
    m3o_downsample_gauge_ex(ts, vals, n, start_ns, step_ns, n_windows, f, count, f + nw, f + 2 * nw, f + 3 * nw,
                            g + 5 * nw, f + 4 * nw);
  size_t k = 0;
  for (size_t w = 0; w < n_windows; w++) {
    if (count[w] == 0) continue;
    ts_out[k] = start_ns + (int64_t)(w + 1) * step_ns;
    val_out[k] = metric_type == 1
                     ? m3o_counter_value_of(agg_type, g[nw + w], count[w], g[2 * nw + w], g[3 * nw + w],
                                            g[4 * nw + w])
                     : m3o_gauge_value_of_ex(agg_type, f[w], count[w], f[nw + w], f[2 * nw + w], f[3 * nw + w],
                                             f[4 * nw + w]);
    k++;
  }
  free(f);
  free(g);
  return k;
}
