/*
 * xf_oracle.c -- TEST INFRASTRUCTURE (CPU oracle), never linked into or called by the
 * product library.  Built by __graft_entry__.build() into tests/libm3tsz_xf_oracle.so and
 * bound by tests/xf_oracle_lib.py; self-contained (it shares no code with oracle/ or
 * tests/agg_oracle.c).
 *
 * Restates what m3tsz_aggregate_tiles_transform does to the value of every flushed window:
 * src/metrics/transformation/{unary,binary,unary_multi}.go and GenericElem.processValue
 * (src/aggregator/aggregator/generic_elem.go:804-950).  Pinned by
 * tests/golden/m3tsz_transform_goldens.json.  NaN payloads are the x86-64 SSE ones, as in Go on
 * amd64.  Build with -ffp-contract=off: every multiply and add is rounded on its own.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

static double f64_from_bits_q(uint64_t b) {
  double d;
  memcpy(&d, &b, 8);
  return d;
}

/* ------------------------------------------------------------------------- */
/* Transformations (transformation.Type ids 1..5) over a series' non-empty     */
/* windows, with the state that carries from one call to the next: the binary */
/* op's previous window (consumedValues) and one running sum per Add position.*/
/* Same layout as m3tsz_transform_state (96 bytes).                            */
/* ------------------------------------------------------------------------- */
typedef struct {
  int32_t has_prev;
  int32_t reserved0;
  int64_t prev_t;
  double prev_v;
  double sum[8];
  uint64_t reserved1;
} m3o_xf_state;

enum { XF_ABSOLUTE = 1, XF_PERSECOND = 2, XF_INCREASE = 3, XF_ADD = 4, XF_RESET = 5 };

/* emptyDatapoint, binary.go:28 (math.NaN()) */
static double xf_empty(void) { return f64_from_bits_q(0x7ff8000000000001ULL); }

/* perSecond, binary.go:49-60 */
double m3o_per_second(int64_t prev_t, double prev_v, int64_t t, double v) {
  if (prev_t >= t || isnan(prev_v) || isnan(v)) return xf_empty();
  double diff = v - prev_v;
  if (diff < 0) return xf_empty();
  return diff * 1e9 / (double)(int64_t)((uint64_t)t - (uint64_t)prev_t);
}

/* increase, binary.go:66-88 */
double m3o_increase(int64_t prev_t, double prev_v, int64_t t, double v) {
  if (prev_t >= t) return xf_empty();
  if (isnan(v)) return xf_empty();
  if (isnan(prev_v)) prev_v = 0;
  double diff = v - prev_v;
  if (diff < 0) return xf_empty();
  return diff;
}

/* One window (end t, value *v) through ops[0..n_ops); returns the Reset datapoint's timestamp (0: none). */
int64_t m3o_transform_window(const int32_t *ops, size_t n_ops, int64_t step, m3o_xf_state *st, int64_t t,
                             double *v) {
  int64_t extra_t = 0;
  for (size_t k = 0; k < n_ops; k++) {
    switch (ops[k]) {
      case XF_ABSOLUTE: *v = fabs(*v); break;
      case XF_ADD:
        if (!isnan(*v)) st->sum[k] += *v;
        *v = st->sum[k];
        break;
      case XF_PERSECOND:
      case XF_INCREASE: {
        int64_t pt = st->has_prev ? st->prev_t : 0;
        double pv = st->has_prev ? st->prev_v : xf_empty();
        double in = *v;
        *v = ops[k] == XF_PERSECOND ? m3o_per_second(pt, pv, t, in) : m3o_increase(pt, pv, t, in);
        st->has_prev = 1;
        st->prev_t = t;
        st->prev_v = in;
        break;
      }
      case XF_RESET: {
        int64_t rw = (int64_t)fmax((double)(step / 2), 1.0);
        extra_t = (int64_t)((uint64_t)t + (uint64_t)rw);
        break;
      }
      default: break;
    }
  }
  return extra_t;
}

/* The flush of n non-empty windows (t[i], v[i]) in order: each window's result, then its Reset datapoint (value 0,
 * unless its timestamp is 0); with discard_nan a NaN result writes neither.  Outputs need 2 * n entries.  Returns
 * the number written. */
size_t m3o_transform_series(const int32_t *ops, size_t n_ops, int discard_nan, int64_t step, m3o_xf_state *st,
                            const int64_t *t, const double *v, size_t n, int64_t *t_out, double *v_out) {
  size_t k = 0;
  for (size_t i = 0; i < n; i++) {
    double x = v[i];
    int64_t extra_t = m3o_transform_window(ops, n_ops, step, st, t[i], &x);
    if (discard_nan && isnan(x)) continue;
    t_out[k] = t[i];
    v_out[k++] = x;
    if (extra_t != 0) {
      t_out[k] = extra_t;
      v_out[k++] = 0.0;
    }
  }
  return k;
}
