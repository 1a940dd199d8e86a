/*
 * elem_oracle.c -- TEST INFRASTRUCTURE (CPU oracle), never linked into or called by the
 * product library.  Built by __graft_entry__.build() into tests/libm3tsz_elem_oracle.so and
 * bound by tests/elem_oracle_lib.py; self-contained (it shares no code with oracle/,
 * tests/agg_oracle.c or tests/xf_oracle.c).
 *
 * Restates what m3tsz_aggregate_tiles_types does with the window values of an element that
 * has several aggregation types: GenericElem.processValue's loop over e.aggTypes
 * (src/aggregator/aggregator/generic_elem.go:830-889) with the transformations of
 * src/metrics/transformation/{unary,binary,unary_multi}.go.  Per window, types in order:
 *   - the Add op at position i is one closure (unary.go:46-54): one sum shared by all types;
 *   - the binary op reads prev = (the previous window's end, consumedValues[j]) and records
 *     consumedValues[j] = its input; the previous window's end is the element's;
 *   - DiscardNaNAggregatedValues drops only that type's datapoint (and its Reset datapoint).
 * Pinned by tests/golden/m3tsz_element_types_goldens.json.  NaN payloads are the x86-64 SSE
 * ones, as in Go on amd64.  Build with -ffp-contract=off.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

/* Same layout as m3tsz_element_state (160 bytes). */
typedef struct {
  int32_t has_prev;      /* a non-empty window has been through the binary op */
  int32_t reserved0;
  int64_t prev_t;        /* its end */
  double prev_v0;        /* consumedValues[0] */
  double sum[8];         /* sum[i]: the Add op at position i, shared by the types */
  uint64_t reserved1;
  double prev_v_more[7]; /* consumedValues[1..7] */
  uint64_t reserved2;
} m3o_elem_state;

enum { EL_ABSOLUTE = 1, EL_PERSECOND = 2, EL_INCREASE = 3, EL_ADD = 4, EL_RESET = 5 };

static double el_bits(uint64_t b) {
  double d;
  memcpy(&d, &b, 8);
  return d;
}

/* emptyDatapoint, binary.go:28 (math.NaN()) */
static double el_empty(void) { return el_bits(0x7ff8000000000001ULL); }

/* binary.go:49-60 */
static double el_per_second(int64_t prev_t, double prev_v, int64_t t, double v) {
  if (prev_t >= t || isnan(prev_v) || isnan(v)) return el_empty();
  double diff = v - prev_v;
  if (diff < 0) return el_empty();
  return diff * 1e9 / (double)(int64_t)((uint64_t)t - (uint64_t)prev_t);
}

/* binary.go:66-88 */
static double el_increase(int64_t prev_t, double prev_v, int64_t t, double v) {
  if (prev_t >= t || isnan(v)) return el_empty();
  if (isnan(prev_v)) prev_v = 0;
  double diff = v - prev_v;
  if (diff < 0) return el_empty();
  return diff;
}

static double *el_prev_v(m3o_elem_state *st, size_t j) { return j == 0 ? &st->prev_v0 : &st->prev_v_more[j - 1]; }

/* The flush of n non-empty windows of an element with n_types types: window i ends at t[i] and type j's value
 * there is v[i * n_types + j].  Type j's datapoints go to t_out / v_out + j * 2n (2n entries each), their count to
 * n_out[j]. */
void m3o_element_series(const int32_t *ops, size_t n_ops, int discard_nan, int64_t step, size_t n_types,
                        m3o_elem_state *st, const int64_t *t, const double *v, size_t n, int64_t *t_out,
                        double *v_out, size_t *n_out) {
  for (size_t j = 0; j < n_types; j++) n_out[j] = 0;
  for (size_t i = 0; i < n; i++) {
    /* cState.prevStartTime: the previous window, the same for every type of this one */
    const int has_prev = st->has_prev;
    const int64_t prev_t = st->prev_t;
    int binary = 0;
    for (size_t j = 0; j < n_types; j++) {
      double x = v[i * n_types + j];
      int64_t extra_t = 0;
      for (size_t k = 0; k < n_ops; k++) {
        switch (ops[k]) {
          case EL_ABSOLUTE: x = fabs(x); break;
          case EL_ADD:
            if (!isnan(x)) st->sum[k] += x;
            x = st->sum[k];
            break;
          case EL_PERSECOND:
          case EL_INCREASE: {
            const int64_t pt = has_prev ? prev_t : 0;
            const double pv = has_prev ? *el_prev_v(st, j) : el_empty();
            const double in = x;
            x = ops[k] == EL_PERSECOND ? el_per_second(pt, pv, t[i], in) : el_increase(pt, pv, t[i], in);
            *el_prev_v(st, j) = in;
            binary = 1;
            break;
          }
          case EL_RESET: extra_t = (int64_t)((uint64_t)t[i] + (uint64_t)(int64_t)fmax((double)(step / 2), 1.0)); break;
          default: break;
        }
      }
      if (discard_nan && isnan(x)) continue;
      int64_t *to = t_out + j * 2 * n;
      double *vo = v_out + j * 2 * n;
      to[n_out[j]] = t[i];
      vo[n_out[j]++] = x;
      if (extra_t != 0) {
        to[n_out[j]] = extra_t;
        vo[n_out[j]++] = 0.0;
      }
    }
    if (binary) {
      st->has_prev = 1;
      st->prev_t = t[i];
    }
  }
}
