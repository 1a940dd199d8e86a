/* CPU oracle of the aggregator's Timer: aggregation.Timer (aggregation/timer.go) over cm.Stream
 * (aggregation/quantile/cm/stream.go, heap.go, list.go), restated in C from the reference's semantics for the tests
 * of the Timer element sets.  Test infrastructure only; built by tests/host_build.build_c_oracle("timer") with
 * oracle/Makefile's flags (-ffp-contract=off: every operation rounded on its own, as amd64 Go).
 *
 * The list is a doubly linked list of heap-allocated samples (the reference's arena and free list are not observable);
 * the two pending heaps are growable arrays with the reference's push and in-place heapsort. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct sample {
  double value;
  int64_t num_ranks, delta;
  struct sample *prev, *next;
} sample;

typedef struct {
  double *a;
  size_t len, cap;
} fheap;

typedef struct {
  sample *head, *tail, *insert_cursor, *compress_cursor;
  size_t len;
  fheap buf_less, buf_more;
  const double *quantiles;
  size_t nq;
  double computed[32];
  int64_t num_values, compress_min_rank;
  int64_t counter, every;
  double eps;
} stream;

/* Go's int64(f) on amd64 (CVTTSD2SQ): truncation, 0x8000000000000000 for NaN and out of range */
static int64_t go_int64(double f) {
  if (!(f >= -9223372036854775808.0 && f < 9223372036854775808.0)) return INT64_MIN;
  return (int64_t)f;
}

static void heap_push(fheap *h, double v) {
  if (h->len == h->cap) {
    h->cap = h->cap ? 2 * h->cap : 16;
    h->a = (double *)realloc(h->a, h->cap * sizeof(double));
  }
  h->a[h->len++] = v;
  size_t i = h->len - 1;
  while (i > 0) {
    size_t parent = (i - 1) / 2;
    if (h->a[parent] <= h->a[i]) break;
    double t = h->a[parent];
    h->a[parent] = h->a[i];
    h->a[i] = t;
    i = parent;
  }
}

static void heap_sort_desc(fheap *h) {
  double *a = h->a;
  for (size_t n = h->len; n > 1; n--) {
    size_t last = n - 1, i = 0, smallest = 0;
    double t = a[0];
    a[0] = a[last];
    a[last] = t;
    for (;;) {
      size_t l = 2 * smallest + 1, r = l + 1;
      if (l < last && a[l] < a[smallest]) smallest = l;
      if (r < last && a[r] < a[smallest]) smallest = r;
      if (smallest == i) break;
      t = a[i];
      a[i] = a[smallest];
      a[smallest] = t;
      i = smallest;
    }
  }
}

static sample *new_sample(double v, int64_t delta) {
  sample *s = (sample *)calloc(1, sizeof(sample));
  s->value = v;
  s->num_ranks = 1;
  s->delta = delta;
  return s;
}

static void list_push_back(stream *st, sample *s) {
  s->prev = st->tail;
  s->next = NULL;
  if (!st->head)
    st->head = s;
  else
    st->tail->next = s;
  st->tail = s;
  st->len++;
}

static void list_insert_before(stream *st, sample *s, sample *mark) {
  sample *prev = mark->prev;
  if (!prev)
    st->head = s;
  else
    prev->next = s;
  mark->prev = s;
  s->next = mark;
  s->prev = prev;
  st->len++;
}

static void list_remove(stream *st, sample *s) {
  if (!s->prev)
    st->head = s->next;
  else
    s->prev->next = s->next;
  if (!s->next)
    st->tail = s->prev;
  else
    s->next->prev = s->prev;
  st->len--;
  free(s);
}

static void reset_insert_cursor(stream *st) {
  fheap t = st->buf_less;
  st->buf_less = st->buf_more;
  st->buf_more = t;
  st->insert_cursor = st->head;
}

static int64_t stream_threshold(const stream *st, int64_t rank) {
  int64_t mn = INT64_MAX;
  double eps = 2.0 * st->eps;
  for (size_t i = 0; i < st->nq; i++) {
    double q = st->quantiles[i];
    int64_t qm;
    if (rank >= go_int64(q * (double)st->num_values))
      qm = go_int64(eps * (double)rank / q);
    else
      qm = go_int64(eps * (double)(st->num_values - rank) / (1.0 - q));
    if (qm < mn) mn = qm;
  }
  return mn;
}

static void stream_insert(stream *st) {
  double comp_value = st->compress_cursor ? st->compress_cursor->value : NAN;
  heap_sort_desc(&st->buf_more);
  double *vals = st->buf_more.a;
  int64_t idx = (int64_t)st->buf_more.len - 1;
  while (st->insert_cursor) {
    sample *curr = st->insert_cursor;
    double ipv = curr->value;
    while (idx >= 0 && vals[idx] <= ipv) {
      double v = vals[idx--];
      list_insert_before(st, new_sample(v, curr->num_ranks + curr->delta - 1), curr);
      if (comp_value >= v) st->compress_min_rank++;
      st->num_values++;
    }
    st->insert_cursor = curr->next;
  }
  while (idx >= 0 && vals[idx] >= st->tail->value) {
    list_push_back(st, new_sample(vals[idx--], 0));
    st->num_values++;
  }
  st->buf_more.len = 0;
  reset_insert_cursor(st);
}

static void stream_compress(stream *st) {
  if (st->len < 3) return;
  if (!st->compress_cursor) {
    st->compress_cursor = st->tail->prev;
    st->compress_min_rank = st->num_values - 1 - st->compress_cursor->num_ranks;
    st->compress_cursor = st->compress_cursor->prev;
  }
  while (st->compress_cursor != st->head) {
    sample *curr = st->compress_cursor, *next = curr->next, *prev = curr->prev;
    int64_t max_rank = st->compress_min_rank + curr->num_ranks + curr->delta;
    int64_t threshold = stream_threshold(st, max_rank);
    st->compress_min_rank -= curr->num_ranks;
    if (curr->num_ranks + next->num_ranks + next->delta <= threshold) {
      if (st->insert_cursor == curr) st->insert_cursor = next;
      next->num_ranks += curr->num_ranks;
      list_remove(st, curr);
    }
    st->compress_cursor = prev;
  }
  st->compress_cursor = NULL;
}

static void stream_add_batch(stream *st, const double *v, size_t n) {
  if (n == 0) return;
  if (st->len == 0) {
    list_push_back(st, new_sample(v[0], 0));
    st->insert_cursor = st->head;
    st->num_values++;
    v++;
    n--;
  }
  double ipv = st->insert_cursor->value;
  int64_t counter = st->counter;
  for (size_t i = 0; i < n; i++) {
    if (v[i] < ipv)
      heap_push(&st->buf_less, v[i]);
    else
      heap_push(&st->buf_more, v[i]);
    if (counter == st->every) {
      stream_insert(st);
      stream_compress(st);
      counter = 0;
    }
    counter++;
  }
  st->counter = counter;
}

static void stream_flush(stream *st) {
  while (st->buf_less.len > 0 || st->buf_more.len > 0) {
    if (st->buf_more.len == 0) reset_insert_cursor(st);
    stream_insert(st);
    stream_compress(st);
  }
  /* calcQuantiles */
  if (st->nq == 0 || st->num_values == 0) return;
  if (st->num_values <= 3) {
    double buf[3];
    int64_t n = 0;
    for (sample *c = st->head; c; c = c->next) buf[n++] = c->value;
    for (size_t i = 0; i < st->nq; i++) {
      int64_t idx = go_int64(st->quantiles[i] * (double)n);
      if (idx >= n) idx = n - 1;
      st->computed[i] = buf[idx];
    }
    return;
  }
  int64_t rank[32], thr[32];
  for (size_t i = 0; i < st->nq; i++) {
    rank[i] = go_int64(ceil(st->quantiles[i] * (double)st->num_values));
    thr[i] = go_int64(ceil((double)stream_threshold(st, rank[i]) / 2.0));
  }
  int64_t min_rank = 0, max_rank = 0;
  size_t idx = 0;
  sample *curr = st->head, *prev = st->head;
  while (curr && idx < st->nq) {
    max_rank = min_rank + curr->num_ranks + curr->delta;
    if (max_rank > rank[idx] + thr[idx] || min_rank > rank[idx]) st->computed[idx++] = prev->value;
    min_rank += curr->num_ranks;
    prev = curr;
    curr = curr->next;
  }
  for (size_t i = idx; i < st->nq; i++)
    if (max_rank >= rank[i] + thr[i] || min_rank > rank[i]) st->computed[i] = prev->value;
}

static double stream_quantile(const stream *st, double q) {
  if (q < 0.0 || q > 1.0) return NAN;
  if (!st->head) return 0.0;
  if (q == 0.0) return st->head->value;
  if (q == 1.0) return st->tail->value;
  for (size_t i = 0; i < st->nq; i++)
    if (st->quantiles[i] >= q) return st->computed[i];
  return NAN;
}

static void stream_free(stream *st) {
  for (sample *c = st->head; c;) {
    sample *n = c->next;
    free(c);
    c = n;
  }
  free(st->buf_less.a);
  free(st->buf_more.a);
}

/* aggregation.Type.Quantile() */
static double type_quantile(int32_t t) {
  switch (t) {
    case 5: case 14: return 0.5;
    case 10: return 0.1;
    case 11: return 0.2;
    case 12: return 0.3;
    case 13: return 0.4;
    case 15: return 0.6;
    case 16: return 0.7;
    case 17: return 0.8;
    case 18: return 0.9;
    case 19: return 0.95;
    case 20: return 0.99;
    case 21: return 0.999;
    case 22: return 0.9999;
    case 23: return 0.25;
    case 24: return 0.75;
    default: return 0.0;
  }
}

/* Types.PooledQuantiles: the quantile types in listed order, Median / P50 once; returns the count */
size_t m3o_timer_quantiles(const int32_t *types, size_t n_types, double *out) {
  size_t n = 0;
  int median = 0;
  for (size_t j = 0; j < n_types; j++) {
    double q = type_quantile(types[j]);
    if (q == 0.0) continue;
    if (types[j] == 5 || types[j] == 14) {
      if (median) continue;
      median = 1;
    }
    out[n++] = q;
  }
  return n;
}

/* One Timer window: the values v[0 .. n) in batches of batch_len[0 .. n_batches) (AddBatch each), then ValueOf of
 * each type into out[0 .. n_types).  *peak (optional): the largest list + pending count seen after a batch. */
void m3o_timer_window(const double *v, const uint32_t *batch_len, size_t n_batches, const int32_t *types,
                      size_t n_types, double eps, int64_t every, double *out, int64_t *peak) {
  double qs[32];
  stream st;
  memset(&st, 0, sizeof(st));
  st.nq = m3o_timer_quantiles(types, n_types, qs);
  st.quantiles = qs;
  st.eps = eps;
  st.every = every;
  int64_t count = 0, pk = 0;
  double sum = 0.0, sum_sq = 0.0;
  size_t off = 0;
  for (size_t b = 0; b < n_batches; b++) {
    size_t n = batch_len[b];
    count += (int64_t)n;
    for (size_t i = 0; i < n; i++) {
      sum += v[off + i];
      sum_sq += v[off + i] * v[off + i];
    }
    stream_add_batch(&st, v + off, n);
    off += n;
    int64_t size = (int64_t)(st.len + st.buf_less.len + st.buf_more.len);
    if (size > pk) pk = size;
  }
  stream_flush(&st);
  for (size_t j = 0; j < n_types; j++) {
    int32_t t = types[j];
    double q = type_quantile(t), r = 0.0;
    if (q > 0.0) {
      r = stream_quantile(&st, q);
    } else if (t == 2) {
      r = stream_quantile(&st, 0.0);
    } else if (t == 3) {
      r = stream_quantile(&st, 1.0);
    } else if (t == 4) {
      r = count == 0 ? 0.0 : sum / (double)count;
    } else if (t == 6) {
      r = (double)count;
    } else if (t == 7) {
      r = sum;
    } else if (t == 8) {
      r = sum_sq;
    } else if (t == 9) { /* aggregation.stdev */
      int64_t div = (int64_t)((uint64_t)count * (uint64_t)(count - 1));
      if (div != 0) {
        double x = ((double)count * sum_sq - sum * sum) / (double)div;
        if (x < 0.0) { /* math.Sqrt of a negative: amd64's invalid-operation NaN */
          uint64_t b = 0xFFF8000000000000ull;
          memcpy(&r, &b, 8);
        } else {
          r = x != x ? x : sqrt(x);
        }
      }
    }
    out[j] = r;
  }
  if (peak) *peak = pk;
  stream_free(&st);
}

/* m3o_timer_window over windows [w0, w1): window w's values v[v_off[w] .. v_off[w + 1]) in batches
 * batch_len[b_off[w] .. b_off[w + 1]); out [w][n_types], peak [w] (optional) */
void m3o_timer_windows(const double *v, const uint64_t *v_off, const uint32_t *batch_len, const uint64_t *b_off,
                       size_t w0, size_t w1, const int32_t *types, size_t n_types, double eps, int64_t every,
                       double *out, int64_t *peak) {
  for (size_t w = w0; w < w1; w++)
    m3o_timer_window(v + v_off[w], batch_len + b_off[w], b_off[w + 1] - b_off[w], types, n_types, eps, every,
                     out + w * n_types, peak ? peak + w : NULL);
}
