/*
 * ann_oracle.c -- TEST INFRASTRUCTURE (CPU oracle), never linked into or called by the
 * product library.  Built by __graft_entry__.build() into tests/libm3tsz_ann_oracle.so and
 * bound by tests/ann_oracle_lib.py; self-contained (it shares no code with oracle/).
 *
 * Restates which annotation each aggregation window of m3tsz_aggregate_tiles_annotated is
 * flushed with, from the reference: Gauge.Update / Counter.Update call MaybeReplaceAnnotation
 * (src/aggregator/aggregation/common.go:47-61, gauge.go:54-57, counter.go:77), so a window keeps
 * the last non-empty annotation it was given, and consumeState.annotation
 * (aggregator/generic_elem.go:567, 915-931) flushes each window with its own.  Pinned by the
 * reference's tests in tests/golden/m3tsz_tile_annotation_goldens.json.
 */
#include <stddef.h>
#include <stdint.h>

/* Window w = floor((ts - start) / step) keeps the annotation of the last datapoint, in stream
 * order, that falls in it and carries one.  ann[i] identifies datapoint i's annotation (-1: none,
 * the iterator's Current() reported an empty one); win_out[w] is the id the window keeps, -1 for
 * none.  Datapoints outside [0, n_windows) count for nothing. */
void m3o_window_annotations(const int64_t *ts, const int64_t *ann, size_t n, int64_t start_ns, int64_t step_ns,
                            size_t n_windows, int64_t *win_out) {
  for (size_t w = 0; w < n_windows; w++) win_out[w] = -1;
  for (size_t i = 0; i < n; i++) {
    if (ann[i] < 0 || ts[i] < start_ns) continue;
    const uint64_t w = (uint64_t)(ts[i] - start_ns) / (uint64_t)step_ns;
    if (w < n_windows) win_out[w] = ann[i];
  }
}
