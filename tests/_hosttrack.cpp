// Host-only TEST shim: compiles the product's track_core.h with g++ (-ffp-contract=off) so the tracker's slot / frame
// clipping, VO pairs, emission ranges and un-normalisation are checked on CPU against data/tuples.py and numpy
// (tests/test_track_host.py).  Not part of the product library.
#include "../geomapnet_b200/csrc/track_core.h"
extern "C" {
long long ht_lag(int T, int skip) { return trackcore::lag(T, skip); }
long long ht_ring_frames(int max_batch, int T, int skip) { return trackcore::ring_frames(max_batch, T, skip); }
long long ht_slot_frame(long long c, int k, int T, int skip, long long last) {
  return trackcore::slot_frame(c, k, T, skip, last);
}
long long ht_first_pending(long long seen, long long lag) { return trackcore::first_pending(seen, lag); }
void ht_vo_pair(int e, int T, int fc, int* i, int* j) { trackcore::vo_pair(e, T, fc, i, j); }
void ht_unnormalize(const double* t, const double* s, const double* m, long long n, double* out) {
  for (long long k = 0; k < n; ++k) out[k] = trackcore::unnormalize(t[k], s[k % 3], m[k % 3]);
}
}
