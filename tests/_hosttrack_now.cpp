// Host-only TEST shim: compiles the product's track_core.h with g++ (-ffp-contract=off) so the zero-lag window
// arithmetic of the tracker (mapnet_track_step_now) is checked on CPU against eval_tables(zero_lag=True)
// (tests/test_track_now_host.py).  Not part of the product library.
#include "../geomapnet_b200/csrc/track_core.h"
extern "C" {
long long htn_lag(int T, int skip) { return trackcore::lag(T, skip); }
long long htn_slot_frame(long long c, int k, int T, int skip, long long last) {
  return trackcore::slot_frame(c, k, T, skip, last);
}
long long htn_first_pending(long long seen, long long lag) { return trackcore::first_pending(seen, lag); }
long long htn_now_first(long long seen, long long lag) { return trackcore::now_first(seen, lag); }
long long htn_now_lead(long long seen, long long n, long long lag) { return trackcore::now_lead(seen, n, lag); }
}
