// Host-only TEST shim: compiles the product's calib_core.h with g++ (-ffp-contract=off) so the calibration scores of
// inference.evaluate_sequence(samples=S) are checked on CPU against numpy / scipy (tests/test_eval_sample_host.py).
// Not part of the product library.
#include "../geomapnet_b200/csrc/calib_core.h"
extern "C" {
// n estimates est7 [n][7] against targ7 [n][7] under cov [n][36]: e [n][6], d2 [n][3], u [n][3], nll [n]
void hc_score(const double* est7, const double* targ7, const double* cov, long long n, double* e, double* d2,
              double* u, double* nll) {
  for (long long i = 0; i < n; ++i) {
    calibcore::error6(est7 + 7 * i, targ7 + 7 * i, e + 6 * i);
    calibcore::score(est7 + 7 * i, targ7 + 7 * i, cov + 36 * i, d2 + 3 * i, u + 3 * i, nll + i);
  }
}
}
