// Calibration score of one Monte-Carlo pose estimate against its target (inference.evaluate_sequence(samples=S)),
// shared by the emit kernel (loader.cu, k_eval_sample_emit) and the host-only test shim (tests/_hostcalib.cpp).
//
// The estimate is (t^, q^) with covariance Sigma [6][6] in (t, log q), the target (t, q); translations in the same
// units as Sigma's translation block.  The error is
//   e = (t^ - t, qlog(q^) - qlog(sigma q)),  sigma = sign(q^ . q) (+1 when the dot product is 0),
// with qlog common/pose_utils.py's (zero for a zero vector part, else arccos(w) v / |v|, w clamped to [-1, 1]).  sigma
// puts the target in the posterior's chart: q and -q are one rotation, and k_pgo_cov maps its posterior to qlog
// coordinates at q^.  The scores are the squared Mahalanobis distances d2 = e' Sigma^-1 e of the 6-DoF error, of the
// translation block and of the log q block (each by its own Cholesky factor), their chi-square CDFs u (6, 3 and 3
// degrees of freedom, in closed form) and the 6-DoF Gaussian negative log-likelihood nll = (d2 + 6 ln 2 pi +
// ln det Sigma) / 2.  A Sigma (or block) that is not positive definite gives NaN in every score that needs it: a
// Cholesky pivot counts as positive above kPivotFloor times its diagonal entry, so that a covariance of rank < n (the
// sample covariance of S <= n draws, whose last pivots are rounding noise of either sign) is reported as not positive
// definite rather than scored against a pivot made of rounding error.
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define CAL_HD __host__ __device__ __forceinline__
#else
#define CAL_HD static inline
#endif

namespace calibcore {

constexpr double kPivotFloor = 1e-12;

// common/pose_utils.py qlog: (arccos(w) * v) / |v|, zero when v is zero
CAL_HD void qlog(const double q[4], double v[3]) {
  if (q[1] == 0.0 && q[2] == 0.0 && q[3] == 0.0) {
    v[0] = v[1] = v[2] = 0.0;
    return;
  }
  const double w = q[0] < -1.0 ? -1.0 : (q[0] > 1.0 ? 1.0 : q[0]);
  const double a = acos(w), n = sqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int k = 0; k < 3; ++k) v[k] = a * q[1 + k] / n;
}

// e [6] of estimate est7 = (t^, q^) against target targ7 = (t, q)
CAL_HD void error6(const double est7[7], const double targ7[7], double e[6]) {
  const double dot = est7[3] * targ7[3] + est7[4] * targ7[4] + est7[5] * targ7[5] + est7[6] * targ7[6];
  const double sg = dot < 0.0 ? -1.0 : 1.0;
  const double qt[4] = {sg * targ7[3], sg * targ7[4], sg * targ7[5], sg * targ7[6]};
  double ve[3], vt[3];
  qlog(est7 + 3, ve);
  qlog(qt, vt);
  for (int k = 0; k < 3; ++k) {
    e[k] = est7[k] - targ7[k];
    e[3 + k] = ve[k] - vt[k];
  }
}

// (d2, ln det) of the n x n block of C [6][6] at (o, o) against x [n]; false (both NaN) when it is not positive definite
// (a pivot not above kPivotFloor times its diagonal entry)
CAL_HD bool mahalanobis(const double C[36], int o, int n, const double* x, double* d2, double* logdet) {
  double L[6][6], y[6];
  double s = 0.0, ld = 0.0;
  for (int j = 0; j < n; ++j) {
    for (int i = j; i < n; ++i) {
      double v = C[6 * (o + i) + o + j];
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      if (i == j) {
        if (!(v > kPivotFloor * C[6 * (o + j) + o + j])) {
          *d2 = *logdet = NAN;
          return false;
        }
        L[j][j] = sqrt(v);
      } else {
        L[i][j] = v / L[j][j];
      }
    }
  }
  for (int i = 0; i < n; ++i) {          // L y = x
    double v = x[i];
    for (int k = 0; k < i; ++k) v -= L[i][k] * y[k];
    y[i] = v / L[i][i];
    s += y[i] * y[i];
    ld += log(L[i][i]);
  }
  *d2 = s;
  *logdet = 2.0 * ld;
  return true;
}

// chi-square CDFs with 6 and 3 degrees of freedom (NaN stays NaN)
CAL_HD double chi2_cdf6(double x) { return 1.0 - exp(-0.5 * x) * (1.0 + 0.5 * x + 0.125 * x * x); }
CAL_HD double chi2_cdf3(double x) {
  return erf(sqrt(0.5 * x)) - sqrt(2.0 * x / 3.14159265358979323846) * exp(-0.5 * x);
}

// d2 [3] (6-DoF, translation, log q), u [3] (their chi-square CDFs) and nll of one estimate
CAL_HD void score(const double est7[7], const double targ7[7], const double C[36], double d2[3], double u[3],
                  double* nll) {
  double e[6], ld, ldb;
  error6(est7, targ7, e);
  mahalanobis(C, 0, 6, e, &d2[0], &ld);
  mahalanobis(C, 0, 3, e, &d2[1], &ldb);
  mahalanobis(C, 3, 3, e + 3, &d2[2], &ldb);
  u[0] = chi2_cdf6(d2[0]);
  u[1] = chi2_cdf3(d2[1]);
  u[2] = chi2_cdf3(d2[2]);
  *nll = 0.5 * (d2[0] + 6.0 * log(2.0 * 3.14159265358979323846) + ld);
}

}  // namespace calibcore
