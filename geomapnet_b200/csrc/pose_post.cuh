// qexp of scripts/eval.py:166 for one predicted or target pose, shared by k_pose_post (pgo.cu) and k_eval_windows
// (loader.cu): numpy on the float32 row, n = linalg.norm(log q); hstack((cos n, sinc(n / pi) * log q)).
//
// The float32 operations are spelled out as _rn intrinsics so that the result does not depend on the file's -fmad
// setting (loader.cu is built with -fmad=false): the squared norm is the contraction nvcc makes of x*x + y*y + z*z under
// its default -fmad=true, so both kernels round exactly as k_pose_post always has.
#pragma once

namespace mapnet {

__device__ __forceinline__ void post_qexp(float x, float y, float z, double* q4) {
  const float nn = sqrtf(__fmaf_rn(z, z, __fmaf_rn(x, x, __fmul_rn(y, y))));
  const float sc = (nn == 0.f) ? 1.f : (float)(sin((double)nn) / (double)nn);
  q4[0] = (double)(float)cos((double)nn);
  q4[1] = (double)__fmul_rn(sc, x); q4[2] = (double)__fmul_rn(sc, y); q4[3] = (double)__fmul_rn(sc, z);
}

// Monte-Carlo dropout post step of one frame (k_sample_post, and the sampled tracker's emit in loader.cu), with the
// arithmetic spelled out as _rn intrinsics so that it does not depend on the file's -fmad setting: these are the
// roundings nvcc makes of k_sample_post's plain expressions under its default -fmad=true.
//   sample_qexp: qexp(v) = (cos n, sin n / n * v), n = |v|, (1, 0, 0, 0) at n = 0
//   sample_stats: cov_out = D C D (may be null), t_std = sqrt(trace of its translation block), q_std_deg =
//   2 sqrt(trace of the log q block) * 180 / pi, D = diag(d)
__device__ __forceinline__ void sample_qexp(double vx, double vy, double vz, double* q4) {
  const double nn = sqrt(__fma_rn(vz, vz, __fma_rn(vx, vx, __dmul_rn(vy, vy))));
  const double f = nn > 0.0 ? sin(nn) / nn : 0.0;
  q4[0] = nn > 0.0 ? cos(nn) : 1.0;
  q4[1] = __dmul_rn(f, vx); q4[2] = __dmul_rn(f, vy); q4[3] = __dmul_rn(f, vz);
}
__device__ __forceinline__ void sample_stats(const double* C, const double d[6], double* cov_out, double* t_std,
                                             double* q_std_deg) {
  if (cov_out != nullptr)
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 6; ++c) cov_out[6 * r + c] = __dmul_rn(__dmul_rn(d[r], C[6 * r + c]), d[c]);
  double tt = 0.0, tq = 0.0;
  for (int k = 0; k < 3; ++k) {
    tt = __dadd_rn(tt, __dmul_rn(__dmul_rn(d[k], C[7 * k]), d[k]));
    tq = __dadd_rn(tq, C[7 * (k + 3)]);
  }
  *t_std = sqrt(tt);
  *q_std_deg = __dmul_rn(__dmul_rn(2.0, sqrt(tq)), 180.0 / 3.14159265358979323846);
}

}  // namespace mapnet
