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

}  // namespace mapnet
