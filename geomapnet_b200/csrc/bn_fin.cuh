// BatchNorm finalize arithmetic of bn.cu: the separate finalize kernel, k_channel_sums and the lazy finalize of the
// consuming element-wise kernels.
// Reference semantics: torch.nn.BatchNorm2d training forward / backward as run by
// /root/reference/models/posenet.py:66 (momentum 0.1, eps 1e-5, unbiased running variance).
#pragma once
#include "common.cuh"

namespace mapnet {

struct BnFin {
  // forward: batch statistics -> mean / invstd / scale / shift, running statistics
  const float *gamma, *beta;
  float *run_mean, *run_var, *mean, *invstd, *scale, *shift;
  int training;
  // backward: main BN then downsample BN
  const float *mscale, *mshift;      // optional: ReLU mask recomputed as (mscale*y + mshift > 0) instead of reading z
  const float *gamma2, *mean2, *invstd2;
  float *dgamma, *dbeta, *coef, *dgamma2, *dbeta2, *coef2;
};

// Finalize performed by the CONSUMING element-wise kernel (bn.cu, k_bn_apply_lazy / k_bn_bwd_apply_lazy / k_stem_pool):
// every block sums the replicas of its own 64-channel slice and derives scale / shift (forward) or the dy = A*g + B*y + C
// coefficients (backward) in its prologue; the blocks with blockIdx.x == 0 also write the per-channel results other
// kernels read later (mean, invstd, scale, shift, running statistics; d gamma, d beta).  This removes the 68 tiny
// finalize launches of a training step from the critical path (measured: 0.27 ms of a 3.9 ms step).  The accumulators
// are per-BatchNorm slots zeroed once per step (nobody resets them between producer and consumers).
struct BnLazy {
  const double* accum;       // [nrep][3 * 512] replicas; nullptr: not lazy (parameters are read from memory)
  int nrep;
  long long M;               // pixels per channel
  double invM, unbias;       // 1 / M and M / (M - 1) from the host: no fp64 division on the consumers' critical path
  BnFin f;
};

#if defined(__CUDACC__)
// s0 = sum y, s1 = sum y^2 over M pixels of channel c
__device__ __forceinline__ void bn_fin_forward(const int c, const double s0, const double s1, const long long M,
                                               const BnFin& f) {
  const double invM = 1.0 / (double)M;
  const double m = s0 * invM;
  double var = s1 * invM - m * m;
  if (var < 0.0) var = 0.0;
  const float mean = (float)m;
  const float invstd = (float)(1.0 / sqrt(var + 1e-5));
  const double unbiased = (M > 1) ? var * (double)M / (double)(M - 1) : var;
  f.run_mean[c] = 0.9f * f.run_mean[c] + 0.1f * mean;
  f.run_var[c] = 0.9f * f.run_var[c] + 0.1f * (float)unbiased;
  f.mean[c] = mean;
  f.invstd[c] = invstd;
  const float sc = f.gamma[c] * invstd;
  f.scale[c] = sc;
  f.shift[c] = f.beta[c] - mean * sc;
}

// s0 = sum g, s1 = sum g*y [, s1d = sum g*yd]:  d gamma, d beta and dy = A*g + B*y + C coefficients
__device__ __forceinline__ void bn_fin_backward(const int c, const int C, const double s0, const double s1,
                                                const double s1d, const long long M, const BnFin& f, const bool ds) {
  const double invM = 1.0 / (double)M;
  {
    const double mu = (double)f.mean[c], is = (double)f.invstd[c];
    const double s2 = is * (s1 - mu * s0);          // sum g * xhat
    f.dgamma[c] = (float)s2;
    f.dbeta[c] = (float)s0;
    const double A = (double)f.gamma[c] * is;
    const double Bc = -A * is * s2 * invM;
    const double Cc = -A * s0 * invM - Bc * mu;
    f.coef[c] = (float)A; f.coef[C + c] = (float)Bc; f.coef[2 * C + c] = (float)Cc;
  }
  if (ds) {
    const double mu = (double)f.mean2[c], is = (double)f.invstd2[c];
    const double s2 = is * (s1d - mu * s0);
    f.dgamma2[c] = (float)s2;
    f.dbeta2[c] = (float)s0;
    const double A = (double)f.gamma2[c] * is;
    const double Bc = -A * is * s2 * invM;
    const double Cc = -A * s0 * invM - Bc * mu;
    f.coef2[c] = (float)A; f.coef2[C + c] = (float)Bc; f.coef2[2 * C + c] = (float)Cc;
  }
}
#endif

}  // namespace mapnet
