// BatchNorm finalize arithmetic of bn.cu (k_channel_sums, k_bn_bwd_finalize_accum and the prologues of the apply kernels)
// and the descriptor through which the training step hands one BatchNorm to bn.cu.
// Reference semantics: torch.nn.BatchNorm2d training forward / backward as run by
// /root/reference/models/posenet.py:66 (momentum 0.1, eps 1e-5, unbiased running variance).
#pragma once
#include "common.cuh"

namespace mapnet {

// Layout of the BatchNorm sum accumulators: replicas of [3][C] doubles (C <= 512), kBnAccStride doubles apart.  Block b of
// a reducing kernel adds into replica b % nrep: same-address fp64 atomics serialise, the replicas keep that chain short.
// k_channel_sums and the stem's pool backward use up to kBnAccReplicas replicas.
constexpr int kBnAccReplicas = 32;
constexpr int kBnAccStride = 3 * 512;

struct BnFin {
  // forward: batch statistics -> mean / invstd / scale / shift, running statistics
  const float *gamma, *beta;
  float *run_mean, *run_var, *mean, *invstd, *scale, *shift;
  // backward: main BN then downsample BN
  const float *mscale, *mshift;      // optional: ReLU mask recomputed as (mscale*y + mshift > 0) instead of reading z
  const float *gamma2, *mean2, *invstd2;
  float *dgamma, *dbeta, *coef, *dgamma2, *dbeta2, *coef2;
};

// One BatchNorm as seen by one launch of bn.cu.  With accum != nullptr the CONSUMING element-wise kernel
// (k_bn_apply / k_bn_bwd_apply / k_stem_pool) finalizes the sums itself (lazy finalize): every block sums the replicas of
// its own 64-channel slice and derives scale / shift (forward) or the dy = A*g + B*y + C coefficients (backward) in its
// prologue; the blocks with blockIdx.x == 0 also write the per-channel results other kernels read later (mean, invstd,
// scale, shift, running statistics; d gamma, d beta).  This removes the 68 tiny finalize launches of a training step from
// the critical path (measured: 0.27 ms of a 3.9 ms step).  The accumulators are per-BatchNorm slots zeroed once per step
// (nobody resets them between producer and consumers).  With accum == nullptr the kernels read scale / shift (forward)
// or coef (backward) from memory, where an earlier finalize left them.
struct BnDesc {
  const double* accum;       // [nrep][kBnAccStride] replicas, or nullptr
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

// backward of one BatchNorm channel from s0 = sum g, s1 = sum g*y:  s2 = sum g * xhat (= d gamma) and the
// dy = A*g + B*y + C coefficients
struct BnBwdCoef { double s2, A, B, C; };
__device__ __forceinline__ BnBwdCoef bn_bwd_coef(const float mean, const float invstd, const float gamma, const double s0,
                                                 const double s1, const double invM) {
  const double mu = (double)mean, is = (double)invstd;
  BnBwdCoef k;
  k.s2 = is * (s1 - mu * s0);
  k.A = (double)gamma * is;
  k.B = -k.A * is * k.s2 * invM;
  k.C = -k.A * s0 * invM - k.B * mu;
  return k;
}

// s0 = sum g, s1 = sum g*y [, s1d = sum g*yd]:  d gamma, d beta and dy = A*g + B*y + C coefficients.
// A null dgamma / dbeta (a frozen parameter) is not written; the coefficients always are.
__device__ __forceinline__ void bn_fin_backward(const int c, const int C, const double s0, const double s1,
                                                const double s1d, const long long M, const BnFin& f, const bool ds) {
  const double invM = 1.0 / (double)M;
  {
    const BnBwdCoef k = bn_bwd_coef(f.mean[c], f.invstd[c], f.gamma[c], s0, s1, invM);
    if (f.dgamma != nullptr) f.dgamma[c] = (float)k.s2;
    if (f.dbeta != nullptr) f.dbeta[c] = (float)s0;
    f.coef[c] = (float)k.A; f.coef[C + c] = (float)k.B; f.coef[2 * C + c] = (float)k.C;
  }
  if (ds) {
    const BnBwdCoef k = bn_bwd_coef(f.mean2[c], f.invstd2[c], f.gamma2[c], s0, s1d, invM);
    if (f.dgamma2 != nullptr) f.dgamma2[c] = (float)k.s2;
    if (f.dbeta2 != nullptr) f.dbeta2[c] = (float)s0;
    f.coef2[c] = (float)k.A; f.coef2[C + c] = (float)k.B; f.coef2[2 * C + c] = (float)k.C;
  }
}
#endif

}  // namespace mapnet
