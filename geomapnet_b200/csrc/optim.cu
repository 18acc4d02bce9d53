// Flat-buffer fused SGD and RMSprop (+ classic L2 weight decay, + global-norm gradient clip, + 1/world gradient
// scale) in one pass over a contiguous run of parameters, built like k_adam (adam.cu).  They replace
// torch.optim.SGD / RMSprop.step and clip_grad_norm (the reference's common/optimizer.py:16-27 and
// common/train.py:357-359) in the CUDA-graph and data-parallel training steps.
//
// Two things make them capturable where k_adam bakes its rate into the launch: the learning rate is read from
// device memory (the reference's SGD recipe changes it every few epochs, common/train.py:265), and SGD's first
// step -- which initialises the momentum buffer instead of decaying it -- is told apart by a device step counter.
// HBM-bound: SGD moves 12 B per parameter (20 B with momentum), RMSprop 20 B (28 B with momentum or centered, 36 B
// with both), 128-bit vectorised.
#include "kernels.h"

namespace mapnet {

// torch.optim.SGD (maximize=False) single-tensor math, d = coef*g:
//   d += wd*p; buf = first ? d : momentum*buf + (1-dampening)*d; d = nesterov ? d + momentum*buf : buf; p -= lr*d
struct SgdArgs {
  float lr, momentum, omd /* 1 - dampening */, wd, coef;
  int has_buf, first, nesterov;
};

__device__ __forceinline__ void sgd_elem(float& p, float g, float& buf, const SgdArgs& a) {
  float d = g * a.coef;
  if (a.wd != 0.f) d = d + a.wd * p;
  if (a.has_buf) {
    buf = a.first ? d : __fmul_rn(a.momentum, buf) + a.omd * d;   // mul_ then add_, as torch rounds
    d = a.nesterov ? d + a.momentum * buf : buf;
  }
  p = p - a.lr * d;
}

__global__ void __launch_bounds__(256)
k_sgd(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf, long long n,
      const float* __restrict__ lr_dev, float momentum, float omd, float wd, int nesterov, float gscale,
      const float* __restrict__ sqnorm, float max_norm, const int* __restrict__ step_dev, int vec) {
  pdl_prologue();
  SgdArgs a;
  a.lr = *lr_dev;
  a.momentum = momentum; a.omd = omd; a.wd = wd; a.nesterov = nesterov;
  a.coef = grad_coef(gscale, sqnorm, max_norm);
  a.has_buf = buf != nullptr;
  a.first = a.has_buf && *step_dev == 1;
  if (!vec) {      // some buffer is not 16-byte aligned (free-standing parameters): scalar grid-stride loop
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
      float b = (a.has_buf && !a.first) ? buf[i] : 0.f;
      sgd_elem(p[i], g[i], b, a);
      if (a.has_buf) buf[i] = b;
    }
    return;
  }
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.has_buf && !a.first) bb = reinterpret_cast<float4*>(buf)[i];    // step 1 does not read the buffer
    float* P = &pp.x; const float* G = &gg.x; float* Bf = &bb.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) sgd_elem(P[k], G[k], Bf[k], a);
    reinterpret_cast<float4*>(p)[i] = pp;
    if (a.has_buf) reinterpret_cast<float4*>(buf)[i] = bb;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (long long i = n4 << 2; i < n; ++i) {
      float b = (a.has_buf && !a.first) ? buf[i] : 0.f;
      sgd_elem(p[i], g[i], b, a);
      if (a.has_buf) buf[i] = b;
    }
  }
}

// torch.optim.RMSprop (maximize=False) single-tensor math, d = coef*g:
//   d += wd*p; sa = alpha*sa + (1-alpha)*d*d
//   centered: ga = lerp(ga, d, 1-alpha), avg = sqrt(sa - ga*ga) + eps;  else avg = sqrt(sa) + eps
//   momentum: buf = momentum*buf + d/avg, p -= lr*buf;  else p -= lr*d/avg
struct RmsArgs {
  float lr, alpha, oma /* 1 - alpha */, eps, wd, momentum, coef;
  int centered, has_buf;
};

__device__ __forceinline__ void rmsprop_elem(float& p, float g, float& sa, float& ga, float& buf, const RmsArgs& a) {
  float d = g * a.coef;
  if (a.wd != 0.f) d = d + a.wd * p;
  sa = __fmul_rn(a.alpha, sa) + a.oma * d * d;
  float avg;
  if (a.centered) {
    // at::lerp's two-sided formula (weight = 1 - alpha)
    ga = a.oma < 0.5f ? ga + a.oma * (d - ga) : d - (d - ga) * (1.f - a.oma);
    avg = sqrtf(sa - ga * ga) + a.eps;
  } else {
    avg = sqrtf(sa) + a.eps;
  }
  if (a.has_buf) {
    buf = __fmul_rn(a.momentum, buf) + d / avg;
    p = p - a.lr * buf;
  } else {
    p = p - a.lr * (d / avg);
  }
}

__global__ void __launch_bounds__(256)
k_rmsprop(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ sq, float* __restrict__ ga,
          float* __restrict__ buf, long long n, const float* __restrict__ lr_dev, float alpha, float oma, float eps,
          float wd, float momentum, float gscale, const float* __restrict__ sqnorm, float max_norm, int vec) {
  pdl_prologue();
  RmsArgs a;
  a.lr = *lr_dev;
  a.alpha = alpha; a.oma = oma; a.eps = eps; a.wd = wd; a.momentum = momentum;
  a.coef = grad_coef(gscale, sqnorm, max_norm);
  a.centered = ga != nullptr;
  a.has_buf = buf != nullptr;
  if (!vec) {      // some buffer is not 16-byte aligned (free-standing parameters): scalar grid-stride loop
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
      float gai = a.centered ? ga[i] : 0.f, bi = a.has_buf ? buf[i] : 0.f;
      rmsprop_elem(p[i], g[i], sq[i], gai, bi, a);
      if (a.centered) ga[i] = gai;
      if (a.has_buf) buf[i] = bi;
    }
    return;
  }
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    float4 ss = reinterpret_cast<float4*>(sq)[i];
    float4 aa = make_float4(0.f, 0.f, 0.f, 0.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.centered) aa = reinterpret_cast<float4*>(ga)[i];
    if (a.has_buf) bb = reinterpret_cast<float4*>(buf)[i];
    float* P = &pp.x; const float* G = &gg.x; float* S = &ss.x; float* A = &aa.x; float* Bf = &bb.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) rmsprop_elem(P[k], G[k], S[k], A[k], Bf[k], a);
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(sq)[i] = ss;
    if (a.centered) reinterpret_cast<float4*>(ga)[i] = aa;
    if (a.has_buf) reinterpret_cast<float4*>(buf)[i] = bb;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (long long i = n4 << 2; i < n; ++i) {
      float gai = a.centered ? ga[i] : 0.f, bi = a.has_buf ? buf[i] : 0.f;
      rmsprop_elem(p[i], g[i], sq[i], gai, bi, a);
      if (a.centered) ga[i] = gai;
      if (a.has_buf) buf[i] = bi;
    }
  }
}

static int optim_grid(long long n) {
  long long grid = ((n >> 2) + 255) / 256;
  if (grid > kNumSMs * 8LL) grid = kNumSMs * 8LL;
  if (grid < 1) grid = 1;
  return (int)grid;
}

static int aligned16(const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

int launch_sgd(float* p, const float* g, float* buf, long long n, const float* lr_dev, float momentum,
               double dampening, float wd, int nesterov, int* step_dev, float gscale, const float* sqnorm_or_null,
               float max_norm, cudaStream_t st) {
  if (step_dev != nullptr) MN_TRY(launch_inc_i32(step_dev, st));
  const int vec = aligned16(p) && aligned16(g) && aligned16(buf);
  const float omd = (float)(1.0 - dampening);      // 1 - dampening rounded once, as torch does
  MN_LAUNCH(k_sgd, optim_grid(n), 256, 0, st, p, g, buf, n, lr_dev, momentum, omd, wd, nesterov ? 1 : 0, gscale,
            sqnorm_or_null, max_norm, (const int*)step_dev, vec);
  MN_LAUNCH_CHECK();
  return 0;
}

int launch_rmsprop(float* p, const float* g, float* square_avg, float* grad_avg, float* buf, long long n,
                   const float* lr_dev, double alpha, float eps, float wd, float momentum, int* step_dev, float gscale,
                   const float* sqnorm_or_null, float max_norm, cudaStream_t st) {
  if (step_dev != nullptr) MN_TRY(launch_inc_i32(step_dev, st));
  const int vec = aligned16(p) && aligned16(g) && aligned16(square_avg) && aligned16(grad_avg) && aligned16(buf);
  const float oma = (float)(1.0 - alpha);
  MN_LAUNCH(k_rmsprop, optim_grid(n), 256, 0, st, p, g, square_avg, grad_avg, buf, n, lr_dev, (float)alpha, oma, eps, wd,
            momentum, gscale, sqnorm_or_null, max_norm, vec);
  MN_LAUNCH_CHECK();
  return 0;
}

}  // namespace mapnet
