// Flat-buffer fused Adam (+ classic L2 weight decay, + global-norm gradient clip,
// + 1/world gradient scale) over the whole parameter vector in one pass.
// Replaces ~10 pointwise launches x 114 tensors of torch.optim.Adam.step and
// clip_grad_norm (/root/reference/common/optimizer.py:21-23,
// /root/reference/common/train.py:357-359; SURVEY.md section 8f-1).  HBM-bound:
// 4 reads + 3 writes of fp32 per parameter, 128-bit vectorised.
#include "kernels.h"

namespace mapnet {

__global__ void __launch_bounds__(256)
k_sqnorm_partial(const float* __restrict__ g, long long n, float* __restrict__ partials, int vec) {
  pdl_prologue();
  double acc = 0.0;
  if (!vec) {      // gradient buffer not 16-byte aligned: scalar grid-stride loop
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
      acc += (double)g[i] * g[i];
  }
  const long long n4 = vec ? (n >> 2) : 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    acc += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
  }
  if (vec && blockIdx.x == 0 && threadIdx.x == 0)
    for (long long i = n4 << 2; i < n; ++i) acc += (double)g[i] * g[i];
  __shared__ double red[8];
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += red[w];
    partials[blockIdx.x] = (float)s;
  }
}
__global__ void k_sqnorm_final(const float* __restrict__ partials, int nblk, float* __restrict__ out,
                               int accumulate) {
  pdl_prologue();
  double s = 0.0;
  for (int i = threadIdx.x; i < nblk; i += 32) s += (double)partials[i];
  s = warp_sum_d(s);
  if (threadIdx.x == 0) out[0] = (accumulate ? out[0] : 0.f) + (float)s;
}

int launch_sqnorm(const float* g, long long n, float* partials, float* out_sq, cudaStream_t st) {
  const int nblk = 296;
  const int vec = (reinterpret_cast<uintptr_t>(g) & 15) == 0;
  MN_LAUNCH(k_sqnorm_partial, nblk, 256, 0, st, g, n, partials, vec);
  MN_LAUNCH_CHECK();
  MN_LAUNCH(k_sqnorm_final, 1, 32, 0, st, partials, nblk, out_sq, 0);
  MN_LAUNCH_CHECK();
  return 0;
}

// torch.optim.Adam (amsgrad=False, maximize=False) single-tensor math:
//   g += wd*p; m = b1*m + (1-b1)*g; v = b2*v + (1-b2)*g*g
//   p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps)
__global__ void k_inc_i32(int* c) {
  pdl_prologue(); *c += 1; }

int launch_inc_i32(int* c, cudaStream_t st) {
  MN_LAUNCH(k_inc_i32, 1, 1, 0, st, c);
  MN_LAUNCH_CHECK();
  return 0;
}

__global__ void __launch_bounds__(256)
k_adam(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
       long long n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2_sqrt,
       float gscale, const float* __restrict__ sqnorm, float max_norm, const int* __restrict__ step_dev, int vec) {
  pdl_prologue();
  if (step_dev != nullptr) {
    // CUDA-graph friendly: the step count lives on the device (bias corrections cannot be
    // baked into a captured launch)
    const double t = (double)(*step_dev);
    bc1 = (float)(1.0 - pow((double)b1, t));
    bc2_sqrt = sqrtf((float)(1.0 - pow((double)b2, t)));
  }
  const float coef = grad_coef(gscale, sqnorm, max_norm);
  const float step = lr / bc1;
  if (!vec) {      // some buffer is not 16-byte aligned (free-standing parameters): scalar grid-stride loop
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
      float gr = g[i] * coef + wd * p[i];
      m[i] = m[i] + (1.f - b1) * (gr - m[i]);
      v[i] = b2 * v[i] + (1.f - b2) * gr * gr;
      p[i] = p[i] - step * (m[i] / (sqrtf(v[i]) / bc2_sqrt + eps));
    }
    return;
  }
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    float* P = &pp.x; const float* G = &gg.x; float* Mm = &mm.x; float* V = &vv.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float gr = G[k] * coef + wd * P[k];
      Mm[k] = Mm[k] + (1.f - b1) * (gr - Mm[k]);          // lerp, as torch does
      V[k] = b2 * V[k] + (1.f - b2) * gr * gr;
      const float denom = sqrtf(V[k]) / bc2_sqrt + eps;
      P[k] = P[k] - step * (Mm[k] / denom);
    }
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (long long i = n4 << 2; i < n; ++i) {
      float gr = g[i] * coef + wd * p[i];
      m[i] = m[i] + (1.f - b1) * (gr - m[i]);
      v[i] = b2 * v[i] + (1.f - b2) * gr * gr;
      p[i] = p[i] - step * (m[i] / (sqrtf(v[i]) / bc2_sqrt + eps));
    }
  }
}

int launch_adam(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                float eps, float wd, float bc1, float bc2, float gscale, const float* sqnorm_or_null,
                float max_norm, int* step_dev, cudaStream_t st) {
  long long grid = ((n >> 2) + 255) / 256;
  if (grid > kNumSMs * 8LL) grid = kNumSMs * 8LL;
  if (grid < 1) grid = 1;
  if (step_dev != nullptr) MN_TRY(launch_inc_i32(step_dev, st));
  const int vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                    reinterpret_cast<uintptr_t>(v)) & 15) == 0;
  MN_LAUNCH(k_adam, (int)grid, 256, 0, st, p, g, m, v, n, lr, beta1, beta2, eps, wd, bc1, sqrtf(bc2), gscale, sqnorm_or_null, max_norm, step_dev, vec);
  MN_LAUNCH_CHECK();
  return 0;
}

}  // namespace mapnet
