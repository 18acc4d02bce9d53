// fp32 CUDA-core implicit-GEMM convolution: fprop, dgrad, wgrad.
//
// This is the STRICT-PARITY path (precision="fp32"): every product and sum is
// fp32 like the reference's cuDNN fp32 convs, so loss/pose match the reference
// PyTorch path to <=1e-4 (BASELINE.json north_star).  It is also the on-GPU
// cross-check for the wgmma kernels in conv_tc.cu.  It is not a CPU fallback
// and not the benchmarked path: the bf16 tensor-core path is.
//
// Replaces cuDNN conv fwd / bwd-data / bwd-filter behind torchvision resnet34
// (SURVEY.md section 2c), reached from /root/reference/models/posenet.py:66.
//
// GEMM views (NHWC activations, weights [N][K] K-major):
//   fprop: C[m=(b,oh,ow)][n=co] = sum_k A[m][k=(kh,kw,ci)] * Wk[n][k]
//   dgrad: C[m=(b,ih,iw)][n=ci] = sum_k dY[..][k=(kh,kw,co)] * Wd[n][k]
//   wgrad: C[m=co][n=(kh,kw,ci)] = sum_{k=pixel} dY[k][m] * X[k@tap][n]   (split-K, fixed-order reduction)
#include "kernels.h"

namespace mapnet {

static const int BM = 64, BN = 64, BK = 16, NT = 256;

template <typename T> struct Ld4 {};
template <> struct Ld4<float> {
  static __device__ __forceinline__ void ld(const float* p, float* o) {
    float4 v = *reinterpret_cast<const float4*>(p);
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
  }
};
template <> struct Ld4<bf16> {
  static __device__ __forceinline__ void ld(const bf16* p, float* o) {
    uint2 r = *reinterpret_cast<const uint2*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
    float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]);
    o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
  }
};

// MODE 0 fprop, 1 dgrad
template <typename T, int MODE>
__global__ void __launch_bounds__(NT)
k_conv_simt(ConvGeom g, const T* __restrict__ src, const float* __restrict__ wmat,
            const T* __restrict__ residual, T* __restrict__ dst) {
  pdl_prologue();
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;
  // GEMM sizes
  const long long M = (MODE == 0) ? g.M_out() : g.M_in();
  const int N = (MODE == 0) ? g.Co : g.Ci;
  const int Cs = (MODE == 0) ? g.Ci : g.Co;        // channels of the gathered tensor
  const int K = g.KH * g.KW * Cs;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // loader coordinates: row lr, 4 consecutive k at lk
  const int lr = t >> 2, lk = (t & 3) * 4;
  const long long am = m0 + lr;
  int pb = 0, ph = 0, pw = 0;
  const bool arow_ok = am < M;
  if (arow_ok) {
    const int Wd = (MODE == 0) ? g.Wo : g.Wi, Hd = (MODE == 0) ? g.Ho : g.Hi;
    long long p = am;
    pw = (int)(p % Wd); p /= Wd;
    ph = (int)(p % Hd);
    pb = (int)(p / Hd);
  }
  const int bn_row = n0 + lr;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += BK) {
    const int k = k0 + lk;
    float av[4] = {0.f, 0.f, 0.f, 0.f};
    if (arow_ok && k < K) {
      const int tap = k / Cs, c = k - tap * Cs;
      const int kh = tap / g.KW, kw = tap - kh * g.KW;
      if (MODE == 0) {
        const int ih = ph * g.stride - g.pad + kh, iw = pw * g.stride - g.pad + kw;
        if (ih >= 0 && ih < g.Hi && iw >= 0 && iw < g.Wi)
          Ld4<T>::ld(src + (((long long)pb * g.Hi + ih) * g.Wi + iw) * g.Ci + c, av);
      } else {
        const int th = ph + g.pad - kh, tw = pw + g.pad - kw;
        if (th >= 0 && tw >= 0 && (th % g.stride) == 0 && (tw % g.stride) == 0) {
          const int oh = th / g.stride, ow = tw / g.stride;
          if (oh < g.Ho && ow < g.Wo)
            Ld4<T>::ld(src + (((long long)pb * g.Ho + oh) * g.Wo + ow) * g.Co + c, av);
        }
      }
    }
    float bv[4] = {0.f, 0.f, 0.f, 0.f};
    if (bn_row < N && k < K) Ld4<float>::ld(wmat + (long long)bn_row * K + k, bv);
#pragma unroll
    for (int i = 0; i < 4; ++i) { As[lk + i][lr] = av[i]; Bs[lk + i][lr] = bv[i]; }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j];
      if (residual != nullptr) v += to_f(residual[m * N + n]);
      dst[m * N + n] = from_f<T>(v);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(NT)
k_conv_simt_wgrad(ConvGeom g, const T* __restrict__ x, const T* __restrict__ dy, float* __restrict__ dw,
                  float* __restrict__ part, long long kchunk) {
  pdl_prologue();
  __shared__ float As[BK][BM + 4];   // [pixel][co]
  __shared__ float Bs[BK][BN + 4];   // [pixel][(tap,ci)]
  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;
  const int M = g.Co, N = g.KH * g.KW * g.Ci;
  const long long Kt = g.M_out();
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const long long kbeg = (long long)blockIdx.z * kchunk;
  long long kend = kbeg + kchunk; if (kend > Kt) kend = Kt;
  const int lp = t >> 4, l4 = (t & 15) * 4;      // pixel-in-tile, 4 consecutive m / n
  // this thread's B columns: n = n0 + l4 .. +3 share one tap
  const int nn = n0 + l4;
  const bool n_ok = nn < N;
  const int tap = n_ok ? nn / g.Ci : 0, ci = n_ok ? nn - tap * g.Ci : 0;
  const int kh = tap / g.KW, kw = tap - kh * g.KW;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (long long k0 = kbeg; k0 < kend; k0 += BK) {
    const long long pix = k0 + lp;
    float av[4] = {0.f, 0.f, 0.f, 0.f}, bv[4] = {0.f, 0.f, 0.f, 0.f};
    if (pix < kend) {
      if (m0 + l4 < M) Ld4<T>::ld(dy + pix * g.Co + m0 + l4, av);
      if (n_ok) {
        long long p = pix;
        const int ow = (int)(p % g.Wo); p /= g.Wo;
        const int oh = (int)(p % g.Ho);
        const int b = (int)(p / g.Ho);
        const int ih = oh * g.stride - g.pad + kh, iw = ow * g.stride - g.pad + kw;
        if (ih >= 0 && ih < g.Hi && iw >= 0 && iw < g.Wi)
          Ld4<T>::ld(x + (((long long)b * g.Hi + ih) * g.Wi + iw) * g.Ci + ci, bv);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) { As[lp][l4 + i] = av[i]; Bs[lp][l4 + i] = bv[i]; }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  // one writer per element: split z STORES into its workspace slice (launch_split_reduce adds the slices up in a
  // fixed order), a single split adds into dw directly
  const bool split = part != nullptr;
  float* out = split ? part + (long long)blockIdx.z * M * N : dw;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      out[(long long)m * N + n] = split ? acc[i][j] : out[(long long)m * N + n] + acc[i][j];
    }
  }
}

template <typename T>
int launch_conv_simt_fprop(const ConvGeom& g, const T* x, const float* w, const T* residual, T* y, cudaStream_t st) {
  MN_CHECK(g.Ci % 4 == 0, "conv_simt: Ci %% 4 != 0");
  dim3 grid(cdiv(g.M_out(), BM), cdiv(g.Co, BN));
  MN_LAUNCH((k_conv_simt<T, 0>), grid, NT, 0, st, g, x, w, residual, y);
  MN_LAUNCH_CHECK();
  return 0;
}
template <typename T>
int launch_conv_simt_dgrad(const ConvGeom& g, const T* dy, const float* w_dg, const T* residual, T* dx, cudaStream_t st) {
  MN_CHECK(g.Co % 4 == 0, "conv_simt: Co %% 4 != 0");
  dim3 grid(cdiv(g.M_in(), BM), cdiv(g.Ci, BN));
  MN_LAUNCH((k_conv_simt<T, 1>), grid, NT, 0, st, g, dy, w_dg, residual, dx);
  MN_LAUNCH_CHECK();
  return 0;
}
template <typename T>
int launch_conv_simt_wgrad(const ConvGeom& g, const T* x, const T* dy, float* dw, cudaStream_t st) {
  MN_CHECK(g.Ci % 4 == 0 && g.Co % 4 == 0, "conv_simt wgrad: channels %% 4 != 0");
  const int gm = cdiv(g.Co, BM), gn = cdiv(g.KH * g.KW * g.Ci, BN);
  const long long Kt = g.M_out();
  long long splits = ((long long)kNumSMs * 4) / ((long long)gm * gn);
  if (splits < 1) splits = 1;
  long long kchunk = (Kt + splits - 1) / splits;
  kchunk = ((kchunk + BK - 1) / BK) * BK;
  if (kchunk < 256) kchunk = 256;
  splits = (Kt + kchunk - 1) / kchunk;
  dim3 grid(gm, gn, (unsigned)splits);
  const long long n = (long long)g.Co * g.KH * g.KW * g.Ci;
  float* part = nullptr;
  if (splits > 1) MN_CUDA(cudaMallocAsync((void**)&part, (size_t)splits * n * sizeof(float), st));   // stream-ordered
  MN_LAUNCH(k_conv_simt_wgrad<T>, grid, NT, 0, st, g, x, dy, dw, part, kchunk);
  MN_LAUNCH_CHECK();
  if (part != nullptr) {
    MN_TRY(launch_split_reduce(part, (int)splits, n, dw, st));
    MN_CUDA(cudaFreeAsync(part, st));
  }
  return 0;
}

template int launch_conv_simt_fprop<float>(const ConvGeom&, const float*, const float*, const float*, float*, cudaStream_t);
template int launch_conv_simt_fprop<bf16>(const ConvGeom&, const bf16*, const float*, const bf16*, bf16*, cudaStream_t);
template int launch_conv_simt_dgrad<float>(const ConvGeom&, const float*, const float*, const float*, float*, cudaStream_t);
template int launch_conv_simt_dgrad<bf16>(const ConvGeom&, const bf16*, const float*, const bf16*, bf16*, cudaStream_t);
template int launch_conv_simt_wgrad<float>(const ConvGeom&, const float*, const float*, float*, cudaStream_t);
template int launch_conv_simt_wgrad<bf16>(const ConvGeom&, const bf16*, const bf16*, float*, cudaStream_t);

}  // namespace mapnet
