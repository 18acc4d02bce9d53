// BatchNorm (training statistics) + ReLU + residual add + stem max-pool, forward
// and backward, on NHWC activations.  HBM-bound: 128-bit vectorised accesses,
// fp32 math, per-thread channel-vector accumulators; block partials are combined with
// fp64 atomics and the LAST block to arrive finalizes (no separate finalize launch).
// One apply kernel per direction: it takes its per-channel parameters either from accumulated sums (finalized in its
// prologue) or from memory (bn_fin.cuh, BnDesc).
//
// Replaces the library calls behind torchvision BasicBlock / ResNet.forward
// (cuDNN BN fwd-training/bwd, THCUNN threshold, TH add, SpatialDilatedMaxPooling;
// SURVEY.md section 2c) that /root/reference/models/posenet.py:66 runs.
#include "kernels.h"
#include "bn_fin.cuh"

namespace mapnet {

static const int kEwThreads = 256;

// ---------------------------------------------------------------------------
// per-channel sums over pixels, finalize fused into the LAST block to arrive:
//   MODE 0: (sum y, sum y^2)            -> batch mean / invstd / scale / shift, running stats
//   MODE 1: (sum g, sum g*y)            -> d gamma, d beta, dy = A*g + B*y + C coefficients
//   MODE 2: (sum g, sum g*y, sum g*yd)  -> the same for the main AND the downsample BN
//   g = dout * [z > 0]
// Block partials are combined with fp64 atomics into the replicated accumulators of bn_fin.cuh (same-address atomics
// serialise at ~30 ns each); the finalizing block sums the replicas and resets them.
// ---------------------------------------------------------------------------
// 8 consecutive per-channel floats (32-byte aligned: channel offsets are multiples of 8) as two
// 128-bit loads; scalar loads here cost 8 L1 wavefronts per warp instruction once C >= 256
__device__ __forceinline__ void ld8(const float* __restrict__ p, float* o) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}


template <typename T, typename TZ, int MODE>
__global__ void __launch_bounds__(kEwThreads)
k_channel_sums(const T* __restrict__ a, const TZ* __restrict__ zmask, const T* __restrict__ y,
               const T* __restrict__ yd, long long M, int C, double* __restrict__ accum,
               unsigned int* __restrict__ counter, BnFin f) {
  pdl_prologue();
  constexpr int NACC = (MODE == 2) ? 3 : 2;
  const int cv = C >> 3;                      // channel vectors per pixel
  const int rows_par = kEwThreads / cv;       // pixels processed in parallel by the block
  const int tx = threadIdx.x % cv, ty = threadIdx.x / cv;
  float acc[NACC][8];
#pragma unroll
  for (int j = 0; j < NACC; ++j)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
  const long long rstep = (long long)gridDim.x * rows_par;
  float msc[8], msh[8];
  const bool ymask = (MODE != 0) && (zmask == nullptr) && (f.mscale != nullptr);
  if (ymask) { ld8(f.mscale + tx * 8, msc); ld8(f.mshift + tx * 8, msh); }
#pragma unroll 4
  for (long long r = (long long)blockIdx.x * rows_par + ty; r < M; r += rstep) {
    const long long off = r * C + tx * 8;
    if (MODE == 0) {
      Vec8<T> v; v.load(a + off);
#pragma unroll
      for (int i = 0; i < 8; ++i) { acc[0][i] += v.v[i]; acc[1][i] += v.v[i] * v.v[i]; }
    } else {
      Vec8<T> g, yy; g.load(a + off); yy.load(y + off);
      if (zmask != nullptr) {
        Vec8<TZ> z; z.load(zmask + off);
#pragma unroll
        for (int i = 0; i < 8; ++i) g.v[i] = (z.v[i] > 0.f) ? g.v[i] : 0.f;
      } else if (ymask) {
#pragma unroll
        for (int i = 0; i < 8; ++i) g.v[i] = (yy.v[i] * msc[i] + msh[i] > 0.f) ? g.v[i] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) { acc[0][i] += g.v[i]; acc[1][i] += g.v[i] * yy.v[i]; }
      if (MODE == 2) {
        Vec8<T> y2; y2.load(yd + off);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[2][i] += g.v[i] * y2.v[i];
      }
    }
  }
  // replicas actually used by this launch: small grids need few (the finalizing block walks them all)
  int nrep = (int)gridDim.x / 16;
  nrep = nrep < 4 ? 4 : (nrep > kBnAccReplicas ? kBnAccReplicas : nrep);
  // reduce across ty through shared memory (rows_par <= 32)
  extern __shared__ float sm[];               // [rows_par][NACC][C]
#pragma unroll
  for (int j = 0; j < NACC; ++j)
#pragma unroll
    for (int i = 0; i < 8; ++i) sm[((size_t)ty * NACC + j) * C + tx * 8 + i] = acc[j][i];
  __syncthreads();
  for (int idx = threadIdx.x; idx < NACC * C; idx += kEwThreads) {
    float s = 0.f;
    for (int t = 0; t < rows_par; ++t) s += sm[(size_t)t * NACC * C + idx];
    atomicAdd(accum + (size_t)(blockIdx.x % nrep) * kBnAccStride + idx, (double)s);
  }
  // ---- last block finalizes ----
  __shared__ unsigned int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // sum the replicas into shared memory (reuse the reduction buffer: NACC*C doubles <= 12 KB... held as
  // doubles in a separate static array to keep precision)
  __shared__ double s_tot[kBnAccStride];
  for (int idx = threadIdx.x; idx < NACC * C; idx += kEwThreads) {
    double t = 0.0;
#pragma unroll 8
    for (int r = 0; r < nrep; ++r) t += __ldcg(accum + (size_t)r * kBnAccStride + idx);
    s_tot[idx] = t;
#pragma unroll 8
    for (int r = 0; r < nrep; ++r) accum[(size_t)r * kBnAccStride + idx] = 0.0;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kEwThreads) {
    const double s0 = s_tot[c], s1 = s_tot[C + c];
    if (MODE == 0) bn_fin_forward(c, s0, s1, M, f);
    else bn_fin_backward(c, C, s0, s1, (MODE == 2) ? s_tot[2 * C + c] : 0.0, M, f, MODE == 2);
  }
  if (threadIdx.x == 0) *counter = 0u;
}

static int sums_grid(long long M, int C) {
  const int rows_par = kEwThreads / (C >> 3);
  long long want = (M + (long long)rows_par * 8 - 1) / ((long long)rows_par * 8);   // >= 8 rows per thread
  const long long cap = (long long)kNumSMs * 4;
  if (want < 1) want = 1;
  return (int)(want < cap ? want : cap);
}

template <typename T, typename TZ>
static int launch_sums(int mode, const T* a, const TZ* zmask, const T* y, const T* yd, long long M, int C,
                       double* accum, unsigned int* counter, const BnFin& f, cudaStream_t st) {
  MN_CHECK(C % 8 == 0 && C >= 8 && (kEwThreads % (C >> 3)) == 0 && C <= 512, "channel_sums: unsupported C=%d", C);
  const int grid = sums_grid(M, C);
  const int rows_par = kEwThreads / (C >> 3);
  const int nacc = (mode == 2) ? 3 : 2;
  const size_t smem = (size_t)rows_par * nacc * C * sizeof(float);
  if (mode == 0) MN_LAUNCH((k_channel_sums<T, TZ, 0>), grid, kEwThreads, smem, st, a, nullptr, nullptr, nullptr, M, C, accum, counter, f);
  else if (mode == 1) MN_LAUNCH((k_channel_sums<T, TZ, 1>), grid, kEwThreads, smem, st, a, zmask, y, nullptr, M, C, accum, counter, f);
  else MN_LAUNCH((k_channel_sums<T, TZ, 2>), grid, kEwThreads, smem, st, a, zmask, y, yd, M, C, accum, counter, f);
  MN_LAUNCH_CHECK();
  return 0;
}

// finalize for backward reductions accumulated in bn_accum by another kernel (the stem's pool backward in the
// CUDA-core modes): same arithmetic as MODE 1 / 2 of k_channel_sums
__global__ void __launch_bounds__(1024)
k_bn_bwd_finalize_accum(long long M, int C, BnFin f, double* __restrict__ accum, int nacc) {
  pdl_prologue();
  __shared__ double ss[3][32][33];
  const int cl = threadIdx.x, r = threadIdx.y;
  const int c = blockIdx.x * 32 + cl;
  double v0 = 0.0, v1 = 0.0, v2 = 0.0;
  if (c < C && r < kBnAccReplicas) {
    double* a = accum + (size_t)r * kBnAccStride;
    v0 = a[c]; v1 = a[C + c];
    a[c] = 0.0; a[C + c] = 0.0;
    if (nacc == 3) { v2 = a[2 * C + c]; a[2 * C + c] = 0.0; }
  }
  ss[0][r][cl] = v0; ss[1][r][cl] = v1; ss[2][r][cl] = v2;
  __syncthreads();
  if (r != 0 || c >= C) return;
  double s0 = 0.0, s1 = 0.0, s1d = 0.0;
#pragma unroll
  for (int k = 0; k < 32; ++k) { s0 += ss[0][k][cl]; s1 += ss[1][k][cl]; s1d += ss[2][k][cl]; }
  bn_fin_backward(c, C, s0, s1, s1d, M, f, nacc == 3);
}

int launch_bn_bwd_finalize_accum(long long M, int C, const BnFin& f, double* accum, cudaStream_t st) {
  MN_CHECK(C <= 512, "bn_bwd_finalize_accum: C=%d", C);
  MN_LAUNCH(k_bn_bwd_finalize_accum, cdiv(C, 32), dim3(32, 32), 0, st, M, C, f, accum, f.gamma2 != nullptr ? 3 : 2);
  MN_LAUNCH_CHECK();
  return 0;
}

// eval-mode scale/shift from the running statistics (no batch statistics)
__global__ void k_bn_eval_scale(int C, const BnFin f) {
  pdl_prologue();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float mean = f.run_mean[c];
  const float invstd = 1.0f / sqrtf(f.run_var[c] + 1e-5f);
  f.mean[c] = mean; f.invstd[c] = invstd;
  const float sc = f.gamma[c] * invstd;
  f.scale[c] = sc; f.shift[c] = f.beta[c] - mean * sc;
}

int launch_bn_eval_scale(int C, const BnFin& f, cudaStream_t st) {
  MN_LAUNCH(k_bn_eval_scale, cdiv(C, 128), 128, 0, st, C, f);
  MN_LAUNCH_CHECK();
  return 0;
}

template <typename T>
int launch_bn_stats(const T* y, long long M, int C, const BnFin& f, double* accum, unsigned int* counter, cudaStream_t st) {
  return launch_sums<T, T>(0, y, nullptr, nullptr, nullptr, M, C, accum, counter, f, st);
}
template int launch_bn_stats<float>(const float*, long long, int, const BnFin&, double*, unsigned int*, cudaStream_t);
template int launch_bn_stats<bf16>(const bf16*, long long, int, const BnFin&, double*, unsigned int*, cudaStream_t);

template <typename T, typename TZ>
int launch_bn_bwd_reduce(const T* dout, const TZ* zmask, const T* y, const T* yd, long long M, int C, const BnFin& f,
                         double* accum, unsigned int* counter, cudaStream_t st) {
  return launch_sums<T, TZ>(yd != nullptr ? 2 : 1, dout, zmask, y, yd, M, C, accum, counter, f, st);
}
#define MN_INST_BWD_REDUCE(TA, TZ) template int launch_bn_bwd_reduce<TA, TZ>(const TA*, const TZ*, const TA*, const TA*, long long, int, const BnFin&, double*, unsigned int*, cudaStream_t);
MN_INST_BWD_REDUCE(float, float)
MN_INST_BWD_REDUCE(bf16, bf16)
MN_INST_BWD_REDUCE(float, hsplit)

// ---------------------------------------------------------------------------
// Apply kernels.  Blocks are laid out (x: pixel groups, y: 64-channel slices) so that a block only needs the
// parameters of 64 channels; its prologue puts them in shared memory, read from memory or finalized from the sums
// (bn_fin.cuh, BnDesc).  Lazy finalize: thread t sums replicas (t >> 6), (t >> 6) + 4, ... of channel cbase + (t & 63)
// -- coalesced 512-byte rows of doubles -- the four partial sums meet in shared memory.  Thread t < 64 then owns
// channel cbase + t.
// ---------------------------------------------------------------------------
template <int NACC>
__device__ __forceinline__ void lazy_sums(const BnDesc& L, const int C, const int cbase, double (*part)[3][64],
                                          double (&s)[3]) {
  const int c = threadIdx.x & 63, rg = threadIdx.x >> 6;
  double t[3] = {0.0, 0.0, 0.0};
  for (int r = rg; r < L.nrep; r += 4) {
    const double* a = L.accum + (size_t)r * kBnAccStride + cbase + c;
#pragma unroll
    for (int j = 0; j < NACC; ++j) t[j] += __ldcg(a + (size_t)j * C);
  }
#pragma unroll
  for (int j = 0; j < NACC; ++j) part[rg][j][c] = t[j];
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 3; ++j) s[j] = (j < NACC) ? (part[0][j][c] + part[1][j][c]) + (part[2][j][c] + part[3][j][c]) : 0.0;
  __syncthreads();                   // `part` may be reused by a second BatchNorm
}

// forward: (scale, shift) of the block's 64 channels into shared memory -- from the sums (lazy) or from memory
__device__ __forceinline__ void lazy_forward_params(const BnDesc& L, const int C, const int cbase, double (*part)[3][64],
                                                    float (*out)[64]) {
  if (L.accum != nullptr) {
    // gamma / beta are fetched before the sums so that the two memory latencies overlap
    float ga = 0.f, be = 0.f;
    if (threadIdx.x < 64) { ga = __ldg(L.f.gamma + cbase + threadIdx.x); be = __ldg(L.f.beta + cbase + threadIdx.x); }
    double s[3];
    lazy_sums<2>(L, C, cbase, part, s);
    if (threadIdx.x < 64) {
      const int c = cbase + threadIdx.x;
      // bn_fin_forward's quantities with the fp64 division and square root taken off the critical path: 1 / M comes
      // from the host and 1 / sqrt is the fp64 rsqrt intrinsic (a few ulp of fp64, i.e. the same fp32 value after
      // rounding except in ~1e-8 of the cases); every block computes the same bits, block x == 0 publishes them
      const double m = s[0] * L.invM;
      double var = s[1] * L.invM - m * m;
      if (var < 0.0) var = 0.0;
      const float mean = (float)m;
      const float invstd = (float)rsqrt(var + 1e-5);
      const float sc = ga * invstd;
      const float sh = be - mean * sc;
      out[0][threadIdx.x] = sc;
      out[1][threadIdx.x] = sh;
      if (blockIdx.x == 0) {
        L.f.mean[c] = mean; L.f.invstd[c] = invstd; L.f.scale[c] = sc; L.f.shift[c] = sh;
        L.f.run_mean[c] = 0.9f * L.f.run_mean[c] + 0.1f * mean;
        L.f.run_var[c] = 0.9f * L.f.run_var[c] + 0.1f * (float)(var * L.unbias);
      }
    }
  } else if (threadIdx.x < 64) {
    out[0][threadIdx.x] = __ldg(L.f.scale + cbase + threadIdx.x);
    out[1][threadIdx.x] = __ldg(L.f.shift + cbase + threadIdx.x);
  }
}

// at most 8 blocks of 256 threads per SM (full occupancy): with 4 loads in flight per thread they cover the HBM
// latency-bandwidth product, and fewer, fatter threads amortise the per-block parameter prologue over more pixels
static int slice_grid_x(long long M, int C) {
  const long long slices = C >> 6;
  long long gx = (M + 31) / 32;
  long long cap = ((long long)kNumSMs * 8) / slices;
  if (cap < 1) cap = 1;
  if (gx > cap) gx = cap;
  return (int)(gx < 1 ? 1 : gx);
}

// The apply kernels request the first pixel's operands BEFORE their prologue (sums -> fp64 math -> shared memory), so
// that the DRAM latency overlaps it: those operands are held raw (Raw8) and converted at first use.  The per-pixel body
// takes each operand from there (PRE) or loads it (every later pixel).
template <bool PRE, typename V, typename R, typename P>
__device__ __forceinline__ void fetch8(V& v, const R& pre, const P* __restrict__ p) { if (PRE) pre.get(v); else v.load(p); }

// ---------------------------------------------------------------------------
// forward apply:  z = relu?( scale*y + shift  [+ zres | + scale2*y2 + shift2] )
// ---------------------------------------------------------------------------
// y (and the downsample branch's conv output) are conv outputs (T); the identity residual and the result are
// forward conv operands (TZ).  RES 0 none, 1 identity tensor, 2 second BN (downsample branch).
template <typename T, typename TZ, int RES>
struct ApplyIn {
  Raw8<T> y, y2; Raw8<TZ> r;
  __device__ __forceinline__ void load(const T* __restrict__ py, const void* __restrict__ res, const long long off) {
    y.load(py + off);
    if (RES == 1) r.load(reinterpret_cast<const TZ*>(res) + off);
    if (RES == 2) y2.load(reinterpret_cast<const T*>(res) + off);
  }
};

// one pixel's 8 channels; p = {scale, shift, scale2, shift2}
template <typename T, typename TZ, int RES, bool PRE>
__device__ __forceinline__ void bn_apply_pixel(const ApplyIn<T, TZ, RES>& pre, const T* __restrict__ y,
                                               const void* __restrict__ res, const float (&p)[4][8], const bool relu,
                                               TZ* __restrict__ z, const long long off) {
  Vec8<T> v; fetch8<PRE>(v, pre.y, y + off);
  float o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] = v.v[k] * p[0][k] + p[1][k];
  if (RES == 1) {
    Vec8<TZ> r; fetch8<PRE>(r, pre.r, reinterpret_cast<const TZ*>(res) + off);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] += r.v[k];
  } else if (RES == 2) {
    Vec8<T> r; fetch8<PRE>(r, pre.y2, reinterpret_cast<const T*>(res) + off);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] += r.v[k] * p[2][k] + p[3][k];
  }
  Vec8<TZ> w;
#pragma unroll
  for (int k = 0; k < 8; ++k) w.v[k] = relu ? fmaxf(o[k], 0.f) : o[k];
  w.store(z + off);
}

// block (x, y) walks pixels x*32 + (t >> 3), ... of channel slice y; thread t owns the 8 channels cbase + 8 * (t & 7)
// (one 128-byte line of bf16 per pixel and slice)
template <typename T, typename TZ, int RES>
__global__ void __launch_bounds__(kEwThreads)
k_bn_apply(const T* __restrict__ y, const void* __restrict__ res, TZ* __restrict__ z, long long M, int C, int relu,
           const BnDesc L1, const BnDesc L2) {
  pdl_prologue();
  __shared__ double part[4][3][64];
  __shared__ float par[4][64];
  const int cbase = blockIdx.y * 64;
  const int cl = (threadIdx.x & 7) * 8;
  const long long p0 = (long long)blockIdx.x * 32 + (threadIdx.x >> 3);
  const long long pstep = (long long)gridDim.x * 32;
  ApplyIn<T, TZ, RES> in0;
  if (p0 < M) in0.load(y, res, p0 * C + cbase + cl);
  lazy_forward_params(L1, C, cbase, part, par);
  if (RES == 2) lazy_forward_params(L2, C, cbase, part, par + 2);
  __syncthreads();
  float p[4][8];
#pragma unroll
  for (int j = 0; j < (RES == 2 ? 4 : 2); ++j)
#pragma unroll
    for (int k = 0; k < 8; ++k) p[j][k] = par[j][cl + k];
  const bool rl = relu != 0;
  if (p0 < M) bn_apply_pixel<T, TZ, RES, true>(in0, y, res, p, rl, z, p0 * C + cbase + cl);
#pragma unroll 4
  for (long long px = p0 + pstep; px < M; px += pstep)
    bn_apply_pixel<T, TZ, RES, false>(in0, y, res, p, rl, z, px * C + cbase + cl);
}

static int ew_grid(long long n) {
  long long g = (n + kEwThreads - 1) / kEwThreads;
  const long long cap = (long long)kNumSMs * 8;       // as slice_grid_x
  return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}

template <typename T, typename TZ>
int launch_bn_apply(const T* y, int res_mode, const void* res, TZ* z, long long M, int C, int relu, const BnDesc& bn,
                    const BnDesc* bn_ds, cudaStream_t st) {
  MN_CHECK(C % 64 == 0 && C <= 512, "bn_apply: C=%d", C);
  MN_CHECK(res_mode != 2 || bn_ds != nullptr, "bn_apply: the downsample BN needs its descriptor too");
  const dim3 grid(slice_grid_x(M, C), C >> 6);
  if (res_mode == 0) MN_LAUNCH((k_bn_apply<T, TZ, 0>), grid, kEwThreads, 0, st, y, nullptr, z, M, C, relu, bn, bn);
  else if (res_mode == 1) MN_LAUNCH((k_bn_apply<T, TZ, 1>), grid, kEwThreads, 0, st, y, res, z, M, C, relu, bn, bn);
  else MN_LAUNCH((k_bn_apply<T, TZ, 2>), grid, kEwThreads, 0, st, y, res, z, M, C, relu, bn, *bn_ds);
  MN_LAUNCH_CHECK();
  return 0;
}
#define MN_INST_BN_APPLY(TA, TZ) template int launch_bn_apply<TA, TZ>(const TA*, int, const void*, TZ*, long long, int, int, const BnDesc&, const BnDesc*, cudaStream_t);
MN_INST_BN_APPLY(float, float)
MN_INST_BN_APPLY(bf16, bf16)
MN_INST_BN_APPLY(float, hsplit)

// ---------------------------------------------------------------------------
// stem: z0 = maxpool3x3s2p1( relu( scale*y0 + shift ) ), argmax position kept
// (first maximum in window scan order wins, as torch's max_pool2d does)
// ---------------------------------------------------------------------------
template <typename T, typename TZ>
__global__ void __launch_bounds__(kEwThreads)
k_stem_pool(const T* __restrict__ y, TZ* __restrict__ z, uint8_t* __restrict__ amax, int B, int H, int W, int Ho, int Wo,
            int C, const BnDesc L) {
  pdl_prologue();
  // lazy finalize of the stem BatchNorm (C == 64: one channel slice, every block derives all 64 scale / shift pairs)
  __shared__ double part[4][3][64];
  __shared__ float par[2][64];
  if (L.accum != nullptr) {
    lazy_forward_params(L, C, 0, part, par);
    __syncthreads();
  }
  const int cv = C >> 3;
  // 32-bit index arithmetic (the launcher checks the element count): 64-bit div / mod per element made this kernel
  // latency-bound (ncu r02a: 89 us for 165 MB, 23 % of DRAM peak)
  const unsigned int nvec = (unsigned int)B * Ho * Wo * cv;
  for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gridDim.x * blockDim.x) {
    const int c0 = (int)(i % cv) * 8;
    unsigned int p = i / cv;
    const int ow = (int)(p % Wo); p /= Wo;
    const int oh = (int)(p % Ho);
    const int b = (int)(p / Ho);
    float best[8]; int bi[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { best[k] = -INFINITY; bi[k] = 0; }
    float sc[8], sh[8];
    if (L.accum != nullptr) {
#pragma unroll
      for (int k = 0; k < 8; ++k) { sc[k] = par[0][c0 + k]; sh[k] = par[1][c0 + k]; }
    } else { ld8(L.f.scale + c0, sc); ld8(L.f.shift + c0, sh); }
    // all nine window loads are issued unconditionally (border taps read a clamped, valid pixel and are masked out
    // below): with the loads under the border branches the compiler kept them serial and the kernel ran at 23 % of the
    // DRAM rate (ncu r02a: 89 us for 165 MB)
    Vec8<T> v[9]; bool ok[9];
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int ih = oh * 2 - 1 + kh;
      const bool okh = (ih >= 0) && (ih < H);
      const int ihc = okh ? ih : oh * 2;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int iw = ow * 2 - 1 + kw;
        const bool okw = (iw >= 0) && (iw < W);
        const int iwc = okw ? iw : ow * 2;
        ok[kh * 3 + kw] = okh && okw;
        v[kh * 3 + kw].load(y + ((size_t)((unsigned int)b * H + ihc) * W + iwc) * C + c0);
      }
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float a = ok[t] ? fmaxf(v[t].v[k] * sc[k] + sh[k], 0.f) : -INFINITY;
        if (a > best[k]) { best[k] = a; bi[k] = t; }
      }
    }
    Vec8<TZ> o;
#pragma unroll
    for (int k = 0; k < 8; ++k) o.v[k] = best[k];
    o.store(z + (size_t)i * 8);
    uint2 packed;
    packed.x = (uint32_t)bi[0] | ((uint32_t)bi[1] << 8) | ((uint32_t)bi[2] << 16) | ((uint32_t)bi[3] << 24);
    packed.y = (uint32_t)bi[4] | ((uint32_t)bi[5] << 8) | ((uint32_t)bi[6] << 16) | ((uint32_t)bi[7] << 24);
    if (amax != nullptr) *reinterpret_cast<uint2*>(amax + (size_t)i * 8) = packed;
  }
}

template <typename T, typename TZ>
int launch_stem_pool(const T* y, TZ* z, uint8_t* amax, int B, int H, int W, int Ho, int Wo, int C, const BnDesc& bn,
                     cudaStream_t st) {
  const long long nvec = (long long)B * Ho * Wo * (C >> 3);
  MN_CHECK(nvec < 2147483647LL, "stem_pool: tensor too large for 32-bit indexing");
  MN_CHECK(bn.accum == nullptr || C == 64, "stem_pool (lazy finalize): C=%d", C);
  MN_LAUNCH((k_stem_pool<T, TZ>), ew_grid(nvec), kEwThreads, 0, st, y, z, amax, B, H, W, Ho, Wo, C, bn);
  MN_LAUNCH_CHECK();
  return 0;
}
#define MN_INST_STEM_POOL(TA, TZ) template int launch_stem_pool<TA, TZ>(const TA*, TZ*, uint8_t*, int, int, int, int, int, int, const BnDesc&, cudaStream_t);
MN_INST_STEM_POOL(float, float)
MN_INST_STEM_POOL(bf16, bf16)
MN_INST_STEM_POOL(float, hsplit)
MN_INST_STEM_POOL(bf16, e4m3)     // fp8 inference: the scale table holds 1 / s (layer1's input scale), the store saturates

// stem backward through max-pool and ReLU:  g0[b,ih,iw,c] = [a0>0] * sum_{windows whose argmax is (ih,iw)} dz
template <typename T>
__global__ void __launch_bounds__(kEwThreads)
k_stem_pool_bwd(const T* __restrict__ dz, const uint8_t* __restrict__ amax, const T* __restrict__ y,
                const float* __restrict__ scale, const float* __restrict__ shift, T* __restrict__ g,
                int B, int H, int W, int Ho, int Wo, int C) {
  pdl_prologue();
  const int cv = C >> 3;
  const long long nvec = (long long)B * H * W * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % cv) * 8;
    long long p = i / cv;
    const int iw = (int)(p % W); p /= W;
    const int ih = (int)(p % H);
    const int b = (int)(p / H);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    // windows (oh,ow) with 2*oh-1 <= ih <= 2*oh+1
    const int oh_lo = (ih >= 1) ? (ih) / 2 : 0;            // ceil((ih-1)/2)
    const int oh_hi = (ih + 1) / 2;
    const int ow_lo = (iw >= 1) ? (iw) / 2 : 0;
    const int ow_hi = (iw + 1) / 2;
    for (int oh = oh_lo; oh <= oh_hi && oh < Ho; ++oh) {
      const int kh = ih - (oh * 2 - 1);
      if (kh < 0 || kh > 2) continue;
      for (int ow = ow_lo; ow <= ow_hi && ow < Wo; ++ow) {
        const int kw = iw - (ow * 2 - 1);
        if (kw < 0 || kw > 2) continue;
        const long long o = (((long long)b * Ho + oh) * Wo + ow) * C + c0;
        const uint2 pk = *reinterpret_cast<const uint2*>(amax + o);
        Vec8<T> d; d.load(dz + o);
        const int pos = kh * 3 + kw;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t word = (k < 4) ? pk.x : pk.y;
          const int idx = (word >> ((k & 3) * 8)) & 0xff;
          if (idx == pos) acc[k] += d.v[k];
        }
      }
    }
    Vec8<T> yy; yy.load(y + i * 8);
    float sc[8], sh[8];
    ld8(scale + c0, sc); ld8(shift + c0, sh);
    Vec8<T> o;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float a = yy.v[k] * sc[k] + sh[k];
      o.v[k] = (a > 0.f) ? acc[k] : 0.f;
    }
    o.store(g + i * 8);
  }
}

// Quad version (H, W even): one thread owns the 2x2 input pixels (2a..2a+1, 2b..2b+1) of 8 channels.
// They are covered by exactly the four pooling windows (a..a+1, b..b+1), so dz / argmax are read
// 4 times per quad instead of 9, and the reductions of the stem BatchNorm backward
// (sum g, sum g*y) are accumulated on the way (accum != nullptr): no separate pass over g and y.
template <typename T>
__global__ void __launch_bounds__(kEwThreads)
k_stem_pool_bwd_quad(const T* __restrict__ dz, const uint8_t* __restrict__ amax, const T* __restrict__ y,
                     const float* __restrict__ scale, const float* __restrict__ shift, T* __restrict__ g,
                     int B, int H, int W, int Ho, int Wo, int C, double* __restrict__ accum) {
  pdl_prologue();
  const int cv = C >> 3;
  const int Hq = H >> 1, Wq = W >> 1;
  const unsigned int nq = (unsigned int)B * Hq * Wq * cv;          // 32-bit index arithmetic (checked by the launcher)
  const unsigned int i0 = blockIdx.x * blockDim.x + threadIdx.x;
  const int c0 = (int)(i0 % cv) * 8;            // loop invariant: the grid stride is a multiple of cv
  float sc[8], sh[8], s0[8], s1[8];
  ld8(scale + c0, sc); ld8(shift + c0, sh);
#pragma unroll
  for (int k = 0; k < 8; ++k) { s0[k] = 0.f; s1[k] = 0.f; }
  for (unsigned int i = i0; i < nq; i += gridDim.x * blockDim.x) {
    unsigned int p = i / cv;
    const int qb = (int)(p % Wq); p /= Wq;
    const int qa = (int)(p % Hq);
    const int b = (int)(p / Hq);
    // windows (qa + dh, qb + dw): gradient and argmax position (kh*3+kw inside the window)
    float d[4][8]; uint2 pk[4];
#pragma unroll
    for (int dh = 0; dh < 2; ++dh)
#pragma unroll
      for (int dw = 0; dw < 2; ++dw) {
        const int oh = qa + dh, ow = qb + dw;
        const int w = dh * 2 + dw;
        if (oh < Ho && ow < Wo) {
          const long long o = (((long long)b * Ho + oh) * Wo + ow) * C + c0;
          pk[w] = *reinterpret_cast<const uint2*>(amax + o);
          Vec8<T> t; t.load(dz + o);
#pragma unroll
          for (int k = 0; k < 8; ++k) d[w][k] = t.v[k];
        } else {
          pk[w] = make_uint2(0xffffffffu, 0xffffffffu);
#pragma unroll
          for (int k = 0; k < 8; ++k) d[w][k] = 0.f;
        }
      }
    // pixel (r, c) of the quad sits at window position: w00 -> (1+r)*3 + (1+c); w01 (c == 1) -> (1+r)*3;
    // w10 (r == 1) -> (1+c); w11 (r == c == 1) -> 0
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const long long off = (((long long)b * H + 2 * qa + r) * W + 2 * qb + c) * C + c0;
        Vec8<T> yy; yy.load(y + off);
        Vec8<T> o;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int sft = (k & 3) * 8;
          const uint32_t i00 = (((k < 4) ? pk[0].x : pk[0].y) >> sft) & 0xff;
          const uint32_t i01 = (((k < 4) ? pk[1].x : pk[1].y) >> sft) & 0xff;
          const uint32_t i10 = (((k < 4) ? pk[2].x : pk[2].y) >> sft) & 0xff;
          const uint32_t i11 = (((k < 4) ? pk[3].x : pk[3].y) >> sft) & 0xff;
          float a = (i00 == (uint32_t)((1 + r) * 3 + 1 + c)) ? d[0][k] : 0.f;
          if (c == 1) a += (i01 == (uint32_t)((1 + r) * 3)) ? d[1][k] : 0.f;
          if (r == 1) a += (i10 == (uint32_t)(1 + c)) ? d[2][k] : 0.f;
          if (r == 1 && c == 1) a += (i11 == 0u) ? d[3][k] : 0.f;
          const float act = yy.v[k] * sc[k] + sh[k];
          o.v[k] = (act > 0.f) ? a : 0.f;
        }
        o.store(g + off);
        if (accum != nullptr) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float gs = to_f(from_f<T>(o.v[k]));       // the value as stored
            s0[k] += gs; s1[k] += gs * yy.v[k];
          }
        }
      }
  }
  if (accum == nullptr) return;
  // block reduction over the threads that share a channel vector, then one fp64 atomic per channel
  extern __shared__ float sm[];                 // [kEwThreads / cv][2][C]
  const int tx = threadIdx.x % cv, ty = threadIdx.x / cv, rows = kEwThreads / cv;
#pragma unroll
  for (int k = 0; k < 8; ++k) { sm[(ty * 2 + 0) * C + tx * 8 + k] = s0[k]; sm[(ty * 2 + 1) * C + tx * 8 + k] = s1[k]; }
  __syncthreads();
  int nrep = (int)gridDim.x / 16;
  nrep = nrep < 4 ? 4 : (nrep > kBnAccReplicas ? kBnAccReplicas : nrep);
  for (int idx = threadIdx.x; idx < 2 * C; idx += kEwThreads) {
    float t = 0.f;
    for (int r = 0; r < rows; ++r) t += sm[r * 2 * C + idx];
    atomicAdd(accum + (size_t)(blockIdx.x % nrep) * kBnAccStride + idx, (double)t);
  }
}

template <typename T>
int launch_stem_pool_bwd(const T* dz, const uint8_t* amax, const T* y, const float* scale, const float* shift,
                         T* g, int B, int H, int W, int Ho, int Wo, int C, cudaStream_t st, double* accum) {
  if ((H % 2) == 0 && (W % 2) == 0 && Ho == H / 2 && Wo == W / 2 && kEwThreads % (C >> 3) == 0) {
    const long long nq = (long long)B * (H / 2) * (W / 2) * (C >> 3);
    MN_CHECK(nq < 2147483647LL, "stem_pool_bwd: tensor too large for 32-bit indexing");
    const size_t smem = accum ? (size_t)(kEwThreads / (C >> 3)) * 2 * C * sizeof(float) : 0;
    MN_LAUNCH(k_stem_pool_bwd_quad<T>, ew_grid(nq), kEwThreads, smem, st, dz, amax, y, scale, shift, g, B, H, W, Ho, Wo, C, accum);
    MN_LAUNCH_CHECK();
    return 0;
  }
  MN_CHECK(accum == nullptr, "stem_pool_bwd: fused reductions need even H, W (got %dx%d)", H, W);
  const long long nvec = (long long)B * H * W * (C >> 3);
  MN_LAUNCH(k_stem_pool_bwd<T>, ew_grid(nvec), kEwThreads, 0, st, dz, amax, y, scale, shift, g, B, H, W, Ho, Wo, C);
  MN_LAUNCH_CHECK();
  return 0;
}
template int launch_stem_pool_bwd<float>(const float*, const uint8_t*, const float*, const float*, const float*, float*, int, int, int, int, int, int, cudaStream_t, double*);
template int launch_stem_pool_bwd<bf16>(const bf16*, const uint8_t*, const bf16*, const float*, const float*, bf16*, int, int, int, int, int, int, cudaStream_t, double*);

// ---------------------------------------------------------------------------
// backward apply: dy = A*g + B*y + C  [, dyd = Ad*g + Bd*yd + Cd] [, gout = g]
// ---------------------------------------------------------------------------
// dout / y / yd / gout: fp32-math tensors (T); zmask: a forward conv operand (TZ); dy / dyd: backward conv operands (TG).
template <typename T, typename TZ, int DS>
struct BwdApplyIn {
  Raw8<T> g, y, yd; Raw8<TZ> z;
  __device__ __forceinline__ void load(const T* __restrict__ dout, const TZ* __restrict__ zmask, const T* __restrict__ py,
                                       const T* __restrict__ pyd, const long long off) {
    g.load(dout + off); y.load(py + off);
    if (zmask != nullptr) z.load(zmask + off);
    if (DS) yd.load(pyd + off);
  }
};

// one pixel's 8 channels; g is gated by the ReLU: zmask > 0 or mscale*y + mshift > 0 (ygate);
// p = {A, B, C, Ad, Bd, Cd, mscale, mshift}
template <typename T, typename TZ, typename TG, int DS, int GOUT, bool PRE>
__device__ __forceinline__ void bn_bwd_apply_pixel(const BwdApplyIn<T, TZ, DS>& pre, const T* __restrict__ dout,
                                                   const TZ* __restrict__ zmask, const T* __restrict__ y,
                                                   const T* __restrict__ yd, const float (&p)[8][8], const bool ygate,
                                                   TG* __restrict__ dy, TG* __restrict__ dyd, T* __restrict__ gout,
                                                   const long long off) {
  Vec8<T> g, yy;
  fetch8<PRE>(g, pre.g, dout + off); fetch8<PRE>(yy, pre.y, y + off);
  if (zmask != nullptr) {
    Vec8<TZ> z; fetch8<PRE>(z, pre.z, zmask + off);
#pragma unroll
    for (int k = 0; k < 8; ++k) g.v[k] = (z.v[k] > 0.f) ? g.v[k] : 0.f;
  } else if (ygate) {
#pragma unroll
    for (int k = 0; k < 8; ++k) g.v[k] = (yy.v[k] * p[6][k] + p[7][k] > 0.f) ? g.v[k] : 0.f;
  }
  Vec8<TG> o;
#pragma unroll
  for (int k = 0; k < 8; ++k) o.v[k] = p[0][k] * g.v[k] + p[1][k] * yy.v[k] + p[2][k];
  o.store(dy + off);
  if (DS) {
    Vec8<T> y2; fetch8<PRE>(y2, pre.yd, yd + off);
    Vec8<TG> o2;
#pragma unroll
    for (int k = 0; k < 8; ++k) o2.v[k] = p[3][k] * g.v[k] + p[4][k] * y2.v[k] + p[5][k];
    o2.store(dyd + off);
  }
  if (GOUT) g.store(gout + off);
}

// Same block layout as k_bn_apply.  With sums (L.accum != nullptr) the block derives A, B, C (and the downsample
// BatchNorm's) for its 64 channels from the sums the producing dgrad / pool-backward kernel accumulated, and
// blockIdx.x == 0 writes d gamma / d beta (and the coefficients, for the record); without, it reads the coefficients.
// gscale != nullptr (strict mode): the coefficients are multiplied by the step's power-of-two scale *gscale in fp32.
template <typename T, typename TZ, typename TG, int DS, int GOUT>
__global__ void __launch_bounds__(kEwThreads)
k_bn_bwd_apply(const T* __restrict__ dout, const TZ* __restrict__ zmask, const T* __restrict__ y, TG* __restrict__ dy,
               const T* __restrict__ yd, TG* __restrict__ dyd, T* __restrict__ gout, long long M, int C,
               const float* __restrict__ gscale, const BnDesc L) {
  pdl_prologue();
  __shared__ double part[4][3][64];
  __shared__ float par[8][64];            // A, B, C, Ad, Bd, Cd, mscale, mshift
  const int cbase = blockIdx.y * 64;
  const int cl = (threadIdx.x & 7) * 8;
  const long long p0 = (long long)blockIdx.x * 32 + (threadIdx.x >> 3);
  const long long pstep = (long long)gridDim.x * 32;
  BwdApplyIn<T, TZ, DS> in0;
  if (p0 < M) in0.load(dout, zmask, y, yd, p0 * C + cbase + cl);
  {
    const int t = threadIdx.x, c = cbase + t;
    // per-channel inputs of the finalize are fetched before the sums so that the memory latencies overlap
    float pmu = 0.f, pis = 0.f, pga = 0.f, pmu2 = 0.f, pis2 = 0.f, pga2 = 0.f, S = 1.f;
    if (t < 64) {
      if (gscale != nullptr) S = __ldg(gscale);
      if (L.accum != nullptr) {
        pmu = __ldg(L.f.mean + c); pis = __ldg(L.f.invstd + c); pga = __ldg(L.f.gamma + c);
        if (DS) { pmu2 = __ldg(L.f.mean2 + c); pis2 = __ldg(L.f.invstd2 + c); pga2 = __ldg(L.f.gamma2 + c); }
      } else {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          par[j][t] = __ldg(L.f.coef + j * C + c) * S;
          if (DS) par[3 + j][t] = __ldg(L.f.coef2 + j * C + c) * S;
        }
      }
      if (L.f.mscale != nullptr) { par[6][t] = __ldg(L.f.mscale + c); par[7][t] = __ldg(L.f.mshift + c); }
    }
    if (L.accum != nullptr) {
      double s[3];
      lazy_sums<DS ? 3 : 2>(L, C, cbase, part, s);
      if (t < 64) {
        const BnBwdCoef k = bn_bwd_coef(pmu, pis, pga, s[0], s[1], L.invM);
        par[0][t] = (float)k.A * S; par[1][t] = (float)k.B * S; par[2][t] = (float)k.C * S;
        if (DS) {
          const BnBwdCoef kd = bn_bwd_coef(pmu2, pis2, pga2, s[0], s[2], L.invM);
          par[3][t] = (float)kd.A * S; par[4][t] = (float)kd.B * S; par[5][t] = (float)kd.C * S;
        }
        if (blockIdx.x == 0) bn_fin_backward(c, C, s[0], s[1], s[2], L.M, L.f, DS != 0);
      }
    }
  }
  __syncthreads();
  const bool ygate = zmask == nullptr && L.f.mscale != nullptr;
  float p[8][8];
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (j < 3 || (DS && j < 6) || (j >= 6 && ygate))
#pragma unroll
      for (int k = 0; k < 8; ++k) p[j][k] = par[j][cl + k];
  if (p0 < M)
    bn_bwd_apply_pixel<T, TZ, TG, DS, GOUT, true>(in0, dout, zmask, y, yd, p, ygate, dy, dyd, gout, p0 * C + cbase + cl);
#pragma unroll 4
  for (long long px = p0 + pstep; px < M; px += pstep)
    bn_bwd_apply_pixel<T, TZ, TG, DS, GOUT, false>(in0, dout, zmask, y, yd, p, ygate, dy, dyd, gout, px * C + cbase + cl);
}

template <typename T, typename TZ, typename TG>
int launch_bn_bwd_apply(const T* dout, const TZ* zmask, const T* y, TG* dy, const T* yd, TG* dyd, T* gout, long long M,
                        int C, const BnDesc& bn, const float* gscale, cudaStream_t st) {
  MN_CHECK(C % 64 == 0 && C <= 512, "bn_bwd_apply: C=%d", C);
  const bool ds = (yd != nullptr), go = (gout != nullptr);
  const dim3 grid(slice_grid_x(M, C), C >> 6);
  if (ds && !go) MN_LAUNCH((k_bn_bwd_apply<T, TZ, TG, 1, 0>), grid, kEwThreads, 0, st, dout, zmask, y, dy, yd, dyd, gout, M, C, gscale, bn);
  else if (!ds && go) MN_LAUNCH((k_bn_bwd_apply<T, TZ, TG, 0, 1>), grid, kEwThreads, 0, st, dout, zmask, y, dy, yd, dyd, gout, M, C, gscale, bn);
  else if (!ds && !go) MN_LAUNCH((k_bn_bwd_apply<T, TZ, TG, 0, 0>), grid, kEwThreads, 0, st, dout, zmask, y, dy, yd, dyd, gout, M, C, gscale, bn);
  else MN_LAUNCH((k_bn_bwd_apply<T, TZ, TG, 1, 1>), grid, kEwThreads, 0, st, dout, zmask, y, dy, yd, dyd, gout, M, C, gscale, bn);
  MN_LAUNCH_CHECK();
  return 0;
}
#define MN_INST_BWD_APPLY(TA, TZ, TG) template int launch_bn_bwd_apply<TA, TZ, TG>(const TA*, const TZ*, const TA*, TG*, const TA*, TG*, TA*, long long, int, const BnDesc&, const float*, cudaStream_t);
MN_INST_BWD_APPLY(float, float, float)
MN_INST_BWD_APPLY(bf16, bf16, bf16)
MN_INST_BWD_APPLY(float, hsplit, hsplit)

}  // namespace mapnet
