// Layout transforms around the conv engines:
//  * pack_weights: fp32 master weights in torch layout [Co,Ci,KH,KW] (the
//    state_dict-compatible storage PyTorch owns, SURVEY.md section 8b) -> K-major GEMM
//    operands [Co][KH][KW][Ci] (fprop/wgrad) and [Ci][KH][KW][Co] (dgrad), in the
//    engine's operand type (fp32 or bf16).  All 36 convs in one launch.
//  * unpack_wgrads: wgrad accumulators [Co][KH][KW][Ci] fp32 -> .grad layout.
//  * stem_im2col: NCHW fp32 input -> [B*Ho*Wo][Kpad] patch matrix of the 7x7/s2/p3
//    stem conv (k = (kh*7+kw)*3+ci, zero padded to Kpad), so the stem runs through
//    the same GEMM engines as a 1x1 conv with Ci=Kpad.
#include "kernels.h"

namespace mapnet {

template <typename TW> __device__ __forceinline__ TW cvt_w(float v);
template <> __device__ __forceinline__ float cvt_w<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 cvt_w<bf16>(float v) { return __float2bfloat16_rn(v); }

// The master conv weights live in params_flat in the order the engines consume them: [Co][KH][KW][Ci] (KRSC,
// mapnet_param_layout == 1; to PyTorch the same memory is the [Co,Ci,KH,KW] parameter in channels_last strides).  The
// operand copy is then a plain fp32 -> TW conversion, and the weight gradients need no re-layout at all -- the two
// transposing passes of round 1 (k_pack_weights 83 us + k_unpack_wgrads 103 us per step, cold) are gone.
// Only the stem keeps torch's [64][3][7][7] order (layout 0): its slab becomes the padded [im2col_k] row of the patch
// GEMM through shared memory.  One block per (group of output channels, conv).
__host__ __device__ inline int pack_group(int n_in) { int g = 4096 / (n_in > 0 ? n_in : 1); return g < 1 ? 1 : (g > 8 ? 8 : g); }

template <typename TW>
__global__ void __launch_bounds__(256)
k_pack_weights(const WeightDesc* __restrict__ descs, const float* __restrict__ params,
               TW* __restrict__ w_krsc, TW* __restrict__ w_dg, int round_bf16) {
  pdl_prologue();
  extern __shared__ float slab[];
  const WeightDesc d = descs[blockIdx.y];
  const int KK = (d.im2col_k > 0) ? 49 : d.KH * d.KW;
  const int n_in = d.Ci_real * KK;
  const int G = (d.im2col_k > 0) ? 1 : pack_group(n_in);
  const int co = blockIdx.x * G;
  if (co >= d.Co) return;
  const int ng = (d.Co - co < G) ? d.Co - co : G;
  const float* src = params + d.p_off + (long long)co * n_in;
  if (d.im2col_k > 0) {
    for (int i = threadIdx.x; i < n_in; i += blockDim.x) slab[i] = src[i];
    __syncthreads();
    TW* dst = w_krsc + d.k_off + (long long)co * d.im2col_k;
    for (int k = threadIdx.x; k < d.im2col_k; k += blockDim.x) {
      float v = 0.f;
      if (d.s2d) {
        const int kh2 = k >> 6, kw2 = (k >> 4) & 3, ch = k & 15;
        if (ch < 12) {
          const int q = ch / 3, c = ch - q * 3;
          const int kh = 2 * kh2 + (q >> 1) - 1, kw = 2 * kw2 + (q & 1) - 1;
          if (kh >= 0 && kh < 7 && kw >= 0 && kw < 7) v = slab[c * 49 + kh * 7 + kw];
        }
      } else if (k < n_in) { const int t = k / d.Ci_real, c = k - t * d.Ci_real; v = slab[c * 49 + t]; }
      if (round_bf16) v = __bfloat162float(__float2bfloat16_rn(v));
      dst[k] = cvt_w<TW>(v);
    }
  } else {
    // same element order on both sides; n_in = KK * Ci is a multiple of 64 and both offsets are 64-float aligned
    TW* dst = w_krsc + d.k_off + (long long)co * n_in;
    const float4* s4 = reinterpret_cast<const float4*>(src);
    for (int jj = threadIdx.x; jj < (ng * n_in) >> 2; jj += blockDim.x) {
      float4 v = __ldg(s4 + jj);
      if (round_bf16) {
        v.x = __bfloat162float(__float2bfloat16_rn(v.x)); v.y = __bfloat162float(__float2bfloat16_rn(v.y));
        v.z = __bfloat162float(__float2bfloat16_rn(v.z)); v.w = __bfloat162float(__float2bfloat16_rn(v.w));
      }
      dst[4 * jj] = cvt_w<TW>(v.x); dst[4 * jj + 1] = cvt_w<TW>(v.y); dst[4 * jj + 2] = cvt_w<TW>(v.z); dst[4 * jj + 3] = cvt_w<TW>(v.w);
    }
  }
}

// w_dg[ci][tap][co] = w_krsc[co][tap][ci]: 32x32 shared-memory tile transpose per filter tap,
// coalesced on both sides (the dgrad engines want Cout as the contiguous K dimension)
template <typename TW>
__global__ void __launch_bounds__(256)
k_transpose_dg(const WeightDesc* __restrict__ descs, const TW* __restrict__ w_krsc, TW* __restrict__ w_dg) {
  pdl_prologue();
  const WeightDesc d = descs[blockIdx.y];
  if (d.im2col_k > 0) return;          // the stem has no dgrad
  const int KK = d.KH * d.KW;
  const int tco = d.Co >> 5, tci = d.Ci >> 5;
  const int ntiles = tco * tci * KK;
  __shared__ TW tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int tap = t % KK;
    const int cit = (t / KK) % tci;
    const int cot = t / (KK * tci);
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
      const int co = cot * 32 + r, ci = cit * 32 + tx;
      tile[r][tx] = w_krsc[d.k_off + ((long long)co * KK + tap) * d.Ci + ci];
    }
    __syncthreads();
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
      const int ci = cit * 32 + r, co = cot * 32 + tx;
      w_dg[d.k_off + ((long long)ci * KK + tap) * d.Co + co] = tile[tx][r];
    }
    __syncthreads();
  }
}

template <typename TW>
int launch_pack_weights(const WeightDesc* d_descs, int nconv, const float* params, TW* w_krsc, TW* w_dg,
                        int max_elems, int round_bf16, cudaStream_t st) {
  dim3 grid(512, nconv);                 // blockIdx.x = output channel group (<= 512), blocks past Co exit
  MN_LAUNCH(k_pack_weights<TW>, grid, 256, 3 * 49 * sizeof(float), st, d_descs, params, w_krsc, w_dg, round_bf16);
  MN_LAUNCH_CHECK();
  if (w_dg != nullptr) {
    dim3 g2(592, nconv);
    MN_LAUNCH(k_transpose_dg<TW>, g2, 256, 0, st, d_descs, w_krsc, w_dg);
    MN_LAUNCH_CHECK();
  }
  return 0;
}
// fp8 inference: one block per (output channel, conv).  The row's amax is an order-independent max, and
// s_w = 2^ceil(log2(amax / 448)) is taken from the exponent (f8_pow2_scale), so the packed weights are exactly reproducible.
__global__ void __launch_bounds__(256)
k_pack_weights_fp8(const WeightDesc* __restrict__ descs, const float* __restrict__ params, uint8_t* __restrict__ w8,
                   float* __restrict__ s_w) {
  pdl_prologue();
  const WeightDesc d = descs[blockIdx.y];
  const int co = blockIdx.x;
  if (d.im2col_k > 0 || co >= d.Co) return;         // the stem stays bf16
  const int n = d.KH * d.KW * d.Ci;
  const float* src = params + d.p_off + (long long)co * n;
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(src[i]));
  __shared__ float red[8];
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
  const float s = f8_pow2_scale(m), inv = 1.f / s;
  if (threadIdx.x == 0) s_w[blockIdx.y * 512 + co] = s;
  uint8_t* dst = w8 + d.k_off + (long long)co * n;
  for (int i = threadIdx.x; 2 * i < n; i += blockDim.x)
    *reinterpret_cast<uint16_t*>(dst + 2 * i) = f8x2_pack(src[2 * i] * inv, src[2 * i + 1] * inv);
}

int launch_pack_weights_fp8(const WeightDesc* d_descs, int nconv, const float* params, uint8_t* w8, float* s_w,
                            cudaStream_t st) {
  MN_LAUNCH(k_pack_weights_fp8, dim3(512, nconv), 256, 0, st, d_descs, params, w8, s_w);
  MN_LAUNCH_CHECK();
  return 0;
}

template int launch_pack_weights<float>(const WeightDesc*, int, const float*, float*, float*, int, int, cudaStream_t);
template int launch_pack_weights<bf16>(const WeightDesc*, int, const float*, bf16*, bf16*, int, int, cudaStream_t);

// ---------------------------------------------------------------------------------
// Strict tensor-core mode (split 16-bit operand planes, common.cuh): weights as hi + lo planes in the
// activations' K order.  A conv with KK filter taps becomes 2*KK "taps" of 2*Ci 16-bit channels:
//   tap  t        holds hi(w) in BOTH plane slots of every 8-channel group,
//   tap  KK + t   holds lo(w) in both,
// so an activation row [xh xl] (the same 8-interleaved K order) against the two taps gives
// xh*wh + xl*wh + xh*wl + xl*wl = (xh + xl) * (wh + wl): every hi/lo cross product, fp32-accumulated by the tensor cores.
//   w_krsc2[co][2*KK][2*Ci]   (fprop, fp16 planes)
//   w_dg2  [ci][2*KK][2*Co]   (dgrad, fp16 planes)
// The stem's patch-matrix row (im2col_k, or 256 for the space-to-depth stem) is treated as ONE tap of that many channels.
// Element offsets into the packed buffers are 4 x the bf16 ones (WeightDesc::k_off * 4).
// ---------------------------------------------------------------------------------
__device__ __forceinline__ void split16(float v, uint16_t& hi, uint16_t& lo) {
  __half h, l; split_f16(v, h, l);
  hi = __half_as_ushort(h); lo = __half_as_ushort(l);
}
// position of (channel c, plane p) inside a pixel's 2*C split channels
__device__ __forceinline__ int split_k(int c, int p) { return ((c >> 3) << 4) + (p << 3) + (c & 7); }

// input: the fp32 K-major matrices launch_pack_weights<float> produces ([rows][KK][C]; rows = Co, C = Ci for
// fprop / wgrad, rows = Ci, C = Co for dgrad); one thread converts 8 channels: coalesced 32-byte loads and stores
__global__ void __launch_bounds__(256)
k_split_weight_rows(const WeightDesc* __restrict__ descs, const float* __restrict__ w_krsc, const float* __restrict__ w_dg,
                    uint16_t* __restrict__ w_krsc2, uint16_t* __restrict__ w_dg2) {
  pdl_prologue();
  const WeightDesc d = descs[blockIdx.y];
  const bool dg = blockIdx.z != 0;
  if (dg && (d.im2col_k > 0 || w_dg2 == nullptr)) return;          // the stem has no dgrad
  const int KK = (d.im2col_k > 0) ? 1 : d.KH * d.KW;
  const int C = (d.im2col_k > 0) ? d.im2col_k : (dg ? d.Co : d.Ci);
  const int rows = dg ? d.Ci : d.Co;
  const float* src = (dg ? w_dg : w_krsc) + d.k_off;
  uint16_t* dst = (dg ? w_dg2 : w_krsc2) + 4 * d.k_off;
  const int cv = C >> 3;
  const long long nvec = (long long)rows * KK * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    const long long rt = i / cv;
    const int t = (int)(rt % KK);
    const long long r = rt / KK;
    Vec8<float> v; v.load(src + i * 8);
    uint4 H, L;
    uint16_t* h = reinterpret_cast<uint16_t*>(&H);
    uint16_t* l = reinterpret_cast<uint16_t*>(&L);
#pragma unroll
    for (int k = 0; k < 8; ++k) split16(v.v[k], h[k], l[k]);
    uint4* o0 = reinterpret_cast<uint4*>(dst + ((r * 2 * KK + t) * 2 * C + c8 * 16));
    uint4* o1 = reinterpret_cast<uint4*>(dst + ((r * 2 * KK + KK + t) * 2 * C + c8 * 16));
    o0[0] = H; o0[1] = H; o1[0] = L; o1[1] = L;
  }
}

// w_krsc_f32 / w_dg_f32: scratch for the fp32 K-major matrices (wk_total floats each)
int launch_pack_weights_split(const WeightDesc* d_descs, int nconv, const float* params, float* w_krsc_f32, float* w_dg_f32,
                              void* w_krsc2, void* w_dg2, int max_elems, cudaStream_t st) {
  MN_TRY(launch_pack_weights<float>(d_descs, nconv, params, w_krsc_f32, w_dg2 != nullptr ? w_dg_f32 : nullptr, max_elems, 0, st));
  dim3 grid(64, nconv, w_dg2 != nullptr ? 2 : 1);
  MN_LAUNCH(k_split_weight_rows, grid, 256, 0, st, d_descs, (const float*)w_krsc_f32, (const float*)w_dg_f32,
            (uint16_t*)w_krsc2, (uint16_t*)w_dg2);
  MN_LAUNCH_CHECK();
  return 0;
}

// one fp32 K-major matrix [rows][KK][C] -> [rows][2*KK][2*C] hi / lo planes (test entry points)
__global__ void __launch_bounds__(256)
k_split_weight_matrix(const float* __restrict__ src, uint16_t* __restrict__ dst, long long rows, int KK, int C) {
  pdl_prologue();
  const int cv = C >> 3;
  const long long nvec = rows * KK * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    const long long rt = i / cv;
    const int t = (int)(rt % KK);
    const long long r = rt / KK;
    Vec8<float> v; v.load(src + i * 8);
    uint4 H, L;
    uint16_t* h = reinterpret_cast<uint16_t*>(&H);
    uint16_t* l = reinterpret_cast<uint16_t*>(&L);
#pragma unroll
    for (int k = 0; k < 8; ++k) split16(v.v[k], h[k], l[k]);
    uint4* o0 = reinterpret_cast<uint4*>(dst + ((r * 2 * KK + t) * 2 * C + c8 * 16));
    uint4* o1 = reinterpret_cast<uint4*>(dst + ((r * 2 * KK + KK + t) * 2 * C + c8 * 16));
    o0[0] = H; o0[1] = H; o1[0] = L; o1[1] = L;
  }
}
int launch_split_weight_matrix(const float* w, void* out, long long rows, int KK, int C, cudaStream_t st) {
  MN_CHECK(C % 8 == 0, "split_weight_matrix: C must be a multiple of 8");
  MN_LAUNCH(k_split_weight_matrix, 256, 256, 0, st, w, (uint16_t*)out, rows, KK, C);
  MN_LAUNCH_CHECK();
  return 0;
}

// fp32 tensor -> split operand planes (test entry points; the training step's element-wise kernels write the
// split form directly)
template <typename TS>
__global__ void __launch_bounds__(256) k_split_tensor(const float* __restrict__ in, TS* __restrict__ out, long long nvec) {
  pdl_prologue();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    Vec8<float> v; v.load(in + i * 8);
    Vec8<TS> o;
#pragma unroll
    for (int k = 0; k < 8; ++k) o.v[k] = v.v[k];
    o.store(out + i * 8);
  }
}
int launch_split_tensor(const float* in, void* out, long long n, cudaStream_t st) {
  MN_CHECK(n % 8 == 0, "split_tensor: element count must be a multiple of 8");
  const long long nvec = n / 8;
  long long grid = (nvec + 255) / 256; if (grid > kNumSMs * 8) grid = kNumSMs * 8; if (grid < 1) grid = 1;
  MN_LAUNCH(k_split_tensor<hsplit>, (int)grid, 256, 0, st, in, (hsplit*)out, nvec);
  MN_LAUNCH_CHECK();
  return 0;
}


__global__ void __launch_bounds__(256)
k_unpack_wgrads(const WeightDesc* __restrict__ descs, const float* __restrict__ dw, float* __restrict__ grads) {
  pdl_prologue();
  extern __shared__ float slab[];
  const WeightDesc d = descs[blockIdx.y];
  if (d.im2col_k > 0) {
    const int co = blockIdx.x;
    if (co >= d.Co) return;
    const float* src = dw + d.k_off + (long long)co * d.im2col_k;
    for (int i = threadIdx.x; i < d.im2col_k; i += blockDim.x) slab[i] = src[i];
    __syncthreads();
    const int n_out = d.Ci_real * 49;
    float* dst = grads + d.p_off + (long long)co * n_out;
    for (int e = threadIdx.x; e < n_out; e += blockDim.x) {
      const int t = e % 49, c = e / 49;
      if (d.s2d) {
        const int kh = t / 7, kw = t - kh * 7;
        const int k = ((kh + 1) >> 1) * 64 + ((kw + 1) >> 1) * 16 + ((((kh + 1) & 1) << 1) | ((kw + 1) & 1)) * 3 + c;
        dst[e] = slab[k];
      } else {
        dst[e] = slab[t * d.Ci_real + c];
      }
    }
    return;
  }
  // every other conv's wgrad engine accumulates straight into grads_flat (KRSC order, mapnet_param_layout == 1)
}

int launch_unpack_wgrads(const WeightDesc* d_descs, int nconv, const float* dw_krsc, float* grads,
                         int max_elems, cudaStream_t st) {
  // only the stem (conv 0, patch-matrix K order) needs a re-layout; nconv is 1
  dim3 grid(64, nconv);
  MN_LAUNCH(k_unpack_wgrads, grid, 256, 256 * sizeof(float), st, d_descs, dw_krsc, grads);
  MN_LAUNCH_CHECK();
  return 0;
}

// One block per output row (b, oh): the 7 input rows x 3 channels it needs are staged in
// shared memory with coalesced loads (3-pixel zero halo left/right, zero rows above/below
// the image), then every thread emits 16-byte slices of the patch matrix (coalesced).
template <typename T>
__global__ void __launch_bounds__(256)
k_stem_im2col(const float* __restrict__ x, T* __restrict__ A, int B, int H, int W, int Ho, int Wo, int Kpad) {
  pdl_prologue();
  extern __shared__ float sx[];          // [3*7][W + 6]
  __shared__ int lut[kStemIm2colK];      // k -> offset of (c,kh,kw) inside sx (-1: zero padding of K)
  const int WP = W + 6;
  const int b = blockIdx.x / Ho, oh = blockIdx.x - b * Ho;
  if (threadIdx.x < kStemIm2colK) {
    const int k = threadIdx.x;
    int off = -1;
    if (k < 147) { const int t = k / 3, c = k - t * 3; const int kh = t / 7, kw = t - kh * 7; off = (c * 7 + kh) * WP + kw; }
    lut[k] = off;
  }
  for (int i = threadIdx.x; i < 21 * WP; i += blockDim.x) {
    const int r = i / WP, col = i - r * WP;
    const int c = r / 7, kh = r - c * 7;
    const int ih = oh * 2 - 3 + kh, iw = col - 3;
    float v = 0.f;
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = __ldg(x + (((long long)b * 3 + c) * H + ih) * W + iw);
    sx[i] = v;
  }
  __syncthreads();
  const int kv = Kpad >> 3;
  T* Arow = A + ((long long)b * Ho + oh) * Wo * Kpad;
  for (int i = threadIdx.x; i < Wo * kv; i += blockDim.x) {
    const int ow = i / kv, k0 = (i - ow * kv) * 8;
    Vec8<T> o;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int off = lut[k0 + j];
      o.v[j] = (off >= 0) ? sx[off + ow * 2] : 0.f;
    }
    o.store(Arow + (long long)i * 8);
  }
}

// Kpad indexes k_stem_im2col's kStemIm2colK-entry k -> offset table.  The 21 staged input rows of W + 6 floats and that
// table share the 48 KB of shared memory a launch gets without opting in, so W <= 570 (a wider frame used to pass a check
// that left the table out and then failed at launch with "invalid argument").
int stem_im2col_check(int W, int Kpad) {
  MN_CHECK(Kpad % 8 == 0 && Kpad >= 147 && Kpad <= kStemIm2colK, "stem_im2col: Kpad %d is not a multiple of 8 in [147, %d]", Kpad,
           kStemIm2colK);
  MN_CHECK(W >= 1 && (size_t)21 * (W + 6) * sizeof(float) + kStemIm2colK * sizeof(int) <= 48 * 1024,
           "stem_im2col: image width %d too large (at most 570)", W);
  return 0;
}

template <typename T>
int launch_stem_im2col(const float* x_nchw, T* A, int B, int H, int W, int Ho, int Wo, int Kpad, cudaStream_t st) {
  MN_TRY(stem_im2col_check(W, Kpad));
  const size_t smem = (size_t)21 * (W + 6) * sizeof(float);
  MN_LAUNCH(k_stem_im2col<T>, B * Ho, 256, smem, st, x_nchw, A, B, H, W, Ho, Wo, Kpad);
  MN_LAUNCH_CHECK();
  return 0;
}
template int launch_stem_im2col<float>(const float*, float*, int, int, int, int, int, int, cudaStream_t);
template int launch_stem_im2col<bf16>(const float*, bf16*, int, int, int, int, int, int, cudaStream_t);
template int launch_stem_im2col<hsplit>(const float*, hsplit*, int, int, int, int, int, int, cudaStream_t);

// ---------------------------------------------------------------------------------
// stem, tensor-core path: space-to-depth instead of a materialised im2col matrix.
// The 7x7/s2/p3 conv on 3 channels is a 4x4/s1 conv on the 2x2 space-to-depth image (12 channels, padded
// to 16; the 7x7 kernel is the 8x8 kernel whose first row and column are zero).  With 16 channels per
// block, the 4 blocks x 16 channels a filter row touches are 64 CONTIGUOUS elements, so the im2col
// operand is an overlapped TMA view of S (pixel stride 16 elements, extent 64): a 4-tap conv with
// "Cin" = 64 that the generic engines run unchanged.  35 MB written and read instead of 403 MB.
// ---------------------------------------------------------------------------------
template <typename TZ>
__global__ void __launch_bounds__(256)
k_stem_s2d(const float* __restrict__ x, TZ* __restrict__ S, int B, int H, int W, int Hs, int Wsp) {
  pdl_prologue();
  const long long n = (long long)B * Hs * Wsp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int bw = (int)(i % Wsp);
    const long long r = i / Wsp;
    const int bh = (int)(r % Hs), b = (int)(r / Hs);
    float v[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) v[k] = 0.f;
#pragma unroll
    for (int pr = 0; pr < 2; ++pr) {
      const int ih = 2 * bh + pr - 4;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int pc = 0; pc < 2; ++pc) {
        const int iw = 2 * bw + pc - 4;
        if (iw < 0 || iw >= W) continue;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[(pr * 2 + pc) * 3 + c] = __ldg(x + (((long long)b * 3 + c) * H + ih) * W + iw);
      }
    }
    Vec8<TZ> o0, o1;
#pragma unroll
    for (int k = 0; k < 8; ++k) { o0.v[k] = v[k]; o1.v[k] = v[8 + k]; }
    o0.store(S + i * 16);
    o1.store(S + i * 16 + 8);
  }
}

int stem_s2d_wsp(int wc) { return (wc + 3 + 3) / 4 * 4; }   // blocks per image row, rows 128 B aligned

// elt_bytes: bytes per stored element (2: bf16; 4: split fp16 planes, where a block of 16 channels is 32 16-bit elements)
void stem_s2d_geometry(int H, int W, int Co, ConvGeom* g, WeightDesc* wd, int elt_bytes) {
  const int hc = (H + 6 - 7) / 2 + 1, wc = (W + 6 - 7) / 2 + 1;
  wd->Co = Co; wd->Ci_real = 3; wd->Ci = 64; wd->KH = 4; wd->KW = 1; wd->im2col_k = 256; wd->s2d = 1;
  g->B = 0; g->Hi = hc + 3; g->Wi = wc; g->Ci = 64; g->Co = Co; g->KH = 4; g->KW = 1; g->stride = 1; g->pad = 0;
  g->Ho = hc; g->Wo = wc;
  g->in_pix_stride = 16 * elt_bytes;
  g->in_row_stride = (long long)stem_s2d_wsp(wc) * 16 * elt_bytes;
  g->in_img_stride = (long long)(hc + 3) * g->in_row_stride;
}

template <typename TZ>
int launch_stem_s2d(const float* x_nchw, TZ* S, int B, int H, int W, int Hs, int Wsp, cudaStream_t st) {
  const long long n = (long long)B * Hs * Wsp;
  long long grid = (n + 255) / 256;
  if (grid > kNumSMs * 8LL) grid = kNumSMs * 8LL;
  MN_LAUNCH(k_stem_s2d<TZ>, (int)grid, 256, 0, st, x_nchw, S, B, H, W, Hs, Wsp);
  MN_LAUNCH_CHECK();
  return 0;
}
template int launch_stem_s2d<bf16>(const float*, bf16*, int, int, int, int, int, cudaStream_t);
template int launch_stem_s2d<hsplit>(const float*, hsplit*, int, int, int, int, int, cudaStream_t);

}  // namespace mapnet
