// Internal launcher declarations for the MapNet kernels.
#pragma once
#include "common.cuh"
#include "bn_fin.cuh"

namespace mapnet {

// Geometry of one convolution (NHWC activations, weights [Co][KH][KW][Ci] "KRSC").
struct ConvGeom {
  int B, Hi, Wi, Ci, Ho, Wo, Co, KH, KW, stride, pad;
  // tensor-core path only: byte strides of the INPUT view when it is not a dense [B,Hi,Wi,Ci] tensor
  // (0 = dense).  The stem uses an overlapped view of its space-to-depth image: a "pixel" is 64
  // consecutive elements and consecutive pixels start 16 elements apart (layout.cu, k_stem_s2d).
  long long in_pix_stride = 0, in_row_stride = 0, in_img_stride = 0;
  // tensor-core path, strict mode: activations / gradients are split 16-bit operand planes (common.cuh: hsplit,
  // 2*C 16-bit "channels" per pixel), the weight matrices hold hi and lo planes as 2*KH*KW taps (layout.cu),
  // outputs are fp32.  fmt_z / fmt_g: element format of the forward / backward operands (0 = fp16, 1 = bf16).
  int split = 0, fmt_z = 1, fmt_g = 1;
  __host__ __device__ long long M_out() const { return (long long)B * Ho * Wo; }
  __host__ __device__ long long M_in() const { return (long long)B * Hi * Wi; }
  __host__ __device__ int Kdim() const { return KH * KW * Ci; }
};

// ---- bn.cu -------------------------------------------------------------------
template <typename T>
int launch_bn_stats(const T* y, long long M, int C, const float* gamma, const float* beta, float* run_mean,
                    float* run_var, float* mean_out, float* invstd_out, float* scale, float* shift, int training,
                    double* accum, unsigned int* counter, cudaStream_t st);
template <typename T, typename TZ>
int launch_bn_bwd_reduce(const T* dout, const TZ* zmask, const T* y, const T* yd, long long M, int C,
                         const float* gamma, const float* mean, const float* invstd, float* dgamma, float* dbeta,
                         float* coef, const float* gamma2, const float* mean2, const float* invstd2,
                         float* dgamma2, float* dbeta2, float* coef2, double* accum, unsigned int* counter,
                         cudaStream_t st, const float* mscale = nullptr, const float* mshift = nullptr);
// res: res_mode 1 -> const TZ* (identity branch), 2 -> const T* (downsample branch conv output)
template <typename T, typename TZ>
int launch_bn_apply(const T* y, const float* scale, const float* shift, int res_mode, const void* res,
                    const float* scale2, const float* shift2, TZ* z, long long M, int C, int relu, cudaStream_t st,
                    const BnLazy* lazy = nullptr, const BnLazy* lazy2 = nullptr);
// lazy (/ lazy2 for the downsample BN): the kernel finalizes the batch statistics itself (bn_fin.cuh, BnLazy)
template <typename T, typename TZ>
int launch_stem_pool(const T* y, const float* scale, const float* shift, TZ* z, uint8_t* amax, int B, int H,
                     int W, int Ho, int Wo, int C, cudaStream_t st, const BnLazy* lazy = nullptr);
template <typename T>
int launch_stem_pool_bwd(const T* dz, const uint8_t* amax, const T* y, const float* scale, const float* shift,
                         T* g, int B, int H, int W, int Ho, int Wo, int C, cudaStream_t st, double* accum = nullptr);
template <typename T, typename TZ, typename TG>
int launch_bn_bwd_apply(const T* dout, const TZ* zmask, const T* y, const float* coef, TG* dy, const T* yd,
                        const float* coefd, TG* dyd, T* gout, long long M, int C, cudaStream_t st,
                        const float* mscale = nullptr, const float* mshift = nullptr, const float* gscale = nullptr,
                        const BnLazy* lazy = nullptr);
// gscale != nullptr (strict mode): dy / dyd are stored multiplied by the device scalar gscale[0] (a power of two)
// lazy: coef / coefd are not read; the kernel derives them from the backward sums (3 per channel when yd != nullptr)

// ---- conv_simt.cu: fp32 CUDA-core implicit GEMM (strict-parity path) -----------
template <typename T>
int launch_conv_simt_fprop(const ConvGeom& g, const T* x, const float* w_krsc, const T* residual, T* y, cudaStream_t st);
template <typename T>
int launch_conv_simt_dgrad(const ConvGeom& g, const T* dy, const float* w_dg /*[Ci][KH][KW][Co]*/, const T* residual, T* dx, cudaStream_t st);
template <typename T>
int launch_conv_simt_wgrad(const ConvGeom& g, const T* x, const T* dy, float* dw_krsc /*zeroed, accumulated*/, cudaStream_t st);

// ---- conv_tc.cu: wgmma / TMA implicit GEMM (bf16 tensor-core path) ---------------
struct TcConvPlan;   // opaque: tile shapes, tap tables and cached TMA tensor maps of one conv
// kind 0 fprop (wmat = [Co][KH][KW][Ci]), 1 dgrad (wmat = [Ci][KH][KW][Co]), 2 wgrad (wmat unused)
int tc_plan_create(TcConvPlan** out, const ConvGeom& g, int kind, const bf16* wmat);
void tc_plan_destroy(TcConvPlan* p);
// dgrad plans of a 3x3 / stride-2 conv only: fold the dgrad of the parallel 1x1 / stride-2 shortcut conv (same
// input and output shapes; wmat2 = [Ci][Co]) into the same launch -- tc_conv_run then takes the shortcut's
// incoming gradient as in1 and writes d(input) of BOTH convs
int tc_plan_add_shortcut(TcConvPlan* p, const bf16* wmat2);
int tc_plan_launches(const TcConvPlan* p);
// dgrad / wgrad plans: multiply the accumulators by the device scalar *inv_scale before they are added to the residual /
// the wgrad buffer (strict mode: the gradient operand planes carry a per-step power-of-two scale)
void tc_plan_set_out_scale(TcConvPlan* p, const float* inv_scale);
int tc_plan_describe(const TcConvPlan* p, char* buf, int cap);      // JSON, host-only (CPU tests of the plan arithmetic)
// fprop: in0 = x, out = y (bf16);  dgrad: in0 = dy [, in1 = the folded shortcut's dy], out = dx (bf16);
// wgrad: in0 = x, in1 = dy, out = fp32 dW (accumulated)
// stats != nullptr (fprop, no residual): per-channel sum / sum of squares of the stored output are
// accumulated into the replica accumulators for the fused BatchNorm statistics
// bwd != nullptr (dgrad only, with stats): the stored gradient is gated by the consumer BN's ReLU
// (zmask > 0, or mscale*y + mshift > 0) and (sum g, sum g*y [, sum g*yd]) are accumulated: the
// reductions of that BN's backward, fused into the producer of its incoming gradient
struct EpiBwd {
  const bf16* y;        // consumer BN input (forward conv output), shaped like the dgrad output
  const bf16* zmask;    // post-ReLU tensor whose sign gates the gradient, or null
  const bf16* yd;       // downsample-branch BN input (third sum), or null
  const float* mscale;  // gate recomputed from y when zmask is null
  const float* mshift;
  const float* oscale;  // strict mode (fp32 output): device scalar multiplied into the accumulators, or null (set by the plan)
};
// fin != nullptr (with stats): the last CTA to flush its sums also finalizes them (bn_fin.cuh) -- forward:
// mean / invstd / scale / shift / running statistics; backward: d gamma, d beta, dy coefficients
struct EpiFin;
int tc_conv_run(TcConvPlan* p, const bf16* in0, const bf16* in1, const bf16* residual, void* out, cudaStream_t st,
                double* stats = nullptr, const EpiBwd* bwd = nullptr, const EpiFin* fin = nullptr);
// finalize of the dgrad-fused reductions: d gamma, d beta and the dy = A*g + B*y + C coefficients
int launch_bn_bwd_finalize_accum(long long M, int C, const float* gamma, const float* mean, const float* invstd,
                                 float* dgamma, float* dbeta, float* coef, const float* gamma2, const float* mean2,
                                 const float* invstd2, float* dgamma2, float* dbeta2, float* coef2, double* accum,
                                 cudaStream_t st);
int launch_bn_finalize_accum(long long M, int C, const float* gamma, const float* beta, float* run_mean,
                             float* run_var, float* mean_out, float* invstd_out, float* scale, float* shift,
                             double* accum, cudaStream_t st);

// true when the driver accepts a tiled tensor map whose second dimension's stride is smaller than the
// first dimension's extent (overlapping windows) -- what the space-to-depth stem view needs
bool tc_overlapped_view_supported();

// ---- layout.cu -----------------------------------------------------------------
struct WeightDesc {   // one conv's weight in the flat parameter buffer and in the packed matrices
  long long p_off;    // float offset in params_flat ([Co,Ci_real,KH,KW] torch layout)
  long long k_off;    // element offset in the KRSC / dgrad packed buffers
  int Co, Ci, Ci_real, KH, KW;   // Ci = packed (padded) channels per tap
  int im2col_k;       // >0: stem conv stored as [Co][im2col_k] with k=(kh*KW+kw)*Ci_real+ci
  int s2d;            // stem, space-to-depth K order: k = kh2*64 + kw2*16 + (pr*2+pc)*3 + ci, (kh,kw) = (2*kh2+pr-1, 2*kw2+pc-1)
};
template <typename TW>
int launch_pack_weights(const WeightDesc* d_descs, int nconv, const float* params, TW* w_krsc, TW* w_dg,
                        int max_elems, int round_bf16, cudaStream_t st);
// strict tensor-core mode: hi / lo operand planes of the weights (layout.cu); fmt 0 = fp16, 1 = bf16
int launch_pack_weights_split(const WeightDesc* d_descs, int nconv, const float* params, float* w_krsc_f32, float* w_dg_f32,
                              void* w_krsc2, void* w_dg2, int max_elems, int fmt_f, int fmt_g, cudaStream_t st);
int launch_split_tensor(const float* in, void* out, long long n, int fmt, cudaStream_t st);
int launch_split_weight_matrix(const float* w, void* out, long long rows, int KK, int C, int fmt, cudaStream_t st);
int launch_unpack_wgrads(const WeightDesc* d_descs, int nconv, const float* dw_krsc, float* grads,
                         int max_elems, cudaStream_t st);
// space-to-depth image of the stem input: S[b][bh][bw][16] bf16, channel (pr*2+pc)*3+c of block (bh,bw)
// = x[b][c][2*bh+pr-4][2*bw+pc-4] (0 outside the image, channels 12..15 = 0), row pitch Wsp blocks
template <typename TZ>
int launch_stem_s2d(const float* x_nchw, TZ* S, int B, int H, int W, int Hs, int Wsp, cudaStream_t st);
// geometry of the stem as the engines see it on that image (B left 0): 4 taps x 64 elements, overlapped view
int stem_s2d_wsp(int wc);
void stem_s2d_geometry(int H, int W, int Co, ConvGeom* g, WeightDesc* wd, int elt_bytes = 2);
template <typename T>
int launch_stem_im2col(const float* x_nchw, T* A, int B, int H, int W, int Ho, int Wo, int Kpad, cudaStream_t st);

// ---- head.cu -------------------------------------------------------------------
template <typename T>
int launch_gap(const T* z, float* feat, int B, int HW, int C, cudaStream_t st);
template <typename T>
int launch_gap_bwd(const float* dfeat, T* dz, int B, int HW, int C, cudaStream_t st);
// dst[i] += part[i] + part[n + i] + ... + part[(splits - 1) * n + i], summed in that order (n % 4 == 0): the
// deterministic second half of a split-K reduction whose splits STORE their partial results
int launch_split_reduce(const float* part, int splits, long long n, float* dst, cudaStream_t st);
int launch_small_gemm(int epi, const float* A, long long sam, long long sak, const float* Bm, long long sbn,
                      long long sbk, float* C, int ldc, int M, int N, int K, const float* bias, float* aux,
                      const float* mask, cudaStream_t st);
int launch_colsum(const float* A, int lda, int M, int N, float* out, cudaStream_t st);
// two NaN-filtered copies of d pred [B,6] (models/posenet.py:28-34 hook semantics, head.cu): out_w for the head's weight /
// bias gradients, out_h for the gradient into the trunk; filter == 0: plain copies
int launch_dpred_filter(const float* in, float* out_w, float* out_h, int B, int filter, cudaStream_t st);
// scale[0] = S = 2^(8 - ceil(log2 max|g|)) (1 when max|g| is 0 or not finite), scale[1] = 1/S
int launch_grad_scale(const float* g, int n, float* scale2, cudaStream_t st);
int launch_dropout_mask(float* mask, long long n, float p, unsigned long long seed, unsigned long long offset,
                        unsigned long long* ctr_dev, unsigned long long ctr_stride, cudaStream_t st);
int launch_head_dh(const float* dpred, const float* wx, const float* wq, const float* mask, const float* fcpre,
                   float* dh, int B, int F, cudaStream_t st);

// ---- loss.cu -------------------------------------------------------------------
int launch_loss(int mode, const float* pred, const float* targ, int N, int Tp, int Tt, const float* s4,
                float* loss, float* dpred, float* ds4, cudaStream_t st);

// ---- adam.cu -------------------------------------------------------------------
int launch_sqnorm(const float* g, long long n, float* partials, float* out_sq, cudaStream_t st);
int launch_adam(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                float eps, float wd, float bc1, float bc2, float gscale, const float* sqnorm_or_null,
                float max_norm, int* step_dev, cudaStream_t st);
int launch_inc_i32(int* c, cudaStream_t st);    // *c += 1 on the device (optimizer step counters)

// Factor every optimizer kernel applies to the raw gradient: gscale (1/world after a sum-allreduce), times
// clip_grad_norm_'s coefficient max_norm / (total_norm + 1e-6) clamped to 1 when sqnorm (the squared norm of the
// unscaled gradient, launch_sqnorm) is given.
__device__ __forceinline__ float grad_coef(float gscale, const float* __restrict__ sqnorm, float max_norm) {
  float coef = gscale;
  if (sqnorm != nullptr) {
    const float total = sqrtf(sqnorm[0]) * gscale;
    float c = max_norm / (total + 1e-6f);
    if (c > 1.0f) c = 1.0f;
    coef *= c;
  }
  return coef;
}

// ---- optim.cu ------------------------------------------------------------------
// SGD / RMSprop on flat buffers; lr_dev is a device float (CUDA-graph capturable rate).  NULL state buffers select
// the variant: no momentum buffer <=> momentum 0, grad_avg <=> centered RMSprop.  step_dev (SGD with momentum:
// required) is incremented first; SGD's step 1 initialises the momentum buffer with the update direction.
int launch_sgd(float* p, const float* g, float* buf, long long n, const float* lr_dev, float momentum,
               double dampening, float wd, int nesterov, int* step_dev, float gscale, const float* sqnorm_or_null,
               float max_norm, cudaStream_t st);
int launch_rmsprop(float* p, const float* g, float* square_avg, float* grad_avg, float* buf, long long n,
                   const float* lr_dev, double alpha, float eps, float wd, float momentum, int* step_dev, float gscale,
                   const float* sqnorm_or_null, float max_norm, cudaStream_t st);

}  // namespace mapnet
