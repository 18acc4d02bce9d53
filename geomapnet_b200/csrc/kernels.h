// Internal launcher declarations for the MapNet kernels.
#pragma once
#include "common.cuh"
#include "bn_fin.cuh"

struct mapnet_preprocess;

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
  // outputs are fp32.  The planes are fp16.
  int split = 0;
  __host__ __device__ long long M_out() const { return (long long)B * Ho * Wo; }
  __host__ __device__ long long M_in() const { return (long long)B * Hi * Wi; }
  __host__ __device__ int Kdim() const { return KH * KW * Ci; }
};

// ---- bn.cu -------------------------------------------------------------------
// accum / counter: the replicated accumulators of bn_fin.cuh and the counter that elects the finalizing block
template <typename T>
int launch_bn_stats(const T* y, long long M, int C, const BnFin& f, double* accum, unsigned int* counter, cudaStream_t st);
// eval mode: mean / invstd / scale / shift from the running statistics
int launch_bn_eval_scale(int C, const BnFin& f, cudaStream_t st);
// f.mscale != nullptr (and zmask == nullptr): the ReLU mask is recomputed from y
template <typename T, typename TZ>
int launch_bn_bwd_reduce(const T* dout, const TZ* zmask, const T* y, const T* yd, long long M, int C, const BnFin& f,
                         double* accum, unsigned int* counter, cudaStream_t st);
// res: res_mode 1 -> const TZ* (identity branch), 2 -> const T* (downsample branch conv output, BatchNorm bn_ds)
template <typename T, typename TZ>
int launch_bn_apply(const T* y, int res_mode, const void* res, TZ* z, long long M, int C, int relu, const BnDesc& bn,
                    const BnDesc* bn_ds, cudaStream_t st);
// amax == nullptr: the argmax positions are not stored (eval-mode inference: no backward follows)
template <typename T, typename TZ>
int launch_stem_pool(const T* y, TZ* z, uint8_t* amax, int B, int H, int W, int Ho, int Wo, int C, const BnDesc& bn,
                     cudaStream_t st);
template <typename T>
int launch_stem_pool_bwd(const T* dz, const uint8_t* amax, const T* y, const float* scale, const float* shift,
                         T* g, int B, int H, int W, int Ho, int Wo, int C, cudaStream_t st, double* accum = nullptr);
// yd != nullptr: dyd of the downsample BatchNorm too (the second BatchNorm of bn.f);  gscale != nullptr (strict mode):
// dy / dyd are stored multiplied by the device scalar gscale[0] (a power of two)
template <typename T, typename TZ, typename TG>
int launch_bn_bwd_apply(const T* dout, const TZ* zmask, const T* y, TG* dy, const T* yd, TG* dyd, T* gout, long long M,
                        int C, const BnDesc& bn, const float* gscale, cudaStream_t st);

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
// tests and micro-benchmarks only: run a wgrad plan on the per-tap engine (taps 0) or the halo engine with 3 / 9
// filter taps per CTA at N tile bn, keeping the plan's K partition
int tc_plan_force_wgrad(TcConvPlan* p, int taps, int bn);
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
  // eval-mode inference (fprop only, set from EpiAffine by tc_conv_run): f = acc * ascale[c] + ashift[c] in fp32 before
  // the residual; aflags = the conv_tc.cu epilogue bits for ReLU and the hi/lo plane output / residual formats
  const float* ascale;
  const float* ashift;
  int aflags;
};
// Inference epilogue of an fprop launch (a frozen BatchNorm folded in as a per-channel affine map):
//   out = relu?( acc * scale[c] + shift[c] [+ residual] ), rounded once, at the store.
// bf16 mode: residual and output bf16.  Strict mode (split plans): out_split = 1 stores the fp16 hi/lo plane form
// (common.cuh: hsplit) the next conv reads as its operand, 0 stores fp32; res_split = 1 reads the residual in that plane
// form (a block input), 0 as fp32 (a downsample branch's output).  Only the combinations the eval-mode ResNet schedule
// uses are built (tc_affine_supported).
struct EpiAffine {
  const float* scale;
  const float* shift;
  int relu, res_split, out_split;
};
bool tc_affine_supported(bool split, bool residual, const EpiAffine& a);
int tc_conv_run(TcConvPlan* p, const bf16* in0, const bf16* in1, const bf16* residual, void* out, cudaStream_t st,
                double* stats = nullptr, const EpiBwd* bwd = nullptr, const EpiAffine* aff = nullptr);
// ---- fp8 inference fprop (k_f8_conv): e4m3 NHWC input, e4m3 K-major weights [Co][KH][KW][Ci], fp32 accumulation.
//   f = acc * scale[c] + shift[c]  (scale = bn_scale * s_in * s_w[c], folded by the caller: powers of two, exact)
//   (+ residual: e4m3 r * *res_scale when res_f8, else bf16) (ReLU), then
//   out_f8: store e4m3(f * *out_inv) (satfinite), else bf16(f);  amax != nullptr: atomicMax of max |f| (bit pattern of a
//   non-negative float) and no store at all -- the calibration pass of the same conv.
// The scalars are read from device memory, so captured graphs stay valid when calibration rewrites them.
struct EpiF8 {
  const float* scale;
  const float* shift;
  const float* res_scale;
  const float* out_inv;
  unsigned int* amax;
  int relu, res_f8, out_f8;
};
// fprop plan over e4m3 operands (1x1 / 3x3, Ci = 64 or a multiple of 128); wmat = e4m3 [Co][KH][KW][Ci]
int tc_plan_create_f8(TcConvPlan** out, const ConvGeom& g, const uint8_t* wmat);
int tc_conv_run_f8(TcConvPlan* p, const uint8_t* in, const void* residual, void* out, const EpiF8& e, cudaStream_t st);
// finalize of backward reductions accumulated in `accum` (the stem's pool backward in the CUDA-core modes): d gamma,
// d beta and the dy = A*g + B*y + C coefficients
int launch_bn_bwd_finalize_accum(long long M, int C, const BnFin& f, double* accum, cudaStream_t st);

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
// strict tensor-core mode: fp16 hi / lo operand planes of the weights (layout.cu)
int launch_pack_weights_split(const WeightDesc* d_descs, int nconv, const float* params, float* w_krsc_f32, float* w_dg_f32,
                              void* w_krsc2, void* w_dg2, int max_elems, cudaStream_t st);
int launch_split_tensor(const float* in, void* out, long long n, cudaStream_t st);
// fp8 inference: per output channel co of every conv, s_w = 2^ceil(log2(amax_co / 448)) (1 when amax_co = 0) into
// s_w[i * 512 + co] and e4m3(w / s_w) into w8 + k_off (the descriptors' non-stem convs; K-major params only)
int launch_pack_weights_fp8(const WeightDesc* d_descs, int nconv, const float* params, uint8_t* w8, float* s_w,
                            cudaStream_t st);
int launch_split_weight_matrix(const float* w, void* out, long long rows, int KK, int C, cudaStream_t st);
int launch_unpack_wgrads(const WeightDesc* d_descs, int nconv, const float* dw_krsc, float* grads,
                         int max_elems, cudaStream_t st);
// space-to-depth image of the stem input: S[b][bh][bw][16] bf16, channel (pr*2+pc)*3+c of block (bh,bw)
// = x[b][c][2*bh+pr-4][2*bw+pc-4] (0 outside the image, channels 12..15 = 0), row pitch Wsp blocks
template <typename TZ>
int launch_stem_s2d(const float* x_nchw, TZ* S, int B, int H, int W, int Hs, int Wsp, cudaStream_t st);
// geometry of the stem as the engines see it on that image (B left 0): 4 taps x 64 elements, overlapped view
int stem_s2d_wsp(int wc);
void stem_s2d_geometry(int H, int W, int Co, ConvGeom* g, WeightDesc* wd, int elt_bytes = 2);
// the im2col stem's patch-matrix row: 7*7*3 = 147 padded to 192 (a multiple of the tensor-core K block)
static constexpr int kStemIm2colK = 192;
// host-side limits of launch_stem_im2col (it calls this first): Kpad a multiple of 8 in [147, kStemIm2colK], W <= 570
int stem_im2col_check(int W, int Kpad);
template <typename T>
int launch_stem_im2col(const float* x_nchw, T* A, int B, int H, int W, int Ho, int Wo, int Kpad, cudaStream_t st);

// ---- head.cu -------------------------------------------------------------------
// scale (device scalar, may be null): multiplies the mean -- the power-of-two scale of an e4m3 tensor
template <typename T>
int launch_gap(const T* z, float* feat, int B, int HW, int C, cudaStream_t st, const float* scale = nullptr);
template <typename T>
int launch_gap_bwd(const float* dfeat, T* dz, int B, int HW, int C, cudaStream_t st);
// dst[i] += part[i] + part[n + i] + ... + part[(splits - 1) * n + i], summed in that order (n % 4 == 0): the
// deterministic second half of a split-K reduction whose splits STORE their partial results
int launch_split_reduce(const float* part, int splits, long long n, float* dst, cudaStream_t st);
int launch_small_gemm(int epi, const float* A, long long sam, long long sak, const float* Bm, long long sbn,
                      long long sbk, float* C, int ldc, int M, int N, int K, const float* bias, float* aux,
                      const float* mask, cudaStream_t st);
// host-only: the split-K plan launch_small_gemm runs for an [M,K] x [N,K]^T product -- the number of K splits (grid.z),
// and through *kchunk the length of every split but the last (K when there is one split)
int small_gemm_split_plan(int epi, int M, int N, int K, int* kchunk);
// Monte-Carlo dropout head (k_head_draws + k_head_stats): S draws of the head for every frame of fcpre [B,F], bit for
// bit the outputs of S consecutive run_head calls from dropout step c (ctr_dev != null: c = *ctr_dev, advanced by S;
// else c = step); samples [B,S,6] (may be null), mean [B,6] and cov [B,6,6] in float64.  stride = max_B * F.
constexpr int kMaxSampleDraws = 1024;
size_t head_sample_smem(int B, int F, int S);     // shared memory of k_head_draws (host-only; <= 48 KB to launch)
int launch_head_sample(const float* fcpre, int B, int F, const float* wx, const float* bx, const float* wq,
                       const float* bq, int S, float p, unsigned long long seed, unsigned long long step,
                       unsigned long long* ctr_dev, unsigned long long stride, float* samples, double* mean,
                       double* cov, cudaStream_t st);
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
// The head's launch sequences, shared by the training step (Net::forward_t / backward_t), the inference engine's
// run_head and mapnet_test_head.  Parameters fc [F][512] + [F], fc_xyz / fc_wpqr [3][F] + [3]; gradients in the same
// shapes, a null gradient pointer is a frozen parameter (nothing computed for it).
struct HeadParams { const float *fc_w, *fc_b, *xyz_w, *xyz_b, *wpqr_w, *wpqr_b; };
struct HeadGrads { float *fc_w, *fc_b, *xyz_w, *xyz_b, *wpqr_w, *wpqr_b; };
// droprate > 0: the dropout mask [B][F] from (seed, flat offset step * stride), or from the device counter *ctr when
// step == ~0 (ctr advanced by one); hdrop = relu(fcpre) * mask, fcpre = feat @ fc_w^T + fc_b; pred [B][6]
int head_forward(const HeadParams& hp, const float* feat, int B, int F, float droprate, unsigned long long seed,
                 unsigned long long step, unsigned long long* ctr, unsigned long long stride, float* mask, float* fcpre,
                 float* hdrop, float* pred, cudaStream_t st);
// dpred [B][6] -> the two NaN-filtered copies dpredw / dpredh, gscale != null: this step's gradient scale of dpredh
// (strict mode), the weight / bias gradients of hg, dh [B][F] (when fc trains or dfeat is wanted) and dfeat [B][512]
// (dfeat != null: the trunk needs its gradient).  mask: the forward's dropout mask, or null.
int head_backward(const HeadParams& hp, const HeadGrads& hg, const float* dpred, int filter_nans, const float* feat,
                  const float* mask, const float* fcpre, const float* hdrop, int B, int F, float* dpredw, float* dpredh,
                  float* gscale, float* dh, float* dfeat, cudaStream_t st);

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

// ---- pgo.cu: pose-graph optimisation of n_windows windows of N poses (k_pgo) --------------------------------------
// w4 = (1/sqrt(sax), 1/sqrt(saq), 1/sqrt(srx), 1/sqrt(srq)) from pgo_weights; n_win_dev (may be null): a device count
// of windows, the blocks beyond it exit; win_fail (may be null): per window 1 / 0, whether its normal matrix was not
// positive definite.  pgo_prepare sets k_pgo's shared-memory limit once (not graph-capturable).  robust_c > 0: the
// absolute factors take the Cauchy loss of scale robust_c (whitened units, iteratively reweighted; k_pgo<true>), and
// w_out (may be null) [n_windows][N] gets each slot's weight at the returned state; 0: the plain k_pgo<false>.
int pgo_prepare();
void pgo_weights(double sax, double saq, double srx, double srq, double w4[4]);
int launch_pgo(const double* poses, const double* vos, double* out, int n_windows, int N, int fc, const double w4[4],
               int n_iters, int exact, int* status, const int* n_win_dev, cudaStream_t st, int* win_fail = nullptr,
               double robust_c = 0.0, double* w_out = nullptr);
// k_pgo_cov: sig7 [n_windows][N][7][7] covariances of the absolute factors, relative weights w_rx = 1/sqrt(srx) and
// w_rq = 1/sqrt(srq), the exact Gauss-Newton step; out [n_windows][N][7] and the posterior cov [n_windows][N][6][6]
// in (t, log q).  n_win_dev, win_fail, status, robust_c and w_out as launch_pgo's (the posterior is taken with the
// weights at the returned state).  pgo_cov_prepare sets its shared-memory limit once.
int pgo_cov_prepare();
int launch_pgo_cov(const double* poses, const double* sig7, const double* vos, double* out, double* cov, int n_windows,
                   int N, int fc, double w_rx, double w_rq, int n_iters, int* status, const int* n_win_dev,
                   int* win_fail, cudaStream_t st, double robust_c = 0.0, double* w_out = nullptr);

// input pipeline internals shared by preprocess.cu and the frame cache (loader.cu)
struct JitterParams;
int preprocess_resize_u8(struct ::mapnet_preprocess* h, const uint8_t* img, int n, uint8_t* out_u8, cudaStream_t st);
int launch_jitter_luma_sum(const uint8_t* u8, const int* frame_index, const JitterParams* jp, unsigned int* sums,
                           long long npix, int n, int gx, cudaStream_t st);
// a plan's output size (Resize's) and the most frames one call takes
int preprocess_geometry(const struct ::mapnet_preprocess* h, int* Hout, int* Wout, int* max_images);
// the inference engine's input from camera frames: n uint8 frames [Hin][Win][3] (device memory, n <= max_images) through
// Resize + ToTensor + Normalize (mean3 / std3: host) straight into the space-to-depth stem operand S [n][Hs][Wsp][16]
// (launch_stem_s2d's layout and values, bit for bit; Hs, Wsp of the plan's output size).  Two launches.
template <typename TZ>
int preprocess_stem_s2d(struct ::mapnet_preprocess* h, const uint8_t* img, int n, const float* mean3, const float* std3,
                        TZ* S, int Hs, int Wsp, cudaStream_t st);

}  // namespace mapnet
