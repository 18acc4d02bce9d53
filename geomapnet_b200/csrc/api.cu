// extern "C" entry points declared in include/mapnet_b200.h.
#include <math.h>

#include <vector>

#include "../../include/mapnet_b200.h"
#include "net.h"
#include "infer.h"

using namespace mapnet;

struct mapnet_trunk { Net net; };
struct mapnet_infer { InferNet net; };

extern "C" {

const char* mapnet_last_error(void) { return get_last_error(); }
int mapnet_abi_version(void) { return 2; }

static int require_device() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    set_last_error("no CUDA device available (%s): this library has no CPU fallback",
                   e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    return 10;
  }
  return 0;
}

int mapnet_trunk_create(mapnet_trunk_t** out, int max_B, int H, int W, int feat_dim, int precision) {
  MN_CHECK(out != nullptr, "trunk_create: null out pointer");
  *out = nullptr;
  if (max_B > 0) MN_TRY(require_device());
  mapnet_trunk* h = new mapnet_trunk();
  int r = h->net.init(max_B, H, W, feat_dim, precision);
  if (r != 0) { h->net.destroy(); delete h; return r; }
  *out = h;
  return 0;
}

// mapnet_trunk_create with Net::init's im2col_stem: 1 gives the tensor-core modes the stem they fall back to when the
// driver rejects overlapped tensor maps (the CUDA-core modes always run it)
int mapnet_test_trunk_create(mapnet_trunk_t** out, int max_B, int H, int W, int feat_dim, int precision, int im2col_stem) {
  MN_CHECK(out != nullptr, "test_trunk_create: null out pointer");
  *out = nullptr;
  MN_CHECK(im2col_stem == 0 || im2col_stem == 1, "test_trunk_create: im2col_stem %d is not 0 or 1", im2col_stem);
  MN_CHECK(precision >= PREC_FP32 && precision <= PREC_TC_SPLIT, "test_trunk_create: precision %d is not a training "
           "precision", precision);
  MN_CHECK(max_B >= 0 && H >= 32 && W >= 32 && feat_dim >= 8 && feat_dim % 4 == 0, "test_trunk_create: bad shape "
           "(max_B %d, %dx%d, feat_dim %d)", max_B, H, W, feat_dim);
  if (max_B > 0) MN_TRY(require_device());
  mapnet_trunk* h = new mapnet_trunk();
  int r = h->net.init(max_B, H, W, feat_dim, precision, im2col_stem);
  if (r != 0) { h->net.destroy(); delete h; return r; }
  *out = h;
  return 0;
}

int mapnet_trunk_destroy(mapnet_trunk_t* h) {
  if (h == nullptr) return 0;
  h->net.destroy();
  delete h;
  return 0;
}

int mapnet_param_count(mapnet_trunk_t* h) { return h ? (int)h->net.table.size() : -1; }

int mapnet_param_info(mapnet_trunk_t* h, int i, char* host_name, int name_cap, int* host_kind, int* host_ndim,
                      int64_t* host_shape4, int64_t* host_offset) {
  MN_CHECK(h != nullptr, "param_info: null handle");
  MN_CHECK(i >= 0 && i < (int)h->net.table.size(), "param_info: index %d out of range", i);
  const ParamEntry& e = h->net.table[i];
  if (host_name && name_cap > 0) { strncpy(host_name, e.name.c_str(), name_cap - 1); host_name[name_cap - 1] = 0; }
  if (host_kind) *host_kind = e.kind;
  if (host_ndim) *host_ndim = e.ndim;
  if (host_shape4) for (int k = 0; k < 4; ++k) host_shape4[k] = e.shape[k];
  if (host_offset) *host_offset = e.offset;
  return 0;
}

int mapnet_param_layout(mapnet_trunk_t* h, int i) {
  if (h == nullptr || i < 0 || i >= (int)h->net.table.size()) return -1;
  return h->net.table[i].layout;
}

int64_t mapnet_params_numel(mapnet_trunk_t* h) { return h ? h->net.n_params : -1; }
int64_t mapnet_bufs_numel(mapnet_trunk_t* h) { return h ? h->net.n_bufs : -1; }

int mapnet_forward(mapnet_trunk_t* h, const float* x, const float* params_flat, float* bufs_flat, int B,
                   int training, float droprate, uint64_t seed, uint64_t step, float* pred, void* stream) {
  MN_CHECK(h != nullptr, "forward: null handle");
  return h->net.forward(x, params_flat, bufs_flat, B, training, droprate, seed, step, pred, (cudaStream_t)stream);
}

int mapnet_backward(mapnet_trunk_t* h, const float* dpred, const float* params_flat, float* grads_flat,
                    int filter_nans, void* stream) {
  MN_CHECK(h != nullptr, "backward: null handle");
  return h->net.backward(dpred, params_flat, grads_flat, filter_nans, -1, (cudaStream_t)stream);
}

int mapnet_backward_part(mapnet_trunk_t* h, int part, const float* dpred, const float* params_flat, float* grads_flat,
                         int filter_nans, void* stream) {
  MN_CHECK(h != nullptr, "backward_part: null handle");
  MN_CHECK(part >= 0 && part <= 2, "backward_part: part %d outside [0, 2]", part);
  return h->net.backward(dpred, params_flat, grads_flat, filter_nans, part, (cudaStream_t)stream);
}

int mapnet_trunk_set_trainable(mapnet_trunk_t* h, const uint8_t* host_mask, int n) {
  MN_CHECK(h != nullptr, "set_trainable: null handle");
  return h->net.set_trainable(host_mask, n);
}

int mapnet_grad_part_range(mapnet_trunk_t* h, int part, int64_t* host_lo, int64_t* host_hi) {
  MN_CHECK(h != nullptr && host_lo && host_hi && part >= 0 && part <= 2, "grad_part_range: bad argument");
  long long lo = 0, hi = 0;
  h->net.part_range(part, &lo, &hi);
  *host_lo = lo; *host_hi = hi;
  return 0;
}

int mapnet_loss_fwd_bwd(int mode, const float* pred, const float* targ, int N, int T_pred, int T_targ,
                        const float* s4, float* loss, float* dpred, float* ds4, void* stream) {
  MN_CHECK(pred && targ && s4 && loss && dpred && ds4, "loss_fwd_bwd: null pointer argument");
  return launch_loss(mode, pred, targ, N, T_pred, T_targ, s4, loss, dpred, ds4, (cudaStream_t)stream);
}

int mapnet_sqnorm(const float* g, int64_t n, float* scratch1024, float* out_sq, void* stream) {
  MN_CHECK(g && scratch1024 && out_sq && n > 0, "sqnorm: bad argument");
  return launch_sqnorm(g, n, scratch1024, out_sq, (cudaStream_t)stream);
}

int mapnet_adam_step(float* p, const float* g, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                     float beta1, float beta2, float eps, float weight_decay, int64_t step, float grad_scale,
                     const float* sqnorm, float max_norm, void* stream) {
  MN_CHECK(p && g && exp_avg && exp_avg_sq && n > 0, "adam_step: bad argument");
  MN_CHECK(step >= 1, "adam_step: step counts from 1 (got %lld)", (long long)step);
  const float bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  const float bc2 = (float)(1.0 - pow((double)beta2, (double)step));
  return launch_adam(p, g, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_scale,
                     sqnorm, max_norm, nullptr, (cudaStream_t)stream);
}

int mapnet_adam_step_dev(float* p, const float* g, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                         float beta1, float beta2, float eps, float weight_decay, int32_t* step_counter,
                         float grad_scale, const float* sqnorm, float max_norm, void* stream) {
  MN_CHECK(p && g && exp_avg && exp_avg_sq && step_counter && n > 0, "adam_step_dev: bad argument");
  return launch_adam(p, g, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, 1.f, 1.f, grad_scale,
                     sqnorm, max_norm, step_counter, (cudaStream_t)stream);
}

int mapnet_sgd_step_dev(float* p, const float* g, float* momentum_buf, int64_t n, const float* lr_dev, float momentum,
                        double dampening, float weight_decay, int nesterov, int32_t* step_counter, float grad_scale,
                        const float* sqnorm, float max_norm, void* stream) {
  MN_CHECK(p && g && lr_dev && n > 0, "sgd_step_dev: bad argument");
  MN_CHECK((momentum_buf != nullptr) == (momentum != 0.f), "sgd_step_dev: momentum_buf must be given exactly when "
           "momentum != 0 (momentum %g)", (double)momentum);
  MN_CHECK(momentum_buf == nullptr || step_counter != nullptr, "sgd_step_dev: momentum needs the step counter");
  MN_CHECK(!nesterov || (momentum > 0.f && dampening == 0.0), "sgd_step_dev: nesterov needs momentum > 0 and "
           "zero dampening");
  return launch_sgd(p, g, momentum_buf, n, lr_dev, momentum, dampening, weight_decay, nesterov, step_counter,
                    grad_scale, sqnorm, max_norm, (cudaStream_t)stream);
}

int mapnet_rmsprop_step_dev(float* p, const float* g, float* square_avg, float* grad_avg, float* momentum_buf,
                            int64_t n, const float* lr_dev, double alpha, float eps, float weight_decay, float momentum,
                            int32_t* step_counter, float grad_scale, const float* sqnorm, float max_norm, void* stream) {
  MN_CHECK(p && g && square_avg && lr_dev && n > 0, "rmsprop_step_dev: bad argument");
  MN_CHECK((momentum_buf != nullptr) == (momentum > 0.f), "rmsprop_step_dev: momentum_buf must be given exactly when "
           "momentum > 0 (momentum %g)", (double)momentum);
  return launch_rmsprop(p, g, square_avg, grad_avg, momentum_buf, n, lr_dev, alpha, eps, weight_decay, momentum,
                        step_counter, grad_scale, sqnorm, max_norm, (cudaStream_t)stream);
}

unsigned long long mapnet_launch_count(void) { return g_launch_count; }

int mapnet_profile(mapnet_trunk_t* h, int enable) {
  MN_CHECK(h != nullptr, "profile: null handle");
  h->net.profile_on = enable ? 1 : 0;
  if (enable) MN_TRY(h->net.prof_reserve(2048));      // no event creation inside the profiled steps
  return 0;
}

int mapnet_profile_read(mapnet_trunk_t* h, double* host_ms3, double* host_flops3, int* host_launches3) {
  MN_CHECK(h != nullptr && host_ms3 && host_flops3 && host_launches3, "profile_read: bad argument");
  return h->net.prof_read(host_ms3, host_flops3, host_launches3);
}

int mapnet_test_conv(int precision, int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride,
                     const void* in0, const void* in1, const void* wmat, void* out, void* stream) {
  MN_TRY(require_device());
  ConvGeom g;
  g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
  g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == PREC_FP32) {
    if (kind == 0) return launch_conv_simt_fprop<float>(g, (const float*)in0, (const float*)wmat, nullptr, (float*)out, st);
    if (kind == 1) return launch_conv_simt_dgrad<float>(g, (const float*)in0, (const float*)wmat, nullptr, (float*)out, st);
    return launch_conv_simt_wgrad<float>(g, (const float*)in0, (const float*)in1, (float*)out, st);
  }
  if (precision == PREC_BF16_SIMT) {
    if (kind == 0) return launch_conv_simt_fprop<bf16>(g, (const bf16*)in0, (const float*)wmat, nullptr, (bf16*)out, st);
    if (kind == 1) return launch_conv_simt_dgrad<bf16>(g, (const bf16*)in0, (const float*)wmat, nullptr, (bf16*)out, st);
    return launch_conv_simt_wgrad<bf16>(g, (const bf16*)in0, (const bf16*)in1, (float*)out, st);
  }
  MN_CHECK(precision == PREC_BF16_TC || precision == PREC_TC_SPLIT, "test_conv: bad precision");
  return mapnet_test_conv_ex(precision, kind, B, Hi, Wi, Ci, Co, k, stride, in0, in1, wmat, nullptr, 0.f, out, stream);
}

// The tensor-core engines of mapnet_test_conv, plus the two strict-mode features the trunk's backward uses:
// a dgrad residual (strict mode: fp32; it may be `out` itself, as in conv_dgrad(conv1, S1, S0, S0)) and the gradient
// out-scale (tc_plan_set_out_scale), a device scalar multiplied into the accumulators before they are stored.
int mapnet_test_conv_ex(int precision, int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride,
                        const void* in0, const void* in1, const void* wmat, const void* residual, float out_scale,
                        void* out, void* stream) {
  MN_CHECK(precision == PREC_BF16_TC || precision == PREC_TC_SPLIT, "test_conv_ex: precision %d is not a tensor-core "
           "training precision (bf16 = %d or tc_split = %d)", precision, PREC_BF16_TC, PREC_TC_SPLIT);
  MN_CHECK(kind >= 0 && kind <= 2, "test_conv_ex: kind %d outside [0, 2]", kind);
  MN_CHECK(B >= 1 && Hi >= 1 && Wi >= 1 && (k == 1 || k == 3) && (stride == 1 || stride == 2) && Ci % 64 == 0 &&
           Co % 64 == 0 && Ci > 0 && Co > 0, "test_conv_ex: bad shape (B %d, %dx%d, Ci %d, Co %d, k %d, stride %d)", B, Hi,
           Wi, Ci, Co, k, stride);
  MN_CHECK(in0 && out && (kind == 2 ? in1 != nullptr : wmat != nullptr), "test_conv_ex: null argument");
  MN_CHECK(residual == nullptr || kind == 1, "test_conv_ex: a residual is a dgrad feature");
  MN_CHECK(out_scale == 0.f || (precision == PREC_TC_SPLIT && kind >= 1 && isfinite(out_scale) && out_scale > 0.f),
           "test_conv_ex: out_scale %g: a positive gradient scale of a strict-mode dgrad / wgrad, or 0", out_scale);
  MN_TRY(require_device());
  ConvGeom g;
  g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
  g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  cudaStream_t st = (cudaStream_t)stream;
  const long long n_in = (long long)B * Hi * Wi * Ci, n_out = (long long)B * g.Ho * g.Wo * Co;
  const int KK = k * k;
  void *s0 = nullptr, *s1 = nullptr, *sw = nullptr;
  float* d_scale = nullptr;
  TcConvPlan* plan = nullptr;
  auto body = [&]() -> int {
    const void *x0 = in0, *x1 = in1, *w = wmat;
    if (precision == PREC_TC_SPLIT) {
      // strict tensor-core mode: fp32 NHWC tensors and fp32 K-major weight matrices in (as for PREC_FP32), fp32 out
      // (and residual); the operands are cut into fp16 hi / lo planes here (the training step's element-wise kernels
      // write that form)
      g.split = 1;
      const long long n0 = (kind == 1) ? n_out : n_in;
      MN_CUDA(cudaMalloc(&s0, (size_t)n0 * 4));
      MN_TRY(launch_split_tensor((const float*)in0, s0, n0, st));
      if (kind == 2) {
        MN_CUDA(cudaMalloc(&s1, (size_t)n_out * 4));
        MN_TRY(launch_split_tensor((const float*)in1, s1, n_out, st));
      } else {
        MN_CUDA(cudaMalloc(&sw, (size_t)Co * KK * Ci * 8));
        if (kind == 0) MN_TRY(launch_split_weight_matrix((const float*)wmat, sw, Co, KK, Ci, st));
        else MN_TRY(launch_split_weight_matrix((const float*)wmat, sw, Ci, KK, Co, st));
      }
      x0 = s0; x1 = s1; w = sw;
    }
    MN_TRY(tc_plan_create(&plan, g, kind, (const bf16*)w));
    if (out_scale != 0.f) {
      MN_CUDA(cudaMalloc((void**)&d_scale, sizeof(float)));
      MN_CUDA(cudaMemcpyAsync(d_scale, &out_scale, sizeof(float), cudaMemcpyHostToDevice, st));
      tc_plan_set_out_scale(plan, d_scale);
    }
    MN_TRY(tc_conv_run(plan, (const bf16*)x0, (const bf16*)x1, (const bf16*)residual, out, st));
    MN_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  const int r = body();
  if (plan) tc_plan_destroy(plan);
  cudaFree(s0); cudaFree(s1); cudaFree(sw); cudaFree(d_scale);
  return r;
}

// JSON description of the plan the tensor-core engines would use for this conv (no device needed).  flags: bit 0 folds
// the downsample shortcut into a stride-2 dgrad; bit 1 describes the strict-mode (split-operand) plan instead of bf16's;
// bit 2 describes the fp8 fprop plan (tc_plan_create_f8).  k == 7 (fprop): the stem as the engines run it, the 4x1 conv
// on the space-to-depth image of an Hi x Wi frame (mapnet_test_conv_affine's k == 7); kind 2 with k == 7: the stem's
// wgrad over that image (mapnet_test_stem_ex)
int mapnet_test_plan_describe(int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, int flags,
                              char* buf, int cap) {
  MN_CHECK(!(flags & 4) || (kind == 0 && !(flags & 3)),
           "test_plan_describe: flag 4 (fp8) describes an fprop plan, without flags 1 or 2");
  ConvGeom g;
  if (k == 7) {
    MN_CHECK((kind == 0 || kind == 2) && Ci == 3 && Co == 64 && stride == 2 && !(flags & 5), "test_plan_describe: the "
             "stem is a 7x7/s2 conv, 3 -> 64, with an fprop and a wgrad");
    WeightDesc wd;
    stem_s2d_geometry(Hi, Wi, 64, &g, &wd, (flags & 2) ? 4 : 2);
  } else {
    g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
    g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  }
  g.B = B;
  if (flags & 2) g.split = 1;
  TcConvPlan* plan = nullptr;
  static const bf16 dummy[8] = {};
  if (flags & 4) MN_TRY(tc_plan_create_f8(&plan, g, (const uint8_t*)dummy));
  else MN_TRY(tc_plan_create(&plan, g, kind, dummy));
  int r = 0;
  if (flags & 1) r = tc_plan_add_shortcut(plan, dummy);
  if (r == 0) r = tc_plan_describe(plan, buf, cap);
  tc_plan_destroy(plan);
  return r;
}

// conv1 (3x3/s2) dgrad with the block's 1x1/s2 downsample dgrad folded in (tc_plan_add_shortcut)
int mapnet_test_dgrad_shortcut(int B, int Hi, int Wi, int Ci, int Co, const void* dy1, const void* dy2,
                               const void* w1_dg, const void* w2_dg, void* dx, void* stream) {
  MN_TRY(require_device());
  MN_CHECK(dy1 && dy2 && w1_dg && w2_dg && dx, "test_dgrad_shortcut: null argument");
  ConvGeom g;
  g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = 3; g.stride = 2; g.pad = 1;
  g.Ho = (Hi + 2 - 3) / 2 + 1; g.Wo = (Wi + 2 - 3) / 2 + 1;
  cudaStream_t st = (cudaStream_t)stream;
  TcConvPlan* plan = nullptr;
  MN_TRY(tc_plan_create(&plan, g, 1, (const bf16*)w1_dg));
  int r = tc_plan_add_shortcut(plan, (const bf16*)w2_dg);
  if (r == 0) r = tc_conv_run(plan, (const bf16*)dy1, (const bf16*)dy2, nullptr, dx, st);
  if (r == 0) { cudaError_t e = cudaStreamSynchronize(st); if (e != cudaSuccess) { set_last_error("test_dgrad_shortcut: %s", cudaGetErrorString(e)); r = 1; } }
  tc_plan_destroy(plan);
  return r;
}

// One wgmma conv launch WITH its fused epilogue, as the training step runs it (bf16 mode):
//   kind 0 (fprop):  out = conv(in0, wmat);  sums[0..1][c] = (sum out, sum out^2) over the stored bf16 values
//                    -- the BatchNorm batch statistics the step takes from the conv epilogue;
//   kind 1 (dgrad):  g = conv_dgrad(in0, wmat) [+ residual], gated by the consumer BatchNorm's ReLU
//                    (zmask > 0, or mscale * y + mshift > 0 when zmask is null), stored as bf16;
//                    sums[0..2][c] = (sum g, sum g*y [, sum g*yd]) over the stored values -- that BatchNorm's
//                    backward reductions.
// host_sums: [3][C] doubles (C = output channels of the launch), replicas already summed.
int mapnet_test_conv_epilogue(int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, const void* in0,
                              const void* wmat, const void* residual, const void* y, const void* zmask, const void* yd,
                              const float* mscale, const float* mshift, void* out, double* host_sums, void* stream) {
  MN_TRY(require_device());
  MN_CHECK((kind == 0 || kind == 1) && in0 && wmat && out && host_sums, "test_conv_epilogue: bad argument");
  ConvGeom g;
  g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
  g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  cudaStream_t st = (cudaStream_t)stream;
  const int C = (kind == 0) ? Co : Ci;
  const size_t acc_doubles = (size_t)kBnAccReplicas * kBnAccStride;
  double* acc = nullptr;
  TcConvPlan* plan = nullptr;
  std::vector<double> h(acc_doubles);
  auto body = [&]() -> int {
    MN_CUDA(cudaMalloc((void**)&acc, acc_doubles * sizeof(double)));
    MN_CUDA(cudaMemsetAsync(acc, 0, acc_doubles * sizeof(double), st));
    MN_TRY(tc_plan_create(&plan, g, kind, (const bf16*)wmat));
    EpiBwd E; memset(&E, 0, sizeof(E));
    if (kind == 1) {
      MN_CHECK(y != nullptr, "test_conv_epilogue: the dgrad epilogue needs y");
      E.y = (const bf16*)y; E.zmask = (const bf16*)zmask; E.yd = (const bf16*)yd; E.mscale = mscale; E.mshift = mshift;
    }
    MN_TRY(tc_conv_run(plan, (const bf16*)in0, nullptr, (const bf16*)residual, out, st, acc, kind == 1 ? &E : nullptr));
    MN_CUDA(cudaMemcpyAsync(h.data(), acc, acc_doubles * sizeof(double), cudaMemcpyDeviceToHost, st));
    MN_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  const int r = body();
  if (r == 0)
    for (int j = 0; j < 3; ++j)
      for (int c = 0; c < C; ++c) {
        double s = 0.0;
        for (int rep = 0; rep < kBnAccReplicas; ++rep) s += h[(size_t)rep * kBnAccStride + (size_t)j * C + c];
        host_sums[(size_t)j * C + c] = s;
      }
  if (plan) tc_plan_destroy(plan);
  cudaFree(acc);
  return r;
}

// the tensor-core stem alone (bf16 mode, no statistics)
int mapnet_test_stem(int B, int H, int W, const float* x_nchw, const float* w_oihw, void* y_out, const void* dy,
                     float* dw_oihw, void* stream) {
  return mapnet_test_stem_ex(PREC_BF16_TC, B, H, W, x_nchw, w_oihw, y_out, dw_oihw ? dy : nullptr, dy ? dw_oihw : nullptr,
                             0.f, nullptr, stream);
}

// The training step's stem (Net::forward_t / backward_t, tensor-core modes): space-to-depth image of the operand type,
// the mode's weight pack, fprop with the BatchNorm-statistics epilogue (host_sums != null), and with dy the wgrad into
// the [64][4][64] patch-matrix accumulator (zeroed first, as backward_t zeroes dw_krsc) re-laid out by k_unpack_wgrads.
// Strict mode: y_out and dy are fp32 (dy cut into fp16 planes here, as the step's element-wise kernels write it) and
// out_scale (0: none) is the wgrad's gradient out-scale.
int mapnet_test_stem_ex(int precision, int B, int H, int W, const float* x_nchw, const float* w_oihw, void* y_out,
                        const void* dy, float* dw_oihw, float out_scale, double* host_sums, void* stream) {
  MN_CHECK(precision == PREC_BF16_TC || precision == PREC_TC_SPLIT, "test_stem_ex: precision %d is not a tensor-core "
           "training precision (bf16 = %d or tc_split = %d)", precision, PREC_BF16_TC, PREC_TC_SPLIT);
  MN_CHECK(B >= 1 && H >= 32 && W >= 32, "test_stem_ex: bad shape (B %d, %dx%d)", B, H, W);
  MN_CHECK(x_nchw && w_oihw && y_out, "test_stem_ex: null argument");
  MN_CHECK((dy == nullptr) == (dw_oihw == nullptr), "test_stem_ex: dy and dw_oihw go together");
  MN_CHECK(out_scale == 0.f || (precision == PREC_TC_SPLIT && dy != nullptr && isfinite(out_scale) && out_scale > 0.f),
           "test_stem_ex: out_scale %g: a positive gradient scale of the strict-mode wgrad, or 0", out_scale);
  MN_TRY(require_device());
  MN_CHECK(tc_overlapped_view_supported(), "test_stem_ex: the driver rejects overlapped tensor maps");
  cudaStream_t st = (cudaStream_t)stream;
  const bool sp = precision == PREC_TC_SPLIT;
  const size_t ez = sp ? 4 : 2;                     // bytes per stored element (split: an fp16 hi / lo pair)
  ConvGeom g; WeightDesc wd; memset(&wd, 0, sizeof(wd));
  stem_s2d_geometry(H, W, 64, &g, &wd, (int)ez);
  g.B = B; wd.p_off = 0; wd.k_off = 0;
  if (sp) g.split = 1;
  const int Hs = g.Hi, Wsp = stem_s2d_wsp(g.Wo);
  const long long n_y = (long long)B * g.Ho * g.Wo * 64;
  const size_t acc_doubles = (size_t)kBnAccReplicas * kBnAccStride;
  void *S = nullptr, *wk = nullptr, *dys = nullptr; float *dwk = nullptr, *f32 = nullptr, *d_scale = nullptr;
  double* acc = nullptr; WeightDesc* d_wd = nullptr;
  TcConvPlan *pf = nullptr, *pw = nullptr;
  std::vector<double> h;
  auto body = [&]() -> int {
    MN_CUDA(cudaMalloc(&S, (size_t)B * Hs * Wsp * 16 * ez));
    MN_CUDA(cudaMalloc(&wk, (size_t)64 * 256 * (sp ? 8 : 2)));
    MN_CUDA(cudaMalloc(&dwk, (size_t)64 * 256 * sizeof(float)));
    MN_CUDA(cudaMalloc(&d_wd, sizeof(WeightDesc)));
    MN_CUDA(cudaMemcpyAsync(d_wd, &wd, sizeof(wd), cudaMemcpyHostToDevice, st));
    MN_CUDA(cudaMemsetAsync(dwk, 0, (size_t)64 * 256 * sizeof(float), st));
    if (sp) {
      MN_CUDA(cudaMalloc(&f32, (size_t)64 * 256 * sizeof(float)));
      MN_TRY(launch_stem_s2d<hsplit>(x_nchw, (hsplit*)S, B, H, W, Hs, Wsp, st));
      MN_TRY(launch_pack_weights_split(d_wd, 1, w_oihw, f32, nullptr, wk, nullptr, 64 * 256, st));
    } else {
      MN_TRY(launch_stem_s2d<bf16>(x_nchw, (bf16*)S, B, H, W, Hs, Wsp, st));
      MN_TRY(launch_pack_weights<bf16>(d_wd, 1, w_oihw, (bf16*)wk, nullptr, 64 * 256, 0, st));
    }
    if (host_sums != nullptr) {
      MN_CUDA(cudaMalloc((void**)&acc, acc_doubles * sizeof(double)));
      MN_CUDA(cudaMemsetAsync(acc, 0, acc_doubles * sizeof(double), st));
    }
    MN_TRY(tc_plan_create(&pf, g, 0, (const bf16*)wk));
    MN_TRY(tc_conv_run(pf, (const bf16*)S, nullptr, nullptr, y_out, st, acc));
    if (dy != nullptr) {
      const void* g_in = dy;
      if (sp) {
        MN_CUDA(cudaMalloc(&dys, (size_t)n_y * 4));
        MN_TRY(launch_split_tensor((const float*)dy, dys, n_y, st));
        g_in = dys;
      }
      MN_TRY(tc_plan_create(&pw, g, 2, nullptr));
      if (out_scale != 0.f) {
        MN_CUDA(cudaMalloc((void**)&d_scale, sizeof(float)));
        MN_CUDA(cudaMemcpyAsync(d_scale, &out_scale, sizeof(float), cudaMemcpyHostToDevice, st));
        tc_plan_set_out_scale(pw, d_scale);
      }
      MN_TRY(tc_conv_run(pw, (const bf16*)S, (const bf16*)g_in, nullptr, dwk, st));
      MN_TRY(launch_unpack_wgrads(d_wd, 1, dwk, dw_oihw, 64 * 256, st));
    }
    if (acc != nullptr) {
      h.resize(acc_doubles);
      MN_CUDA(cudaMemcpyAsync(h.data(), acc, acc_doubles * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    MN_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  const int r = body();
  if (r == 0 && host_sums != nullptr)
    for (int j = 0; j < 2; ++j)
      for (int c = 0; c < 64; ++c) {
        double s = 0.0;
        for (int rep = 0; rep < kBnAccReplicas; ++rep) s += h[(size_t)rep * kBnAccStride + (size_t)j * 64 + c];
        host_sums[(size_t)j * 64 + c] = s;
      }
  if (pf) tc_plan_destroy(pf);
  if (pw) tc_plan_destroy(pw);
  cudaFree(S); cudaFree(wk); cudaFree(dwk); cudaFree(dys); cudaFree(f32); cudaFree(d_scale); cudaFree(acc);
  cudaFree(d_wd);
  return r;
}

// The CUDA-core engines (fp32 and bf16_simt) as Net::conv_fprop / conv_dgrad / conv_wgrad launch them: NHWC activations
// and gradients of the mode's type, fp32 K-major weights, fp32 dW accumulated into `out`.  A residual (dgrad only, out's
// type and shape) is added before the store; it may be `out` itself, as in Net::backward_t's conv_dgrad(conv1, S1, S0, S0).
int mapnet_test_conv_simt(int precision, int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride,
                          const void* in0, const void* in1, const void* wmat, const void* residual, void* out, void* stream) {
  MN_CHECK(precision == PREC_FP32 || precision == PREC_BF16_SIMT, "test_conv_simt: precision %d is not a CUDA-core "
           "precision (fp32 = %d or bf16_simt = %d)", precision, PREC_FP32, PREC_BF16_SIMT);
  MN_CHECK(kind >= 0 && kind <= 2, "test_conv_simt: kind %d outside [0, 2]", kind);
  MN_CHECK(B >= 1 && Hi >= 1 && Wi >= 1 && (k == 1 || k == 3) && (stride == 1 || stride == 2) && Ci > 0 && Co > 0 &&
           Ci % 4 == 0 && Co % 4 == 0, "test_conv_simt: bad shape (B %d, %dx%d, Ci %d, Co %d, k %d, stride %d)", B, Hi,
           Wi, Ci, Co, k, stride);
  MN_CHECK(in0 && out && (kind == 2 ? in1 != nullptr : wmat != nullptr), "test_conv_simt: null argument");
  MN_CHECK(residual == nullptr || kind == 1, "test_conv_simt: a residual is a dgrad feature");
  MN_TRY(require_device());
  ConvGeom g;
  g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
  g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  cudaStream_t st = (cudaStream_t)stream;
  const float* w = (const float*)wmat;
  if (precision == PREC_FP32) {
    if (kind == 0) MN_TRY(launch_conv_simt_fprop<float>(g, (const float*)in0, w, nullptr, (float*)out, st));
    else if (kind == 1) MN_TRY(launch_conv_simt_dgrad<float>(g, (const float*)in0, w, (const float*)residual, (float*)out, st));
    else MN_TRY(launch_conv_simt_wgrad<float>(g, (const float*)in0, (const float*)in1, (float*)out, st));
  } else {
    if (kind == 0) MN_TRY(launch_conv_simt_fprop<bf16>(g, (const bf16*)in0, w, nullptr, (bf16*)out, st));
    else if (kind == 1) MN_TRY(launch_conv_simt_dgrad<bf16>(g, (const bf16*)in0, w, (const bf16*)residual, (bf16*)out, st));
    else MN_TRY(launch_conv_simt_wgrad<bf16>(g, (const bf16*)in0, (const bf16*)in1, (float*)out, st));
  }
  MN_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// The training step's im2col stem (Net::forward_t / backward_t when stem_s2d is off: always in the CUDA-core modes, the
// fallback of the tensor-core modes): k_stem_im2col's [B*Hc*Wc][192] patch matrix of the operand type, the mode's weight
// pack into the [64][192] row, the 1x1 GEMM view (Ci = 192) fprop -- in the tensor-core modes with the BatchNorm-statistics
// epilogue when host_sums != NULL -- and with dy the wgrad into the zeroed [64][192] accumulator, re-laid out into
// dw_oihw [64,3,7,7] by k_unpack_wgrads.  a_out (optional) receives the patch matrix.  Types as mapnet_test_stem_ex, with
// the CUDA-core modes' y_out / dy fp32 (fp32) or bf16 (bf16_simt).
int mapnet_test_stem_im2col(int precision, int B, int H, int W, const float* x_nchw, const float* w_oihw, void* a_out,
                            void* y_out, const void* dy, float* dw_oihw, float out_scale, double* host_sums, void* stream) {
  MN_CHECK(precision >= PREC_FP32 && precision <= PREC_TC_SPLIT, "test_stem_im2col: precision %d is not a training "
           "precision", precision);
  MN_CHECK(B >= 1 && H >= 32 && W >= 32, "test_stem_im2col: bad shape (B %d, %dx%d)", B, H, W);
  MN_TRY(stem_im2col_check(W, kStemIm2colK));
  MN_CHECK(x_nchw && w_oihw && y_out, "test_stem_im2col: null argument");
  MN_CHECK((dy == nullptr) == (dw_oihw == nullptr), "test_stem_im2col: dy and dw_oihw go together");
  MN_CHECK(out_scale == 0.f || (precision == PREC_TC_SPLIT && dy != nullptr && isfinite(out_scale) && out_scale > 0.f),
           "test_stem_im2col: out_scale %g: a positive gradient scale of the strict-mode wgrad, or 0", out_scale);
  const bool tc = precision == PREC_BF16_TC || precision == PREC_TC_SPLIT;
  MN_CHECK(host_sums == nullptr || tc, "test_stem_im2col: the BatchNorm-statistics epilogue is a tensor-core feature "
           "(the CUDA-core modes take the statistics from k_channel_sums)");
  MN_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  const bool sp = precision == PREC_TC_SPLIT;
  const size_t ez = (precision == PREC_BF16_TC || precision == PREC_BF16_SIMT) ? 2 : 4;   // split: an fp16 hi / lo pair
  const int K = kStemIm2colK;
  const int Hc = (H - 1) / 2 + 1, Wc = (W - 1) / 2 + 1;
  ConvGeom g;                                      // the GEMM view: a 1x1 conv over the patch matrix
  g.B = B; g.Hi = g.Ho = Hc; g.Wi = g.Wo = Wc; g.Ci = K; g.Co = 64; g.KH = g.KW = 1; g.stride = 1; g.pad = 0;
  if (sp) g.split = 1;
  WeightDesc wd; memset(&wd, 0, sizeof(wd));
  wd.Co = 64; wd.Ci = K; wd.Ci_real = 3; wd.KH = wd.KW = 1; wd.im2col_k = K;
  const long long M = (long long)B * Hc * Wc, n_y = M * 64;
  const size_t acc_doubles = (size_t)kBnAccReplicas * kBnAccStride;
  void *A = nullptr, *wk = nullptr, *dys = nullptr; float *dwk = nullptr, *f32 = nullptr, *d_scale = nullptr;
  double* acc = nullptr; WeightDesc* d_wd = nullptr;
  TcConvPlan *pf = nullptr, *pw = nullptr;
  std::vector<double> h;
  auto body = [&]() -> int {
    MN_CUDA(cudaMalloc(&A, (size_t)M * K * ez));
    MN_CUDA(cudaMalloc(&wk, (size_t)64 * K * (sp ? 8 : (precision == PREC_BF16_TC ? 2 : 4))));
    MN_CUDA(cudaMalloc(&dwk, (size_t)64 * K * sizeof(float)));
    MN_CUDA(cudaMalloc(&d_wd, sizeof(WeightDesc)));
    MN_CUDA(cudaMemcpyAsync(d_wd, &wd, sizeof(wd), cudaMemcpyHostToDevice, st));
    MN_CUDA(cudaMemsetAsync(dwk, 0, (size_t)64 * K * sizeof(float), st));
    if (precision == PREC_FP32 || precision == PREC_BF16_SIMT) {
      if (precision == PREC_FP32) MN_TRY(launch_stem_im2col<float>(x_nchw, (float*)A, B, H, W, Hc, Wc, K, st));
      else MN_TRY(launch_stem_im2col<bf16>(x_nchw, (bf16*)A, B, H, W, Hc, Wc, K, st));
      MN_TRY(launch_pack_weights<float>(d_wd, 1, w_oihw, (float*)wk, nullptr, 64 * K, precision == PREC_BF16_SIMT, st));
    } else if (sp) {
      MN_CUDA(cudaMalloc(&f32, (size_t)64 * K * sizeof(float)));
      MN_TRY(launch_stem_im2col<hsplit>(x_nchw, (hsplit*)A, B, H, W, Hc, Wc, K, st));
      MN_TRY(launch_pack_weights_split(d_wd, 1, w_oihw, f32, nullptr, wk, nullptr, 64 * K, st));
    } else {
      MN_TRY(launch_stem_im2col<bf16>(x_nchw, (bf16*)A, B, H, W, Hc, Wc, K, st));
      MN_TRY(launch_pack_weights<bf16>(d_wd, 1, w_oihw, (bf16*)wk, nullptr, 64 * K, 0, st));
    }
    if (a_out != nullptr) MN_CUDA(cudaMemcpyAsync(a_out, A, (size_t)M * K * ez, cudaMemcpyDeviceToDevice, st));
    if (host_sums != nullptr) {
      MN_CUDA(cudaMalloc((void**)&acc, acc_doubles * sizeof(double)));
      MN_CUDA(cudaMemsetAsync(acc, 0, acc_doubles * sizeof(double), st));
    }
    if (precision == PREC_FP32) MN_TRY(launch_conv_simt_fprop<float>(g, (const float*)A, (const float*)wk, nullptr, (float*)y_out, st));
    else if (precision == PREC_BF16_SIMT) MN_TRY(launch_conv_simt_fprop<bf16>(g, (const bf16*)A, (const float*)wk, nullptr, (bf16*)y_out, st));
    else {
      MN_TRY(tc_plan_create(&pf, g, 0, (const bf16*)wk));
      MN_TRY(tc_conv_run(pf, (const bf16*)A, nullptr, nullptr, y_out, st, acc));
    }
    if (dy != nullptr) {
      if (precision == PREC_FP32) MN_TRY(launch_conv_simt_wgrad<float>(g, (const float*)A, (const float*)dy, dwk, st));
      else if (precision == PREC_BF16_SIMT) MN_TRY(launch_conv_simt_wgrad<bf16>(g, (const bf16*)A, (const bf16*)dy, dwk, st));
      else {
        const void* g_in = dy;
        if (sp) {
          MN_CUDA(cudaMalloc(&dys, (size_t)n_y * 4));
          MN_TRY(launch_split_tensor((const float*)dy, dys, n_y, st));
          g_in = dys;
        }
        MN_TRY(tc_plan_create(&pw, g, 2, nullptr));
        if (out_scale != 0.f) {
          MN_CUDA(cudaMalloc((void**)&d_scale, sizeof(float)));
          MN_CUDA(cudaMemcpyAsync(d_scale, &out_scale, sizeof(float), cudaMemcpyHostToDevice, st));
          tc_plan_set_out_scale(pw, d_scale);
        }
        MN_TRY(tc_conv_run(pw, (const bf16*)A, (const bf16*)g_in, nullptr, dwk, st));
      }
      MN_TRY(launch_unpack_wgrads(d_wd, 1, dwk, dw_oihw, 64 * K, st));
    }
    if (acc != nullptr) {
      h.resize(acc_doubles);
      MN_CUDA(cudaMemcpyAsync(h.data(), acc, acc_doubles * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    MN_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  const int r = body();
  if (r == 0 && host_sums != nullptr)
    for (int j = 0; j < 2; ++j)
      for (int c = 0; c < 64; ++c) {
        double s = 0.0;
        for (int rep = 0; rep < kBnAccReplicas; ++rep) s += h[(size_t)rep * kBnAccStride + (size_t)j * 64 + c];
        host_sums[(size_t)j * 64 + c] = s;
      }
  if (pf) tc_plan_destroy(pf);
  if (pw) tc_plan_destroy(pw);
  cudaFree(A); cudaFree(wk); cudaFree(dwk); cudaFree(dys); cudaFree(f32); cudaFree(d_scale); cudaFree(acc);
  cudaFree(d_wd);
  return r;
}

// One wgmma fprop launch with the inference epilogue (conv_tc.cu, EPI_AFFINE): out = relu?(conv * scale + shift
// [+ residual]).  flags: bit 0 ReLU, bit 1 (strict mode) residual in hi/lo plane form, bit 2 (strict mode) output in
// hi/lo plane form.  k == 7: the stem as the engine runs it (in0 = fp32 NCHW image, wmat = fp32 [Co][3][7][7]).
// Otherwise bf16 mode: in0 / residual / out bf16 NHWC, wmat bf16 [Co][k][k][Ci]; strict mode: fp32 NHWC in0 / residual
// and fp32 [Co][k][k][Ci] wmat, cut into fp16 hi/lo planes here (the engine's operands are stored in that form).
int mapnet_test_conv_affine(int precision, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, const void* in0,
                            const void* wmat, const float* scale, const float* shift, const void* residual, int flags,
                            void* out, void* stream) {
  MN_CHECK(precision == PREC_BF16_TC || precision == PREC_TC_SPLIT, "test_conv_affine: precision %d is not supported "
           "(bf16 = %d or tc_split = %d)", precision, PREC_BF16_TC, PREC_TC_SPLIT);
  MN_CHECK(in0 && wmat && scale && shift && out && B >= 1, "test_conv_affine: bad argument");
  MN_CHECK(k != 7 || (Ci == 3 && Co == 64 && stride == 2 && residual == nullptr), "test_conv_affine: the stem is 7x7/s2, 3 -> 64, no residual");
  MN_TRY(require_device());
  const bool sp = precision == PREC_TC_SPLIT;
  EpiAffine a;
  a.scale = scale; a.shift = shift; a.relu = flags & 1; a.res_split = (flags >> 1) & 1; a.out_split = (flags >> 2) & 1;
  MN_CHECK(tc_affine_supported(sp, residual != nullptr, a), "test_conv_affine: epilogue variant not built (flags %d, "
           "residual %d)", flags, residual != nullptr);
  cudaStream_t st = (cudaStream_t)stream;
  ConvGeom g; WeightDesc wd; memset(&wd, 0, sizeof(wd));
  if (k == 7) {
    stem_s2d_geometry(Hi, Wi, 64, &g, &wd, sp ? 4 : 2);
    MN_CHECK(tc_overlapped_view_supported(), "test_conv_affine: the driver rejects overlapped tensor maps");
  } else {
    g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
    g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  }
  g.B = B;
  if (sp) g.split = 1;
  const long long n_out = (long long)B * g.Ho * g.Wo * Co;
  void *x = nullptr, *w = nullptr, *r = nullptr, *f32 = nullptr; WeightDesc* d_wd = nullptr;
  TcConvPlan* plan = nullptr;
  auto body = [&]() -> int {
    const void* xin = in0; const void* win = wmat; const void* rin = residual;
    if (k == 7) {
      const int Wsp = stem_s2d_wsp(g.Wo);
      MN_CUDA(cudaMalloc(&x, (size_t)B * g.Hi * Wsp * 16 * (sp ? 4 : 2)));
      MN_CUDA(cudaMalloc(&w, (size_t)64 * 256 * (sp ? 8 : 2)));
      MN_CUDA(cudaMalloc((void**)&d_wd, sizeof(WeightDesc)));
      MN_CUDA(cudaMemcpyAsync(d_wd, &wd, sizeof(wd), cudaMemcpyHostToDevice, st));
      if (sp) {
        MN_CUDA(cudaMalloc(&f32, (size_t)64 * 256 * 4));
        MN_TRY(launch_stem_s2d<hsplit>((const float*)in0, (hsplit*)x, B, Hi, Wi, g.Hi, Wsp, st));
        MN_TRY(launch_pack_weights_split(d_wd, 1, (const float*)wmat, (float*)f32, nullptr, w, nullptr, 64 * 256, st));
      } else {
        MN_TRY(launch_stem_s2d<bf16>((const float*)in0, (bf16*)x, B, Hi, Wi, g.Hi, Wsp, st));
        MN_TRY(launch_pack_weights<bf16>(d_wd, 1, (const float*)wmat, (bf16*)w, nullptr, 64 * 256, 0, st));
      }
      xin = x; win = w;
    } else if (sp) {
      const long long n_in = (long long)B * Hi * Wi * Ci;
      MN_CUDA(cudaMalloc(&x, (size_t)n_in * 4));
      MN_TRY(launch_split_tensor((const float*)in0, x, n_in, st));
      MN_CUDA(cudaMalloc(&w, (size_t)Co * k * k * Ci * 8));
      MN_TRY(launch_split_weight_matrix((const float*)wmat, w, Co, k * k, Ci, st));
      if (residual != nullptr && a.res_split) {
        MN_CUDA(cudaMalloc(&r, (size_t)n_out * 4));
        MN_TRY(launch_split_tensor((const float*)residual, r, n_out, st));
        rin = r;
      }
      xin = x; win = w;
    }
    MN_TRY(tc_plan_create(&plan, g, 0, (const bf16*)win));
    MN_TRY(tc_conv_run(plan, (const bf16*)xin, nullptr, (const bf16*)rin, out, st, nullptr, nullptr, &a));
    MN_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  const int rc = body();
  if (plan) tc_plan_destroy(plan);
  cudaFree(x); cudaFree(w); cudaFree(r); cudaFree(f32); cudaFree(d_wd);
  return rc;
}

// One k_f8_conv launch (conv_tc.cu): in0 e4m3 NHWC [B,Hi,Wi,Ci], wmat e4m3 [Co][k][k][Ci], scale / shift fp32 [Co] (the
// folded table), residual e4m3 (flags bit 1, scaled by *res_scale) or bf16, out e4m3 (flags bit 2, stored as f * *out_inv)
// or bf16; flags bit 0 ReLU, bit 3 calibration pass: max |f| into *amax (out untouched).
int mapnet_test_conv_fp8(int B, int Hi, int Wi, int Ci, int Co, int k, int stride, const void* in0, const void* wmat,
                         const float* scale, const float* shift, const void* residual, const float* res_scale,
                         const float* out_inv, int flags, void* out, unsigned int* amax, void* stream) {
  MN_CHECK(in0 && wmat && scale && shift && B >= 1 && (out || (flags & 8)), "test_conv_fp8: bad argument");
  MN_CHECK(k == 1 || k == 3, "test_conv_fp8: k must be 1 or 3");
  MN_CHECK(!(flags & 8) || amax != nullptr, "test_conv_fp8: the calibration pass needs amax");
  MN_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  ConvGeom g;
  g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
  g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  EpiF8 e; memset(&e, 0, sizeof(e));
  e.scale = scale; e.shift = shift; e.relu = flags & 1; e.res_f8 = (flags >> 1) & 1; e.out_f8 = (flags >> 2) & 1;
  e.res_scale = res_scale; e.out_inv = out_inv; e.amax = (flags & 8) ? amax : nullptr;
  TcConvPlan* plan = nullptr;
  int rc = tc_plan_create_f8(&plan, g, (const uint8_t*)wmat);
  if (rc == 0) rc = tc_conv_run_f8(plan, (const uint8_t*)in0, residual, out, e, st);
  if (rc == 0 && cudaStreamSynchronize(st) != cudaSuccess) { set_last_error("test_conv_fp8: %s", cudaGetErrorString(cudaGetLastError())); rc = 1; }
  if (plan) tc_plan_destroy(plan);
  return rc;
}

}  // extern "C"

// ---- the element-wise kernels of bn.cu / head.cu one launch sequence at a time (tests/test_gpu_bn_pool.py) ----
// Per-BatchNorm state: kTestBnRows rows of C floats (rows as in include/mapnet_b200.h), uploaded from host_params before
// every pass and copied back into host_out after it.
enum { TB_GAMMA, TB_BETA, TB_RMEAN, TB_RVAR, TB_MEAN, TB_INVSTD, TB_SCALE, TB_SHIFT, TB_MSCALE, TB_MSHIFT, TB_DGAMMA,
       TB_DBETA, TB_COEF, kTestBnRows = TB_COEF + 3 };

static bool test_prec_ok(int p) {
  return p == PREC_FP32 || p == PREC_BF16_TC || p == PREC_BF16_SIMT || p == PREC_TC_SPLIT;
}

// the (A, Z, G) element types Net uses for a training precision
template <typename Fn>
static int with_test_types(int precision, Fn&& fn) {
  if (precision == PREC_FP32) return fn(TypesF32());
  if (precision == PREC_TC_SPLIT) return fn(TypesSplitHH());
  return fn(TypesBF16());
}

struct TestBnState {
  float* d = nullptr;          // [nbn][kTestBnRows][C]
  double* accum = nullptr;     // [slot][kBnAccReplicas][kBnAccStride]
  unsigned int* counter = nullptr;
  float* gscale = nullptr;
  int nbn = 0, C = 0;
  float* row(int bn, int r) const { return d + ((size_t)bn * kTestBnRows + r) * C; }
  double* acc(int slot) const { return accum + (size_t)slot * kBnAccReplicas * kBnAccStride; }
  // nslots accumulator slots of kBnAccReplicas replicas (zeroed) and one counter
  int alloc(int nbn_, int C_, int nslots, cudaStream_t st) {
    nbn = nbn_; C = C_;
    const size_t acc_bytes = (size_t)nslots * kBnAccReplicas * kBnAccStride * sizeof(double);
    MN_CUDA(cudaMalloc((void**)&d, (size_t)nbn * kTestBnRows * C * sizeof(float)));
    MN_CUDA(cudaMalloc((void**)&accum, acc_bytes));
    MN_CUDA(cudaMalloc((void**)&counter, sizeof(unsigned int)));
    MN_CUDA(cudaMalloc((void**)&gscale, sizeof(float)));
    MN_CUDA(cudaMemsetAsync(accum, 0, acc_bytes, st));
    MN_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), st));
    return 0;
  }
  void release() { cudaFree(d); cudaFree(accum); cudaFree(counter); cudaFree(gscale); }
  int upload(const float* host_params, cudaStream_t st) {
    MN_CUDA(cudaMemcpyAsync(d, host_params, (size_t)nbn * kTestBnRows * C * sizeof(float), cudaMemcpyHostToDevice, st));
    return 0;
  }
  // host_sums [nrep][3][C] into the replica layout of bn_fin.cuh (replica r at kBnAccStride * r)
  int upload_sums(int slot, const double* host_sums, int nrep, cudaStream_t st) {
    MN_CUDA(cudaMemcpy2DAsync(acc(slot), kBnAccStride * sizeof(double), host_sums, 3 * (size_t)C * sizeof(double),
                              3 * (size_t)C * sizeof(double), nrep, cudaMemcpyHostToDevice, st));
    return 0;
  }
  int download(float* host_out, cudaStream_t st) {
    MN_CUDA(cudaMemcpyAsync(host_out, d, (size_t)nbn * kTestBnRows * C * sizeof(float), cudaMemcpyDeviceToHost, st));
    MN_CUDA(cudaStreamSynchronize(st));
    return 0;
  }
  BnFin fwd(int bn) const {
    BnFin f; memset(&f, 0, sizeof(f));
    f.gamma = row(bn, TB_GAMMA); f.beta = row(bn, TB_BETA); f.run_mean = row(bn, TB_RMEAN); f.run_var = row(bn, TB_RVAR);
    f.mean = row(bn, TB_MEAN); f.invstd = row(bn, TB_INVSTD); f.scale = row(bn, TB_SCALE); f.shift = row(bn, TB_SHIFT);
    return f;
  }
  // the backward of BatchNorm 0 [and of the downsample BatchNorm 1]; gate 2: the ReLU gate recomputed from y
  BnFin bwd(bool ds, int gate) const {
    BnFin f; memset(&f, 0, sizeof(f));
    f.gamma = row(0, TB_GAMMA); f.mean = row(0, TB_MEAN); f.invstd = row(0, TB_INVSTD);
    f.dgamma = row(0, TB_DGAMMA); f.dbeta = row(0, TB_DBETA); f.coef = row(0, TB_COEF);
    if (gate == 2) { f.mscale = row(0, TB_MSCALE); f.mshift = row(0, TB_MSHIFT); }
    if (ds) {
      f.gamma2 = row(1, TB_GAMMA); f.mean2 = row(1, TB_MEAN); f.invstd2 = row(1, TB_INVSTD);
      f.dgamma2 = row(1, TB_DGAMMA); f.dbeta2 = row(1, TB_DBETA); f.coef2 = row(1, TB_COEF);
    }
    return f;
  }
  BnDesc desc(const BnFin& f, long long M, bool sums, int bn, int nrep, bool forward) const {
    BnDesc L; memset(&L, 0, sizeof(L));
    if (sums) { L.accum = acc(bn); L.nrep = nrep; }
    L.M = M; L.invM = 1.0 / (double)M;
    L.unbias = (forward && M > 1) ? (double)M / (double)(M - 1) : 1.0;
    L.f = f;
    return L;
  }
};

// forward per-channel parameters of BatchNorm bn as Net derives them: source 0 k_channel_sums over y (finalize by the
// last block), 2 k_bn_eval_scale; sources 1 (lazy: the consumer finalizes) and 3 (scale / shift as given) launch nothing
template <typename T>
static int test_bn_forward_params(const TestBnState& s, int bn, int source, const T* y, long long M, cudaStream_t st) {
  if (source == 0) return launch_bn_stats<T>(y, M, s.C, s.fwd(bn), s.acc(bn), s.counter, st);
  if (source == 2) return launch_bn_eval_scale(s.C, s.fwd(bn), st);
  return 0;
}

extern "C" {

int mapnet_test_bn_forward(int precision, int res_mode, int relu, int source, int64_t M, int C, const void* y,
                           const void* res, void* z, const float* host_params, const double* host_sums, int nrep,
                           float* host_out, void* stream) {
  MN_CHECK(test_prec_ok(precision), "test_bn_forward: precision %d is not a training precision", precision);
  MN_CHECK(res_mode >= 0 && res_mode <= 2, "test_bn_forward: res_mode %d outside [0, 2]", res_mode);
  MN_CHECK(source >= 0 && source <= 3, "test_bn_forward: source %d outside [0, 3]", source);
  MN_CHECK(M >= 1 && C >= 64 && C <= 512 && C % 64 == 0, "test_bn_forward: need M >= 1 and C a multiple of 64 in "
           "[64, 512] (got M %lld, C %d)", (long long)M, C);
  MN_CHECK(y && z && host_params && host_out, "test_bn_forward: null argument");
  MN_CHECK(res_mode == 0 || res != nullptr, "test_bn_forward: res_mode %d needs res (%s)", res_mode,
           res_mode == 2 ? "the downsample branch's conv output, second BatchNorm" : "the identity branch");
  MN_CHECK(source != 1 || (host_sums && nrep >= 1 && nrep <= kBnAccReplicas), "test_bn_forward: the lazy source needs "
           "host_sums and 1 <= nrep <= %d (got %d)", kBnAccReplicas, nrep);
  MN_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  const int nbn = res_mode == 2 ? 2 : 1;
  const int passes = source == 0 ? 2 : 1;     // source 0: the reduction twice on the same accumulators and counter
  TestBnState s;
  auto body = [&]() -> int {
    MN_TRY(s.alloc(nbn, C, nbn, st));
    for (int pass = 0; pass < passes; ++pass) {
      MN_TRY(s.upload(host_params, st));
      if (source == 1)
        for (int bn = 0; bn < nbn; ++bn) MN_TRY(s.upload_sums(bn, host_sums + (size_t)bn * nrep * 3 * C, nrep, st));
      MN_TRY(with_test_types(precision, [&](auto tp) -> int {
        typedef typename decltype(tp)::A T;
        typedef typename decltype(tp)::Z TZ;
        MN_TRY(test_bn_forward_params<T>(s, 0, source, (const T*)y, M, st));
        if (nbn == 2) MN_TRY(test_bn_forward_params<T>(s, 1, source, (const T*)res, M, st));
        const BnDesc l1 = s.desc(s.fwd(0), M, source == 1, 0, nrep, true);
        const BnDesc l2 = s.desc(s.fwd(nbn - 1), M, source == 1, nbn - 1, nrep, true);
        return launch_bn_apply<T, TZ>((const T*)y, res_mode, res, (TZ*)z, M, C, relu, l1, nbn == 2 ? &l2 : nullptr, st);
      }));
      MN_TRY(s.download(host_out + (size_t)pass * nbn * kTestBnRows * C, st));
    }
    return 0;
  };
  const int r = body();
  s.release();
  return r;
}

int mapnet_test_bn_backward(int precision, int source, int gate, int64_t M, int C, const void* dout, const void* zmask,
                            const void* y, const void* yd, void* dy, void* dyd, void* gout, const float* host_params,
                            const double* host_sums, int nrep, float gscale, float* host_out, void* stream) {
  MN_CHECK(test_prec_ok(precision), "test_bn_backward: precision %d is not a training precision", precision);
  MN_CHECK(source == 0 || source == 1, "test_bn_backward: source %d is neither 0 (reduce) nor 1 (lazy)", source);
  MN_CHECK(gate >= 0 && gate <= 2, "test_bn_backward: gate %d outside [0, 2]", gate);
  MN_CHECK(M >= 1 && C >= 64 && C <= 512 && C % 64 == 0, "test_bn_backward: need M >= 1 and C a multiple of 64 in "
           "[64, 512] (got M %lld, C %d)", (long long)M, C);
  MN_CHECK(dout && y && dy && host_params && host_out, "test_bn_backward: null argument");
  MN_CHECK((gate == 1) == (zmask != nullptr), "test_bn_backward: zmask is given exactly when gate == 1");
  MN_CHECK((yd != nullptr) == (dyd != nullptr), "test_bn_backward: yd and dyd go together (downsample BatchNorm)");
  MN_CHECK(source != 1 || (host_sums && nrep >= 1 && nrep <= kBnAccReplicas), "test_bn_backward: the lazy source needs "
           "host_sums and 1 <= nrep <= %d (got %d)", kBnAccReplicas, nrep);
  MN_CHECK(gscale >= 0.f, "test_bn_backward: gscale %g < 0", (double)gscale);
  MN_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  const bool ds = yd != nullptr;
  const int nbn = ds ? 2 : 1;
  const int passes = source == 0 ? 2 : 1;
  TestBnState s;
  auto body = [&]() -> int {
    MN_TRY(s.alloc(nbn, C, nbn, st));
    MN_CUDA(cudaMemcpyAsync(s.gscale, &gscale, sizeof(float), cudaMemcpyHostToDevice, st));
    for (int pass = 0; pass < passes; ++pass) {
      MN_TRY(s.upload(host_params, st));
      if (source == 1) MN_TRY(s.upload_sums(0, host_sums, nrep, st));
      MN_TRY(with_test_types(precision, [&](auto tp) -> int {
        typedef typename decltype(tp)::A T;
        typedef typename decltype(tp)::Z TZ;
        typedef typename decltype(tp)::G TG;
        const BnFin f = s.bwd(ds, gate);
        if (source == 0)
          MN_TRY((launch_bn_bwd_reduce<T, TZ>((const T*)dout, (const TZ*)zmask, (const T*)y, (const T*)yd, M, C, f,
                                              s.acc(0), s.counter, st)));
        return launch_bn_bwd_apply<T, TZ, TG>((const T*)dout, (const TZ*)zmask, (const T*)y, (TG*)dy, (const T*)yd,
                                              (TG*)dyd, (T*)gout, M, C, s.desc(f, M, source == 1, 0, nrep, false),
                                              gscale > 0.f ? s.gscale : nullptr, st);
      }));
      MN_TRY(s.download(host_out + (size_t)pass * nbn * kTestBnRows * C, st));
    }
    return 0;
  };
  const int r = body();
  s.release();
  return r;
}

int mapnet_test_stem_pool(int precision, int source, int bsource, int B, int Hc, int Wc, const void* y, void* z,
                          void* amax, const void* dz, void* g, void* dy, const float* host_params,
                          const double* host_sums, int nrep, float* host_out, void* stream) {
  const bool f8 = precision == PREC_FP8;
  MN_CHECK(test_prec_ok(precision) || f8, "test_stem_pool: precision %d is neither a training precision nor fp8",
           precision);
  MN_CHECK(source >= 0 && source <= 3, "test_stem_pool: source %d outside [0, 3]", source);
  MN_CHECK(B >= 1 && Hc >= 1 && Wc >= 1, "test_stem_pool: bad shape %dx%dx%d", B, Hc, Wc);
  MN_CHECK(y && z && host_params && host_out, "test_stem_pool: null argument");
  MN_CHECK(!f8 || (source == 3 && dz == nullptr), "test_stem_pool: fp8 is the inference pool (source 3, no backward)");
  MN_CHECK(source != 1 || (host_sums && nrep >= 1 && nrep <= kBnAccReplicas), "test_stem_pool: the lazy source needs "
           "host_sums and 1 <= nrep <= %d (got %d)", kBnAccReplicas, nrep);
  const bool even = Hc % 2 == 0 && Wc % 2 == 0;
  if (dz != nullptr) {
    MN_CHECK(amax && g && dy && source != 3, "test_stem_pool: the backward needs amax, g, dy and batch statistics");
    MN_CHECK(bsource == 0 || bsource == 1, "test_stem_pool: bsource %d is neither 0 nor 1 (lazy)", bsource);
    MN_CHECK(bsource == 0 || even, "test_stem_pool: the lazy backward needs even Hc, Wc (got %dx%d)", Hc, Wc);
  }
  MN_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  const int C = 64;
  const int Ho = (Hc - 1) / 2 + 1, Wo = (Wc - 1) / 2 + 1;
  const long long M = (long long)B * Hc * Wc;
  TestBnState s;
  auto body = [&]() -> int {
    MN_TRY(s.alloc(1, C, 2, st));        // slot 0: the forward sums, slot 1: the backward's (as Net's two slots)
    MN_TRY(s.upload(host_params, st));
    if (source == 1) MN_TRY(s.upload_sums(0, host_sums, nrep, st));
    const BnDesc lf = s.desc(s.fwd(0), M, source == 1, 0, nrep, true);
    if (f8) {
      MN_TRY((launch_stem_pool<bf16, e4m3>((const bf16*)y, (e4m3*)z, (uint8_t*)amax, B, Hc, Wc, Ho, Wo, C, lf, st)));
      return s.download(host_out, st);
    }
    MN_TRY(with_test_types(precision, [&](auto tp) -> int {
      typedef typename decltype(tp)::A T;
      typedef typename decltype(tp)::Z TZ;
      typedef typename decltype(tp)::G TG;
      MN_TRY(test_bn_forward_params<T>(s, 0, source, (const T*)y, M, st));
      MN_TRY((launch_stem_pool<T, TZ>((const T*)y, (TZ*)z, (uint8_t*)amax, B, Hc, Wc, Ho, Wo, C, lf, st)));
      if (dz == nullptr) return 0;
      // the stem's backward as Net runs it: even sizes accumulate the BatchNorm sums in the pool backward (finalized by
      // k_bn_bwd_finalize_accum, or lazily by the apply kernel over kBnAccReplicas replicas), odd sizes reduce afterwards
      const BnFin fb = s.bwd(false, 0);
      if (even) {
        MN_TRY(launch_stem_pool_bwd<T>((const T*)dz, (const uint8_t*)amax, (const T*)y, s.row(0, TB_SCALE),
                                       s.row(0, TB_SHIFT), (T*)g, B, Hc, Wc, Ho, Wo, C, st, s.acc(1)));
        if (bsource == 0) MN_TRY(launch_bn_bwd_finalize_accum(M, C, fb, s.acc(1), st));
      } else {
        MN_TRY(launch_stem_pool_bwd<T>((const T*)dz, (const uint8_t*)amax, (const T*)y, s.row(0, TB_SCALE),
                                       s.row(0, TB_SHIFT), (T*)g, B, Hc, Wc, Ho, Wo, C, st));
        MN_TRY((launch_bn_bwd_reduce<T, TZ>((const T*)g, (const TZ*)nullptr, (const T*)y, nullptr, M, C, fb, s.acc(1),
                                            s.counter, st)));
      }
      return launch_bn_bwd_apply<T, TZ, TG>((const T*)g, (const TZ*)nullptr, (const T*)y, (TG*)dy, nullptr, nullptr,
                                            nullptr, M, C, s.desc(fb, M, bsource == 1, 1, kBnAccReplicas, false),
                                            nullptr, st);
    }));
    return s.download(host_out, st);
  };
  const int r = body();
  s.release();
  return r;
}

int mapnet_test_gap(int precision, int B, int HW, int C, const void* z, float* feat, const float* dfeat, void* dz,
                    void* stream) {
  MN_CHECK(test_prec_ok(precision), "test_gap: precision %d is not a training precision", precision);
  MN_CHECK(B >= 1 && HW >= 1 && C >= 8 && C <= 2048 && C % 8 == 0, "test_gap: bad shape B %d HW %d C %d", B, HW, C);
  MN_CHECK(z && feat && dfeat && dz, "test_gap: null argument");
  MN_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  MN_TRY(with_test_types(precision, [&](auto tp) -> int {
    typedef typename decltype(tp)::A T;
    typedef typename decltype(tp)::Z TZ;
    MN_TRY(launch_gap<TZ>((const TZ*)z, feat, B, HW, C, st));
    return launch_gap_bwd<T>(dfeat, (T*)dz, B, HW, C, st);
  }));
  MN_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// ---- eval-mode inference engine (infer.cu) ----
int64_t mapnet_infer_arena_bytes(int max_B, int H, int W, int precision) {
  return InferNet::arena_bytes(max_B, H, W, precision);
}

int mapnet_infer_create(mapnet_infer_t** out, int max_B, int H, int W, int feat_dim, int precision) {
  MN_CHECK(out != nullptr, "infer_create: null out pointer");
  *out = nullptr;
  // argument errors first: nothing is allocated or launched for a call that cannot succeed
  MN_CHECK(precision == PREC_BF16_TC || precision == PREC_TC_SPLIT || precision == PREC_FP8, "infer_create: precision %d "
           "is not supported (bf16 = %d, tc_split = %d or fp8 = %d)", precision, PREC_BF16_TC, PREC_TC_SPLIT, PREC_FP8);
  MN_CHECK(max_B >= 1 && H >= 32 && W >= 32, "infer_create: need max_B >= 1 and H, W >= 32 (got %d, %d, %d)", max_B, H, W);
  MN_CHECK(feat_dim >= 8 && feat_dim % 4 == 0, "infer_create: feat_dim must be a multiple of 4");
  MN_TRY(require_device());
  mapnet_infer* h = new mapnet_infer();
  int r = h->net.init(max_B, H, W, feat_dim, precision);
  if (r != 0) { h->net.destroy(); delete h; return r; }
  *out = h;
  return 0;
}

int mapnet_infer_load(mapnet_infer_t* h, const float* params_flat, const float* bufs_flat, void* stream) {
  MN_CHECK(h != nullptr, "infer_load: null handle");
  return h->net.load(params_flat, bufs_flat, (cudaStream_t)stream);
}

int mapnet_infer_forward(mapnet_infer_t* h, const float* x, int B, float droprate, uint64_t seed, uint64_t step,
                         float* pred, void* stream) {
  MN_CHECK(h != nullptr, "infer_forward: null handle");
  return h->net.forward(x, B, droprate, seed, step, pred, (cudaStream_t)stream);
}

int mapnet_infer_forward_frames(mapnet_infer_t* h, mapnet_preprocess_t* pre, const void* frames_nhwc_u8, int B,
                                const float* mean3, const float* std3, float droprate, uint64_t seed, uint64_t step,
                                float* pred, void* stream) {
  MN_CHECK(h != nullptr, "infer_forward_frames: null handle");
  return h->net.forward_frames(pre, (const uint8_t*)frames_nhwc_u8, B, mean3, std3, droprate, seed, step, pred,
                               (cudaStream_t)stream);
}

int mapnet_infer_sample(mapnet_infer_t* h, const float* x, int B, int S, float droprate, uint64_t seed, uint64_t step,
                        float* samples, double* mean, double* cov, void* stream) {
  MN_CHECK(h != nullptr, "infer_sample: null handle");
  return h->net.sample(x, B, S, droprate, seed, step, samples, mean, cov, (cudaStream_t)stream);
}

int mapnet_infer_sample_frames(mapnet_infer_t* h, mapnet_preprocess_t* pre, const void* frames_nhwc_u8, int B,
                               const float* mean3, const float* std3, int S, float droprate, uint64_t seed,
                               uint64_t step, float* samples, double* mean, double* cov, void* stream) {
  MN_CHECK(h != nullptr, "infer_sample_frames: null handle");
  return h->net.sample_frames(pre, (const uint8_t*)frames_nhwc_u8, B, mean3, std3, S, droprate, seed, step, samples,
                              mean, cov, (cudaStream_t)stream);
}

// host-only: launch_small_gemm's split-K plan of one product
int mapnet_test_small_gemm_plan(int epi, int M, int N, int K, int* splits, int* kchunk) {
  MN_CHECK(epi >= 0 && epi <= 2 && M >= 1 && N >= 1 && K >= 1 && splits != nullptr && kchunk != nullptr,
           "test_small_gemm_plan: bad argument");
  *splits = small_gemm_split_plan(epi, M, N, K, kchunk);
  return 0;
}

// The pose head as the training step runs it (head_forward, then with dpred head_backward with every parameter
// trained) on caller-owned fp32 device tensors.  params / grads: fc_w [F][512], fc_b [F], xyz_w [3][F], xyz_b [3],
// wpqr_w [3][F], wpqr_b [3], packed in that order.
int mapnet_test_head(int B, int F, const float* feat, const float* params, float droprate, uint64_t seed, uint64_t step,
                     uint64_t stride, uint64_t* ctr, float* mask, float* fcpre, float* hdrop, float* pred,
                     const float* dpred, int filter_nans, float* dh, float* dfeat, float* grads, float* scale2,
                     void* stream) {
  MN_CHECK(B >= 1 && F >= 8 && F % 4 == 0, "test_head: need B >= 1 and F a multiple of 4, >= 8 (got B %d, F %d)", B, F);
  MN_CHECK(feat && params && fcpre && hdrop && pred, "test_head: null argument");
  MN_CHECK(droprate >= 0.f && droprate < 1.f, "test_head: droprate %g outside [0, 1)", (double)droprate);
  MN_CHECK(droprate == 0.f || (mask != nullptr && stride >= (uint64_t)B * F && (step != ~0ULL || ctr != nullptr)),
           "test_head: dropout needs mask, stride >= B * F (got %llu) and, at step ~0, the device counter ctr",
           (unsigned long long)stride);
  MN_CHECK(dpred == nullptr || (dh && dfeat && grads), "test_head: the backward needs dh, dfeat and grads");
  MN_CHECK(scale2 == nullptr || dpred != nullptr, "test_head: the gradient scale is a backward output");
  MN_TRY(require_device());
  cudaStream_t st = (cudaStream_t)stream;
  const long long F512 = (long long)F * 512;
  const HeadParams hp{params, params + F512, params + F512 + F, params + F512 + 4 * F, params + F512 + 4 * F + 3,
                      params + F512 + 7 * F + 3};
  float* dpf = nullptr;
  auto body = [&]() -> int {
    MN_TRY(head_forward(hp, feat, B, F, droprate, seed, step, (unsigned long long*)ctr, stride, mask, fcpre, hdrop, pred,
                        st));
    if (dpred != nullptr) {
      const HeadGrads hg{grads, grads + F512, grads + F512 + F, grads + F512 + 4 * F, grads + F512 + 4 * F + 3,
                         grads + F512 + 7 * F + 3};
      MN_CUDA(cudaMalloc((void**)&dpf, (size_t)B * 12 * sizeof(float)));
      MN_TRY(head_backward(hp, hg, dpred, filter_nans, feat, droprate > 0.f ? mask : nullptr, fcpre, hdrop, B, F, dpf,
                           dpf + (size_t)B * 6, scale2, dh, dfeat, st));
    }
    MN_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  const int r = body();
  cudaFree(dpf);
  return r;
}

// The weight-pack table of a parameter-table-only trunk in one precision; fp8 uses the bf16 table, as InferNet::init.
// im2col_stem: the tensor-core modes' fallback stem layout (the CUDA-core modes always have it; the fp8 engine never).
static int pack_spec(Net* spec, int H, int W, int precision, int im2col_stem, const char* what) {
  MN_CHECK(precision >= PREC_FP32 && precision <= PREC_FP8, "%s: precision %d outside [0, 4]", what, precision);
  MN_CHECK(im2col_stem == 0 || im2col_stem == 1, "%s: im2col_stem %d is not 0 or 1", what, im2col_stem);
  MN_CHECK(!(im2col_stem && precision == PREC_FP8), "%s: the fp8 engine has no im2col stem", what);
  return spec->init(0, H, W, 2048, precision == PREC_FP8 ? PREC_BF16_TC : precision, im2col_stem);
}

int mapnet_test_weight_table(int H, int W, int precision, int im2col_stem, int64_t* out, int cap) {
  MN_CHECK(out != nullptr, "test_weight_table: null out pointer");
  Net* spec = new Net();
  int r = pack_spec(spec, H, W, precision, im2col_stem, "test_weight_table");
  const int n = (int)spec->convs.size();
  if (r == 0 && cap < 2 + 9 * n) {
    set_last_error("test_weight_table: cap %d < %d (2 + 9 per conv)", cap, 2 + 9 * n);
    r = 2;
  }
  if (r == 0) {
    out[0] = n;
    out[1] = spec->wk_total;
    for (int i = 0; i < n; ++i) {
      const WeightDesc& d = spec->convs[i].wd;
      const int64_t row[9] = {d.p_off, d.k_off, d.Co, d.Ci, d.Ci_real, d.KH, d.KW, d.im2col_k, d.s2d};
      for (int k = 0; k < 9; ++k) out[2 + 9 * i + k] = row[k];
    }
  }
  spec->destroy();
  delete spec;
  return r;
}

// The production pack of one precision: Net::forward_t's (fp32, bf16_simt, bf16, tc_split with its dgrad planes) or
// InferNet::load's fp8 pair, over the descriptors of a parameter-table-only trunk.
int mapnet_test_pack_weights(int precision, int im2col_stem, int H, int W, const float* params_flat, void* krsc_out, void* dg_out,
                             float* s_w_out, void* stream) {
  MN_CHECK(params_flat && krsc_out && dg_out, "test_pack_weights: null argument");
  MN_CHECK((s_w_out != nullptr) == (precision == PREC_FP8), "test_pack_weights: s_w_out is given exactly for fp8 "
           "(precision %d)", precision);
  Net* spec = new Net();
  int r = pack_spec(spec, H, W, precision, im2col_stem, "test_pack_weights");
  WeightDesc* d_wd = nullptr;
  float* f32 = nullptr;
  auto body = [&]() -> int {
    MN_TRY(require_device());
    for (const void* p : {(const void*)params_flat, (const void*)krsc_out, (const void*)dg_out, (const void*)s_w_out}) {
      if (p == nullptr) continue;
      cudaPointerAttributes at;
      MN_CUDA(cudaPointerGetAttributes(&at, p));
      MN_CHECK(at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged,
               "test_pack_weights: params_flat and the outputs must be device memory");
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int nconv = (int)spec->convs.size();
    const long long wk = spec->wk_total;
    std::vector<WeightDesc> wd;
    for (auto& c : spec->convs) wd.push_back(c.wd);
    MN_CUDA(cudaMalloc((void**)&d_wd, wd.size() * sizeof(WeightDesc)));
    MN_CUDA(cudaMemcpy(d_wd, wd.data(), wd.size() * sizeof(WeightDesc), cudaMemcpyHostToDevice));
    if (precision == PREC_FP32 || precision == PREC_BF16_SIMT) {
      MN_TRY(launch_pack_weights<float>(d_wd, nconv, params_flat, (float*)krsc_out, (float*)dg_out, spec->max_w_elems,
                                        precision == PREC_BF16_SIMT, st));
    } else if (precision == PREC_BF16_TC) {
      MN_TRY(launch_pack_weights<bf16>(d_wd, nconv, params_flat, (bf16*)krsc_out, (bf16*)dg_out, spec->max_w_elems, 0, st));
    } else if (precision == PREC_TC_SPLIT) {
      MN_CUDA(cudaMalloc((void**)&f32, (size_t)wk * 2 * sizeof(float)));     // the fp32 K-major matrices (Net's w_*_f32)
      MN_TRY(launch_pack_weights_split(d_wd, nconv, params_flat, f32, f32 + wk, krsc_out, dg_out, spec->max_w_elems, st));
    } else {
      MN_TRY(launch_pack_weights<bf16>(d_wd, 1, params_flat, (bf16*)dg_out, nullptr, spec->max_w_elems, 0, st));
      MN_TRY(launch_pack_weights_fp8(d_wd, nconv, params_flat, (uint8_t*)krsc_out, s_w_out, st));
    }
    MN_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  if (r == 0) r = body();
  cudaFree(f32);
  cudaFree(d_wd);
  spec->destroy();
  delete spec;
  return r;
}

// The stem operand of the inference engine from one of its two sources: uint8 frames through pre (the fused vertical
// pass), or float32 images of pre's output size through k_stem_s2d (what mapnet_infer_forward writes).
int mapnet_test_stem_operand(int precision, mapnet_preprocess_t* pre, const void* frames_nhwc_u8, const float* x_nchw,
                             int B, const float* mean3, const float* std3, void* S, void* stream) {
  MN_CHECK(precision == PREC_BF16_TC || precision == PREC_TC_SPLIT || precision == PREC_FP8,
           "test_stem_operand: precision %d has no space-to-depth stem operand", precision);
  MN_CHECK(pre != nullptr && S != nullptr && (frames_nhwc_u8 == nullptr) != (x_nchw == nullptr),
           "test_stem_operand: need pre, S and exactly one of frames / x");
  int H = 0, W = 0, max_images = 0;
  MN_TRY(preprocess_geometry(pre, &H, &W, &max_images));
  const int hc = (H - 1) / 2 + 1, Hs = hc + 3, Wsp = stem_s2d_wsp((W - 1) / 2 + 1);
  cudaStream_t st = (cudaStream_t)stream;
  const bool sp = precision == PREC_TC_SPLIT;
  if (frames_nhwc_u8 != nullptr) {
    const uint8_t* f = (const uint8_t*)frames_nhwc_u8;
    return sp ? preprocess_stem_s2d<hsplit>(pre, f, B, mean3, std3, (hsplit*)S, Hs, Wsp, st)
              : preprocess_stem_s2d<bf16>(pre, f, B, mean3, std3, (bf16*)S, Hs, Wsp, st);
  }
  MN_CHECK(B >= 1, "test_stem_operand: batch %d", B);
  return sp ? launch_stem_s2d<hsplit>(x_nchw, (hsplit*)S, B, H, W, Hs, Wsp, st)
            : launch_stem_s2d<bf16>(x_nchw, (bf16*)S, B, H, W, Hs, Wsp, st);
}

int mapnet_infer_calibrate(mapnet_infer_t* h, const float* x, int B, void* stream) {
  MN_CHECK(h != nullptr, "infer_calibrate: null handle");
  return h->net.calibrate(x, B, (cudaStream_t)stream);
}

int mapnet_infer_act_scales(mapnet_infer_t* h, float* host_out, int cap) {
  MN_CHECK(h != nullptr, "infer_act_scales: null handle");
  const int r = h->net.act_scales(host_out, cap, nullptr);
  return r < 0 ? r : 0;
}

int mapnet_infer_destroy(mapnet_infer_t* h) {
  if (h == nullptr) return 0;
  h->net.destroy();
  delete h;
  return 0;
}

// wgrad of one stride-1 (or any) conv on a chosen engine, keeping the plan's K partition: taps -1 = the planner's
// choice, 0 = the per-tap engine, 3 / 9 = the halo engine with that many filter taps per CTA at N tile bn.  dw is
// accumulated onto (one split) or has the splits' sum added to it, as in the training step.  iters 0: one run;
// iters > 0: 3 warm-up runs, then the average ms of `iters` runs into *host_ms (tools/bench_conv.py)
int mapnet_test_wgrad(int taps, int bn, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, const void* x,
                      const void* dy, void* dw, int iters, float* host_ms) {
  MN_TRY(require_device());
  ConvGeom g;
  g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
  g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  TcConvPlan* plan = nullptr;
  MN_TRY(tc_plan_create(&plan, g, 2, nullptr));
  cudaStream_t st = 0;
  int r = taps >= 0 ? tc_plan_force_wgrad(plan, taps, bn) : 0;
  auto run = [&]() { return tc_conv_run(plan, (const bf16*)x, (const bf16*)dy, nullptr, dw, st); };
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (r == 0 && iters <= 0) r = run();
  if (r == 0 && iters > 0) {
    for (int i = 0; i < 3 && r == 0; ++i) r = run();
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0, st);
    for (int i = 0; i < iters && r == 0; ++i) r = run();
    cudaEventRecord(e1, st);
  }
  const cudaError_t e = cudaStreamSynchronize(st);
  if (r == 0 && e != cudaSuccess) { set_last_error("test_wgrad: %s", cudaGetErrorString(e)); r = 1; }
  if (r == 0 && iters > 0 && host_ms != nullptr) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    *host_ms = ms / iters;
  }
  if (e0) cudaEventDestroy(e0);
  if (e1) cudaEventDestroy(e1);
  tc_plan_destroy(plan);
  return r;
}

// micro-benchmark of one wgmma conv launch configuration (plan built once, CUDA-event timing)
int mapnet_bench_conv(int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, const void* in0,
                      const void* in1, const void* wmat, void* out, int iters, float* host_ms) {
  MN_TRY(require_device());
  ConvGeom g;
  g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
  g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  TcConvPlan* plan = nullptr;
  MN_TRY(tc_plan_create(&plan, g, kind, (const bf16*)wmat));
  cudaStream_t st = 0;
  int r = 0;
  // MAPNET_BENCH_EPI=1: the epilogue variants the training step really runs -- fprop with the fused BatchNorm
  // statistics, dgrad with the ReLU gate + BatchNorm-backward sums (gate tensor and Y = the input operand's
  // sibling buffers; the values are irrelevant for timing); =2 additionally isolates each launch with an event
  // record (what bench.py's per-conv brackets do: no programmatic overlap with the neighbours)
  static int epi = -1;
  if (epi < 0) { const char* e = getenv("MAPNET_BENCH_EPI"); epi = e ? atoi(e) : 0; }
  double* stats = nullptr;
  EpiBwd E; memset(&E, 0, sizeof(E));
  const bf16* res = nullptr;
  if (epi && kind != 2) {
    if (cudaMalloc((void**)&stats, kBnAccReplicas * kBnAccStride * sizeof(double)) != cudaSuccess) { set_last_error("bench_conv: cudaMalloc"); tc_plan_destroy(plan); return 1; }
    cudaMemset(stats, 0, kBnAccReplicas * kBnAccStride * sizeof(double));
    if (kind == 1) { E.y = (const bf16*)out; E.zmask = (const bf16*)out; res = (const bf16*)out; }   // shaped like the output
  }
  cudaEvent_t iso;
  cudaEventCreate(&iso);
  auto run = [&]() {
    int rc = tc_conv_run(plan, (const bf16*)in0, (const bf16*)in1, res, out, st, stats, (kind == 1 && stats) ? &E : nullptr);
    if (epi == 2) cudaEventRecord(iso, st);
    return rc;
  };
  for (int i = 0; i < 3 && r == 0; ++i) r = run();
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0, st);
  for (int i = 0; i < iters && r == 0; ++i) r = run();
  cudaEventRecord(e1, st);
  cudaError_t e = cudaEventSynchronize(e1);
  if (r == 0 && e != cudaSuccess) { set_last_error("bench_conv: %s", cudaGetErrorString(e)); r = 1; }
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  if (host_ms) *host_ms = ms / (iters > 0 ? iters : 1);
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(iso);
  if (stats) cudaFree(stats);
  tc_plan_destroy(plan);
  return r;
}

}  // extern "C"
