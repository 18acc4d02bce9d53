// extern "C" entry points declared in include/mapnet_b200.h.
#include <math.h>

#include <vector>

#include "../../include/mapnet_b200.h"
#include "net.h"

using namespace mapnet;

struct mapnet_trunk { Net net; };

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
  if (precision == PREC_TC_SPLIT) {
    // strict tensor-core mode: fp32 NHWC tensors and fp32 K-major weight matrices in (as for PREC_FP32), fp32 out;
    // the operands are cut into fp16 hi / lo planes here (the training step's element-wise kernels write that form)
    g.split = 1; g.fmt_z = 0; g.fmt_g = 0;
    const long long n_in = (long long)B * Hi * Wi * Ci, n_out = (long long)B * g.Ho * g.Wo * Co;
    const int KK = k * k;
    void *s0 = nullptr, *s1 = nullptr, *sw = nullptr;
    TcConvPlan* plan = nullptr;
    auto body = [&]() -> int {
      const long long n0 = (kind == 1) ? n_out : n_in;
      MN_CUDA(cudaMalloc(&s0, (size_t)n0 * 4));
      MN_TRY(launch_split_tensor((const float*)in0, s0, n0, 0, st));
      if (kind == 2) {
        MN_CUDA(cudaMalloc(&s1, (size_t)n_out * 4));
        MN_TRY(launch_split_tensor((const float*)in1, s1, n_out, 0, st));
      } else {
        MN_CUDA(cudaMalloc(&sw, (size_t)Co * KK * Ci * 8));
        if (kind == 0) MN_TRY(launch_split_weight_matrix((const float*)wmat, sw, Co, KK, Ci, 0, st));
        else MN_TRY(launch_split_weight_matrix((const float*)wmat, sw, Ci, KK, Co, 0, st));
      }
      MN_TRY(tc_plan_create(&plan, g, kind, (const bf16*)sw));
      MN_TRY(tc_conv_run(plan, (const bf16*)s0, (const bf16*)s1, nullptr, out, st));
      MN_CUDA(cudaStreamSynchronize(st));
      return 0;
    };
    const int r = body();
    if (plan) tc_plan_destroy(plan);
    cudaFree(s0); cudaFree(s1); cudaFree(sw);
    return r;
  }
  MN_CHECK(precision == PREC_BF16_TC, "test_conv: bad precision");
  TcConvPlan* plan = nullptr;
  MN_TRY(tc_plan_create(&plan, g, kind, (const bf16*)wmat));
  int r = tc_conv_run(plan, (const bf16*)in0, (const bf16*)in1, nullptr, out, st);
  if (r == 0) { cudaError_t e = cudaStreamSynchronize(st); if (e != cudaSuccess) { set_last_error("test_conv: %s", cudaGetErrorString(e)); r = 1; } }
  tc_plan_destroy(plan);
  return r;
}

// JSON description of the plan the tensor-core engines would use for this conv (no device needed)
int mapnet_test_plan_describe(int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, int with_shortcut,
                              char* buf, int cap) {
  ConvGeom g;
  g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Co = Co; g.KH = g.KW = k; g.stride = stride; g.pad = (k - 1) / 2;
  g.Ho = (Hi + 2 * g.pad - k) / stride + 1; g.Wo = (Wi + 2 * g.pad - k) / stride + 1;
  TcConvPlan* plan = nullptr;
  static const bf16 dummy[8] = {};
  MN_TRY(tc_plan_create(&plan, g, kind, dummy));
  int r = 0;
  if (with_shortcut) r = tc_plan_add_shortcut(plan, dummy);
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
  const size_t acc_doubles = 32 * 3 * 512;
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
        for (int rep = 0; rep < 32; ++rep) s += h[(size_t)rep * 3 * 512 + (size_t)j * C + c];
        host_sums[(size_t)j * C + c] = s;
      }
  if (plan) tc_plan_destroy(plan);
  cudaFree(acc);
  return r;
}

// the tensor-core stem alone: space-to-depth image -> packed weights -> fprop [-> wgrad -> .grad layout]
int mapnet_test_stem(int B, int H, int W, const float* x_nchw, const float* w_oihw, void* y_out, const void* dy,
                     float* dw_oihw, void* stream) {
  MN_TRY(require_device());
  MN_CHECK(B >= 1 && H >= 32 && W >= 32 && x_nchw && w_oihw && y_out, "test_stem: bad argument");
  MN_CHECK(tc_overlapped_view_supported(), "test_stem: the driver rejects overlapped tensor maps");
  cudaStream_t st = (cudaStream_t)stream;
  ConvGeom g; WeightDesc wd; memset(&wd, 0, sizeof(wd));
  stem_s2d_geometry(H, W, 64, &g, &wd);
  g.B = B; wd.p_off = 0; wd.k_off = 0;
  const int Hs = g.Hi, Wsp = stem_s2d_wsp(g.Wo);
  bf16 *S = nullptr, *wk = nullptr; float* dwk = nullptr; WeightDesc* d_wd = nullptr;
  TcConvPlan *pf = nullptr, *pw = nullptr;
  int r = 0;
  auto body = [&]() -> int {
    MN_CUDA(cudaMalloc(&S, (size_t)B * Hs * Wsp * 16 * sizeof(bf16)));
    MN_CUDA(cudaMalloc(&wk, (size_t)64 * 256 * sizeof(bf16)));
    MN_CUDA(cudaMalloc(&dwk, (size_t)64 * 256 * sizeof(float)));
    MN_CUDA(cudaMalloc(&d_wd, sizeof(WeightDesc)));
    MN_CUDA(cudaMemcpyAsync(d_wd, &wd, sizeof(wd), cudaMemcpyHostToDevice, st));
    MN_CUDA(cudaMemsetAsync(dwk, 0, (size_t)64 * 256 * sizeof(float), st));
    MN_TRY(launch_stem_s2d<bf16>(x_nchw, S, B, H, W, Hs, Wsp, st));
    MN_TRY(launch_pack_weights<bf16>(d_wd, 1, w_oihw, wk, nullptr, 64 * 256, 0, st));
    MN_TRY(tc_plan_create(&pf, g, 0, wk));
    MN_TRY(tc_conv_run(pf, S, nullptr, nullptr, y_out, st));
    if (dy != nullptr && dw_oihw != nullptr) {
      MN_TRY(tc_plan_create(&pw, g, 2, nullptr));
      MN_TRY(tc_conv_run(pw, S, (const bf16*)dy, nullptr, dwk, st));
      MN_TRY(launch_unpack_wgrads(d_wd, 1, dwk, dw_oihw, 64 * 256, st));
    }
    MN_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  r = body();
  if (pf) tc_plan_destroy(pf);
  if (pw) tc_plan_destroy(pw);
  cudaFree(S); cudaFree(wk); cudaFree(dwk); cudaFree(d_wd);
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
    if (cudaMalloc((void**)&stats, 32 * 3 * 512 * sizeof(double)) != cudaSuccess) { set_last_error("bench_conv: cudaMalloc"); tc_plan_destroy(plan); return 1; }
    cudaMemset(stats, 0, 32 * 3 * 512 * sizeof(double));
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
