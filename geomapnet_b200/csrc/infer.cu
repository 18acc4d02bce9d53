// Eval-mode PoseNet(ResNet-34) inference: a frozen snapshot replayed through the wgmma fprop engine.
//
// In the forward of an eval-mode ResNet every BatchNorm is a fixed per-channel affine map, so each conv's epilogue
// applies it to the fp32 accumulator, adds the residual, applies the ReLU and rounds once at the store (conv_tc.cu,
// EPI_AFFINE).  Compared with the live eval forward (Net::forward_t with training = 0) there is no per-call weight pack,
// no dgrad operand, no BatchNorm launch, no separate apply pass, no stem argmax and no training arena: one launch per
// conv, plus the stem operand, the pool and the head (docs: DESIGN.md section 7).
//
// The schedule shares Net's parameter table and layer geometry (a spec-only Net, max_B = 0) and owns its resources:
// the packed fprop operands, a per-channel scale / shift table computed by the same k_bn_eval_scale the live eval
// forward runs, an fp32 copy of the head and an activation arena that holds only the live set of one block.
//
// fp8 (PREC_FP8): the stem conv stays on the bf16 engine; the pool output and every block's h and output are e4m3, each
// with one power-of-two scale, and every other conv runs k_f8_conv on e4m3 weights with a power-of-two scale per output
// channel.  Its epilogue applies S[c] = bn_scale[c] * s_in * s_w[c] (exact: powers of two), adds the residual (e4m3 *
// s_res, or the bf16 downsample output), applies the ReLU and stores e4m3(f / s_out).  The activation scales come from
// calibration over the engine's own schedule (calibrate): each tensor's scale is taken from the values its epilogue
// would quantize with every earlier tensor already quantized, so a CPU emulation with the same scales reproduces the
// engine's rounding points.
#include "infer.h"

#include <math.h>

#include <string.h>

namespace mapnet {

static long long align_up(long long v, long long a) { return (v + a - 1) / a * a; }

int InferNet::alloc(void** p, size_t bytes) {
  if (bytes == 0) bytes = 16;
  MN_CUDA(cudaMalloc(p, align_up((long long)bytes, 256)));
  allocs.push_back(*p);
  return 0;
}

// ---- fp8 calibration kernels (one launch each per tensor, at calibration time only) ----
// max |y| of a bf16 tensor into *amax (bit pattern): the stem output, whose max is the pool output's (every stem pixel
// lies in some pooling window, and max pooling keeps the largest value)
__global__ void k_f8_amax_bf16(const bf16* __restrict__ y, long long n8, unsigned int* __restrict__ amax) {
  pdl_prologue();
  float m = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    Vec8<bf16> v; v.load(y + 8 * i);
#pragma unroll
    for (int k = 0; k < 8; ++k) m = fmaxf(m, fabsf(v.v[k]));
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) atomicMax(amax, __float_as_uint(m));
}
// tensor t's scale from its amax: slots[n + t] = s, slots[2n + t] = 1 / s; fill[0..nfill) = 1 / s (the pool's map)
__global__ void k_f8_set_scale(float* __restrict__ slots, int n, int t, float* __restrict__ fill, int nfill) {
  pdl_prologue();
  const float s = f8_pow2_scale(__uint_as_float(reinterpret_cast<const unsigned int*>(slots)[t]));
  if (threadIdx.x == 0) { slots[n + t] = s; slots[2 * n + t] = 1.f / s; }
  for (int i = threadIdx.x; i < nfill; i += blockDim.x) fill[i] = 1.f / s;
}
// the epilogue table of one conv: S[c] = bn_scale[c] * s_in * s_w[c] (two power-of-two factors: exact)
__global__ void k_f8_fold(const float* __restrict__ bn_scale, const float* __restrict__ s_w, const float* __restrict__ s_in,
                          float* __restrict__ S, int C) {
  pdl_prologue();
  for (int c = threadIdx.x; c < C; c += blockDim.x) S[c] = bn_scale[c] * __ldg(s_in) * s_w[c];
}

int InferNet::sizes(const Net& n, int precision, Sizes* s) {
  const bool f8 = precision == PREC_FP8;
  const long long ez = (n.precision == PREC_TC_SPLIT) ? 4 : 2;       // operand element (bf16 / hi+lo fp16 planes)
  const long long ea = (n.precision == PREC_TC_SPLIT) ? 4 : 2;       // conv output element (bf16 / fp32)
  const long long eb = f8 ? 1 : ez;                                   // block tensors (fp8: e4m3)
  const ConvGeom& g0 = n.convs[0].g;
  s->a0 = n.stem_s2d ? (long long)g0.Hi * stem_s2d_wsp(n.Wc) * 16 * ez : (long long)n.Hc * n.Wc * g0.Ci * ez;
  s->y0 = (long long)n.Hc * n.Wc * 64 * ea;
  long long act = (long long)n.Hp * n.Wp * 64, ds = 0;
  for (const BlockL& b : n.blocks) {
    const long long e = (long long)b.Ho * b.Wo * b.Cout;
    if (e > act) act = e;
    if (b.convd >= 0 && e > ds) ds = e;
  }
  s->act = act * eb;
  s->ds = ds * ea;
  s->head = (512 + 3LL * n.feat_dim) * 4;     // feat, fc output (pre-ReLU and dropped), dropout mask
  return 0;
}

long long InferNet::arena_bytes(int max_B, int H, int W, int precision) {
  if (precision != PREC_BF16_TC && precision != PREC_TC_SPLIT && precision != PREC_FP8) {
    set_last_error("infer: precision %d is not supported (bf16 = %d, tc_split = %d or fp8 = %d)", precision, PREC_BF16_TC,
                   PREC_TC_SPLIT, PREC_FP8);
    return -2;
  }
  if (max_B < 1 || H < 32 || W < 32) { set_last_error("infer: need max_B >= 1 and H, W >= 32 (got %d, %d, %d)", max_B, H, W); return -2; }
  Net n = Net();
  if (n.init(0, H, W, 2048, precision == PREC_FP8 ? PREC_BF16_TC : precision) != 0) return -2;
  Sizes s;
  sizes(n, precision, &s);
  const long long slots = precision == PREC_FP8 ? f8_slot_bytes(n) : 0;
  n.destroy();
  return (long long)max_B * (s.a0 + s.y0 + 3 * s.act + s.ds + s.head) + slots;
}

int InferNet::init(int max_B_, int H_, int W_, int feat_dim_, int precision_) {
  max_B = max_B_; H = H_; W = W_; feat_dim = feat_dim_; precision = precision_;
  loaded = false; calibrated = false; plan_B = 0;
  wk = nullptr; d_wdescs = nullptr; affine = head = ident = eval_scratch = nullptr;
  wk8 = nullptr; s_w = f8_table = pool_map = f8_slots = nullptr; n_f8 = 0;
  A0 = y0 = ds = nullptr; act[0] = act[1] = act[2] = nullptr;
  feat = fcpre = hdrop = mask = nullptr; drop_ctr = nullptr;
  const bool f8 = precision == PREC_FP8;
  MN_CHECK(precision == PREC_BF16_TC || precision == PREC_TC_SPLIT || f8,
           "infer_create: precision %d is not supported (bf16 = %d, tc_split = %d or fp8 = %d)", precision, PREC_BF16_TC,
           PREC_TC_SPLIT, PREC_FP8);
  MN_CHECK(max_B >= 1 && H >= 32 && W >= 32, "infer_create: need max_B >= 1 and H, W >= 32 (got %d, %d, %d)", max_B, H, W);
  MN_TRY(spec.init(0, H, W, feat_dim, f8 ? PREC_BF16_TC : precision));     // fp8: the stem's operands are bf16
  MN_CHECK(!spec.stem_s2d || tc_overlapped_view_supported(),
           "infer_create: the driver rejects the overlapped tensor map of the space-to-depth stem");
  Sizes s;
  sizes(spec, precision, &s);
  const long long Bm = max_B;
  MN_TRY(alloc(&A0, (size_t)(Bm * s.a0)));
  MN_TRY(alloc(&y0, (size_t)(Bm * s.y0)));
  for (int i = 0; i < 3; ++i) MN_TRY(alloc(&act[i], (size_t)(Bm * s.act)));
  MN_TRY(alloc(&ds, (size_t)(Bm * s.ds)));
  MN_TRY(alloc((void**)&feat, (size_t)Bm * 512 * 4));
  MN_TRY(alloc((void**)&fcpre, (size_t)Bm * feat_dim * 4));
  MN_TRY(alloc((void**)&hdrop, (size_t)Bm * feat_dim * 4));
  MN_TRY(alloc((void**)&mask, (size_t)Bm * feat_dim * 4));
  // snapshot storage
  if (f8) {
    const int nconv = (int)spec.convs.size();
    MN_CHECK(spec.convs[0].wd.k_off == 0, "infer_create: the stem's packed weights must come first");
    MN_TRY(alloc(&wk, (size_t)spec.convs[1].wd.k_off * 2));            // the stem's bf16 operand only
    MN_TRY(alloc((void**)&wk8, (size_t)spec.wk_total));
    MN_TRY(alloc((void**)&s_w, (size_t)nconv * 512 * 4));
    MN_TRY(alloc((void**)&f8_table, (size_t)nconv * 512 * 4));
    n_f8 = f8_tensors(spec);
    MN_TRY(alloc((void**)&pool_map, (size_t)f8_slot_bytes(spec)));
    MN_CUDA(cudaMemset(pool_map, 0, (size_t)f8_slot_bytes(spec)));
    f8_slots = pool_map + 128;
  } else {
    MN_TRY(alloc(&wk, (size_t)spec.wk_total * (precision == PREC_TC_SPLIT ? 8 : 2)));
  }
  std::vector<WeightDesc> wd;
  for (auto& c : spec.convs) wd.push_back(c.wd);
  MN_TRY(alloc((void**)&d_wdescs, wd.size() * sizeof(WeightDesc)));
  MN_CUDA(cudaMemcpy(d_wdescs, wd.data(), wd.size() * sizeof(WeightDesc), cudaMemcpyHostToDevice));
  long long nf = 0;
  for (auto& b : spec.bns) nf += 2LL * b.C;
  MN_TRY(alloc((void**)&affine, (size_t)nf * 4));
  float* p = affine;
  for (auto& b : spec.bns) { bn_scale.push_back(p); p += b.C; bn_shift.push_back(p); p += b.C; }
  MN_TRY(alloc((void**)&head, (size_t)(spec.wpqr_b + 3 - spec.fc_w) * 4));
  MN_TRY(alloc((void**)&ident, 128 * 4));
  { float h[128]; for (int i = 0; i < 128; ++i) h[i] = i < 64 ? 1.f : 0.f;
    MN_CUDA(cudaMemcpy(ident, h, sizeof(h), cudaMemcpyHostToDevice)); }
  MN_TRY(alloc((void**)&eval_scratch, 2 * 512 * 4));
  MN_TRY(alloc((void**)&drop_ctr, 16));
  MN_CUDA(cudaMemset(drop_ctr, 0, 16));
  return 0;
}

void InferNet::destroy() {
  for (auto* p : plans) tc_plan_destroy(p);
  plans.clear();
  for (void* p : allocs) cudaFree(p);
  allocs.clear();
  spec.destroy();
  loaded = false;
}

// Snapshot: the packed fprop operands, the eval-mode scale / shift of every BatchNorm and the head.  Nothing here is
// read from params / bufs again.
int InferNet::load(const float* params, const float* bufs, cudaStream_t st) {
  MN_CHECK(params != nullptr && bufs != nullptr, "infer_load: null pointer argument");
  for (const float* p : {params, bufs}) {       // the snapshot is read by kernels: refuse host memory before a launch
    cudaPointerAttributes at;
    MN_CUDA(cudaPointerGetAttributes(&at, p));
    MN_CHECK(at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged,
             "infer_load: params_flat / bufs_flat must be device memory");
  }
  const int nconv = (int)spec.convs.size();
  calibrated = false;          // fp8: the activation scales belong to the previous weights
  if (precision == PREC_FP8) {
    MN_TRY(launch_pack_weights<bf16>(d_wdescs, 1, params, (bf16*)wk, nullptr, spec.max_w_elems, 0, st));   // the stem
    MN_TRY(launch_pack_weights_fp8(d_wdescs, nconv, params, wk8, s_w, st));
  } else if (precision == PREC_BF16_TC) {
    MN_TRY(launch_pack_weights<bf16>(d_wdescs, nconv, params, (bf16*)wk, nullptr, spec.max_w_elems, 0, st));
  } else {
    float* f32 = nullptr;       // the fp32 K-major matrices the hi / lo planes are cut from (load time only)
    MN_CUDA(cudaMallocAsync((void**)&f32, (size_t)spec.wk_total * 4, st));
    const int r = launch_pack_weights_split(d_wdescs, nconv, params, f32, nullptr, wk, nullptr, spec.max_w_elems, st);
    MN_CUDA(cudaFreeAsync(f32, st));
    MN_TRY(r);
  }
  for (size_t i = 0; i < spec.bns.size(); ++i) {
    const BNL& b = spec.bns[i];
    // the arithmetic of the live eval forward (running statistics are only read)
    BnFin f; memset(&f, 0, sizeof(f));
    f.gamma = params + b.g_off; f.beta = params + b.b_off;
    f.run_mean = const_cast<float*>(bufs + b.rm_off); f.run_var = const_cast<float*>(bufs + b.rv_off);
    f.mean = eval_scratch; f.invstd = eval_scratch + 512; f.scale = bn_scale[i]; f.shift = bn_shift[i];
    MN_TRY(launch_bn_eval_scale(b.C, f, st));
  }
  MN_CUDA(cudaMemcpyAsync(head, params + spec.fc_w, (size_t)(spec.wpqr_b + 3 - spec.fc_w) * 4, cudaMemcpyDeviceToDevice, st));
  loaded = true;
  return 0;
}

int InferNet::ensure_plans(int B) {
  if (plan_B == B) return 0;
  for (auto* p : plans) tc_plan_destroy(p);
  plans.assign(spec.convs.size(), nullptr);
  const bool sp = precision == PREC_TC_SPLIT;
  for (size_t i = 0; i < spec.convs.size(); ++i) {
    ConvGeom g = spec.convs[i].g; g.B = B;
    if (sp) g.split = 1;
    if (precision == PREC_FP8 && i > 0) {
      MN_TRY(tc_plan_create_f8(&plans[i], g, wk8 + spec.convs[i].wd.k_off));
      continue;
    }
    const bf16* w = (const bf16*)wk + (sp ? 4 : 1) * spec.convs[i].wd.k_off;
    MN_TRY(tc_plan_create(&plans[i], g, 0, w));
  }
  plan_B = B;
  return 0;
}

int InferNet::conv(int ci, const void* in, const void* residual, void* out, int relu, int res_split, int out_split,
                   cudaStream_t st) {
  const int bi = spec.convs[ci].bn;
  EpiAffine a;
  a.scale = bn_scale[bi]; a.shift = bn_shift[bi]; a.relu = relu; a.res_split = res_split; a.out_split = out_split;
  return tc_conv_run(plans[ci], (const bf16*)in, nullptr, (const bf16*)residual, out, st, nullptr, nullptr, &a);
}

// the stem operand A0 of frames x [B,3,H,W]: the space-to-depth image (or the im2col matrix), in the stem's operand type
int InferNet::stem_operand(const float* x, int B, cudaStream_t st) {
  const Net& n = spec;
  if (precision == PREC_TC_SPLIT) {
    if (n.stem_s2d) return launch_stem_s2d<hsplit>(x, (hsplit*)A0, B, H, W, n.convs[0].g.Hi, stem_s2d_wsp(n.Wc), st);
    return launch_stem_im2col<hsplit>(x, (hsplit*)A0, B, H, W, n.Hc, n.Wc, n.convs[0].g.Ci, st);
  }
  if (n.stem_s2d) return launch_stem_s2d<bf16>(x, (bf16*)A0, B, H, W, n.convs[0].g.Hi, stem_s2d_wsp(n.Wc), st);
  return launch_stem_im2col<bf16>(x, (bf16*)A0, B, H, W, n.Hc, n.Wc, n.convs[0].g.Ci, st);
}

// everything after the stem operand: stem conv .. head
int InferNet::trunk(int B, float droprate, unsigned long long seed, unsigned long long step, float* pred, cudaStream_t st) {
  MN_TRY(features(B, st));
  return run_head(B, droprate, seed, step, pred, st);
}

// stem conv .. global average pool: feat [B,512]
int InferNet::features(int B, cudaStream_t st) {
  if (precision == PREC_FP8) {
    int last = 0;
    MN_TRY(run_f8(B, false, &last, st));
    return launch_gap<e4m3>((const e4m3*)act[last], feat, B, spec.Hf * spec.Wf, 512, st, f8_slots + 2 * n_f8 - 1);
  }
  if (precision == PREC_TC_SPLIT) return forward_t<TypesSplitHH>(B, st);
  return forward_t<TypesBF16>(B, st);
}

template <typename P>
int InferNet::forward_t(int B, cudaStream_t st) {
  typedef typename P::A T;        // stem / downsample conv outputs (bf16, or fp32 in strict mode)
  typedef typename P::Z TZ;       // conv operands (bf16, or fp16 hi/lo planes)
  const int sp = (precision == PREC_TC_SPLIT) ? 1 : 0;
  const Net& n = spec;
  MN_TRY(ensure_plans(B));
  // stem: operand image (A0, already written) -> conv + BN + ReLU (epilogue) -> 3x3/s2 max pool
  MN_TRY(conv(0, A0, nullptr, y0, 1, 0, 0, st));
  BnDesc id; memset(&id, 0, sizeof(id));        // the stem's BatchNorm and ReLU are in the conv epilogue: identity map
  id.f.scale = ident; id.f.shift = ident + 64;
  MN_TRY((launch_stem_pool<T, TZ>((const T*)y0, (TZ*)act[0], nullptr, B, n.Hc, n.Wc, n.Hp, n.Wp, 64, id, st)));
  // blocks: (input, h, output) rotate through the three arena tensors
  int xi = 0;
  for (const BlockL& bl : n.blocks) {
    void* xin = act[xi];
    void* h = act[(xi + 1) % 3];
    void* out = act[(xi + 2) % 3];
    MN_TRY(conv(bl.conv1, xin, nullptr, h, 1, 0, sp, st));
    if (bl.convd >= 0) {
      MN_TRY(conv(bl.convd, xin, nullptr, ds, 0, 0, 0, st));
      MN_TRY(conv(bl.conv2, h, ds, out, 1, 0, sp, st));
    } else {
      MN_TRY(conv(bl.conv2, h, xin, out, 1, sp, sp, st));
    }
    xi = (xi + 2) % 3;
  }
  return launch_gap<TZ>((const TZ*)act[xi], feat, B, n.Hf * n.Wf, 512, st);
}

// head on feat: exactly the calls of Net::forward_t, on the snapshot's copy of the head parameters
int InferNet::run_head(int B, float droprate, unsigned long long seed, unsigned long long step, float* pred,
                       cudaStream_t st) {
  const Net& n = spec;
  const float* hp = head - n.fc_w;      // indexed with the flat-buffer offsets
  return head_forward(n.head_params(hp), feat, B, feat_dim, droprate, seed, step, drop_ctr,
                      (unsigned long long)max_B * feat_dim, mask, fcpre, hdrop, pred, st);
}

// S Monte-Carlo dropout draws of the head on feat: the fc product once, without a mask (fcpre is the same for every
// draw), then launch_head_sample, which forms every draw's mask and products in run_head's order (head.cu)
int InferNet::sample_head(int B, int S, float droprate, unsigned long long seed, unsigned long long step, float* samples,
                          double* mean, double* cov, cudaStream_t st) {
  const Net& n = spec;
  const float* hp = head - n.fc_w;
  MN_TRY(launch_small_gemm(1, feat, 512, 1, hp + n.fc_w, 512, 1, hdrop, feat_dim, B, feat_dim, 512, hp + n.fc_b, fcpre,
                           nullptr, st));
  const bool dev_ctr = (step == ~0ULL);
  return launch_head_sample(fcpre, B, feat_dim, hp + n.xyz_w, hp + n.xyz_b, hp + n.wpqr_w, hp + n.wpqr_b, S, droprate,
                            seed, dev_ctr ? 0ULL : step, dev_ctr ? drop_ctr : nullptr,
                            (unsigned long long)max_B * feat_dim, samples, mean, cov, st);
}

// the checks shared by sample and sample_frames (before any launch)
int InferNet::check_sample(const char* what, int S, float droprate, const double* mean, const double* cov) const {
  MN_CHECK(S >= 2 && S <= kMaxSampleDraws, "%s: S = %d draws outside [2, %d]", what, S, kMaxSampleDraws);
  MN_CHECK(droprate > 0.f && droprate < 1.f, "%s: droprate %f outside (0,1): without dropout every draw is the same pose",
           what, droprate);
  MN_CHECK(mean != nullptr && cov != nullptr, "%s: null pointer argument", what);
  MN_CHECK(head_sample_smem(max_B, feat_dim, S) <= 48 * 1024, "%s: feat_dim %d is too large for the draw kernel", what,
           feat_dim);
  return 0;
}

int InferNet::sample(const float* x, int B, int S, float droprate, unsigned long long seed, unsigned long long step,
                     float* samples, double* mean, double* cov, cudaStream_t st) {
  MN_CHECK(loaded, "infer_sample: no snapshot loaded (call mapnet_infer_load first)");
  MN_CHECK(precision != PREC_FP8 || calibrated,
           "infer_sample: the fp8 engine has no activation scales for this snapshot (call mapnet_infer_calibrate)");
  MN_CHECK(B >= 1 && B <= max_B, "infer_sample: batch %d outside [1, max_B=%d]", B, max_B);
  MN_CHECK(x != nullptr, "infer_sample: null pointer argument");
  MN_TRY(check_sample("infer_sample", S, droprate, mean, cov));
  MN_TRY(ensure_plans(B));
  MN_TRY(stem_operand(x, B, st));
  MN_TRY(features(B, st));
  return sample_head(B, S, droprate, seed, step, samples, mean, cov, st);
}

int InferNet::forward(const float* x, int B, float droprate, unsigned long long seed, unsigned long long step, float* pred,
                      cudaStream_t st) {
  MN_CHECK(loaded, "infer_forward: no snapshot loaded (call mapnet_infer_load first)");
  MN_CHECK(precision != PREC_FP8 || calibrated,
           "infer_forward: the fp8 engine has no activation scales for this snapshot (call mapnet_infer_calibrate)");
  MN_CHECK(B >= 1 && B <= max_B, "infer_forward: batch %d outside [1, max_B=%d]", B, max_B);
  MN_CHECK(x != nullptr && pred != nullptr, "infer_forward: null pointer argument");
  MN_CHECK(droprate >= 0.f && droprate < 1.f, "infer_forward: droprate %f outside [0,1)", droprate);
  MN_TRY(ensure_plans(B));
  MN_TRY(stem_operand(x, B, st));
  return trunk(B, droprate, seed, step, pred, st);
}

// Camera frames in: Resize + ToTensor + Normalize written by pre straight into the stem operand (two launches instead
// of pre's two and the stem operand's one), then the forward from the stem conv on.  Every check comes before the first
// launch.
int InferNet::forward_frames(struct ::mapnet_preprocess* pre, const uint8_t* frames, int B, const float* mean3,
                             const float* std3, float droprate, unsigned long long seed, unsigned long long step,
                             float* pred, cudaStream_t st) {
  MN_CHECK(pred != nullptr, "infer_forward_frames: null pointer argument");
  MN_TRY(check_frames("infer_forward_frames", pre, frames, B, mean3, std3));
  MN_CHECK(droprate >= 0.f && droprate < 1.f, "infer_forward_frames: droprate %f outside [0,1)", droprate);
  MN_TRY(frames_operand(pre, frames, B, mean3, std3, st));
  return trunk(B, droprate, seed, step, pred, st);
}

// S Monte-Carlo dropout draws from camera frames: forward_frames' stem operand and trunk, then sample_head
int InferNet::sample_frames(struct ::mapnet_preprocess* pre, const uint8_t* frames, int B, const float* mean3,
                            const float* std3, int S, float droprate, unsigned long long seed, unsigned long long step,
                            float* samples, double* mean, double* cov, cudaStream_t st) {
  MN_TRY(check_frames("infer_sample_frames", pre, frames, B, mean3, std3));
  MN_TRY(check_sample("infer_sample_frames", S, droprate, mean, cov));
  MN_TRY(frames_operand(pre, frames, B, mean3, std3, st));
  MN_TRY(features(B, st));
  return sample_head(B, S, droprate, seed, step, samples, mean, cov, st);
}

// the checks of a call on camera frames through pre (host-only)
int InferNet::check_frames(const char* what, struct ::mapnet_preprocess* pre, const uint8_t* frames, int B,
                           const float* mean3, const float* std3) const {
  MN_CHECK(loaded, "%s: no snapshot loaded (call mapnet_infer_load first)", what);
  MN_CHECK(precision != PREC_FP8 || calibrated,
           "%s: the fp8 engine has no activation scales for this snapshot (call mapnet_infer_calibrate)", what);
  MN_CHECK(pre != nullptr && frames != nullptr && mean3 != nullptr && std3 != nullptr, "%s: null pointer argument", what);
  int Ho = 0, Wo = 0, max_images = 0;
  MN_TRY(preprocess_geometry(pre, &Ho, &Wo, &max_images));
  MN_CHECK(Ho == H && Wo == W, "%s: the preprocess plan resizes to %dx%d, the engine takes %dx%d", what, Ho, Wo, H, W);
  MN_CHECK(B >= 1 && B <= max_B && B <= max_images,
           "%s: batch %d outside [1, min(max_B=%d, the plan's max_images=%d)]", what, B, max_B, max_images);
  MN_CHECK(spec.stem_s2d, "%s: the engine's stem has no space-to-depth operand", what);
  for (int c = 0; c < 3; ++c)
    MN_CHECK(std3[c] > 0.f, "%s: std[%d] = %f must be positive", what, c, std3[c]);
  return 0;
}

// the stem operand written from camera frames by pre (after check_frames)
int InferNet::frames_operand(struct ::mapnet_preprocess* pre, const uint8_t* frames, int B, const float* mean3,
                             const float* std3, cudaStream_t st) {
  MN_TRY(ensure_plans(B));
  const int Hs = spec.convs[0].g.Hi, Wsp = stem_s2d_wsp(spec.Wc);
  if (precision == PREC_TC_SPLIT) return preprocess_stem_s2d<hsplit>(pre, frames, B, mean3, std3, (hsplit*)A0, Hs, Wsp, st);
  return preprocess_stem_s2d<bf16>(pre, frames, B, mean3, std3, (bf16*)A0, Hs, Wsp, st);
}

// one fp8 conv: t_in / t_res / t_out index the e4m3 tensors' scales (t_res < 0: bf16 residual or none; t_out < 0: bf16
// output).  Calibrating, the epilogue table is folded with the input's new scale, and an e4m3 output's scale is taken
// from an amax pass of the same epilogue before the storing pass.
int InferNet::conv_f8(int ci, const void* in, int t_in, const void* res, int t_res, void* out, int t_out, int relu,
                      bool calib, cudaStream_t st) {
  const int bi = spec.convs[ci].bn, C = spec.convs[ci].g.Co;
  float* S = f8_table + (size_t)ci * 512;
  float* scale = f8_slots + n_f8;
  float* inv = f8_slots + 2 * n_f8;
  EpiF8 e; memset(&e, 0, sizeof(e));
  e.scale = S; e.shift = bn_shift[bi]; e.relu = relu;
  e.res_f8 = t_res >= 0; e.res_scale = t_res >= 0 ? scale + t_res : nullptr;
  e.out_f8 = t_out >= 0; e.out_inv = t_out >= 0 ? inv + t_out : nullptr;
  if (calib) {
    MN_LAUNCH(k_f8_fold, 1, 512, 0, st, bn_scale[bi], s_w + (size_t)ci * 512, scale + t_in, S, C);
    MN_LAUNCH_CHECK();
    if (t_out >= 0) {
      EpiF8 a = e;
      a.amax = reinterpret_cast<unsigned int*>(f8_slots) + t_out;
      MN_TRY(tc_conv_run_f8(plans[ci], (const uint8_t*)in, res, nullptr, a, st));
      MN_LAUNCH(k_f8_set_scale, 1, 32, 0, st, f8_slots, n_f8, t_out, (float*)nullptr, 0);
      MN_LAUNCH_CHECK();
    }
  }
  return tc_conv_run_f8(plans[ci], (const uint8_t*)in, res, out, e, st);
}

int InferNet::run_f8(int B, bool calib, int* last, cudaStream_t st) {
  const Net& n = spec;
  MN_TRY(ensure_plans(B));
  MN_TRY(conv(0, A0, nullptr, y0, 1, 0, 0, st));
  if (calib) {
    MN_CUDA(cudaMemsetAsync(f8_slots, 0, (size_t)n_f8 * 4, st));
    const long long n8 = (long long)B * n.Hc * n.Wc * 64 / 8;
    MN_LAUNCH(k_f8_amax_bf16, (int)(n8 / 256 + 1 < 4 * kNumSMs ? n8 / 256 + 1 : 4 * kNumSMs), 256, 0, st, (const bf16*)y0,
              n8, reinterpret_cast<unsigned int*>(f8_slots));
    MN_LAUNCH_CHECK();
    MN_LAUNCH(k_f8_set_scale, 1, 64, 0, st, f8_slots, n_f8, 0, pool_map, 64);
    MN_LAUNCH_CHECK();
  }
  BnDesc id; memset(&id, 0, sizeof(id));
  id.f.scale = pool_map; id.f.shift = pool_map + 64;
  MN_TRY((launch_stem_pool<bf16, e4m3>((const bf16*)y0, (e4m3*)act[0], nullptr, B, n.Hc, n.Wc, n.Hp, n.Wp, 64, id, st)));
  int xi = 0, t_in = 0;
  for (size_t b = 0; b < n.blocks.size(); ++b) {
    const BlockL& bl = n.blocks[b];
    void* xin = act[xi];
    void* h = act[(xi + 1) % 3];
    void* out = act[(xi + 2) % 3];
    const int t_h = 1 + 2 * (int)b, t_out = 2 + 2 * (int)b;
    MN_TRY(conv_f8(bl.conv1, xin, t_in, nullptr, -1, h, t_h, 1, calib, st));
    if (bl.convd >= 0) {
      MN_TRY(conv_f8(bl.convd, xin, t_in, nullptr, -1, ds, -1, 0, calib, st));
      MN_TRY(conv_f8(bl.conv2, h, t_h, ds, -1, out, t_out, 1, calib, st));
    } else {
      MN_TRY(conv_f8(bl.conv2, h, t_h, xin, t_in, out, t_out, 1, calib, st));
    }
    xi = (xi + 2) % 3;
    t_in = t_out;
  }
  *last = xi;
  return 0;
}

int InferNet::calibrate(const float* x, int B, cudaStream_t st) {
  MN_CHECK(precision == PREC_FP8, "infer_calibrate: only the fp8 engine has activation scales (precision %d)", precision);
  MN_CHECK(loaded, "infer_calibrate: no snapshot loaded (call mapnet_infer_load first)");
  MN_CHECK(B >= 1 && B <= max_B, "infer_calibrate: %d calibration frames outside [1, max_B=%d]", B, max_B);
  MN_CHECK(x != nullptr, "infer_calibrate: null pointer argument");
  int last = 0;
  MN_TRY(ensure_plans(B));
  MN_TRY(stem_operand(x, B, st));
  MN_TRY(run_f8(B, true, &last, st));
  calibrated = true;
  return 0;
}

int InferNet::act_scales(float* host, int cap, cudaStream_t st) {
  MN_CHECK(precision == PREC_FP8, "infer_act_scales: only the fp8 engine has activation scales (precision %d)", precision);
  MN_CHECK(calibrated, "infer_act_scales: not calibrated");
  MN_CHECK(host != nullptr && cap >= n_f8, "infer_act_scales: need room for %d scales", n_f8);
  MN_CUDA(cudaMemcpyAsync(host, f8_slots + n_f8, (size_t)n_f8 * 4, cudaMemcpyDeviceToHost, st));
  MN_CUDA(cudaStreamSynchronize(st));
  return n_f8;
}

}  // namespace mapnet
