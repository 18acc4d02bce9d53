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
#include "infer.h"

#include <string.h>

namespace mapnet {

static long long align_up(long long v, long long a) { return (v + a - 1) / a * a; }

int InferNet::alloc(void** p, size_t bytes) {
  if (bytes == 0) bytes = 16;
  MN_CUDA(cudaMalloc(p, align_up((long long)bytes, 256)));
  allocs.push_back(*p);
  return 0;
}

int InferNet::sizes(const Net& n, Sizes* s) {
  const long long ez = (n.precision == PREC_TC_SPLIT) ? 4 : 2;       // operand element (bf16 / hi+lo fp16 planes)
  const long long ea = (n.precision == PREC_TC_SPLIT) ? 4 : 2;       // conv output element (bf16 / fp32)
  const ConvGeom& g0 = n.convs[0].g;
  s->a0 = n.stem_s2d ? (long long)g0.Hi * stem_s2d_wsp(n.Wc) * 16 * ez : (long long)n.Hc * n.Wc * g0.Ci * ez;
  s->y0 = (long long)n.Hc * n.Wc * 64 * ea;
  long long act = (long long)n.Hp * n.Wp * 64, ds = 0;
  for (const BlockL& b : n.blocks) {
    const long long e = (long long)b.Ho * b.Wo * b.Cout;
    if (e > act) act = e;
    if (b.convd >= 0 && e > ds) ds = e;
  }
  s->act = act * ez;
  s->ds = ds * ea;
  s->head = (512 + 3LL * n.feat_dim) * 4;     // feat, fc output (pre-ReLU and dropped), dropout mask
  return 0;
}

long long InferNet::arena_bytes(int max_B, int H, int W, int precision) {
  if (precision != PREC_BF16_TC && precision != PREC_TC_SPLIT) {
    set_last_error("infer: precision %d is not supported (bf16 = %d or tc_split = %d)", precision, PREC_BF16_TC,
                   PREC_TC_SPLIT);
    return -2;
  }
  if (max_B < 1 || H < 32 || W < 32) { set_last_error("infer: need max_B >= 1 and H, W >= 32 (got %d, %d, %d)", max_B, H, W); return -2; }
  Net n = Net();
  if (n.init(0, H, W, 2048, precision) != 0) return -2;
  Sizes s;
  sizes(n, &s);
  n.destroy();
  return (long long)max_B * (s.a0 + s.y0 + 3 * s.act + s.ds + s.head);
}

int InferNet::init(int max_B_, int H_, int W_, int feat_dim_, int precision_) {
  max_B = max_B_; H = H_; W = W_; feat_dim = feat_dim_; precision = precision_;
  loaded = false; plan_B = 0;
  wk = nullptr; d_wdescs = nullptr; affine = head = ident = eval_scratch = nullptr;
  A0 = y0 = ds = nullptr; act[0] = act[1] = act[2] = nullptr;
  feat = fcpre = hdrop = mask = nullptr; drop_ctr = nullptr;
  MN_CHECK(precision == PREC_BF16_TC || precision == PREC_TC_SPLIT,
           "infer_create: precision %d is not supported (bf16 = %d or tc_split = %d)", precision, PREC_BF16_TC, PREC_TC_SPLIT);
  MN_CHECK(max_B >= 1 && H >= 32 && W >= 32, "infer_create: need max_B >= 1 and H, W >= 32 (got %d, %d, %d)", max_B, H, W);
  MN_TRY(spec.init(0, H, W, feat_dim, precision));
  MN_CHECK(!spec.stem_s2d || tc_overlapped_view_supported(),
           "infer_create: the driver rejects the overlapped tensor map of the space-to-depth stem");
  Sizes s;
  sizes(spec, &s);
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
  MN_TRY(alloc(&wk, (size_t)spec.wk_total * (precision == PREC_TC_SPLIT ? 8 : 2)));
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
  if (precision == PREC_BF16_TC) {
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

template <typename P>
int InferNet::forward_t(const float* x, int B, float droprate, unsigned long long seed, unsigned long long step,
                        float* pred, cudaStream_t st) {
  typedef typename P::A T;        // stem / downsample conv outputs (bf16, or fp32 in strict mode)
  typedef typename P::Z TZ;       // conv operands (bf16, or fp16 hi/lo planes)
  const int sp = (precision == PREC_TC_SPLIT) ? 1 : 0;
  const Net& n = spec;
  MN_TRY(ensure_plans(B));
  // stem: operand image -> conv + BN + ReLU (epilogue) -> 3x3/s2 max pool
  if (n.stem_s2d) MN_TRY(launch_stem_s2d<TZ>(x, (TZ*)A0, B, H, W, n.convs[0].g.Hi, stem_s2d_wsp(n.Wc), st));
  else MN_TRY(launch_stem_im2col<TZ>(x, (TZ*)A0, B, H, W, n.Hc, n.Wc, n.convs[0].g.Ci, st));
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
  // head: exactly the calls of Net::forward_t, on the snapshot's copy of the head parameters
  const float* hp = head - n.fc_w;      // indexed with the flat-buffer offsets
  MN_TRY(launch_gap<TZ>((const TZ*)act[xi], feat, B, n.Hf * n.Wf, 512, st));
  const float* mk = nullptr;
  if (droprate > 0.f) {
    const unsigned long long stride = (unsigned long long)max_B * feat_dim;
    const bool dev_ctr = (step == ~0ULL);
    MN_TRY(launch_dropout_mask(mask, (long long)B * feat_dim, droprate, seed, dev_ctr ? 0ULL : step * stride,
                               dev_ctr ? drop_ctr : nullptr, stride, st));
    mk = mask;
  }
  MN_TRY(launch_small_gemm(1, feat, 512, 1, hp + n.fc_w, 512, 1, hdrop, feat_dim, B, feat_dim, 512, hp + n.fc_b, fcpre, mk, st));
  MN_TRY(launch_small_gemm(0, hdrop, feat_dim, 1, hp + n.xyz_w, feat_dim, 1, pred, 6, B, 3, feat_dim, hp + n.xyz_b, nullptr, nullptr, st));
  MN_TRY(launch_small_gemm(0, hdrop, feat_dim, 1, hp + n.wpqr_w, feat_dim, 1, pred + 3, 6, B, 3, feat_dim, hp + n.wpqr_b, nullptr, nullptr, st));
  return 0;
}

int InferNet::forward(const float* x, int B, float droprate, unsigned long long seed, unsigned long long step, float* pred,
                      cudaStream_t st) {
  MN_CHECK(loaded, "infer_forward: no snapshot loaded (call mapnet_infer_load first)");
  MN_CHECK(B >= 1 && B <= max_B, "infer_forward: batch %d outside [1, max_B=%d]", B, max_B);
  MN_CHECK(x != nullptr && pred != nullptr, "infer_forward: null pointer argument");
  MN_CHECK(droprate >= 0.f && droprate < 1.f, "infer_forward: droprate %f outside [0,1)", droprate);
  if (precision == PREC_TC_SPLIT) return forward_t<TypesSplitHH>(x, B, droprate, seed, step, pred, st);
  return forward_t<TypesBF16>(x, B, droprate, seed, step, pred, st);
}

}  // namespace mapnet
