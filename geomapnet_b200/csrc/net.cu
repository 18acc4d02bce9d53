// PoseNet(ResNet-34) training step plan: explicit forward and backward schedules
// over a static activation arena -- no autograd graph inside the trunk.
//
// Mirrors the graph that /root/reference/models/posenet.py:65-73 runs through
// torchvision resnet34 (BasicBlock [3,4,6,3]; conv-BN-ReLU-conv-BN-(+id|1x1s2
// conv+BN)-ReLU; SURVEY.md section 8a-1..3) with training-mode BatchNorm.
#include "net.h"
#include "bn_fin.cuh"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include <type_traits>

namespace mapnet {

// ---- error string ------------------------------------------------------------
unsigned long long g_launch_count = 0;

int pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("MAPNET_PDL"); v = (e && atoi(e) == 0) ? 0 : 1; }
  return v;
}
static thread_local char g_err[1024] = "";
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_last_error() { return g_err; }

static const int kStages[4][3] = {{64, 3, 1}, {128, 4, 2}, {256, 6, 2}, {512, 3, 2}};
static const int kStemK = kStemIm2colK;

static long long align_up(long long v, long long a) { return (v + a - 1) / a * a; }
static int conv_out(int n, int k, int s, int p) { return (n + 2 * p - k) / s + 1; }

int Net::alloc(void** p, size_t bytes) {
  if (bytes == 0) bytes = 16;
  MN_CUDA(cudaMalloc(p, bytes));
  allocs.push_back(*p);
  return 0;
}

void Net::build_table() {
  table.clear();
  n_params = n_bufs = n_nbt = 0;
  auto add = [&](const std::string& name, int kind, std::initializer_list<long long> shp) {
    ParamEntry e;
    e.name = name; e.kind = kind; e.layout = 0; e.ndim = (int)shp.size(); e.numel = 1;
    int i = 0;
    for (long long s : shp) { e.shape[i++] = s; e.numel *= s; }
    for (; i < 4; ++i) e.shape[i] = 1;
    if (kind == 0) { e.offset = n_params; n_params = align_up(n_params + e.numel, 64); }
    else if (kind == 1) { e.offset = n_bufs; n_bufs = align_up(n_bufs + e.numel, 64); }
    else { e.offset = n_nbt; n_nbt += 1; }
    table.push_back(e);
    return (int)table.size() - 1;
  };
  auto add_bn = [&](const std::string& p, int C) {
    BNL b; b.C = C;
    b.g_off = table[add(p + ".weight", 0, {C})].offset;
    b.b_off = table[add(p + ".bias", 0, {C})].offset;
    b.rm_off = table[add(p + ".running_mean", 1, {C})].offset;
    b.rv_off = table[add(p + ".running_var", 1, {C})].offset;
    add(p + ".num_batches_tracked", 2, {});
    b.mean = b.invstd = b.scale = b.shift = b.coef = nullptr;
    bns.push_back(b);
    return (int)bns.size() - 1;
  };
  wk_total = 0; max_w_elems = 0;
  auto add_conv = [&](const std::string& name, int Ci, int Co, int k, int stride, int Hi, int Wi, bool stem) {
    ConvL c;
    const int pidx = add(name + ".weight", 0, {Co, stem ? 3 : Ci, k, k});
    table[pidx].layout = stem ? 0 : 1;     // [Co][KH][KW][Ci] in the flat buffers (what the engines read and accumulate)
    c.wd.p_off = table[pidx].offset;
    c.wd.k_off = wk_total;
    c.wd.Co = Co; c.wd.Ci_real = stem ? 3 : Ci;
    c.wd.s2d = 0;
    if (stem && stem_s2d) {
      // 4 taps (filter rows of the space-to-depth image) x 64 contiguous elements (4 blocks x 16 channels)
      stem_s2d_geometry(Hi, Wi, Co, &c.g, &c.wd, (int)elt());
    } else if (stem) {
      c.wd.Ci = kStemK; c.wd.KH = c.wd.KW = 1; c.wd.im2col_k = kStemK;
      c.g.Hi = conv_out(Hi, 7, 2, 3); c.g.Wi = conv_out(Wi, 7, 2, 3);   // GEMM view: 1x1 conv over the patch matrix
      c.g.Ho = c.g.Hi; c.g.Wo = c.g.Wi; c.g.Ci = kStemK; c.g.Co = Co; c.g.KH = c.g.KW = 1; c.g.stride = 1; c.g.pad = 0;
    } else {
      c.wd.Ci = Ci; c.wd.KH = c.wd.KW = k; c.wd.im2col_k = 0;
      c.g.Hi = Hi; c.g.Wi = Wi; c.g.Ci = Ci; c.g.Co = Co; c.g.KH = c.g.KW = k; c.g.stride = stride; c.g.pad = (k - 1) / 2;
      c.g.Ho = conv_out(Hi, k, stride, c.g.pad); c.g.Wo = conv_out(Wi, k, stride, c.g.pad);
    }
    c.g.B = 0;
    const long long ne = (long long)Co * c.wd.KH * c.wd.KW * c.wd.Ci;
    wk_total += align_up(ne, 512);        // 1 KB-aligned (bf16) matrices: TMA base alignment
    if (ne > max_w_elems) max_w_elems = (int)ne;
    c.bn = -1;
    convs.push_back(c);
    return (int)convs.size() - 1;
  };

  const std::string fe = "feature_extractor.";
  Hc = conv_out(H, 7, 2, 3); Wc = conv_out(W, 7, 2, 3);
  Hp = conv_out(Hc, 3, 2, 1); Wp = conv_out(Wc, 3, 2, 1);
  int c0 = add_conv(fe + "conv1", 3, 64, 7, 2, H, W, true);
  convs[c0].bn = add_bn(fe + "bn1", 64);
  int inpl = 64, h = Hp, w = Wp;
  for (int li = 0; li < 4; ++li) {
    const int planes = kStages[li][0], nblk = kStages[li][1];
    for (int b = 0; b < nblk; ++b) {
      const int s = (b == 0) ? kStages[li][2] : 1;
      char pre[64];
      snprintf(pre, sizeof(pre), "%slayer%d.%d.", fe.c_str(), li + 1, b);
      BlockL bl;
      bl.Hi = h; bl.Wi = w; bl.Cin = inpl; bl.Cout = planes; bl.stride = s;
      bl.conv1 = add_conv(std::string(pre) + "conv1", inpl, planes, 3, s, h, w, false);
      convs[bl.conv1].bn = add_bn(std::string(pre) + "bn1", planes);
      bl.Ho = convs[bl.conv1].g.Ho; bl.Wo = convs[bl.conv1].g.Wo;
      bl.conv2 = add_conv(std::string(pre) + "conv2", planes, planes, 3, 1, bl.Ho, bl.Wo, false);
      convs[bl.conv2].bn = add_bn(std::string(pre) + "bn2", planes);
      bl.convd = -1;
      if (s != 1 || inpl != planes) {
        bl.convd = add_conv(std::string(pre) + "downsample.0", inpl, planes, 1, s, h, w, false);
        convs[bl.convd].bn = add_bn(std::string(pre) + "downsample.1", planes);
      }
      bl.y1 = bl.h = bl.y2 = bl.yd = bl.out = nullptr;
      bl.ds_fold = 0;          // set by ensure_tc_plans on the tensor-core path only
      blocks.push_back(bl);
      inpl = planes; h = bl.Ho; w = bl.Wo;
    }
  }
  Hf = h; Wf = w;
  fc_w = table[add(fe + "fc.weight", 0, {feat_dim, 512})].offset;
  fc_b = table[add(fe + "fc.bias", 0, {feat_dim})].offset;
  xyz_w = table[add("fc_xyz.weight", 0, {3, feat_dim})].offset;
  xyz_b = table[add("fc_xyz.bias", 0, {3})].offset;
  wpqr_w = table[add("fc_wpqr.weight", 0, {3, feat_dim})].offset;
  wpqr_b = table[add("fc_wpqr.bias", 0, {3})].offset;
}

int Net::init(int max_B_, int H_, int W_, int feat_dim_, int precision_, int im2col_stem) {
  max_B = max_B_; H = H_; W = W_; feat_dim = feat_dim_; precision = precision_;
  MN_CHECK(max_B >= 0 && H >= 32 && W >= 32, "create: need max_B>=0 and H,W>=32 (got %d,%d,%d)", max_B, H, W);
  MN_CHECK(precision >= 0 && precision <= 3, "create: bad precision %d", precision);
  MN_CHECK(feat_dim >= 8 && feat_dim % 4 == 0, "create: feat_dim must be a multiple of 4");
  last_B = 0; last_training = 0; last_has_mask = 0; tc_B = 0; profile_on = 0; prof_pool_used = 0;
  bwd_pre = false; bwd_next_part = 0;
  side = nullptr; ring_pos = 0; cur_grads = nullptr; dw_stem_elems = 0;
  for (int i = 0; i < 4; ++i) { ring[i] = nullptr; ring_ready[i] = ring_done[i] = nullptr; ring_pending[i] = false; }
  stem_s2d = !im2col_stem && tc() && (max_B == 0 || tc_overlapped_view_supported());
  Hc = conv_out(H, 7, 2, 3); Wc = conv_out(W, 7, 2, 3);        // (build_table sets them again)
  stem_fuse = (Hc % 2 == 0) && (Wc % 2 == 0);
  { const char* e = getenv("MAPNET_TC_FUSE_BWD"); fuse_bwd = (precision == PREC_BF16_TC) && (e ? atoi(e) != 0 : 1); }
  stats_target = nullptr; bn_slots = nullptr; bn_slots_bytes = 0;
  { const char* e = getenv("MAPNET_TC_DS_FOLD"); ds_fold = (precision == PREC_BF16_TC) && (e ? atoi(e) != 0 : 1); }
  build_table();
  {
    std::vector<uint8_t> all;
    for (auto& e : table) if (e.kind == 0) all.push_back(1);
    MN_TRY(set_trainable(all.data(), (int)all.size()));
  }
  if (max_B == 0) return 0;      // spec-only handle: parameter table, no device memory
  const size_t es = elt();
  const long long Bm = max_B;
  MN_TRY(alloc(&A0, (size_t)(Bm * Hc * Wc * kStemK) * es));
  MN_TRY(alloc(&y0, (size_t)(Bm * Hc * Wc * 64) * es));
  MN_TRY(alloc(&z0, (size_t)(Bm * Hp * Wp * 64) * es));
  MN_TRY(alloc((void**)&amax0, (size_t)(Bm * Hp * Wp * 64)));
  scratch_elems = Bm * Hc * Wc * 64;
  for (int i = 0; i < 7; ++i) MN_TRY(alloc(&scratch[i], (size_t)scratch_elems * es));
  ring[0] = scratch[1]; ring[1] = scratch[2]; ring[2] = scratch[5]; ring[3] = scratch[6];
  ring_pos = 0;
  {
    int lo = 0, hi = 0;
    MN_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));       // lo = numerically greatest = lowest priority
    MN_CUDA(cudaStreamCreateWithPriority(&side, cudaStreamNonBlocking, lo));
    for (int i = 0; i < 4; ++i) {
      MN_CUDA(cudaEventCreateWithFlags(&ring_ready[i], cudaEventDisableTiming));
      MN_CUDA(cudaEventCreateWithFlags(&ring_done[i], cudaEventDisableTiming));
      ring_pending[i] = false;
    }
  }
  for (auto& bl : blocks) {
    const size_t n = (size_t)(Bm * bl.Ho * bl.Wo * bl.Cout) * es;
    MN_TRY(alloc(&bl.y1, n)); MN_TRY(alloc(&bl.h, n)); MN_TRY(alloc(&bl.y2, n)); MN_TRY(alloc(&bl.out, n));
    if (bl.convd >= 0) MN_TRY(alloc(&bl.yd, n));
  }
  const size_t wes = (precision == PREC_BF16_TC) ? 2 : (precision == PREC_TC_SPLIT ? 8 : 4);
  MN_TRY(alloc(&w_krsc, (size_t)wk_total * wes));
  MN_TRY(alloc(&w_dg, (size_t)wk_total * wes));
  w_krsc_f32 = w_dg_f32 = nullptr;
  if (precision == PREC_TC_SPLIT) {      // fp32 K-major matrices the hi / lo planes are cut from
    MN_TRY(alloc((void**)&w_krsc_f32, (size_t)wk_total * 4));
    MN_TRY(alloc((void**)&w_dg_f32, (size_t)wk_total * 4));
  }
  dw_stem_elems = align_up((long long)convs[0].wd.Co * convs[0].wd.KH * convs[0].wd.KW * convs[0].wd.Ci, 512);
  MN_TRY(alloc((void**)&dw_krsc, (size_t)dw_stem_elems * 4));       // the stem's wgrad (conv 0, k_off == 0)
  std::vector<WeightDesc> wd;
  for (auto& c : convs) wd.push_back(c.wd);
  MN_TRY(alloc((void**)&d_wdescs, wd.size() * sizeof(WeightDesc)));
  MN_CUDA(cudaMemcpy(d_wdescs, wd.data(), wd.size() * sizeof(WeightDesc), cudaMemcpyHostToDevice));
  MN_TRY(alloc((void**)&bn_accum, kBnAccReplicas * kBnAccStride * sizeof(double) + 64));
  MN_CUDA(cudaMemset(bn_accum, 0, kBnAccReplicas * kBnAccStride * sizeof(double) + 64));
  bn_counter = (unsigned int*)(bn_accum + kBnAccReplicas * kBnAccStride);
  MN_CHECK(bns.size() <= 36, "trunk: %d BatchNorm layers (36 accumulator slots)", (int)bns.size());
  bn_slots_bytes = (size_t)(72 * kSlotReplicas + kStemBwdReplicas) * kSlotStride * sizeof(double);
  MN_TRY(alloc((void**)&bn_slots, bn_slots_bytes));
  MN_CUDA(cudaMemset(bn_slots, 0, bn_slots_bytes));
  long long small = 0;
  for (auto& b : bns) small += 7LL * b.C;
  MN_TRY(alloc((void**)&bn_small, (size_t)small * sizeof(float)));
  float* p = bn_small;
  for (auto& b : bns) {
    b.mean = p; p += b.C; b.invstd = p; p += b.C; b.scale = p; p += b.C; b.shift = p; p += b.C;
    b.coef = p; p += 3 * b.C;
  }
  MN_TRY(alloc((void**)&feat, (size_t)Bm * 512 * 4));
  MN_TRY(alloc((void**)&fcpre, (size_t)Bm * feat_dim * 4));
  MN_TRY(alloc((void**)&hdrop, (size_t)Bm * feat_dim * 4));
  MN_TRY(alloc((void**)&mask, (size_t)Bm * feat_dim * 4));
  MN_TRY(alloc((void**)&dh, (size_t)Bm * feat_dim * 4));
  MN_TRY(alloc((void**)&dfeat, (size_t)Bm * 512 * 4));
  MN_TRY(alloc((void**)&dpredf, (size_t)Bm * 6 * 4 * 2));      // two NaN-filtered copies of d pred (head.cu)
  MN_TRY(alloc((void**)&sq_partials, 1024 * 4));
  MN_TRY(alloc((void**)&sq_out, 16));
  MN_TRY(alloc((void**)&drop_ctr, 16));
  MN_TRY(alloc((void**)&gscale, 16));
  { const float one[2] = {1.f, 1.f}; MN_CUDA(cudaMemcpy(gscale, one, sizeof(one), cudaMemcpyHostToDevice)); }
  MN_CUDA(cudaMemset(drop_ctr, 0, 16));
  return 0;
}

int Net::set_trainable(const uint8_t* host_mask, int n) {
  int nk = 0;
  for (auto& e : table) nk += (e.kind == 0);
  MN_CHECK(host_mask != nullptr, "set_trainable: null mask");
  MN_CHECK(n == nk, "set_trainable: mask has %d entries, the parameter table %d trainable ones", n, nk);
  std::map<long long, bool> by_off;       // parameter offset -> needs a gradient
  int k = 0;
  for (auto& e : table) if (e.kind == 0) by_off[e.offset] = host_mask[k++] != 0;
  for (auto& c : convs) c.train = by_off[c.wd.p_off];
  for (auto& b : bns) { b.train_g = by_off[b.g_off]; b.train_b = by_off[b.b_off]; }
  train_fc_w = by_off[fc_w]; train_fc_b = by_off[fc_b];
  train_xyz_w = by_off[xyz_w]; train_xyz_b = by_off[xyz_b];
  train_wpqr_w = by_off[wpqr_w]; train_wpqr_b = by_off[wpqr_b];
  auto conv_trains = [&](int ci) { return ci >= 0 && (convs[ci].train || bns[convs[ci].bn].train_g || bns[convs[ci].bn].train_b); };
  bwd_lo = (int)blocks.size();
  for (int bi = (int)blocks.size() - 1; bi >= 0; --bi)
    if (conv_trains(blocks[bi].conv1) || conv_trains(blocks[bi].conv2) || conv_trains(blocks[bi].convd)) bwd_lo = bi;
  if (conv_trains(0)) bwd_lo = -1;
  return 0;
}

void Net::destroy() {
  for (auto& kv : tc_sets)
    for (auto* v : {&kv.second.fprop, &kv.second.dgrad, &kv.second.wgrad})
      for (auto* p : *v) tc_plan_destroy(p);
  tc_sets.clear();
  tc_fprop.clear(); tc_dgrad.clear(); tc_wgrad.clear();
  tc_B = 0;
  for (void* p : allocs) cudaFree(p);
  allocs.clear();
  if (side != nullptr) {
    cudaStreamSynchronize(side);
    for (int i = 0; i < 4; ++i) { if (ring_ready[i]) cudaEventDestroy(ring_ready[i]); if (ring_done[i]) cudaEventDestroy(ring_done[i]); }
    cudaStreamDestroy(side);
    side = nullptr;
  }
  for (cudaEvent_t e : prof_pool) cudaEventDestroy(e);
  prof_pool.clear();
}

// ---- conv dispatch -------------------------------------------------------------
// events come from a pool that is only ever grown: creating two events per conv launch inside the profiled
// step made the host the bottleneck and the idle gaps landed inside the brackets
int Net::prof_event(cudaEvent_t* e) {
  if (prof_pool_used == prof_pool.size()) {
    cudaEvent_t ev;
    MN_CUDA(cudaEventCreate(&ev));
    prof_pool.push_back(ev);
  }
  *e = prof_pool[prof_pool_used++];
  return 0;
}
int Net::prof_reserve(int n_events) {
  while ((int)prof_pool.size() < n_events) {
    cudaEvent_t ev;
    MN_CUDA(cudaEventCreate(&ev));
    prof_pool.push_back(ev);
  }
  return 0;
}
int Net::prof_begin(cudaStream_t st, cudaEvent_t* e0) {
  if (!profile_on) return 0;
  MN_TRY(prof_event(e0));
  MN_CUDA(cudaEventRecord(*e0, st));
  return 0;
}
void Net::prof_end(cudaStream_t st, cudaEvent_t e0, int cls, double flops) {
  if (!profile_on) return;
  ProfRec r; r.e0 = e0; r.cls = cls; r.flops = flops;
  if (prof_event(&r.e1) != 0) return;
  cudaEventRecord(r.e1, st);
  prof.push_back(r);
}
int Net::prof_read(double* ms3, double* flops3, int* launches3) {
  for (int i = 0; i < 3; ++i) { ms3[i] = 0; flops3[i] = 0; launches3[i] = 0; }
  MN_CUDA(cudaDeviceSynchronize());
  // MAPNET_PROFILE_DUMP=<path>: one line per bracketed launch (class, algorithmic GFLOP, microseconds), in launch order
  const char* dump = getenv("MAPNET_PROFILE_DUMP");
  FILE* df = (dump && dump[0]) ? fopen(dump, "a") : nullptr;
  for (auto& r : prof) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.e0, r.e1);
    ms3[r.cls] += ms; flops3[r.cls] += r.flops; launches3[r.cls] += 1;
    if (df) fprintf(df, "%s %.3f GF %.2f us %.0f TF\n", r.cls == 0 ? "fprop" : (r.cls == 1 ? "dgrad" : "wgrad"), r.flops * 1e-9,
                    ms * 1e3, ms > 0 ? r.flops / (ms * 1e-3) * 1e-12 : 0.0);
  }
  if (df) { fprintf(df, "---\n"); fclose(df); }
  prof.clear();
  prof_pool_used = 0;
  return 0;
}

static double conv_flops(const ConvGeom& g, int B, bool stem) {
  // algorithmic MACs of the convolution (the stem's zero padding of K to 192 is not counted)
  const double k = stem ? 147.0 : (double)g.KH * g.KW * g.Ci;
  return 2.0 * (double)B * g.Ho * g.Wo * g.Co * k;
}

// The CUDA-core engine works on one element type; it is only reachable in the modes whose A / Z / G types coincide.
template <typename P> struct SimtConv {
  static constexpr bool ok = std::is_same<typename P::A, typename P::Z>::value && std::is_same<typename P::A, typename P::G>::value;
};

template <typename P>
int Net::conv_fprop(int ci, const typename P::Z* x, const typename P::A* residual, typename P::A* y, int B, cudaStream_t st) {
  ConvGeom g = convs[ci].g; g.B = B;
  cudaEvent_t e0 = nullptr;
  MN_TRY(prof_begin(st, &e0));
  int r;
  if (tc())
    r = tc_conv_run(tc_fprop[ci], (const bf16*)x, nullptr, (const bf16*)residual, y, st, stats_target);
  else if constexpr (SimtConv<P>::ok)
    r = launch_conv_simt_fprop<typename P::A>(g, x, (const float*)w_krsc + convs[ci].wd.k_off, residual, y, st);
  else { set_last_error("conv_fprop: no CUDA-core engine for split operands"); r = 2; }
  prof_end(st, e0, 0, conv_flops(g, B, ci == 0));
  return r;
}
template <typename P>
int Net::conv_dgrad(int ci, const typename P::G* dy, const typename P::A* residual, typename P::A* dx, int B, cudaStream_t st,
                    const EpiBwd* bwd, const typename P::G* dy_shortcut, int ci_shortcut) {
  ConvGeom g = convs[ci].g; g.B = B;
  cudaEvent_t e0 = nullptr;
  MN_TRY(prof_begin(st, &e0));
  int r;
  double flops = conv_flops(g, B, false);
  if (tc()) {
    // dy_shortcut: the block's downsample-conv dgrad rides in the same launch (tc_plan_add_shortcut)
    r = tc_conv_run(tc_dgrad[ci], (const bf16*)dy, (const bf16*)dy_shortcut, (const bf16*)residual, dx, st, bwd ? stats_target : nullptr, bwd);
    if (dy_shortcut != nullptr) { ConvGeom gs = convs[ci_shortcut].g; gs.B = B; flops += conv_flops(gs, B, false); }
  } else if constexpr (SimtConv<P>::ok) {
    MN_CHECK(dy_shortcut == nullptr, "conv_dgrad: folded shortcut is a tensor-core path feature");
    r = launch_conv_simt_dgrad<typename P::A>(g, dy, (const float*)w_dg + convs[ci].wd.k_off, residual, dx, st);
  } else { set_last_error("conv_dgrad: no CUDA-core engine for split operands"); r = 2; }
  prof_end(st, e0, 1, flops);
  return r;
}
// next slot of the d(conv output) ring, safe to overwrite on `st`
void* Net::ring_next(cudaStream_t st) {
  const int slot = ring_pos++ & 3;
  if (ring_pending[slot]) { cudaStreamWaitEvent(st, ring_done[slot], 0); ring_pending[slot] = false; }
  return ring[slot];
}
int Net::ring_slot(const void* p) const {
  for (int i = 0; i < 4; ++i) if (ring[i] == p) return i;
  return -1;
}
int Net::wgrad_join(cudaStream_t st) {
  for (int i = 0; i < 4; ++i)
    if (ring_pending[i]) { MN_CUDA(cudaStreamWaitEvent(st, ring_done[i], 0)); ring_pending[i] = false; }
  return 0;
}

template <typename P>
int Net::conv_wgrad(int ci, const typename P::Z* x, const typename P::G* dy, int B, cudaStream_t st) {
  ConvGeom g = convs[ci].g; g.B = B;
  const int slot = ring_slot(dy);
  if (!profile_on && slot >= 0) {
    // fork: the side stream picks the gradient up where the compute stream has just finished writing it
    MN_CUDA(cudaEventRecord(ring_ready[slot], st));
    MN_CUDA(cudaStreamWaitEvent(side, ring_ready[slot], 0));
    int r;
    if (tc()) r = tc_conv_run(tc_wgrad[ci], (const bf16*)x, (const bf16*)dy, nullptr, wgrad_out(ci), side);
    else if constexpr (SimtConv<P>::ok) r = launch_conv_simt_wgrad<typename P::A>(g, x, dy, wgrad_out(ci), side);
    else { set_last_error("conv_wgrad: no CUDA-core engine for split operands"); r = 2; }
    MN_CUDA(cudaEventRecord(ring_done[slot], side));
    ring_pending[slot] = true;
    return r;
  }
  cudaEvent_t e0 = nullptr;
  MN_TRY(prof_begin(st, &e0));
  int r;
  if (tc()) r = tc_conv_run(tc_wgrad[ci], (const bf16*)x, (const bf16*)dy, nullptr, wgrad_out(ci), st);
  else if constexpr (SimtConv<P>::ok) r = launch_conv_simt_wgrad<typename P::A>(g, x, dy, wgrad_out(ci), st);
  else { set_last_error("conv_wgrad: no CUDA-core engine for split operands"); r = 2; }
  prof_end(st, e0, 2, conv_flops(g, B, ci == 0));
  return r;
}

int Net::ensure_tc_plans(int B) {
  if (!tc() || tc_B == B) return 0;
  auto it = tc_sets.find(B);
  if (it != tc_sets.end()) {
    const TcPlanSet& s = it->second;
    tc_fprop = s.fprop; tc_dgrad = s.dgrad; tc_wgrad = s.wgrad;
    for (size_t k = 0; k < blocks.size(); ++k) blocks[k].ds_fold = s.ds_fold[k];
    tc_B = B;
    return 0;
  }
  tc_B = 0;
  tc_fprop.assign(convs.size(), nullptr);
  tc_dgrad.assign(convs.size(), nullptr);
  tc_wgrad.assign(convs.size(), nullptr);
  const int r = build_tc_plans(B);
  if (r != 0) {       // free what was built; the next call at this B starts over
    for (auto* v : {&tc_fprop, &tc_dgrad, &tc_wgrad}) { for (auto* p : *v) tc_plan_destroy(p); v->clear(); }
    return r;
  }
  TcPlanSet& s = tc_sets[B];
  s.fprop = tc_fprop; s.dgrad = tc_dgrad; s.wgrad = tc_wgrad;
  for (auto& bl : blocks) s.ds_fold.push_back(bl.ds_fold);
  tc_B = B;
  return 0;
}

int Net::build_tc_plans(int B) {
  for (size_t i = 0; i < convs.size(); ++i) {
    ConvGeom g = convs[i].g; g.B = B;
    const bool sp = precision == PREC_TC_SPLIT;
    if (sp) g.split = 1;
    const bf16* wk = (const bf16*)w_krsc + (sp ? 4 : 1) * convs[i].wd.k_off;     // split planes: 4 x the 16-bit elements
    const bf16* wd = (const bf16*)w_dg + (sp ? 4 : 1) * convs[i].wd.k_off;
    MN_TRY(tc_plan_create(&tc_fprop[i], g, 0, wk));
    if (i > 0) MN_TRY(tc_plan_create(&tc_dgrad[i], g, 1, wd));
    MN_TRY(tc_plan_create(&tc_wgrad[i], g, 2, nullptr));
    if (sp) {       // fp16 gradient planes carry the step's power-of-two scale: divide it out
      if (i > 0) tc_plan_set_out_scale(tc_dgrad[i], gscale + 1);
      tc_plan_set_out_scale(tc_wgrad[i], gscale + 1);
    }
  }
  // stride-2 blocks: the 1x1 downsample dgrad becomes one more tap of conv1's (single-launch) dgrad
  for (auto& bl : blocks) {
    bl.ds_fold = 0;
    if (!ds_fold || bl.convd < 0 || convs[bl.conv1].g.stride != 2 || convs[bl.conv1].g.KH != 3) continue;
    if (tc_plan_launches(tc_dgrad[bl.conv1]) != 1) continue;       // MAPNET_TC_DGRAD_MERGE=0: per-class launches
    MN_TRY(tc_plan_add_shortcut(tc_dgrad[bl.conv1], (const bf16*)w_dg + convs[bl.convd].wd.k_off));
    bl.ds_fold = 1;
  }
  return 0;
}

template <typename P>
int Net::bn_forward(int bi, const typename P::A* y, long long M, const float* params, float* bufs, int training,
                    cudaStream_t st) {
  typedef typename P::A T;
  const BnFin f = lazy_forward(bi, M, params, bufs, false).f;
  if (!training) return launch_bn_eval_scale(bns[bi].C, f, st);
  return launch_bn_stats<T>(y, M, bns[bi].C, f, bn_accum, bn_counter, st);
}

BnDesc Net::lazy_forward(int bi, long long M, const float* params, float* bufs, bool sums) {
  BnDesc L; memset(&L, 0, sizeof(L));
  BNL& b = bns[bi];
  if (sums) { L.accum = fwd_slot(bi); L.nrep = kSlotReplicas; }
  L.M = M;
  L.invM = 1.0 / (double)M; L.unbias = (M > 1) ? (double)M / (double)(M - 1) : 1.0;
  L.f.gamma = params + b.g_off; L.f.beta = params + b.b_off; L.f.run_mean = bufs + b.rm_off; L.f.run_var = bufs + b.rv_off;
  L.f.mean = b.mean; L.f.invstd = b.invstd; L.f.scale = b.scale; L.f.shift = b.shift;
  return L;
}
BnDesc Net::lazy_backward(int bi, int bi_ds, long long M, const float* params, float* grads, bool sums) {
  BnDesc L; memset(&L, 0, sizeof(L));
  BNL& b = bns[bi];
  if (sums) { L.accum = bwd_slot(bi); L.nrep = (bi == convs[0].bn) ? kStemBwdReplicas : kSlotReplicas; }
  L.M = M;
  L.invM = 1.0 / (double)M; L.unbias = 1.0;
  L.f.gamma = params + b.g_off; L.f.mean = b.mean; L.f.invstd = b.invstd;
  // a frozen gamma / beta gets no gradient: its grads_flat entries keep the zero of the pass's opening memset
  L.f.dgamma = b.train_g ? grads + b.g_off : nullptr; L.f.dbeta = b.train_b ? grads + b.b_off : nullptr; L.f.coef = b.coef;
  if (bi_ds >= 0) {
    BNL& d = bns[bi_ds];
    L.f.gamma2 = params + d.g_off; L.f.mean2 = d.mean; L.f.invstd2 = d.invstd;
    L.f.dgamma2 = d.train_g ? grads + d.g_off : nullptr; L.f.dbeta2 = d.train_b ? grads + d.b_off : nullptr;
    L.f.coef2 = d.coef;
  }
  return L;
}

// ---- forward -------------------------------------------------------------------
template <typename P>
int Net::forward_t(const float* x, const float* params, float* bufs, int B, int training, float droprate,
                   unsigned long long seed, unsigned long long step, float* pred, cudaStream_t st) {
  typedef typename P::A T;        // conv outputs
  typedef typename P::Z TZ;       // forward conv operands
  MN_TRY(ensure_tc_plans(B));
  // operand copies of the master weights (they change every optimizer step)
  if (precision == PREC_BF16_TC)
    MN_TRY(launch_pack_weights<bf16>(d_wdescs, (int)convs.size(), params, (bf16*)w_krsc, (bf16*)w_dg, max_w_elems, 0, st));
  else if (precision == PREC_TC_SPLIT)
    MN_TRY(launch_pack_weights_split(d_wdescs, (int)convs.size(), params, w_krsc_f32, w_dg_f32, w_krsc, w_dg, max_w_elems, st));
  else
    MN_TRY(launch_pack_weights<float>(d_wdescs, (int)convs.size(), params, (float*)w_krsc, (float*)w_dg, max_w_elems,
                                      precision == PREC_BF16_SIMT, st));
  // stem: im2col -> GEMM -> BN -> ReLU -> maxpool
  if (stem_s2d) {
    if constexpr (std::is_same<TZ, float>::value) { MN_CHECK(false, "forward: the space-to-depth stem is a tensor-core path feature"); }
    else MN_TRY(launch_stem_s2d<TZ>(x, (TZ*)A0, B, H, W, Hc + 3, stem_s2d_wsp(Wc), st));
  }
  else MN_TRY(launch_stem_im2col<TZ>(x, (TZ*)A0, B, H, W, Hc, Wc, kStemK, st));
  // lazy finalize: the conv epilogues accumulate into per-BatchNorm slots (zeroed here, once per step, for both passes)
  // and the consuming element-wise kernels finalize them -- no finalize launches
  const bool lazy = tc() && training;
  if (lazy) MN_CUDA(cudaMemsetAsync(bn_slots, 0, bn_slots_bytes, st));
  stats_target = lazy ? fwd_slot(convs[0].bn) : nullptr;
  MN_TRY(conv_fprop<P>(0, (const TZ*)A0, nullptr, (T*)y0, B, st));
  if (!lazy) MN_TRY(bn_forward<P>(convs[0].bn, (const T*)y0, (long long)B * Hc * Wc, params, bufs, training, st));
  MN_TRY((launch_stem_pool<T, TZ>((const T*)y0, (TZ*)z0, amax0, B, Hc, Wc, Hp, Wp, 64,
                                  lazy_forward(convs[0].bn, (long long)B * Hc * Wc, params, bufs, lazy), st)));
  const TZ* zin = (const TZ*)z0;
  for (auto& bl : blocks) {
    const long long Mo = (long long)B * bl.Ho * bl.Wo;
    const BnDesc l1 = lazy_forward(convs[bl.conv1].bn, Mo, params, bufs, lazy);
    const BnDesc l2 = lazy_forward(convs[bl.conv2].bn, Mo, params, bufs, lazy);
    stats_target = lazy ? fwd_slot(convs[bl.conv1].bn) : nullptr;
    MN_TRY(conv_fprop<P>(bl.conv1, zin, nullptr, (T*)bl.y1, B, st));
    if (!lazy) MN_TRY(bn_forward<P>(convs[bl.conv1].bn, (const T*)bl.y1, Mo, params, bufs, training, st));
    MN_TRY((launch_bn_apply<T, TZ>((const T*)bl.y1, 0, nullptr, (TZ*)bl.h, Mo, bl.Cout, 1, l1, nullptr, st)));
    stats_target = lazy ? fwd_slot(convs[bl.conv2].bn) : nullptr;
    MN_TRY(conv_fprop<P>(bl.conv2, (const TZ*)bl.h, nullptr, (T*)bl.y2, B, st));
    if (!lazy) MN_TRY(bn_forward<P>(convs[bl.conv2].bn, (const T*)bl.y2, Mo, params, bufs, training, st));
    if (bl.convd >= 0) {
      const BnDesc ld = lazy_forward(convs[bl.convd].bn, Mo, params, bufs, lazy);
      stats_target = lazy ? fwd_slot(convs[bl.convd].bn) : nullptr;
      MN_TRY(conv_fprop<P>(bl.convd, zin, nullptr, (T*)bl.yd, B, st));
      if (!lazy) MN_TRY(bn_forward<P>(convs[bl.convd].bn, (const T*)bl.yd, Mo, params, bufs, training, st));
      MN_TRY((launch_bn_apply<T, TZ>((const T*)bl.y2, 2, bl.yd, (TZ*)bl.out, Mo, bl.Cout, 1, l2, &ld, st)));
    } else {
      MN_TRY((launch_bn_apply<T, TZ>((const T*)bl.y2, 1, zin, (TZ*)bl.out, Mo, bl.Cout, 1, l2, nullptr, st)));
    }
    zin = (const TZ*)bl.out;
  }
  stats_target = nullptr;
  // head
  MN_TRY(launch_gap<TZ>(zin, feat, B, Hf * Wf, 512, st));
  MN_TRY(head_forward(head_params(params), feat, B, feat_dim, droprate, seed, step, drop_ctr,
                      (unsigned long long)max_B * feat_dim, mask, fcpre, hdrop, pred, st));
  last_B = B; last_training = training; last_has_mask = droprate > 0.f;
  bwd_next_part = 0;
  return 0;
}

// ---- backward ------------------------------------------------------------------
// The backward pass runs in up to three PARTS so that a data-parallel caller can start the allreduce of a part's
// gradients while the next part computes (geomapnet_b200/ddp.py): part 0 = head + layer4 (64 % of the parameters,
// final after 20 % of the backward FLOPs), part 1 = layer3, part 2 = layer2, layer1, stem.  part < 0: everything.
int Net::part_of_block(int bi) const { return blocks[bi].Cout >= 512 ? 0 : (blocks[bi].Cout >= 256 ? 1 : 2); }
void Net::part_range(int part, long long* lo, long long* hi) const {
  // float offsets into the flat parameter / gradient buffer; the table is in forward order, parts are contiguous
  long long first[3] = {n_params, n_params, 0};
  for (size_t bi = 0; bi < blocks.size(); ++bi) {
    const int p = part_of_block((int)bi);
    const long long off = convs[blocks[bi].conv1].wd.p_off;
    if (p < 2 && off < first[p]) first[p] = off;
  }
  if (part == 0) { *lo = first[0]; *hi = n_params; }
  else if (part == 1) { *lo = first[1]; *hi = first[0]; }
  else { *lo = 0; *hi = first[1]; }
}

template <typename P>
int Net::backward_t(const float* dpred, const float* params, float* grads, int filter_nans, int part, cudaStream_t st) {
  typedef typename P::A T;        // conv outputs, gradients w.r.t. block outputs (fp32 math tensors)
  typedef typename P::Z TZ;       // forward conv operands
  typedef typename P::G TG;       // backward conv operands (gradients w.r.t. conv outputs)
  MN_CHECK(last_B > 0 && last_training, "backward: no training-mode forward precedes this call");
  const int B = last_B;
  const int F = feat_dim;
  MN_CHECK(part <= 0 || bwd_next_part == part, "backward: part %d called out of order (next is %d)", part, bwd_next_part);
  bwd_next_part = (part < 0 || part == 2) ? 0 : part + 1;
  const bool do_head = part <= 0, do_stem = part < 0 || part == 2;
  // the wgrad engines ACCUMULATE (split-K atomics) straight into grads_flat -- conv weights are stored in the engines'
  // KRSC order there (mapnet_param_layout) -- except the stem, whose patch-matrix gradient is re-laid out from dw_krsc
  cur_grads = grads;
  if (do_head) {
    MN_CUDA(cudaMemsetAsync(grads, 0, (size_t)n_params * 4, st));
    MN_CUDA(cudaMemsetAsync(dw_krsc, 0, (size_t)dw_stem_elems * 4, st));
  }
  // S0: d(block output), S3: gated gradient of the identity branch, S4: d h -- T;  S1 / S2: d(conv output) -- TG
  // (S1 / S2 are slots of the ring the asynchronous wgrads read from: re-pointed before every write)
  T* S0 = (T*)scratch[0]; TG* S1 = (TG*)scratch[1]; TG* S2 = (TG*)scratch[2]; T* S3 = (T*)scratch[3]; T* S4 = (T*)scratch[4];

  // ---- head (models/posenet.py:67-73 backward, NaN filter :28-34) ----
  float* dpredh = dpredf + (size_t)max_B * 6;         // second filtered copy (gradient into the trunk)
  // strict mode: the backward conv operands are fp16 planes; ONE power-of-two scale per step (from max|d pred|)
  // places every gradient tensor inside fp16's window, the consuming conv epilogues divide it out again
  const float* gs = (precision == PREC_TC_SPLIT) ? gscale : nullptr;
  const bool trunk = bwd_lo < (int)blocks.size();       // a conv or BatchNorm parameter needs a gradient
  if (do_head) {
    HeadGrads hg;
    hg.fc_w = train_fc_w ? grads + fc_w : nullptr; hg.fc_b = train_fc_b ? grads + fc_b : nullptr;
    hg.xyz_w = train_xyz_w ? grads + xyz_w : nullptr; hg.xyz_b = train_xyz_b ? grads + xyz_b : nullptr;
    hg.wpqr_w = train_wpqr_w ? grads + wpqr_w : nullptr; hg.wpqr_b = train_wpqr_b ? grads + wpqr_b : nullptr;
    MN_TRY(head_backward(head_params(params), hg, dpred, filter_nans, feat, last_has_mask ? mask : nullptr, fcpre, hdrop,
                         B, F, dpredf, dpredh, (trunk && gs != nullptr) ? gscale : nullptr, dh, trunk ? dfeat : nullptr, st));
    if (trunk) MN_TRY(launch_gap_bwd<T>(dfeat, S0, B, Hf * Wf, 512, st));
    bwd_pre = false;
  }

  // ---- residual blocks, last to first ----
  // fuse_bwd (wgmma path): the dgrad that PRODUCES a BatchNorm's incoming gradient gates it with that
  // BN's ReLU and accumulates its backward reductions in the epilogue (conv_tc.cu, EpiBwd), so only the apply pass
  // remains, and it finalizes the sums itself (BnDesc).  `pre` = S0 arrives gated with the BN2 sums of this block pending.
  // Frozen parameters: the pass stops at the lowest block that trains (lo), and that block computes no gradient w.r.t.
  // its input (conv1 and downsample dgrad) unless the stem trains.
  bool pre = bwd_pre;
  const int lo = bwd_lo > 0 ? bwd_lo : 0;
  for (int bi = (int)blocks.size() - 1; bi >= lo; --bi) {
    if (part >= 0 && part_of_block(bi) != part) continue;
    BlockL& bl = blocks[bi];
    const bool dgrad_in = bi > bwd_lo;
    const TZ* zin = (bi == 0) ? (const TZ*)z0 : (const TZ*)blocks[bi - 1].out;
    const long long Mo = (long long)B * bl.Ho * bl.Wo;
    const int C = bl.Cout;
    BNL& b1 = bns[convs[bl.conv1].bn];
    const bool ds = bl.convd >= 0;
    const T* gres = S3;       // gated d out, the gradient of the identity branch
    // out = relu(bn2(y2) + idt): g = dout*[out>0]; BN2 (and downsample BN) backward.  With `pre`, S0 is already gated
    // and its sums are in the BN2 slot.
    S1 = (TG*)ring_next(st);
    if (ds) S2 = (TG*)ring_next(st);
    {
      const BnDesc d2 = lazy_backward(convs[bl.conv2].bn, ds ? convs[bl.convd].bn : -1, Mo, params, grads, pre);
      const TZ* zmask = pre ? nullptr : (const TZ*)bl.out;
      const T* yd = ds ? (const T*)bl.yd : nullptr;
      if (!pre) MN_TRY((launch_bn_bwd_reduce<T, TZ>(S0, zmask, (const T*)bl.y2, yd, Mo, C, d2.f, bn_accum, bn_counter, st)));
      // identity branch: the gated gradient is written to S3, unless S0 already holds it (conv1's dgrad adds it in place)
      T* gout = (ds || pre || !dgrad_in) ? nullptr : S3;
      MN_TRY((launch_bn_bwd_apply<T, TZ, TG>(S0, zmask, (const T*)bl.y2, S1, yd, ds ? S2 : nullptr, gout, Mo, C, d2, gs, st)));
      if (!ds && pre) gres = S0;
    }
    // conv2
    if (convs[bl.conv2].train) MN_TRY(conv_wgrad<P>(bl.conv2, (const TZ*)bl.h, S1, B, st));
    // h = relu(bn1(y1)) has no residual: its ReLU mask is recomputed from y1 (scale*y+shift > 0),
    // one tensor read less in both backward passes
    const TG* dy2 = S1;
    S1 = (TG*)ring_next(st);      // d y1 goes to a fresh slot: conv2's wgrad may still be reading d y2
    if (fuse_bwd) {
      EpiBwd e1; memset(&e1, 0, sizeof(e1));
      e1.y = (const bf16*)bl.y1; e1.mscale = b1.scale; e1.mshift = b1.shift;
      stats_target = bwd_slot(convs[bl.conv1].bn);
      MN_TRY(conv_dgrad<P>(bl.conv2, dy2, nullptr, S4, B, st, &e1));
      stats_target = nullptr;
      MN_TRY((launch_bn_bwd_apply<T, TZ, TG>(S4, nullptr, (const T*)bl.y1, S1, nullptr, nullptr, nullptr, Mo, C,
                                             lazy_backward(convs[bl.conv1].bn, -1, Mo, params, grads, true), gs, st)));
    } else {
      MN_TRY(conv_dgrad<P>(bl.conv2, dy2, nullptr, S4, B, st));
      BnDesc d1 = lazy_backward(convs[bl.conv1].bn, -1, Mo, params, grads, false);
      d1.f.mscale = b1.scale; d1.f.mshift = b1.shift;
      MN_TRY((launch_bn_bwd_reduce<T, TZ>(S4, nullptr, (const T*)bl.y1, nullptr, Mo, C, d1.f, bn_accum, bn_counter, st)));
      MN_TRY((launch_bn_bwd_apply<T, TZ, TG>(S4, nullptr, (const T*)bl.y1, S1, nullptr, nullptr, nullptr, Mo, C, d1, gs, st)));
    }
    // conv1 (+ downsample conv): d zin; with fuse_bwd it is gated by the previous block's output ReLU
    // and carries that block's BN2 (+ downsample BN) reductions
    // (armed only when block bi - 1 runs: otherwise nothing would consume the sums)
    const bool next_pre = fuse_bwd && bi > lo;
    EpiBwd e2; memset(&e2, 0, sizeof(e2));
    if (next_pre) {
      BlockL& pb = blocks[bi - 1];
      e2.y = (const bf16*)pb.y2; e2.zmask = (const bf16*)pb.out;
      e2.yd = (pb.convd >= 0) ? (const bf16*)pb.yd : nullptr;
      stats_target = bwd_slot(convs[pb.conv2].bn);      // consumed at the top of the next iteration
    }
    if (convs[bl.conv1].train) MN_TRY(conv_wgrad<P>(bl.conv1, zin, S1, B, st));
    if (ds && convs[bl.convd].train) MN_TRY(conv_wgrad<P>(bl.convd, zin, S2, B, st));
    if (dgrad_in && ds && bl.ds_fold) {
      MN_TRY(conv_dgrad<P>(bl.conv1, S1, nullptr, S0, B, st, next_pre ? &e2 : nullptr, S2, bl.convd));
    } else if (dgrad_in && ds) {
      MN_TRY(conv_dgrad<P>(bl.convd, S2, nullptr, S0, B, st));
      MN_TRY(conv_dgrad<P>(bl.conv1, S1, S0, S0, B, st, next_pre ? &e2 : nullptr));
    } else if (dgrad_in) {
      MN_TRY(conv_dgrad<P>(bl.conv1, S1, gres, S0, B, st, next_pre ? &e2 : nullptr));
    }
    stats_target = nullptr;
    pre = next_pre;
  }
  bwd_pre = pre;
  // ---- stem: maxpool -> ReLU -> BN -> conv (no input gradient: nothing consumes it) ----
  const bool stem = do_stem && bwd_lo < 0, stem_w = stem && convs[0].train;
  if (stem) {
    S2 = (TG*)ring_next(st);
    BNL& b0 = bns[convs[0].bn];
    const long long M0 = (long long)B * Hc * Wc;
    const BnDesc d0 = lazy_backward(convs[0].bn, -1, M0, params, grads, tc() && stem_fuse);
    if (stem_fuse) {
      // the pool/ReLU backward accumulates the stem BN's (sum g, sum g*y) while it has g and y in registers
      MN_TRY(launch_stem_pool_bwd<T>(S0, amax0, (const T*)y0, b0.scale, b0.shift, S4, B, Hc, Wc, Hp, Wp, 64, st,
                                     tc() ? bwd_slot(convs[0].bn) : bn_accum));
      if (!tc()) MN_TRY(launch_bn_bwd_finalize_accum(M0, 64, d0.f, bn_accum, st));
    } else {
      MN_TRY(launch_stem_pool_bwd<T>(S0, amax0, (const T*)y0, b0.scale, b0.shift, S4, B, Hc, Wc, Hp, Wp, 64, st));
      MN_TRY((launch_bn_bwd_reduce<T, TZ>(S4, (const TZ*)nullptr, (const T*)y0, nullptr, M0, 64, d0.f, bn_accum, bn_counter, st)));
    }
    MN_TRY((launch_bn_bwd_apply<T, TZ, TG>(S4, (const TZ*)nullptr, (const T*)y0, S2, nullptr, nullptr, nullptr, M0, 64, d0, gs, st)));
    if (stem_w) MN_TRY(conv_wgrad<P>(0, (const TZ*)A0, S2, B, st));
  }
  MN_TRY(wgrad_join(st));       // every asynchronous wgrad of this part has landed in grads_flat (the stem's in dw_krsc)
  if (stem_w) MN_TRY(launch_unpack_wgrads(d_wdescs, 1, dw_krsc, grads, max_w_elems, st));
  return 0;
}

int Net::forward(const float* x, const float* params, float* bufs, int B, int training, float droprate,
                 unsigned long long seed, unsigned long long step, float* pred, cudaStream_t st) {
  MN_CHECK(B >= 1 && B <= max_B, "forward: batch %d outside [1, max_B=%d]", B, max_B);
  MN_CHECK(x && params && bufs && pred, "forward: null pointer argument");
  MN_CHECK(droprate >= 0.f && droprate < 1.f, "forward: droprate %f outside [0,1)", droprate);
  if (precision == PREC_FP32) return forward_t<TypesF32>(x, params, bufs, B, training, droprate, seed, step, pred, st);
  if (precision == PREC_TC_SPLIT) return forward_t<TypesSplitHH>(x, params, bufs, B, training, droprate, seed, step, pred, st);
  return forward_t<TypesBF16>(x, params, bufs, B, training, droprate, seed, step, pred, st);
}

int Net::backward(const float* dpred, const float* params, float* grads, int filter_nans, int part, cudaStream_t st) {
  MN_CHECK(dpred && params && grads, "backward: null pointer argument");
  MN_CHECK(part >= -1 && part <= 2, "backward: part %d outside [-1, 2]", part);
  if (precision == PREC_FP32) return backward_t<TypesF32>(dpred, params, grads, filter_nans, part, st);
  if (precision == PREC_TC_SPLIT) return backward_t<TypesSplitHH>(dpred, params, grads, filter_nans, part, st);
  return backward_t<TypesBF16>(dpred, params, grads, filter_nans, part, st);
}

}  // namespace mapnet
