// Host-side plan of the PoseNet(ResNet-34) training step: parameter table,
// layer geometry, activation arena, forward / backward schedules.
#pragma once
#include <string>
#include <vector>

#include "kernels.h"
#include "bn_fin.cuh"

namespace mapnet {

// PREC_TC_SPLIT: strict tensor-core mode -- fp32-stored conv outputs, conv operands as split fp16 hi/lo planes (22
// significant bits), every product formed by 4 wgmma MMAs (hi*hi + hi*lo + lo*hi + lo*lo), fp32 accumulation
enum Precision { PREC_FP32 = 0, PREC_BF16_TC = 1, PREC_BF16_SIMT = 2, PREC_TC_SPLIT = 3 };

struct ParamEntry {
  std::string name;
  int kind;               // 0 trainable fp32 (params_flat), 1 fp32 buffer (bufs_flat), 2 int64 num_batches_tracked
  int layout;             // 0: elements in torch's contiguous order of `shape`; 1: conv weight [Co,Ci,KH,KW] stored as
                          //    [Co][KH][KW][Ci] (torch.channels_last strides) -- every conv except the stem
  int ndim;
  long long shape[4];
  long long numel;
  long long offset;       // element offset in its flat buffer (kind 2: index into the nbt vector)
};

struct ConvL {
  ConvGeom g;             // B filled per call; for the stem this is the 1x1 "GEMM" view over the im2col matrix
  WeightDesc wd;
  int bn;
};

struct BNL {
  int C;
  long long g_off, b_off, rm_off, rv_off;
  float *mean, *invstd, *scale, *shift, *coef;   // device, [C] each (coef [3C])
};

struct BlockL {
  int conv1, conv2, convd;       // indices into convs (convd = -1: identity)
  int Hi, Wi, Ho, Wo, Cin, Cout, stride;
  void *y1, *h, *y2, *yd, *out;  // activation buffers (T)
  int ds_fold;                   // the downsample dgrad is folded into conv1's dgrad launch (wgmma path)
};

struct Net {
  int max_B, H, W, feat_dim, precision;
  int Hc, Wc, Hp, Wp;            // stem conv / pooled sizes
  int Hf, Wf;                    // final feature map size
  std::vector<ParamEntry> table;
  long long n_params, n_bufs, n_nbt;
  std::vector<ConvL> convs;
  std::vector<BNL> bns;
  std::vector<BlockL> blocks;
  long long wk_total;            // packed weight elements
  int max_w_elems;
  // parameter offsets of the head
  long long fc_w, fc_b, xyz_w, xyz_b, wpqr_w, wpqr_b;

  // device memory owned by the handle
  std::vector<void*> allocs;
  void *A0, *y0, *z0; uint8_t* amax0;
  void* scratch[7]; long long scratch_elems;
  // Weight-gradient convolutions run on a second, LOW-priority stream: nothing in the backward chain waits for dW, so
  // they fill the SM time the chain leaves idle (latency-bound finalize / head / loss kernels, kernel tails) instead of
  // sitting in it.  The gradients they read (d conv output) rotate through a ring of four buffers; a slot is rewritten
  // only after the wgrad that read it has finished (event), and every part of the backward pass ends with a join.
  cudaStream_t side; int wgrad_async;
  void* ring[4]; cudaEvent_t ring_ready[4], ring_done[4]; bool ring_pending[4]; int ring_pos;
  void* ring_next(cudaStream_t st);
  int ring_slot(const void* p) const;
  int wgrad_join(cudaStream_t st);
  void *w_krsc, *w_dg; float* dw_krsc; WeightDesc* d_wdescs;
  float* cur_grads;              // grads_flat of the running backward pass
  long long dw_stem_elems;       // floats in dw_krsc (the stem's patch-matrix weight gradient)
  // where conv ci's wgrad engine accumulates: grads_flat at the parameter's offset (KRSC order), the stem in dw_krsc
  float* wgrad_out(int ci) { return ci == 0 ? dw_krsc : cur_grads + convs[ci].wd.p_off; }
  float *w_krsc_f32, *w_dg_f32;  // strict mode: fp32 K-major matrices the hi / lo weight planes are cut from
  int split_fmt_z, split_fmt_g;  // strict mode: element format of the forward / backward operand planes (0 fp16, 1 bf16)
  float* gscale;                 // strict mode, device: {S, 1/S} -- this step's power-of-two gradient scale
  double* bn_accum; unsigned int* bn_counter;
  // lazy BatchNorm finalize (bn_fin.cuh, BnLazy): one accumulator slot per BatchNorm and direction, zeroed once per step.
  // Slots 0..35 forward statistics, 36..71 backward reductions (8 replicas x [3][512] doubles each, what the conv
  // epilogues spread their flushes over), slot 72 (32 replicas) the stem's backward sums from the pool-backward kernel.
  double* bn_slots; size_t bn_slots_bytes;
  int lazy_fin;                  // consumers finalize the sums themselves (env MAPNET_BN_LAZY_FIN, tensor-core modes)
  double* stats_target;          // where the next conv_fprop / conv_dgrad with fused sums accumulates (nullptr: bn_accum)
  static constexpr int kSlotReplicas = 8, kStemBwdReplicas = 32, kSlotStride = 3 * 512;
  double* fwd_slot(int bn) { return bn_slots + (size_t)bn * kSlotReplicas * kSlotStride; }
  double* bwd_slot(int bn) { return bn_slots + (size_t)(bn == convs[0].bn ? 72 : 36 + bn) * kSlotReplicas * kSlotStride; }
  BnLazy lazy_forward(int bi, long long M, const float* params, float* bufs);
  BnLazy lazy_backward(int bi, int bi_ds, long long M, const float* params, float* grads);
  float *feat, *fcpre, *hdrop, *mask, *dh, *dfeat, *dpredf;
  float* bn_small;               // backing store of the BN small arrays
  float *sq_partials, *sq_out;
  unsigned long long* drop_ctr;  // device-side dropout step counter (graph capture)

  // tensor-core plans (precision == PREC_BF16_TC), rebuilt when B changes
  std::vector<TcConvPlan*> tc_fprop, tc_dgrad, tc_wgrad;
  int tc_B;

  // state of the last forward
  int last_B, last_training, last_has_mask;

  // optional per-conv-launch timing (bench.py roofline): CUDA events around every conv call
  struct ProfRec { cudaEvent_t e0, e1; int cls; double flops; };
  int profile_on;
  int stem_s2d;                  // stem conv on an overlapped view of the space-to-depth image (env MAPNET_STEM_S2D)
  int stem_fuse;                 // stem BN backward reductions inside the pool backward (env MAPNET_STEM_FUSE)
  int fuse_fin;                  // BN finalize inside the last CTA of the accumulating conv (env MAPNET_TC_FUSE_FIN)
  int fuse_bwd;                  // BN backward reductions accumulated in the dgrad epilogue (env MAPNET_TC_FUSE_BWD)
  int fuse_stats;                // BN statistics accumulated in the wgmma conv epilogue (env MAPNET_TC_FUSE_STATS)
  int ds_fold;                   // fold each 1x1/s2 downsample dgrad into its block's conv1 dgrad (env MAPNET_TC_DS_FOLD)
  std::vector<ProfRec> prof;
  std::vector<cudaEvent_t> prof_pool; size_t prof_pool_used;
  int prof_event(cudaEvent_t* e);
  int prof_reserve(int n_events);
  int prof_begin(cudaStream_t st, cudaEvent_t* e0);
  void prof_end(cudaStream_t st, cudaEvent_t e0, int cls, double flops);
  int prof_read(double* ms3, double* flops3, int* launches3);   // classes: 0 fprop, 1 dgrad, 2 wgrad

  size_t elt() const { return (precision == PREC_FP32 || precision == PREC_TC_SPLIT) ? 4 : 2; }
  bool tc() const { return precision == PREC_BF16_TC || precision == PREC_TC_SPLIT; }

  int init(int max_B, int H, int W, int feat_dim, int precision);
  void destroy();
  int forward(const float* x, const float* params, float* bufs, int B, int training, float droprate,
              unsigned long long seed, unsigned long long step, float* pred, cudaStream_t st);
  // part: -1 = the whole backward pass; 0, 1, 2 = its three parts, called in that order (net.cu: part_of_block)
  int backward(const float* dpred, const float* params, float* grads, int filter_nans, int part, cudaStream_t st);
  int part_of_block(int bi) const;
  void part_range(int part, long long* lo, long long* hi) const;
  bool bwd_pre; int bwd_next_part;      // state carried between the parts of one backward pass

 private:
  int alloc(void** p, size_t bytes);
  void build_table();
  // P: element-type bundle of the precision mode (common.cuh: TypesF32 / TypesBF16 / TypesSplitHH / TypesSplitHB)
  template <typename P> int forward_t(const float* x, const float* params, float* bufs, int B, int training,
                                      float droprate, unsigned long long seed, unsigned long long step,
                                      float* pred, cudaStream_t st);
  template <typename P> int backward_t(const float* dpred, const float* params, float* grads, int filter_nans,
                                       int part, cudaStream_t st);
  template <typename P> int conv_fprop(int ci, const typename P::Z* x, const typename P::A* residual, typename P::A* y, int B,
                                       cudaStream_t st, bool with_stats = false, const EpiFin* fin = nullptr);
  template <typename P> int conv_dgrad(int ci, const typename P::G* dy, const typename P::A* residual, typename P::A* dx, int B,
                                       cudaStream_t st, const EpiBwd* bwd = nullptr, const EpiFin* fin = nullptr,
                                       const typename P::G* dy_shortcut = nullptr, int ci_shortcut = -1);
  EpiFin fin_forward(int bi, long long M, const float* params, float* bufs);
  EpiFin fin_backward(int bi, int bi_ds, long long M, const float* params, float* grads);
  template <typename P> int conv_wgrad(int ci, const typename P::Z* x, const typename P::G* dy, int B, cudaStream_t st);
  template <typename P> int bn_forward(int bi, const typename P::A* y, long long M, const float* params, float* bufs,
                                       int training, cudaStream_t st);
  int ensure_tc_plans(int B);
};

}  // namespace mapnet
