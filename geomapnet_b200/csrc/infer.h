// Eval-mode PoseNet(ResNet-34) inference engine: a frozen snapshot of the weights and BatchNorm running statistics
// and a forward-only schedule in which every BatchNorm (+ residual) (+ ReLU) runs inside its conv's wgmma epilogue.
// Precisions: bf16, tc_split, and fp8 (PREC_FP8: e4m3 operands for every conv but the stem, calibrated scales).
#pragma once
#include <vector>

#include "net.h"

namespace mapnet {

struct InferNet {
  Net spec;                      // parameter table and layer geometry (created with max_B = 0: owns no device memory)
  int max_B, H, W, feat_dim, precision;
  bool loaded;
  bool calibrated;               // fp8: activation scales taken for the current snapshot
  std::vector<void*> allocs;
  // snapshot (mapnet_infer_load)
  void* wk;                      // packed fprop operands only: bf16, or fp16 hi/lo planes (4 x 16-bit per element)
  WeightDesc* d_wdescs;
  float* affine;                 // per BatchNorm: scale[C], shift[C] (k_bn_eval_scale on the running statistics)
  std::vector<float*> bn_scale, bn_shift;
  float* head;                   // fp32 copy of fc, fc_xyz, fc_wpqr (weights and biases, flat-buffer layout)
  float* ident;                  // 64 ones, 64 zeros: the stem pool's affine (the conv epilogue already applied BN + ReLU)
  float* eval_scratch;           // mean / invstd outputs of k_bn_eval_scale (not kept)
  // fp8 snapshot: the stem keeps its bf16 operand in wk; every other conv reads e4m3 weights with a power-of-two scale
  // per output channel, and every e4m3 activation tensor (the pool output, each block's h and output: n_f8 of them, in
  // schedule order) has one power-of-two scale from calibration
  uint8_t* wk8;                  // e4m3 [Co][KH][KW][Ci] at each conv's k_off
  float* s_w;                    // [conv][512] weight scales
  float* f8_table;               // [conv][512] S = bn_scale * s_in * s_w: the epilogue's scale table (calibration)
  float* pool_map;               // the stem pool's affine map into layer1's e4m3 input: 64 x 1/s_pool, 64 x 0 (16-byte
                                 // aligned: read as float4), followed by f8_slots
  float* f8_slots;               // [n_f8] amax (bit patterns), [n_f8] s, [n_f8] 1/s
  int n_f8;
  // activation arena: stem operand, stem output, three rotating block tensors (input, h, output), downsample output
  void *A0, *y0, *act[3], *ds;
  float *feat, *fcpre, *hdrop, *mask;
  unsigned long long* drop_ctr;  // device dropout step counter (step == ~0: graph-capturable)
  std::vector<TcConvPlan*> plans;
  int plan_B;

  int init(int max_B, int H, int W, int feat_dim, int precision);
  void destroy();
  int load(const float* params, const float* bufs, cudaStream_t st);
  int forward(const float* x, int B, float droprate, unsigned long long seed, unsigned long long step, float* pred,
              cudaStream_t st);
  // the same forward on uint8 camera frames [B][Hin][Win][3] that pre resizes to (H, W) (mapnet_infer_forward_frames)
  int forward_frames(struct ::mapnet_preprocess* pre, const uint8_t* frames, int B, const float* mean3, const float* std3,
                     float droprate, unsigned long long seed, unsigned long long step, float* pred, cudaStream_t st);
  // S Monte-Carlo dropout draws of the head per frame, from one trunk forward (mapnet_infer_sample): samples [B,S,6]
  // (may be null), mean [B,6] and cov [B,6,6] in float64
  int sample(const float* x, int B, int S, float droprate, unsigned long long seed, unsigned long long step,
             float* samples, double* mean, double* cov, cudaStream_t st);
  int sample_frames(struct ::mapnet_preprocess* pre, const uint8_t* frames, int B, const float* mean3, const float* std3,
                    int S, float droprate, unsigned long long seed, unsigned long long step, float* samples,
                    double* mean, double* cov, cudaStream_t st);
  // fp8: the activation scales, progressively over the engine's own schedule on frames x [B,3,H,W] (B <= max_B)
  int calibrate(const float* x, int B, cudaStream_t st);
  int act_scales(float* host, int cap, cudaStream_t st);

  // bytes of the activation arena for max_B images (host-only: from the shapes); < 0 on a bad argument
  static long long arena_bytes(int max_B, int H, int W, int precision);

 private:
  struct Sizes { long long a0, y0, act, ds, head; };   // bytes per image
  static int sizes(const Net& spec, int precision, Sizes* s);
  static int f8_tensors(const Net& spec) { return 1 + 2 * (int)spec.blocks.size(); }
  static long long f8_slot_bytes(const Net& spec) { return 4LL * (3 * f8_tensors(spec) + 128); }
  int alloc(void** p, size_t bytes);
  int ensure_plans(int B);
  int stem_operand(const float* x, int B, cudaStream_t st);
  int check_frames(const char* what, struct ::mapnet_preprocess* pre, const uint8_t* frames, int B, const float* mean3,
                   const float* std3) const;
  int frames_operand(struct ::mapnet_preprocess* pre, const uint8_t* frames, int B, const float* mean3,
                     const float* std3, cudaStream_t st);
  int check_sample(const char* what, int S, float droprate, const double* mean, const double* cov) const;
  int trunk(int B, float droprate, unsigned long long seed, unsigned long long step, float* pred, cudaStream_t st);
  int features(int B, cudaStream_t st);           // stem conv .. global average pool: feat
  template <typename P> int forward_t(int B, cudaStream_t st);
  int conv(int ci, const void* in, const void* residual, void* out, int relu, int res_split, int out_split,
           cudaStream_t st);
  int run_head(int B, float droprate, unsigned long long seed, unsigned long long step, float* pred, cudaStream_t st);
  int sample_head(int B, int S, float droprate, unsigned long long seed, unsigned long long step, float* samples,
                  double* mean, double* cov, cudaStream_t st);
  // fp8 schedule (stem conv .. last block) on the stem operand A0; calib: take every tensor's scale first.  Returns the
  // index of the last block's output in act[] through *last.
  int run_f8(int B, bool calib, int* last, cudaStream_t st);
  int conv_f8(int ci, const void* in, int t_in, const void* res, int t_res, void* out, int t_out, int relu, bool calib,
              cudaStream_t st);
};

}  // namespace mapnet
