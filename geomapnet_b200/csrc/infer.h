// Eval-mode PoseNet(ResNet-34) inference engine: a frozen snapshot of the weights and BatchNorm running statistics
// and a forward-only schedule in which every BatchNorm (+ residual) (+ ReLU) runs inside its conv's wgmma epilogue.
#pragma once
#include <vector>

#include "net.h"

namespace mapnet {

struct InferNet {
  Net spec;                      // parameter table and layer geometry (created with max_B = 0: owns no device memory)
  int max_B, H, W, feat_dim, precision;
  bool loaded;
  std::vector<void*> allocs;
  // snapshot (mapnet_infer_load)
  void* wk;                      // packed fprop operands only: bf16, or fp16 hi/lo planes (4 x 16-bit per element)
  WeightDesc* d_wdescs;
  float* affine;                 // per BatchNorm: scale[C], shift[C] (k_bn_eval_scale on the running statistics)
  std::vector<float*> bn_scale, bn_shift;
  float* head;                   // fp32 copy of fc, fc_xyz, fc_wpqr (weights and biases, flat-buffer layout)
  float* ident;                  // 64 ones, 64 zeros: the stem pool's affine (the conv epilogue already applied BN + ReLU)
  float* eval_scratch;           // mean / invstd outputs of k_bn_eval_scale (not kept)
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

  // bytes of the activation arena for max_B images (host-only: from the shapes); < 0 on a bad argument
  static long long arena_bytes(int max_B, int H, int W, int precision);

 private:
  struct Sizes { long long a0, y0, act, ds, head; };   // bytes per image
  static int sizes(const Net& spec, Sizes* s);
  int alloc(void** p, size_t bytes);
  int ensure_plans(int B);
  template <typename P> int forward_t(const float* x, int B, float droprate, unsigned long long seed,
                                      unsigned long long step, float* pred, cudaStream_t st);
  int conv(int ci, const void* in, const void* residual, void* out, int relu, int res_split, int out_split,
           cudaStream_t st);
};

}  // namespace mapnet
