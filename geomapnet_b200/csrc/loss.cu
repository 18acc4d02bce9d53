// Fused criterion forward + backward in ONE launch: absolute L1 pose loss and the
// relative-pose (VO) term -- calc_vos_simple (MapNet) or calc_vos in log-quaternion
// space (MapNet++), plus d loss/d pred and d loss/d (sax,saq,srx,srq).
// Replaces ~12 (PoseNet) to ~11 000 (MapNet++ fwd+bwd, N=16,T=5) ATen launches of
// /root/reference/common/criterion.py:42-52,76-109,137-184 and
// /root/reference/common/pose_utils.py:234-260 (SURVEY.md section 2c).  Latency-bound:
// one block, one thread per pose, warp-shuffle reductions, no atomics.
#include "kernels.h"
#include "loss_core.h"

#include "../../include/mapnet_b200.h"

namespace mapnet {

__global__ void __launch_bounds__(256)
k_loss(int mode, const float* __restrict__ pred, const float* __restrict__ targ, int N, int Tp, int Tt,
       const float* __restrict__ s4, float* __restrict__ loss, float* __restrict__ dpred,
       float* __restrict__ ds4) {
  pdl_prologue();
  __shared__ float red[8][4];
  float s[4] = {s4[0], s4[1], s4[2], s4[3]};
  const losscore::Cfg c = losscore::make_cfg(mode, N, Tp, Tt, s);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const int total = N * Tp;
  for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
    const int n = idx / Tp, i = idx - n * Tp;
    float g[6];
    losscore::pose_contrib(c, pred, targ, n, i, g, acc);
#pragma unroll
    for (int k = 0; k < 6; ++k) dpred[(long long)idx * 6 + k] = g[k];
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) acc[k] = warp_sum(acc[k]);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) red[w][k] = acc[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float sums[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ww = 0; ww < (int)(blockDim.x >> 5); ++ww)
#pragma unroll
      for (int k = 0; k < 4; ++k) sums[k] += red[ww][k];
    float L, ds[4];
    losscore::finalize(mode, N, Tp, s, sums, &L, ds);
    loss[0] = L;
#pragma unroll
    for (int k = 0; k < 4; ++k) ds4[k] = ds[k];
  }
}

int launch_loss(int mode, const float* pred, const float* targ, int N, int Tp, int Tt, const float* s4,
                float* loss, float* dpred, float* ds4, cudaStream_t st) {
  MN_CHECK(mode >= 0 && mode <= 3, "loss: bad mode %d", mode);
  MN_CHECK(N > 0 && Tp > 0 && Tt > 0, "loss: empty batch (N=%d Tp=%d Tt=%d)", N, Tp, Tt);
  if (mode == losscore::POSENET) MN_CHECK(Tp == 1 && Tt == 1, "loss: posenet mode wants [N,6] tensors");
  if (mode == losscore::MAPNET) MN_CHECK(Tt == Tp, "loss: mapnet mode wants targ [N,T,6] like pred");
  if (mode == losscore::ONLINE) MN_CHECK(Tp % 2 == 0 && Tt == Tp - 1, "loss: online mode wants pred [N,2T,6], targ [N,2T-1,6]");
  if (mode == losscore::ONLINE_GPS) MN_CHECK(Tp % 2 == 0 && Tt == Tp, "loss: online_gps mode wants pred, targ [N,2T,6]");
  MN_LAUNCH(k_loss, 1, 256, 0, st, mode, pred, targ, N, Tp, Tt, s4, loss, dpred, ds4);
  MN_LAUNCH_CHECK();
  return 0;
}

// The loss value of every batch of a validation pass: block b gathers the pred / targ rows of its items into shared
// memory as [N_b,T,6] and then runs k_loss's forward on them -- the same thread mapping, per-thread accumulation
// order and reduction tree -- so losses[b] is bit for bit what k_loss returns for that batch.  No atomics.
// d loss / d s4 is stored too (to a scratch row per batch): k_loss shares exp(-s) * mean between the loss and that
// gradient, and with the gradient dropped the compiler fuses the loss's multiply-add, which rounds differently.
__global__ void __launch_bounds__(256)
k_batch_losses(int mode, const float* __restrict__ pred, const float* __restrict__ targ,
               const int* __restrict__ pred_rows, const int* __restrict__ targ_rows, int T,
               const int* __restrict__ batch_items, const float* __restrict__ s4, float* __restrict__ losses,
               float* __restrict__ ds_scratch) {
  pdl_prologue();
  extern __shared__ float sm[];
  __shared__ float red[8][4];
  const int i0 = batch_items[blockIdx.x], N = batch_items[blockIdx.x + 1] - i0;
  const int total = N * T;
  float* sp = sm;
  float* st = sm + (size_t)total * 6;
  for (int r = threadIdx.x; r < total; r += blockDim.x) {
    const float* p = pred + 6LL * pred_rows[(long long)i0 * T + r];
    const float* t = targ + 6LL * targ_rows[(long long)i0 * T + r];
#pragma unroll
    for (int k = 0; k < 6; ++k) { sp[r * 6 + k] = p[k]; st[r * 6 + k] = t[k]; }
  }
  __syncthreads();
  float s[4] = {s4[0], s4[1], s4[2], s4[3]};
  const losscore::Cfg c = losscore::make_cfg(mode, N, T, T, s);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
    const int n = idx / T, i = idx - n * T;
    float g[6];
    losscore::pose_contrib(c, sp, st, n, i, g, acc);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) acc[k] = warp_sum(acc[k]);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) red[w][k] = acc[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float sums[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ww = 0; ww < (int)(blockDim.x >> 5); ++ww)
#pragma unroll
      for (int k = 0; k < 4; ++k) sums[k] += red[ww][k];
    float L, ds[4];
    losscore::finalize(mode, N, T, s, sums, &L, ds);
    losses[blockIdx.x] = L;
#pragma unroll
    for (int k = 0; k < 4; ++k) ds_scratch[blockIdx.x * 4 + k] = ds[k];
  }
}

static bool device_memory(const void* ptr) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, ptr) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

}  // namespace mapnet

using namespace mapnet;

extern "C" int mapnet_batch_losses(int mode, const float* pred, int n_pred, const float* targ, int n_targ,
                                   const int32_t* pred_rows, const int32_t* targ_rows, int T, const int32_t* batch_items,
                                   int n_batches, const float* s4, float* losses, void* stream) {
  MN_CHECK(pred && targ && pred_rows && targ_rows && batch_items && s4 && losses, "batch_losses: null argument");
  MN_CHECK(mode == losscore::POSENET || mode == losscore::MAPNET,
           "batch_losses: mode %d: only posenet (0) and mapnet (1) are validated", mode);
  MN_CHECK(T >= 1 && (mode != losscore::POSENET || T == 1), "batch_losses: T = %d (posenet mode wants T = 1)", T);
  MN_CHECK(n_batches >= 1 && n_pred >= 1 && n_targ >= 1, "batch_losses: bad count (%d batches, %d pred, %d targ rows)",
           n_batches, n_pred, n_targ);
  MN_CHECK(batch_items[0] == 0, "batch_losses: batch_items[0] = %d, must be 0", batch_items[0]);
  int max_rows = 0;
  for (int b = 0; b < n_batches; ++b) {
    MN_CHECK(batch_items[b + 1] > batch_items[b], "batch_losses: batch %d is empty or batch_items decrease (%d, %d)", b,
             batch_items[b], batch_items[b + 1]);
    const long long rows = (long long)(batch_items[b + 1] - batch_items[b]) * T;
    MN_CHECK(rows * 12 * sizeof(float) <= 200 * 1024, "batch_losses: batch %d has %lld poses (at most %d)", b, rows,
             (int)(200 * 1024 / (12 * sizeof(float))));
    if (rows > max_rows) max_rows = (int)rows;
  }
  const long long n_rows = (long long)batch_items[n_batches] * T;
  MN_CHECK(n_rows < (1LL << 30), "batch_losses: %lld rows", n_rows);
  for (long long r = 0; r < n_rows; ++r)
    MN_CHECK(pred_rows[r] >= 0 && pred_rows[r] < n_pred && targ_rows[r] >= 0 && targ_rows[r] < n_targ,
             "batch_losses: row %lld = (pred %d, targ %d) outside the %d predictions / %d targets", r, pred_rows[r],
             targ_rows[r], n_pred, n_targ);
  MN_CHECK(device_memory(pred) && device_memory(targ) && device_memory(s4) && device_memory(losses),
           "batch_losses: pred, targ, s4 and losses must be device memory");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = (size_t)max_rows * 12 * sizeof(float);
  if (smem > 48 * 1024) MN_CUDA(cudaFuncSetAttribute(k_batch_losses, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const size_t n_tab = 2 * (size_t)n_rows + n_batches + 1;
  int32_t* d = nullptr;                // the index tables and the ds scratch, stream-ordered: freed after the kernel
  MN_CUDA(cudaMallocAsync((void**)&d, (n_tab + 4 * (size_t)n_batches) * sizeof(int32_t), st));
  MN_CUDA(cudaMemcpyAsync(d, pred_rows, (size_t)n_rows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  MN_CUDA(cudaMemcpyAsync(d + n_rows, targ_rows, (size_t)n_rows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  MN_CUDA(cudaMemcpyAsync(d + 2 * n_rows, batch_items, (size_t)(n_batches + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  MN_LAUNCH(k_batch_losses, n_batches, 256, smem, st, mode, pred, targ, (const int*)d, (const int*)(d + n_rows), T,
            (const int*)(d + 2 * n_rows), s4, losses, (float*)(d + n_tab));
  MN_LAUNCH_CHECK();
  MN_CUDA(cudaFreeAsync(d, st));
  return 0;
}
