// Device-resident training set (geomapnet_b200/data/loader.py): every frame's Resize(256) output cached once in HBM,
// and the per-step batch assembly out of it (gather, ColorJitter, ToTensor + Normalize, targets) in one launch.
//
// Compiled with -fmad=false (geomapnet_b200/build.py): the VO targets are calc_vo_logq_safe
// (common/pose_utils.py:276-288) in float32, and without contracted multiply-adds the quaternion arithmetic of
// pose_math.h rounds where the reference's float32 torch / numpy code does (max error 6e-7 of max(|VO|, 1) against
// the reference, 1.0e-6 with contraction).  The pixel arithmetic uses explicit _rn intrinsics and is unaffected.
#include <cstring>

#include "kernels.h"
#include "preprocess_core.h"
#include "jitter_core.h"
#include "pose_math.h"
#include "pose_post.cuh"

#include "../../include/mapnet_b200.h"

namespace mapnet {

// ---- frame cache: the training set resized once (Resize(256) is deterministic and precedes ColorJitter, so its uint8
// output is what every epoch starts from), and the per-step batch assembly out of it.
struct TargRow { int a, b; };       // target row: b < 0 -> pose row a; else calc_vo_logq_safe(pose a, pose b)

// One image per blockIdx.y: gather frame frame_index[n] of the cache, [ColorJitter], ToTensor + Normalize, float32 NCHW
// into the caller's buffer.  Block (0, 0) also writes the n_targ target rows.
__global__ void __launch_bounds__(256)
k_loader_assemble(const uint8_t* __restrict__ frames, const int* __restrict__ frame_index,
                  const JitterParams* __restrict__ jp, const unsigned int* __restrict__ sums, float* __restrict__ out,
                  long long npix, float m0, float m1, float m2, float s0, float s1, float s2,
                  const float* __restrict__ poses, const TargRow* __restrict__ rows, int n_targ, float* __restrict__ targ) {
  pdl_prologue();
  const int n = blockIdx.y;
  if (blockIdx.x == 0 && n == 0) {
    for (int k = threadIdx.x; k < n_targ; k += blockDim.x) {
      const TargRow r = rows[k];
      const float* pa = poses + 6LL * r.a;
      float* o = targ + 6LL * k;
      if (r.b < 0) {
#pragma unroll
        for (int c = 0; c < 6; ++c) o[c] = pa[c];
      } else {
        const float* pb = poses + 6LL * r.b;
        posemath::Pose6 p0, p1;
        p0.t = posemath::v3(pa[0], pa[1], pa[2]); p0.l = posemath::v3(pa[3], pa[4], pa[5]);
        p1.t = posemath::v3(pb[0], pb[1], pb[2]); p1.l = posemath::v3(pb[3], pb[4], pb[5]);
        const posemath::Pose6 v = posemath::calc_vo_logq_safe(p0, p1);
        o[0] = v.t.x; o[1] = v.t.y; o[2] = v.t.z; o[3] = v.l.x; o[4] = v.l.y; o[5] = v.l.z;
      }
    }
  }
  const uint8_t* base = frames + (long long)frame_index[n] * npix * 3;
  const float mean[3] = {m0, m1, m2}, stdev[3] = {s0, s1, s2};
  float* dst = out + (long long)n * 3 * npix;
  if (jp == nullptr) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
#pragma unroll
      for (int c = 0; c < 3; ++c) dst[c * npix + i] = pre_normalize(base[3 * i + c], mean[c], stdev[c]);
    }
    return;
  }
  const JitterParams P = jp[n];
  // int(ImageStat.Stat(L).mean[0] + 0.5): double division of the exact integer sum
  const int gray_mean = (int)((double)sums[n] / (double)npix + 0.5);
  const uint8_t shift = jit_hue_shift(P.factor[JIT_HUE]);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    uint8_t px[3] = {base[3 * i], base[3 * i + 1], base[3 * i + 2]};
#pragma unroll
    for (int k = 0; k < 4; ++k) jit_apply(P.order[k], P.factor[P.order[k]], gray_mean, shift, px);
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[c * npix + i] = pre_normalize(px[c], mean[c], stdev[c]);
  }
}

// ---- evaluation windows (inference.evaluate_sequence): per-frame predictions -> the [L,T] windows scripts/eval.py
// post-processes.  Rows 0 .. n_win*T-1: pred7 / targ7 of window slot r; rows n_win*T .. +n_vo-1: VO k.  Translations
// stay normalised (PGO works on them), the quaternions are post_qexp of the float32 log q, as mapnet_pose_post.
__device__ __forceinline__ posemath::Pose6 ld_pose6(const float* p) {
  posemath::Pose6 o;
  o.t = posemath::v3(p[0], p[1], p[2]); o.l = posemath::v3(p[3], p[4], p[5]);
  return o;
}
__device__ __forceinline__ void st_pose7(const float* p6, double* o7) {
  o7[0] = (double)p6[0]; o7[1] = (double)p6[1]; o7[2] = (double)p6[2];
  post_qexp(p6[3], p6[4], p6[5], o7 + 3);
}

__global__ void __launch_bounds__(128)
k_eval_windows(const float* __restrict__ pred6, const float* __restrict__ poses, const float* __restrict__ vo_poses,
               const int* __restrict__ frame, const int* __restrict__ slot, int n_rows, const TargRow* __restrict__ vo_rows,
               int n_vo, double* __restrict__ pred7, double* __restrict__ targ7, double* __restrict__ vos7) {
  pdl_prologue();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n_rows) {
    st_pose7(pred6 + 6LL * slot[r], pred7 + 7LL * r);
    st_pose7(poses + 6LL * frame[r], targ7 + 7LL * r);
  } else if (r < n_rows + n_vo) {
    const int k = r - n_rows;
    const TargRow p = vo_rows[k];
    // calc_vos_safe / calc_vos_safe_fc (common/pose_utils.py:276-304) on the VO library's float32 poses, as the
    // MFOnline targets of k_loader_assemble
    const posemath::Pose6 v = posemath::calc_vo_logq_safe(ld_pose6(vo_poses + 6LL * p.a), ld_pose6(vo_poses + 6LL * p.b));
    const float v6[6] = {v.t.x, v.t.y, v.t.z, v.l.x, v.l.y, v.l.z};
    st_pose7(v6, vos7 + 7LL * k);
  }
}

}  // namespace mapnet

using namespace mapnet;

// Per-call records (frame indices, jitter records, target rows) go through a ring of staging slots, each a pinned host
// block and a device block with the same layout and an event that marks the assembly that last read it.  The host never
// waits unless it is kSlots calls ahead of the device, and assemblies may run on different streams.
struct mapnet_frame_cache {
  static constexpr int kSlots = 4;
  mapnet_preprocess_t* pre;           // the resize of one ingest chunk
  int chunk, Hout, Wout;
  int L, max_images, max_targ;
  uint8_t* frames;                    // [L][Hout][Wout][3]
  size_t slot_bytes, off_rows, off_idx, off_sums;
  uint8_t* host;                      // pinned, kSlots x slot_bytes
  uint8_t* dev;                       // kSlots x slot_bytes
  cudaEvent_t done[kSlots];
  int next;
};

extern "C" {

static bool device_memory(const void* ptr) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, ptr) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

int mapnet_frame_cache_create(mapnet_frame_cache_t** out, int n_frames, int Hin, int Win, int size, int chunk,
                              int max_images, int max_targ) {
  MN_CHECK(out != nullptr && n_frames >= 1 && chunk >= 1 && max_images >= 1 && max_targ >= 0,
           "frame_cache_create: bad argument");
  *out = nullptr;
  mapnet_preprocess_t* pre = nullptr;
  MN_TRY(mapnet_preprocess_create(&pre, Hin, Win, size, chunk));
  mapnet_frame_cache* h = new mapnet_frame_cache();
  h->pre = pre; h->chunk = chunk;
  mapnet_preprocess_output_size(pre, &h->Hout, &h->Wout);
  h->L = n_frames; h->max_images = max_images; h->max_targ = max_targ; h->next = 0;
  const size_t npix = (size_t)h->Hout * h->Wout;
  int r = 0;
  if (npix * 255 >= 4294967295ull) { set_last_error("frame_cache_create: image too large for the 32-bit luma sum"); r = 1; }
  h->off_rows = (size_t)max_images * sizeof(JitterParams);
  h->off_idx = h->off_rows + (size_t)max_targ * sizeof(TargRow);
  h->off_sums = h->off_idx + (size_t)max_images * sizeof(int);
  h->slot_bytes = (h->off_sums + (size_t)max_images * sizeof(unsigned int) + 255) / 256 * 256;
  if (r == 0 && cudaMalloc((void**)&h->frames, (size_t)n_frames * npix * 3) != cudaSuccess) {
    set_last_error("frame_cache_create: cudaMalloc of %d frames of %dx%d failed", n_frames, h->Hout, h->Wout); r = 1;
  }
  if (r == 0 && cudaMalloc((void**)&h->dev, h->slot_bytes * mapnet_frame_cache::kSlots) != cudaSuccess) {
    set_last_error("frame_cache_create: cudaMalloc of the staging slots failed"); r = 1;
  }
  if (r == 0 && cudaMallocHost((void**)&h->host, h->slot_bytes * mapnet_frame_cache::kSlots) != cudaSuccess) {
    set_last_error("frame_cache_create: cudaMallocHost of the staging slots failed"); r = 1;
  }
  for (int s = 0; r == 0 && s < mapnet_frame_cache::kSlots; ++s)
    if (cudaEventCreateWithFlags(&h->done[s], cudaEventDisableTiming) != cudaSuccess) {
      set_last_error("frame_cache_create: cudaEventCreate failed"); r = 1;
    }
  if (r != 0) { cudaGetLastError(); mapnet_frame_cache_destroy(h); return r; }
  *out = h;
  return 0;
}

int mapnet_frame_cache_ingest(mapnet_frame_cache_t* h, const void* frames_nhwc_u8, int first, int n, void* stream) {
  MN_CHECK(h != nullptr && frames_nhwc_u8 != nullptr, "frame_cache_ingest: null argument");
  MN_CHECK(n >= 1 && n <= h->chunk, "frame_cache_ingest: %d frames outside [1, chunk=%d]", n, h->chunk);
  MN_CHECK(first >= 0 && first <= h->L - n, "frame_cache_ingest: frames [%d, %d) outside the cache's [0, %d)", first,
           first + n, h->L);
  MN_CHECK(device_memory(frames_nhwc_u8), "frame_cache_ingest: frames must be device memory");
  return preprocess_resize_u8(h->pre, (const uint8_t*)frames_nhwc_u8, n, h->frames + (size_t)first * h->Hout * h->Wout * 3,
                              (cudaStream_t)stream);
}

int mapnet_frame_cache_assemble(mapnet_frame_cache_t* h, int n, const int32_t* frame_index, const void* jitter,
                                const float* poses_dev, int n_poses, const int32_t* targ_rows, int n_targ,
                                const float* mean3, const float* std3, float* out_nchw, float* targ_out, void* stream) {
  MN_CHECK(h != nullptr && frame_index != nullptr && mean3 != nullptr && std3 != nullptr && out_nchw != nullptr,
           "frame_cache_assemble: null argument");
  MN_CHECK(n >= 1 && n <= h->max_images, "frame_cache_assemble: %d images outside [1, max_images=%d]", n, h->max_images);
  MN_CHECK(n_targ >= 0 && n_targ <= h->max_targ, "frame_cache_assemble: %d target rows outside [0, max_targ=%d]", n_targ,
           h->max_targ);
  for (int c = 0; c < 3; ++c) MN_CHECK(std3[c] > 0.f, "frame_cache_assemble: std[%d] = %f must be positive", c, std3[c]);
  for (int i = 0; i < n; ++i)
    MN_CHECK(frame_index[i] >= 0 && frame_index[i] < h->L, "frame_cache_assemble: frame_index[%d] = %d outside [0, %d)", i,
             frame_index[i], h->L);
  const JitterParams* jp = (const JitterParams*)jitter;
  for (int i = 0; jp != nullptr && i < n; ++i) {
    int seen = 0;
    for (int k = 0; k < 4; ++k) if (jp[i].order[k] >= 0 && jp[i].order[k] < 4) seen |= 1 << jp[i].order[k];
    MN_CHECK(seen == 15, "frame_cache_assemble: jitter record %d: order is not a permutation of 0..3", i);
  }
  const TargRow* rows = (const TargRow*)targ_rows;
  if (n_targ > 0) {
    MN_CHECK(poses_dev != nullptr && targ_rows != nullptr && targ_out != nullptr, "frame_cache_assemble: null target argument");
    for (int k = 0; k < n_targ; ++k)
      MN_CHECK(rows[k].a >= 0 && rows[k].a < n_poses && rows[k].b >= -1 && rows[k].b < n_poses,
               "frame_cache_assemble: target row %d = (%d, %d) outside the %d poses", k, rows[k].a, rows[k].b, n_poses);
    MN_CHECK(device_memory(poses_dev) && device_memory(targ_out), "frame_cache_assemble: poses / targets must be device memory");
  }
  MN_CHECK(device_memory(out_nchw), "frame_cache_assemble: out must be device memory");
  cudaStream_t st = (cudaStream_t)stream;
  const int s = h->next;
  h->next = (s + 1) % mapnet_frame_cache::kSlots;
  MN_CUDA(cudaEventSynchronize(h->done[s]));     // the assembly that last read this slot has finished
  uint8_t* hs = h->host + (size_t)s * h->slot_bytes;
  uint8_t* ds = h->dev + (size_t)s * h->slot_bytes;
  if (jp != nullptr) memcpy(hs, jp, (size_t)n * sizeof(JitterParams));
  if (n_targ > 0) memcpy(hs + h->off_rows, rows, (size_t)n_targ * sizeof(TargRow));
  memcpy(hs + h->off_idx, frame_index, (size_t)n * sizeof(int));
  MN_CUDA(cudaMemcpyAsync(ds, hs, h->off_sums, cudaMemcpyHostToDevice, st));
  const long long npix = (long long)h->Hout * h->Wout;
  int gx = (int)((npix + 255) / 256); if (gx > 64) gx = 64;
  const int* d_idx = (const int*)(ds + h->off_idx);
  const JitterParams* d_jp = jp != nullptr ? (const JitterParams*)ds : nullptr;
  unsigned int* d_sums = (unsigned int*)(ds + h->off_sums);
  if (jp != nullptr) {
    MN_CUDA(cudaMemsetAsync(d_sums, 0, (size_t)n * sizeof(unsigned int), st));
    MN_TRY(launch_jitter_luma_sum(h->frames, d_idx, d_jp, d_sums, npix, n, gx, st));
  }
  MN_LAUNCH(k_loader_assemble, dim3(gx, n), 256, 0, st, (const uint8_t*)h->frames, d_idx, d_jp, (const unsigned int*)d_sums,
            out_nchw, npix, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2], poses_dev,
            (const TargRow*)(ds + h->off_rows), n_targ, targ_out);
  MN_LAUNCH_CHECK();
  MN_CUDA(cudaEventRecord(h->done[s], st));
  return 0;
}

int mapnet_eval_windows(const float* pred6, int n_pred, const float* poses, const float* vo_poses, int n_poses,
                        const int32_t* frame, const int32_t* slot, int n_rows, const int32_t* vo_rows, int n_vo,
                        double* pred7, double* targ7, double* vos7, void* stream) {
  MN_CHECK(pred6 != nullptr && poses != nullptr && frame != nullptr && slot != nullptr && pred7 != nullptr &&
           targ7 != nullptr, "eval_windows: null argument");
  MN_CHECK(n_rows >= 1 && n_pred >= 1 && n_poses >= 1 && n_vo >= 0, "eval_windows: bad count");
  MN_CHECK(n_vo == 0 || (vo_poses != nullptr && vo_rows != nullptr && vos7 != nullptr),
           "eval_windows: %d VO rows need vo_poses, vo_rows and vos7", n_vo);
  MN_CHECK((long long)n_rows + n_vo < (1LL << 31), "eval_windows: %d + %d rows", n_rows, n_vo);
  for (int r = 0; r < n_rows; ++r)
    MN_CHECK(frame[r] >= 0 && frame[r] < n_poses && slot[r] >= 0 && slot[r] < n_pred,
             "eval_windows: row %d = (frame %d, slot %d) outside the %d poses / %d predictions", r, frame[r], slot[r],
             n_poses, n_pred);
  for (int k = 0; k < 2 * n_vo; ++k)
    MN_CHECK(vo_rows[k] >= 0 && vo_rows[k] < n_poses, "eval_windows: VO row %d = (%d, %d) outside the %d poses", k / 2,
             vo_rows[k & ~1], vo_rows[k | 1], n_poses);
  MN_CHECK(device_memory(pred6) && device_memory(poses) && device_memory(pred7) && device_memory(targ7) &&
           (n_vo == 0 || (device_memory(vo_poses) && device_memory(vos7))), "eval_windows: tensors must be device memory");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t bytes = (2 * (size_t)n_rows + 2 * (size_t)n_vo) * sizeof(int32_t);
  int32_t* d = nullptr;                // the index tables, stream-ordered: freed once the kernel has read them
  MN_CUDA(cudaMallocAsync((void**)&d, bytes, st));
  MN_CUDA(cudaMemcpyAsync(d, frame, (size_t)n_rows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  MN_CUDA(cudaMemcpyAsync(d + n_rows, slot, (size_t)n_rows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (n_vo > 0) MN_CUDA(cudaMemcpyAsync(d + 2 * n_rows, vo_rows, 2 * (size_t)n_vo * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  MN_LAUNCH(k_eval_windows, (int)cdiv((long long)n_rows + n_vo, 128), 128, 0, st, pred6, poses, vo_poses, (const int*)d,
            (const int*)(d + n_rows), n_rows, (const TargRow*)(d + 2 * n_rows), n_vo, pred7, targ7, vos7);
  MN_LAUNCH_CHECK();
  MN_CUDA(cudaFreeAsync(d, st));
  return 0;
}

int mapnet_frame_cache_destroy(mapnet_frame_cache_t* h) {
  if (h == nullptr) return 0;
  for (int s = 0; s < mapnet_frame_cache::kSlots; ++s)
    if (h->done[s] != nullptr) { cudaEventSynchronize(h->done[s]); cudaEventDestroy(h->done[s]); }
  mapnet_preprocess_destroy(h->pre);
  cudaFree(h->frames); cudaFree(h->dev); cudaFreeHost(h->host);
  delete h;
  return 0;
}

}  // extern "C"
