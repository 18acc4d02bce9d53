// GPU-side input pipeline (SURVEY.md section 8 row f2): the arithmetic is checked bit-exactly on the CPU against
// Pillow / torchvision through tests/_hostpre.cpp, the kernels against torchvision on the GPU (tests/test_gpu_preprocess.py).
//
// Replaces, for a batch of equally sized uint8 frames already in device memory, the per-image CPU transform stack
// of /root/reference/scripts/train.py:119-128 / scripts/eval.py:97-101:
//   transforms.Resize(256) (Pillow bilinear, 8-bit fixed point, two passes) [-> ColorJitter] -> ToTensor ->
//   Normalize(mean, sqrt(var)),
// and the frame gather of the MF / MFOnline tuple datasets (dataset_loaders/composite.py:60-97,117-126): output image
// n is cut from frame frame_index[n] of a device-resident sequence, so a [N,T,3,H',W'] batch of tuples is ONE call.
// ColorJitter (jitter_core.h) needs the mean luma of each image in its state just before the contrast adjustment, so the
// jitter path is: vertical pass -> uint8 image; a reduction pass that applies the adjustments preceding contrast on the
// fly and sums the luma per image; a final pass that applies all four adjustments + ToTensor + Normalize.
// At ~15 k img/s per GPU the reference's 5 DataLoader workers (mapnet.ini:13) fall short by two orders of magnitude.
//
// HBM-bound byte work: a 640x480 frame is 0.92 MB in, 0.26 MB of intermediate, 1.05 MB (fp32 CHW) out.  Pass 1
// (horizontal) and pass 2 (vertical + ToTensor + Normalize) are separate kernels because Pillow rounds to uint8
// between the passes; consecutive threads walk consecutive output columns, so pass-2 stores are fully coalesced
// and pass-1 / pass-2 loads hit the same few source rows from L1/L2.
#include "kernels.h"
#include "preprocess_core.h"
#include "jitter_core.h"

#include "../../include/mapnet_b200.h"

namespace mapnet {

struct PreprocessPlan {
  int Hin, Win, Hout, Wout, ksh, ksv, max_images;
  int *d_bh, *d_kh, *d_bv, *d_kv;     // bounds / fixed-point weights of the two passes
  uint8_t* d_tmp;                     // [max_images][Hin][Wout][3] after the horizontal pass
  uint8_t* d_u8;                      // [max_images][Hout][Wout][3] resized image (jitter path), allocated on first use
  unsigned int* d_sums;               // [max_images] luma sums (jitter path)
};

__global__ void __launch_bounds__(256)
k_pre_resize_h(const uint8_t* __restrict__ img, const int* __restrict__ frame_index, uint8_t* __restrict__ tmp,
               const int* __restrict__ bounds, const int* __restrict__ kk, int ksize, long long rows /* n*Hin */, int Hin,
               int Win, int Wout) {
  pdl_prologue();
  const long long total = rows * Wout;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xx = (int)(i % Wout);
    const long long row = i / Wout;
    const int xmin = bounds[2 * xx], n = bounds[2 * xx + 1];
    long long srow = row;
    if (frame_index != nullptr) {       // tuple gather: output image row / Hin is cut from frame frame_index[.]
      const long long im = row / Hin;
      srow = (long long)frame_index[im] * Hin + (row - im * Hin);
    }
    const uint8_t* src = img + (srow * Win + xmin) * 3;
    const int* k = kk + (long long)xx * ksize;
    uint8_t* dst = tmp + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[c] = pre_resample(src + c, 3, n, k);
  }
}

__global__ void __launch_bounds__(256)
k_pre_resize_v_norm(const uint8_t* __restrict__ tmp, float* __restrict__ out, uint8_t* __restrict__ out_u8,
                    const int* __restrict__ bounds, const int* __restrict__ kk, int ksize, int nimg, int Hin, int Hout,
                    int Wout, float m0, float m1, float m2, float s0, float s1, float s2) {
  pdl_prologue();
  const long long total = (long long)nimg * Hout * Wout;
  const float mean[3] = {m0, m1, m2}, stdev[3] = {s0, s1, s2};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xx = (int)(i % Wout);
    const long long r = i / Wout;
    const int yy = (int)(r % Hout);
    const long long n = r / Hout;
    const int ymin = bounds[2 * yy], cnt = bounds[2 * yy + 1];
    const uint8_t* src = tmp + ((n * Hin + ymin) * Wout + xx) * 3;
    const int* k = kk + (long long)yy * ksize;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const uint8_t u = pre_resample(src + c, (long long)Wout * 3, cnt, k);
      if (out != nullptr) out[((n * 3 + c) * Hout + yy) * Wout + xx] = pre_normalize(u, mean[c], stdev[c]);
      if (out_u8 != nullptr) out_u8[i * 3 + c] = u;
    }
  }
}

// Inference from camera frames: pass 2 (vertical resample + ToTensor + Normalize) written straight into the inference
// engine's space-to-depth stem operand, the layout of k_stem_s2d (layout.cu): S[b][bh][bw][16], channel (pr*2+pc)*3+c
// of block (bh, bw) is pixel (2*bh+pr-4, 2*bw+pc-4) of the resized image, zero outside it and in channels 12..15.  The
// float32 image is never stored: each value is the pre_normalize result k_stem_s2d would have read, converted once by
// the same Vec8 store, so S is bitwise what k_stem_s2d writes over k_pre_resize_v_norm's output.  One thread per 2x2
// block: a warp reads 32 consecutive 6-byte pixel pairs of each intermediate row it needs and writes 32 consecutive
// blocks (1 KB in bf16).
template <typename TZ>
__global__ void __launch_bounds__(256)
k_pre_resize_v_s2d(const uint8_t* __restrict__ tmp, TZ* __restrict__ S, const int* __restrict__ bounds,
                   const int* __restrict__ kk, int ksize, int nimg, int Hin, int Hout, int Wout, int Hs, int Wsp,
                   float m0, float m1, float m2, float s0, float s1, float s2) {
  pdl_prologue();
  const long long total = (long long)nimg * Hs * Wsp;
  const float mean[3] = {m0, m1, m2}, stdev[3] = {s0, s1, s2};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int bw = (int)(i % Wsp);
    const long long r = i / Wsp;
    const int bh = (int)(r % Hs);
    const long long n = r / Hs;
    float v[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) v[k] = 0.f;
#pragma unroll
    for (int pr = 0; pr < 2; ++pr) {
      const int yy = 2 * bh + pr - 4;
      if (yy < 0 || yy >= Hout) continue;
      const int ymin = bounds[2 * yy], cnt = bounds[2 * yy + 1];
      const int* k = kk + (long long)yy * ksize;
#pragma unroll
      for (int pc = 0; pc < 2; ++pc) {
        const int xx = 2 * bw + pc - 4;
        if (xx < 0 || xx >= Wout) continue;
        const uint8_t* src = tmp + ((n * Hin + ymin) * Wout + xx) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c)
          v[(pr * 2 + pc) * 3 + c] = pre_normalize(pre_resample(src + c, (long long)Wout * 3, cnt, k), mean[c], stdev[c]);
      }
    }
    Vec8<TZ> o0, o1;
#pragma unroll
    for (int k = 0; k < 8; ++k) { o0.v[k] = v[k]; o1.v[k] = v[8 + k]; }
    o0.store(S + i * 16);
    o1.store(S + i * 16 + 8);
  }
}

// ColorJitter, pass A: per image, the luma sum of the image in its state just before the contrast adjustment.
// frame_index: nullptr (image n is image n of u8) or the frame cache's gather (image n is frame frame_index[n])
__global__ void __launch_bounds__(256)
k_jitter_luma_sum(const uint8_t* __restrict__ u8, const int* __restrict__ frame_index, const JitterParams* __restrict__ jp,
                  unsigned int* __restrict__ sums, long long npix /* per image */) {
  pdl_prologue();
  const int n = blockIdx.y;
  const JitterParams P = jp[n];
  int npre = 0;
  while (npre < 4 && P.order[npre] != JIT_CONTRAST) ++npre;
  const uint8_t shift = jit_hue_shift(P.factor[JIT_HUE]);
  unsigned int acc = 0;
  const uint8_t* base = u8 + (long long)(frame_index != nullptr ? frame_index[n] : n) * npix * 3;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    uint8_t px[3] = {base[3 * i], base[3 * i + 1], base[3 * i + 2]};
    for (int k = 0; k < npre; ++k) jit_apply(P.order[k], P.factor[P.order[k]], 0, shift, px);
    acc += jit_luma(px[0], px[1], px[2]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc != 0) atomicAdd(sums + n, acc);
}

// ColorJitter, pass B: all four adjustments in the image's order, then ToTensor + Normalize
__global__ void __launch_bounds__(256)
k_jitter_norm(const uint8_t* __restrict__ u8, const JitterParams* __restrict__ jp, const unsigned int* __restrict__ sums,
              float* __restrict__ out, uint8_t* __restrict__ out_u8, int Hout, int Wout, float m0, float m1, float m2,
              float s0, float s1, float s2) {
  pdl_prologue();
  const int n = blockIdx.y;
  const long long npix = (long long)Hout * Wout;
  const JitterParams P = jp[n];
  // int(ImageStat.Stat(L).mean[0] + 0.5): double division of the exact integer sum
  const int gray_mean = (int)((double)sums[n] / (double)npix + 0.5);
  const uint8_t shift = jit_hue_shift(P.factor[JIT_HUE]);
  const float mean[3] = {m0, m1, m2}, stdev[3] = {s0, s1, s2};
  const uint8_t* base = u8 + (long long)n * npix * 3;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    uint8_t px[3] = {base[3 * i], base[3 * i + 1], base[3 * i + 2]};
#pragma unroll
    for (int k = 0; k < 4; ++k) jit_apply(P.order[k], P.factor[P.order[k]], gray_mean, shift, px);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      out[((long long)n * 3 + c) * npix + i] = pre_normalize(px[c], mean[c], stdev[c]);
      if (out_u8 != nullptr) out_u8[((long long)n * npix + i) * 3 + c] = px[c];
    }
  }
}

static int upload(const std::vector<int>& v, int** d) {
  MN_CUDA(cudaMalloc((void**)d, v.size() * sizeof(int)));
  MN_CUDA(cudaMemcpy(*d, v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice));
  return 0;
}

}  // namespace mapnet

using namespace mapnet;

struct mapnet_preprocess {
  PreprocessPlan p;
};

namespace mapnet {
// ---- used by the frame cache (loader.cu) --------------------------------------------------------------------------
// Resize n frames (n <= the plan's max_images) into uint8 [n][Hout][Wout][3] at out_u8.
int preprocess_resize_u8(mapnet_preprocess_t* h, const uint8_t* img, int n, uint8_t* out_u8, cudaStream_t st) {
  PreprocessPlan& p = h->p;
  MN_CHECK(n >= 1 && n <= p.max_images, "preprocess_resize_u8: %d images outside [1, max_images=%d]", n, p.max_images);
  const long long t1 = (long long)n * p.Hin * p.Wout, t2 = (long long)n * p.Hout * p.Wout;
  const int g1 = (int)((t1 + 255) / 256 < (long long)kNumSMs * 16 ? (t1 + 255) / 256 : (long long)kNumSMs * 16);
  const int g2 = (int)((t2 + 255) / 256 < (long long)kNumSMs * 16 ? (t2 + 255) / 256 : (long long)kNumSMs * 16);
  MN_LAUNCH(k_pre_resize_h, g1, 256, 0, st, img, (const int*)nullptr, p.d_tmp, p.d_bh, p.d_kh, p.ksh, (long long)n * p.Hin,
            p.Hin, p.Win, p.Wout);
  MN_LAUNCH_CHECK();
  MN_LAUNCH(k_pre_resize_v_norm, g2, 256, 0, st, p.d_tmp, (float*)nullptr, out_u8, p.d_bv, p.d_kv, p.ksv, n, p.Hin, p.Hout,
            p.Wout, 0.f, 0.f, 0.f, 1.f, 1.f, 1.f);
  MN_LAUNCH_CHECK();
  return 0;
}
int launch_jitter_luma_sum(const uint8_t* u8, const int* frame_index, const JitterParams* jp, unsigned int* sums,
                           long long npix, int n, int gx, cudaStream_t st) {
  MN_LAUNCH(k_jitter_luma_sum, dim3(gx, n), 256, 0, st, u8, frame_index, jp, sums, npix);
  MN_LAUNCH_CHECK();
  return 0;
}

// ---- used by the inference engine (infer.cu) ----------------------------------------------------------------------
int preprocess_geometry(const mapnet_preprocess_t* h, int* Hout, int* Wout, int* max_images) {
  MN_CHECK(h != nullptr, "preprocess: null plan");
  *Hout = h->p.Hout; *Wout = h->p.Wout; *max_images = h->p.max_images;
  return 0;
}
template <typename TZ>
int preprocess_stem_s2d(mapnet_preprocess_t* h, const uint8_t* img, int n, const float* mean3, const float* std3, TZ* S,
                        int Hs, int Wsp, cudaStream_t st) {
  MN_CHECK(h != nullptr && img != nullptr && mean3 != nullptr && std3 != nullptr && S != nullptr,
           "preprocess_stem_s2d: null argument");
  PreprocessPlan& p = h->p;
  MN_CHECK(n >= 1 && n <= p.max_images, "preprocess_stem_s2d: %d images outside [1, max_images=%d]", n, p.max_images);
  for (int c = 0; c < 3; ++c) MN_CHECK(std3[c] > 0.f, "preprocess_stem_s2d: std[%d] = %f must be positive", c, std3[c]);
  const long long t1 = (long long)n * p.Hin * p.Wout, t2 = (long long)n * Hs * Wsp;
  const int g1 = (int)((t1 + 255) / 256 < (long long)kNumSMs * 16 ? (t1 + 255) / 256 : (long long)kNumSMs * 16);
  const int g2 = (int)((t2 + 255) / 256 < (long long)kNumSMs * 16 ? (t2 + 255) / 256 : (long long)kNumSMs * 16);
  MN_LAUNCH(k_pre_resize_h, g1, 256, 0, st, img, (const int*)nullptr, p.d_tmp, p.d_bh, p.d_kh, p.ksh, (long long)n * p.Hin,
            p.Hin, p.Win, p.Wout);
  MN_LAUNCH_CHECK();
  MN_LAUNCH(k_pre_resize_v_s2d<TZ>, g2, 256, 0, st, (const uint8_t*)p.d_tmp, S, (const int*)p.d_bv, (const int*)p.d_kv,
            p.ksv, n, p.Hin, p.Hout, p.Wout, Hs, Wsp, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2]);
  MN_LAUNCH_CHECK();
  return 0;
}
template int preprocess_stem_s2d<bf16>(mapnet_preprocess_t*, const uint8_t*, int, const float*, const float*, bf16*, int,
                                       int, cudaStream_t);
template int preprocess_stem_s2d<hsplit>(mapnet_preprocess_t*, const uint8_t*, int, const float*, const float*, hsplit*,
                                         int, int, cudaStream_t);
}  // namespace mapnet


extern "C" {

int mapnet_preprocess_create(mapnet_preprocess_t** out, int Hin, int Win, int size, int max_images) {
  MN_CHECK(out != nullptr && Hin >= 1 && Win >= 1 && size >= 1 && max_images >= 1, "preprocess_create: bad argument");
  *out = nullptr;
  int ndev = 0;
  MN_CHECK(cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0, "preprocess_create: no CUDA device (this library has no CPU fallback)");
  mapnet_preprocess* h = new mapnet_preprocess();
  PreprocessPlan& p = h->p;
  memset(&p, 0, sizeof(p));
  p.Hin = Hin; p.Win = Win; p.max_images = max_images;
  pre_resize_output_size(Hin, Win, size, &p.Hout, &p.Wout);
  std::vector<int> bh, kh, bv, kv;
  p.ksh = pre_compute_coeffs(Win, p.Wout, bh, kh);
  p.ksv = pre_compute_coeffs(Hin, p.Hout, bv, kv);
  int r = upload(bh, &p.d_bh);
  if (r == 0) r = upload(kh, &p.d_kh);
  if (r == 0) r = upload(bv, &p.d_bv);
  if (r == 0) r = upload(kv, &p.d_kv);
  if (r == 0 && cudaMalloc((void**)&p.d_tmp, (size_t)max_images * Hin * p.Wout * 3) != cudaSuccess) {
    set_last_error("preprocess_create: cudaMalloc of the intermediate image failed");
    r = 1;
  }
  if (r != 0) { mapnet_preprocess_destroy(h); return r; }
  *out = h;
  return 0;
}

int mapnet_preprocess_output_size(const mapnet_preprocess_t* h, int* Hout, int* Wout) {
  MN_CHECK(h != nullptr && Hout != nullptr && Wout != nullptr, "preprocess_output_size: null argument");
  *Hout = h->p.Hout; *Wout = h->p.Wout;
  return 0;
}

int mapnet_preprocess_run(mapnet_preprocess_t* h, const void* img_nhwc_u8, int n, const float* mean3, const float* std3,
                          float* out_nchw, void* out_u8_or_null, void* stream) {
  return mapnet_preprocess_run_ex(h, img_nhwc_u8, n, nullptr, nullptr, mean3, std3, out_nchw, out_u8_or_null, stream);
}

int mapnet_preprocess_run_ex(mapnet_preprocess_t* h, const void* img_nhwc_u8, int n, const int32_t* frame_index_dev,
                             const void* jitter_dev, const float* mean3, const float* std3, float* out_nchw,
                             void* out_u8_or_null, void* stream) {
  MN_CHECK(h != nullptr && img_nhwc_u8 != nullptr && mean3 != nullptr && std3 != nullptr && out_nchw != nullptr,
           "preprocess_run: null argument");
  PreprocessPlan& p = h->p;
  MN_CHECK(n >= 1 && n <= p.max_images, "preprocess_run: %d images outside [1, max_images=%d]", n, p.max_images);
  for (int c = 0; c < 3; ++c) MN_CHECK(std3[c] > 0.f, "preprocess_run: std[%d] = %f must be positive", c, std3[c]);
  cudaStream_t st = (cudaStream_t)stream;
  const long long t1 = (long long)n * p.Hin * p.Wout, t2 = (long long)n * p.Hout * p.Wout;
  const int g1 = (int)((t1 + 255) / 256 < (long long)kNumSMs * 16 ? (t1 + 255) / 256 : (long long)kNumSMs * 16);
  const int g2 = (int)((t2 + 255) / 256 < (long long)kNumSMs * 16 ? (t2 + 255) / 256 : (long long)kNumSMs * 16);
  MN_LAUNCH(k_pre_resize_h, g1, 256, 0, st, (const uint8_t*)img_nhwc_u8, (const int*)frame_index_dev, p.d_tmp, p.d_bh, p.d_kh,
            p.ksh, (long long)n * p.Hin, p.Hin, p.Win, p.Wout);
  MN_LAUNCH_CHECK();
  if (jitter_dev == nullptr) {
    MN_LAUNCH(k_pre_resize_v_norm, g2, 256, 0, st, p.d_tmp, out_nchw, (uint8_t*)out_u8_or_null, p.d_bv, p.d_kv, p.ksv, n,
              p.Hin, p.Hout, p.Wout, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2]);
    MN_LAUNCH_CHECK();
    return 0;
  }
  // ColorJitter between Resize and ToTensor (scripts/train.py:121-126)
  if (p.d_u8 == nullptr) {
    MN_CUDA(cudaMalloc((void**)&p.d_u8, (size_t)p.max_images * p.Hout * p.Wout * 3));
    MN_CUDA(cudaMalloc((void**)&p.d_sums, (size_t)p.max_images * sizeof(unsigned int)));
  }
  const long long npix = (long long)p.Hout * p.Wout;
  MN_CHECK(npix * 255 < 4294967295LL, "preprocess_run: image too large for the 32-bit luma sum");
  MN_LAUNCH(k_pre_resize_v_norm, g2, 256, 0, st, p.d_tmp, (float*)nullptr, p.d_u8, p.d_bv, p.d_kv, p.ksv, n,
            p.Hin, p.Hout, p.Wout, 0.f, 0.f, 0.f, 1.f, 1.f, 1.f);
  MN_LAUNCH_CHECK();
  MN_CUDA(cudaMemsetAsync(p.d_sums, 0, (size_t)n * sizeof(unsigned int), st));
  int gx = (int)((npix + 255) / 256); if (gx > 64) gx = 64;
  MN_LAUNCH(k_jitter_luma_sum, dim3(gx, n), 256, 0, st, (const uint8_t*)p.d_u8, (const int*)nullptr,
            (const JitterParams*)jitter_dev, p.d_sums, npix);
  MN_LAUNCH_CHECK();
  MN_LAUNCH(k_jitter_norm, dim3(gx, n), 256, 0, st, (const uint8_t*)p.d_u8, (const JitterParams*)jitter_dev,
            (const unsigned int*)p.d_sums, out_nchw, (uint8_t*)out_u8_or_null, p.Hout, p.Wout, mean3[0], mean3[1], mean3[2],
            std3[0], std3[1], std3[2]);
  MN_LAUNCH_CHECK();
  return 0;
}

int mapnet_preprocess_destroy(mapnet_preprocess_t* h) {
  if (h == nullptr) return 0;
  cudaFree(h->p.d_bh); cudaFree(h->p.d_kh); cudaFree(h->p.d_bv); cudaFree(h->p.d_kv); cudaFree(h->p.d_tmp);
  cudaFree(h->p.d_u8); cudaFree(h->p.d_sums);
  delete h;
  return 0;
}

}  // extern "C"
