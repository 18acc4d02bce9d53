// Shared device/host helpers for the MapNet hot path (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace mapnet {

typedef __nv_bfloat16 bf16;

// ---- error plumbing: no exception crosses the C boundary -------------------
void set_last_error(const char* fmt, ...);
const char* get_last_error();

#define MN_CUDA(expr)                                                           \
  do {                                                                          \
    cudaError_t _e = (expr);                                                    \
    if (_e != cudaSuccess) {                                                    \
      mapnet::set_last_error("%s:%d CUDA error %d (%s) in %s", __FILE__,        \
                             __LINE__, (int)_e, cudaGetErrorString(_e), #expr); \
      return 1;                                                                 \
    }                                                                           \
  } while (0)

#define MN_CHECK(cond, ...)                         \
  do {                                              \
    if (!(cond)) {                                  \
      mapnet::set_last_error(__VA_ARGS__);          \
      return 2;                                     \
    }                                               \
  } while (0)

#define MN_TRY(expr)          \
  do {                        \
    int _r = (expr);          \
    if (_r != 0) return _r;   \
  } while (0)

extern unsigned long long g_launch_count;   // kernels launched by this library (host-side counter)
#define MN_LAUNCH_CHECK()              \
  do {                                 \
    ++mapnet::g_launch_count;          \
    MN_CUDA(cudaGetLastError());       \
  } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// SMs of the target GPU (H100 SXM): persistent grids and split-K factors are sized for it
static constexpr int kNumSMs = 132;

// ---- programmatic dependent launch -------------------------------------------
// Every kernel of the library starts with pdl_prologue(): it lets the NEXT kernel in the stream be
// scheduled early (its blocks then sit in griddepcontrol.wait) and itself waits until the PREVIOUS
// kernel has completed and flushed.  Nothing touches global memory before the wait, so the
// semantics are those of a serialized stream; what overlaps is launch latency, block scheduling
// and per-block setup (barrier init, descriptor prefetch) -- worth it because a
// training step is ~290 launches of 2-40 us each.  MAPNET_PDL=0 disables the launch attribute.
#if defined(__CUDACC__)
__device__ __forceinline__ void pdl_prologue() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
#endif
int pdl_enabled();

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                   Args&&... args) {
  cudaLaunchConfig_t cfg; memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#define MN_LAUNCH(kern, grid, block, smem, st, ...)                                        \
  do {                                                                                     \
    MN_CUDA(mapnet::launch_k(kern, dim3(grid), dim3(block), (size_t)(smem), st, __VA_ARGS__)); \
  } while (0)

// ---- activation element access ---------------------------------------------
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16_rn(v); }

// 8-wide channel vectors: 16 B for bf16, 2x16 B for fp32.  All activation
// tensors are NHWC with C % 8 == 0 (C in {8(padded stem),64,128,256,512}).
template <typename T> struct Vec8;
template <> struct Vec8<float> {
  float v[8];
  __device__ __forceinline__ void load(const float* p) {
    float4 a = *reinterpret_cast<const float4*>(p);
    float4 b = *reinterpret_cast<const float4*>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  __device__ __forceinline__ void store(float* p) const {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
};
template <> struct Vec8<bf16> {
  float v[8];
  __device__ __forceinline__ void load(const bf16* p) {
    uint4 r = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 f = __bfloat1622float2(h[i]);
      v[2 * i] = f.x; v[2 * i + 1] = f.y;
    }
  }
  __device__ __forceinline__ void store(bf16* p) const {
    uint4 r;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = r;
  }
};

// ---- split 16-bit operand planes (strict tensor-core mode) --------------------------------
// A value x is stored as hi + lo with hi = fp16(x), lo = fp16(x - hi): 22 significant bits, |x| <= 65504
// (saturating), absolute error max(2^-22 |x|, 2^-25).  Storage layout per 8
// consecutive channels: 8 x hi (16 B) then 8 x lo (16 B) -- one logical element is 4 bytes, so the NHWC
// indexing of the element-wise kernels (pointer + 8*i) is unchanged, and the conv engines see a 16-bit tensor
// with 2C "channels" whose K order is (c/8, plane, c%8); the packed weight matrices use the same K order
// (layout.cu), so every hi/lo cross product is formed by ordinary wgmma MMAs.  Only Vec8 access is defined.
struct hsplit { uint32_t raw; };

__device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
  float c = fminf(fmaxf(v, -65504.f), 65504.f);        // saturate instead of overflowing to inf
  c = (v != v) ? v : c;                                 // NaN stays NaN
  hi = __float2half_rn(c);
  lo = __float2half_rn(c - __half2float(hi));
}

template <> struct Vec8<hsplit> {
  float v[8];
  __device__ __forceinline__ void load(const hsplit* p) {
    const uint4 a = *reinterpret_cast<const uint4*>(p);
    const uint4 b = *(reinterpret_cast<const uint4*>(p) + 1);
    const __half2* h = reinterpret_cast<const __half2*>(&a);
    const __half2* l = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 fh = __half22float2(h[i]), fl = __half22float2(l[i]);
      v[2 * i] = fh.x + fl.x; v[2 * i + 1] = fh.y + fl.y;
    }
  }
  __device__ __forceinline__ void store(hsplit* p) const {
    uint4 a, b;
    __half* h = reinterpret_cast<__half*>(&a);
    __half* l = reinterpret_cast<__half*>(&b);
#pragma unroll
    for (int i = 0; i < 8; ++i) split_f16(v[i], h[i], l[i]);
    *reinterpret_cast<uint4*>(p) = a;
    *(reinterpret_cast<uint4*>(p) + 1) = b;
  }
};
// ---- e4m3 activations (fp8 inference) -------------------------------------------------------
// One byte per element; the tensor's power-of-two scale lives elsewhere (infer.cu), so Vec8 moves the scaled values:
// load dequantizes without the scale, store rounds to nearest even and saturates to +-448 (cvt.rn.satfinite).
struct e4m3 { uint8_t raw; };

__device__ __forceinline__ uint16_t f8x2_pack(float a, float b) {
  return (uint16_t)__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
}
__device__ __forceinline__ float2 f8x2_unpack(uint16_t v) {
  const __half2 h = __half2(__nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)v, __NV_E4M3));
  return __half22float2(h);
}
__device__ __forceinline__ uint2 f8x8_pack(const float (&v)[8]) {
  uint2 r;
  r.x = (uint32_t)f8x2_pack(v[0], v[1]) | ((uint32_t)f8x2_pack(v[2], v[3]) << 16);
  r.y = (uint32_t)f8x2_pack(v[4], v[5]) | ((uint32_t)f8x2_pack(v[6], v[7]) << 16);
  return r;
}
__device__ __forceinline__ void f8x8_unpack(const uint2 r, float (&v)[8]) {
  float2 t;
  t = f8x2_unpack((uint16_t)(r.x & 0xffffu)); v[0] = t.x; v[1] = t.y;
  t = f8x2_unpack((uint16_t)(r.x >> 16)); v[2] = t.x; v[3] = t.y;
  t = f8x2_unpack((uint16_t)(r.y & 0xffffu)); v[4] = t.x; v[5] = t.y;
  t = f8x2_unpack((uint16_t)(r.y >> 16)); v[6] = t.x; v[7] = t.y;
}
// The scale of an e4m3 tensor or weight row with max |x| = amax: the smallest power of two s with 448 * s >= amax, i.e.
// 2^ceil(log2(amax / 448)), taken from the exponent so that no rounded division or logarithm is involved (amax =
// m * 2^k, m in [0.5, 1), 448 = 0.875 * 2^9).  amax 0 gives 1; s stays >= 2^-126 so 1 / s is finite.
__host__ __device__ inline float f8_pow2_scale(float amax) {
  if (!(amax > 0.f)) return 1.f;
  if (amax > 3.4028234663852886e38f) return ldexpf(1.f, 120);
  int k;
  const float m = frexpf(amax, &k);
  int e = (m <= 0.875f) ? k - 9 : k - 8;
  if (e < -126) e = -126;
  return ldexpf(1.f, e);
}
template <> struct Vec8<e4m3> {
  float v[8];
  __device__ __forceinline__ void load(const e4m3* p) { f8x8_unpack(*reinterpret_cast<const uint2*>(p), v); }
  __device__ __forceinline__ void store(e4m3* p) const { *reinterpret_cast<uint2*>(p) = f8x8_pack(v); }
};

// The same 8 elements held RAW: issue the loads early (software pipelining across a prologue or a barrier -- a warp
// issues in order, so an early load whose conversion follows at once would stall right there), convert at first use.
template <typename T> struct Raw8;
template <> struct Raw8<float> {
  float4 a, b;
  __device__ __forceinline__ void load(const float* p) {
    a = *reinterpret_cast<const float4*>(p); b = *reinterpret_cast<const float4*>(p + 4);
  }
  __device__ __forceinline__ void get(Vec8<float>& o) const {
    o.v[0] = a.x; o.v[1] = a.y; o.v[2] = a.z; o.v[3] = a.w; o.v[4] = b.x; o.v[5] = b.y; o.v[6] = b.z; o.v[7] = b.w;
  }
};
template <> struct Raw8<bf16> {
  uint4 r;
  __device__ __forceinline__ void load(const bf16* p) { r = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void get(Vec8<bf16>& o) const {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(h[i]); o.v[2 * i] = f.x; o.v[2 * i + 1] = f.y; }
  }
};
template <> struct Raw8<hsplit> {
  uint4 a, b;
  __device__ __forceinline__ void load(const hsplit* p) {
    a = *reinterpret_cast<const uint4*>(p); b = *(reinterpret_cast<const uint4*>(p) + 1);
  }
  __device__ __forceinline__ void get(Vec8<hsplit>& o) const {
    const __half2* h = reinterpret_cast<const __half2*>(&a);
    const __half2* l = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 fh = __half22float2(h[i]), fl = __half22float2(l[i]);
      o.v[2 * i] = fh.x + fl.x; o.v[2 * i + 1] = fh.y + fl.y;
    }
  }
};
// Element types of one precision mode: A = conv outputs and everything derived by fp32 math from them
// (what BatchNorm reads, gradients w.r.t. block outputs), Z = forward conv operands (post-BN/ReLU activations,
// the stem operand), G = backward conv operands (gradients w.r.t. conv outputs).
struct TypesF32 { typedef float A; typedef float Z; typedef float G; };
struct TypesBF16 { typedef bf16 A; typedef bf16 Z; typedef bf16 G; };
struct TypesSplitHH { typedef float A; typedef hsplit Z; typedef hsplit G; };

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace mapnet
