// wgmma / TMA implicit-GEMM convolution engines for sm_90a (bf16 operands,
// fp32 accumulation in registers): fprop, dgrad, wgrad of every ResNet-34 conv.
//
// Replaces cuDNN conv fwd / bwd-data / bwd-filter behind torchvision resnet34
// (reference models/posenet.py:66; SURVEY.md section 2c) with hand-written kernels:
//
//  k_tc_conv  (fprop, dgrad)  D[pixel][cout] = sum_{tap,c} A_tap[pixel][c] * W[cout][tap][c]
//     * im2col is done ON THE FLY by TMA: the A tile of one (tap, 64-channel block)
//       is a 4-D box {64 ch, TW, TH, TN} of the NHWC activation tensor at the tap's
//       spatial offset; out-of-bounds pixels (padding, ragged edges) are zero-filled
//       by the TMA unit.  Stride-2 convs read parity views of the tensor (4 maps).
//     * warp-specialised, persistent CTAs: warp 8 = TMA producer, warps 0-7 = two
//       consumer warpgroups, each issuing wgmma m64nBNk16 for 64 of the tile's 128
//       pixel rows (N = 64/128, K = 16) and then running the epilogue on its own
//       rows (registers -> shared memory -> +residual -> bf16 -> global) while the
//       producer already streams the next tile's operands.
//  k_tc_wgrad  dW[cout][tap][c] += sum_pixels dY[pixel][cout] * X_tap[pixel][c]
//     * both operands are MN-major (pixels = K): two 64-channel X chunks form the
//       128 rows of A (one per consumer warpgroup), dY supplies up to 128 columns of B;
//       split-K over pixel tiles, the splits' partial dW added up in a fixed order into the flat
//       wgrad buffer (k_wgrad_reduce).
//  k_halo_wgrad  the same dW for stride-1 3x3 convs with the same K partition: per k-block one X halo and one dY
//     tile, 3 or 9 filter taps read from the halo by descriptor (tc_plan_create picks the engine per conv).
#include <cudaTypedefs.h>

#include <stdarg.h>
#include <stdlib.h>

#include <vector>

#include "kernels.h"
#include "tc_ptx.cuh"

namespace mapnet {

using namespace ptx;

// ---------------------------------------------------------------------------------
// host: tensor-map encoding through the driver entry point (no libcuda link dependency)
// ---------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
  }
  return fn;
}

// 4-D NHWC view: dims {C, W, H, N} with byte strides; box {box0, bw, bh, bn}; OOB -> 0.  bf16 tiles are 64 channels
// in 128B-swizzled rows; e4m3 tiles (UINT8) are 128- or 64-channel rows with the matching swizzle.
static int encode_act_map(CUtensorMap* m, const void* base, int C, int Wd, int Hd, int Nd, long long sw_bytes,
                          long long sh_bytes, long long sn_bytes, int bw, int bh, int bn,
                          CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, int box0 = 64,
                          CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  auto fn = get_encode_fn();
  MN_CHECK(fn != nullptr, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)Wd, (cuuint64_t)Hd, (cuuint64_t)Nd};
  cuuint64_t strides[3] = {(cuuint64_t)sw_bytes, (cuuint64_t)sh_bytes, (cuuint64_t)sn_bytes};
  cuuint32_t box[4] = {(cuuint32_t)box0, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
  cuuint32_t es[4] = {1u, 1u, 1u, 1u};
  CUresult r = fn(m, dt, 4, const_cast<void*>(base), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MN_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(act %dx%dx%dx%d box %d,%d,%d) failed: %d", C, Wd, Hd, Nd, bw, bh, bn, (int)r);
  return 0;
}
// 2-D weight matrix [rows][K] (K contiguous): box {box0, brows} (bf16: 64 elements; e4m3: 128 or 64 bytes)
static int encode_w_map(CUtensorMap* m, const void* base, int K, int rows, int brows,
                        CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, int box0 = 64,
                        CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  auto fn = get_encode_fn();
  MN_CHECK(fn != nullptr, "cuTensorMapEncodeTiled entry point not available");
  const int elt = (dt == CU_TENSOR_MAP_DATA_TYPE_UINT8) ? 1 : 2;
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * elt};
  cuuint32_t box[2] = {(cuuint32_t)box0, (cuuint32_t)brows};
  cuuint32_t es[2] = {1u, 1u};
  CUresult r = fn(m, dt, 2, const_cast<void*>(base), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MN_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(weights K=%d rows=%d) failed: %d", K, rows, (int)r);
  return 0;
}

bool tc_overlapped_view_supported() {
  static int ok = -1;
  if (ok < 0) {
    // encode only (nothing is dereferenced): 64-element rows that start 16 elements apart
    CUtensorMap m;
    auto fn = get_encode_fn();
    ok = 0;
    if (fn != nullptr) {
      cuuint64_t dims[4] = {64, 128, 131, 2};
      cuuint64_t strides[3] = {32, 132 * 32, 131ull * 132 * 32};
      cuuint32_t box[4] = {64, 16, 8, 1};
      cuuint32_t es[4] = {1, 1, 1, 1};
      void* base = nullptr;
      if (cudaMalloc(&base, 4096) == cudaSuccess) {
        CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        ok = (r == CUDA_SUCCESS) ? 1 : 0;
        cudaFree(base);
      }
    }
  }
  return ok == 1;
}

// ---------------------------------------------------------------------------------
// device parameter blocks
// ---------------------------------------------------------------------------------
// map: bits 0..1 = activation tensor map (A operand), bit 2 = the SECOND weight matrix (mapB2: the 1x1
// downsample conv folded into a stride-2 dgrad, see tc_plan_add_shortcut)
struct TapDesc { int dh, dw, map, kidx; };

// One output class of a launch.  fprop and stride-1 dgrad have a single class; a stride-2 dgrad has
// s*s parity classes -- output pixels (jh*os+oa, jw*os+ob) -- each with its own subset of the filter
// taps.  All classes of a launch share the tile box and the tile grid (sized for the largest class).
struct ClassDesc { int Hs, Ws, oa, ob, tap0, num_taps; };

struct ConvParams {
  // M space: (n, jh, jw) over [Nimg, Hs, Ws] of the tile's class; tile box TN x TH x TW = 128 pixels
  int Nimg, TW, TH, TN, tiles_w, tiles_h, tiles_n, n_tiles_m, n_tiles_n;
  int n_classes;
  ClassDesc cls[4];
  // K space
  int cblocks, Cs;
  TapDesc taps[20];        // strict (split-operand) mode: every filter tap appears twice (hi and lo weight planes)
  // output tensor [Nimg, Hout, Wout, Cout]; pixel (n, jh*os+oa, jw*os+ob)
  int Hout, Wout, Cout, os;
  int debug;     // micro-benchmark only: 1 = skip the MMAs, 2 = skip the TMA loads (results are garbage)
  int fmt_a, fmt_b;        // wgmma operand element formats (equal): 0 = fp16, 1 = bf16
  int out32;               // strict mode: output (and residual) are fp32 tensors
};

// work item -> (class, N tile, M tile): classes are laid out one after the other (heaviest first), inside a class the
// N tile varies fastest
struct TileCoord { int cls, tn, tm; };
__device__ __forceinline__ TileCoord decode_tile(const int tile, const int per_class, const int n_tiles_n) {
  TileCoord t;
  t.cls = tile / per_class;
  const int r = tile - t.cls * per_class;
  t.tm = r / n_tiles_n;
  t.tn = r - t.tm * n_tiles_n;
  return t;
}

struct WgradChunk { int dh, dw, map, c0, tap; };   // one 64-channel slice of X at one filter tap
struct WgradTap { int dh, dw, map; };

struct WgradParams {
  int Nimg, Ho, Wo, TW, TH, TN, tiles_w, tiles_h, tiles_n, n_pix_tiles;
  int n_chunks;            // total X chunks = taps * cpt
  int cpt;                 // 64-element chunks per tap: Ci/64 (strict mode: 2*Ci/64 chunks of the split planes)
  int n_mtiles;            // ceil(n_chunks / 2)
  int n_ntiles, BN;        // Co tiles of BN columns (strict mode: columns of the split planes, 2*Co in all)
  int splits, tiles_per_split;
  int Ci, Co, KK;          // dW layout [Co][KK][Ci] (real channels)
  int debug;               // micro-benchmark only: 3 = skip the atomic epilogue
  int split;               // strict mode: X and dY are split 16-bit planes, the four hi/lo products are summed
  int fmt_a, fmt_b;        // wgmma operand element formats (equal): 0 = fp16, 1 = bf16
  const float* oscale;     // device scalar multiplied into the accumulators before they are stored, or null
  float* partial;          // splits > 1: split s stores its dW slice at partial + s * part_stride (no atomics), or null
  long long part_stride;   // Co * KK * Ci
  WgradTap taps[16];
  // stride-1 3x3 convs run from a staged input halo (k_halo_wgrad) when halo_taps != 0; the K partition above
  // (box, splits, tiles_per_split) is the per-tap engine's either way
  int halo_taps;           // 3: one filter row per CTA (one consumer warpgroup), 9: all three rows (three warpgroups)
  int halo_bn;             // its N tile (64 or 128; 9 taps: 64)
  int RW, HR;              // halo box: RW = TW + 2 rounded up to 8 pixels wide, HR = TH + halo_taps / 3 - 1 rows high
  int halo_bytes;          // 128 * RW * HR * TN
  int halo_sbo;            // bytes between the two 8-pixel groups of a k16 step inside the halo
  int step_row[4];         // halo row of the first pixel of k16 step j of a k-block (filter tap (0, 0) of the halo)
};
// chunk c = (tap c / cpt, 64-element block c % cpt)
__device__ __forceinline__ WgradChunk wgrad_chunk(const WgradParams& P, int c) {
  WgradChunk ch;
  ch.tap = c / P.cpt;
  ch.c0 = (c - ch.tap * P.cpt) * 64;
  ch.dh = P.taps[ch.tap].dh; ch.dw = P.taps[ch.tap].dw; ch.map = P.taps[ch.tap].map;
  return ch;
}

// x[32] per lane -> lane L ends with sum over the warp's lanes of x[L] (in x[0])
__device__ __forceinline__ void warp_transpose_reduce(float (&x)[32], int lane) {
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    const bool up = (lane & s) != 0;
#pragma unroll
    for (int k = 0; k < s; ++k) {
      const float send = up ? x[k] : x[k + s];
      const float keep = up ? x[k + s] : x[k];
      x[k] = keep + __shfl_xor_sync(0xffffffffu, send, s);
    }
  }
}

// ---------------------------------------------------------------------------------
// Shared epilogue of the fprop / dgrad engines: one 32-column chunk of a warp's 32 accumulator rows.
//   f = acc (+ residual)                                  every mode
//   dgrad with E.y:  f = gate ? f : 0                     the consumer BN's ReLU gate, so the stored
//                                                         gradient is already masked
//   store bf16(f)
//   statistics of the values AS STORED (rows outside the tensor count as 0):
//     fprop:  (sum f, sum f^2)                            BatchNorm batch statistics
//     dgrad:  (sum g, sum g*y [, sum g*yd])               BatchNorm backward reductions of the BN
//                                                         (and downsample BN) that consumes g
// which removes the separate reduction pass over dY and Y of every BatchNorm backward.
//
// The wgmma accumulator fragment scatters a row over four lanes in 8-byte pieces: touching global memory in
// that layout costs a wavefront per lane per 8 bytes.  Each warpgroup therefore stages its 64 accumulator rows
// once in shared memory (row stride BN + 4 floats: conflict-free reads) and re-reads them in the COALESCED
// layout -- lane L owns 8 consecutive columns (16 bytes of bf16) p = L&3 of rows 8i + (L>>2), i = 0..3, of a
// 32-row quarter -- in which every global load and store instruction covers 8 rows x 64 contiguous bytes, and
// everything else (residual, gate, statistics) happens in that layout.
// ---------------------------------------------------------------------------------
// Two consumer warpgroups (warps 0-7) and one TMA producer warp (warp 8).  In the epilogue the two warps that
// share a 32-row quarter of the tile split its 32-column chunks (even / odd chunks).
static constexpr int kEpiWarps = 8;
static constexpr int kEpiSplit = 2;                      // warps per 32-row quarter
static constexpr int kEpiThreads = 32 * kEpiWarps;
static constexpr int kProducerWarp = kEpiWarps;
static constexpr int kConvThreads = kEpiThreads + 32;

// Epilogue variants (template flags): the flags are launch-uniform, and specialising on them keeps every
// variant's chunk body straight-line code (runtime flags cost ~3x: branches fence the scheduler and the
// four epilogue warps are latency-, not throughput-bound).
enum : int {
  EPI_RES = 1,      // + residual
  EPI_STATS = 2,    // fprop: (sum f, sum f^2)
  EPI_BWD = 4,      // dgrad: gate + (sum g, sum g*y); gate = mscale*y+mshift > 0 unless EPI_ZMASK
  EPI_ZMASK = 8,    // gate = zmask > 0
  EPI_YD = 16,      // third sum over the downsample-branch BN input
  EPI_OUT32 = 32,   // strict mode: fp32 output and residual (combines with EPI_RES / EPI_STATS only)
  // eval-mode inference (fprop, never with EPI_STATS / EPI_BWD): f = acc*s[c] + t[c] (+ residual) (ReLU), one rounding
  EPI_AFFINE = 64,
  EPI_RELU = 128,   // with EPI_AFFINE
  EPI_HOUT = 256,   // with EPI_OUT32: store fp16 hi/lo planes (common.cuh: hsplit) instead of fp32
  EPI_HRES = 512,   // with EPI_OUT32 | EPI_RES: the residual is in hi/lo plane form
  // fp8 inference (k_f8_conv only, with EPI_AFFINE: the scale table is bn_scale * s_in * s_w, see EpiF8)
  EPI_F8OUT = 1024, // store e4m3(f / s_out) (satfinite) instead of bf16
  EPI_F8RES = 2048, // with EPI_RES: the residual is e4m3, dequantized as r * s_res
  EPI_AMAX = 4096,  // calibration: record max |f| over the tensor's rows, store nothing
};

// The fp8 engine's epilogue operands: EpiBwd's affine fields plus the device scalars of the e4m3 tensors involved
struct EpiF8Dev : EpiBwd {
  const float* res_scale;   // s_res (EPI_F8RES)
  const float* out_inv;     // 1 / s_out (EPI_F8OUT)
  unsigned int* amax;       // EPI_AMAX: max |f| as the bit pattern of a non-negative float (atomicMax)
};

struct EpiRegs { uint4 r[4], y[4], z[4], d[4]; };

__device__ __forceinline__ void unpack8(const uint4& u, float (&o)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    o[2 * i] = t.x; o[2 * i + 1] = t.y;
  }
}

// x[8] per lane -> the sum over the 8 lanes that share (lane & 3), column (lane >> 2) of the 8 in x[0]
__device__ __forceinline__ void group_reduce8(float (&x)[8], int lane) {
#pragma unroll
  for (int s = 4; s >= 1; s >>= 1) {          // lane bits 4, 3, 2 <-> column bits 2, 1, 0
    const bool up = (lane & (s << 2)) != 0;
#pragma unroll
    for (int k = 0; k < s; ++k) {
      const float send = up ? x[k] : x[k + s];
      const float keep = up ? x[k + s] : x[k];
      x[k] = keep + __shfl_xor_sync(0xffffffffu, send, s << 2);
    }
  }
}

// statistics land on lane L for column  col0 + epi_stat_col(L)
__device__ __forceinline__ int epi_stat_col(int lane) { return 8 * (lane & 3) + (lane >> 2); }

// issue one chunk's operand loads (they do not depend on the accumulator).  Rows outside the tensor have
// their offset clamped to row 0 by the caller, so no load needs a guard.
template <int F>
__device__ __forceinline__ void epi_issue_loads(EpiRegs& G, const long long (&rowoff)[4], const int coff,
                                                const bf16* residual, const EpiBwd& E, const int lane) {
  const int po = coff + 8 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long off = rowoff[i] + po;
    if ((F & EPI_RES) && (F & EPI_OUT32)) {       // fp32 residual: 8 floats, second half in the (otherwise unused) y slot
      const float* rp = reinterpret_cast<const float*>(residual) + off;
      G.r[i] = *reinterpret_cast<const uint4*>(rp);
      G.y[i] = *reinterpret_cast<const uint4*>(rp + 4);
    } else if ((F & EPI_RES) && (F & EPI_F8RES)) {   // 8 e4m3 values in the low half of the r slot
      const uint2 v = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(residual) + off);
      G.r[i].x = v.x; G.r[i].y = v.y;
    } else if (F & EPI_RES) G.r[i] = *reinterpret_cast<const uint4*>(residual + off);   // may alias `out`: plain load
    if (F & EPI_BWD) G.y[i] = __ldg(reinterpret_cast<const uint4*>(E.y + off));
    if (F & EPI_ZMASK) G.z[i] = __ldg(reinterpret_cast<const uint4*>(E.zmask + off));
    if (F & EPI_YD) G.d[i] = __ldg(reinterpret_cast<const uint4*>(E.yd + off));
  }
}

// write this thread's wgmma accumulator fragment (rows 16*wq + lane/4 (+8), columns 8j + 2*(lane%4) (+1)) into
// the warpgroup's staging rows
template <int BN>
__device__ __forceinline__ void acc_to_stage(const float (&d)[BN / 2], float* __restrict__ stg, const int wq, const int lane) {
  constexpr int RS = BN + 4;
  float* r0 = stg + (16 * wq + (lane >> 2)) * RS + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2*>(r0 + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(r0 + 8 * RS + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

// one 32-column chunk of a warp's 32 staged rows (row stride RS floats).  EP: EpiBwd, or EpiF8Dev for the fp8 engine's
// flags (EPI_F8OUT / EPI_F8RES / EPI_AMAX; with EPI_AMAX s0 is the running max |f| of the rows inside the tensor)
template <int F, int RS, typename EP>
__device__ __forceinline__ void epi_chunk(const float* __restrict__ scr, const EpiRegs& G,
                                          const long long (&rowoff)[4], const bool (&rstore)[4], const float (&rw)[4],
                                          const int coff, const int col0, bf16* out, const EP& E, const int lane,
                                          float& s0, float& s1, float& s2) {
  const int p = lane & 3, rr = lane >> 2;
  float4 lo[4], hi[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4* src = reinterpret_cast<const float4*>(scr + (8 * i + rr) * RS + 8 * p);
    lo[i] = src[0]; hi[i] = src[1];
  }
  float msc[8], msh[8];
  if (((F & EPI_BWD) && !(F & EPI_ZMASK)) || (F & EPI_AFFINE)) {
    const float4* a = reinterpret_cast<const float4*>(((F & EPI_AFFINE) ? E.ascale : E.mscale) + col0 + 8 * p);
    const float4* b = reinterpret_cast<const float4*>(((F & EPI_AFFINE) ? E.ashift : E.mshift) + col0 + 8 * p);
    const float4 a0 = __ldg(a), a1 = __ldg(a + 1), b0 = __ldg(b), b1 = __ldg(b + 1);
    msc[0] = a0.x; msc[1] = a0.y; msc[2] = a0.z; msc[3] = a0.w; msc[4] = a1.x; msc[5] = a1.y; msc[6] = a1.z; msc[7] = a1.w;
    msh[0] = b0.x; msh[1] = b0.y; msh[2] = b0.z; msh[3] = b0.w; msh[4] = b1.x; msh[5] = b1.y; msh[6] = b1.z; msh[7] = b1.w;
  }
  float c0[8], c1[8], c2[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { c0[k] = 0.f; c1[k] = 0.f; c2[k] = 0.f; }
  float osc = 1.f;
  if (F & EPI_OUT32) { if (E.oscale != nullptr) osc = __ldg(E.oscale); }
  float rsc = 1.f, oinv = 1.f;
  if constexpr ((F & EPI_F8RES) != 0) rsc = __ldg(E.res_scale);
  if constexpr ((F & EPI_F8OUT) != 0) oinv = __ldg(E.out_inv);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float f[8] = {lo[i].x, lo[i].y, lo[i].z, lo[i].w, hi[i].x, hi[i].y, hi[i].z, hi[i].w};
    float yv[8];
    if (F & EPI_OUT32) {
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] *= osc;
    }
    if (F & EPI_AFFINE) {        // the same expression as k_bn_apply's, on the fp32 accumulator
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] = f[k] * msc[k] + msh[k];
    }
    if ((F & EPI_RES) && (F & EPI_HRES)) {       // hi planes in the r slot, lo planes in the y slot (Vec8<hsplit>::load)
      const __half2* h = reinterpret_cast<const __half2*>(&G.r[i]);
      const __half2* l = reinterpret_cast<const __half2*>(&G.y[i]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 fh = __half22float2(h[k]), fl = __half22float2(l[k]);
        f[2 * k] += fh.x + fl.x; f[2 * k + 1] += fh.y + fl.y;
      }
    } else if ((F & EPI_RES) && (F & EPI_F8RES)) {      // r * s_res is exact (s_res a power of two)
      float r[8];
      f8x8_unpack(make_uint2(G.r[i].x, G.r[i].y), r);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] += r[k] * rsc;
    } else if ((F & EPI_RES) && (F & EPI_OUT32)) {
      const float4 r0 = *reinterpret_cast<const float4*>(&G.r[i]), r1 = *reinterpret_cast<const float4*>(&G.y[i]);
      f[0] += r0.x; f[1] += r0.y; f[2] += r0.z; f[3] += r0.w; f[4] += r1.x; f[5] += r1.y; f[6] += r1.z; f[7] += r1.w;
    } else if (F & EPI_RES) {
      float r[8];
      unpack8(G.r[i], r);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] += r[k];
    }
    if (F & EPI_BWD) {
      unpack8(G.y[i], yv);
      if (F & EPI_ZMASK) {
        float z[8];
        unpack8(G.z[i], z);
#pragma unroll
        for (int k = 0; k < 8; ++k) f[k] = (z[k] > 0.f) ? f[k] : 0.f;
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) f[k] = (yv[k] * msc[k] + msh[k] > 0.f) ? f[k] : 0.f;
      }
    }
    if (F & EPI_RELU) {
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] = fmaxf(f[k], 0.f);
    }
    if constexpr ((F & EPI_AMAX) != 0) {           // calibration pass: the values the storing pass would quantize
#pragma unroll
      for (int k = 0; k < 8; ++k) s0 = fmaxf(s0, rw[i] != 0.f ? fabsf(f[k]) : 0.f);
      continue;
    } else if constexpr ((F & EPI_F8OUT) != 0) {   // f / s_out is exact; one rounding, at the e4m3 cast
      float q[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) q[k] = f[k] * oinv;
      const uint2 pk = f8x8_pack(q);
      if (rstore[i]) *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(out) + rowoff[i] + coff + 8 * p) = pk;
      continue;
    }
    uint4 o;
    if (F & EPI_HOUT) {          // 8 hi then 8 lo fp16 values: the operand form the next conv reads
      if (rstore[i]) {
        uint4 a, b;
        __half* h = reinterpret_cast<__half*>(&a);
        __half* l = reinterpret_cast<__half*>(&b);
#pragma unroll
        for (int k = 0; k < 8; ++k) split_f16(f[k], h[k], l[k]);
        uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<float*>(out) + rowoff[i] + coff + 8 * p);
        op[0] = a; op[1] = b;
      }
    } else if (F & EPI_OUT32) {
      if (rstore[i]) {
        float* op = reinterpret_cast<float*>(out) + rowoff[i] + coff + 8 * p;
        *reinterpret_cast<float4*>(op) = make_float4(f[0], f[1], f[2], f[3]);
        *reinterpret_cast<float4*>(op + 4) = make_float4(f[4], f[5], f[6], f[7]);
      }
    } else {
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
      for (int k = 0; k < 4; ++k) h[k] = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
      if (rstore[i]) *reinterpret_cast<uint4*>(out + rowoff[i] + coff + 8 * p) = o;
    }
    if (F & (EPI_STATS | EPI_BWD)) {
      // the values AS STORED; rw = 1 for rows inside the tensor, 0 outside
      float x[8];
      if (F & EPI_OUT32) {
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = f[k];
      } else unpack8(o, x);
#pragma unroll
      for (int k = 0; k < 8; ++k) x[k] *= rw[i];
      if (F & EPI_BWD) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { c0[k] += x[k]; c1[k] += x[k] * yv[k]; }
        if (F & EPI_YD) {
          float u[8];
          unpack8(G.d[i], u);
#pragma unroll
          for (int k = 0; k < 8; ++k) c2[k] += x[k] * u[k];
        }
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) { c0[k] += x[k]; c1[k] += x[k] * x[k]; }
      }
    }
  }
  if (F & (EPI_STATS | EPI_BWD)) {
    group_reduce8(c0, lane);
    group_reduce8(c1, lane);
    s0 += c0[0];
    s1 += c1[0];
    if (F & EPI_YD) { group_reduce8(c2, lane); s2 += c2[0]; }
  }
}

// One accumulator tile (this warp's 32 staged rows x BN columns): walk the warp's 32-column chunks.
template <int F, int BN, typename EP>
__device__ __forceinline__ void epi_tile(const float* __restrict__ rows, float (*stw)[BN / 32][32],
                                         const long long (&rowoff)[4], const bool (&rvalid)[4], const bool do_store,
                                         const int tn, const bf16* residual, bf16* out, const EP& E, const int lane,
                                         const int half) {
  bool rstore[4]; float rw[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { rstore[i] = rvalid[i] && do_store; rw[i] = rvalid[i] ? 1.f : 0.f; }
#pragma unroll 1
  for (int cc = half; cc < BN / 32; cc += kEpiSplit) {
    EpiRegs G;
    epi_issue_loads<F>(G, rowoff, cc * 32, residual, E, lane);
    epi_chunk<F, BN + 4>(rows + cc * 32, G, rowoff, rstore, rw, cc * 32, tn * BN + cc * 32, out, E, lane,
                         stw[0][cc][lane], stw[1][cc][lane], stw[2][cc][lane]);
  }
}

// launch-uniform dispatch over the variants the network uses
template <int BN, bool AFF>
__device__ __forceinline__ void epi_tile_dispatch(const int mode, const float* __restrict__ rows,
                                                  float (*stw)[BN / 32][32], const long long (&rowoff)[4],
                                                  const bool (&rvalid)[4], const bool do_store, const int tn,
                                                  const bf16* residual, bf16* out, const EpiBwd& E, const int lane,
                                                  const int half) {
#define MN_EPI_CASE(Fv) case (Fv): epi_tile<(Fv), BN>(rows, stw, rowoff, rvalid, do_store, tn, residual, out, E, lane, half); break;
  if constexpr (AFF) {
    // eval-mode inference, its own kernel instantiations (k_tc_conv<BN, true>) so that the training kernels keep
    // their register allocation: stem / conv1 (ReLU), downsample (no ReLU), conv2 (+ block input or downsample
    // output, ReLU)
    switch (mode) {
      MN_EPI_CASE(EPI_AFFINE | EPI_RELU)
      MN_EPI_CASE(EPI_AFFINE)
      MN_EPI_CASE(EPI_AFFINE | EPI_RES | EPI_RELU)
      MN_EPI_CASE(EPI_OUT32 | EPI_AFFINE | EPI_RELU)
      MN_EPI_CASE(EPI_OUT32 | EPI_AFFINE | EPI_RELU | EPI_HOUT)
      MN_EPI_CASE(EPI_OUT32 | EPI_AFFINE)
      MN_EPI_CASE(EPI_OUT32 | EPI_AFFINE | EPI_RES | EPI_RELU | EPI_HOUT)
      MN_EPI_CASE(EPI_OUT32 | EPI_AFFINE | EPI_RES | EPI_HRES | EPI_RELU | EPI_HOUT)
      default: __trap();
    }
    return;
  }
  switch (mode) {
    MN_EPI_CASE(0)
    MN_EPI_CASE(EPI_RES)
    MN_EPI_CASE(EPI_STATS)
    MN_EPI_CASE(EPI_BWD)
    MN_EPI_CASE(EPI_BWD | EPI_RES)
    MN_EPI_CASE(EPI_BWD | EPI_ZMASK)
    MN_EPI_CASE(EPI_BWD | EPI_ZMASK | EPI_RES)
    MN_EPI_CASE(EPI_BWD | EPI_ZMASK | EPI_YD)
    MN_EPI_CASE(EPI_BWD | EPI_ZMASK | EPI_RES | EPI_YD)
    MN_EPI_CASE(EPI_OUT32)
    MN_EPI_CASE(EPI_OUT32 | EPI_RES)
    MN_EPI_CASE(EPI_OUT32 | EPI_STATS)
    default: __trap();
  }
#undef MN_EPI_CASE
}

// the affine epilogue bits of a launch (host and device): what tc_affine_supported checks and epi_mode_of dispatches on
__host__ __device__ __forceinline__ int affine_mode(const bool split, const bool residual, const int relu, const int res_split,
                                                   const int out_split) {
  int m = EPI_AFFINE | (residual ? EPI_RES : 0) | (relu ? EPI_RELU : 0);
  if (split) m |= EPI_OUT32 | (out_split ? EPI_HOUT : 0) | ((residual && res_split) ? EPI_HRES : 0);
  return m;
}

bool tc_affine_supported(bool split, bool residual, const EpiAffine& a) {
  if (a.scale == nullptr || a.shift == nullptr) return false;
  if (!split && (a.res_split || a.out_split)) return false;
  static const int built[] = {
      EPI_AFFINE | EPI_RELU, EPI_AFFINE, EPI_AFFINE | EPI_RES | EPI_RELU, EPI_OUT32 | EPI_AFFINE | EPI_RELU,
      EPI_OUT32 | EPI_AFFINE | EPI_RELU | EPI_HOUT, EPI_OUT32 | EPI_AFFINE,
      EPI_OUT32 | EPI_AFFINE | EPI_RES | EPI_RELU | EPI_HOUT,
      EPI_OUT32 | EPI_AFFINE | EPI_RES | EPI_HRES | EPI_RELU | EPI_HOUT};
  const int m = affine_mode(split, residual, a.relu, a.res_split, a.out_split);
  for (int b : built) if (b == m) return true;
  return false;
}

template <bool AFF>
__device__ __forceinline__ int epi_mode_of(const bf16* residual, const double* stats, const EpiBwd& E, const int out32) {
  int m = (residual != nullptr) ? EPI_RES : 0;
  if (out32) m |= EPI_OUT32;
  if (AFF) {
    m |= EPI_AFFINE | E.aflags;
  } else if (E.y != nullptr) {
    m |= EPI_BWD;
    if (E.zmask != nullptr) m |= EPI_ZMASK;
    if (E.yd != nullptr) m |= EPI_YD;
  } else if (stats != nullptr) {
    m |= EPI_STATS;
  }
  return m;
}

// ---- statistics flush (epilogue warps only: kEpiThreads threads, named barrier 1) ----
static constexpr int kConvReplicas = 8;        // accumulator replicas the conv engines spread their flushes over

__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, %0;" ::"n"(kEpiThreads) : "memory"); }

// Combine the four epilogue warps' running column sums of N tile `tn` in shared memory and add them to this
// CTA's accumulator replica: one fp64 atomic per (statistic, column) per CTA.
template <int BN>
__device__ __forceinline__ void epi_flush(float (*all)[3][BN / 32][32], double* __restrict__ stats, const int Cout,
                                          const int tn, const bool third, const int etid) {
  epi_bar();                                    // every warp's sums for this N tile are in shared memory
  double* acc = stats + (size_t)(blockIdx.x % kConvReplicas) * kBnAccStride;   // bn_fin.cuh layout
  const int nstat = third ? 3 : 2;
#pragma unroll 1
  for (int e = etid; e < nstat * BN; e += kEpiThreads) {
    const int j = e / BN, rem = e - j * BN, i = rem >> 5, l = rem & 31;
    const float t = all[0][j][i][l] + all[1][j][i][l] + all[2][j][i][l] + all[3][j][i][l];
    all[0][j][i][l] = 0.f; all[1][j][i][l] = 0.f; all[2][j][i][l] = 0.f; all[3][j][i][l] = 0.f;
    atomicAdd(acc + (size_t)j * Cout + tn * BN + i * 32 + epi_stat_col(l), (double)t);
  }
  epi_bar();                                    // zeroed before any warp accumulates the next N tile
}

// as many stages as fit in 227 KB next to the accumulator staging rows: the engines are bound by bytes in flight
static constexpr int conv_stages(int BN) { return BN <= 64 ? 7 : 4; }
static constexpr size_t conv_smem_bytes(int BN) {
  return (size_t)conv_stages(BN) * (128 * 128 + BN * 128) + (size_t)128 * (BN + 4) * 4 + 1024;
}
// wgrad runs two CTAs per SM, each with half the stages that would fit for one: the store epilogue of one CTA overlaps
// the other CTA's MMAs instead of idling the tensor cores (measured: 587 -> 781 TF/s on layer3/4 wgrad)
static constexpr int wgrad_stages(int BN) { return (BN <= 64 ? 9 : 6) / 2; }

// named barrier of one consumer warpgroup (barrier 0 is __syncthreads, 1 is epi_bar)
__device__ __forceinline__ void wg_bar(const int wg) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); }

// release a pipeline stage: one thread per consumer warpgroup arrives on the stage's empty barrier
__device__ __forceinline__ void release_stage(const uint32_t empty_bar, const bool arriver) {
  if (arriver) mbar_arrive(empty_bar);
}

// Mainloop of one tile for one consumer warpgroup: kblocks k-blocks, each KSTEPS wgmma instructions (bf16: 64 channels
// as four K=16 steps; e4m3: 128 or 64 channels as four or two K=32 steps -- 32 bytes of a row per step either way).  A
// stage is handed back as soon as the wgmma group that read it has retired (one group stays in flight behind the next).
// a_off / a_step: this warpgroup's A rows inside a stage and the byte step per instruction; b_step likewise for B.
template <int BN, int FMT, int TA, int TB, int KSTEPS = 4>
__device__ __forceinline__ void mma_tile(float (&d)[BN / 2], const int kblocks, int& stage, uint32_t& phase,
                                         const int STAGES, const uint32_t stage_bytes, const uint32_t smem_base,
                                         const uint32_t a_off, const uint32_t a_step, const uint32_t b_off,
                                         const uint32_t b_step, const uint64_t adesc, const uint64_t bdesc,
                                         const uint32_t full0, const uint32_t empty0, const bool arriver,
                                         const bool skip_mma) {
  int prev = -1;
  for (int kb = 0; kb < kblocks; ++kb) {
    mbar_wait(full0 + 8 * stage, phase);
    // One thread releases the stage for its whole warpgroup, which is only safe while every warp has passed the wait
    // above.  The wgmma instructions (.sync.aligned) keep the four warps together; without them a warp could fall a
    // whole ring behind, miss a phase of the full barrier and wait forever.
    if (skip_mma) wg_bar(threadIdx.x >> 7);
    if (!skip_mma) {
      const uint32_t sa = smem_base + stage * stage_bytes + a_off;
      const uint32_t sb = smem_base + stage * stage_bytes + b_off;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < KSTEPS; ++k)
        wgmma_k16<TA, TB>(WgmmaTag<BN, FMT>(), d, smem_desc(adesc, sa + k * a_step), smem_desc(bdesc, sb + k * b_step),
                          (kb > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_fence_acc(d);
    }
    if (prev >= 0) release_stage(empty0 + 8 * prev, arriver);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_acc(d);
  if (prev >= 0) release_stage(empty0 + 8 * prev, arriver);
  if (kblocks == 0 || skip_mma) {         // no filter tap reaches this output class (or MMAs skipped): D = 0
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  }
}

// ---------------------------------------------------------------------------------
// fprop / dgrad kernel
// ---------------------------------------------------------------------------------
// TMA producer of the fprop / dgrad engines (one elected lane): every (work item, filter tap, channel block) of this
// CTA into the stage ring.  KB: channels per block of the activation tensor (bf16: 64; e4m3: 128 or 64 = one 128- or
// 64-byte row), which is also the K extent of the weight box.
template <int STAGES, uint32_t A_BYTES, uint32_t STAGE_BYTES, int BN, int KB>
__device__ __forceinline__ void conv_producer(const ConvParams& P, const CUtensorMap* mapA0, const CUtensorMap* mapA1,
                                              const CUtensorMap* mapA2, const CUtensorMap* mapA3, const CUtensorMap* mapB,
                                              const CUtensorMap* mapB2, const uint32_t smem_base, const uint32_t full0,
                                              const uint32_t empty0, const int first_tile, const int total_tiles,
                                              const int tile_step, const int per_class) {
  int stage = 0; uint32_t phase = 0;
  for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
    const TileCoord tc = decode_tile(tile, per_class, P.n_tiles_n);
    const ClassDesc cd = P.cls[tc.cls];
    const int tn = tc.tn;
    int tm = tc.tm;
    const int tw = tm % P.tiles_w; tm /= P.tiles_w;
    const int th = tm % P.tiles_h;
    const int tb = tm / P.tiles_h;
    const int jw0 = tw * P.TW, jh0 = th * P.TH, n0 = tb * P.TN;
    for (int t = cd.tap0; t < cd.tap0 + cd.num_taps; ++t) {
      const TapDesc tap = P.taps[t];
      const int am = tap.map & 3;
      const CUtensorMap* mA = (am == 0) ? mapA0 : (am == 1) ? mapA1 : (am == 2) ? mapA2 : mapA3;
      const CUtensorMap* mB = (tap.map & 4) ? mapB2 : mapB;
      for (int cb = 0; cb < P.cblocks; ++cb) {
        mbar_wait(empty0 + 8 * stage, phase ^ 1);
        const uint32_t sa = smem_base + stage * STAGE_BYTES;
        if (P.debug == 2) { mbar_arrive(full0 + 8 * stage); if (++stage == STAGES) { stage = 0; phase ^= 1; } continue; }
        mbar_expect_tx(full0 + 8 * stage, STAGE_BYTES);
        tma_load_4d(sa, mA, full0 + 8 * stage, cb * KB, jw0 + tap.dw, jh0 + tap.dh, n0);
        tma_load_2d(sa + A_BYTES, mB, full0 + 8 * stage, tap.kidx * P.Cs + cb * KB, tn * BN);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  }
}

// the 4 output rows this lane owns in the coalesced epilogue layout (tile row q*32 + 8i + (lane>>2)) of M tile tm:
// element offsets of (row, column col0), and whether the row lies inside the tensor
__device__ __forceinline__ void tile_rows(const ConvParams& P, const ClassDesc& cd, int tm, const int q, const int lane,
                                          const int col0, long long (&rowoff)[4], bool (&rvalid)[4]) {
  const int tw = tm % P.tiles_w; tm /= P.tiles_w;
  const int th = tm % P.tiles_h;
  const int tb = tm / P.tiles_h;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = q * 32 + 8 * i + (lane >> 2);
    const int lw = m % P.TW;
    const int lh = (m / P.TW) % P.TH;
    const int ln = m / (P.TW * P.TH);
    const int jw = tw * P.TW + lw, jh = th * P.TH + lh, n = tb * P.TN + ln;
    rvalid[i] = (jw < cd.Ws) && (jh < cd.Hs) && (n < P.Nimg);
    const long long pix = ((long long)n * P.Hout + (jh * P.os + cd.oa)) * P.Wout + (jw * P.os + cd.ob);
    rowoff[i] = (rvalid[i] ? pix * P.Cout : 0) + col0;     // outside rows: clamped, loads stay in bounds
  }
}

// AFF: the eval-mode inference epilogues (EPI_AFFINE) instead of the training ones.
template <int BN, bool AFF = false>
__global__ void __launch_bounds__(kConvThreads, 1)
k_tc_conv(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
          const __grid_constant__ CUtensorMap mapA2, const __grid_constant__ CUtensorMap mapA3,
          const __grid_constant__ CUtensorMap mapB, const __grid_constant__ CUtensorMap mapB2,
          const __grid_constant__ ConvParams P, const bf16* __restrict__ residual,
          bf16* __restrict__ out, double* __restrict__ stats, const EpiBwd E) {
  constexpr int STAGES = conv_stages(BN);
  constexpr uint32_t A_BYTES = 128 * 128;        // 128 pixels x 64 ch bf16
  constexpr uint32_t B_BYTES = BN * 128;
  constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int RS = BN + 4;                     // floats per accumulator staging row
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B swizzle atoms
  const uint32_t smem_base = __shfl_sync(0xffffffffu, (smem_u32(smem_raw) + 1023u) & ~1023u, 0);
  __shared__ __align__(8) uint64_t bars[2 * STAGES];
  const uint32_t full0 = __shfl_sync(0xffffffffu, smem_u32(&bars[0]), 0), empty0 = smem_u32(&bars[STAGES]);

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
  const int lane = threadIdx.x & 31;

  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&mapA0); prefetch_tmap(&mapB);
    for (int i = 0; i < STAGES; ++i) { mbar_init(full0 + 8 * i, 1); mbar_init(empty0 + 8 * i, 2); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_prologue();      // nothing above touches global memory: setup overlaps the previous kernel's tail

  // work items: (M tile, N tile) per class; the persistent CTAs take them round-robin
  const int per_class = P.n_tiles_m * P.n_tiles_n;
  const int total_tiles = per_class * P.n_classes;
  const int first_tile = blockIdx.x;
  const int tile_step = gridDim.x;

  if (warp == kProducerWarp) {
    // ===================== TMA producer =====================
    if (elect_one())
      conv_producer<STAGES, A_BYTES, STAGE_BYTES, BN, 64>(P, &mapA0, &mapA1, &mapA2, &mapA3, &mapB, &mapB2, smem_base, full0,
                                                         empty0, first_tile, total_tiles, tile_step, per_class);
  } else {
    // ===================== consumer warpgroups: MMAs, then the epilogue of their own 64 rows =====================
    const int wg = warp >> 2;               // accumulator rows 64*wg .. 64*wg + 63 of the tile
    const int wq = warp & 3;
    const int q = 2 * wg + (wq >> 1);       // the 32-row quarter this warp's epilogue walks
    const int half = wq & 1;                // which of the quarter's chunk subsets
    const bool arriver = (threadIdx.x & 127) == 0;
    float* stg = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw)) + STAGES * STAGE_BYTES);
    const int epi_mode = epi_mode_of<AFF>(residual, stats, E, P.out32);
    constexpr uint64_t DESC_BASE = make_smem_desc_base(16, 1024);
    int stage = 0; uint32_t phase = 0;
    // running column sums of this warp, [statistic][chunk][lane] (lane <-> column epi_stat_col(lane)); kept in
    // shared memory so that the chunk loop can stay ROLLED (unrolled, the epilogue's code size stalls the
    // epilogue warps on instruction fetch)
    __shared__ float epi_stats[4][3][BN / 32][32];
    float (*stw)[BN / 32][32] = epi_stats[q];
#pragma unroll 1
    for (int i = half; i < BN / 32; i += kEpiSplit) { stw[0][i][lane] = 0.f; stw[1][i][lane] = 0.f; stw[2][i][lane] = 0.f; }
    int st_tn = -1;
    const int etid = warp * 32 + lane;
    auto flush_stats = [&](int tn_flush) { epi_flush<BN>(epi_stats, stats, P.Cout, tn_flush, E.yd != nullptr, etid); };
    for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
      const TileCoord tc = decode_tile(tile, per_class, P.n_tiles_n);
      const ClassDesc cd = P.cls[tc.cls];
      const int kblocks = cd.num_taps * P.cblocks;
      const int tn = tc.tn;
      float d[BN / 2];
      if (P.fmt_a)
        mma_tile<BN, 1, 0, 0>(d, kblocks, stage, phase, STAGES, STAGE_BYTES, smem_base, wg * 64 * 128, 32, A_BYTES, 32,
                              DESC_BASE, DESC_BASE, full0, empty0, arriver, P.debug == 1);
      else
        mma_tile<BN, 0, 0, 0>(d, kblocks, stage, phase, STAGES, STAGE_BYTES, smem_base, wg * 64 * 128, 32, A_BYTES, 32,
                              DESC_BASE, DESC_BASE, full0, empty0, arriver, P.debug == 1);
      // inference launches carry no statistics (tc_conv_run checks it): no flush is compiled into those kernels
      if (!AFF && stats != nullptr && tn != st_tn) { if (st_tn >= 0) flush_stats(st_tn); st_tn = tn; }
      long long rowoff[4]; bool rvalid[4];
      tile_rows(P, cd, tc.tm, q, lane, tn * BN, rowoff, rvalid);
      if (P.debug == 3) continue;           // micro-benchmark: no epilogue work at all
      wg_bar(wg);                             // the previous tile's staged rows have been read
      acc_to_stage<BN>(d, stg + wg * 64 * RS, wq, lane);
      wg_bar(wg);
      epi_tile_dispatch<BN, AFF>(epi_mode, stg + q * 32 * RS, stw, rowoff, rvalid, P.debug != 4, tn, residual, out, E, lane,
                            half);
    }
    if (!AFF && stats != nullptr && st_tn >= 0) flush_stats(st_tn);
  }
}

// ---------------------------------------------------------------------------------
// fp8 inference fprop: e4m3 operands, fp32 accumulation, the affine epilogue on a folded table
// ---------------------------------------------------------------------------------
// The pipeline of k_tc_conv (producer warp, mbarrier ring, persistent tiles, coalesced epilogue) with e4m3 tiles.  A
// k-block is one row of KB bytes = KB channels per pixel: KB = 128 keeps bf16's stage layout, 128B swizzle and 32-byte
// instruction step (four m64nBNk32 per stage); KB = 64 (the Cin = 64 convs) uses 64B-swizzled rows, two instructions
// per stage and twice the stages in the same shared memory.
static constexpr int f8_stages(int BN, int KB) { return KB == 128 ? conv_stages(BN) : 2 * conv_stages(BN); }
static constexpr size_t f8_smem_bytes(int BN, int KB) {
  return (size_t)f8_stages(BN, KB) * (128 * KB + BN * KB) + (size_t)128 * (BN + 4) * 4 + 1024;
}

// launch-uniform dispatch over the variants the fp8 schedule uses (EpiF8::mode)
template <int BN>
__device__ __forceinline__ void f8_epi_dispatch(const int mode, const float* __restrict__ rows, float (*stw)[BN / 32][32],
                                                const long long (&rowoff)[4], const bool (&rvalid)[4], const int tn,
                                                const void* residual, void* out, const EpiF8Dev& E, const int lane,
                                                const int half) {
#define MN_F8_CASE(Fv) case (Fv): epi_tile<(Fv), BN>(rows, stw, rowoff, rvalid, true, tn, (const bf16*)residual, (bf16*)out, E, lane, half); break;
  switch (mode) {
    MN_F8_CASE(EPI_AFFINE | EPI_RELU | EPI_F8OUT)                         // conv1
    MN_F8_CASE(EPI_AFFINE)                                                // downsample: bf16 out
    MN_F8_CASE(EPI_AFFINE | EPI_RES | EPI_RELU | EPI_F8OUT)               // conv2 after a downsample (bf16 residual)
    MN_F8_CASE(EPI_AFFINE | EPI_RES | EPI_F8RES | EPI_RELU | EPI_F8OUT)   // conv2, identity (e4m3 residual)
    MN_F8_CASE(EPI_AFFINE | EPI_RELU | EPI_AMAX)                          // calibration of the three above
    MN_F8_CASE(EPI_AFFINE | EPI_RES | EPI_RELU | EPI_AMAX)
    MN_F8_CASE(EPI_AFFINE | EPI_RES | EPI_F8RES | EPI_RELU | EPI_AMAX)
    default: __trap();
  }
#undef MN_F8_CASE
}

template <int BN, int KB>
__global__ void __launch_bounds__(kConvThreads, 1)
k_f8_conv(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
          const __grid_constant__ CUtensorMap mapA2, const __grid_constant__ CUtensorMap mapA3,
          const __grid_constant__ CUtensorMap mapB, const __grid_constant__ ConvParams P, const void* __restrict__ residual,
          void* __restrict__ out, const EpiF8Dev E) {
  static_assert(KB == 128 || KB == 64, "e4m3 k-blocks are 128- or 64-byte rows");
  constexpr int STAGES = f8_stages(BN, KB);
  constexpr uint32_t A_BYTES = 128 * KB;         // 128 pixels x KB channels
  constexpr uint32_t B_BYTES = BN * KB;
  constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int RS = BN + 4;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = __shfl_sync(0xffffffffu, (smem_u32(smem_raw) + 1023u) & ~1023u, 0);
  __shared__ __align__(8) uint64_t bars[2 * STAGES];
  const uint32_t full0 = __shfl_sync(0xffffffffu, smem_u32(&bars[0]), 0), empty0 = smem_u32(&bars[STAGES]);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&mapA0); prefetch_tmap(&mapB);
    for (int i = 0; i < STAGES; ++i) { mbar_init(full0 + 8 * i, 1); mbar_init(empty0 + 8 * i, 2); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_prologue();
  const int per_class = P.n_tiles_m * P.n_tiles_n;
  const int total_tiles = per_class * P.n_classes;
  if (warp == kProducerWarp) {
    if (elect_one())
      conv_producer<STAGES, A_BYTES, STAGE_BYTES, BN, KB>(P, &mapA0, &mapA1, &mapA2, &mapA3, &mapB, &mapB, smem_base, full0,
                                                         empty0, blockIdx.x, total_tiles, gridDim.x, per_class);
    return;
  }
  const int wg = warp >> 2, wq = warp & 3;
  const int q = 2 * wg + (wq >> 1), half = wq & 1;
  const bool arriver = (threadIdx.x & 127) == 0;
  float* stg = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw)) + STAGES * STAGE_BYTES);
  constexpr uint64_t DESC_BASE = KB == 128 ? make_smem_desc_base(16, 1024) : make_smem_desc_base_sw64(16, 512);
  // EPI_AMAX: per-warp running max |f| of each (chunk, lane), as the training kernels keep their column sums
  __shared__ float epi_amax[4][3][BN / 32][32];
  float (*stw)[BN / 32][32] = epi_amax[q];
  for (int i = half; i < BN / 32; i += kEpiSplit) stw[0][i][lane] = 0.f;
  int stage = 0; uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const TileCoord tc = decode_tile(tile, per_class, P.n_tiles_n);
    const ClassDesc cd = P.cls[tc.cls];
    float d[BN / 2];
    mma_tile<BN, 2, 0, 0, KB / 32>(d, cd.num_taps * P.cblocks, stage, phase, STAGES, STAGE_BYTES, smem_base, wg * 64 * KB,
                                   32, A_BYTES, 32, DESC_BASE, DESC_BASE, full0, empty0, arriver, false);
    long long rowoff[4]; bool rvalid[4];
    tile_rows(P, cd, tc.tm, q, lane, tc.tn * BN, rowoff, rvalid);
    wg_bar(wg);
    acc_to_stage<BN>(d, stg + wg * 64 * RS, wq, lane);
    wg_bar(wg);
    f8_epi_dispatch<BN>(E.aflags, stg + q * 32 * RS, stw, rowoff, rvalid, tc.tn, residual, out, E, lane, half);
  }
  if (E.aflags & EPI_AMAX) {        // the bit patterns of non-negative floats order as the floats do
    float m = 0.f;
    for (int i = half; i < BN / 32; i += kEpiSplit) m = fmaxf(m, stw[0][i][lane]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) atomicMax(E.amax, __float_as_uint(m));
  }
}

// ---------------------------------------------------------------------------------
// wgrad epilogue: this thread's accumulator fragment -- rows r = 16*wq + lane/4 and r + 8 of X chunk `ch`
// (input channels), columns 8j + 2*(lane%4) (+1) from col0 (output channels) -- into dW[co][tap][ci] at `dw`.
// Every element has exactly one writer per launch (split): with one split it is added into the gradient buffer
// (which may already hold a gradient to accumulate onto), with several it is STORED into the split's slice of the
// workspace and k_wgrad_reduce adds the slices up in a fixed order -- the result does not depend on CTA timing.
// Strict mode: rows and columns index the split planes -- row r of a 64-element chunk is channel
// (r/16)*8 + r%8 of plane (r/8)%2, columns likewise -- so the four hi/lo products of one (co, ci) pair are the
// cells (r, c), (r+8, c), (r, c+8), (r+8, c+8), all held by the same thread: summed in registers, one atomic.
// ---------------------------------------------------------------------------------
template <int BN, int JG = 4>
__device__ __forceinline__ void wgrad_store(const WgradParams& P, float* __restrict__ dw, const float (&d)[BN / 2],
                                            const WgradChunk& ch, const int col0, const int wq, const int lane) {
  const int r = 16 * wq + (lane >> 2);
  const int c = 2 * (lane & 3);
  const bool store = P.partial != nullptr;
  auto put = [&](float* p, const float v) { if (store) *p = v; else *p += v; };
  if (!P.split) {
    // Adding into dw reads it first.  The compiler cannot tell that the addresses differ, so one `+=` at a time makes
    // every load wait for the previous store: BN / 2 dependent DRAM round trips per thread (measured on H100: more than
    // half of a layer4 wgrad).  Groups of 4 * JG loads (JG j values x 2 x 2) are issued together before their adds and
    // stores instead.
    // element (co = col0 + c + k, row r) is at p0 + k * cstride
    float* p0 = dw + ((long long)(col0 + c) * P.KK + ch.tap) * P.Ci + ch.c0 + r;
    const int cstride = P.KK * P.Ci;
    const int kend = P.Co - col0 - c;          // k < kend: inside the tensor
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += JG) {
      float old[JG][2][2];
#pragma unroll
      for (int j = 0; j < JG; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int k = 8 * (j0 + j) + e;
          const bool ld = !store && k < kend;
          old[j][e][0] = ld ? p0[k * cstride] : 0.f;
          old[j][e][1] = ld ? p0[k * cstride + 8] : 0.f;
        }
#pragma unroll
      for (int j = 0; j < JG; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int k = 8 * (j0 + j) + e;
          if (k < kend) {
            const float v0 = d[4 * (j0 + j) + e], v1 = d[4 * (j0 + j) + 2 + e];
            p0[k * cstride] = store ? v0 : old[j][e][0] + v0;
            p0[k * cstride + 8] = store ? v1 : old[j][e][1] + v1;
          }
        }
    }
    return;
  }
  const float osc = (P.oscale != nullptr) ? __ldg(P.oscale) : 1.f;
  // real input channel of rows r / r + 8: chunk offset c0 (in split elements) -> c0/2 real channels
  const int ci = (ch.c0 >> 1) + ((r >> 4) << 3) + (r & 7);
#pragma unroll
  for (int g = 0; g < BN / 16; ++g)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float s = d[8 * g + e] + d[8 * g + 2 + e] + d[8 * g + 4 + e] + d[8 * g + 6 + e];
      const int co = ((col0 + 16 * g) >> 1) + c + e;
      if (co < P.Co) put(dw + ((long long)co * P.KK + ch.tap) * P.Ci + ci, s * osc);
    }
}

// ---------------------------------------------------------------------------------
// wgrad kernel: one CTA per (M-tile of 2 X chunks, N-tile of BN couts, K split); consumer warpgroup j owns chunk j
// ---------------------------------------------------------------------------------
// two CTAs per SM (wgrad_stages)
template <int BN>
__global__ void __launch_bounds__(kConvThreads, 2)
k_tc_wgrad(const __grid_constant__ CUtensorMap mapX0, const __grid_constant__ CUtensorMap mapX1,
           const __grid_constant__ CUtensorMap mapX2, const __grid_constant__ CUtensorMap mapX3,
           const __grid_constant__ CUtensorMap mapDY, const __grid_constant__ WgradParams P,
           float* __restrict__ dw) {
  constexpr int STAGES = wgrad_stages(BN);
  constexpr uint32_t CHUNK_BYTES = 64 * 128;     // 64 pixels x 64 ch bf16
  constexpr uint32_t A_BYTES = 2 * CHUNK_BYTES;
  constexpr uint32_t B_BYTES = (BN / 64) * CHUNK_BYTES;
  constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = __shfl_sync(0xffffffffu, (smem_u32(smem_raw) + 1023u) & ~1023u, 0);
  __shared__ __align__(8) uint64_t bars[2 * STAGES];
  const uint32_t full0 = __shfl_sync(0xffffffffu, smem_u32(&bars[0]), 0), empty0 = smem_u32(&bars[STAGES]);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
  const int lane = threadIdx.x & 31;

  // unit decode
  int u = blockIdx.x;
  const int split = u % P.splits; u /= P.splits;
  const int nt = u % P.n_ntiles;
  const int mt = u / P.n_ntiles;
  const int c_lo = mt * 2;
  const int n_valid_chunks = (c_lo + 1 < P.n_chunks) ? 2 : 1;
  const int t_beg = split * P.tiles_per_split;
  int t_end = t_beg + P.tiles_per_split; if (t_end > P.n_pix_tiles) t_end = P.n_pix_tiles;
  const int ksteps = (t_end > t_beg) ? (t_end - t_beg) : 0;

  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&mapX0); prefetch_tmap(&mapDY);
    for (int i = 0; i < STAGES; ++i) { mbar_init(full0 + 8 * i, 1); mbar_init(empty0 + 8 * i, 2); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_prologue();      // nothing above touches global memory: setup overlaps the previous kernel's tail

  if (warp == kProducerWarp) {
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      const WgradChunk ch0 = wgrad_chunk(P, c_lo);
      const WgradChunk ch1 = wgrad_chunk(P, (n_valid_chunks == 2) ? c_lo + 1 : c_lo);
      const CUtensorMap* m0 = (ch0.map == 0) ? &mapX0 : (ch0.map == 1) ? &mapX1 : (ch0.map == 2) ? &mapX2 : &mapX3;
      const CUtensorMap* m1 = (ch1.map == 0) ? &mapX0 : (ch1.map == 1) ? &mapX1 : (ch1.map == 2) ? &mapX2 : &mapX3;
      for (int t = t_beg; t < t_end; ++t) {
        int tt = t;
        const int tw = tt % P.tiles_w; tt /= P.tiles_w;
        const int th = tt % P.tiles_h;
        const int tb = tt / P.tiles_h;
        const int ow0 = tw * P.TW, oh0 = th * P.TH, n0 = tb * P.TN;
        mbar_wait(empty0 + 8 * stage, phase ^ 1);
        const uint32_t sa = smem_base + stage * STAGE_BYTES;
        mbar_expect_tx(full0 + 8 * stage, STAGE_BYTES);
        tma_load_4d(sa, m0, full0 + 8 * stage, ch0.c0, ow0 + ch0.dw, oh0 + ch0.dh, n0);
        tma_load_4d(sa + CHUNK_BYTES, m1, full0 + 8 * stage, ch1.c0, ow0 + ch1.dw, oh0 + ch1.dh, n0);
#pragma unroll
        for (int j = 0; j < BN / 64; ++j)
          tma_load_4d(sa + A_BYTES + j * CHUNK_BYTES, &mapDY, full0 + 8 * stage, nt * BN + j * 64, ow0, oh0, n0);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    const int wg = warp >> 2;                 // X chunk c_lo + wg = accumulator rows
    // MN-major, 128B swizzle: LBO = stride between 64-element MN chunks, SBO = 8-pixel group stride;
    // 64 pixels per stage = 4 x K16, 16 pixel rows = 2048 B
    constexpr uint64_t DESC_BASE = make_smem_desc_base(CHUNK_BYTES, 1024);
    int stage = 0; uint32_t phase = 0;
    float d[BN / 2];
    const bool arriver = (threadIdx.x & 127) == 0;
    if (P.fmt_a)
      mma_tile<BN, 1, 1, 1>(d, ksteps, stage, phase, STAGES, STAGE_BYTES, smem_base, wg * CHUNK_BYTES, 2048, A_BYTES,
                            2048, DESC_BASE, DESC_BASE, full0, empty0, arriver, false);
    else
      mma_tile<BN, 0, 1, 1>(d, ksteps, stage, phase, STAGES, STAGE_BYTES, smem_base, wg * CHUNK_BYTES, 2048, A_BYTES,
                            2048, DESC_BASE, DESC_BASE, full0, empty0, arriver, false);
    float* dst = (P.partial != nullptr) ? P.partial + (long long)split * P.part_stride : dw;
    if (ksteps > 0 && wg < n_valid_chunks && P.debug != 3)
      wgrad_store<BN>(P, dst, d, wgrad_chunk(P, c_lo + wg), nt * BN, warp & 3, lane);
  }
}

// ---------------------------------------------------------------------------------
// stride-1 3x3 wgrad from a staged input halo: one CTA per (64-channel X block, tap group, N tile of BN, K split)
// ---------------------------------------------------------------------------------
// k_tc_wgrad loads every filter tap's X box on its own, although the nine boxes of one pixel box are shifted views of
// one halo, and loads the dY tile again for every M tile: its operand stream, not its MMAs, bounds it.  Here each
// k-block loads the halo of the pixel box (NWG filter rows; zero outside the tensor, as the per-tap boxes are) and the
// dY tile once.  Tap (kh0 + wg, kw) of k16 step j is a descriptor into the halo at row step_row[j] + wg * RW + kw: the
// same pixels in the same order as the per-tap box, so every dW element sees the same wgmma k16 steps as in
// k_tc_wgrad and comes out bit for bit the same.  NWG consumer warpgroups, one per filter row, hold three accumulators
// each (one per filter column).  The 128B swizzle of a shifted start row follows from its address (the halo is
// 1024-byte aligned, the descriptor's base offset stays 0).
static constexpr uint32_t halo_max_bytes(int NWG) { return NWG == 3 ? 28672u : 16384u; }   // 224 / 128 halo rows
static constexpr int halo_stages(int BN, int NWG) { return (NWG == 1 && BN == 64) ? 4 : 6; }
static constexpr int halo_ctas_per_sm(int BN, int NWG) { return (NWG == 1 && BN == 64) ? 2 : 1; }
static constexpr size_t halo_smem_bytes(int BN, int NWG) {
  return (size_t)halo_stages(BN, NWG) * (halo_max_bytes(NWG) + BN * 128) + 1024;
}

template <int BN, int NWG>
__global__ void __launch_bounds__(NWG * 128 + 32, halo_ctas_per_sm(BN, NWG))
k_halo_wgrad(const __grid_constant__ CUtensorMap mapH, const __grid_constant__ CUtensorMap mapDY,
                const __grid_constant__ WgradParams P, float* __restrict__ dw) {
  static_assert(NWG == 1 || (NWG == 3 && BN == 64), "9 taps hold 3 x 64 x BN accumulators per warpgroup: BN 64 only");
  constexpr int STAGES = halo_stages(BN, NWG);
  constexpr uint32_t HALO_BYTES = halo_max_bytes(NWG);
  constexpr uint32_t CHUNK_BYTES = 64 * 128;
  constexpr uint32_t STAGE_BYTES = HALO_BYTES + BN * 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = __shfl_sync(0xffffffffu, (smem_u32(smem_raw) + 1023u) & ~1023u, 0);
  __shared__ __align__(8) uint64_t bars[2 * STAGES];
  const uint32_t full0 = __shfl_sync(0xffffffffu, smem_u32(&bars[0]), 0), empty0 = smem_u32(&bars[STAGES]);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  int u = blockIdx.x;
  const int split = u % P.splits; u /= P.splits;
  const int n_nt = P.Co / BN;
  const int nt = u % n_nt; u /= n_nt;
  const int kh0 = (u % (3 / NWG)) * NWG;      // first filter row of this CTA
  const int cb = u / (3 / NWG);               // 64-channel X block
  const int t_beg = split * P.tiles_per_split;
  int t_end = t_beg + P.tiles_per_split; if (t_end > P.n_pix_tiles) t_end = P.n_pix_tiles;
  const int ksteps = (t_end > t_beg) ? (t_end - t_beg) : 0;

  if (warp == 4 * NWG && lane == 0) {
    prefetch_tmap(&mapH); prefetch_tmap(&mapDY);
    for (int i = 0; i < STAGES; ++i) { mbar_init(full0 + 8 * i, 1); mbar_init(empty0 + 8 * i, NWG); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_prologue();

  if (warp == 4 * NWG) {
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      const uint32_t tx = (uint32_t)P.halo_bytes + BN * 128;
      for (int t = t_beg; t < t_end; ++t) {
        int tt = t;
        const int tw = tt % P.tiles_w; tt /= P.tiles_w;
        const int th = tt % P.tiles_h;
        const int tb = tt / P.tiles_h;
        const int ow0 = tw * P.TW, oh0 = th * P.TH, n0 = tb * P.TN;
        mbar_wait(empty0 + 8 * stage, phase ^ 1);
        const uint32_t sa = smem_base + stage * STAGE_BYTES;
        mbar_expect_tx(full0 + 8 * stage, tx);
        tma_load_4d(sa, &mapH, full0 + 8 * stage, cb * 64, ow0 - 1, oh0 + kh0 - 1, n0);
#pragma unroll
        for (int j = 0; j < BN / 64; ++j)
          tma_load_4d(sa + HALO_BYTES + j * CHUNK_BYTES, &mapDY, full0 + 8 * stage, nt * BN + j * 64, ow0, oh0, n0);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    const int wg = warp >> 2;                 // filter row kh0 + wg
    const uint64_t adesc = make_smem_desc_base(CHUNK_BYTES, (uint32_t)P.halo_sbo);
    constexpr uint64_t BDESC = make_smem_desc_base(CHUNK_BYTES, 1024);
    uint32_t arow[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) arow[j] = (uint32_t)(P.step_row[j] + wg * P.RW) * 128u;
    const bool arriver = (threadIdx.x & 127) == 0;
    float d[3][BN / 2];
    int stage = 0, prev = -1; uint32_t phase = 0;
    for (int kb = 0; kb < ksteps; ++kb) {
      mbar_wait(full0 + 8 * stage, phase);
      const uint32_t sa = smem_base + stage * STAGE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint64_t db = smem_desc(BDESC, sa + HALO_BYTES + j * 2048);
#pragma unroll
        for (int kw = 0; kw < 3; ++kw)
          wgmma_k16<1, 1>(WgmmaTag<BN, 1>(), d[kw], smem_desc(adesc, sa + arow[j] + kw * 128), db,
                          (kb > 0 || j > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) wgmma_fence_acc(d[kw]);
      if (prev >= 0) release_stage(empty0 + 8 * prev, arriver);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) wgmma_fence_acc(d[kw]);
    if (prev >= 0) release_stage(empty0 + 8 * prev, arriver);
    float* dst = (P.partial != nullptr) ? P.partial + (long long)split * P.part_stride : dw;
    if (ksteps > 0) {
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        WgradChunk ch;
        ch.tap = (kh0 + wg) * 3 + kw; ch.c0 = cb * 64; ch.dh = 0; ch.dw = 0; ch.map = 0;
        wgrad_store<BN, NWG == 3 ? 2 : 4>(P, dst, d[kw], ch, nt * BN, warp & 3, lane);   // 9 taps: within 128 registers
      }
    }
  }
}

// dw[i] += sum over splits s = 0, 1, ... of part[s * stride + i], added in that order (4 elements per thread).  The
// loads of 8 splits are issued together before their adds: one dependent DRAM round trip per split would make the
// kernel latency-bound (tens of splits, few elements per thread).
__global__ void k_wgrad_reduce(const float4* __restrict__ part, const long long stride4, const int splits,
                               const long long n4, float4* __restrict__ dw) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k0 = 0; k0 < splits; k0 += 8) {
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        v[j] = (k0 + j < splits) ? part[(long long)(k0 + j) * stride4 + i] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s.x += v[j].x; s.y += v[j].y; s.z += v[j].z; s.w += v[j].w; }
    }
    float4 o = dw[i];
    o.x += s.x; o.y += s.y; o.z += s.z; o.w += s.w;
    dw[i] = o;
  }
}

// ---------------------------------------------------------------------------------
// host plans
// ---------------------------------------------------------------------------------
struct ConvLaunch {
  ConvParams P;
  CUtensorMap mapA[4], mapB, mapB2;
  int n_maps;
  // parity views: (a,b) of map i
  int pa[4], pb[4];
};

struct TcConvPlan {
  ConvGeom g;
  int kind;
  const bf16* wmat;
  const bf16* wmat2;                    // dgrad weight matrix [Ci][Co2] of a folded 1x1/stride-2 shortcut conv, or null
  int BN;
  std::vector<ConvLaunch> launches;    // fprop: 1; dgrad: 1 (stride 1) or 4 (stride 2)
  // wgrad
  WgradParams WP;
  CUtensorMap mapX[4], mapDY;
  int wpa[4], wpb[4], w_nmaps;
  int shortcut_flops_k;                 // K of the folded shortcut (0: none), for the callers' FLOP accounting
  // cached pointers the maps were encoded for
  const void *c_in0, *c_in1;
  bool smem_attr_set;
  bool smem_attr_aff;                   // ... for the inference (EPI_AFFINE) instantiation of the fprop kernel
  const float* out_scale;              // strict mode dgrad / wgrad: device scalar applied to the accumulators, or null
  float* ws;                            // wgrad with split-K: per-split dW slices (allocated at the first run)
  int f8_kb;                            // fp8 fprop plan (tc_plan_create_f8): bytes per k-block row, 128 or 64; else 0
};

static void pick_box(int Wd, int Hd, int pixels, int* TW, int* TH, int* TN) {
  int tw = 8;
  while (tw < Wd && tw < pixels) tw *= 2;
  int th = 1;
  while (tw * th < pixels && th < Hd) th *= 2;
  int tn = pixels / (tw * th);
  if (tn < 1) tn = 1;
  *TW = tw; *TH = th; *TN = tn;
}

// N tile by a small cost model: wider tiles re-use the A operand more, but must still leave enough work items to
// occupy the SMs.  A k-block costs max(bytes staged / ingest rate, MMA issue time) plus a fixed cost per work item
// (prologue, epilogue).  The constants -- ~55 B per cycle of TMA ingest, 580 / 600 cycles of issue per k-block, ~2000
// cycles per work item -- are carried over from a fit to an earlier tensor-memory engine on another GPU and have NOT
// been measured for these wgmma engines on H100: treat the model as a ranking heuristic between BN = 64 and 128.  On
// H100 the engines stage 20-47 B per cycle per SM and keep 79-93 % of their time with the loads skipped
// (profiles/h100_conv_bound.md): ingest and MMA issue plus epilogue are nearly balanced, neither alone bounds a launch.
// BN is 64 or 128 because a consumer warpgroup holds its 64 x BN fp32 accumulator in registers.  MAPNET_TC_BN=64|128
// forces the choice (where Cout allows it).
static int forced_bn() {
  static int f = -1;
  if (f < 0) { const char* e = getenv("MAPNET_TC_BN"); f = e ? atoi(e) : 0; }
  return f;
}
static double kblock_cycles(int bn) {
  const double bytes = 16384.0 + bn * 128.0;
  const double issue = bn <= 64 ? 580.0 : 600.0;
  return (bytes / 55.0 > issue) ? bytes / 55.0 : issue;
}
// `ncls` classes of `mtiles` M tiles each, class c with kb[c] k-blocks per tile (a stride-2 dgrad launched as ONE
// grid over its parity classes); work items are dealt round-robin to the persistent CTAs, heaviest class first
static int choose_bn_classes(int Cout, long long mtiles, int ncls, const int* kb) {
  int best = 64;
  double best_t = 1e30;
  for (int bn = 64; bn <= 128; bn *= 2) {
    if (Cout % bn != 0) continue;
    if (forced_bn() && bn != forced_bn() && Cout % forced_bn() == 0) continue;
    const long long per_class = mtiles * (Cout / bn);
    const double per_kb = kblock_cycles(bn);
    // slot j gets items j, j + slots, ...: the busiest slot bounds the launch
    double t = 0.0;
    const long long total = per_class * ncls;
    for (int j = 0; j < kNumSMs && j < total; ++j) {
      double tj = 0.0;
      for (long long it = j; it < total; it += kNumSMs) tj += kb[it / per_class] * per_kb + 2000.0;
      if (tj > t) t = tj;
    }
    if (t < best_t) { best_t = t; best = bn; }
  }
  return best;
}

static int choose_bn(int Cout, long long Mpix, int kblocks) {
  const long long mtiles = (Mpix + 127) / 128;
  const int kb[1] = {kblocks};
  return choose_bn_classes(Cout, mtiles, 1, kb);
}

// Halo geometry of a stride-1 3x3 wgrad plan for `taps` (3 or 9) filter taps per CTA, into P.  False when the pixel
// box does not suit k_halo_wgrad: every k16 step must be two runs of 8 consecutive halo rows, the same distance
// apart in every step (that distance is the descriptor's SBO), and the halo must fit its stage slot.
static bool wgrad_halo_geometry(WgradParams& P, int taps) {
  const int RW = (P.TW + 2 + 7) / 8 * 8, HR = P.TH + taps / 3 - 1;
  const long long bytes = 128LL * RW * HR * P.TN;
  if (P.TW % 8 != 0 || bytes > (long long)halo_max_bytes(taps / 3)) return false;
  auto row = [&](int q) { return ((q / (P.TW * P.TH)) * HR + (q / P.TW) % P.TH) * RW + q % P.TW; };
  const int sbo = row(8) - row(0);
  for (int j = 0; j < 4; ++j) {
    for (int i = 1; i < 8; ++i)
      if (row(16 * j + i) != row(16 * j) + i || row(16 * j + 8 + i) != row(16 * j + 8) + i) return false;
    if (row(16 * j + 8) - row(16 * j) != sbo) return false;
  }
  P.RW = RW; P.HR = HR; P.halo_bytes = (int)bytes; P.halo_sbo = sbo * 128;
  for (int j = 0; j < 4; ++j) P.step_row[j] = row(16 * j);
  return true;
}

static bool wgrad_halo_allowed(const ConvGeom& g, const WgradParams& P, int taps, int bn) {
  if (g.split || g.stride != 1 || g.KH != 3 || g.KW != 3 || g.pad != 1 || g.in_pix_stride != 0) return false;
  if (!((taps == 3 && (bn == 64 || bn == 128)) || (taps == 9 && bn == 64)) || g.Co % bn != 0) return false;
  WgradParams Q = P;
  return wgrad_halo_geometry(Q, taps);
}

// Switch a wgrad plan to the halo engine (taps 3 / 9, N tile bn) or back to the per-tap engine (taps 0).  The K
// partition stays as it is: only the units of the grid change.
static void wgrad_use_engine(TcConvPlan* p, int taps, int bn) {
  WgradParams& P = p->WP;
  P.halo_taps = taps; P.halo_bn = taps ? bn : 0;
  if (taps) wgrad_halo_geometry(P, taps);
  p->c_in0 = p->c_in1 = nullptr;         // the X tensor map's box changes
  p->smem_attr_set = false;
}

static int wgrad_units(const WgradParams& P, int taps, int bn) {
  return taps ? (P.Ci / 64) * (9 / taps) * (P.Co / bn) : P.n_mtiles * P.n_ntiles;
}

// Cycles of the busiest SM for one wgrad engine: waves x CTAs sharing the SM x k-blocks per CTA x max(MMA clocks,
// operand bytes / L2 rate) per k-block.  MMA clocks: m64nBNk16 is 64 * BN * 16 MACs at 2048 per clock per SM.  Operand
// bytes: per-tap engine 2 X chunks + the dY tile; halo engine the halo + the dY tile.  CTAs per SM come from the
// kernels' shared memory and registers (checked with -Xptxas -v): per-tap 2, halo 3 taps at BN 64 2, else 1.  The L2
// rate is the operand stream the fprop / dgrad engines reach on H100 (20-47 B/clk/SM, profiles/h100_conv_bound.md).
static constexpr double kWgradL2BytesPerClk = 40.0;
static double wgrad_cost(const WgradParams& P0, int taps, int bn) {
  WgradParams P = P0;
  if (taps) wgrad_halo_geometry(P, taps);
  const double mma = (taps ? taps : 2) * 4 * bn / 2.0;
  const double bytes = (taps ? P.halo_bytes : 2 * 8192) + bn * 128.0;
  const int cps = taps ? ((taps == 3 && bn == 64) ? halo_ctas_per_sm(64, 1) : 1) : 2;
  const long long per_sm = cdiv((long long)wgrad_units(P, taps, bn) * P.splits, kNumSMs);
  const long long waves = (per_sm + cps - 1) / cps, conc = per_sm < cps ? per_sm : cps;
  const double per_kb = mma > bytes / kWgradL2BytesPerClk ? mma : bytes / kWgradL2BytesPerClk;
  return (double)waves * conc * P.tiles_per_split * per_kb;
}

static int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }
static int posmod(int a, int b) { int r = a % b; return r < 0 ? r + b : r; }

int tc_plan_create(TcConvPlan** out, const ConvGeom& g, int kind, const bf16* wmat) {
  *out = nullptr;
  MN_CHECK(g.stride == 1 || g.stride == 2, "tc conv: stride %d unsupported", g.stride);
  MN_CHECK(g.Ci % 64 == 0 && g.Co % 64 == 0, "tc conv: channels must be multiples of 64 (Ci=%d Co=%d)", g.Ci, g.Co);
  MN_CHECK((g.KH == g.KW && (g.KH == 1 || g.KH == 3)) || (g.KH == 4 && g.KW == 1 && g.stride == 1 && g.pad == 0 && kind != 1),
           "tc conv: kernel %dx%d unsupported", g.KH, g.KW);
  MN_CHECK(g.in_pix_stride == 0 || (g.stride == 1 && kind != 1), "tc conv: strided input views only for stride-1 fprop / wgrad");
  TcConvPlan* p = new TcConvPlan();
  p->g = g; p->kind = kind; p->wmat = wmat; p->wmat2 = nullptr; p->shortcut_flops_k = 0;
  p->c_in0 = p->c_in1 = nullptr; p->smem_attr_set = false; p->smem_attr_aff = false; p->out_scale = nullptr; p->ws = nullptr;
  p->f8_kb = 0;
  const int s = g.stride, pad = g.pad, KK = g.KH * g.KW;
  // strict mode: the engines see 2*C 16-bit channels per pixel and every filter tap twice (hi / lo weight planes)
  const int SP = g.split ? 2 : 1;
  MN_CHECK(!g.split || KK <= 9, "tc conv: strict mode supports up to 9 filter taps");
  if (kind == 0) {
    // ---------------- fprop ----------------
    p->BN = choose_bn(g.Co, g.M_out(), SP * KK * (SP * g.Ci / 64));
    ConvLaunch L; memset(&L, 0, sizeof(L));
    ConvParams& P = L.P;
    { const char* e = getenv("MAPNET_TC_DEBUG"); P.debug = e ? atoi(e) : 0; }
    P.fmt_a = P.fmt_b = g.split ? 0 : 1; P.out32 = g.split;
    P.Nimg = g.B;
    P.n_classes = 1;
    P.cls[0].Hs = g.Ho; P.cls[0].Ws = g.Wo; P.cls[0].oa = 0; P.cls[0].ob = 0; P.cls[0].tap0 = 0; P.cls[0].num_taps = SP * KK;
    pick_box(g.Wo, g.Ho, 128, &P.TW, &P.TH, &P.TN);
    P.tiles_w = cdiv(g.Wo, P.TW); P.tiles_h = cdiv(g.Ho, P.TH); P.tiles_n = cdiv(g.B, P.TN);
    P.n_tiles_m = P.tiles_w * P.tiles_h * P.tiles_n; P.n_tiles_n = g.Co / p->BN;
    P.cblocks = SP * g.Ci / 64; P.Cs = SP * g.Ci;
    P.Hout = g.Ho; P.Wout = g.Wo; P.Cout = g.Co; P.os = 1;
    L.n_maps = 0;
    for (int pass = 0; pass < SP; ++pass)
    for (int kh = 0; kh < g.KH; ++kh)
      for (int kw = 0; kw < g.KW; ++kw) {
        TapDesc& t = P.taps[pass * KK + kh * g.KW + kw];
        t.kidx = pass * KK + kh * g.KW + kw;
        if (s == 1) { t.dh = kh - pad; t.dw = kw - pad; t.map = 0; L.pa[0] = L.pb[0] = 0; if (L.n_maps < 1) L.n_maps = 1; }
        else {
          const int a = posmod(kh - pad, 2), b = posmod(kw - pad, 2);
          t.dh = floordiv(kh - pad, 2); t.dw = floordiv(kw - pad, 2);
          int mi = -1;
          for (int i = 0; i < L.n_maps; ++i) if (L.pa[i] == a && L.pb[i] == b) mi = i;
          if (mi < 0) { mi = L.n_maps++; L.pa[mi] = a; L.pb[mi] = b; }
          t.map = mi;
        }
      }
    p->launches.push_back(L);
  } else if (kind == 1) {
    // ---------------- dgrad: gather over dY [B,Ho,Wo,Co], output dX [B,Hi,Wi,Ci] ----------------
    // A stride-s dgrad is s*s parity classes of output pixels (a, b) = (ih % s, iw % s), each reached by its own
    // subset of the filter taps (3x3/s2: 4, 2, 2 and 1 taps; 1x1/s2: 1, 0, 0, 0).
    struct ClassTaps { int a, b, n; TapDesc t[18]; };
    ClassTaps ct[4]; int ncls = 0;
    for (int a = 0; a < s; ++a)
      for (int b = 0; b < s; ++b) {
        if (cdiv(g.Hi - a, s) <= 0 || cdiv(g.Wi - b, s) <= 0) continue;
        ClassTaps& c = ct[ncls++];
        c.a = a; c.b = b; c.n = 0;
        for (int kh = 0; kh < g.KH; ++kh)
          for (int kw = 0; kw < g.KW; ++kw) {
            const int eh = a + pad - kh, ew = b + pad - kw;
            if (posmod(eh, s) != 0 || posmod(ew, s) != 0) continue;
            TapDesc& t = c.t[c.n++];
            t.dh = floordiv(eh, s); t.dw = floordiv(ew, s); t.map = 0; t.kidx = kh * g.KW + kw;
          }
        if (g.split) {                      // the same taps again against the lo weight planes
          const int n1 = c.n;
          for (int k = 0; k < n1; ++k) { c.t[c.n] = c.t[k]; c.t[c.n].kidx += KK; ++c.n; }
        }
      }
    int merge = 1;       // read per plan (not cached): the A/B parity test flips it between trunks
    { const char* e = getenv("MAPNET_TC_DGRAD_MERGE"); if (e) merge = atoi(e); }
    if (s == 1 || merge) {
      // ONE launch over all classes, heaviest class first (the persistent CTAs take work items round-robin).
      // As four launches of 1..4 taps on 1/4 of the pixels each stride-2 dgrad would be four single short waves.
      for (int i = 1; i < ncls; ++i)              // stable insertion sort by tap count, descending
        for (int j = i; j > 0 && ct[j].n > ct[j - 1].n; --j) { ClassTaps tmp = ct[j]; ct[j] = ct[j - 1]; ct[j - 1] = tmp; }
      const int Hs0 = cdiv(g.Hi, s), Ws0 = cdiv(g.Wi, s);      // the largest class (a = b = 0)
      ConvLaunch L; memset(&L, 0, sizeof(L));
      ConvParams& P = L.P;
      { const char* e = getenv("MAPNET_TC_DEBUG"); P.debug = e ? atoi(e) : 0; }
      P.fmt_a = P.fmt_b = g.split ? 0 : 1; P.out32 = g.split;
      P.Nimg = g.B;
      pick_box(Ws0, Hs0, 128, &P.TW, &P.TH, &P.TN);
      P.tiles_w = cdiv(Ws0, P.TW); P.tiles_h = cdiv(Hs0, P.TH); P.tiles_n = cdiv(g.B, P.TN);
      P.n_tiles_m = P.tiles_w * P.tiles_h * P.tiles_n;
      int kbs[4];
      for (int i = 0; i < ncls; ++i) kbs[i] = ct[i].n * (SP * g.Co / 64);
      p->BN = choose_bn_classes(g.Ci, P.n_tiles_m, ncls, kbs);
      P.n_tiles_n = g.Ci / p->BN;
      P.cblocks = SP * g.Co / 64; P.Cs = SP * g.Co;
      P.Hout = g.Hi; P.Wout = g.Wi; P.Cout = g.Ci; P.os = s;
      P.n_classes = ncls;
      int nt = 0;
      for (int i = 0; i < ncls; ++i) {
        ClassDesc& c = P.cls[i];
        c.Hs = cdiv(g.Hi - ct[i].a, s); c.Ws = cdiv(g.Wi - ct[i].b, s); c.oa = ct[i].a; c.ob = ct[i].b;
        c.tap0 = nt; c.num_taps = ct[i].n;
        for (int k = 0; k < ct[i].n; ++k) P.taps[nt++] = ct[i].t[k];
      }
      L.n_maps = 1; L.pa[0] = L.pb[0] = 0;
      p->launches.push_back(L);
    } else {
      // one launch per class: size the tiles for one class
      p->BN = choose_bn(g.Ci, g.M_in() / (s * s), SP * ((KK + s * s - 1) / (s * s)) * (SP * g.Co / 64));
      for (int i = 0; i < ncls; ++i) {
        ConvLaunch L; memset(&L, 0, sizeof(L));
        ConvParams& P = L.P;
        P.fmt_a = P.fmt_b = g.split ? 0 : 1; P.out32 = g.split;
        P.Nimg = g.B;
        P.n_classes = 1;
        ClassDesc& c = P.cls[0];
        c.Hs = cdiv(g.Hi - ct[i].a, s); c.Ws = cdiv(g.Wi - ct[i].b, s); c.oa = ct[i].a; c.ob = ct[i].b;
        c.tap0 = 0; c.num_taps = ct[i].n;
        for (int k = 0; k < ct[i].n; ++k) P.taps[k] = ct[i].t[k];
        pick_box(c.Ws, c.Hs, 128, &P.TW, &P.TH, &P.TN);
        P.tiles_w = cdiv(c.Ws, P.TW); P.tiles_h = cdiv(c.Hs, P.TH); P.tiles_n = cdiv(g.B, P.TN);
        P.n_tiles_m = P.tiles_w * P.tiles_h * P.tiles_n; P.n_tiles_n = g.Ci / p->BN;
        P.cblocks = SP * g.Co / 64; P.Cs = SP * g.Co;
        P.Hout = g.Hi; P.Wout = g.Wi; P.Cout = g.Ci; P.os = s;
        L.n_maps = 1; L.pa[0] = L.pb[0] = 0;
        p->launches.push_back(L);
      }
    }
  } else {
    // ---------------- wgrad ----------------
    WgradParams& P = p->WP; memset(&P, 0, sizeof(P));
    { const char* e = getenv("MAPNET_TC_DEBUG"); P.debug = e ? atoi(e) : 0; }
    const int CoS = SP * g.Co, CiS = SP * g.Ci;      // GEMM N / M extents in 16-bit operand elements
    p->BN = (CoS % 128 == 0) ? 128 : 64;      // 64 x BN fp32 accumulator per consumer warpgroup in registers
    P.split = g.split; P.fmt_a = P.fmt_b = g.split ? 0 : 1;
    P.BN = p->BN; P.Nimg = g.B; P.Ho = g.Ho; P.Wo = g.Wo; P.Ci = g.Ci; P.Co = g.Co; P.KK = KK;
    pick_box(g.Wo, g.Ho, 64, &P.TW, &P.TH, &P.TN);
    P.tiles_w = cdiv(g.Wo, P.TW); P.tiles_h = cdiv(g.Ho, P.TH); P.tiles_n = cdiv(g.B, P.TN);
    P.n_pix_tiles = P.tiles_w * P.tiles_h * P.tiles_n;
    P.cpt = CiS / 64;
    P.n_chunks = KK * P.cpt;
    MN_CHECK(KK <= 16, "tc wgrad: too many filter taps");
    P.n_mtiles = cdiv(P.n_chunks, 2); P.n_ntiles = CoS / p->BN;
    p->w_nmaps = 0;
    for (int kh = 0; kh < g.KH; ++kh)
      for (int kw = 0; kw < g.KW; ++kw) {
        WgradTap& c = P.taps[kh * g.KW + kw];
        if (s == 1) { c.dh = kh - pad; c.dw = kw - pad; c.map = 0; p->wpa[0] = p->wpb[0] = 0; if (p->w_nmaps < 1) p->w_nmaps = 1; }
        else {
          const int a = posmod(kh - pad, 2), b = posmod(kw - pad, 2);
          c.dh = floordiv(kh - pad, 2); c.dw = floordiv(kw - pad, 2);
          int mi = -1;
          for (int i = 0; i < p->w_nmaps; ++i) if (p->wpa[i] == a && p->wpb[i] == b) mi = i;
          if (mi < 0) { mi = p->w_nmaps++; p->wpa[mi] = a; p->wpb[mi] = b; }
          c.map = mi;
        }
      }
    const int units = P.n_mtiles * P.n_ntiles;
    int splits = (kNumSMs * 2) / units; if (splits < 1) splits = 1;
    if (splits > P.n_pix_tiles) splits = P.n_pix_tiles;
    P.tiles_per_split = cdiv(P.n_pix_tiles, splits);
    P.splits = cdiv(P.n_pix_tiles, P.tiles_per_split);
    // the engine with the lowest modelled cost; the per-tap engine unless a halo engine is strictly cheaper
    static const int kHalo[3][2] = {{3, 64}, {3, 128}, {9, 64}};
    int taps = 0, bn = p->BN;
    double best = wgrad_cost(P, 0, p->BN);
    for (const auto& v : kHalo) {
      if (!wgrad_halo_allowed(g, P, v[0], v[1])) continue;
      const double c = wgrad_cost(P, v[0], v[1]);
      if (c < best) { best = c; taps = v[0]; bn = v[1]; }
    }
    wgrad_use_engine(p, taps, bn);
  }
  *out = p;
  return 0;
}

void tc_plan_destroy(TcConvPlan* p) {
  if (p != nullptr && p->ws != nullptr) cudaFree(p->ws);
  delete p;
}
void tc_plan_set_out_scale(TcConvPlan* p, const float* inv_scale) { if (p != nullptr) p->out_scale = inv_scale; }

int tc_plan_force_wgrad(TcConvPlan* p, int taps, int bn) {
  MN_CHECK(p != nullptr && p->kind == 2, "tc_plan_force_wgrad: not a wgrad plan");
  MN_CHECK(taps == 0 || wgrad_halo_allowed(p->g, p->WP, taps, bn),
           "tc_plan_force_wgrad: no halo engine with %d taps at BN %d for this conv", taps, bn);
  wgrad_use_engine(p, taps, bn);
  return 0;
}

// Fold the dgrad of the block's 1x1 / stride-2 downsample conv into the (merged) dgrad of its 3x3 / stride-2 conv1:
// both produce d(block input), the shortcut only reaches the pixel class (0, 0), where it is one more filter tap
// that reads the OTHER incoming gradient (tc_conv_run's in1, shaped like in0) against the shortcut's own weight
// matrix wmat2 = [Ci][Co].  Replaces 4 launches, a zero-filled full-size tensor and its re-read as a residual.
int tc_plan_add_shortcut(TcConvPlan* p, const bf16* wmat2) {
  MN_CHECK(p != nullptr && wmat2 != nullptr, "tc_plan_add_shortcut: null argument");
  MN_CHECK(p->kind == 1 && !p->g.split && p->g.stride == 2 && p->g.KH == 3 && p->launches.size() == 1,
           "tc_plan_add_shortcut: needs a merged 3x3 stride-2 dgrad plan (bf16 mode)");
  ConvParams& P = p->launches[0].P;
  ClassDesc& c = P.cls[P.n_classes - 1];
  MN_CHECK(c.oa == 0 && c.ob == 0 && c.tap0 + c.num_taps == 9 && p->wmat2 == nullptr,
           "tc_plan_add_shortcut: unexpected class layout");
  TapDesc& t = P.taps[9];
  t.dh = 0; t.dw = 0; t.map = 1 | 4; t.kidx = 0;        // activation map 1 (= in1), second weight matrix
  c.num_taps += 1;
  p->wmat2 = wmat2;
  p->shortcut_flops_k = p->g.Co;
  p->c_in0 = p->c_in1 = nullptr;
  return 0;
}
// Host-only description of a plan as JSON (tests/test_tc_plan.py emulates it on the CPU: the tap / parity-class /
// tile arithmetic is host logic and is checked without a GPU against torch's convolutions).
int tc_plan_describe(const TcConvPlan* p, char* buf, int cap) {
  MN_CHECK(p != nullptr && buf != nullptr && cap > 0, "tc_plan_describe: bad argument");
  int n = 0;
  bool ovf = false;
  auto put = [&](const char* fmt, ...) {
    if (ovf) return;
    va_list ap;
    va_start(ap, fmt);
    const int w = vsnprintf(buf + n, (size_t)(cap - n), fmt, ap);
    va_end(ap);
    if (w < 0 || w >= cap - n) ovf = true; else n += w;
  };
  put("{\"kind\":%d,\"BN\":%d,\"shortcut\":%d,\"f8_kb\":%d", p->kind, p->BN, p->wmat2 != nullptr ? 1 : 0, p->f8_kb);
  if (p->kind == 2) {
    const WgradParams& P = p->WP;
    put(",\"wgrad\":{\"TW\":%d,\"TH\":%d,\"TN\":%d,\"tiles_w\":%d,\"tiles_h\":%d,\"tiles_n\":%d,\"n_pix_tiles\":%d,"
        "\"n_chunks\":%d,\"n_mtiles\":%d,\"n_ntiles\":%d,\"BN\":%d,\"splits\":%d,\"tiles_per_split\":%d,\"Ci\":%d,\"Co\":%d,"
        "\"KK\":%d,\"maps\":[",
        P.TW, P.TH, P.TN, P.tiles_w, P.tiles_h, P.tiles_n, P.n_pix_tiles, P.n_chunks, P.n_mtiles, P.n_ntiles, P.BN,
        P.splits, P.tiles_per_split, P.Ci, P.Co, P.KK);
    for (int i = 0; i < p->w_nmaps; ++i) put("%s[%d,%d]", i ? "," : "", p->wpa[i], p->wpb[i]);
    put("],\"chunks\":[");
    for (int i = 0; i < P.n_chunks; ++i) {
      const int tap = i / P.cpt, c0 = (i - tap * P.cpt) * 64;
      put("%s[%d,%d,%d,%d,%d]", i ? "," : "", P.taps[tap].dh, P.taps[tap].dw, P.taps[tap].map, c0, tap);
    }
    // the engine that runs it: taps 0 = k_tc_wgrad (BN above), 3 / 9 = k_halo_wgrad
    const int bn = P.halo_taps ? P.halo_bn : P.BN;
    put("],\"engine\":{\"taps\":%d,\"BN\":%d,\"units\":%d,\"grid\":%d,\"RW\":%d,\"HR\":%d,\"halo_bytes\":%d,"
        "\"sbo\":%d,\"step_row\":[%d,%d,%d,%d]}}",
        P.halo_taps, bn, wgrad_units(P, P.halo_taps, bn), wgrad_units(P, P.halo_taps, bn) * P.splits,
        P.halo_taps ? P.RW : 0, P.halo_taps ? P.HR : 0, P.halo_taps ? P.halo_bytes : 0, P.halo_taps ? P.halo_sbo : 0,
        P.step_row[0], P.step_row[1], P.step_row[2], P.step_row[3]);
  } else {
    put(",\"launches\":[");
    for (size_t li = 0; li < p->launches.size(); ++li) {
      const ConvLaunch& L = p->launches[li];
      const ConvParams& P = L.P;
      put("%s{\"TW\":%d,\"TH\":%d,\"TN\":%d,\"tiles_w\":%d,\"tiles_h\":%d,\"tiles_n\":%d,\"n_tiles_m\":%d,\"n_tiles_n\":%d,"
          "\"cblocks\":%d,\"Cs\":%d,\"Hout\":%d,\"Wout\":%d,\"Cout\":%d,\"os\":%d,\"Nimg\":%d,\"maps\":[",
          li ? "," : "", P.TW, P.TH, P.TN, P.tiles_w, P.tiles_h, P.tiles_n, P.n_tiles_m, P.n_tiles_n, P.cblocks, P.Cs,
          P.Hout, P.Wout, P.Cout, P.os, P.Nimg);
      for (int i = 0; i < L.n_maps; ++i) put("%s[%d,%d]", i ? "," : "", L.pa[i], L.pb[i]);
      put("],\"classes\":[");
      for (int c = 0; c < P.n_classes; ++c) {
        const ClassDesc& cd = P.cls[c];
        put("%s{\"Hs\":%d,\"Ws\":%d,\"oa\":%d,\"ob\":%d,\"taps\":[", c ? "," : "", cd.Hs, cd.Ws, cd.oa, cd.ob);
        for (int t = cd.tap0; t < cd.tap0 + cd.num_taps; ++t)
          put("%s[%d,%d,%d,%d]", t > cd.tap0 ? "," : "", P.taps[t].dh, P.taps[t].dw, P.taps[t].map, P.taps[t].kidx);
        put("]}");
      }
      put("]}");
    }
    put("]");
  }
  put("}");
  MN_CHECK(!ovf, "tc_plan_describe: buffer of %d bytes is too small", cap);
  return 0;
}

int tc_plan_launches(const TcConvPlan* p) { return p->kind == 2 ? 1 : (int)p->launches.size(); }

template <typename K>
static int set_smem(K kernel, size_t bytes) {
  MN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}

// activation map (optionally a stride-2 parity view) over [N, Hd, Wd, C]
static int encode_view(CUtensorMap* m, const bf16* base, int N, int Hd, int Wd, int C, int s, int a, int b, int bw,
                       int bh, int bn, const ConvGeom* gv = nullptr) {
  if (gv != nullptr && gv->in_pix_stride != 0)      // explicit (possibly overlapping) strides, stride-1 only
    return encode_act_map(m, base, C, Wd, Hd, N, gv->in_pix_stride, gv->in_row_stride, gv->in_img_stride, bw, bh, bn);
  const long long rowb = (long long)Wd * C * 2, imgb = (long long)Hd * rowb;
  if (s == 1) return encode_act_map(m, base, C, Wd, Hd, N, (long long)C * 2, rowb, imgb, bw, bh, bn);
  const int Hq = cdiv(Hd - a, 2), Wq = cdiv(Wd - b, 2);
  const bf16* vb = base + ((long long)a * Wd + b) * C;
  return encode_act_map(m, vb, C, Wq > 0 ? Wq : 1, Hq > 0 ? Hq : 1, N, (long long)C * 4, rowb * 2, imgb, bw, bh, bn);
}

// fp8 fprop plan: the bf16 fprop plan's tiles and taps with e4m3 k-blocks (128 channels, or 64 when Ci = 64)
int tc_plan_create_f8(TcConvPlan** out, const ConvGeom& g, const uint8_t* wmat) {
  *out = nullptr;
  MN_CHECK(!g.split && g.in_pix_stride == 0 && g.KH == g.KW && (g.KH == 1 || g.KH == 3),
           "tc fp8 conv: dense 1x1 / 3x3 convs only");
  MN_CHECK(g.Ci % 64 == 0 && (g.Ci == 64 || g.Ci % 128 == 0), "tc fp8 conv: Ci must be 64 or a multiple of 128 (got %d)", g.Ci);
  MN_TRY(tc_plan_create(out, g, 0, (const bf16*)wmat));
  TcConvPlan* p = *out;
  ConvParams& P = p->launches[0].P;
  p->f8_kb = (g.Ci % 128 == 0) ? 128 : 64;
  P.cblocks = g.Ci / p->f8_kb;
  P.Cs = g.Ci;
  P.fmt_a = P.fmt_b = 2;
  p->BN = choose_bn(g.Co, g.M_out(), g.KH * g.KW * P.cblocks);
  P.n_tiles_n = g.Co / p->BN;
  return 0;
}

int tc_conv_run_f8(TcConvPlan* p, const uint8_t* in, const void* residual, void* out, const EpiF8& e, cudaStream_t st) {
  MN_CHECK(p != nullptr && p->f8_kb != 0, "tc_conv_run_f8: not an fp8 plan");
  MN_CHECK(e.scale != nullptr && e.shift != nullptr, "tc_conv_run_f8: null scale / shift table");
  const bool res = residual != nullptr;
  int mode = EPI_AFFINE | (res ? EPI_RES : 0) | (e.relu ? EPI_RELU : 0) | ((res && e.res_f8) ? EPI_F8RES : 0);
  mode |= e.amax != nullptr ? EPI_AMAX : (e.out_f8 ? EPI_F8OUT : 0);
  static const int built[] = {
      EPI_AFFINE | EPI_RELU | EPI_F8OUT, EPI_AFFINE, EPI_AFFINE | EPI_RES | EPI_RELU | EPI_F8OUT,
      EPI_AFFINE | EPI_RES | EPI_F8RES | EPI_RELU | EPI_F8OUT, EPI_AFFINE | EPI_RELU | EPI_AMAX,
      EPI_AFFINE | EPI_RES | EPI_RELU | EPI_AMAX, EPI_AFFINE | EPI_RES | EPI_F8RES | EPI_RELU | EPI_AMAX};
  bool ok = false;
  for (int b : built) ok = ok || b == mode;
  MN_CHECK(ok, "tc_conv_run_f8: epilogue variant not built (residual %d relu %d res_f8 %d out_f8 %d amax %d)", res, e.relu,
           e.res_f8, e.out_f8, e.amax != nullptr);
  MN_CHECK(!(mode & EPI_F8RES) || e.res_scale != nullptr, "tc_conv_run_f8: an e4m3 residual needs its scale");
  MN_CHECK(!(mode & EPI_F8OUT) || e.out_inv != nullptr, "tc_conv_run_f8: an e4m3 output needs 1 / its scale");
  MN_CHECK(out != nullptr || (mode & EPI_AMAX), "tc_conv_run_f8: null output");
  const ConvGeom& g = p->g;
  ConvLaunch& L = p->launches[0];
  const int kb = p->f8_kb;
  const CUtensorMapSwizzle swz = kb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  if (p->c_in0 != in) {
    const long long rowb = (long long)g.Wi * g.Ci, imgb = (long long)g.Hi * rowb;
    for (int i = 0; i < L.n_maps; ++i) {
      if (g.stride == 1) {
        MN_TRY(encode_act_map(&L.mapA[i], in, g.Ci, g.Wi, g.Hi, g.B, g.Ci, rowb, imgb, L.P.TW, L.P.TH, L.P.TN,
                              CU_TENSOR_MAP_DATA_TYPE_UINT8, kb, swz));
      } else {       // stride-2 parity view (a, b), as encode_view builds it for bf16
        const int a = L.pa[i], b = L.pb[i];
        const int Hq = cdiv(g.Hi - a, 2), Wq = cdiv(g.Wi - b, 2);
        MN_TRY(encode_act_map(&L.mapA[i], in + ((long long)a * g.Wi + b) * g.Ci, g.Ci, Wq > 0 ? Wq : 1, Hq > 0 ? Hq : 1,
                              g.B, 2LL * g.Ci, 2 * rowb, imgb, L.P.TW, L.P.TH, L.P.TN, CU_TENSOR_MAP_DATA_TYPE_UINT8, kb, swz));
      }
    }
    for (int i = L.n_maps; i < 4; ++i) L.mapA[i] = L.mapA[0];
    MN_TRY(encode_w_map(&L.mapB, p->wmat, g.KH * g.KW * g.Ci, g.Co, p->BN, CU_TENSOR_MAP_DATA_TYPE_UINT8, kb, swz));
    p->c_in0 = in;
  }
  EpiF8Dev E; memset(&E, 0, sizeof(E));
  E.ascale = e.scale; E.ashift = e.shift; E.aflags = mode;
  E.res_scale = e.res_scale; E.out_inv = e.out_inv; E.amax = e.amax;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, ConvParams, const void*, void*, EpiF8Dev) =
      (kb == 128) ? ((p->BN == 64) ? k_f8_conv<64, 128> : k_f8_conv<128, 128>)
                  : ((p->BN == 64) ? k_f8_conv<64, 64> : k_f8_conv<128, 64>);
  const size_t smem = (kb == 128) ? f8_smem_bytes(p->BN, 128) : f8_smem_bytes(p->BN, 64);
  if (!p->smem_attr_set) {
    MN_TRY(set_smem(kern, smem));
    p->smem_attr_set = true;
  }
  const int items = L.P.n_tiles_m * L.P.n_tiles_n;
  MN_LAUNCH(kern, items < kNumSMs ? items : kNumSMs, kConvThreads, smem, st, L.mapA[0], L.mapA[1], L.mapA[2], L.mapA[3],
            L.mapB, L.P, residual, out, E);
  MN_LAUNCH_CHECK();
  return 0;
}

int tc_conv_run(TcConvPlan* p, const bf16* in0, const bf16* in1, const bf16* residual, void* out, cudaStream_t st,
                double* stats, const EpiBwd* bwd, const EpiAffine* aff) {
  MN_CHECK(p != nullptr, "tc_conv_run: null plan");
  if (aff != nullptr) {
    MN_CHECK(p->kind == 0 && stats == nullptr && bwd == nullptr,
             "tc_conv_run: the affine (inference) epilogue is an fprop epilogue without statistics");
    MN_CHECK(tc_affine_supported(p->g.split != 0, residual != nullptr, *aff),
             "tc_conv_run: affine epilogue variant not built (split %d residual %d relu %d res_split %d out_split %d)",
             p->g.split, residual != nullptr, aff->relu, aff->res_split, aff->out_split);
  }
  EpiBwd E; memset(&E, 0, sizeof(E));
  if (bwd != nullptr) {
    MN_CHECK(p->kind == 1 && stats != nullptr && bwd->y != nullptr, "tc_conv_run: backward statistics need a dgrad plan, accumulators and Y");
    MN_CHECK(bwd->zmask != nullptr || (bwd->mscale != nullptr && bwd->mshift != nullptr), "tc_conv_run: backward statistics need a gate (zmask or mscale/mshift)");
    MN_CHECK(bwd->yd == nullptr || bwd->zmask != nullptr, "tc_conv_run: the downsample sum is only built for zmask-gated gradients");
    E = *bwd;
  } else {
    MN_CHECK(stats == nullptr || residual == nullptr, "tc_conv_run: fprop statistics with a fused residual are not built");
  }
  MN_CHECK(!p->g.split || bwd == nullptr, "tc_conv_run: the fused BatchNorm-backward epilogue is a bf16-mode feature");
  E.oscale = p->out_scale;
  if (aff != nullptr) {
    E.ascale = aff->scale; E.ashift = aff->shift;
    E.aflags = affine_mode(p->g.split != 0, residual != nullptr, aff->relu, aff->res_split, aff->out_split) &
               (EPI_RELU | EPI_HOUT | EPI_HRES);
  }
  const ConvGeom& g = p->g;
  const int SP = g.split ? 2 : 1;
  const int nsm = kNumSMs;
  if (p->kind == 0 || p->kind == 1) {
    MN_CHECK(p->wmat2 == nullptr || in1 != nullptr, "tc_conv_run: a dgrad plan with a folded shortcut needs the shortcut's gradient as in1");
    if (p->c_in0 != in0 || (p->wmat2 != nullptr && p->c_in1 != in1)) {
      for (auto& L : p->launches) {
        if (p->kind == 0) {
          for (int i = 0; i < L.n_maps; ++i)
            MN_TRY(encode_view(&L.mapA[i], in0, g.B, g.Hi, g.Wi, SP * g.Ci, g.stride, L.pa[i], L.pb[i], L.P.TW, L.P.TH, L.P.TN, &g));
          MN_TRY(encode_w_map(&L.mapB, p->wmat, SP * g.KH * g.KW * SP * g.Ci, g.Co, p->BN));
        } else {
          MN_TRY(encode_view(&L.mapA[0], in0, g.B, g.Ho, g.Wo, SP * g.Co, 1, 0, 0, L.P.TW, L.P.TH, L.P.TN));
          MN_TRY(encode_w_map(&L.mapB, p->wmat, SP * g.KH * g.KW * SP * g.Co, g.Ci, p->BN));
          if (p->wmat2 != nullptr) {
            MN_TRY(encode_view(&L.mapA[1], in1, g.B, g.Ho, g.Wo, g.Co, 1, 0, 0, L.P.TW, L.P.TH, L.P.TN));
            MN_TRY(encode_w_map(&L.mapB2, p->wmat2, g.Co, g.Ci, p->BN));
            L.n_maps = 2;
          }
        }
        for (int i = L.n_maps; i < 4; ++i) L.mapA[i] = L.mapA[0];
        if (p->wmat2 == nullptr) L.mapB2 = L.mapB;
      }
      p->c_in0 = in0; p->c_in1 = in1;
    }
    const size_t smem = conv_smem_bytes(p->BN);
    void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, ConvParams, const bf16*, bf16*, double*, EpiBwd) =
        (aff != nullptr) ? ((p->BN == 64) ? k_tc_conv<64, true> : k_tc_conv<128, true>)
                         : ((p->BN == 64) ? k_tc_conv<64> : k_tc_conv<128>);
    if (!p->smem_attr_set || p->smem_attr_aff != (aff != nullptr)) {
      MN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      p->smem_attr_set = true;
      p->smem_attr_aff = (aff != nullptr);
    }
    for (auto& L : p->launches) {
      const int items = L.P.n_tiles_m * L.P.n_tiles_n * L.P.n_classes;     // persistent CTAs: at most one per SM
      MN_LAUNCH(kern, items < nsm ? items : nsm, kConvThreads, smem, st, L.mapA[0], L.mapA[1], L.mapA[2], L.mapA[3], L.mapB,
                L.mapB2, L.P, residual, (bf16*)out, stats, E);
      MN_LAUNCH_CHECK();
    }
    return 0;
  }
  // wgrad: in0 = x [B,Hi,Wi,Ci], in1 = dy [B,Ho,Wo,Co]
  WgradParams& P = p->WP;
  P.oscale = p->out_scale;
  if (p->c_in0 != in0 || p->c_in1 != in1) {
    if (P.halo_taps) {       // the halo box: RW x HR pixels per image
      MN_TRY(encode_view(&p->mapX[0], in0, g.B, g.Hi, g.Wi, g.Ci, 1, 0, 0, P.RW, P.HR, P.TN));
    } else {
      for (int i = 0; i < p->w_nmaps; ++i)
        MN_TRY(encode_view(&p->mapX[i], in0, g.B, g.Hi, g.Wi, SP * g.Ci, g.stride, p->wpa[i], p->wpb[i], P.TW, P.TH, P.TN, &g));
    }
    for (int i = p->w_nmaps; i < 4; ++i) p->mapX[i] = p->mapX[0];
    MN_TRY(encode_view(&p->mapDY, in1, g.B, g.Ho, g.Wo, SP * g.Co, 1, 0, 0, P.TW, P.TH, P.TN));
    p->c_in0 = in0; p->c_in1 = in1;
  }
  void (*k1)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, WgradParams, float*) =
      (p->BN == 64) ? k_tc_wgrad<64> : k_tc_wgrad<128>;
  void (*kh)(CUtensorMap, CUtensorMap, WgradParams, float*) =
      P.halo_taps == 9 ? k_halo_wgrad<64, 3> : P.halo_bn == 64 ? k_halo_wgrad<64, 1> : k_halo_wgrad<128, 1>;
  const size_t smem = !P.halo_taps ? (size_t)wgrad_stages(p->BN) * (2 * 8192 + (p->BN / 64) * 8192) + 1024
                      : P.halo_taps == 9 ? halo_smem_bytes(64, 3) : P.halo_bn == 64 ? halo_smem_bytes(64, 1)
                                                                                    : halo_smem_bytes(128, 1);
  if (!p->smem_attr_set) {
    if (P.halo_taps) MN_TRY(set_smem(kh, smem));
    else MN_TRY(set_smem(k1, smem));
    p->smem_attr_set = true;
  }
  const int grid = wgrad_units(P, P.halo_taps, P.halo_taps ? P.halo_bn : p->BN) * P.splits;
  P.part_stride = (long long)g.Co * P.KK * g.Ci;
  P.partial = nullptr;
  if (P.splits > 1) {
    // split-K partial sums go through a workspace and a fixed-order reduction instead of float atomics, so that the
    // gradient is bit-identical from run to run.  Allocated at the first (eager) run, before any graph capture.
    if (p->ws == nullptr) MN_CUDA(cudaMalloc(&p->ws, (size_t)P.splits * P.part_stride * sizeof(float)));
    P.partial = p->ws;
  }
  if (P.halo_taps)
    MN_LAUNCH(kh, grid, (P.halo_taps / 3) * 128 + 32, smem, st, p->mapX[0], p->mapDY, P, (float*)out);
  else
    MN_LAUNCH(k1, grid, kConvThreads, smem, st, p->mapX[0], p->mapX[1], p->mapX[2], p->mapX[3], p->mapDY, P, (float*)out);
  MN_LAUNCH_CHECK();
  if (P.splits > 1) {
    MN_TRY(launch_split_reduce(p->ws, P.splits, P.part_stride, (float*)out, st));
  }
  return 0;
}

int launch_split_reduce(const float* part, int splits, long long n, float* dst, cudaStream_t st) {
  MN_CHECK(n % 4 == 0, "split reduce: %lld elements, not a multiple of 4", n);
  MN_CHECK((((uintptr_t)part | (uintptr_t)dst) & 15) == 0, "split reduce: workspace / destination not 16-byte aligned");
  const long long n4 = n / 4;
  const long long grid = (n4 + 255) / 256 < kNumSMs * 8LL ? (n4 + 255) / 256 : kNumSMs * 8LL;
  MN_LAUNCH(k_wgrad_reduce, (int)(grid > 0 ? grid : 1), 256, 0, st, (const float4*)part, n4, splits, n4, (float4*)dst);
  MN_LAUNCH_CHECK();
  return 0;
}

}  // namespace mapnet
