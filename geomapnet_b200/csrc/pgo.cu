// Batched pose-graph optimisation (SURVEY.md section 8 row f3): one thread block per window.
//
// Replaces, for a whole batch of windows at once, /root/reference/common/pose_utils.py:458-804 -- PoseGraph /
// PoseGraphFC.optimize and optimize_poses -- which scripts/eval.py:172-178 calls once per frame on the N poses a
// MapNet tuple predicts, each call a dense numpy Gauss-Newton: stack the Jacobian J of every constraint, H = J'J,
// b = J'r, Cholesky-solve H x = -b, update on the manifold; 10 iterations.
//
// Same state and constraints (file:line in the reference):
//   state z_i = (t_i, q_i), q = (w, x, y, z) not renormalised; increments x_i = (dt, dqm), q <- q * (cos|dqm|, sinc(|dqm|/pi) dqm)
//                                                                                         (update_on_manifold :552-575)
//   unary     (:473-483, :516-523)  r = L_a (z_i - pose_i),   J_t = I,  J_q = m_rot(q_i)              (m_rot :444-456)
//   pairwise  (:486-505, :526-549)  r_t = R(q_i)^-1 (t_j - t_i) - vo_t,  J = (-dqstq_t(q_i), +dqstq_t(q_i)) w.r.t. (t_i, t_j)
//                                   r_q = q_i^-1 * q_j - vo_q,           J = (dpsq_p(q_j) m_rot(q_i), dpsq_q(q_i) m_rot(q_j))
//                                   (the rotation derivative of r_t is commented out in the reference and absent here)
//   edges: consecutive poses (PoseGraph) or every pair i < j in row-major order (PoseGraphFC :648-703)
//   weights: L = chol(I / s)' = I / sqrt(s) for each of sax, saq, srx, srq (:593-597)
//   linear solve (:605-608): R = cholesky(H) (upper); y = solve_triangular(R.T, -b) -- called with scipy's default
//   lower=False, so LAPACK reads only the upper triangle of R' (its diagonal): y = -b / diag(R); x = solve_triangular(R, y).
//   The reference's step is therefore R^-1 diag(R)^-1 (-b), NOT H^-1 (-b); reproduced literally (flags bit 0 = 0) because
//   that is what scripts/eval.py computes; flags bit 0 = 1 does the forward substitution (the Gauss-Newton step).
// H and b are accumulated constraint by constraint (J is never materialised); transforms3d's qmult / qinverse /
// rotate_vector (third party, `transforms3d` in environment.yml:19, not vendored) are restated from its published
// source: Hamilton product, conj(q) / (q.q), and q * (0, v) * conj(q).  fp64 throughout, as numpy computes.
// Latency-bound small dense algebra: 6N <= 96 unknowns per window, H (<= 73.7 KB) lives in shared memory.
#include <math.h>

#include "kernels.h"
#include "pose_post.cuh"
#include "track_core.h"
#include "../../include/mapnet_b200.h"

namespace mapnet {

static constexpr int kPgoMaxN = 16;
static constexpr int kPgoThreads = 128;

struct Q4 { double w, x, y, z; };
__device__ __forceinline__ Q4 q_mul(const Q4& a, const Q4& b) {
  return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}
__device__ __forceinline__ Q4 q_conj(const Q4& a) { return {a.w, -a.x, -a.y, -a.z}; }
__device__ __forceinline__ Q4 q_inv(const Q4& a) {           // transforms3d.quaternions.qinverse
  const double n = a.w * a.w + a.x * a.x + a.y * a.y + a.z * a.z;
  return {a.w / n, -a.x / n, -a.y / n, -a.z / n};
}
// transforms3d.quaternions.rotate_vector(v, q) = (q * (0, v) * conj(q))[1:]
__device__ __forceinline__ void q_rotate(const double v[3], const Q4& q, double out[3]) {
  const Q4 r = q_mul(q, q_mul(Q4{0.0, v[0], v[1], v[2]}, q_conj(q)));
  out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
// columns 1..3 of dpq_q(p) (:385-396): m_rot(p), 4 x 3
__device__ __forceinline__ void m_rot(const Q4& p, double M[4][3]) {
  M[0][0] = -p.x; M[0][1] = -p.y; M[0][2] = -p.z;
  M[1][0] = p.w;  M[1][1] = -p.z; M[1][2] = p.y;
  M[2][0] = p.z;  M[2][1] = p.w;  M[2][2] = -p.x;
  M[3][0] = -p.y; M[3][1] = p.x;  M[3][2] = p.w;
}
// dpsq_q(p) (:398-409) and dpsq_p(q) (:411-422), 4 x 4
__device__ __forceinline__ void dpsq_q(const Q4& p, double J[4][4]) {
  J[0][0] = p.w;  J[0][1] = -p.x; J[0][2] = -p.y; J[0][3] = -p.z;
  J[1][0] = -p.x; J[1][1] = p.w;  J[1][2] = p.z;  J[1][3] = -p.y;
  J[2][0] = -p.y; J[2][1] = -p.z; J[2][2] = p.w;  J[2][3] = p.x;
  J[3][0] = -p.z; J[3][1] = p.y;  J[3][2] = -p.x; J[3][3] = p.w;
}
__device__ __forceinline__ void dpsq_p(const Q4& q, double J[4][4]) {
  J[0][0] = q.w; J[0][1] = q.x;  J[0][2] = q.y;  J[0][3] = q.z;
  J[1][0] = q.x; J[1][1] = -q.w; J[1][2] = -q.z; J[1][3] = q.y;
  J[2][0] = q.y; J[2][1] = q.z;  J[2][2] = -q.w; J[2][3] = -q.x;
  J[3][0] = q.z; J[3][1] = -q.y; J[3][2] = q.x;  J[3][3] = -q.w;
}
// dqstq_t(q) (:434-442): (w^2 - v.v) I + 2 v v' - 2 w skew(v)
__device__ __forceinline__ void dqstq_t(const Q4& q, double D[3][3]) {
  const double v[3] = {q.x, q.y, q.z};
  const double c = q.w * q.w - (q.x * q.x + q.y * q.y + q.z * q.z);
  const double S[3][3] = {{0.0, -q.z, q.y}, {q.z, 0.0, -q.x}, {-q.y, q.x, 0.0}};
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) D[a][b] = (a == b ? c : 0.0) + 2.0 * v[a] * v[b] - 2.0 * q.w * S[a][b];
}

// Cauchy weight of an absolute factor whose whitened residual is r [7]: omega = 1 / (1 + |r|^2 / c^2), the IRLS
// weight of rho(s) = c^2 log(1 + s / c^2) (rho'(s) = omega).  s / c^2 is summed as (r_k / c)^2, so a zero residual gives
// omega = 1 and an overflowing one omega = 0 for every finite c > 0, never 0 / 0.
__device__ __forceinline__ double cauchy_weight(const double r[7], double c) {
  double u = 0.0;
#pragma unroll
  for (int a = 0; a < 7; ++a) {
    const double e = r[a] / c;
    u += e * e;
  }
  return 1.0 / (1.0 + u);
}

// k_pgo's absolute factor of slot i at state z: its Cauchy weight at scale c (residual (w_ax (t - t0), w_aq (q - q0)))
__device__ __forceinline__ double pgo_point_weight(const double* z, const double* P, int i, double w_ax, double w_aq,
                                                   double c) {
  double r[7];
#pragma unroll
  for (int a = 0; a < 7; ++a) r[a] = (a < 3 ? w_ax : w_aq) * (z[7 * i + a] - P[7 * i + a]);
  return cauchy_weight(r, c);
}

// One window per block.  Constraints are dealt to threads; each thread accumulates into the shared H / b with
// double atomics (a few hundred constraints x <= 144 entries: contention is irrelevant next to the Cholesky).
// n_win_dev (may be null): the device count of windows to optimise; the blocks beyond it exit, so a captured graph can
// keep a fixed grid while the count changes from replay to replay.  win_fail (may be null): per window, 1 when its
// normal matrix was not positive definite, else 0, so a caller can tell which windows failed.
// kRobust: iteratively reweighted Gauss-Newton for the Cauchy loss on the absolute factors -- in every iteration the
// unary work item of slot i weighs its H and b contributions by omega_i = cauchy_weight at the iteration's starting
// state (scale c, whitened units); w_out (may be null) [W][N] gets omega at the returned state.  The step rule (exact)
// is unchanged.  Without kRobust, c and w_out are not read.
template <bool kRobust>
__global__ void __launch_bounds__(kPgoThreads)
k_pgo(const double* __restrict__ poses, const double* __restrict__ vos, double* __restrict__ out, int N, int fc,
      double w_ax, double w_aq, double w_rx, double w_rq, int n_iters, int exact, int* __restrict__ status,
      const int* __restrict__ n_win_dev, int* __restrict__ win_fail, double c, double* __restrict__ w_out) {
  pdl_prologue();
  if (n_win_dev != nullptr && (int)blockIdx.x >= *n_win_dev) return;
  extern __shared__ double sm[];
  const int D = 6 * N;
  double* H = sm;                 // D x D
  double* bv = H + D * D;         // D
  double* z = bv + D;             // 7 N
  double* xs = z + 7 * N;         // D
  const int W = blockIdx.x;
  const int E = fc ? N * (N - 1) / 2 : N - 1;
  const double* P = poses + (size_t)W * N * 7;
  const double* V = vos + (size_t)W * E * 7;
  for (int i = threadIdx.x; i < 7 * N; i += blockDim.x) z[i] = P[i];
  __shared__ int s_fail;
  if (threadIdx.x == 0) s_fail = 0;
  __syncthreads();
  for (int it = 0; it < n_iters; ++it) {
    for (int i = threadIdx.x; i < D * D + D; i += blockDim.x) H[i] = 0.0;
    __syncthreads();
    // ---- unary constraints + pairwise constraints: work items 0..N-1 unary, N..N+E-1 edges ----
    for (int f = threadIdx.x; f < N + E; f += blockDim.x) {
      if (f < N) {
        const int i = f;
        const Q4 q = {z[7 * i + 3], z[7 * i + 4], z[7 * i + 5], z[7 * i + 6]};
        double om = 1.0;                         // the slot's Cauchy weight (1: plain least squares)
        if constexpr (kRobust) om = pgo_point_weight(z, P, i, w_ax, w_aq, c);
        const double wx2 = kRobust ? om * (w_ax * w_ax) : w_ax * w_ax;
        // translation: J = w_ax I, r = w_ax (t - t0)
        for (int a = 0; a < 3; ++a) {
          atomicAdd(&H[(6 * i + a) * D + 6 * i + a], wx2);
          atomicAdd(&bv[6 * i + a], wx2 * (z[7 * i + a] - P[7 * i + a]));
        }
        double M[4][3], r[4];
        m_rot(q, M);
        for (int a = 0; a < 4; ++a) {
          r[a] = w_aq * (z[7 * i + 3 + a] - P[7 * i + 3 + a]);
          for (int b = 0; b < 3; ++b) M[a][b] *= w_aq;
        }
        for (int a = 0; a < 3; ++a) {
          for (int b = 0; b < 3; ++b) {
            double s = 0.0;
            for (int k = 0; k < 4; ++k) s += M[k][a] * M[k][b];
            atomicAdd(&H[(6 * i + 3 + a) * D + 6 * i + 3 + b], kRobust ? om * s : s);
          }
          double s = 0.0;
          for (int k = 0; k < 4; ++k) s += M[k][a] * r[k];
          atomicAdd(&bv[6 * i + 3 + a], kRobust ? om * s : s);
        }
      } else {
        int e = f - N, i, j;
        if (!fc) { i = e; j = e + 1; }
        else {                                   // row-major enumeration of the pairs i < j
          i = 0;
          int rem = e;
          while (rem >= N - 1 - i) { rem -= N - 1 - i; ++i; }
          j = i + 1 + rem;
        }
        const Q4 qi = {z[7 * i + 3], z[7 * i + 4], z[7 * i + 5], z[7 * i + 6]};
        const Q4 qj = {z[7 * j + 3], z[7 * j + 4], z[7 * j + 5], z[7 * j + 6]};
        // translation residual and Jacobian
        double Dt[3][3], rt[3];
        dqstq_t(qi, Dt);
        const double dv[3] = {z[7 * j] - z[7 * i], z[7 * j + 1] - z[7 * i + 1], z[7 * j + 2] - z[7 * i + 2]};
        q_rotate(dv, q_inv(qi), rt);
        for (int a = 0; a < 3; ++a) {
          rt[a] = w_rx * (rt[a] - V[7 * e + a]);
          for (int b = 0; b < 3; ++b) Dt[a][b] *= w_rx;
        }
        // J = [-Dt at t_i, +Dt at t_j]
        for (int a = 0; a < 3; ++a) {
          double g = 0.0;
          for (int k = 0; k < 3; ++k) g += Dt[k][a] * rt[k];
          atomicAdd(&bv[6 * i + a], -g);
          atomicAdd(&bv[6 * j + a], g);
          for (int b = 0; b < 3; ++b) {
            double s = 0.0;
            for (int k = 0; k < 3; ++k) s += Dt[k][a] * Dt[k][b];
            atomicAdd(&H[(6 * i + a) * D + 6 * i + b], s);
            atomicAdd(&H[(6 * j + a) * D + 6 * j + b], s);
            atomicAdd(&H[(6 * i + a) * D + 6 * j + b], -s);
            atomicAdd(&H[(6 * j + a) * D + 6 * i + b], -s);
          }
        }
        // rotation residual and Jacobian
        double A4[4][4], B4[4][4], Mi[4][3], Mj[4][3], Ja[4][3], Jb[4][3], rq[4];
        dpsq_p(qj, A4); dpsq_q(qi, B4); m_rot(qi, Mi); m_rot(qj, Mj);
        for (int a = 0; a < 4; ++a)
          for (int b = 0; b < 3; ++b) {
            double sa = 0.0, sb = 0.0;
            for (int k = 0; k < 4; ++k) { sa += A4[a][k] * Mi[k][b]; sb += B4[a][k] * Mj[k][b]; }
            Ja[a][b] = w_rq * sa; Jb[a][b] = w_rq * sb;
          }
        const Q4 qvo = q_mul(q_inv(qi), qj);
        rq[0] = w_rq * (qvo.w - V[7 * e + 3]); rq[1] = w_rq * (qvo.x - V[7 * e + 4]);
        rq[2] = w_rq * (qvo.y - V[7 * e + 5]); rq[3] = w_rq * (qvo.z - V[7 * e + 6]);
        for (int a = 0; a < 3; ++a) {
          double ga = 0.0, gb = 0.0;
          for (int k = 0; k < 4; ++k) { ga += Ja[k][a] * rq[k]; gb += Jb[k][a] * rq[k]; }
          atomicAdd(&bv[6 * i + 3 + a], ga);
          atomicAdd(&bv[6 * j + 3 + a], gb);
          for (int b = 0; b < 3; ++b) {
            double saa = 0.0, sbb = 0.0, sab = 0.0, sba = 0.0;
            for (int k = 0; k < 4; ++k) {
              saa += Ja[k][a] * Ja[k][b]; sbb += Jb[k][a] * Jb[k][b];
              sab += Ja[k][a] * Jb[k][b]; sba += Jb[k][a] * Ja[k][b];
            }
            atomicAdd(&H[(6 * i + 3 + a) * D + 6 * i + 3 + b], saa);
            atomicAdd(&H[(6 * j + 3 + a) * D + 6 * j + 3 + b], sbb);
            atomicAdd(&H[(6 * i + 3 + a) * D + 6 * j + 3 + b], sab);
            atomicAdd(&H[(6 * j + 3 + a) * D + 6 * i + 3 + b], sba);
          }
        }
      }
    }
    __syncthreads();
    // ---- Cholesky H = R' R (upper R stored in place, row-major), right-looking, one column per step ----
    for (int k = 0; k < D; ++k) {
      if (threadIdx.x == 0) {
        const double d = H[k * D + k];
        if (!(d > 0.0)) s_fail = 1;           // scipy.linalg.cholesky would raise LinAlgError here
        H[k * D + k] = sqrt(d > 0.0 ? d : 1.0);
      }
      __syncthreads();
      const double rkk = H[k * D + k];
      for (int j = k + 1 + threadIdx.x; j < D; j += blockDim.x) H[k * D + j] /= rkk;
      __syncthreads();
      for (int idx = threadIdx.x; idx < (D - k - 1) * (D - k - 1); idx += blockDim.x) {
        const int i = k + 1 + idx / (D - k - 1), j = k + 1 + idx % (D - k - 1);
        if (j >= i) H[i * D + j] -= H[k * D + i] * H[k * D + j];
      }
      __syncthreads();
    }
    // ---- y = -b / diag(R) (reference, see header) or R' y = -b (exact); then R x = y (thread 0: D <= 96) ----
    if (threadIdx.x == 0) {
      for (int i = 0; i < D; ++i) {
        double s = -bv[i];
        if (exact) for (int k = 0; k < i; ++k) s -= H[k * D + i] * xs[k];
        xs[i] = s / H[i * D + i];
      }
      for (int i = D - 1; i >= 0; --i) {
        double s = xs[i];
        for (int k = i + 1; k < D; ++k) s -= H[i * D + k] * xs[k];
        xs[i] = s / H[i * D + i];
      }
    }
    __syncthreads();
    // ---- update on the manifold ----
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      z[7 * i] += xs[6 * i]; z[7 * i + 1] += xs[6 * i + 1]; z[7 * i + 2] += xs[6 * i + 2];
      const double mx = xs[6 * i + 3], my = xs[6 * i + 4], mz = xs[6 * i + 5];
      const double n = sqrt(mx * mx + my * my + mz * mz);
      const double sc = (n == 0.0) ? 1.0 : sin(n) / n;          // np.sinc(n / pi)
      const Q4 dq = {cos(n), sc * mx, sc * my, sc * mz};
      const Q4 q = q_mul(Q4{z[7 * i + 3], z[7 * i + 4], z[7 * i + 5], z[7 * i + 6]}, dq);
      z[7 * i + 3] = q.w; z[7 * i + 4] = q.x; z[7 * i + 5] = q.y; z[7 * i + 6] = q.z;
    }
    __syncthreads();
  }
  double* O = out + (size_t)W * N * 7;
  for (int i = threadIdx.x; i < 7 * N; i += blockDim.x) O[i] = z[i];
  if constexpr (kRobust) {
    if (w_out != nullptr)
      for (int i = threadIdx.x; i < N; i += blockDim.x) w_out[(size_t)W * N + i] = pgo_point_weight(z, P, i, w_ax, w_aq, c);
  }
  if (threadIdx.x == 0 && s_fail && status != nullptr) atomicExch(status, 1);
  if (threadIdx.x == 0 && win_fail != nullptr) win_fail[W] = s_fail;
}

int pgo_prepare() {
  static bool attr = false;
  if (!attr) {
    const int smem = (int)(96 * 96 + 96 * 2 + 7 * 16) * 8;
    MN_CUDA(cudaFuncSetAttribute(k_pgo<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    MN_CUDA(cudaFuncSetAttribute(k_pgo<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = true;
  }
  return 0;
}

int launch_pgo(const double* poses, const double* vos, double* out, int n_windows, int N, int fc, const double w4[4],
               int n_iters, int exact, int* status, const int* n_win_dev, cudaStream_t st, int* win_fail,
               double robust_c, double* w_out) {
  MN_TRY(pgo_prepare());
  const int D = 6 * N;
  const size_t smem = (size_t)(D * D + D + 7 * N + D) * sizeof(double);
  if (robust_c > 0.0) {
    MN_LAUNCH(k_pgo<true>, n_windows, kPgoThreads, smem, st, poses, vos, out, N, fc, w4[0], w4[1], w4[2], w4[3],
              n_iters, exact, status, n_win_dev, win_fail, robust_c, w_out);
  } else {
    MN_LAUNCH(k_pgo<false>, n_windows, kPgoThreads, smem, st, poses, vos, out, N, fc, w4[0], w4[1], w4[2], w4[3],
              n_iters, exact, status, n_win_dev, win_fail, 0.0, (double*)nullptr);
  }
  MN_LAUNCH_CHECK();
  return 0;
}

void pgo_weights(double sax, double saq, double srx, double srq, double w4[4]) {
  w4[0] = 1.0 / sqrt(sax); w4[1] = 1.0 / sqrt(saq); w4[2] = 1.0 / sqrt(srx); w4[3] = 1.0 / sqrt(srq);
}

// ---- covariance-weighted pose graph (mapnet_pgo_optimize_cov, inference.SampledTracker).  k_pgo's state, relative
// factors and manifold update, with a full 7 x 7 covariance S7 = C C' per absolute factor (residual C^-1 (z - p),
// Jacobian C^-1 blockdiag(I, m_rot(q))), the exact Gauss-Newton step, and the posterior covariance of every slot:
// the 6 x 6 diagonal blocks of H^-1 at the returned state, mapped from (dt, x) to (t, log q).
//
// Deterministic: every factor first writes its Jacobian products into its own shared-memory record, then one thread
// per H / b entry adds the records that touch it in a fixed order (no atomics).  The Cholesky and the inverse
// R^-1 are right-looking over the block; the two triangular solves run in warp 0 with three rows per lane in
// registers (D <= 96), so they need shuffles instead of block barriers.
static constexpr int kUnaryRec = 42;      // per slot: JtJ [6][6], Jtr [6]
static constexpr int kEdgeRec = 45;       // per edge: Tt [3][3], gt [3], Haa, Hbb, Hab [3][3], ga [3], gb [3]

// index of the relative factor between slots i < j, -1 when there is none (the order of trackcore::vo_pair)
__device__ __forceinline__ int pgo_edge(int i, int j, int N, int fc) {
  if (!fc) return j == i + 1 ? i : -1;
  return i * (N - 1) - i * (i - 1) / 2 + (j - i - 1);
}

// G(q) = d qlog(q * dq(x)) / dx at x = 0 = Jlog(q) m_rot(q), qlog(w, u) = atan2(|u|, w) u / |u|
__device__ __forceinline__ void qlog_jac(const Q4& q, double G[3][3]) {
  const double u[3] = {q.x, q.y, q.z};
  const double s2 = u[0] * u[0] + u[1] * u[1] + u[2] * u[2], s = sqrt(s2), n2 = q.w * q.w + s2;
  double f, c;                            // d qlog / du = f I + c u u',  d qlog / dw = -u / n2
  const double t = s / q.w;
  if (q.w > 0.0 && t < 1e-2) {            // series in t = |u| / w: atan(t) / t and (w / n2 - f) / s2
    const double t2 = t * t;
    f = (1.0 + t2 * (-1.0 / 3.0 + t2 * (1.0 / 5.0 + t2 * (-1.0 / 7.0 + t2 / 9.0)))) / q.w;
    c = (-2.0 / 3.0 + t2 * (4.0 / 5.0 + t2 * (-6.0 / 7.0 + t2 * (8.0 / 9.0)))) / (q.w * q.w * q.w);
  } else {
    f = atan2(s, q.w) / s;
    c = (q.w / n2 - f) / s2;
  }
  double J[3][4];
  for (int a = 0; a < 3; ++a) {
    J[a][0] = -u[a] / n2;
    for (int b = 0; b < 3; ++b) J[a][1 + b] = (a == b ? f : 0.0) + c * u[a] * u[b];
  }
  double M[4][3];
  m_rot(q, M);
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      double v = 0.0;
      for (int k = 0; k < 4; ++k) v += J[a][k] * M[k][b];
      G[a][b] = v;
    }
}

// H (D x D) and b at state z: each factor's record, then one thread per entry sums the records touching it.
// kRobust: slot i's record is weighed by its Cauchy weight at z (scale c), which it also writes to w_out[i] when
// w_out is not null.
template <bool kRobust>
__device__ void pgo_cov_normal(const double* z, const double* P, const double* Li, const double* V, int N, int fc,
                               int E, double w_rx, double w_rq, double* rec, double* H, double* bv, double c,
                               double* w_out) {
  const int D = 6 * N;
  double* ru = rec;                       // [N][kUnaryRec]
  double* re = rec + N * kUnaryRec;       // [E][kEdgeRec]
  for (int f = threadIdx.x; f < N + E; f += blockDim.x) {
    if (f < N) {
      const int i = f;
      const Q4 q = {z[7 * i + 3], z[7 * i + 4], z[7 * i + 5], z[7 * i + 6]};
      double M[4][3], d[7], r[7], J[7][6];
      m_rot(q, M);
      for (int a = 0; a < 7; ++a) d[a] = z[7 * i + a] - P[7 * i + a];
      const double* L = Li + 49 * i;      // C^-1, lower triangular
      for (int a = 0; a < 7; ++a) {
        double v = 0.0;
        for (int b = 0; b <= a; ++b) v += L[7 * a + b] * d[b];
        r[a] = v;
        for (int cc = 0; cc < 3; ++cc) J[a][cc] = a >= cc ? L[7 * a + cc] : 0.0;
        for (int cc = 0; cc < 3; ++cc) {
          double s = 0.0;
          for (int b = 3; b <= a; ++b) s += L[7 * a + b] * M[b - 3][cc];
          J[a][3 + cc] = s;
        }
      }
      double om = 1.0;                      // the slot's Cauchy weight (1: plain least squares)
      if constexpr (kRobust) {
        om = cauchy_weight(r, c);
        if (w_out != nullptr) w_out[i] = om;
      }
      double* o = ru + kUnaryRec * i;
      for (int a = 0; a < 6; ++a) {
        for (int b = 0; b < 6; ++b) {
          double s = 0.0;
          for (int k = 0; k < 7; ++k) s += J[k][a] * J[k][b];
          o[6 * a + b] = kRobust ? om * s : s;
        }
        double s = 0.0;
        for (int k = 0; k < 7; ++k) s += J[k][a] * r[k];
        o[36 + a] = kRobust ? om * s : s;
      }
    } else {
      const int e = f - N;
      int i, j;
      trackcore::vo_pair(e, N, fc, &i, &j);
      const Q4 qi = {z[7 * i + 3], z[7 * i + 4], z[7 * i + 5], z[7 * i + 6]};
      const Q4 qj = {z[7 * j + 3], z[7 * j + 4], z[7 * j + 5], z[7 * j + 6]};
      double* o = re + kEdgeRec * e;
      double Dt[3][3], rt[3];
      dqstq_t(qi, Dt);
      const double dv[3] = {z[7 * j] - z[7 * i], z[7 * j + 1] - z[7 * i + 1], z[7 * j + 2] - z[7 * i + 2]};
      q_rotate(dv, q_inv(qi), rt);
      for (int a = 0; a < 3; ++a) {
        rt[a] = w_rx * (rt[a] - V[7 * e + a]);
        for (int b = 0; b < 3; ++b) Dt[a][b] *= w_rx;
      }
      for (int a = 0; a < 3; ++a) {
        double g = 0.0;
        for (int k = 0; k < 3; ++k) g += Dt[k][a] * rt[k];
        o[9 + a] = g;
        for (int b = 0; b < 3; ++b) {
          double s = 0.0;
          for (int k = 0; k < 3; ++k) s += Dt[k][a] * Dt[k][b];
          o[3 * a + b] = s;
        }
      }
      double A4[4][4], B4[4][4], Mi[4][3], Mj[4][3], Ja[4][3], Jb[4][3], rq[4];
      dpsq_p(qj, A4); dpsq_q(qi, B4); m_rot(qi, Mi); m_rot(qj, Mj);
      for (int a = 0; a < 4; ++a)
        for (int b = 0; b < 3; ++b) {
          double sa = 0.0, sb = 0.0;
          for (int k = 0; k < 4; ++k) { sa += A4[a][k] * Mi[k][b]; sb += B4[a][k] * Mj[k][b]; }
          Ja[a][b] = w_rq * sa; Jb[a][b] = w_rq * sb;
        }
      const Q4 qvo = q_mul(q_inv(qi), qj);
      rq[0] = w_rq * (qvo.w - V[7 * e + 3]); rq[1] = w_rq * (qvo.x - V[7 * e + 4]);
      rq[2] = w_rq * (qvo.y - V[7 * e + 5]); rq[3] = w_rq * (qvo.z - V[7 * e + 6]);
      for (int a = 0; a < 3; ++a) {
        double ga = 0.0, gb = 0.0;
        for (int k = 0; k < 4; ++k) { ga += Ja[k][a] * rq[k]; gb += Jb[k][a] * rq[k]; }
        o[39 + a] = ga; o[42 + a] = gb;
        for (int b = 0; b < 3; ++b) {
          double saa = 0.0, sbb = 0.0, sab = 0.0;
          for (int k = 0; k < 4; ++k) { saa += Ja[k][a] * Ja[k][b]; sbb += Jb[k][a] * Jb[k][b]; sab += Ja[k][a] * Jb[k][b]; }
          o[12 + 3 * a + b] = saa; o[21 + 3 * a + b] = sbb; o[30 + 3 * a + b] = sab;
        }
      }
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < D * D + D; idx += blockDim.x) {
    if (idx < D * D) {
      const int row = idx / D, col = idx % D, i = row / 6, a = row % 6, j = col / 6, b = col % 6;
      const bool tt = a < 3 && b < 3, qq = a >= 3 && b >= 3;
      double v;
      if (i == j) {
        v = ru[kUnaryRec * i + 6 * a + b];
        for (int m = 0; m < N; ++m) {
          const int e = m == i ? -1 : pgo_edge(i < m ? i : m, i < m ? m : i, N, fc);
          if (e < 0) continue;
          const double* o = re + kEdgeRec * e;
          if (tt) v += o[3 * a + b];
          else if (qq) v += o[(i < m ? 12 : 21) + 3 * (a - 3) + (b - 3)];
        }
      } else {
        const int e = pgo_edge(i < j ? i : j, i < j ? j : i, N, fc);
        const double* o = re + kEdgeRec * (e < 0 ? 0 : e);
        v = 0.0;
        if (e >= 0 && tt) v = -o[3 * a + b];
        else if (e >= 0 && qq) v = i < j ? o[30 + 3 * (a - 3) + (b - 3)] : o[30 + 3 * (b - 3) + (a - 3)];
      }
      H[idx] = v;
    } else {
      const int row = idx - D * D, i = row / 6, a = row % 6;
      double v = ru[kUnaryRec * i + 36 + a];
      for (int m = 0; m < N; ++m) {
        const int e = m == i ? -1 : pgo_edge(i < m ? i : m, i < m ? m : i, N, fc);
        if (e < 0) continue;
        const double* o = re + kEdgeRec * e;
        if (a < 3) v += i < m ? -o[9 + a] : o[9 + a];
        else v += o[(i < m ? 39 : 42) + a - 3];
      }
      bv[row] = v;
    }
  }
  __syncthreads();
}

// H = R' R in place (upper R, row-major), right-looking over the block, as k_pgo factors; a pivot <= 0 sets *fail
__device__ void pgo_cov_cholesky(double* H, int D, int* fail) {
  for (int k = 0; k < D; ++k) {
    if (threadIdx.x == 0) {
      const double d = H[k * D + k];
      if (!(d > 0.0)) *fail = 1;
      H[k * D + k] = sqrt(d > 0.0 ? d : 1.0);
    }
    __syncthreads();
    const double rkk = H[k * D + k];
    for (int j = k + 1 + threadIdx.x; j < D; j += blockDim.x) H[k * D + j] /= rkk;
    __syncthreads();
    for (int idx = threadIdx.x; idx < (D - k - 1) * (D - k - 1); idx += blockDim.x) {
      const int i = k + 1 + idx / (D - k - 1), j = k + 1 + idx % (D - k - 1);
      if (j >= i) H[i * D + j] -= H[k * D + i] * H[k * D + j];
    }
    __syncthreads();
  }
}

// warp 0: xs = -(R'R)^-1 b, rows lane, lane + 32, lane + 64 in registers
__device__ void pgo_cov_solve(const double* R, const double* bv, int D, double* xs) {
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  double y[3];
#pragma unroll
  for (int s = 0; s < 3; ++s) y[s] = lane + 32 * s < D ? -bv[lane + 32 * s] : 0.0;
  for (int k = 0; k < D; ++k) {             // R' y = -b
    const int ks = k >> 5;
    double yk = ks == 0 ? y[0] : (ks == 1 ? y[1] : y[2]);
    yk = __shfl_sync(0xffffffffu, yk, k & 31) / R[k * D + k];
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int i = lane + 32 * s;
      if (i == k) y[s] = yk;
      else if (i > k && i < D) y[s] -= R[k * D + i] * yk;
    }
  }
  for (int k = D - 1; k >= 0; --k) {        // R x = y
    const int ks = k >> 5;
    double xk = ks == 0 ? y[0] : (ks == 1 ? y[1] : y[2]);
    xk = __shfl_sync(0xffffffffu, xk, k & 31) / R[k * D + k];
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int i = lane + 32 * s;
      if (i == k) y[s] = xk;
      else if (i < k) y[s] -= R[i * D + k] * xk;
    }
  }
#pragma unroll
  for (int s = 0; s < 3; ++s)
    if (lane + 32 * s < D) xs[lane + 32 * s] = y[s];
}

// One window per block (kPgoThreads threads).  poses [W][N][7] (the absolute poses p), sig7 [W][N][7][7] (their
// covariances), vos [W][E][7] -> out [W][N][7], cov [W][N][6][6]; n_win_dev, win_fail and status as for k_pgo.
// kRobust: the absolute factors are Cauchy-weighted as in k_pgo<true>, each iteration's weights taken at its starting
// state; the posterior's normal matrix is built at the returned state with the weights at that state, which w_out
// (may be null) [W][N] gets.  Without kRobust, c and w_out are not read.
template <bool kRobust>
__global__ void __launch_bounds__(kPgoThreads)
k_pgo_cov(const double* __restrict__ poses, const double* __restrict__ sig7, const double* __restrict__ vos,
          double* __restrict__ out, double* __restrict__ cov, int N, int fc, double w_rx, double w_rq, int n_iters,
          int* __restrict__ status, const int* __restrict__ n_win_dev, int* __restrict__ win_fail, double c,
          double* __restrict__ w_out) {
  pdl_prologue();
  if (n_win_dev != nullptr && (int)blockIdx.x >= *n_win_dev) return;
  extern __shared__ double sm[];
  const int D = 6 * N, W = blockIdx.x;
  const int E = fc ? N * (N - 1) / 2 : N - 1;
  double* H = sm;                         // D x D
  double* bv = H + D * D;                 // D
  double* xs = bv + D;                    // D
  double* z = xs + D;                     // 7 N
  double* Li = z + 7 * N;                 // N x [7][7]: C^-1
  double* rec = Li + 49 * N;              // factor records, then the posterior blocks [N][36]
  const double* P = poses + (size_t)W * N * 7;
  const double* V = vos + (size_t)W * E * 7;
  __shared__ int s_fail;
  if (threadIdx.x == 0) s_fail = 0;
  for (int i = threadIdx.x; i < 7 * N; i += blockDim.x) z[i] = P[i];
  // prologue: C = chol(S7) and C^-1 per slot
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const double* S = sig7 + ((size_t)W * N + i) * 49;
    double C[7][7];
    bool ok = true;
    for (int c = 0; c < 7; ++c) {
      for (int r = c; r < 7; ++r) {
        double v = S[7 * r + c];
        for (int k = 0; k < c; ++k) v -= C[r][k] * C[c][k];
        if (r == c) {
          if (!(v > 0.0)) { ok = false; v = 1.0; }
          C[c][c] = sqrt(v);
        } else {
          C[r][c] = v / C[c][c];
        }
      }
    }
    double* L = Li + 49 * i;
    for (int c = 0; c < 7; ++c)             // C L = I, column by column
      for (int r = 0; r < 7; ++r) {
        double v = r == c ? 1.0 : 0.0;
        for (int k = c; k < r; ++k) v -= C[r][k] * L[7 * k + c];
        L[7 * r + c] = r < c ? 0.0 : v / C[r][r];
      }
    if (!ok) atomicExch(&s_fail, 1);
  }
  __syncthreads();
  for (int it = 0; it <= n_iters; ++it) {
    pgo_cov_normal<kRobust>(z, P, Li, V, N, fc, E, w_rx, w_rq, rec, H, bv, c,
                            kRobust && it == n_iters && w_out != nullptr ? w_out + (size_t)W * N : nullptr);
    pgo_cov_cholesky(H, D, &s_fail);
    if (it == n_iters) break;               // the posterior's factor, at the returned state
    pgo_cov_solve(H, bv, D, xs);
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      z[7 * i] += xs[6 * i]; z[7 * i + 1] += xs[6 * i + 1]; z[7 * i + 2] += xs[6 * i + 2];
      const double mx = xs[6 * i + 3], my = xs[6 * i + 4], mz = xs[6 * i + 5];
      const double n = sqrt(mx * mx + my * my + mz * mz);
      const double sc = (n == 0.0) ? 1.0 : sin(n) / n;
      const Q4 dq = {cos(n), sc * mx, sc * my, sc * mz};
      const Q4 q = q_mul(Q4{z[7 * i + 3], z[7 * i + 4], z[7 * i + 5], z[7 * i + 6]}, dq);
      z[7 * i + 3] = q.w; z[7 * i + 4] = q.x; z[7 * i + 5] = q.y; z[7 * i + 6] = q.z;
    }
    __syncthreads();
  }
  // Q = R^-1 (upper), right-looking from the last row: Q[a][c] (a < c) kept in H[c][a], its diagonal in xs
  for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
    const int r = idx / D, c = idx % D;
    if (c < r) H[idx] = 0.0;
  }
  for (int i = threadIdx.x; i < D; i += blockDim.x) xs[i] = 1.0;
  __syncthreads();
  for (int m = D - 1; m >= 0; --m) {
    const double rmm = H[m * D + m];
    for (int c = m + threadIdx.x; c < D; c += blockDim.x) {
      if (c == m) xs[m] /= rmm;
      else H[c * D + m] /= rmm;
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < m * (D - m); idx += blockDim.x) {
      const int a = idx / (D - m), c = m + idx % (D - m);
      const double qmc = c == m ? xs[m] : H[c * D + m];
      H[c * D + a] -= H[a * D + m] * qmc;
    }
    __syncthreads();
  }
  // P = Q Q': the 6 x 6 diagonal block of each slot
  double* Pb = rec;
  for (int idx = threadIdx.x; idx < 36 * N; idx += blockDim.x) {
    const int i = idx / 36, a = 6 * i + (idx % 36) / 6, b = 6 * i + idx % 6;
    const int c0 = a > b ? a : b;
    double v = (c0 == a ? xs[a] : H[c0 * D + a]) * (c0 == b ? xs[b] : H[c0 * D + b]);
    for (int c = c0 + 1; c < D; ++c) v += H[c * D + a] * H[c * D + b];
    Pb[idx] = v;
  }
  __syncthreads();
  double* O = out + (size_t)W * N * 7;
  for (int i = threadIdx.x; i < 7 * N; i += blockDim.x) O[i] = z[i];
  for (int i = threadIdx.x; i < N; i += blockDim.x) {   // cov = B P B', B = blockdiag(I, G(q))
    double G[3][3], B[6][6] = {};
    qlog_jac(Q4{z[7 * i + 3], z[7 * i + 4], z[7 * i + 5], z[7 * i + 6]}, G);
    for (int a = 0; a < 3; ++a) {
      B[a][a] = 1.0;
      for (int b = 0; b < 3; ++b) B[3 + a][3 + b] = G[a][b];
    }
    const double* Pi = Pb + 36 * i;
    double BP[6][6];
    for (int a = 0; a < 6; ++a)
      for (int b = 0; b < 6; ++b) {
        double v = 0.0;
        for (int k = 0; k < 6; ++k) v += B[a][k] * Pi[6 * k + b];
        BP[a][b] = v;
      }
    double* o = cov + ((size_t)W * N + i) * 36;
    for (int a = 0; a < 6; ++a)
      for (int b = 0; b < 6; ++b) {
        double v = 0.0;
        for (int k = 0; k < 6; ++k) v += BP[a][k] * B[b][k];
        o[6 * a + b] = v;
      }
  }
  if (threadIdx.x == 0 && s_fail && status != nullptr) atomicExch(status, 1);
  if (threadIdx.x == 0 && win_fail != nullptr) win_fail[W] = s_fail;
}

static size_t pgo_cov_smem(int N) {
  const int D = 6 * N, E = N * (N - 1) / 2;
  const int rec = N * kUnaryRec + E * kEdgeRec;
  return (size_t)(D * D + 2 * D + 7 * N + 49 * N + (rec > 36 * N ? rec : 36 * N)) * sizeof(double);
}

int pgo_cov_prepare() {
  static bool attr = false;
  if (!attr) {
    MN_CUDA(cudaFuncSetAttribute(k_pgo_cov<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)pgo_cov_smem(kPgoMaxN)));
    MN_CUDA(cudaFuncSetAttribute(k_pgo_cov<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)pgo_cov_smem(kPgoMaxN)));
    attr = true;
  }
  return 0;
}

int launch_pgo_cov(const double* poses, const double* sig7, const double* vos, double* out, double* cov, int n_windows,
                   int N, int fc, double w_rx, double w_rq, int n_iters, int* status, const int* n_win_dev,
                   int* win_fail, cudaStream_t st, double robust_c, double* w_out) {
  MN_TRY(pgo_cov_prepare());
  if (robust_c > 0.0) {
    MN_LAUNCH(k_pgo_cov<true>, n_windows, kPgoThreads, pgo_cov_smem(N), st, poses, sig7, vos, out, cov, N, fc, w_rx,
              w_rq, n_iters, status, n_win_dev, win_fail, robust_c, w_out);
  } else {
    MN_LAUNCH(k_pgo_cov<false>, n_windows, kPgoThreads, pgo_cov_smem(N), st, poses, sig7, vos, out, cov, N, fc, w_rx,
              w_rq, n_iters, status, n_win_dev, win_fail, 0.0, (double*)nullptr);
  }
  MN_LAUNCH_CHECK();
  return 0;
}

}  // namespace mapnet

using namespace mapnet;

extern "C" int mapnet_pgo_optimize(const double* poses, const double* vos, double* out, int n_windows, int N, int fc_vos,
                                   double sax, double saq, double srx, double srq, int n_iters, int flags, int* status_dev,
                                   void* stream) {
  MN_CHECK(poses && vos && out && n_windows >= 1, "pgo_optimize: bad argument");
  MN_CHECK(N >= 2 && N <= kPgoMaxN, "pgo_optimize: window of %d poses outside [2, %d]", N, kPgoMaxN);
  MN_CHECK(sax > 0 && saq > 0 && srx > 0 && srq > 0 && n_iters >= 0, "pgo_optimize: covariances must be positive");
  int ndev = 0;
  MN_CHECK(cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0, "pgo_optimize: no CUDA device (this library has no CPU fallback)");
  double w4[4];
  pgo_weights(sax, saq, srx, srq, w4);
  return launch_pgo(poses, vos, out, n_windows, N, fc_vos ? 1 : 0, w4, n_iters, flags & 1, status_dev, nullptr,
                    (cudaStream_t)stream);
}

extern "C" int mapnet_pgo_optimize_cov(const double* poses, const double* sig7, const double* vos, double* out,
                                       double* cov, int n_windows, int N, int fc_vos, double srx, double srq,
                                       int n_iters, int* status_dev, void* stream) {
  MN_CHECK(poses && sig7 && vos && out && cov && n_windows >= 1, "pgo_optimize_cov: bad argument");
  MN_CHECK(N >= 2 && N <= kPgoMaxN, "pgo_optimize_cov: window of %d poses outside [2, %d]", N, kPgoMaxN);
  MN_CHECK(srx > 0 && srq > 0 && n_iters >= 0, "pgo_optimize_cov: covariances must be positive");
  int ndev = 0;
  MN_CHECK(cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0,
           "pgo_optimize_cov: no CUDA device (this library has no CPU fallback)");
  return launch_pgo_cov(poses, sig7, vos, out, cov, n_windows, N, fc_vos ? 1 : 0, 1.0 / sqrt(srx), 1.0 / sqrt(srq),
                        n_iters, status_dev, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int mapnet_pgo_optimize_robust(const double* poses, const double* vos, double* out, int n_windows, int N,
                                          int fc_vos, double sax, double saq, double srx, double srq, int n_iters,
                                          int flags, double c, double* w, int* status_dev, void* stream) {
  MN_CHECK(poses && vos && out && n_windows >= 1, "pgo_optimize_robust: bad argument");
  MN_CHECK(N >= 2 && N <= kPgoMaxN, "pgo_optimize_robust: window of %d poses outside [2, %d]", N, kPgoMaxN);
  MN_CHECK(sax > 0 && saq > 0 && srx > 0 && srq > 0 && n_iters >= 0,
           "pgo_optimize_robust: covariances must be positive");
  MN_CHECK(c > 0 && isfinite(c), "pgo_optimize_robust: the Cauchy scale c = %g must be finite and positive", c);
  int ndev = 0;
  MN_CHECK(cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0,
           "pgo_optimize_robust: no CUDA device (this library has no CPU fallback)");
  double w4[4];
  pgo_weights(sax, saq, srx, srq, w4);
  return launch_pgo(poses, vos, out, n_windows, N, fc_vos ? 1 : 0, w4, n_iters, flags & 1, status_dev, nullptr,
                    (cudaStream_t)stream, nullptr, c, w);
}

extern "C" int mapnet_pgo_optimize_cov_robust(const double* poses, const double* sig7, const double* vos, double* out,
                                              double* cov, int n_windows, int N, int fc_vos, double srx, double srq,
                                              int n_iters, double c, double* w, int* status_dev, void* stream) {
  MN_CHECK(poses && sig7 && vos && out && cov && n_windows >= 1, "pgo_optimize_cov_robust: bad argument");
  MN_CHECK(N >= 2 && N <= kPgoMaxN, "pgo_optimize_cov_robust: window of %d poses outside [2, %d]", N, kPgoMaxN);
  MN_CHECK(srx > 0 && srq > 0 && n_iters >= 0, "pgo_optimize_cov_robust: covariances must be positive");
  MN_CHECK(c > 0 && isfinite(c), "pgo_optimize_cov_robust: the Cauchy scale c = %g must be finite and positive", c);
  int ndev = 0;
  MN_CHECK(cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0,
           "pgo_optimize_cov_robust: no CUDA device (this library has no CPU fallback)");
  return launch_pgo_cov(poses, sig7, vos, out, cov, n_windows, N, fc_vos ? 1 : 0, 1.0 / sqrt(srx), 1.0 / sqrt(srq),
                        n_iters, status_dev, nullptr, nullptr, (cudaStream_t)stream, c, w);
}

// qexp + un-normalisation of a batch of 6-vectors (scripts/eval.py:163-181): out[i] = (t * pose_s + pose_m, qexp(logq))
namespace mapnet {
__global__ void k_pose_post(const float* __restrict__ p6, double* __restrict__ out7, long long n, double m0, double m1,
                            double m2, double s0, double s1, double s2, int unnormalize) {
  pdl_prologue();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double ms[3] = {m0, m1, m2}, ss[3] = {s0, s1, s2};
  for (int k = 0; k < 3; ++k) {
    const double t = (double)p6[6 * i + k];
    out7[7 * i + k] = unnormalize ? t * ss[k] + ms[k] : t;
  }
  post_qexp(p6[6 * i + 3], p6[6 * i + 4], p6[6 * i + 5], out7 + 7 * i + 3);
}
}  // namespace mapnet

extern "C" int mapnet_pose_post(const float* pred6, double* out7, int64_t n, const double* pose_m3, const double* pose_s3,
                                void* stream) {
  MN_CHECK(pred6 && out7 && n >= 1, "pose_post: bad argument");
  const int un = (pose_m3 != nullptr && pose_s3 != nullptr) ? 1 : 0;
  MN_LAUNCH(k_pose_post, cdiv(n, 128), 128, 0, (cudaStream_t)stream, pred6, out7, (long long)n, un ? pose_m3[0] : 0.0,
            un ? pose_m3[1] : 0.0, un ? pose_m3[2] : 0.0, un ? pose_s3[0] : 1.0, un ? pose_s3[1] : 1.0, un ? pose_s3[2] : 1.0, un);
  MN_LAUNCH_CHECK();
  return 0;
}

// Monte-Carlo dropout poses in metric units (mapnet_sample_post), float64 throughout: with D = diag(pose_s, 1, 1, 1),
// pose7 = (mean_t * pose_s + pose_m, qexp(mean_logq)), qexp(v) = (cos n, sin n / n * v) with n = |v| ((1, 0, 0, 0) at
// n = 0), cov_metric = D cov D, t_std = sqrt(trace of cov_metric's translation block) and q_std_deg = 2 sqrt(trace of
// the log q block) * 180 / pi (a log q perturbation dv turns the rotation by about 2 |dv|).
namespace mapnet {
__global__ void k_sample_post(const double* __restrict__ mean, const double* __restrict__ cov, long long n, double m0,
                              double m1, double m2, double s0, double s1, double s2, double* __restrict__ pose7,
                              double* __restrict__ cov_out, double* __restrict__ t_std, double* __restrict__ q_std_deg) {
  pdl_prologue();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* mu = mean + 6 * i;
  const double* C = cov + 36 * i;
  const double ms[3] = {m0, m1, m2}, d[6] = {s0, s1, s2, 1.0, 1.0, 1.0};
  if (pose7 != nullptr) {
    double* o = pose7 + 7 * i;
    for (int k = 0; k < 3; ++k) o[k] = mu[k] * d[k] + ms[k];
    sample_qexp(mu[3], mu[4], mu[5], o + 3);
  }
  sample_stats(C, d, cov_out != nullptr ? cov_out + 36 * i : nullptr, t_std + i, q_std_deg + i);
}
}  // namespace mapnet

extern "C" int mapnet_sample_post(const double* mean, const double* cov, int64_t n, const double* pose_m3,
                                  const double* pose_s3, double* pose7, double* cov_metric, double* t_std,
                                  double* q_std_deg, void* stream) {
  MN_CHECK(mean && cov && t_std && q_std_deg && n >= 1, "sample_post: bad argument");
  MN_CHECK((pose_m3 == nullptr) == (pose_s3 == nullptr), "sample_post: pose_m3 and pose_s3 go together");
  const int un = pose_m3 != nullptr;
  MN_LAUNCH(k_sample_post, cdiv(n, 128), 128, 0, (cudaStream_t)stream, mean, cov, (long long)n, un ? pose_m3[0] : 0.0,
            un ? pose_m3[1] : 0.0, un ? pose_m3[2] : 0.0, un ? pose_s3[0] : 1.0, un ? pose_s3[1] : 1.0,
            un ? pose_s3[2] : 1.0, pose7, cov_metric, t_std, q_std_deg);
  MN_LAUNCH_CHECK();
  return 0;
}
