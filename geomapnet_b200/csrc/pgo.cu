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

// One window per block.  Constraints are dealt to threads; each thread accumulates into the shared H / b with
// double atomics (a few hundred constraints x <= 144 entries: contention is irrelevant next to the Cholesky).
__global__ void __launch_bounds__(kPgoThreads)
k_pgo(const double* __restrict__ poses, const double* __restrict__ vos, double* __restrict__ out, int N, int fc,
      double w_ax, double w_aq, double w_rx, double w_rq, int n_iters, int exact, int* __restrict__ status) {
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
    for (int c = threadIdx.x; c < N + E; c += blockDim.x) {
      if (c < N) {
        const int i = c;
        const Q4 q = {z[7 * i + 3], z[7 * i + 4], z[7 * i + 5], z[7 * i + 6]};
        // translation: J = w_ax I, r = w_ax (t - t0)
        for (int a = 0; a < 3; ++a) {
          atomicAdd(&H[(6 * i + a) * D + 6 * i + a], w_ax * w_ax);
          atomicAdd(&bv[6 * i + a], w_ax * w_ax * (z[7 * i + a] - P[7 * i + a]));
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
            atomicAdd(&H[(6 * i + 3 + a) * D + 6 * i + 3 + b], s);
          }
          double s = 0.0;
          for (int k = 0; k < 4; ++k) s += M[k][a] * r[k];
          atomicAdd(&bv[6 * i + 3 + a], s);
        }
      } else {
        int e = c - N, i, j;
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
  if (threadIdx.x == 0 && s_fail && status != nullptr) atomicExch(status, 1);
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
  const int D = 6 * N;
  const size_t smem = (size_t)(D * D + D + 7 * N + D) * sizeof(double);
  static bool attr = false;
  if (!attr) { MN_CUDA(cudaFuncSetAttribute(k_pgo, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(96 * 96 + 96 * 2 + 7 * 16) * 8)); attr = true; }
  MN_LAUNCH(k_pgo, n_windows, kPgoThreads, smem, (cudaStream_t)stream, poses, vos, out, N, fc_vos ? 1 : 0, 1.0 / sqrt(sax),
            1.0 / sqrt(saq), 1.0 / sqrt(srx), 1.0 / sqrt(srq), n_iters, flags & 1, status_dev);
  MN_LAUNCH_CHECK();
  return 0;
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
