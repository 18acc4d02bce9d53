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
#include "track_core.h"
#include "calib_core.h"

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

// calc_vos_safe / calc_vos_safe_fc (common/pose_utils.py:276-304) of VO pair p on the VO library's float32 poses, as the
// MFOnline targets of k_loader_assemble
__device__ __forceinline__ void eval_vo(const float* vo_poses, const TargRow p, double* o7) {
  const posemath::Pose6 v = posemath::calc_vo_logq_safe(ld_pose6(vo_poses + 6LL * p.a), ld_pose6(vo_poses + 6LL * p.b));
  const float v6[6] = {v.t.x, v.t.y, v.t.z, v.l.x, v.l.y, v.l.z};
  st_pose7(v6, o7);
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
    eval_vo(vo_poses, vo_rows[k], vos7 + 7LL * k);
  }
}

// ---- streaming pose-graph tracker (mapnet_track_*, inference.Tracker): eval.py's windows over frames as they arrive.
// Device state of one sequence (one per stream of a multi-stream tracker): `seen` frames so far; status: 1 once a
// window's normal matrix was not positive definite.  The count of windows the current call solves sits apart, with the
// per-window failure flags of a multi-stream call: written by the gather for the PGO launch and the emit.
struct TrackDev {
  long long seen;
  int status, pad;
};

// what a tracker handle is created with: window geometry, PGO weights, pose statistics (single and multi-stream)
struct TrackCfg {
  int T, skip, fc, max_batch, E, max_win;   // max_win: the most windows one call completes, max(max_batch, lag)
  long long R, lag;
  double w4[4];                             // PGO weights 1/sqrt(sigma) of sax, saq, srx, srq
  int un;
  double m[3], s[3];
};

// the device state of every tracker handle: n_streams sequences (1 for the single-stream trackers), their rings of R
// frames and the windows of one call.  The sampled trackers' buffers (ring49, win49, cov36) are null for point factors.
struct TrackHandle : TrackCfg {
  int n_streams;
  double sax, saq;                          // the floors of the absolute factors' covariances (sampled)
  TrackDev* st;                             // [n_streams]
  int* n_win;                               // the windows of the current call, written by the gather
  int* win_fail;                            // [max_win]: the PGO's per-window failure flags (multi-stream)
  double *ring7, *ring49;                   // [n_streams][R][7], [n_streams][R][7][7]: p and S7 of the last R frames
  float* ring_vo;                           // [n_streams][R][6]: their VO-library poses
  double *win7, *win49, *vos7, *opt7, *cov36;   // [max_win][T][7], [.][T][49], [.][E][7], [.][T][7], [.][T][36]
  double robust_c;                          // > 0: the Cauchy scale of the absolute factors (fixed before the first step)
  bool started;                             // a step or flush has been enqueued: robust_c is fixed
};

__device__ __forceinline__ const float* track_src(const float* fresh, const float* ring, long long f, long long seen,
                                                  long long R) {
  return f >= seen ? fresh + 6 * (f - seen) : ring + 6 * (f % R);
}

__device__ __forceinline__ void track_emit_pose(const double* p, int un, const double ms[3], const double ss[3],
                                                double* o) {
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] = un ? trackcore::unnormalize(p[k], ss[k], ms[k]) : p[k];
#pragma unroll
  for (int k = 3; k < 7; ++k) o[k] = p[k];
}

// ---- Monte-Carlo tracker (mapnet_track_sample_*, inference.SampledTracker): mapnet_track_*'s windows, with each
// frame's S-draw mean (t, log q) and covariance Sigma [6][6] (float64, mapnet_infer_sample_frames' outputs) in place of
// its one draw.  A new frame's absolute pose p = (mean_t, qexp(mean_v)) (k_sample_post's qexp) and its factor covariance
// S7 = A Sigma A' + diag(sax I3, saq I4), A = blockdiag(I3, E(mean_v)), are formed into rings of R frames; the
// windows gather them, k_pgo_cov solves them, and the emit writes per window row pose7 [7], cov [36] = D cov D,
// t_std, q_std_deg (k_sample_post's statistics), kTrackSampleRow doubles.
static constexpr int kTrackSampleRow = 45;

// E(v) = d qexp(v) / dv (4 x 3): row 0 -sinc(n) v', rows 1..3 sinc(n) I + g(n) v v', g = (n cos n - sin n) / n^3
// (its series below n = 0.1, where the difference cancels), sinc(n) = sin n / n
__device__ __forceinline__ void qexp_jac(const double v[3], double Ej[4][3]) {
  const double n2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2], n = sqrt(n2);
  const double sc = n > 0.0 ? sin(n) / n : 1.0;
  const double g = n < 0.1 ? -1.0 / 3.0 + n2 * (1.0 / 30.0 + n2 * (-1.0 / 840.0 + n2 * (1.0 / 45360.0 -
                                                                                      n2 / 3991680.0)))
                           : (n * cos(n) - sin(n)) / (n2 * n);
  for (int b = 0; b < 3; ++b) {
    Ej[0][b] = -sc * v[b];
    for (int a = 0; a < 3; ++a) Ej[1 + a][b] = (a == b ? sc : 0.0) + g * v[a] * v[b];
  }
}

// one frame's absolute pose p7 = (mean_t, qexp(mean_v)) from its draws' mean [6]
__device__ __forceinline__ void sample_pose7(const double* mu, double p7[7]) {
  p7[0] = mu[0]; p7[1] = mu[1]; p7[2] = mu[2];
  sample_qexp(mu[3], mu[4], mu[5], p7 + 3);
}

// one frame's absolute pose p7 and factor covariance S7 [7][7] from its draws' mean [6] and covariance [36]
__device__ __forceinline__ void sample_factor(const double* mu, const double* C, double sax, double saq, double p7[7],
                                              double S7[49]) {
  sample_pose7(mu, p7);
  double Ej[4][3];
  qexp_jac(mu + 3, Ej);
  double A[7][6] = {};
  for (int a = 0; a < 3; ++a) A[a][a] = 1.0;
  for (int a = 0; a < 4; ++a)
    for (int b = 0; b < 3; ++b) A[3 + a][3 + b] = Ej[a][b];
  for (int r = 0; r < 7; ++r)
    for (int c = 0; c < 7; ++c) {
      double v = 0.0;
      for (int k = 0; k < 6; ++k) {
        double ac = 0.0;
        for (int l = 0; l < 6; ++l) ac += C[6 * k + l] * A[c][l];
        v += A[r][k] * ac;
      }
      S7[7 * r + c] = v + (r == c ? (r < 3 ? sax : saq) : 0.0);
    }
}

// mapnet_test_sample_factor: sample_factor of n frames, the tracker's own arithmetic, for tests that compose its windows
__global__ void __launch_bounds__(128)
k_test_sample_factor(const double* __restrict__ mean, const double* __restrict__ cov, long long n, double sax,
                     double saq, double* __restrict__ p7, double* __restrict__ s7) {
  pdl_prologue();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) sample_factor(mean + 6 * i, cov + 36 * i, sax, saq, p7 + 7 * i, s7 + 49 * i);
}

__device__ __forceinline__ void track_sample_row(const double* p7, const double* C, int un, const double ms[3],
                                                 const double ss[3], double* o) {
  track_emit_pose(p7, un, ms, ss, o);
  const double d[6] = {ss[0], ss[1], ss[2], 1.0, 1.0, 1.0};
  sample_stats(C, d, o + 7, o + 43, o + 44);
}

// ---- the factors a window slot holds: everything the point and the sampled trackers do differently.  A factor is
// formed from input row b of a call into ring slot q or window slot q (a pure function of the row, so every copy is
// bit for bit the ring's), copied from ring slot q into window slot r, and an optimised window slot becomes an
// output row of kRow doubles; pgo launches the matching pose-graph optimisation of the call's windows.
// Point factors: p7 = st_pose7 of the engine's float32 (t, log q); k_pgo.
struct PointFactor {
  static constexpr int kRow = 7;
  const float* pred6;                       // [B][6], null for a flush
  double *ring7, *win7;
  const double* opt7;

  PointFactor(const TrackHandle& h, const float* pred6_)
      : pred6(pred6_), ring7(h.ring7), win7(h.win7), opt7(h.opt7) {}
  __device__ __forceinline__ void form(long long b, bool ring, long long q) const {
    st_pose7(pred6 + 6 * b, (ring ? ring7 : win7) + 7 * q);
  }
  __device__ __forceinline__ void nan_slot(long long r) const {
    const float nan = __int_as_float(0x7fc00000);
    const float v6[6] = {nan, nan, nan, nan, nan, nan};
    st_pose7(v6, win7 + 7 * r);
  }
  __device__ __forceinline__ void copy(long long q, long long r) const {
#pragma unroll
    for (int c = 0; c < 7; ++c) win7[7 * r + c] = ring7[7 * q + c];
  }
  __device__ __forceinline__ void row(long long k, int un, const double ms[3], const double ss[3], double* o) const {
    track_emit_pose(opt7 + 7 * k, un, ms, ss, o);
  }
  int pgo(const TrackHandle& h, int nw, int* status, const int* n_win_dev, int* win_fail, cudaStream_t st) const {
    return launch_pgo(h.win7, h.vos7, h.opt7, nw, h.T, h.fc, h.w4, 10, 0, status, n_win_dev, st, win_fail,
                      h.robust_c);
  }
};

// Sampled factors: p7 and S7 = sample_factor of the frame's float64 mean [6] and covariance [36]; k_pgo_cov, whose
// posterior cov36 the output rows carry.
struct SampleFactor {
  static constexpr int kRow = kTrackSampleRow;
  const double *mean, *cov;                 // [B][6], [B][36], null for a flush
  double sax, saq;
  double *ring7, *ring49, *win7, *win49;
  const double *opt7, *cov36;

  SampleFactor(const TrackHandle& h, const double* mean_, const double* cov_)
      : mean(mean_), cov(cov_), sax(h.sax), saq(h.saq), ring7(h.ring7), ring49(h.ring49), win7(h.win7),
        win49(h.win49), opt7(h.opt7), cov36(h.cov36) {}
  // window slots alone, without a tracker (k_eval_sample_windows)
  SampleFactor(const double* mean_, const double* cov_, double sax_, double saq_, double* win7_, double* win49_)
      : mean(mean_), cov(cov_), sax(sax_), saq(saq_), ring7(nullptr), ring49(nullptr), win7(win7_), win49(win49_),
        opt7(nullptr), cov36(nullptr) {}
  // the frame's mean and covariance through the read-only path into registers first: the struct's pointers carry no
  // restrict, so sample_factor reading them in place would reload the covariance after every store of S7
  __device__ __forceinline__ void form(long long b, bool ring, long long q) const {
    double mu[6], C[36];
#pragma unroll
    for (int c = 0; c < 6; ++c) mu[c] = __ldg(mean + 6 * b + c);
#pragma unroll
    for (int c = 0; c < 36; ++c) C[c] = __ldg(cov + 36 * b + c);
    sample_factor(mu, C, sax, saq, (ring ? ring7 : win7) + 7 * q, (ring ? ring49 : win49) + 49 * q);
  }
  __device__ __forceinline__ void nan_slot(long long r) const {
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    for (int c = 0; c < 7; ++c) win7[7 * r + c] = nan;
    for (int c = 0; c < 49; ++c) win49[49 * r + c] = nan;
  }
  __device__ __forceinline__ void copy(long long q, long long r) const {
    for (int c = 0; c < 7; ++c) win7[7 * r + c] = ring7[7 * q + c];
    for (int c = 0; c < 49; ++c) win49[49 * r + c] = ring49[49 * q + c];
  }
  __device__ __forceinline__ void row(long long k, int un, const double ms[3], const double ss[3], double* o) const {
    track_sample_row(opt7 + 7 * k, cov36 + 36 * k, un, ms, ss, o);
  }
  int pgo(const TrackHandle& h, int nw, int* status, const int* n_win_dev, int* win_fail, cudaStream_t st) const {
    return launch_pgo_cov(h.win7, h.win49, h.vos7, h.opt7, h.cov36, nw, h.T, h.fc, h.w4[2], h.w4[3], 10, status,
                          n_win_dev, win_fail, st, h.robust_c);
  }
};

// One thread per row: the n new frames into the rings (their factors, the VO-library pose as given), then slot
// (w, k) of every completed window w < n_win (rows n .. n + max_win*T - 1), then VO (w, e) (the next max_win*E rows).
// A slot's frame comes from this call's inputs when it is new, else from the ring: R = max_batch + (T-1)*skip frames
// hold every older frame a window of this call reaches, none of them in a ring slot this call writes.  The values are
// k_eval_windows': the frame's factor (st_pose7 of the float32 pose for point factors), calc_vo_logq_safe of the
// float32 VO-library poses.  A zero-lag call (now) gathers the n windows that end at its frames instead, from centre
// now_first(seen); *n_win_dev is the count of completed windows either way.
template <class F>
__global__ void __launch_bounds__(128)
k_track_gather(F fac, const float* __restrict__ vo6, int n, int flush, int now, const TrackDev* __restrict__ st,
               int* __restrict__ n_win_dev, float* __restrict__ ring_vo, long long R, int T, int skip, int fc,
               int max_win, double* __restrict__ vos7) {
  pdl_prologue();
  const long long seen = st->seen, total = seen + n, lag = trackcore::lag(T, skip);
  const long long pending = trackcore::first_pending(seen, lag);
  const int n_done = (int)((flush ? total : trackcore::first_pending(total, lag)) - pending);
  const long long first = now ? trackcore::now_first(seen, lag) : pending;
  const int n_win = now ? n : n_done;
  const int E = fc ? T * (T - 1) / 2 : T - 1;
  long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0) *n_win_dev = n_done;
  // the input row b whose factor this thread forms into ring slot q (a new frame) or window slot q: one call site,
  // so the threads of a warp that form a frame's ring copy and its window copies run the formation together
  const bool ring = r < n;
  long long b, q;
  if (ring) {
    b = r; q = (seen + r) % R;
#pragma unroll
    for (int c = 0; c < 6; ++c) ring_vo[6 * q + c] = vo6[6 * r + c];
  } else if (r - n < (long long)max_win * T) {
    r -= n;
    const int w = (int)(r / T), k = (int)(r % T);
    if (w >= n_win) return;
    const long long f = trackcore::slot_frame(first + w, k, T, skip, total - 1);
    if (f < seen) { fac.copy(f % R, r); return; }
    b = f - seen; q = r;
  } else {
    r -= n + (long long)max_win * T;
    if (r >= (long long)max_win * E) return;
    const int w = (int)(r / E), e = (int)(r % E);
    if (w >= n_win) return;
    int i, j;
    trackcore::vo_pair(e, T, fc, &i, &j);
    const long long fa = trackcore::slot_frame(first + w, i, T, skip, total - 1);
    const long long fb = trackcore::slot_frame(first + w, j, T, skip, total - 1);
    const posemath::Pose6 v = posemath::calc_vo_logq_safe(ld_pose6(track_src(vo6, ring_vo, fa, seen, R)),
                                                          ld_pose6(track_src(vo6, ring_vo, fb, seen, R)));
    const float v6[6] = {v.t.x, v.t.y, v.t.z, v.l.x, v.l.y, v.l.z};
    st_pose7(v6, vos7 + 7 * r);
    return;
  }
  fac.form(b, ring, q);
}

// One thread per completed window: its optimised middle slot, translations un-normalised as _window_errors does
// (un = 0: kept), into out row w; thread 0 advances the frame counter by the call's n frames.  With now (a zero-lag
// call: n windows, the last n_win of them completed) thread w also writes window w's last slot into now row w, and the
// completed window n - n_win + j feeds out row j.
template <class F>
__global__ void __launch_bounds__(128)
k_track_emit(F fac, TrackDev* __restrict__ st, const int* __restrict__ n_win_dev, int n, int T, int un, double m0,
             double m1, double m2, double s0, double s1, double s2, double* __restrict__ out,
             double* __restrict__ now) {
  pdl_prologue();
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const int n_win = *n_win_dev;
  if (w == 0) st->seen += n;
  const double ms[3] = {m0, m1, m2}, ss[3] = {s0, s1, s2};
  const long long mid = (long long)w * T + T / 2, last = (long long)w * T + T - 1;
  if (now == nullptr) {
    if (w < n_win) fac.row(mid, un, ms, ss, out + F::kRow * (long long)w);
    return;
  }
  if (w >= n) return;
  fac.row(last, un, ms, ss, now + F::kRow * (long long)w);
  const int lead = n - n_win;
  if (w >= lead) fac.row(mid, un, ms, ss, out + F::kRow * (long long)(w - lead));
}

// ---- multi-stream trackers (mapnet_track_multi_*, inference.MultiTracker; mapnet_track_multi_sample_*,
// inference.SampledMultiTracker): the same windows for n_streams independent sequences, one set of launches per call.
// Per stream: its frames so far and its status word; the rings are [n_streams][R].  The host keeps count of every
// stream and builds one record per frame of a call, so the kernels find every window without reading a counter:
// stream, rank among that stream's frames in the call, that stream's frame count in the call, absolute frame index,
// the output row of the frame's completed window (-1: none yet), and (a per-row field) the record whose completed
// window is output row b (-1 once the call's rows are done).
struct MTrackRec { int stream, rank, count, frame, row, win; };

// one window of a multi-stream call: its stream, centre, the last frame its slots may reach and the stream's first
// frame in this call (slots from there on come from the call's inputs)
struct MWin {
  int s;
  long long c, last, f0;
};

// Window w of a call, false when the call has no window w.  A step's windows are the completed ones in output-row
// order (rec[w].win), a zero-lag step's the one that ends at each record's frame (record w); a flush of stream
// flush_s >= 0 solves that stream's pending windows, clipped at its last frame.
__device__ __forceinline__ bool mtrack_window(const MTrackRec* rec, int B, int w, int now, int flush_s,
                                              const TrackDev* st, int n_streams, long long lag, MWin* o) {
  if (flush_s >= 0) {
    const long long seen = st[flush_s].seen, first = trackcore::first_pending(seen, lag);
    if (w >= seen - first) return false;
    o->s = flush_s; o->c = first + w; o->last = seen - 1; o->f0 = seen;
    return true;
  }
  if (w >= B) return false;
  const int b = now ? w : rec[w].win;
  if (b < 0 || b >= B) return false;
  const MTrackRec r = rec[b];
  if (r.stream < 0 || r.stream >= n_streams) return false;
  o->s = r.stream;
  o->c = trackcore::now_first(r.frame, lag);       // frame (f - lag)'s window ends at f
  o->f0 = (long long)r.frame - r.rank;
  o->last = o->f0 + r.count - 1;
  return true;
}

// input row of new frame f of window m's stream: the record of that stream at rank f - f0 (the call's only search)
__device__ __forceinline__ int mtrack_input(const MTrackRec* rec, int B, const MWin& m, long long f) {
  const int rank = (int)(f - m.f0);
  for (int b = 0; b < B; ++b)
    if (rec[b].stream == m.s && rec[b].rank == rank) return b;
  return -1;
}

__device__ __forceinline__ posemath::Pose6 mtrack_vo(const float* vo6, const float* ring_vo, const MTrackRec* rec,
                                                     int B, const MWin& m, long long f, long long R) {
  if (f >= m.f0) {
    const int b = mtrack_input(rec, B, m, f);
    if (b >= 0) return ld_pose6(vo6 + 6LL * b);
    const float nan = __int_as_float(0x7fc00000);   // an inconsistent record table: a visible NaN, no stray read
    const float v6[6] = {nan, nan, nan, nan, nan, nan};
    return ld_pose6(v6);
  }
  return ld_pose6(ring_vo + 6 * (m.s * R + f % R));
}

// k_track_gather for B frames of several streams (records rec) or a flush of stream flush_s: rows 0 .. B-1 write
// the new frames into their streams' rings, then slot (w, k) of window w < max_win, then VO (w, e).  The values are
// k_track_gather's (the factors, calc_vo_logq_safe), so each window is bit for bit the single-stream tracker's.  Thread
// 0 writes the count of windows the PGO and the emit read: the completed windows of a step (the records with a row), B
// for a zero-lag step, the stream's pending windows for a flush.
template <class F>
__global__ void __launch_bounds__(128)
k_track_multi_gather(F fac, const float* __restrict__ vo6, const MTrackRec* __restrict__ rec, int B, int now,
                     int flush_s, const TrackDev* __restrict__ st, int n_streams, int* __restrict__ n_win_dev,
                     float* __restrict__ ring_vo, long long R, int T, int skip, int fc, int max_win,
                     double* __restrict__ vos7) {
  pdl_prologue();
  const long long lag = trackcore::lag(T, skip);
  const int E = fc ? T * (T - 1) / 2 : T - 1;
  long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0) {
    int n = 0;
    if (flush_s >= 0) n = (int)(st[flush_s].seen - trackcore::first_pending(st[flush_s].seen, lag));
    else if (now) n = B;
    else while (n < B && rec[n].win >= 0) ++n;
    *n_win_dev = n;
  }
  // one formation call site for ring and window slots, as in k_track_gather
  const bool ring = r < B;
  long long b, q;
  if (ring) {
    const MTrackRec x = rec[r];
    if (x.stream < 0 || x.stream >= n_streams) return;
    b = r; q = x.stream * R + x.frame % R;
#pragma unroll
    for (int c = 0; c < 6; ++c) ring_vo[6 * q + c] = vo6[6 * r + c];
  } else if (r - B < (long long)max_win * T) {
    r -= B;
    const int w = (int)(r / T), k = (int)(r % T);
    MWin m;
    if (!mtrack_window(rec, B, w, now, flush_s, st, n_streams, lag, &m)) return;
    const long long f = trackcore::slot_frame(m.c, k, T, skip, m.last);
    if (f < m.f0) { fac.copy(m.s * R + f % R, r); return; }
    b = mtrack_input(rec, B, m, f);
    if (b < 0) { fac.nan_slot(r); return; }         // an inconsistent record table: a visible NaN, no stray read
    q = r;
  } else {
    r -= B + (long long)max_win * T;
    if (r >= (long long)max_win * E) return;
    const int w = (int)(r / E), e = (int)(r % E);
    MWin m;
    if (!mtrack_window(rec, B, w, now, flush_s, st, n_streams, lag, &m)) return;
    int i, j;
    trackcore::vo_pair(e, T, fc, &i, &j);
    const long long fa = trackcore::slot_frame(m.c, i, T, skip, m.last);
    const long long fb = trackcore::slot_frame(m.c, j, T, skip, m.last);
    const posemath::Pose6 v = posemath::calc_vo_logq_safe(mtrack_vo(vo6, ring_vo, rec, B, m, fa, R),
                                                          mtrack_vo(vo6, ring_vo, rec, B, m, fb, R));
    const float v6[6] = {v.t.x, v.t.y, v.t.z, v.l.x, v.l.y, v.l.z};
    st_pose7(v6, vos7 + 7 * r);
    return;
  }
  fac.form(b, ring, q);
}

// k_track_emit for several streams: window w's middle slot into out row w (a zero-lag step: into row rec[w].row
// when the window completed a frame, and its last slot into now row w); a window the PGO marked failed (its normal
// matrix, or a slot's S7, not positive definite) sets its own stream's status; the last record of each stream in the
// call sets that stream's frame count.
template <class F>
__global__ void __launch_bounds__(128)
k_track_multi_emit(F fac, const int* __restrict__ win_fail, const MTrackRec* __restrict__ rec, int B, int flush_s,
                   TrackDev* __restrict__ st, int n_streams, const int* __restrict__ n_win_dev, int T, int un,
                   double m0, double m1, double m2, double s0, double s1, double s2, double* __restrict__ out,
                   double* __restrict__ now) {
  pdl_prologue();
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const double ms[3] = {m0, m1, m2}, ss[3] = {s0, s1, s2};
  const long long mid = (long long)w * T + T / 2, last = (long long)w * T + T - 1;
  if (w < B) {
    const MTrackRec q = rec[w];
    const bool ok = q.stream >= 0 && q.stream < n_streams;
    if (ok && q.rank == q.count - 1) st[q.stream].seen = (long long)q.frame + 1;
    if (now != nullptr) {
      if (!ok) return;
      fac.row(last, un, ms, ss, now + F::kRow * (long long)w);
      if (q.row >= 0) fac.row(mid, un, ms, ss, out + F::kRow * (long long)q.row);
      if (win_fail[w]) atomicExch(&st[q.stream].status, 1);
      return;
    }
  }
  if (now != nullptr || w >= *n_win_dev) return;
  int s = flush_s;
  if (s < 0) {
    const int b = rec[w].win;
    s = b >= 0 && b < B ? rec[b].stream : -1;
    if (s < 0 || s >= n_streams) return;
  }
  fac.row(mid, un, ms, ss, out + F::kRow * (long long)w);
  if (win_fail[w]) atomicExch(&st[s].status, 1);
}

// ---- Monte-Carlo evaluation windows (mapnet_eval_sample_*, inference.evaluate_sequence(samples=S)): every frame's
// S-draw mean [6] and covariance [36] once, shared by every window slot that holds it, as the sampled trackers share
// them.  One thread per row: slot r < n_rows gets the factor (p7, S7) of frame row slot[r], formed by SampleFactor as
// the tracker forms it into its rings (bit for bit), and VO k the row k_eval_windows writes.
__global__ void __launch_bounds__(128)
k_eval_sample_windows(SampleFactor fac, const float* __restrict__ vo_poses, const int* __restrict__ slot, int n_rows,
                      const TargRow* __restrict__ vo_rows, int n_vo, double* __restrict__ vos7) {
  pdl_prologue();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n_rows) fac.form(slot[r], false, r);
  else if (r < n_rows + n_vo) eval_vo(vo_poses, vo_rows[r - n_rows], vos7 + 7LL * (r - n_rows));
}

// One thread per item i: its estimate as a kTrackSampleRow row (track_sample_row: pose7 un-normalised as
// _window_errors does, D cov D, t_std, q_std_deg) -- slot `keep` of its optimised window (opt7 / post36 rows i*T + keep)
// or, without a pose graph (opt7 null), the draws' own mean and covariance of frame row slot[i] -- its target (st_pose7
// of poses[frame[i]], un-normalised alike) and calibcore::score of the row's pose7 and covariance against the target.
__global__ void __launch_bounds__(128)
k_eval_sample_emit(const double* __restrict__ mean, const double* __restrict__ cov, const double* __restrict__ opt7,
                   const double* __restrict__ post36, int T, int keep, const float* __restrict__ poses,
                   const int* __restrict__ frame, const int* __restrict__ slot, int n, int un, double m0, double m1,
                   double m2, double s0, double s1, double s2, double* __restrict__ out, double* __restrict__ targ7,
                   double* __restrict__ d2, double* __restrict__ u, double* __restrict__ nll) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double ms[3] = {m0, m1, m2}, ss[3] = {s0, s1, s2};
  double* o = out + (long long)kTrackSampleRow * i;
  if (opt7 != nullptr) {
    const long long r = (long long)i * T + keep;
    track_sample_row(opt7 + 7 * r, post36 + 36 * r, un, ms, ss, o);
  } else {
    double mu[6], p7[7];
    for (int c = 0; c < 6; ++c) mu[c] = mean[6LL * slot[i] + c];
    sample_pose7(mu, p7);
    track_sample_row(p7, cov + 36LL * slot[i], un, ms, ss, o);
  }
  double t7[7];
  st_pose7(poses + 6LL * frame[i], t7);
  double* tg = targ7 + 7LL * i;
  track_emit_pose(t7, un, ms, ss, tg);
  calibcore::score(o, tg, o + 7, d2 + 3LL * i, u + 3LL * i, nll + i);
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

// the checks both Monte-Carlo evaluation entry points share: the frame rows' count, every slot row and every frame or
// VO pose index inside its table
static int eval_sample_rows(const char* who, int n_pred, int n_poses, const int32_t* frame, const int32_t* slot,
                            int n_rows, const int32_t* vo_rows, int n_vo) {
  for (int r = 0; r < n_rows; ++r) {
    MN_CHECK((frame == nullptr || (frame[r] >= 0 && frame[r] < n_poses)) && slot[r] >= 0 && slot[r] < n_pred,
             "%s: row %d = (frame %d, slot %d) outside the %d poses / %d frame rows", who, r,
             frame != nullptr ? frame[r] : 0, slot[r], n_poses, n_pred);
  }
  for (int k = 0; k < 2 * n_vo; ++k)
    MN_CHECK(vo_rows[k] >= 0 && vo_rows[k] < n_poses, "%s: VO row %d = (%d, %d) outside the %d poses", who, k / 2,
             vo_rows[k & ~1], vo_rows[k | 1], n_poses);
  return 0;
}

int mapnet_eval_sample_windows(const double* mean6, const double* cov36, int n_pred, double sax, double saq,
                               const float* vo_poses, int n_poses, const int32_t* slot, int n_rows,
                               const int32_t* vo_rows, int n_vo, double* p7, double* s7, double* vos7, void* stream) {
  MN_CHECK(mean6 != nullptr && cov36 != nullptr && slot != nullptr && p7 != nullptr && s7 != nullptr,
           "eval_sample_windows: null argument");
  MN_CHECK(n_rows >= 1 && n_pred >= 1 && n_poses >= 1 && n_vo >= 0, "eval_sample_windows: bad count");
  MN_CHECK(sax > 0 && saq > 0, "eval_sample_windows: sax = %g and saq = %g must be positive", sax, saq);
  MN_CHECK(n_vo == 0 || (vo_poses != nullptr && vo_rows != nullptr && vos7 != nullptr),
           "eval_sample_windows: %d VO rows need vo_poses, vo_rows and vos7", n_vo);
  MN_CHECK((long long)n_rows + n_vo < (1LL << 31), "eval_sample_windows: %d + %d rows", n_rows, n_vo);
  MN_TRY(eval_sample_rows("eval_sample_windows", n_pred, n_poses, nullptr, slot, n_rows, vo_rows, n_vo));
  MN_CHECK(device_memory(mean6) && device_memory(cov36) && device_memory(p7) && device_memory(s7) &&
           (n_vo == 0 || (device_memory(vo_poses) && device_memory(vos7))),
           "eval_sample_windows: tensors must be device memory");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t bytes = ((size_t)n_rows + 2 * (size_t)n_vo) * sizeof(int32_t);
  int32_t* d = nullptr;                // the index tables, stream-ordered: freed once the kernel has read them
  MN_CUDA(cudaMallocAsync((void**)&d, bytes, st));
  MN_CUDA(cudaMemcpyAsync(d, slot, (size_t)n_rows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (n_vo > 0) MN_CUDA(cudaMemcpyAsync(d + n_rows, vo_rows, 2 * (size_t)n_vo * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  MN_LAUNCH(k_eval_sample_windows, (int)cdiv((long long)n_rows + n_vo, 128), 128, 0, st,
            SampleFactor(mean6, cov36, sax, saq, p7, s7), vo_poses, (const int*)d, n_rows,
            (const TargRow*)(d + n_rows), n_vo, vos7);
  MN_LAUNCH_CHECK();
  MN_CUDA(cudaFreeAsync(d, st));
  return 0;
}

int mapnet_eval_sample_emit(const double* mean6, const double* cov36, int n_pred, const double* opt7,
                            const double* post36, int T, int keep, const float* poses, int n_poses,
                            const int32_t* frame, const int32_t* slot, int n, const double* pose_m3,
                            const double* pose_s3, double* out, double* targ7, double* d2, double* u, double* nll,
                            void* stream) {
  MN_CHECK(poses != nullptr && frame != nullptr && out != nullptr && targ7 != nullptr && d2 != nullptr &&
           u != nullptr && nll != nullptr, "eval_sample_emit: null argument");
  MN_CHECK(opt7 != nullptr ? post36 != nullptr : (mean6 != nullptr && cov36 != nullptr && slot != nullptr),
           "eval_sample_emit: need opt7 and post36, or mean6, cov36 and slot");
  MN_CHECK(n >= 1 && n_poses >= 1 && (opt7 != nullptr || n_pred >= 1), "eval_sample_emit: bad count");
  MN_CHECK(T >= 1 && keep >= 0 && keep < T && (long long)n * T < (1LL << 31),
           "eval_sample_emit: slot %d of windows of %d outside the window", keep, T);
  MN_CHECK((pose_m3 == nullptr) == (pose_s3 == nullptr), "eval_sample_emit: pose_m3 and pose_s3 go together");
  if (opt7 != nullptr) {
    for (int i = 0; i < n; ++i)
      MN_CHECK(frame[i] >= 0 && frame[i] < n_poses, "eval_sample_emit: item %d: frame %d outside the %d poses", i,
               frame[i], n_poses);
  } else {
    MN_TRY(eval_sample_rows("eval_sample_emit", n_pred, n_poses, frame, slot, n, nullptr, 0));
  }
  MN_CHECK(device_memory(poses) && device_memory(out) && device_memory(targ7) && device_memory(d2) &&
           device_memory(u) && device_memory(nll) &&
           (opt7 != nullptr ? device_memory(opt7) && device_memory(post36) : device_memory(mean6) && device_memory(cov36)),
           "eval_sample_emit: tensors must be device memory");
  cudaStream_t st = (cudaStream_t)stream;
  const int un = pose_m3 != nullptr;
  const size_t rows = opt7 != nullptr ? 1 : 2;
  int32_t* d = nullptr;                // frame (and slot) of every item, stream-ordered as in mapnet_eval_windows
  MN_CUDA(cudaMallocAsync((void**)&d, rows * (size_t)n * sizeof(int32_t), st));
  MN_CUDA(cudaMemcpyAsync(d, frame, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (opt7 == nullptr) MN_CUDA(cudaMemcpyAsync(d + n, slot, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  MN_LAUNCH(k_eval_sample_emit, (int)cdiv(n, 128), 128, 0, st, mean6, cov36, opt7, post36, T, keep, poses,
            (const int*)d, opt7 != nullptr ? nullptr : (const int*)(d + n), n, un, un ? pose_m3[0] : 0.0,
            un ? pose_m3[1] : 0.0, un ? pose_m3[2] : 0.0, un ? pose_s3[0] : 1.0, un ? pose_s3[1] : 1.0,
            un ? pose_s3[2] : 1.0, out, targ7, d2, u, nll);
  MN_LAUNCH_CHECK();
  MN_CUDA(cudaFreeAsync(d, st));
  return 0;
}

}  // extern "C"

// checks a tracker's arguments (messages prefixed with `who`) and fills c; nothing is allocated or launched
static int track_config(TrackCfg* c, const char* who, int T, int skip, int fc_vos, int max_batch, const double* sigmas4,
                        const double* pose_m3, const double* pose_s3) {
  MN_CHECK(T >= 2 && T <= 16, "%s: windows of %d frames outside [2, 16]", who, T);
  MN_CHECK(skip >= 1 && max_batch >= 1, "%s: skip = %d and max_batch = %d must be >= 1", who, skip, max_batch);
  for (int k = 0; k < 4; ++k) MN_CHECK(sigmas4[k] > 0, "%s: sigma %d = %g must be positive", who, k, sigmas4[k]);
  MN_CHECK((pose_m3 == nullptr) == (pose_s3 == nullptr), "%s: pose_m3 and pose_s3 go together", who);
  const long long lag = trackcore::lag(T, skip), R = trackcore::ring_frames(max_batch, T, skip);
  MN_CHECK(R < (1LL << 26), "%s: a ring of %lld frames", who, R);
  int ndev = 0;
  MN_CHECK(cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0, "%s: no CUDA device (this library has no CPU fallback)",
           who);
  MN_TRY(pgo_prepare());
  c->T = T; c->skip = skip; c->fc = fc_vos ? 1 : 0; c->max_batch = max_batch;
  c->E = c->fc ? T * (T - 1) / 2 : T - 1;
  c->lag = lag; c->R = R;
  c->max_win = (int)(lag > max_batch ? lag : max_batch);
  pgo_weights(sigmas4[0], sigmas4[1], sigmas4[2], sigmas4[3], c->w4);
  c->un = pose_m3 != nullptr;
  for (int k = 0; k < 3; ++k) { c->m[k] = c->un ? pose_m3[k] : 0.0; c->s[k] = c->un ? pose_s3[k] : 1.0; }
  return 0;
}

struct mapnet_track : TrackHandle {};
struct mapnet_track_sample : TrackHandle {};
struct mapnet_track_multi : TrackHandle {};
struct mapnet_track_multi_sample : TrackHandle {};

template <class H>
static int track_destroy(H* h) {
  if (h == nullptr) return 0;
  cudaFree(h->st); cudaFree(h->n_win); cudaFree(h->ring7); cudaFree(h->ring49); cudaFree(h->ring_vo);
  cudaFree(h->win7); cudaFree(h->win49); cudaFree(h->vos7); cudaFree(h->opt7); cudaFree(h->cov36);
  delete h;
  return 0;
}

// every tracker's create: the checks, then one allocation per buffer, with the byte count in the failure message of
// the multi-stream trackers (multi); sampled trackers also hold the p / S7 rings and the posterior covariances
template <class H>
static int track_create(H** out, const char* who, bool multi, bool sampled, int n_streams, int T, int skip,
                        int fc_vos, int max_batch, const double* sigmas4, const double* pose_m3,
                        const double* pose_s3) {
  MN_CHECK(out != nullptr && sigmas4 != nullptr, "%s: null argument", who);
  *out = nullptr;
  MN_CHECK(n_streams >= 1 && n_streams <= MAPNET_TRACK_MAX_STREAMS, "%s: %d streams outside [1, %d]", who, n_streams,
           MAPNET_TRACK_MAX_STREAMS);
  TrackCfg c;
  MN_TRY(track_config(&c, who, T, skip, fc_vos, max_batch, sigmas4, pose_m3, pose_s3));
  if (sampled) MN_TRY(pgo_cov_prepare());
  const size_t W = (size_t)c.max_win, WT = W * c.T, ring = (size_t)n_streams * (size_t)c.R;
  const size_t P = sampled ? 7 + 49 : 7;                     // doubles per ring frame and window slot of the factors
  const size_t frame_bytes = P * sizeof(double) + 6 * sizeof(float);       // 472 B per sampled ring frame
  const size_t bytes = ring * frame_bytes + WT * (P + 7 + (sampled ? 36 : 0)) * sizeof(double) +
                       W * c.E * 7 * sizeof(double) + (size_t)n_streams * sizeof(TrackDev) + (W + 1) * sizeof(int);
  MN_CHECK(ring < (1ull << 31), "%s: %d streams x rings of %lld frames = %zu frames (%.3f GB) exceed 2^31 ring frames",
           who, n_streams, c.R, ring, bytes / 1e9);
  H* h = new H();
  static_cast<TrackCfg&>(*h) = c;
  h->n_streams = n_streams;
  h->sax = sigmas4[0]; h->saq = sigmas4[1];
  bool ok = cudaMalloc((void**)&h->st, (size_t)n_streams * sizeof(TrackDev)) == cudaSuccess &&
            cudaMalloc((void**)&h->n_win, (W + 1) * sizeof(int)) == cudaSuccess &&
            cudaMalloc((void**)&h->ring7, ring * 7 * sizeof(double)) == cudaSuccess &&
            (!sampled || cudaMalloc((void**)&h->ring49, ring * 49 * sizeof(double)) == cudaSuccess) &&
            cudaMalloc((void**)&h->ring_vo, ring * 6 * sizeof(float)) == cudaSuccess &&
            cudaMalloc((void**)&h->win7, WT * 7 * sizeof(double)) == cudaSuccess &&
            (!sampled || cudaMalloc((void**)&h->win49, WT * 49 * sizeof(double)) == cudaSuccess) &&
            cudaMalloc((void**)&h->vos7, W * c.E * 7 * sizeof(double)) == cudaSuccess &&
            cudaMalloc((void**)&h->opt7, WT * 7 * sizeof(double)) == cudaSuccess &&
            (!sampled || cudaMalloc((void**)&h->cov36, WT * 36 * sizeof(double)) == cudaSuccess) &&
            cudaMemset(h->st, 0, (size_t)n_streams * sizeof(TrackDev)) == cudaSuccess &&
            cudaMemset(h->n_win, 0, (W + 1) * sizeof(int)) == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    if (!multi)
      set_last_error("%s: device allocation of a ring of %lld frames and %d windows failed", who, c.R, c.max_win);
    else if (!sampled)
      set_last_error("%s: device allocation of %zu bytes (%d streams x rings of %lld frames, %d windows) failed", who,
                     bytes, n_streams, c.R, c.max_win);
    else
      set_last_error("%s: device allocation of %zu bytes (%d streams x rings of %lld frames of %zu B, %d windows) "
                     "failed", who, bytes, n_streams, c.R, frame_bytes, c.max_win);
    track_destroy(h);
    return 1;
  }
  h->win_fail = h->n_win + 1;
  *out = h;
  return 0;
}

// stream s (every stream when s = -1) starts a new sequence, stream-ordered
static int track_reset(TrackHandle* h, int s, cudaStream_t stream) {
  const size_t n = s < 0 ? (size_t)h->n_streams : 1;
  MN_CUDA(cudaMemsetAsync(h->st + (s < 0 ? 0 : s), 0, n * sizeof(TrackDev), stream));
  return 0;
}

// the Cauchy scale c of every window's absolute factors from now on; refused once the handle has enqueued a step or
// a flush, so every window of the handle's life (and every graph that captured its launches) has the same loss
static int track_set_robust(TrackHandle* h, const char* who, double c) {
  MN_CHECK(h != nullptr, "%s: null handle", who);
  MN_CHECK(c > 0 && isfinite(c), "%s: the Cauchy scale c = %g must be finite and positive", who, c);
  MN_CHECK(!h->started, "%s: the handle has already stepped; set the robust loss before the first step", who);
  h->robust_c = c;
  return 0;
}

static int track_status(TrackHandle* h, int s, int64_t* frames_seen, int* failed, cudaStream_t stream) {
  TrackDev d;
  MN_CUDA(cudaMemcpyAsync(&d, h->st + s, sizeof(TrackDev), cudaMemcpyDeviceToHost, stream));
  MN_CUDA(cudaStreamSynchronize(stream));
  if (frames_seen != nullptr) *frames_seen = d.seen;
  if (failed != nullptr) *failed = d.status;
  return 0;
}

// the three launches of a single-stream call: n new frames (a step) or none (flush), out [max_win][kRow]; with now
// [n][kRow] a zero-lag step, which solves all n of its windows, so the PGO needs no device count
template <class F>
static int track_launch(TrackHandle* h, F fac, const float* vo6, int n, int flush, double* out, double* now,
                        cudaStream_t st) {
  const int nw = flush ? (int)(h->lag < h->max_win ? h->lag : h->max_win) : n;   // the grid's windows
  const long long rows = n + (long long)nw * (h->T + h->E);
  h->started = true;
  MN_LAUNCH(k_track_gather<F>, cdiv(rows, 128), 128, 0, st, fac, vo6, n, flush, now != nullptr ? 1 : 0,
            (const TrackDev*)h->st, h->n_win, h->ring_vo, h->R, h->T, h->skip, h->fc, nw, h->vos7);
  MN_LAUNCH_CHECK();
  MN_TRY(fac.pgo(*h, nw, &h->st->status, now != nullptr ? nullptr : h->n_win, nullptr, st));
  MN_LAUNCH(k_track_emit<F>, cdiv(nw, 128), 128, 0, st, fac, h->st, (const int*)h->n_win, n, h->T, h->un, h->m[0],
            h->m[1], h->m[2], h->s[0], h->s[1], h->s[2], out, now);
  MN_LAUNCH_CHECK();
  return 0;
}

// the three launches of a multi-stream call: B frames with records rec (a step; with now a zero-lag step, which
// solves all B of its windows) or a flush of stream flush_s (B = 0); out [max_win][kRow], now [B][kRow] or null
template <class F>
static int track_multi_launch(TrackHandle* h, F fac, const float* vo6, const MTrackRec* rec, int B, int flush_s,
                              double* out, double* now, cudaStream_t st) {
  const int nw = flush_s >= 0 ? (int)(h->lag < h->max_win ? h->lag : h->max_win) : B;    // the grid's windows
  const int zl = now != nullptr ? 1 : 0;
  const long long rows = B + (long long)nw * (h->T + h->E);
  h->started = true;
  MN_LAUNCH(k_track_multi_gather<F>, cdiv(rows, 128), 128, 0, st, fac, vo6, rec, B, zl, flush_s,
            (const TrackDev*)h->st, h->n_streams, h->n_win, h->ring_vo, h->R, h->T, h->skip, h->fc, nw, h->vos7);
  MN_LAUNCH_CHECK();
  MN_TRY(fac.pgo(*h, nw, nullptr, zl ? nullptr : h->n_win, h->win_fail, st));
  MN_LAUNCH(k_track_multi_emit<F>, cdiv(nw > B ? nw : B, 128), 128, 0, st, fac, (const int*)h->win_fail, rec, B,
            flush_s, h->st, h->n_streams, (const int*)h->n_win, h->T, h->un, h->m[0], h->m[1], h->m[2], h->s[0],
            h->s[1], h->s[2], out, now);
  MN_LAUNCH_CHECK();
  return 0;
}

extern "C" {

int mapnet_track_create(mapnet_track_t** out, int T, int skip, int fc_vos, int max_batch, const double* sigmas4,
                        const double* pose_m3, const double* pose_s3) {
  return track_create(out, "track_create", false, false, 1, T, skip, fc_vos, max_batch, sigmas4, pose_m3, pose_s3);
}

int mapnet_track_step(mapnet_track_t* h, const float* pred6, const float* vo6, int B, double* out7, void* stream) {
  MN_CHECK(h != nullptr, "track_step: null handle");
  MN_CHECK(pred6 != nullptr && vo6 != nullptr && out7 != nullptr, "track_step: null argument");
  MN_CHECK(B >= 1 && B <= h->max_batch, "track_step: %d frames outside [1, max_batch=%d]", B, h->max_batch);
  return track_launch(h, PointFactor(*h, pred6), vo6, B, 0, out7, nullptr, (cudaStream_t)stream);
}

int mapnet_track_step_now(mapnet_track_t* h, const float* pred6, const float* vo6, int B, double* out7, double* now7,
                          void* stream) {
  MN_CHECK(h != nullptr, "track_step_now: null handle");
  MN_CHECK(pred6 != nullptr && vo6 != nullptr && out7 != nullptr && now7 != nullptr, "track_step_now: null argument");
  MN_CHECK(B >= 1 && B <= h->max_batch, "track_step_now: %d frames outside [1, max_batch=%d]", B, h->max_batch);
  return track_launch(h, PointFactor(*h, pred6), vo6, B, 0, out7, now7, (cudaStream_t)stream);
}

int mapnet_track_flush(mapnet_track_t* h, double* out7, void* stream) {
  MN_CHECK(h != nullptr, "track_flush: null handle");
  MN_CHECK(out7 != nullptr, "track_flush: null argument");
  if (h->lag == 0) return 0;                 // every window was complete when its last frame arrived
  return track_launch(h, PointFactor(*h, nullptr), nullptr, 0, 1, out7, nullptr, (cudaStream_t)stream);
}

int mapnet_track_reset(mapnet_track_t* h, void* stream) {
  MN_CHECK(h != nullptr, "track_reset: null handle");
  return track_reset(h, -1, (cudaStream_t)stream);
}

int mapnet_track_status(mapnet_track_t* h, int64_t* frames_seen, int* failed, void* stream) {
  MN_CHECK(h != nullptr, "track_status: null handle");
  return track_status(h, 0, frames_seen, failed, (cudaStream_t)stream);
}

int mapnet_track_set_robust(mapnet_track_t* h, double c) { return track_set_robust(h, "track_set_robust", c); }

int mapnet_track_destroy(mapnet_track_t* h) { return track_destroy(h); }

int mapnet_track_sample_create(mapnet_track_sample_t** out, int T, int skip, int fc_vos, int max_batch,
                               const double* sigmas4, const double* pose_m3, const double* pose_s3) {
  return track_create(out, "track_sample_create", false, true, 1, T, skip, fc_vos, max_batch, sigmas4, pose_m3,
                      pose_s3);
}

int mapnet_track_sample_step(mapnet_track_sample_t* h, const double* mean6, const double* cov36, const float* vo6, int B,
                             double* out, void* stream) {
  MN_CHECK(h != nullptr, "track_sample_step: null handle");
  MN_CHECK(mean6 != nullptr && cov36 != nullptr && vo6 != nullptr && out != nullptr, "track_sample_step: null argument");
  MN_CHECK(B >= 1 && B <= h->max_batch, "track_sample_step: %d frames outside [1, max_batch=%d]", B, h->max_batch);
  return track_launch(h, SampleFactor(*h, mean6, cov36), vo6, B, 0, out, nullptr, (cudaStream_t)stream);
}

int mapnet_track_sample_step_now(mapnet_track_sample_t* h, const double* mean6, const double* cov36, const float* vo6,
                                 int B, double* out, double* now, void* stream) {
  MN_CHECK(h != nullptr, "track_sample_step_now: null handle");
  MN_CHECK(mean6 != nullptr && cov36 != nullptr && vo6 != nullptr && out != nullptr && now != nullptr,
           "track_sample_step_now: null argument");
  MN_CHECK(B >= 1 && B <= h->max_batch, "track_sample_step_now: %d frames outside [1, max_batch=%d]", B, h->max_batch);
  return track_launch(h, SampleFactor(*h, mean6, cov36), vo6, B, 0, out, now, (cudaStream_t)stream);
}

int mapnet_track_sample_flush(mapnet_track_sample_t* h, double* out, void* stream) {
  MN_CHECK(h != nullptr, "track_sample_flush: null handle");
  MN_CHECK(out != nullptr, "track_sample_flush: null argument");
  if (h->lag == 0) return 0;
  return track_launch(h, SampleFactor(*h, nullptr, nullptr), nullptr, 0, 1, out, nullptr, (cudaStream_t)stream);
}

int mapnet_track_sample_reset(mapnet_track_sample_t* h, void* stream) {
  MN_CHECK(h != nullptr, "track_sample_reset: null handle");
  return track_reset(h, -1, (cudaStream_t)stream);
}

int mapnet_track_sample_status(mapnet_track_sample_t* h, int64_t* frames_seen, int* failed, void* stream) {
  MN_CHECK(h != nullptr, "track_sample_status: null handle");
  return track_status(h, 0, frames_seen, failed, (cudaStream_t)stream);
}

int mapnet_test_sample_factor(const double* mean6, const double* cov36, int64_t n, double sax, double saq, double* p7,
                              double* s7, void* stream) {
  MN_CHECK(mean6 != nullptr && cov36 != nullptr && p7 != nullptr && s7 != nullptr && n >= 1,
           "test_sample_factor: bad argument");
  MN_CHECK(sax > 0 && saq > 0, "test_sample_factor: sax = %g and saq = %g must be positive", sax, saq);
  MN_LAUNCH(k_test_sample_factor, cdiv(n, 128), 128, 0, (cudaStream_t)stream, mean6, cov36, (long long)n, sax, saq, p7,
            s7);
  MN_LAUNCH_CHECK();
  return 0;
}

int mapnet_track_sample_set_robust(mapnet_track_sample_t* h, double c) { return track_set_robust(h, "track_sample_set_robust", c); }

int mapnet_track_sample_destroy(mapnet_track_sample_t* h) { return track_destroy(h); }

int mapnet_track_multi_create(mapnet_track_multi_t** out, int n_streams, int T, int skip, int fc_vos, int max_batch,
                              const double* sigmas4, const double* pose_m3, const double* pose_s3) {
  return track_create(out, "track_multi_create", true, false, n_streams, T, skip, fc_vos, max_batch, sigmas4, pose_m3,
                      pose_s3);
}

int mapnet_track_multi_step(mapnet_track_multi_t* h, const float* pred6, const float* vo6, const int32_t* rec, int B,
                            double* out7, double* now7, void* stream) {
  MN_CHECK(h != nullptr, "track_multi_step: null handle");
  MN_CHECK(pred6 != nullptr && vo6 != nullptr && rec != nullptr && out7 != nullptr, "track_multi_step: null argument");
  MN_CHECK(B >= 1 && B <= h->max_batch, "track_multi_step: %d frames outside [1, max_batch=%d]", B, h->max_batch);
  return track_multi_launch(h, PointFactor(*h, pred6), vo6, (const MTrackRec*)rec, B, -1, out7, now7,
                            (cudaStream_t)stream);
}

int mapnet_track_multi_flush(mapnet_track_multi_t* h, int s, double* out7, void* stream) {
  MN_CHECK(h != nullptr, "track_multi_flush: null handle");
  MN_CHECK(out7 != nullptr, "track_multi_flush: null argument");
  MN_CHECK(s >= 0 && s < h->n_streams, "track_multi_flush: stream %d outside [0, %d)", s, h->n_streams);
  if (h->lag == 0) return 0;                 // every window was complete when its last frame arrived
  return track_multi_launch(h, PointFactor(*h, nullptr), nullptr, nullptr, 0, s, out7, nullptr, (cudaStream_t)stream);
}

int mapnet_track_multi_reset(mapnet_track_multi_t* h, int s, void* stream) {
  MN_CHECK(h != nullptr, "track_multi_reset: null handle");
  MN_CHECK(s >= -1 && s < h->n_streams, "track_multi_reset: stream %d outside [-1, %d)", s, h->n_streams);
  return track_reset(h, s, (cudaStream_t)stream);
}

int mapnet_track_multi_status(mapnet_track_multi_t* h, int s, int64_t* frames_seen, int* failed, void* stream) {
  MN_CHECK(h != nullptr, "track_multi_status: null handle");
  MN_CHECK(s >= 0 && s < h->n_streams, "track_multi_status: stream %d outside [0, %d)", s, h->n_streams);
  return track_status(h, s, frames_seen, failed, (cudaStream_t)stream);
}

int mapnet_track_multi_set_robust(mapnet_track_multi_t* h, double c) { return track_set_robust(h, "track_multi_set_robust", c); }

int mapnet_track_multi_destroy(mapnet_track_multi_t* h) { return track_destroy(h); }

int mapnet_track_multi_sample_create(mapnet_track_multi_sample_t** out, int n_streams, int T, int skip, int fc_vos,
                                     int max_batch, const double* sigmas4, const double* pose_m3,
                                     const double* pose_s3) {
  return track_create(out, "track_multi_sample_create", true, true, n_streams, T, skip, fc_vos, max_batch, sigmas4,
                      pose_m3, pose_s3);
}

int mapnet_track_multi_sample_step(mapnet_track_multi_sample_t* h, const double* mean6, const double* cov36,
                                   const float* vo6, const int32_t* rec, int B, double* out, double* now,
                                   void* stream) {
  MN_CHECK(h != nullptr, "track_multi_sample_step: null handle");
  MN_CHECK(mean6 != nullptr && cov36 != nullptr && vo6 != nullptr && rec != nullptr && out != nullptr,
           "track_multi_sample_step: null argument");
  MN_CHECK(B >= 1 && B <= h->max_batch, "track_multi_sample_step: %d frames outside [1, max_batch=%d]", B,
           h->max_batch);
  return track_multi_launch(h, SampleFactor(*h, mean6, cov36), vo6, (const MTrackRec*)rec, B, -1, out, now,
                            (cudaStream_t)stream);
}

int mapnet_track_multi_sample_flush(mapnet_track_multi_sample_t* h, int s, double* out, void* stream) {
  MN_CHECK(h != nullptr, "track_multi_sample_flush: null handle");
  MN_CHECK(out != nullptr, "track_multi_sample_flush: null argument");
  MN_CHECK(s >= 0 && s < h->n_streams, "track_multi_sample_flush: stream %d outside [0, %d)", s, h->n_streams);
  if (h->lag == 0) return 0;                 // every window was complete when its last frame arrived
  return track_multi_launch(h, SampleFactor(*h, nullptr, nullptr), nullptr, nullptr, 0, s, out, nullptr,
                            (cudaStream_t)stream);
}

int mapnet_track_multi_sample_reset(mapnet_track_multi_sample_t* h, int s, void* stream) {
  MN_CHECK(h != nullptr, "track_multi_sample_reset: null handle");
  MN_CHECK(s >= -1 && s < h->n_streams, "track_multi_sample_reset: stream %d outside [-1, %d)", s, h->n_streams);
  return track_reset(h, s, (cudaStream_t)stream);
}

int mapnet_track_multi_sample_status(mapnet_track_multi_sample_t* h, int s, int64_t* frames_seen, int* failed,
                                     void* stream) {
  MN_CHECK(h != nullptr, "track_multi_sample_status: null handle");
  MN_CHECK(s >= 0 && s < h->n_streams, "track_multi_sample_status: stream %d outside [0, %d)", s, h->n_streams);
  return track_status(h, s, frames_seen, failed, (cudaStream_t)stream);
}

int mapnet_track_multi_sample_set_robust(mapnet_track_multi_sample_t* h, double c) { return track_set_robust(h, "track_multi_sample_set_robust", c); }

int mapnet_track_multi_sample_destroy(mapnet_track_multi_sample_t* h) { return track_destroy(h); }

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
