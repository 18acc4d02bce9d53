// Pose / log-quaternion math of the relative-pose loss, forward AND hand-derived
// reverse mode, as plain fp32 inline functions usable from device code (loss.cu)
// and from a host-only test shim (tests/_hostmath.cpp) so the derivatives are
// checked on CPU against the reference's autograd goldens.
//
// Follows /root/reference/common/pose_utils.py operation by operation:
//   qexp_t :73-84   qlog_t :86-96   qmult :44-62   qinv :64-71
//   rotate_vec_by_q :120-132   compose_pose_quaternion :134-146
//   invert_pose_quaternion :148-157   calc_vo :159-165   calc_vo_logq :167-179
// clamp() passes gradient only inside its range and norm()'s sub-gradient at 0
// is 0, as torch autograd defines them (SURVEY.md section 7 hard part 7).
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define PM_HD __host__ __device__ __forceinline__
#else
#define PM_HD static inline
#endif

namespace posemath {

struct V3 { float x, y, z; };
struct Q4 { float s; V3 v; };

PM_HD V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
PM_HD V3 add(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
PM_HD V3 sub(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
PM_HD V3 mul(V3 a, float k) { return v3(a.x * k, a.y * k, a.z * k); }
PM_HD V3 divs(V3 a, float k) { return v3(a.x / k, a.y / k, a.z / k); }
PM_HD V3 neg(V3 a) { return v3(-a.x, -a.y, -a.z); }
PM_HD float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
PM_HD V3 cross(V3 a, V3 b) {
  return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
PM_HD float norm3(V3 a) { return sqrtf(a.x * a.x + a.y * a.y + a.z * a.z); }

// ---- qexp_t ----------------------------------------------------------------
PM_HD Q4 qexp(V3 l) {
  float m = norm3(l);
  float n = fmaxf(m, 1e-8f);
  Q4 q;
  q.s = cosf(n);
  q.v = divs(mul(l, sinf(n)), n);
  return q;
}
// returns d/dl given upstream gq
PM_HD V3 qexp_bwd(V3 l, Q4 gq) {
  float m = norm3(l);
  float n = fmaxf(m, 1e-8f);
  float sn = sinf(n), cn = cosf(n);
  V3 u = mul(l, sn);
  V3 gu = divs(gq.v, n);
  float gn = -dot(gq.v, u) / (n * n);
  V3 gl = mul(gu, sn);
  gn += dot(gu, l) * cn;
  gn += gq.s * (-sn);
  float gm = (m >= 1e-8f) ? gn : 0.0f;         // clamp(min) backward
  if (m > 0.0f) gl = add(gl, mul(divs(l, m), gm));   // norm backward, 0 at the origin
  return gl;
}

// ---- qlog_t ----------------------------------------------------------------
PM_HD V3 qlog(Q4 q) {
  float m = norm3(q.v);
  float n = fmaxf(m, 1e-8f);
  float c = fminf(fmaxf(q.s, -1.0f), 1.0f);
  float a = acosf(c);
  return divs(mul(q.v, a), n);
}
PM_HD Q4 qlog_bwd(Q4 q, V3 go) {
  float m = norm3(q.v);
  float n = fmaxf(m, 1e-8f);
  float c = fminf(fmaxf(q.s, -1.0f), 1.0f);
  float a = acosf(c);
  // o = (q.v * a) / n
  V3 gw = divs(go, n);                       // grad wrt w = q.v * a
  float gn = -dot(go, mul(q.v, a)) / (n * n);
  Q4 g;
  g.v = mul(gw, a);
  float ga = dot(gw, q.v);
  float gm = (m >= 1e-8f) ? gn : 0.0f;
  if (m > 0.0f) g.v = add(g.v, mul(divs(q.v, m), gm));
  float gc = ga * (-(1.0f / sqrtf(1.0f - c * c)));   // acos'; 0 * inf = NaN as in torch
  g.s = (q.s >= -1.0f && q.s <= 1.0f) ? gc : 0.0f;
  return g;
}

// ---- rotate_vec_by_q -------------------------------------------------------
PM_HD V3 rotate(V3 t, Q4 q) {
  V3 b = cross(q.v, t);
  V3 c = mul(cross(q.v, b), 2.0f);
  b = mul(mul(b, 2.0f), q.s);
  return add(add(t, b), c);
}
PM_HD void rotate_bwd(V3 t, Q4 q, V3 g, V3* gt, Q4* gq) {
  V3 b0 = cross(q.v, t);
  // out = t + 2*b0*qs + 2*(qv x b0)
  V3 g_t = g;
  // c = 2 * (qv x b0)
  V3 g_qv = mul(cross(b0, g), 2.0f);
  V3 g_b0 = mul(cross(g, q.v), 2.0f);
  // b = 2*b0*qs
  g_b0 = add(g_b0, mul(g, 2.0f * q.s));
  float g_qs = 2.0f * dot(b0, g);
  // b0 = qv x t
  g_qv = add(g_qv, cross(t, g_b0));
  g_t = add(g_t, cross(g_b0, q.v));
  *gt = g_t;
  gq->s = g_qs;
  gq->v = g_qv;
}

// ---- qmult (Hamilton product + normalize) ----------------------------------
PM_HD Q4 qmult_raw(Q4 a, Q4 b) {
  Q4 r;
  r.s = a.s * b.s - dot(a.v, b.v);
  r.v = add(add(mul(a.v, b.s), mul(b.v, a.s)), cross(a.v, b.v));
  return r;
}
PM_HD float norm4(Q4 q) { return sqrtf(q.s * q.s + q.v.x * q.v.x + q.v.y * q.v.y + q.v.z * q.v.z); }
PM_HD Q4 qmult(Q4 a, Q4 b) {
  Q4 r = qmult_raw(a, b);
  float n = norm4(r);
  Q4 q;
  q.s = r.s / n;
  q.v = divs(r.v, n);
  return q;
}
PM_HD void qmult_bwd(Q4 a, Q4 b, Q4 gq, Q4* ga, Q4* gb) {
  Q4 r = qmult_raw(a, b);
  float n = norm4(r);
  // q = r / n
  float d = gq.s * r.s + dot(gq.v, r.v);
  float gn = -d / (n * n);
  Q4 gr;
  gr.s = gq.s / n + gn * (r.s / n);
  gr.v = add(divs(gq.v, n), mul(divs(r.v, n), gn));
  // raw product
  ga->s = gr.s * b.s + dot(gr.v, b.v);
  gb->s = gr.s * a.s + dot(gr.v, a.v);
  ga->v = add(add(mul(b.v, -gr.s), mul(gr.v, b.s)), cross(b.v, gr.v));
  gb->v = add(add(mul(a.v, -gr.s), mul(gr.v, a.s)), cross(gr.v, a.v));
}

// ---- calc_vo_logq: relative pose of p1 in the frame of p0 -------------------
struct Pose6 { V3 t; V3 l; };

PM_HD Pose6 calc_vo_logq(Pose6 p0, Pose6 p1) {
  Q4 q0 = qexp(p0.l), q1 = qexp(p1.l);
  Q4 q0i; q0i.s = q0.s; q0i.v = neg(q0.v);                // qinv
  V3 tinv = neg(rotate(p0.t, q0i));                        // invert_pose_quaternion
  Q4 q = qmult(q0i, q1);                                   // compose_pose_quaternion
  V3 t = add(tinv, rotate(p1.t, q0i));
  Pose6 o; o.t = t; o.l = qlog(q);
  return o;
}

PM_HD void calc_vo_logq_bwd(Pose6 p0, Pose6 p1, Pose6 go, Pose6* g0, Pose6* g1) {
  Q4 q0 = qexp(p0.l), q1 = qexp(p1.l);
  Q4 q0i; q0i.s = q0.s; q0i.v = neg(q0.v);
  Q4 q = qmult(q0i, q1);
  // qlog
  Q4 gq = qlog_bwd(q, go.l);
  // qmult
  Q4 g_q0i, g_q1;
  qmult_bwd(q0i, q1, gq, &g_q0i, &g_q1);
  // t = tinv + rotate(p1.t, q0i)
  V3 g_t1; Q4 g_qa;
  rotate_bwd(p1.t, q0i, go.t, &g_t1, &g_qa);
  g_q0i.s += g_qa.s; g_q0i.v = add(g_q0i.v, g_qa.v);
  // tinv = -rotate(p0.t, q0i)
  V3 g_t0; Q4 g_qb;
  rotate_bwd(p0.t, q0i, neg(go.t), &g_t0, &g_qb);
  g_q0i.s += g_qb.s; g_q0i.v = add(g_q0i.v, g_qb.v);
  // q0i = (q0.s, -q0.v)
  Q4 g_q0; g_q0.s = g_q0i.s; g_q0.v = neg(g_q0i.v);
  g0->t = g_t0; g0->l = qexp_bwd(p0.l, g_q0);
  g1->t = g_t1; g1->l = qexp_bwd(p1.l, g_q1);
}

// ---- calc_vo_logq_safe (:276-288): the VO targets of MFOnline's validation half ----------------
// qexp_t_safe / qlog_t_safe run numpy's qexp / qlog (:307-327) on float32 rows, so every operation is float32:
// qexp = (cos n, sinc(n / pi) q) with np.sinc(x) = sin(pi x) / (pi x); qlog has no clamp, as the reference.
PM_HD Q4 qexp_safe(V3 l) {
  const float n = sqrtf(l.x * l.x + l.y * l.y + l.z * l.z);
  const float pi = 3.14159265358979323846f;
  const float x = n / pi;
  const float y = pi * (x == 0.0f ? 1.0e-20f : x);
  Q4 q;
  q.s = cosf(n);
  q.v = mul(l, sinf(y) / y);
  return q;
}
PM_HD V3 qlog_safe(Q4 q) {
  if (q.v.x == 0.0f && q.v.y == 0.0f && q.v.z == 0.0f) return v3(0.0f, 0.0f, 0.0f);
  return divs(mul(q.v, acosf(q.s)), norm3(q.v));
}
PM_HD Pose6 calc_vo_logq_safe(Pose6 p0, Pose6 p1) {
  Q4 q0 = qexp_safe(p0.l), q1 = qexp_safe(p1.l);
  Q4 q0i; q0i.s = q0.s; q0i.v = neg(q0.v);                // qinv
  Pose6 o;
  o.t = rotate(sub(p1.t, p0.t), q0i);
  o.l = qlog_safe(qmult(q0i, q1));
  return o;
}

PM_HD float sgnf(float d) { return (d > 0.0f) ? 1.0f : ((d < 0.0f) ? -1.0f : 0.0f); }

}  // namespace posemath
