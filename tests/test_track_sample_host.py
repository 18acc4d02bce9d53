"""Host-side checks of the covariance-weighted pose graph and inference.SampledTracker (no GPU needed): the entry points
are declared, exported and refuse bad arguments before any launch, every SampledTracker argument error is raised
before the device is touched, and a numpy float64 restatement of the factor model (the oracle the GPU tests compare
k_pgo_cov and the tracker against) has Jacobians that match central finite differences and, with no sampled
covariance, the reference's unary factor."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import pgo_oracle as po
from test_track_host import _stub_predictor      # an open Predictor without an engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN = [0.5, 0.44, 0.45]
STD = [0.21, 0.23, 0.22]


# ---- the oracle: numpy float64, dense Jacobians ---------------------------------------------------------------------
def qexp(v):
    n = np.linalg.norm(v)
    return np.concatenate(([math.cos(n)], (math.sin(n) / n) * v)) if n > 0 else np.array([1.0, 0.0, 0.0, 0.0])


def qexp_jac(v):
    """E(v) = d qexp(v) / dv, 4 x 3; g(n) = (n cos n - sin n) / n^3 by its series below n = 0.1"""
    v = np.asarray(v, dtype=np.float64)
    n = np.linalg.norm(v)
    sc = math.sin(n) / n if n > 0 else 1.0
    if n < 0.1:
        g = sum((-1) ** k * 2 * k / math.factorial(2 * k + 1) * n ** (2 * k - 2) for k in range(1, 7))
    else:
        g = (n * math.cos(n) - math.sin(n)) / n ** 3
    return np.vstack((-sc * v[None], sc * np.eye(3) + g * np.outer(v, v)))


def qlog(q):
    u = np.asarray(q[1:], dtype=np.float64)
    s = np.linalg.norm(u)
    return math.atan2(s, q[0]) * u / s if s > 0 else np.zeros(3)


def qlog_jac(q):
    """G(q) = d qlog(q * dq(x)) / dx at x = 0 = Jlog(q) m_rot(q)"""
    w, u = float(q[0]), np.asarray(q[1:], dtype=np.float64)
    s2 = float(u @ u)
    s, n2 = math.sqrt(s2), w * w + s2
    t = s / w if w != 0 else np.inf
    if w > 0 and t < 1e-2:
        f = sum((-1) ** k * t ** (2 * k) / (2 * k + 1) for k in range(6)) / w
        c = sum((-1) ** k * 2 * k / (2 * k + 1) * t ** (2 * k - 2) for k in range(1, 6)) / w ** 3
    else:
        f = math.atan2(s, w) / s
        c = (w / n2 - f) / s2
    Jl = np.hstack(((-u / n2)[:, None], f * np.eye(3) + c * np.outer(u, u)))
    return Jl @ po.m_rot(np.asarray(q, dtype=np.float64))


def factor(mu, sigma, sax, saq):
    """(p [7], S7 [7,7]) of a frame's draws' mean mu [6] and covariance sigma [6,6]"""
    A = np.zeros((7, 6))
    A[:3, :3] = np.eye(3)
    A[3:, 3:] = qexp_jac(mu[3:])
    S7 = A @ sigma @ A.T + np.diag([sax] * 3 + [saq] * 4)
    return np.concatenate((mu[:3], qexp(mu[3:]))), S7


def unary(z, p, S7):
    """(residual [7], Jacobian [7,6] w.r.t. slot (dt, x)) of the absolute factor at slot state z [7]"""
    Ci = np.linalg.inv(np.linalg.cholesky(S7))
    J0 = np.zeros((7, 6))
    J0[:3, :3] = np.eye(3)
    J0[3:, 3:] = po.m_rot(z[3:])
    return Ci @ (z - p), Ci @ J0


def _normal(z, poses, S7s, vos, fc, srx, srq):
    N = len(poses)
    rows, res = [], []
    for i in range(N):
        r, J = unary(z[7 * i:7 * i + 7], poses[i], S7s[i])
        Jf = np.zeros((7, 6 * N))
        Jf[:, 6 * i:6 * i + 6] = J
        rows.append(Jf); res.append(r)
    L_rx, L_rq = np.eye(3) / math.sqrt(srx), np.eye(4) / math.sqrt(srq)
    for k, (i, j) in enumerate(po.edges(N, fc)):                          # pgo_oracle.optimize's relative factors
        qi, qj = z[7 * i + 3:7 * i + 7], z[7 * j + 3:7 * j + 7]
        dt = po.dqstq_t(qi)
        jt = np.zeros((3, 6 * N)); jt[:, 6 * i:6 * i + 3] = -dt; jt[:, 6 * j:6 * j + 3] = dt
        rt = po.rotate_vector(z[7 * j:7 * j + 3] - z[7 * i:7 * i + 3], po.qinverse(qi)) - vos[k, :3]
        rows.append(L_rx @ jt); res.append(L_rx @ rt)
        jr = np.zeros((4, 6 * N))
        jr[:, 6 * i + 3:6 * i + 6] = po.dpsq_p(qj) @ po.m_rot(qi)
        jr[:, 6 * j + 3:6 * j + 6] = po.dpsq_q(qi) @ po.m_rot(qj)
        rows.append(L_rq @ jr); res.append(L_rq @ (po.qmult(po.qinverse(qi), qj) - vos[k, 3:]))
    J, r = np.vstack(rows), np.concatenate(res)
    return J.T @ J, J.T @ r


def optimize_cov(poses, S7s, vos, fc=False, srx=1.0, srq=1.0, n_iters=10):
    """one window: poses [N,7], S7s [N,7,7], vos [E,7] -> (poses [N,7], cov [N,6,6] in (t, log q))"""
    poses = np.asarray(poses, dtype=np.float64)
    N = len(poses)
    z = poses.reshape(-1).copy()
    for _ in range(n_iters):
        H, b = _normal(z, poses, S7s, vos, fc, srx, srq)
        x = np.linalg.solve(H, -b)                                        # the Gauss-Newton step
        for i in range(N):
            z[7 * i:7 * i + 3] += x[6 * i:6 * i + 3]
            qm = x[6 * i + 3:6 * i + 6]
            n = np.linalg.norm(qm)
            z[7 * i + 3:7 * i + 7] = po.qmult(z[7 * i + 3:7 * i + 7], np.concatenate(([math.cos(n)], np.sinc(n / np.pi) * qm)))
    H, _ = _normal(z, poses, S7s, vos, fc, srx, srq)
    np.linalg.cholesky(H)                                                 # raises where the kernel flags the window
    P = np.linalg.inv(H)
    cov = np.empty((N, 6, 6))
    for i in range(N):
        B = np.eye(6)
        B[3:, 3:] = qlog_jac(z[7 * i + 3:7 * i + 7])
        cov[i] = B @ P[6 * i:6 * i + 6, 6 * i:6 * i + 6] @ B.T
    return z.reshape(-1, 7), cov


def random_window(rng, N, fc, lq_max=2.5):
    """poses [N,7] with log q up to lq_max, coupled random SPD S7s [N,7,7], vos [E,7] near the poses' own"""
    lq = rng.standard_normal((N, 3))
    lq *= (rng.uniform(0, lq_max, N) / np.linalg.norm(lq, axis=1))[:, None]
    mu = np.hstack((rng.standard_normal((N, 3)), lq))
    poses = np.stack([np.concatenate((m[:3], qexp(m[3:]))) for m in mu])
    S7s = []
    for _ in range(N):
        A = rng.standard_normal((7, 7)) * 0.1
        S7s.append(A @ A.T + np.diag(rng.uniform(0.01, 0.1, 7)))
    vos = []
    for i, j in po.edges(N, fc):
        t = po.rotate_vector(poses[j, :3] - poses[i, :3], po.qinverse(poses[i, 3:]))
        q = po.qmult(po.qinverse(poses[i, 3:]), poses[j, 3:])
        vos.append(np.concatenate((t, q)) + rng.standard_normal(7) * 0.05)
    return poses, np.stack(S7s), np.stack(vos)


def _fd(f, x, h=1e-6):
    x = np.asarray(x, dtype=np.float64)
    cols = []
    for k in range(x.size):
        e = np.zeros_like(x); e[k] = h
        cols.append((f(x + e) - f(x - e)) / (2 * h))
    return np.stack(cols, -1)


def _boxplus(z, x):
    n = np.linalg.norm(x[3:])
    dq = np.concatenate(([math.cos(n)], np.sinc(n / np.pi) * x[3:]))
    return np.concatenate((z[:3] + x[:3], po.qmult(z[3:], dq)))


# ---- oracle checks --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0.0, 1e-9, 1e-3, 0.0999, 0.1001, 1.0, 2.5])
def test_qexp_jacobian_matches_finite_differences(n):
    rng = np.random.default_rng(int(n * 1e4) + 1)
    d = rng.standard_normal(3)
    v = d / np.linalg.norm(d) * n
    np.testing.assert_allclose(qexp_jac(v), _fd(qexp, v), rtol=0, atol=1e-8)
    if n == 0:
        np.testing.assert_array_equal(qexp_jac(v), np.vstack((np.zeros((1, 3)), np.eye(3))))


@pytest.mark.parametrize("seed", range(6))
def test_qlog_jacobian_matches_finite_differences(seed):
    rng = np.random.default_rng(seed)
    lq = rng.standard_normal(3) * [1e-4, 0.3, 1.0, 1.5, 2.5, 1e-9][seed]
    q = qexp(lq) * (1.0 + 0.01 * seed)                      # PGO states are not renormalised
    f = lambda x: qlog(po.qmult(q, qexp(x)))
    np.testing.assert_allclose(qlog_jac(q), _fd(f, np.zeros(3)), rtol=0, atol=1e-7)
    np.testing.assert_allclose(qlog_jac(np.array([1.0, 0.0, 0.0, 0.0])), np.eye(3), rtol=0, atol=0)


@pytest.mark.parametrize("seed", range(4))
def test_unary_jacobian_including_the_whitening_matches_finite_differences(seed):
    rng = np.random.default_rng(10 + seed)
    poses, S7s, _ = random_window(rng, 2, False)
    z = np.concatenate((poses[1, :3] + 0.1, po.qmult(poses[1, 3:], qexp(rng.standard_normal(3) * 0.2))))
    _, J = unary(z, poses[0], S7s[0])
    np.testing.assert_allclose(J, _fd(lambda x: unary(_boxplus(z, x), poses[0], S7s[0])[0], np.zeros(6)),
                               rtol=0, atol=1e-6 * np.abs(J).max())


def test_zero_sampled_covariance_gives_the_reference_unary_factor():
    rng = np.random.default_rng(3)
    sax, saq = 0.7, 0.2
    for n in (0.0, 0.5, 2.5):
        mu = np.concatenate((rng.standard_normal(3), rng.standard_normal(3)))
        mu[3:] *= n / np.linalg.norm(mu[3:])
        p, S7 = factor(mu, np.zeros((6, 6)), sax, saq)
        np.testing.assert_array_equal(S7, np.diag([sax] * 3 + [saq] * 4))
        z = np.concatenate((p[:3] + 0.3, p[3:] * 1.1))
        r, J = unary(z, p, S7)
        # pgo_oracle.optimize's unary rows: L_ax (t - t0), L_aq (q - q0), Jacobians L_ax I, L_aq m_rot(q)
        np.testing.assert_allclose(r, np.concatenate(((z[:3] - p[:3]) / math.sqrt(sax), (z[3:] - p[3:]) / math.sqrt(saq))),
                                   rtol=1e-15, atol=0)
        want = np.zeros((7, 6))
        want[:3, :3] = np.eye(3) / math.sqrt(sax)
        want[3:, 3:] = po.m_rot(z[3:]) / math.sqrt(saq)
        np.testing.assert_allclose(J, want, rtol=1e-15, atol=0)


def test_oracle_with_reference_factors_is_the_exact_solve_of_pgo_oracle():
    rng = np.random.default_rng(4)
    for fc in (False, True):
        poses, _, vos = random_window(rng, 5, fc)
        S7s = np.stack([np.diag([0.3] * 3 + [0.05] * 4)] * 5)
        got, _ = optimize_cov(poses, S7s, vos, fc, 2.0, 3.0)
        want = po.optimize(poses, vos, 0.3, 0.05, 2.0, 3.0, fc=fc, exact_solve=True)
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


# ---- C ABI and Python argument errors, before any launch ------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


def test_entry_points_are_declared_exported_and_refuse_bad_arguments_without_a_launch(L):
    from geomapnet_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mapnet_b200.h")).read(), flags=re.S)
    for name in _lib.TRACK_SAMPLE_API + ["mapnet_pgo_optimize_cov", "mapnet_test_sample_factor"]:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in _lib.EXPORTED and hasattr(L, name)
    n0 = L.mapnet_launch_count()
    out = ctypes.c_void_p()
    sig = (ctypes.c_double * 4)(1.0, 1.0, 1.0, 1.0)
    m3 = (ctypes.c_double * 3)(0.0, 0.0, 0.0)
    for T, skip, mb, s, pm, ps, msg in [
            (1, 1, 4, sig, None, None, b"outside [2, 16]"), (17, 1, 4, sig, None, None, b"outside [2, 16]"),
            (3, 0, 4, sig, None, None, b"must be >= 1"), (3, 1, 0, sig, None, None, b"must be >= 1"),
            (3, 1, 4, (ctypes.c_double * 4)(1.0, 0.0, 1.0, 1.0), None, None, b"positive"),
            (3, 1, 4, (ctypes.c_double * 4)(1.0, 1.0, -1.0, 1.0), None, None, b"positive"),
            (3, 1, 4, sig, m3, None, b"go together"), (3, 1, 4, None, None, None, b"null argument")]:
        assert L.mapnet_track_sample_create(ctypes.byref(out), T, skip, 0, mb, s, pm, ps) != 0, (T, skip, mb)
        assert msg in L.mapnet_last_error(), (msg, L.mapnet_last_error())
        assert b"track_sample_create" in L.mapnet_last_error()
        assert not out.value
    for rc in (L.mapnet_track_sample_step(None, None, None, None, 1, None, None),
               L.mapnet_track_sample_step_now(None, None, None, None, 1, None, None, None),
               L.mapnet_track_sample_flush(None, None, None), L.mapnet_track_sample_reset(None, None),
               L.mapnet_track_sample_status(None, None, None, None)):
        assert rc != 0 and b"null handle" in L.mapnet_last_error()
    assert L.mapnet_track_sample_destroy(None) == 0
    p = ctypes.c_void_p(16)
    for args, msg in [((None, p, p, p, p, 1, 3, 0, 1.0, 1.0, 10, None, None), b"bad argument"),
                      ((p, p, p, p, None, 1, 3, 0, 1.0, 1.0, 10, None, None), b"bad argument"),
                      ((p, p, p, p, p, 0, 3, 0, 1.0, 1.0, 10, None, None), b"bad argument"),
                      ((p, p, p, p, p, 1, 1, 0, 1.0, 1.0, 10, None, None), b"outside [2, 16]"),
                      ((p, p, p, p, p, 1, 17, 0, 1.0, 1.0, 10, None, None), b"outside [2, 16]"),
                      ((p, p, p, p, p, 1, 3, 0, 0.0, 1.0, 10, None, None), b"positive"),
                      ((p, p, p, p, p, 1, 3, 0, 1.0, -2.0, 10, None, None), b"positive")]:
        assert L.mapnet_pgo_optimize_cov(*args) != 0
        assert msg in L.mapnet_last_error() and b"pgo_optimize_cov" in L.mapnet_last_error()
    for args, msg in [((None, p, 1, 1.0, 1.0, p, p, None), b"bad argument"),
                      ((p, p, 0, 1.0, 1.0, p, p, None), b"bad argument"),
                      ((p, p, 1, 1.0, 1.0, p, None, None), b"bad argument"),
                      ((p, p, 1, 0.0, 1.0, p, p, None), b"positive"),
                      ((p, p, 1, 1.0, -1.0, p, p, None), b"positive")]:
        assert L.mapnet_test_sample_factor(*args) != 0
        assert msg in L.mapnet_last_error() and b"test_sample_factor" in L.mapnet_last_error()
    assert L.mapnet_launch_count() == n0


def test_sampled_tracker_argument_errors_before_any_launch(L):
    from geomapnet_b200.inference import Localizer, SampledTracker, Tracker
    pr = _stub_predictor()
    loc = Localizer(pr, MEAN, STD)
    n0 = L.mapnet_launch_count()
    with pytest.raises(ValueError, match="no dropout"):
        SampledTracker(loc, 8, 3)                        # droprate 0
    pr.droprate = 0.5
    for obj in (pr, None):
        with pytest.raises(TypeError, match="Localizer"):
            SampledTracker(obj, 8, 3)
    for S in (1, 0, 1025, 2.0, True, "8"):
        with pytest.raises(ValueError, match="S must be"):
            SampledTracker(loc, S, 3)
    for steps in (1, 17):
        with pytest.raises(ValueError, match="steps"):
            SampledTracker(loc, 8, steps)
    for k in ("sax", "saq", "srx", "srq"):
        with pytest.raises(ValueError, match="positive"):
            SampledTracker(loc, 8, 3, **{k: 0.0})
    st = SampledTracker(loc, 8, 7, skip=10, vo_fc=True, sax=1e-4, saq=1e-4, srx=20, srq=20)
    assert isinstance(st, Tracker) and st.lag == 30 and st.seen == 0 and st.S == 8
    f2, v2 = torch.zeros(2, 48, 64, 3, dtype=torch.uint8), torch.zeros(2, 6)
    for frames, vo, msg in [(f2, torch.zeros(3, 6), "vo_poses must be \\[2, 6\\]"),
                            (f2[0], torch.zeros(1, 6), "vo_poses must be \\[6\\]"),
                            (f2, torch.zeros(2, 6, dtype=torch.int32), "float"),
                            (torch.zeros(2, 48, 64, 3), v2, "uint8")]:
        for call in (st, st.step):
            with pytest.raises(ValueError, match=msg):
                call(frames, vo)
    st.reset()
    assert st.seen == 0
    st.close()
    for call in (lambda: st(f2, v2), st.flush, st.reset):
        with pytest.raises(ValueError, match="SampledTracker is closed"):
            call()
    st = SampledTracker(loc, 8, 3)
    pr._params = None
    for call in (lambda: st(f2, v2), lambda: st.step(f2, v2), st.flush):
        with pytest.raises(ValueError, match="Predictor is closed"):
            call()
    assert L.mapnet_launch_count() == n0
