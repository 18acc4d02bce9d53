"""Host-side checks of the Cauchy-weighted pose graphs (no GPU needed): a numpy float64 iteratively reweighted
Gauss-Newton for the point graph (on oracle/pgo_oracle.py's factors) and the covariance graph (on
test_track_sample_host's factors) -- the oracle the GPU tests compare k_pgo<true> and k_pgo_cov<true> against -- that
is the plain oracle exactly when c = inf, silences a gross outlier at c = 2, and whose weight is the derivative of the
Cauchy loss; and every robust_c / c argument error, raised before any launch."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import pgo_oracle as po
from test_track_host import _stub_predictor      # an open Predictor without an engine
from test_track_sample_host import _normal, optimize_cov, qexp, qlog_jac, random_window, unary

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN = [0.5, 0.44, 0.45]
STD = [0.21, 0.23, 0.22]
BAD_C = [0.0, -1.0, float("nan"), float("inf"), -float("inf"), "2", True, object(), [2.0], 1j]


# ---- the oracle -----------------------------------------------------------------------------------------------------
def cauchy_weight(r, c):
    """w = 1 / (1 + |r|^2 / c^2) of a whitened residual r, |r|^2 / c^2 summed as (r_k / c)^2 as the kernels sum it"""
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + float(np.sum((np.asarray(r, dtype=np.float64) / c) ** 2)))


def rho(s, c):
    return c * c * math.log1p(s / (c * c))


def _update(z, x, N):
    for i in range(N):                                                    # pgo_oracle.optimize's manifold update
        z[7 * i:7 * i + 3] += x[6 * i:6 * i + 3]
        qm = x[6 * i + 3:6 * i + 6]
        n = np.linalg.norm(qm)
        z[7 * i + 3:7 * i + 7] = po.qmult(z[7 * i + 3:7 * i + 7], np.concatenate(([math.cos(n)], np.sinc(n / np.pi) * qm)))


def point_weights(z, poses, sax, saq, c):
    N = len(poses)
    return np.array([cauchy_weight(np.concatenate(((z[7 * i:7 * i + 3] - poses[i, :3]) / math.sqrt(sax),
                                                   (z[7 * i + 3:7 * i + 7] - poses[i, 3:]) / math.sqrt(saq))), c)
                     for i in range(N)])


def optimize_robust(poses, vos, sax=1, saq=1, srx=1, srq=1, n_iters=10, fc=False, exact_solve=False, c=math.inf):
    """pgo_oracle.optimize with slot i's two absolute rows weighed by w_i (its Cauchy weight at the iteration's
    starting state) in H = J' W J and b = J' W r.  -> (poses [N,7], w [N] at the returned state)"""
    poses = np.asarray(poses, dtype=np.float64)
    vos = np.asarray(vos, dtype=np.float64)
    N = len(poses)
    z = poses.copy().reshape(-1)
    L_ax, L_aq = np.eye(3) / math.sqrt(sax), np.eye(4) / math.sqrt(saq)
    L_rx, L_rq = np.eye(3) / math.sqrt(srx), np.eye(4) / math.sqrt(srq)
    for _ in range(n_iters):
        om = point_weights(z, poses, sax, saq, c)
        rows, res, wrow = [], [], []
        for i in range(N):
            jt = np.zeros((3, 6 * N)); jt[:, 6 * i:6 * i + 3] = np.eye(3)
            rows.append(L_ax @ jt); res.append(L_ax @ (z[7 * i:7 * i + 3] - poses[i, :3]))
            jr = np.zeros((4, 6 * N)); jr[:, 6 * i + 3:6 * i + 6] = po.m_rot(z[7 * i + 3:7 * i + 7])
            rows.append(L_aq @ jr); res.append(L_aq @ (z[7 * i + 3:7 * i + 7] - poses[i, 3:]))
            wrow.append(np.full(7, om[i]))
        for k, (i, j) in enumerate(po.edges(N, fc)):
            qi, qj = z[7 * i + 3:7 * i + 7], z[7 * j + 3:7 * j + 7]
            dt = po.dqstq_t(qi)
            jt = np.zeros((3, 6 * N)); jt[:, 6 * i:6 * i + 3] = -dt; jt[:, 6 * j:6 * j + 3] = dt
            rt = po.rotate_vector(z[7 * j:7 * j + 3] - z[7 * i:7 * i + 3], po.qinverse(qi)) - vos[k, :3]
            rows.append(L_rx @ jt); res.append(L_rx @ rt)
            jr = np.zeros((4, 6 * N))
            jr[:, 6 * i + 3:6 * i + 6] = po.dpsq_p(qj) @ po.m_rot(qi)
            jr[:, 6 * j + 3:6 * j + 6] = po.dpsq_q(qi) @ po.m_rot(qj)
            rows.append(L_rq @ jr); res.append(L_rq @ (po.qmult(po.qinverse(qi), qj) - vos[k, 3:]))
            wrow.append(np.ones(7))
        J, r, wr = np.vstack(rows), np.concatenate(res), np.concatenate(wrow)
        H, b = (J.T * wr) @ J, (J.T * wr) @ r
        R = np.linalg.cholesky(H).T
        y = np.linalg.solve(R.T, -b) if exact_solve else -b / np.diag(R)
        _update(z, np.linalg.solve(R, y), N)
    return z.reshape(-1, 7), point_weights(z, poses, sax, saq, c)


def cov_weights(z, poses, S7s, c):
    return np.array([cauchy_weight(unary(z[7 * i:7 * i + 7], poses[i], S7s[i])[0], c) for i in range(len(poses))])


def _normal_robust(z, poses, S7s, vos, fc, srx, srq, c):
    """(H, b, w) at z: test_track_sample_host._normal with slot i's absolute factor weighed by w_i"""
    H, b = _normal(z, poses, S7s, vos, fc, srx, srq)
    om = cov_weights(z, poses, S7s, c)
    for i in range(len(poses)):
        r, J = unary(z[7 * i:7 * i + 7], poses[i], S7s[i])
        sl = slice(6 * i, 6 * i + 6)
        H[sl, sl] += (om[i] - 1.0) * (J.T @ J)
        b[sl] += (om[i] - 1.0) * (J.T @ r)
    return H, b, om


def optimize_cov_robust(poses, S7s, vos, fc=False, srx=1.0, srq=1.0, n_iters=10, c=math.inf):
    """test_track_sample_host.optimize_cov, reweighted: -> (poses [N,7], cov [N,6,6], w [N] at the returned state)"""
    poses = np.asarray(poses, dtype=np.float64)
    N = len(poses)
    z = poses.reshape(-1).copy()
    for _ in range(n_iters):
        H, b, _ = _normal_robust(z, poses, S7s, vos, fc, srx, srq, c)
        _update(z, np.linalg.solve(H, -b), N)
    H, _, om = _normal_robust(z, poses, S7s, vos, fc, srx, srq, c)
    np.linalg.cholesky(H)
    P = np.linalg.inv(H)
    cov = np.empty((N, 6, 6))
    for i in range(N):
        B = np.eye(6)
        B[3:, 3:] = qlog_jac(z[7 * i + 3:7 * i + 7])
        cov[i] = B @ P[6 * i:6 * i + 6, 6 * i:6 * i + 6] @ B.T
    return z.reshape(-1, 7), cov, om


def outlier_window(rng, N, fc, sigma, shift):
    """(poses, outlier poses, vos): a smooth window with translation noise of sigma, VOs exactly the noise-free
    window's, and the same poses with slot N // 2's translation moved `shift` sigmas"""
    lq = np.cumsum(rng.standard_normal((N, 3)) * 0.05, 0)
    t = np.cumsum(rng.standard_normal((N, 3)) * 0.3, 0)
    poses = np.hstack((t, np.stack([qexp(v) for v in lq])))
    vos = np.stack([np.concatenate((po.rotate_vector(poses[j, :3] - poses[i, :3], po.qinverse(poses[i, 3:])),
                                    po.qmult(po.qinverse(poses[i, 3:]), poses[j, 3:]))) for i, j in po.edges(N, fc)])
    noisy = poses + np.hstack((rng.standard_normal((N, 3)) * sigma, np.zeros((N, 4))))
    bad = noisy.copy()
    k = N // 2
    d = rng.standard_normal(3)
    bad[k, :3] += shift * sigma * d / np.linalg.norm(d)
    return noisy, bad, vos


# ---- oracle checks --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fc", [False, True])
@pytest.mark.parametrize("exact", [False, True])
def test_infinite_scale_is_the_plain_point_oracle_exactly(fc, exact):
    rng = np.random.default_rng(1 + fc + 2 * exact)
    for N in (2, 3, 7):
        poses, _, vos = random_window(rng, N, fc, lq_max=1.0)
        got, w = optimize_robust(poses, vos, 0.3, 0.05, 2.0, 3.0, fc=fc, exact_solve=exact)
        np.testing.assert_array_equal(got, po.optimize(poses, vos, 0.3, 0.05, 2.0, 3.0, fc=fc, exact_solve=exact))
        np.testing.assert_array_equal(w, np.ones(N))


@pytest.mark.parametrize("fc", [False, True])
def test_infinite_scale_is_the_plain_covariance_oracle_exactly(fc):
    rng = np.random.default_rng(5 + fc)
    for N in (2, 3, 7):
        poses, S7s, vos = random_window(rng, N, fc)
        got, cov, w = optimize_cov_robust(poses, S7s, vos, fc, 2.0, 3.0)
        want, want_cov = optimize_cov(poses, S7s, vos, fc, 2.0, 3.0)
        np.testing.assert_array_equal(got, want)
        np.testing.assert_array_equal(cov, want_cov)
        np.testing.assert_array_equal(w, np.ones(N))


def _deviation(a, b, skip):
    keep = [i for i in range(len(a)) if i != skip]
    return float(np.abs(a[keep] - b[keep]).max())


@pytest.mark.parametrize("fc", [False, True])
def test_a_30_sigma_outlier_is_silenced_at_c_2_in_the_point_graph(fc):
    sigma, N = 0.1, 7
    sax = saq = sigma ** 2
    srx = srq = 1e-2
    noisy, bad, vos = outlier_window(np.random.default_rng(11 + fc), N, fc, sigma, 30.0)
    clean, _ = optimize_robust(noisy, vos, sax, saq, srx, srq, fc=fc, exact_solve=True)
    plain, _ = optimize_robust(bad, vos, sax, saq, srx, srq, fc=fc, exact_solve=True)
    robust, w = optimize_robust(bad, vos, sax, saq, srx, srq, fc=fc, exact_solve=True, c=2.0)
    assert w[N // 2] < 0.01 and np.delete(w, N // 2).min() > 0.3, w
    d_plain, d_robust = _deviation(plain, clean, N // 2), _deviation(robust, clean, N // 2)
    assert d_robust < sigma and d_robust < 0.3 * d_plain, (d_robust, d_plain)
    assert d_plain > 2 * sigma, d_plain


@pytest.mark.parametrize("fc", [False, True])
def test_a_30_sigma_outlier_is_silenced_at_c_2_in_the_covariance_graph(fc):
    sigma, N = 0.1, 7
    noisy, bad, vos = outlier_window(np.random.default_rng(21 + fc), N, fc, sigma, 30.0)
    S7s = np.stack([np.diag([sigma ** 2] * 7)] * N)
    clean, _, _ = optimize_cov_robust(noisy, S7s, vos, fc, 1e-2, 1e-2)
    plain, _, _ = optimize_cov_robust(bad, S7s, vos, fc, 1e-2, 1e-2)
    robust, cov, w = optimize_cov_robust(bad, S7s, vos, fc, 1e-2, 1e-2, c=2.0)
    assert w[N // 2] < 0.01 and np.delete(w, N // 2).min() > 0.3, w
    d_plain, d_robust = _deviation(plain, clean, N // 2), _deviation(robust, clean, N // 2)
    assert d_robust < sigma and d_robust < 0.3 * d_plain, (d_robust, d_plain)
    assert np.isfinite(cov).all()


@pytest.mark.parametrize("c", [0.5, 1.0, 2.0, 4.0, 30.0])
def test_the_weight_is_the_derivative_of_the_cauchy_loss(c):
    rng = np.random.default_rng(int(c * 10))
    for _ in range(8):
        r = rng.standard_normal(7) * rng.uniform(0.0, 5.0) * c
        s, h = float(r @ r), 1e-6 * max(1.0, float(r @ r))
        fd = (rho(s + h, c) - rho(s - h, c)) / (2 * h)
        assert abs(cauchy_weight(r, c) - fd) < 1e-8, (c, s)
    assert cauchy_weight(np.zeros(7), 1e-300) == 1.0 and cauchy_weight(np.full(7, 1e300), 1e-300) == 0.0
    assert cauchy_weight(np.full(7, 1e3), 1e300) == 1.0


# ---- C ABI and Python argument errors, before any launch ------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


def test_entry_points_are_declared_exported_and_refuse_bad_arguments_without_a_launch(L):
    from geomapnet_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mapnet_b200.h")).read(), flags=re.S)
    for name in _lib.ROBUST_API:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in _lib.EXPORTED and hasattr(L, name)
    assert L.mapnet_abi_version() == 2
    n0 = L.mapnet_launch_count()
    p = ctypes.c_void_p(16)
    for c in (0.0, -1.0, float("nan"), float("inf"), -float("inf")):
        assert L.mapnet_pgo_optimize_robust(p, p, p, 1, 3, 0, 1.0, 1.0, 1.0, 1.0, 10, 0, c, p, None, None) != 0
        assert b"pgo_optimize_robust" in L.mapnet_last_error() and b"finite and positive" in L.mapnet_last_error()
        assert L.mapnet_pgo_optimize_cov_robust(p, p, p, p, p, 1, 3, 0, 1.0, 1.0, 10, c, p, None, None) != 0
        assert b"pgo_optimize_cov_robust" in L.mapnet_last_error() and b"finite and positive" in L.mapnet_last_error()
    for args, msg in [((None, p, p, 1, 3, 0, 1.0, 1.0, 1.0, 1.0, 10, 0, 2.0, p, None, None), b"bad argument"),
                      ((p, p, p, 0, 3, 0, 1.0, 1.0, 1.0, 1.0, 10, 0, 2.0, p, None, None), b"bad argument"),
                      ((p, p, p, 1, 17, 0, 1.0, 1.0, 1.0, 1.0, 10, 0, 2.0, p, None, None), b"outside [2, 16]"),
                      ((p, p, p, 1, 3, 0, 0.0, 1.0, 1.0, 1.0, 10, 0, 2.0, p, None, None), b"positive")]:
        assert L.mapnet_pgo_optimize_robust(*args) != 0
        assert msg in L.mapnet_last_error() and b"pgo_optimize_robust" in L.mapnet_last_error()
    for args, msg in [((p, None, p, p, p, 1, 3, 0, 1.0, 1.0, 10, 2.0, p, None, None), b"bad argument"),
                      ((p, p, p, p, p, 1, 1, 0, 1.0, 1.0, 10, 2.0, p, None, None), b"outside [2, 16]"),
                      ((p, p, p, p, p, 1, 3, 0, 1.0, -1.0, 10, 2.0, p, None, None), b"positive")]:
        assert L.mapnet_pgo_optimize_cov_robust(*args) != 0
        assert msg in L.mapnet_last_error() and b"pgo_optimize_cov_robust" in L.mapnet_last_error()
    for name in _lib.ROBUST_API[2:]:
        assert getattr(L, name)(None, 2.0) != 0 and b"null handle" in L.mapnet_last_error(), name
    assert L.mapnet_launch_count() == n0


def test_python_entry_points_refuse_a_bad_robust_c_before_any_launch(L):
    from geomapnet_b200.common.pgo import check_robust_c, optimize_pose_windows, optimize_pose_windows_cov
    from geomapnet_b200.inference import (Localizer, MultiTracker, SampledMultiTracker, SampledTracker, Tracker,
                                          evaluate_sequence, pgo)
    assert check_robust_c(None) is None and check_robust_c(2) == 2.0 and check_robust_c(np.float32(0.5)) == 0.5
    pr = _stub_predictor()
    loc = Localizer(pr, MEAN, STD)
    n0 = L.mapnet_launch_count()
    p7, v7, s7 = torch.zeros(1, 3, 7), torch.zeros(1, 2, 7), torch.zeros(1, 3, 7, 7)
    for c in BAD_C:
        with pytest.raises(ValueError, match="robust_c"):
            optimize_pose_windows(p7, v7, robust_c=c)
        with pytest.raises(ValueError, match="robust_c"):
            optimize_pose_windows_cov(p7, s7, v7, robust_c=c)
        with pytest.raises(ValueError, match="robust_c"):
            pgo(p7, v7, robust_c=c)
        with pytest.raises(ValueError, match="robust_c"):
            evaluate_sequence(None, None, robust_c=c)
        with pytest.raises(ValueError, match="robust_c"):
            Tracker(loc, 3, robust_c=c)
        with pytest.raises(ValueError, match="robust_c"):
            MultiTracker(loc, 2, 3, robust_c=c)
    pr.droprate = 0.5
    for c in BAD_C:
        with pytest.raises(ValueError, match="robust_c"):
            SampledTracker(loc, 8, 3, robust_c=c)
        with pytest.raises(ValueError, match="robust_c"):
            SampledMultiTracker(loc, 8, 2, 3, robust_c=c)
    trk = SampledMultiTracker(loc, 8, 2, 7, skip=10, vo_fc=True, robust_c=2)
    assert trk.robust_c == 2.0 and isinstance(trk.robust_c, float) and not trk.h      # no handle until the first call
    assert Tracker(loc, 3).robust_c is None
    assert L.mapnet_launch_count() == n0
