"""Host-side checks of inference.evaluate_sequence(samples=S) (no GPU needed): the calibration arithmetic of
csrc/calib_core.h, compiled for the host, against an independent numpy / scipy float64 oracle (random SPD
covariances, rotations past 90 degrees, q = -q^, q = q^ with a zero vector part, near-identity rotations, covariances
that are not positive definite), a coverage check of the scores on errors drawn from the covariance itself, the
entry points' exports and argument errors, and every Python argument error raised before any launch."""
import ctypes
import math
import os
import re
import subprocess
import tempfile
import types

import numpy as np
import pytest
import torch
from scipy import stats

from test_track_host import _stub_predictor      # an open Predictor without an engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests")


@pytest.fixture(scope="module")
def hc():
    d = tempfile.mkdtemp(prefix="hostcalib")
    so = os.path.join(d, "libhostcalib.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(HERE, "_hostcalib.cpp")])
    lib = ctypes.CDLL(so)
    lib.hc_score.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_longlong] + [ctypes.c_void_p] * 4
    return lib


@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


def _score(hc, est7, targ7, cov):
    """calib_core.h on the host: (e [n,6], d2 [n,3], u [n,3], nll [n])"""
    est7, targ7 = (np.ascontiguousarray(a, dtype=np.float64) for a in (est7, targ7))
    cov = np.ascontiguousarray(cov, dtype=np.float64).reshape(-1, 36)
    n = est7.shape[0]
    e, d2, u, nll = np.empty((n, 6)), np.empty((n, 3)), np.empty((n, 3)), np.empty(n)
    hc.hc_score(est7.ctypes.data, targ7.ctypes.data, cov.ctypes.data, n, e.ctypes.data, d2.ctypes.data, u.ctypes.data,
                nll.ctypes.data)
    return e, d2, u, nll


# ---- the oracle: numpy / scipy float64 ------------------------------------------------------------------------------
def qexp(v):
    n = np.linalg.norm(v)
    return np.concatenate(([math.cos(n)], math.sin(n) / n * np.asarray(v))) if n > 0 else np.array([1.0, 0, 0, 0])


def qlog(q):
    """common/pose_utils.py:307-317, w clamped to [-1, 1]"""
    q = np.asarray(q, dtype=np.float64)
    if np.all(q[1:] == 0):
        return np.zeros(3)
    return np.arccos(np.clip(q[0], -1.0, 1.0)) * q[1:] / np.linalg.norm(q[1:])


def oracle(est7, targ7, cov):
    """(e [6], d2 [3], nll) of one estimate; NaN where the covariance (block) has no Cholesky factor"""
    sg = -1.0 if est7[3:] @ targ7[3:] < 0 else 1.0
    e = np.concatenate((est7[:3] - targ7[:3], qlog(est7[3:]) - qlog(sg * targ7[3:])))

    def maha(C, x):
        try:
            np.linalg.cholesky(C)
        except np.linalg.LinAlgError:
            return math.nan, math.nan
        return float(x @ np.linalg.solve(C, x)), float(np.linalg.slogdet(C)[1])
    d6, ld = maha(cov, e)
    d2 = np.array([d6, maha(cov[:3, :3], e[:3])[0], maha(cov[3:, 3:], e[3:])[0]])
    return e, d2, 0.5 * (d6 + 6 * math.log(2 * math.pi) + ld)


def _spd(rng, scale=1.0):
    A = rng.standard_normal((6, 6)) * scale
    return A @ A.T + np.diag(rng.uniform(0.05, 0.5, 6)) * scale ** 2


def _case(rng, lq, dq=0.1, dt=0.5):
    """an estimate with log q of norm lq and a target near it"""
    d = rng.standard_normal(3)
    v = d / np.linalg.norm(d) * lq
    est = np.concatenate((rng.standard_normal(3) * 3, qexp(v)))
    targ = np.concatenate((est[:3] + rng.standard_normal(3) * dt, qexp(v + rng.standard_normal(3) * dq)))
    return est, targ


def _cases():
    rng = np.random.default_rng(11)
    est, targ, cov = [], [], []

    def add(e, t, c):
        est.append(e); targ.append(t); cov.append(c)
    for k in range(40):                                   # random SPD, |log q| from 0.05 to 2.9 (w < 0 past pi/2)
        e, t = _case(rng, 0.05 + 2.85 * k / 39)
        add(e, t, _spd(rng, [0.1, 1.0, 3.0][k % 3]))
    for lq in (1.7, 2.5, 3.0):                            # w < 0, target on the other side of the sphere: -q
        e, t = _case(rng, lq)
        add(e, np.concatenate((t[:3], -t[3:])), _spd(rng))
    e, _ = _case(rng, 1.2)
    add(e, np.concatenate((e[:3] + 0.3, -e[3:])), _spd(rng))                           # q = -q^
    q1 = np.array([1.0, 0.0, 0.0, 0.0])
    add(np.concatenate(([1.0, 2.0, 3.0], q1)), np.concatenate(([1.5, 2.0, 2.5], q1)), _spd(rng))   # zero vector parts
    for n in (1e-12, 1e-9, 1e-6):                         # near-identity rotations
        d = rng.standard_normal((2, 3))
        add(np.concatenate(([0.1, 0.2, 0.3], qexp(d[0] * n))), np.concatenate(([0.0, 0.2, 0.4], qexp(d[1] * n))),
            _spd(rng, 1e-3))
    return np.stack(est), np.stack(targ), np.stack(cov)


# ---- the arithmetic against the oracle ------------------------------------------------------------------------------
def test_scores_match_the_float64_oracle(hc):
    est, targ, cov = _cases()
    e, d2, u, nll = _score(hc, est, targ, cov)
    for i in range(est.shape[0]):
        we, wd2, wnll = oracle(est[i], targ[i], cov[i])
        np.testing.assert_allclose(e[i], we, rtol=0, atol=1e-15 * max(1.0, np.abs(we).max()), err_msg=str(i))
        np.testing.assert_allclose(d2[i], wd2, rtol=1e-12, atol=1e-300, err_msg=str(i))
        np.testing.assert_allclose(nll[i], wnll, rtol=1e-12, atol=0, err_msg=str(i))
        np.testing.assert_allclose(u[i], stats.chi2.cdf(d2[i], [6, 3, 3]), rtol=0, atol=1e-13, err_msg=str(i))
        np.testing.assert_allclose(u[i], stats.chi2.cdf(wd2, [6, 3, 3]), rtol=0, atol=1e-13, err_msg=str(i))
    assert np.isfinite(d2).all() and np.isfinite(u).all() and np.isfinite(nll).all()


def test_the_target_is_taken_in_the_estimates_chart(hc):
    est, targ, cov = _cases()
    e, _, _, _ = _score(hc, est, targ, cov)
    flip = np.concatenate((targ[:, :3], -targ[:, 3:]), 1)            # -q is the same rotation: the same error
    e2, _, _, _ = _score(hc, est, flip, cov)
    assert np.array_equal(e, e2)
    k = 43                                                           # q = -q^ exactly: no rotation error at all
    assert np.array_equal(targ[k, 3:], -est[k, 3:]) and np.array_equal(e[k, 3:], np.zeros(3))
    k = 44                                                           # two zero vector parts
    assert np.array_equal(e[k], [-0.5, 0.0, 0.5, 0.0, 0.0, 0.0])
    e0, d0, u0, _ = _score(hc, est[:1], est[:1], cov[:1])            # the target itself
    assert np.array_equal(e0, np.zeros((1, 6))) and np.array_equal(d0, np.zeros((1, 3)))
    assert np.array_equal(u0, np.zeros((1, 3)))


def test_covariances_that_are_not_positive_definite_give_nan(hc):
    rng = np.random.default_rng(3)
    est, targ = _case(rng, 0.7)
    good = _spd(rng)
    covs = []
    c = good.copy(); c[0, 0] = -1.0; covs.append(c)                  # the translation block fails
    c = good.copy(); c[5, 5] = 0.0; c[5, :5] = c[:5, 5] = 0.0; covs.append(c)      # the log q block is singular
    w, V = np.linalg.eigh(good)
    covs.append(V @ np.diag(np.concatenate(([-1e-3], w[1:]))) @ V.T)              # indefinite, blocks may be fine
    draws = rng.standard_normal((4, 6))                              # the sample covariance of S = 4 draws: rank 3
    covs.append(np.cov(draws, rowvar=False))
    draws = rng.standard_normal((6, 6))                              # S = 6: rank 5
    covs.append(np.cov(draws, rowvar=False))
    n = len(covs)
    e, d2, u, nll = _score(hc, np.tile(est, (n, 1)), np.tile(targ, (n, 1)), np.stack(covs))
    assert np.isnan(d2[:, 0]).all() and np.isnan(u[:, 0]).all() and np.isnan(nll).all()
    assert np.isnan(d2[0, 1]) and np.isfinite(d2[0, 2]) and np.isnan(d2[1, 2]) and np.isfinite(d2[1, 1])
    for k in (3, 4):                    # S - 1 >= 3: both 3 x 3 blocks of the sample covariance are positive definite
        np.testing.assert_allclose(d2[k, 1:], [oracle(est, targ, covs[k])[1][1], oracle(est, targ, covs[k])[1][2]],
                                   rtol=1e-10)
        assert np.isfinite(u[k, 1:]).all()


def test_coverage_of_errors_drawn_from_the_covariance(hc):
    """errors e ~ N(0, Sigma), targets t = t^ - e_t, q = qexp(qlog(q^) - e_v): each column of (u <= p).mean() is p"""
    rng = np.random.default_rng(2026)
    n = 20000
    C = _spd(rng, 0.05)
    Lc = np.linalg.cholesky(C)
    err = rng.standard_normal((n, 6)) @ Lc.T
    est = np.zeros((n, 7))
    est[:, :3] = rng.standard_normal((n, 3))
    v = rng.standard_normal((n, 3))
    v *= (rng.uniform(0.0, 2.5, n) / np.linalg.norm(v, axis=1))[:, None]
    est[:, 3:] = np.stack([qexp(x) for x in v])
    targ = np.zeros((n, 7))
    targ[:, :3] = est[:, :3] - err[:, :3]
    targ[:, 3:] = np.stack([qexp(qlog(est[i, 3:]) - err[i, 3:]) for i in range(n)])
    e, d2, u, _ = _score(hc, est, targ, np.broadcast_to(C, (n, 6, 6)))
    assert np.abs(e - err).max() < 1e-9
    for p in (0.5, 0.9, 0.95, 0.99):
        cov = (u <= p).mean(0)
        assert np.abs(cov - p).max() <= 0.01, (p, cov)


# ---- C ABI and Python argument errors, before any launch ------------------------------------------------------------
def test_entry_points_are_declared_exported_and_refuse_bad_arguments_without_a_launch(L):
    from geomapnet_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mapnet_b200.h")).read(), flags=re.S)
    for name in _lib.EVAL_SAMPLE_API:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in _lib.EXPORTED and hasattr(L, name)
    n0 = L.mapnet_launch_count()
    p = ctypes.c_void_p(16)
    slot = np.array([0, 1, 2, 1], np.int32)
    bad_slot = np.array([0, 1, 3, 1], np.int32)
    vo = np.array([0, 1, 1, 2], np.int32)
    bad_vo = np.array([0, 1, 1, 5], np.int32)
    S, V, BS, BV = (a.ctypes.data for a in (slot, vo, bad_slot, bad_vo))
    for args, msg in [
            ((None, p, 3, 1.0, 1.0, p, 5, S, 4, V, 2, p, p, p, None), b"eval_sample_windows: null argument"),
            ((p, p, 3, 1.0, 1.0, p, 5, None, 4, V, 2, p, p, p, None), b"eval_sample_windows: null argument"),
            ((p, p, 3, 1.0, 1.0, p, 5, S, 4, V, 2, p, None, p, None), b"eval_sample_windows: null argument"),
            ((p, p, 3, 1.0, 1.0, p, 5, S, 0, V, 2, p, p, p, None), b"eval_sample_windows: bad count"),
            ((p, p, 0, 1.0, 1.0, p, 5, S, 4, V, 2, p, p, p, None), b"eval_sample_windows: bad count"),
            ((p, p, 3, 1.0, 1.0, p, 5, S, 4, V, -1, p, p, p, None), b"eval_sample_windows: bad count"),
            ((p, p, 3, 0.0, 1.0, p, 5, S, 4, V, 2, p, p, p, None),
             b"eval_sample_windows: sax = 0 and saq = 1 must be positive"),
            ((p, p, 3, 1.0, 1.0, None, 5, S, 4, V, 2, p, p, p, None),
             b"eval_sample_windows: 2 VO rows need vo_poses, vo_rows and vos7"),
            ((p, p, 3, 1.0, 1.0, p, 5, BS, 4, V, 2, p, p, p, None),
             b"eval_sample_windows: row 2 = (frame 0, slot 3) outside the 5 poses / 3 frame rows"),
            ((p, p, 3, 1.0, 1.0, p, 2, S, 4, V, 2, p, p, p, None),
             b"eval_sample_windows: VO row 1 = (1, 2) outside the 2 poses"),
            ((p, p, 3, 1.0, 1.0, p, 5, S, 4, BV, 2, p, p, p, None),
             b"eval_sample_windows: VO row 1 = (1, 5) outside the 5 poses")]:
        assert L.mapnet_eval_sample_windows(*args) != 0, msg
        assert L.mapnet_last_error() == msg, (msg, L.mapnet_last_error())
    fr = np.array([0, 4, 2], np.int32)
    bad_fr = np.array([0, 5, 2], np.int32)
    sl = np.array([0, 1, 2], np.int32)
    bad_sl = np.array([0, 1, -1], np.int32)
    F, BF, SL, BSL = (a.ctypes.data for a in (fr, bad_fr, sl, bad_sl))
    m3 = (ctypes.c_double * 3)(0.0, 0.0, 0.0)
    for args, msg in [
            ((p, p, 3, None, None, 3, 1, None, 5, F, SL, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: null argument"),
            ((p, p, 3, None, None, 3, 1, p, 5, F, SL, 3, None, None, p, p, p, None, p, None),
             b"eval_sample_emit: null argument"),
            ((p, p, 3, p, None, 3, 1, p, 5, F, SL, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: need opt7 and post36, or mean6, cov36 and slot"),
            ((None, p, 3, None, None, 3, 1, p, 5, F, SL, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: need opt7 and post36, or mean6, cov36 and slot"),
            ((p, p, 3, None, None, 3, 1, p, 5, F, None, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: need opt7 and post36, or mean6, cov36 and slot"),
            ((p, p, 3, None, None, 3, 1, p, 5, F, SL, 0, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: bad count"),
            ((p, p, 0, None, None, 3, 1, p, 5, F, SL, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: bad count"),
            ((p, p, 3, None, None, 3, 3, p, 5, F, SL, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: slot 3 of windows of 3 outside the window"),
            ((p, p, 3, None, None, 0, 0, p, 5, F, SL, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: slot 0 of windows of 0 outside the window"),
            ((p, p, 3, None, None, 3, 1, p, 5, F, SL, 3, m3, None, p, p, p, p, p, None),
             b"eval_sample_emit: pose_m3 and pose_s3 go together"),
            ((p, p, 3, None, None, 3, 1, p, 5, BF, SL, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: row 1 = (frame 5, slot 1) outside the 5 poses / 3 frame rows"),
            ((p, p, 3, None, None, 3, 1, p, 5, F, BSL, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: row 2 = (frame 2, slot -1) outside the 5 poses / 3 frame rows"),
            ((None, None, 0, p, p, 3, 1, p, 5, BF, None, 3, None, None, p, p, p, p, p, None),
             b"eval_sample_emit: item 1: frame 5 outside the 5 poses")]:
        assert L.mapnet_eval_sample_emit(*args) != 0, msg
        assert L.mapnet_last_error() == msg, (msg, L.mapnet_last_error())
    assert L.mapnet_launch_count() == n0


def _stub_dataset(**kw):
    """the host part of a DeviceDataset on cuda:0, with no cache behind it"""
    from geomapnet_b200.data import DeviceDataset, ItemLayout
    ds = DeviceDataset.__new__(DeviceDataset)
    ItemLayout.__init__(ds, 6, **kw)
    ds.device, ds.h, ds.vo_poses, ds.max_batch, ds.Ho, ds.Wo = torch.device("cuda", 0), object(), None, 6, 16, 16
    return ds


def test_python_argument_errors_before_any_launch(L):
    import torchvision
    from geomapnet_b200.inference import evaluate_sequence
    from geomapnet_b200.models.posenet import PoseNet, MapNet
    n0 = L.mapnet_launch_count()
    pr = _stub_predictor()
    pr.net = types.SimpleNamespace(precision="bf16")
    ds = _stub_dataset(steps=3)
    with pytest.raises(ValueError, match="no dropout"):
        evaluate_sequence(pr, ds, samples=8)                 # droprate 0
    pr.droprate = 0.5
    for S in (1, 0, 1025, 2.0, True, "8"):
        with pytest.raises(ValueError, match="S must be"):
            evaluate_sequence(pr, ds, samples=S)
    for k in ("sax", "saq", "srx", "srq"):
        with pytest.raises(ValueError, match="positive"):
            evaluate_sequence(pr, ds, samples=8, **{k: 0.0})
    with pytest.raises(TypeError, match="unknown covariance"):
        evaluate_sequence(pr, ds, samples=8, sigma=1.0)
    with pytest.raises(ValueError, match="zero_lag"):
        evaluate_sequence(pr, _stub_dataset(steps=3, variable_skip=True), zero_lag=True, samples=8)
    with pytest.raises(ValueError, match="vo_fc"):
        evaluate_sequence(pr, ds, vo_fc=True, samples=8)
    with pytest.raises(ValueError, match="ColorJitter"):
        evaluate_sequence(pr, _stub_dataset(steps=3, color_jitter=0.4), samples=8)
    with pytest.raises(ValueError, match="MFOnline"):
        evaluate_sequence(pr, _stub_dataset(steps=3, online=True, n_val_frames=6), samples=8)
    # a live fp32 model has no sampled engine (model and dataset both on the CPU, so nothing else stops the call)
    model = MapNet(PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False,
                                 precision="fp32"))
    cpu = _stub_dataset(steps=3)
    cpu.device = torch.device("cpu")
    np.random.seed(0)
    state = np.random.get_state()[1].copy()
    with pytest.raises(ValueError, match="no sampled engine"):
        evaluate_sequence(model, cpu, samples=8)
    assert np.array_equal(np.random.get_state()[1], state)        # no window was drawn
    assert L.mapnet_launch_count() == n0
