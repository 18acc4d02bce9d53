"""GPU tests of the Cauchy-weighted pose graphs: k_pgo<true> (both step rules) and k_pgo_cov<true> against the float64
IRLS oracle of test_robust_pgo_host (poses, posterior covariances and weights), k_pgo_cov<true> bit for bit
reproducible, a scale of 1e300 equal to the plain kernels, and the four trackers with robust_c bit for bit
evaluate_sequence(robust_c=...) at equal chunking (zero-lag rows and flushes included), multi-stream handles bit for bit
single-stream ones, one engine replay and three tracking launches per chunk, and the scale fixed once a handle steps."""
import ctypes

import numpy as np
import pytest
import torch

from test_robust_pgo_host import optimize_cov_robust, optimize_robust
from test_track_sample_host import random_window

pytestmark = pytest.mark.gpu

C = 1.5                                  # small enough that random windows give weights well below 1
C_COV = 0.03                             # the same for random_window's broad S7 (whitened residuals of ~0.03)


def _batch(N, fc, W, seed):
    rng = np.random.default_rng(seed)
    ws = [random_window(rng, N, fc, lq_max=1.0) for _ in range(W)]
    return [np.stack([w[k] for w in ws]) for k in range(3)]      # poses [W,N,7], S7s [W,N,7,7], vos [W,E,7]


# ---------------------------------------------------------------------------------------------------------------------
# 1. kernels against the oracle, reproducibility, c -> infinity
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [2, 3, 7, 16])
@pytest.mark.parametrize("fc", [False, True])
def test_point_kernel_matches_the_irls_oracle(N, fc):
    from geomapnet_b200.common.pgo import optimize_pose_windows
    poses, _, vos = _batch(N, fc, 3, 100 + N + fc)
    sig = dict(sax=0.3, saq=0.05, srx=2.0, srq=3.0)
    for exact in (False, True):
        got, w = optimize_pose_windows(torch.from_numpy(poses), torch.from_numpy(vos), fc_vos=fc, exact_solve=exact,
                                       robust_c=C, **sig)
        got, w = got.cpu().numpy(), w.cpu().numpy()
        assert w.shape == (3, N) and (w > 0).all() and (w <= 1).all()
        for k in range(3):
            want, ww = optimize_robust(poses[k], vos[k], fc=fc, exact_solve=exact, c=C, **sig)
            np.testing.assert_allclose(got[k], want, rtol=0, atol=1e-10, err_msg=str((N, fc, exact, k)))
            np.testing.assert_allclose(w[k], ww, rtol=0, atol=1e-10, err_msg=str((N, fc, exact, k)))
        plain = optimize_pose_windows(torch.from_numpy(poses), torch.from_numpy(vos), fc_vos=fc, exact_solve=exact,
                                      **sig)
        far, wf = optimize_pose_windows(torch.from_numpy(poses), torch.from_numpy(vos), fc_vos=fc, exact_solve=exact,
                                        robust_c=1e300, **sig)
        np.testing.assert_allclose(far.cpu().numpy(), plain.cpu().numpy(), rtol=0, atol=1e-12)
        assert (wf == 1.0).all()


@pytest.mark.parametrize("N", [2, 3, 7, 16])
@pytest.mark.parametrize("fc", [False, True])
def test_covariance_kernel_matches_the_irls_oracle_and_is_reproducible(N, fc):
    from geomapnet_b200.common.pgo import optimize_pose_windows_cov
    poses, S7s, vos = _batch(N, fc, 3, 200 + N + fc)
    args = [torch.from_numpy(a) for a in (poses, S7s, vos)]
    run = lambda: [t.cpu().numpy() for t in optimize_pose_windows_cov(*args, fc_vos=fc, srx=2.0, srq=3.0,
                                                                      robust_c=C_COV)]
    got, cov, w = run()
    assert w.min() < 0.95, w.min()
    for k in range(3):
        want, want_cov, ww = optimize_cov_robust(poses[k], S7s[k], vos[k], fc, 2.0, 3.0, c=C_COV)
        np.testing.assert_allclose(got[k], want, rtol=0, atol=1e-10, err_msg=str((N, fc, k)))
        np.testing.assert_allclose(cov[k], want_cov, rtol=1e-8, atol=1e-8 * np.abs(want_cov).max(), err_msg=str(k))
        np.testing.assert_allclose(w[k], ww, rtol=0, atol=1e-10, err_msg=str((N, fc, k)))
    again = run()
    for a, b in zip(again, (got, cov, w)):
        assert np.array_equal(a, b)
    plain = optimize_pose_windows_cov(*args, fc_vos=fc, srx=2.0, srq=3.0)
    far = optimize_pose_windows_cov(*args, fc_vos=fc, srx=2.0, srq=3.0, robust_c=1e300)
    for a, b in zip(far[:2], plain):
        np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=0, atol=1e-12)
    assert (far[2] == 1.0).all()


# ---------------------------------------------------------------------------------------------------------------------
# 2. trackers against evaluate_sequence(robust_c=...)
# ---------------------------------------------------------------------------------------------------------------------
from test_gpu_track import seq, _chunks, _assert_bitwise, MEAN, STD, POSE_M, POSE_S, SIG, L_SEQ  # noqa: E402


def _point_model(droprate=0.0):
    from oracle import weights
    from helpers import make_product_model
    model, _ = make_product_model(weights.make_state(5), "mapnet", "bf16", droprate=droprate)
    return model


def _steps(trk, frames, vo, sizes, now):
    """(every pose of the sequence, flush included; the zero-lag rows when now)"""
    outs, nows, lo = [], [], 0
    for n in sizes:
        if now:
            nw, _, p = trk.step(frames[lo:lo + n], vo[lo:lo + n])
            nows.append(nw)
        else:
            _, p = trk(frames[lo:lo + n], vo[lo:lo + n])
        outs.append(p)
        lo += n
    outs.append(trk.flush()[1])
    cat = (lambda xs: torch.cat(xs)) if torch.is_tensor(outs[0]) else \
        (lambda xs: {k: torch.cat([x[k] for x in xs]) for k in xs[0]})
    return cat(outs), (cat(nows) if now else None)


@pytest.mark.parametrize("T,skip,fc", [(3, 2, False), (7, 3, True)])
def test_tracker_is_bitwise_robust_evaluate_sequence(seq, T, skip, fc):
    from geomapnet_b200.data import DeviceDataset
    from geomapnet_b200.inference import Localizer, Predictor, Tracker, evaluate_sequence
    fr, frames, poses, vo = seq
    ds = DeviceDataset(fr, MEAN, STD, poses=poses, steps=T, skip=skip, vo_poses=vo)
    pr = Predictor(_point_model(), max_batch=8)
    plain = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, **SIG)
    for zero_lag in (False, True):
        want = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, zero_lag, robust_c=C, **SIG)
        assert want["w"].shape == (L_SEQ,) and want["w"].min() < 0.9 and want["w"].max() <= 1.0
        loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
        trk = Tracker(loc, steps=T, skip=skip, vo_fc=fc, robust_c=C, **SIG)
        got, now = _steps(trk, frames, vo, _chunks(L_SEQ, 8), zero_lag)
        _assert_bitwise(now if zero_lag else got, want["pred7"], (T, skip, fc, zero_lag))
        trk.close(); loc.close()
    lagged = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, robust_c=C, **SIG)
    assert not torch.equal(lagged["pred7"], plain["pred7"])
    pr.close(); ds.close()


def test_sampled_tracker_is_bitwise_robust_evaluate_sequence(seq):
    from test_gpu_eval_sample import _dataset, _est, _twins, _assert_bitwise as _assert_est
    from test_gpu_track_sample import S, SIG as SSIG
    from geomapnet_b200.inference import Localizer, SampledTracker, evaluate_sequence
    fr, frames, poses, vo = seq
    T, skip, fc = 7, 3, True
    for zero_lag, var in ((False, False), (True, False), (False, True)):
        ds = _dataset(fr, poses, vo, steps=T, skip=skip, variable_skip=var)
        pa, pb = _twins(8, "bf16")
        got = evaluate_sequence(pa, ds, POSE_M, POSE_S, fc, zero_lag, samples=S, robust_c=C, **SSIG)
        assert got["w"].shape == (L_SEQ,) and torch.isfinite(got["w"]).all()
        if not var:
            loc = Localizer(pb, MEAN, STD, POSE_M, POSE_S)
            st = SampledTracker(loc, S, steps=T, skip=skip, vo_fc=fc, robust_c=C, **SSIG)
            est, now = _steps(st, frames, vo, _chunks(L_SEQ, 8), zero_lag)
            _assert_est(_est(got), now if zero_lag else est, ("sampled", zero_lag))
            st.close(); loc.close()
        pa.close(); pb.close(); ds.close()


def _flat(x):
    return x.reshape(x.shape[0], int(np.prod(x.shape[1:])))


def test_multi_stream_trackers_are_bitwise_single_stream_ones(seq):
    from geomapnet_b200.inference import (Localizer, MultiTracker, Predictor, SampledMultiTracker, SampledTracker,
                                          Tracker)
    from test_gpu_eval_sample import _twins
    from test_gpu_track_sample import S, SIG as SSIG
    _, frames, _, vo = seq
    T, skip, fc, K, n = 7, 3, True, 2, 40
    pr = Predictor(_point_model(), max_batch=8)
    loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
    mt = MultiTracker(loc, K, steps=T, skip=skip, vo_fc=fc, robust_c=C, **SIG)
    order = np.repeat(np.arange(K), n).reshape(K, n).T.reshape(-1)        # the streams' frames interleaved
    idx = np.concatenate([np.arange(n) + s * n for s in range(K)]).reshape(K, n).T.reshape(-1)
    rows = {s: [] for s in range(K)}
    for lo in range(0, K * n, 6):
        sid, _, p = mt(frames[idx[lo:lo + 6]], vo[idx[lo:lo + 6]], order[lo:lo + 6])
        for s in range(K):
            rows[s].append(p[(sid == s).to(p.device)])
    for s in range(K):
        got = torch.cat(rows[s] + [mt.flush(s)[1]])
        trk = Tracker(loc, steps=T, skip=skip, vo_fc=fc, robust_c=C, **SIG)
        want, _ = _steps(trk, frames[s * n:(s + 1) * n], vo[s * n:(s + 1) * n], _chunks(n, 8), False)
        _assert_bitwise(got, want, ("stream", s))
        trk.close()
    mt.close(); loc.close(); pr.close()
    # one stream of a SampledMultiTracker is the SampledTracker, given the same per-frame draws
    pa, pb = _twins(8, "bf16")
    la, lb = Localizer(pa, MEAN, STD, POSE_M, POSE_S), Localizer(pb, MEAN, STD, POSE_M, POSE_S)
    smt = SampledMultiTracker(la, S, 1, steps=T, skip=skip, vo_fc=fc, robust_c=C, **SSIG)
    st = SampledTracker(lb, S, steps=T, skip=skip, vo_fc=fc, robust_c=C, **SSIG)
    for lo, m in zip(np.cumsum([0] + _chunks(n, 8))[:-1], _chunks(n, 8)):
        _, _, a = smt(frames[lo:lo + m], vo[lo:lo + m], [0] * m)
        _, b = st(frames[lo:lo + m], vo[lo:lo + m])
        for k in b:
            _assert_bitwise(_flat(a[k]), _flat(b[k]), k)
    a, b = smt.flush(0)[1], st.flush()[1]
    for k in b:
        _assert_bitwise(_flat(a[k]), _flat(b[k]), ("flush", k))
    smt.close(); st.close(); la.close(); lb.close(); pa.close(); pb.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. launches, and the scale fixed once a handle has stepped
# ---------------------------------------------------------------------------------------------------------------------
def test_one_replay_and_three_tracking_launches_per_chunk_and_the_scale_is_fixed(seq):
    from geomapnet_b200 import _lib
    from geomapnet_b200.inference import Localizer, Predictor, Tracker
    _, frames, _, vo = seq
    pr = Predictor(_point_model(), max_batch=4)
    loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
    trk = Tracker(loc, steps=7, skip=3, vo_fc=True, robust_c=C, **SIG)
    trk(frames[:4], vo[:4])                               # captures the chunk's graph
    lib = _lib.lib()
    c0 = lib.mapnet_launch_count()
    trk(frames[4:12], vo[4:12])                           # two chunks: replays only
    assert lib.mapnet_launch_count() == c0
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        trk(frames[12:16], vo[12:16])
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    for k in ("k_track_gather<mapnet::PointFactor>", "k_pgo<true>", "k_track_emit<mapnet::PointFactor>"):
        assert sum(k in nm for nm in names) == 1, (k, names)
    assert sum("k_pgo" in nm for nm in names) == 1, names
    rc = lib.mapnet_track_set_robust(trk.h, 4.0)          # the handle has stepped: its scale stays
    assert rc != 0 and b"first step" in lib.mapnet_last_error()
    assert lib.mapnet_launch_count() == c0
    trk.close(); loc.close(); pr.close()
