"""GPU tests of inference.evaluate_sequence(samples=S), Monte-Carlo dropout on a labelled sequence: bit for bit a
SampledTracker fed the same frames at equal chunking (its step() rows under zero_lag, with and without pose
statistics), the dropout counter left where Predictor.sample leaves it, Localizer.sample's estimates without VO poses,
the composition of Predictor.sample, the tracker's factors and optimize_pose_windows_cov under variable_skip, the
device calibration scores against the float64 oracle of test_eval_sample_host, and one gather, one k_pgo_cov and one
emit launch per sequence."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from test_eval_sample_host import oracle
from test_gpu_track_sample import (MEAN, STD, POSE_M, POSE_S, SIG, S, L_SEQ, CONFIGS, _assert_close, _chunks, _factors,
                                   _pair, _rel, _tracker, _track)
from oracle import pgo_oracle as po

pytestmark = pytest.mark.gpu

EST = ("pose7", "cov", "t_std", "q_std_deg")


@pytest.fixture(scope="module")
def seq():
    """uint8 frames [L,480,640,3] (host and device), the targets (a smooth trajectory, normalised t and log q) and the
    VO library's noisy estimates of it"""
    rng = np.random.default_rng(7)
    fr = rng.integers(0, 256, (L_SEQ, 480, 640, 3), dtype=np.uint8)
    s = np.arange(L_SEQ)[:, None] / 10.0
    t = np.concatenate([np.sin(s), np.cos(0.7 * s), 0.1 * s], 1)
    lq = np.concatenate([0.2 * np.sin(0.3 * s), 0.1 * np.cos(0.5 * s), 0.05 * s], 1)
    poses = np.concatenate([t, lq], 1).astype(np.float32)
    vo = (poses + rng.standard_normal((L_SEQ, 6)) * 0.02).astype(np.float32)
    return fr, torch.from_numpy(fr).cuda(), poses, vo


def _dataset(fr, poses, vo=None, **kw):
    from geomapnet_b200.data import DeviceDataset
    return DeviceDataset(fr, MEAN, STD, poses=poses, vo_poses=vo, **kw)


def _est(got):
    return {k: got["pred7" if k == "pose7" else k] for k in EST}


def _assert_bitwise(got, want, what, keys=EST):
    for k in keys:
        assert got[k].shape == want[k].shape, (what, k, tuple(got[k].shape), tuple(want[k].shape))
        bad = (got[k] != want[k]).reshape(got[k].shape[0], -1).any(1).nonzero().flatten().tolist()
        assert not bad, (what, k, "items differ:", bad[:10])


# ---------------------------------------------------------------------------------------------------------------------
# 1. bitwise SampledTracker, 2. the dropout counter
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
def test_bitwise_sampled_tracker(seq, precision):
    fr, frames, poses, vo = seq
    for T, skip, fc in CONFIGS:
        ds = _dataset(fr, poses, vo, steps=T, skip=skip)
        for B in ((1, 8, 32) if (T, skip, fc) == CONFIGS[-1] else (8,)):
            from geomapnet_b200.inference import evaluate_sequence
            pa, pb = _twins(B, precision)
            got = evaluate_sequence(pa, ds, POSE_M, POSE_S, fc, samples=S, **SIG)
            assert got["n_frames"] == L_SEQ
            loc, st = _tracker(pb, T, skip, fc)
            want, _ = _track(st, frames, vo, _chunks(L_SEQ, B))
            _assert_bitwise(_est(got), want, (precision, T, skip, fc, B))
            st.close(); loc.close(); pa.close(); pb.close()
        ds.close()


def _twins(B, precision):
    """two Predictors of one model of `precision` with equal seeds and counters, as test_gpu_track_sample's _pair"""
    from geomapnet_b200.inference import Predictor
    from test_gpu_track_sample import _model
    model = _model(5, precision=precision)
    pa, pb = Predictor(model, max_batch=B), Predictor(model, max_batch=B)
    pa.seed = pb.seed = 20261018
    return pa, pb


def test_zero_lag_and_normalised_rows_equal_the_trackers(seq):
    from geomapnet_b200.inference import evaluate_sequence
    fr, frames, poses, vo = seq
    T, skip, fc = CONFIGS[-1]
    ds = _dataset(fr, poses, vo, steps=T, skip=skip)
    for zero_lag, metric in ((True, True), (False, False), (True, False)):
        pa, pb = _pair(8)
        stats_ = (POSE_M, POSE_S) if metric else (None, None)
        got = evaluate_sequence(pa, ds, *stats_, fc, zero_lag, samples=S, **SIG)
        loc, st = _tracker(pb, T, skip, fc, metric=metric)
        want, now = _track(st, frames, vo, _chunks(L_SEQ, 8), now=zero_lag)
        _assert_bitwise(_est(got), now if zero_lag else want, (zero_lag, metric))
        st.close(); loc.close(); pa.close(); pb.close()
    ds.close()


def test_dropout_counter_ends_where_predictor_sample_leaves_it(seq):
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.inference import evaluate_sequence
    fr, frames, poses, vo = seq
    T, skip, fc = CONFIGS[0]
    ds = _dataset(fr, poses, vo, steps=T, skip=skip)
    pa, pb = _pair(16)
    evaluate_sequence(pa, ds, POSE_M, POSE_S, fc, samples=S, **SIG)
    pipe = ImagePipeline(MEAN, STD)
    pb.sample(pipe(frames), S)                            # the same chunks of 16
    x = pipe(frames[:5])
    a, b = pa.sample(x, S, keep_samples=True), pb.sample(x, S, keep_samples=True)
    assert all(torch.equal(a[k], b[k]) for k in a)
    pa.close(); pb.close(); ds.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. without VO poses: Localizer.sample
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("steps", [None, 3])
def test_without_vo_poses_the_estimates_are_localizer_samples(seq, steps):
    from geomapnet_b200.inference import Localizer, evaluate_sequence
    fr, frames, poses, _ = seq
    ds = _dataset(fr, poses, steps=steps, skip=2)
    for metric in (False, True):
        pa, pb = _pair(8)
        stats_ = (POSE_M, POSE_S) if metric else ()
        got = evaluate_sequence(pa, ds, *stats_, samples=S)
        loc = Localizer(pb, MEAN, STD, *stats_)
        want = loc.sample(frames, S)
        if not metric:
            _assert_bitwise(_est(got), want, (steps, metric))
        else:
            _assert_bitwise(_est(got), want, (steps, metric), ("cov", "t_std", "q_std_deg"))
            assert torch.equal(got["pred7"][:, 3:], want["pose7"][:, 3:])
            assert _rel(got["pred7"][:, :3].cpu(), want["pose7"][:, :3].cpu()) <= 1e-15
        loc.close(); pa.close(); pb.close()
    ds.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. variable_skip against the composition, 5. the device scores against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _compose(mean, cov, vo, windows, fc, keep):
    """each window's slots from the tracker's factors (mapnet_test_sample_factor), its VOs (mapnet_eval_windows),
    optimize_pose_windows_cov, slot `keep`, metric: dict(pose7, cov, t_std, q_std_deg)"""
    from geomapnet_b200 import _lib
    from geomapnet_b200.common.pgo import optimize_pose_windows_cov
    n, (W, T) = mean.shape[0], windows.shape
    p7, s7 = _factors(mean, cov, SIG["sax"], SIG["saq"])
    pairs = po.edges(T, fc)
    vo_rows = np.ascontiguousarray(windows[:, np.asarray(pairs)], dtype=np.int32)
    E = len(pairs)
    vo_dev = torch.as_tensor(vo[:n]).cuda().contiguous()
    dummy = torch.zeros((n, 6), dtype=torch.float32, device="cuda")
    w7, t7 = (torch.empty((W, T, 7), dtype=torch.float64, device="cuda") for _ in range(2))
    vos7 = torch.empty((W, E, 7), dtype=torch.float64, device="cuda")
    flat = np.ascontiguousarray(windows.reshape(-1), dtype=np.int32)
    _lib.check(_lib.lib().mapnet_eval_windows(dummy.data_ptr(), n, dummy.data_ptr(), vo_dev.data_ptr(), n,
                                              flat.ctypes.data, flat.ctypes.data, W * T, vo_rows.ctypes.data, W * E,
                                              w7.data_ptr(), t7.data_ptr(), vos7.data_ptr(), _lib.stream_ptr()),
               "mapnet_eval_windows")
    ix = torch.from_numpy(windows.astype(np.int64)).cuda()
    z, cv = optimize_pose_windows_cov(p7[ix], s7[ix], vos7, fc_vos=fc, srx=SIG["srx"], srq=SIG["srq"])
    z, cv = z[:, keep], cv[:, keep]
    d = torch.tensor(list(POSE_S) + [1.0] * 3, dtype=torch.float64, device="cuda")
    m = torch.tensor(POSE_M, dtype=torch.float64, device="cuda")
    z = torch.cat((z[:, :3] * d[:3] + m, z[:, 3:]), -1)
    cv = d[:, None] * cv * d[None, :]
    tt = cv[:, 0, 0] + cv[:, 1, 1] + cv[:, 2, 2]
    tq = cv[:, 3, 3] + cv[:, 4, 4] + cv[:, 5, 5]
    return dict(pose7=z, cov=cv, t_std=tt.sqrt(), q_std_deg=2.0 * tq.sqrt() * (180.0 / math.pi))


def test_variable_skip_equals_the_composition_and_scores_match_the_oracle(seq):
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.inference import evaluate_sequence
    fr, frames, poses, vo = seq
    T, skip, fc = 5, 3, True
    ds = _dataset(fr, poses, vo, steps=T, skip=skip, variable_skip=True)
    pa, pb = _pair(16)
    np.random.seed(4)
    got = evaluate_sequence(pa, ds, POSE_M, POSE_S, fc, samples=S, **SIG)
    np.random.seed(4)
    windows = ds.eval_tables(vo_fc=fc)["windows"]
    assert len(set(np.diff(windows, axis=1).ravel().tolist())) > 1          # the skips do vary
    out = pb.sample(ImagePipeline(MEAN, STD)(frames), S)
    want = _compose(out["mean"].cpu().numpy(), out["cov"].cpu().numpy(), vo, windows, fc, T // 2)
    _assert_close(_est(got), want, "variable_skip")
    # the targets: poses[i] (the middle slot of window i), qexp'd as mapnet_eval_windows, un-normalised
    t = poses.astype(np.float64)
    n = np.linalg.norm(poses[:, 3:].astype(np.float32), axis=1).astype(np.float64)
    targ = got["targ7"].cpu().numpy()
    assert np.array_equal(targ[:, :3], t[:, :3] * np.asarray(POSE_S) + np.asarray(POSE_M))
    assert np.abs(targ[:, 3] - np.cos(n)).max() < 1e-7
    te, qe = got["t_err"].cpu().numpy(), got["q_err"].cpu().numpy()
    p = got["pred7"].cpu().numpy()
    np.testing.assert_allclose(te, np.linalg.norm(p[:, :3] - targ[:, :3], axis=1), rtol=1e-14)
    dq = np.clip(np.abs((p[:, 3:] * targ[:, 3:]).sum(1)), -1, 1)
    np.testing.assert_allclose(qe, 2 * np.arccos(dq) * 180 / np.pi, rtol=1e-12, atol=1e-12)
    # 5. the device scores against the float64 oracle, at the host tolerances
    d2, u, nll = (got[k].cpu().numpy() for k in ("d2", "u", "nll"))
    cov = got["cov"].cpu().numpy()
    assert np.isfinite(d2).all() and np.isfinite(nll).all()
    for i in range(L_SEQ):
        _, wd2, wnll = oracle(p[i], targ[i], cov[i])
        np.testing.assert_allclose(d2[i], wd2, rtol=1e-12, err_msg=str(i))
        np.testing.assert_allclose(nll[i], wnll, rtol=1e-12, err_msg=str(i))
        np.testing.assert_allclose(u[i], stats.chi2.cdf(d2[i], [6, 3, 3]), rtol=0, atol=1e-13, err_msg=str(i))
    pa.close(); pb.close(); ds.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. launches
# ---------------------------------------------------------------------------------------------------------------------
def test_one_gather_one_pgo_and_one_emit_per_sequence(seq):
    from geomapnet_b200.inference import evaluate_sequence
    fr, _, poses, vo = seq
    T, skip, fc = CONFIGS[-1]
    for use_vo in (True, False):
        ds = _dataset(fr, poses, vo if use_vo else None, steps=T, skip=skip)
        pa, _ = _pair(16)
        evaluate_sequence(pa, ds, POSE_M, POSE_S, fc and use_vo, samples=S, **SIG)     # captures the graphs
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            evaluate_sequence(pa, ds, POSE_M, POSE_S, fc and use_vo, samples=S, **SIG)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        count = lambda k: sum(k in n for n in names)
        assert count("k_eval_sample_emit") == 1, names
        assert count("k_eval_sample_windows") == (1 if use_vo else 0), names
        assert count("k_pgo_cov") == (1 if use_vo else 0), names
        assert count("k_pgo") == count("k_pgo_cov") and count("k_eval_windows") == 0
        assert count("k_head_draws") == len(_chunks(L_SEQ, 16)), names                 # one engine replay per chunk
        pa.close(); ds.close()
