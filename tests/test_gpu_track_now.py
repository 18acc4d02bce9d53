"""GPU tests of the zero-lag tracker output (Tracker.step, csrc/loader.cu mapnet_track_step_now): every frame's pose
from the window that ends at it, in the call that brings it.  Bit for bit evaluate_sequence(zero_lag=True) at equal
chunking, bit for bit the composition of the same Predictor calls with mapnet_eval_windows, pgo, slot steps-1 and the
un-normalisation for any call sizes, with dropout, mixed with lagged calls, across reset / flush / refresh and in fp8;
the same launches per chunk as a lagged call; and the reference's PGO (oracle/pgo_oracle.py) on the same windows."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# the fixtures of test_gpu_track.py: data/7Scenes/chess/stats.txt of the reference (row 0 the mean, row 1 the
# variance, which Normalize takes the square root of), a 97-frame 480x640 sequence, three (steps, skip, vo_fc)
MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]
STD = [float(np.sqrt(v)) for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
POSE_M, POSE_S = [0.5, -1.25, 2.0], [1.5, 0.75, 2.5]
SIG = dict(sax=1.0, saq=0.5, srx=20.0, srq=20.0)
L_SEQ, H_IN, W_IN = 97, 480, 640
CONFIGS = [(3, 2, False), (4, 5, False), (7, 3, True)]          # (steps, skip, vo_fc): lags 2, 5, 9
SIZES = [1, 8, 3, 13, 5, 8, 2, 1, 7]                             # 13 > max_batch = 8: two chunks


@pytest.fixture(scope="module")
def seq():
    """uint8 frames [L,480,640,3], a smooth trajectory (normalised t, log q) as the targets and the VO library's noisy
    estimates of it"""
    rng = np.random.default_rng(7)
    fr = rng.integers(0, 256, (L_SEQ, H_IN, W_IN, 3), dtype=np.uint8)
    s = np.arange(L_SEQ)[:, None] / 10.0
    t = np.concatenate([np.sin(s), np.cos(0.7 * s), 0.1 * s], 1)
    lq = np.concatenate([0.2 * np.sin(0.3 * s), 0.1 * np.cos(0.5 * s), 0.05 * s], 1)
    poses = np.concatenate([t, lq], 1).astype(np.float32)
    vo = (poses + rng.standard_normal(poses.shape) * 0.02).astype(np.float32)
    return fr, torch.from_numpy(fr).cuda(), poses, vo


def _model(precision, seed=5, droprate=0.0):
    from oracle import weights
    from helpers import make_product_model
    model, _ = make_product_model(weights.make_state(seed), "mapnet", precision, droprate=droprate)
    return model


def _tracker(pr, T, skip, fc, metric=True):
    from geomapnet_b200.inference import Localizer, Tracker
    loc = Localizer(pr, MEAN, STD, *((POSE_M, POSE_S) if metric else ()))
    return loc, Tracker(loc, steps=T, skip=skip, vo_fc=fc, **SIG)


def _chunks(L, B):
    return [min(B, L - lo) for lo in range(0, L, B)]


def _track(trk, frames, vo, sizes, steps=None):
    """(every zero-lag pose [L,7] of the step calls, every smoothed pose [L,7]): calls of `sizes` frames (step() where
    steps[k], else a lagged call), then flush; checks the emitted ranges as it goes"""
    nows, out, nxt, lo = [], [], 0, 0
    for k, n in enumerate(sizes):
        if steps is None or steps[k]:
            now, first, p = trk.step(frames[lo:lo + n], vo[lo:lo + n])
            assert now.dtype == torch.float64 and now.shape == (n, 7) and now.is_cuda
            nows.append(now)
        else:
            first, p = trk(frames[lo:lo + n], vo[lo:lo + n])
        assert first == nxt and p.dtype == torch.float64 and p.shape[1] == 7 and p.is_cuda, (first, nxt)
        assert p.shape[0] == max(lo + n - trk.lag, 0) - max(lo - trk.lag, 0)
        out.append(p)
        nxt += p.shape[0]
        lo += n
    first, p = trk.flush()
    assert first == nxt and nxt + p.shape[0] == lo and trk.seen == 0
    return (torch.cat(nows) if nows else None), torch.cat(out + [p])


def _windows(pr, frames, vo, sizes, T, skip, fc, zero_lag):
    """ImagePipeline -> Predictor (one call per entry of sizes) -> the windows (eval.py's, or those that end at each
    frame) through mapnet_eval_windows: (pred7 [L,T,7], vos7 [L,E,7]) as k_pgo takes them"""
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.data.tuples import mf_indices
    pipe = ImagePipeline(MEAN, STD)
    los = np.cumsum([0] + list(sizes))
    pred6 = torch.cat([pr(pipe(frames[a:b])) for a, b in zip(los[:-1], los[1:])]).contiguous()
    L = pred6.shape[0]
    lag = (T - 1 - T // 2) * skip if zero_lag else 0
    windows = np.ascontiguousarray(np.stack([mf_indices(i - lag, L, T, skip) for i in range(L)]), dtype=np.int32)
    pairs = [(i, j) for i in range(T) for j in range(i + 1, T)] if fc else [(i, i + 1) for i in range(T - 1)]
    vo_rows = np.ascontiguousarray(windows[:, np.asarray(pairs)], dtype=np.int32)
    E = vo_rows.shape[1]
    vo_dev = torch.as_tensor(vo[:L]).cuda().contiguous()
    pred7 = torch.empty((L, T, 7), dtype=torch.float64, device="cuda")
    targ7, vos7 = torch.empty_like(pred7), torch.empty((L, E, 7), dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().mapnet_eval_windows(
        pred6.data_ptr(), L, pred6.data_ptr(), vo_dev.data_ptr(), L, windows.ctypes.data, windows.ctypes.data, L * T,
        vo_rows.ctypes.data, L * E, pred7.data_ptr(), targ7.data_ptr(), vos7.data_ptr(), _lib.stream_ptr()),
        "mapnet_eval_windows")
    return pred7, vos7


def _composition(pr, frames, vo, sizes, T, skip, fc, metric=True, zero_lag=True):
    """_windows -> pgo -> slot T-1 (zero_lag) or T//2, un-normalised as _window_errors does"""
    from geomapnet_b200.inference import pgo
    pred7, vos7 = _windows(pr, frames, vo, sizes, T, skip, fc, zero_lag)
    keep = pgo(pred7, vos7, fc_vos=fc, **SIG)[:, T - 1 if zero_lag else T // 2]
    if not metric:
        return keep
    m = torch.as_tensor(np.asarray(POSE_M, dtype=np.float64), device="cuda")
    s = torch.as_tensor(np.asarray(POSE_S, dtype=np.float64), device="cuda")
    return torch.cat((keep[:, :3] * s + m, keep[:, 3:]), -1)


def _assert_bitwise(got, want, what):
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    bad = (got != want).any(1).nonzero().flatten().tolist()
    assert not bad, (what, "frames differ:", bad[:10], float((got - want).abs().max()))


# ---------------------------------------------------------------------------------------------------------------------
# 1. bitwise evaluate_sequence(zero_lag=True), 3. a sequence shorter than the lag
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
def test_step_is_bitwise_zero_lag_evaluate_sequence(precision, seq):
    from geomapnet_b200.data import DeviceDataset
    from geomapnet_b200.inference import Predictor, evaluate_sequence
    fr, frames, poses, vo = seq
    model = _model(precision)
    for T, skip, fc in CONFIGS:
        ds = DeviceDataset(fr, MEAN, STD, poses=poses, steps=T, skip=skip, vo_poses=vo)
        for B in (1, 8, 32):
            pr = Predictor(model, max_batch=B)
            want = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, zero_lag=True, **SIG)
            loc, trk = _tracker(pr, T, skip, fc)
            now, smoothed = _track(trk, frames, vo, _chunks(L_SEQ, B))
            _assert_bitwise(now, want["pred7"], (precision, T, skip, fc, B))
            _, fresh = _tracker(pr, T, skip, fc)
            _assert_bitwise(smoothed, _track(fresh, frames, vo, _chunks(L_SEQ, B), steps=[False] * 99)[1],
                            ("smoothed", precision, T, skip, fc, B))
            trk.close(); fresh.close(); loc.close(); pr.close()
        ds.close()


def test_zero_lag_evaluation_keeps_the_last_slot_and_its_target(seq):
    """evaluate_sequence(zero_lag=True) errors are those of the last slot against the frame's own target: the target
    the middle slot of eval.py's window of the same frame holds"""
    from geomapnet_b200.data import DeviceDataset
    from geomapnet_b200.inference import Predictor, evaluate_sequence, pose_errors
    fr, _, poses, vo = seq
    T, skip, fc, L = 7, 3, True, 40
    ds = DeviceDataset(fr[:L], MEAN, STD, poses=poses[:L], steps=T, skip=skip, vo_poses=vo[:L])
    pr = Predictor(_model("bf16"), max_batch=8)
    got = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, zero_lag=True, **SIG)
    lagged = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, **SIG)
    _assert_bitwise(got["targ7"], lagged["targ7"], "targets")
    assert not torch.equal(got["pred7"], lagged["pred7"])
    t_err, q_err = pose_errors(got["pred7"], got["targ7"])
    assert torch.equal(got["t_err"], t_err) and torch.equal(got["q_err"], q_err) and got["n_frames"] == L
    pr.close(); ds.close()


def test_a_sequence_shorter_than_the_lag_gets_every_zero_lag_pose_in_its_call(seq):
    from geomapnet_b200.data import DeviceDataset
    from geomapnet_b200.inference import Predictor, evaluate_sequence
    fr, frames, poses, vo = seq
    T, skip, fc, L = 7, 3, True, 6                        # lag 9
    pr = Predictor(_model("bf16"), max_batch=4)
    ds = DeviceDataset(fr[:L], MEAN, STD, poses=poses[:L], steps=T, skip=skip, vo_poses=vo[:L])
    want_now = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, zero_lag=True, **SIG)["pred7"]
    want = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, **SIG)["pred7"]
    loc, trk = _tracker(pr, T, skip, fc)
    for lo, n in ((0, 4), (4, 2)):
        now, first, p = trk.step(frames[lo:lo + n], vo[lo:lo + n])
        assert first == 0 and p.shape == (0, 7)
        _assert_bitwise(now, want_now[lo:lo + n], ("zero-lag, frames", lo, n))
    first, got = trk.flush()
    assert first == 0
    _assert_bitwise(got, want, "flush")
    trk.close(); loc.close(); pr.close(); ds.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. any call sizes, 4. dropout
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,skip,fc", CONFIGS)
def test_varying_call_sizes_equal_the_composition_of_those_calls(seq, T, skip, fc):
    from geomapnet_b200.inference import Predictor
    _, frames, _, vo = seq
    pr = Predictor(_model("bf16"), max_batch=8)
    for metric in (True, False):                          # without pose_m / pose_s the translations stay normalised
        loc, trk = _tracker(pr, T, skip, fc, metric)
        now, smoothed = _track(trk, frames, vo, SIZES)
        _assert_bitwise(now, _composition(pr, frames, vo, SIZES, T, skip, fc, metric), (T, skip, fc, metric))
        _assert_bitwise(smoothed, _composition(pr, frames, vo, SIZES, T, skip, fc, metric, zero_lag=False),
                        ("smoothed", T, skip, fc, metric))
        trk.close(); loc.close()
    pr.close()


def test_dropout_windows_reuse_each_frames_one_draw(seq):
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.inference import Predictor, post
    _, frames, _, vo = seq
    T, skip, fc = 4, 5, False
    pa = Predictor(_model("bf16", seed=3, droprate=0.5), max_batch=8)
    pb = Predictor(_model("bf16", seed=3, droprate=0.5), max_batch=8)
    pb.seed = pa.seed
    loc, trk = _tracker(pa, T, skip, fc)
    now, _ = _track(trk, frames, vo, SIZES)
    _assert_bitwise(now, _composition(pb, frames, vo, SIZES, T, skip, fc), "droprate 0.5")
    # the counters end equal: the next forward of either draws the same mask
    f = frames[:3]
    assert torch.equal(loc(f), post(pb(ImagePipeline(MEAN, STD)(f)), POSE_M, POSE_S))
    trk.close(); loc.close(); pa.close(); pb.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. mixed calls, reset / flush, refresh, fp8
# ---------------------------------------------------------------------------------------------------------------------
def test_mixed_calls_and_steps_share_one_sequence(seq):
    from geomapnet_b200.inference import Predictor
    _, frames, _, vo = seq
    T, skip, fc = 7, 3, True
    pr = Predictor(_model("bf16"), max_batch=8)
    loc, trk = _tracker(pr, T, skip, fc)
    now_all, smoothed_all = _track(trk, frames, vo, SIZES)
    for steps in ([k % 2 == 0 for k in range(len(SIZES))], [k % 2 == 1 for k in range(len(SIZES))]):
        now, smoothed = _track(trk, frames, vo, SIZES, steps)
        _assert_bitwise(smoothed, smoothed_all, ("smoothed", steps))
        los = np.cumsum([0] + SIZES)
        want = torch.cat([now_all[los[k]:los[k + 1]] for k in range(len(SIZES)) if steps[k]])
        _assert_bitwise(now, want, ("zero-lag", steps))
    # reset and flush start a new sequence
    a, b = frames[40:80], vo[40:80]
    _, fresh = _tracker(pr, T, skip, fc)
    want = _track(fresh, a, b, _chunks(40, 8))
    trk.step(frames[:21], vo[:21])                        # an abandoned sequence
    trk.reset()
    assert trk.seen == 0
    for what in ("after reset", "after flush"):
        got = _track(trk, a, b, _chunks(40, 8))
        _assert_bitwise(got[0], want[0], ("zero-lag", what))
        _assert_bitwise(got[1], want[1], ("smoothed", what))
    fresh.close(); trk.close(); loc.close(); pr.close()


def test_refresh_changes_the_output_to_the_new_snapshot(seq):
    from geomapnet_b200.common.optimizer import Optimizer
    from geomapnet_b200.inference import Predictor
    _, frames, _, vo = seq
    T, skip, fc = 4, 5, False
    model = _model("bf16", seed=9)
    pr = Predictor(model, max_batch=8)
    loc, trk = _tracker(pr, T, skip, fc)
    sizes = _chunks(30, 8)
    before = _track(trk, frames, vo, sizes)[0]
    opt = Optimizer(params=model.parameters(), method="adam", base_lr=1e-2, weight_decay=0.0)
    model.train()
    x = torch.randn(2, 2, 3, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    out = model(x.requires_grad_(True))
    opt.learner.zero_grad()
    out.square().sum().backward()
    opt.learner.step()
    assert torch.equal(_track(trk, frames, vo, sizes)[0], before)      # frozen until refresh
    pr.refresh()
    after = _track(trk, frames, vo, sizes)[0]
    assert not torch.equal(after, before)
    _assert_bitwise(after, _composition(pr, frames, vo, sizes, T, skip, fc), "refreshed")
    trk.close(); loc.close(); pr.close()


def test_fp8_predictor_equals_its_own_composition(seq):
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.inference import Predictor
    _, frames, _, vo = seq
    T, skip, fc = 7, 3, True
    pr = Predictor(_model("bf16"), max_batch=8, precision="fp8", calibration=ImagePipeline(MEAN, STD)(frames[:8]))
    loc, trk = _tracker(pr, T, skip, fc)
    sizes = _chunks(40, 8)
    _assert_bitwise(_track(trk, frames, vo, sizes)[0], _composition(pr, frames, vo, sizes, T, skip, fc), "fp8")
    trk.close(); loc.close(); pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. launches and captures, argument errors on a live handle
# ---------------------------------------------------------------------------------------------------------------------
def test_one_replay_of_the_engine_and_three_tracking_launches_per_chunk(seq):
    """2 preprocess + 43 engine launches in the eager run before the capture, the same 45 + gather, k_pgo and emit in
    the capture; a replay makes no library call, and a shape met before makes no new capture"""
    from geomapnet_b200 import _lib
    from geomapnet_b200.inference import Predictor
    _, frames, _, vo = seq
    lib = _lib.lib()
    pr = Predictor(_model("bf16"), max_batch=4)
    loc, trk = _tracker(pr, 4, 5, False)
    pr._engine(256, 341)                                  # the engine's creation and snapshot load are not counted
    lo = 0
    for B in (1, 4):
        c0 = lib.mapnet_launch_count()
        trk.step(frames[lo:lo + B], vo[lo:lo + B])
        c1 = lib.mapnet_launch_count()
        assert c1 - c0 == (2 + 43) + (2 + 43 + 3), (B, c1 - c0)
        lo += B
    assert len(trk._now_graphs) == 2 and not trk._graphs
    c1 = lib.mapnet_launch_count()
    for B in (4, 1, 4, 4, 1):
        trk.step(frames[lo:lo + B], vo[lo:lo + B])
        lo += B
    trk.step(frames[lo:lo + 9], vo[lo:lo + 9])             # chunks of 4, 4 and 1
    assert lib.mapnet_launch_count() == c1 and len(trk._now_graphs) == 2
    trk.close(); loc.close(); pr.close()


def test_step_now_refuses_frame_counts_outside_max_batch(seq):
    from geomapnet_b200 import _lib
    from geomapnet_b200.inference import Predictor
    lib = _lib.lib()
    pr = Predictor(_model("bf16"), max_batch=4)
    loc, trk = _tracker(pr, 4, 5, False)
    h = trk._handle()
    buf = torch.zeros(8, 7, dtype=torch.float64, device="cuda")
    n0 = lib.mapnet_launch_count()
    for B in (0, -1, 5):
        assert lib.mapnet_track_step_now(h, buf.data_ptr(), buf.data_ptr(), B, buf.data_ptr(), buf.data_ptr(),
                                         None) != 0
        assert b"outside [1, max_batch=4]" in lib.mapnet_last_error()
    assert lib.mapnet_launch_count() == n0
    seen, failed = ctypes.c_int64(-1), ctypes.c_int(-1)
    assert lib.mapnet_track_status(h, ctypes.byref(seen), ctypes.byref(failed), None) == 0
    assert (seen.value, failed.value) == (0, 0)
    trk.close(); loc.close(); pr.close()


def test_single_frames_and_host_arrays_agree(seq):
    from geomapnet_b200.inference import Predictor
    fr, frames, _, vo = seq
    pr = Predictor(_model("bf16"), max_batch=4)
    loc, trk = _tracker(pr, 3, 2, False)
    want = _track(trk, frames, vo, [4, 4, 4])
    nows, outs = [], []
    for i in range(12):                                   # one [H,W,3] frame and one [6] VO pose per call
        f = fr[i] if i % 3 == 0 else (torch.from_numpy(fr[i]) if i % 3 == 1 else frames[i])
        v = vo[i].astype(np.float64) if i % 2 else torch.from_numpy(vo[i])
        now, _, p = trk.step(f, v)
        assert now.shape == (1, 7)
        nows.append(now); outs.append(p)
    outs.append(trk.flush()[1])
    _assert_bitwise(torch.cat(nows), want[0], "single frames, zero-lag")
    _assert_bitwise(torch.cat(outs), want[1], "single frames, smoothed")
    trk.close(); loc.close(); pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. the reference's pose-graph optimisation
# ---------------------------------------------------------------------------------------------------------------------
# oracle/pgo_oracle.py restates the reference's PoseGraph / PoseGraphFC in numpy float64 and is pinned to them at
# 1e-11 (goldens) and 1e-12 (live classes) by test_pgo_oracle.py.  k_pgo computes the same 10 iterations in float64
# with its own summation order (shared-memory atomics, a right-looking Cholesky), and test_gpu_inference.py bounds it
# against the oracle at 1e-9 absolute on poses of the same O(1) scale as the normalised ones here.  The zero-lag
# windows are the same problems, warm-up windows included (repeated frame 0, identity VOs), so the same 1e-9 applies.
ORACLE_ATOL = 1e-9


@pytest.mark.parametrize("T,skip,fc", CONFIGS)
def test_zero_lag_poses_match_the_reference_pgo(seq, T, skip, fc):
    from oracle import pgo_oracle as P
    from geomapnet_b200.inference import Predictor
    _, frames, _, vo = seq
    L = 40
    pr = Predictor(_model("bf16"), max_batch=8)
    loc, trk = _tracker(pr, T, skip, fc, metric=False)
    sizes = _chunks(L, 8)
    now, _ = _track(trk, frames[:L], vo[:L], sizes)
    pred7, vos7 = _windows(pr, frames, vo, sizes, T, skip, fc, zero_lag=True)
    pred7, vos7, now = pred7.cpu().numpy(), vos7.cpu().numpy(), now.cpu().numpy()
    err = max(np.abs(now[i] - P.optimize(pred7[i], vos7[i], SIG["sax"], SIG["saq"], SIG["srx"], SIG["srq"],
                                         fc=fc)[T - 1]).max() for i in range(L))
    print("T=%d skip=%d fc=%s: max |now7 - oracle| = %.3e" % (T, skip, fc, err))
    assert err <= ORACLE_ATOL
    trk.close(); loc.close(); pr.close()
