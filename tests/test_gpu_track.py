"""GPU tests of inference.Tracker (MapNet+PGO over a camera stream, csrc/loader.cu mapnet_track_*): bit for bit
evaluate_sequence on a DeviceDataset of the same frames at equal chunking, bit for bit the composition of the same
Predictor calls with mapnet_eval_windows, pgo and the un-normalisation for any call sizes, with dropout, across reset /
flush / refresh and in fp8, and one graph replay of the engine's launches plus three tracking launches per chunk."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# data/7Scenes/chess/stats.txt of the reference: row 0 the mean, row 1 the variance (Normalize takes its square root)
MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]
STD = [float(np.sqrt(v)) for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
POSE_M, POSE_S = [0.5, -1.25, 2.0], [1.5, 0.75, 2.5]
SIG = dict(sax=1.0, saq=0.5, srx=20.0, srq=20.0)
L_SEQ, H_IN, W_IN = 97, 480, 640
CONFIGS = [(3, 2, False), (4, 5, False), (7, 3, True)]          # (steps, skip, vo_fc)


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


def _track(trk, frames, vo, sizes):
    """every pose of the sequence: the calls of `sizes` frames, then flush; checks the emitted ranges as it goes"""
    out, nxt, lo = [], 0, 0
    for n in sizes:
        first, p = trk(frames[lo:lo + n], vo[lo:lo + n])
        assert first == nxt and p.dtype == torch.float64 and p.shape[1] == 7 and p.is_cuda, (first, nxt)
        assert p.shape[0] == max(lo + n - trk.lag, 0) - max(lo - trk.lag, 0)
        out.append(p)
        nxt += p.shape[0]
        lo += n
    first, p = trk.flush()
    assert first == nxt and nxt + p.shape[0] == lo and trk.seen == 0
    return torch.cat(out + [p])


def _chunks(L, B):
    return [min(B, L - lo) for lo in range(0, L, B)]


def _composition(pr, frames, vo, sizes, T, skip, fc, metric=True):
    """ImagePipeline -> Predictor (one call per entry of sizes) -> eval.py's windows (mapnet_eval_windows) -> pgo ->
    the middle slot, un-normalised as _window_errors does"""
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.data.tuples import mf_indices
    from geomapnet_b200.inference import pgo
    pipe = ImagePipeline(MEAN, STD)
    los = np.cumsum([0] + list(sizes))
    pred6 = torch.cat([pr(pipe(frames[a:b])) for a, b in zip(los[:-1], los[1:])]).contiguous()
    L = pred6.shape[0]
    windows = np.ascontiguousarray(np.stack([mf_indices(i, L, T, skip) for i in range(L)]), dtype=np.int32)
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
    mid = pgo(pred7, vos7, fc_vos=fc, **SIG)[:, T // 2]
    if not metric:
        return mid
    m = torch.as_tensor(np.asarray(POSE_M, dtype=np.float64), device="cuda")
    s = torch.as_tensor(np.asarray(POSE_S, dtype=np.float64), device="cuda")
    return torch.cat((mid[:, :3] * s + m, mid[:, 3:]), -1)


def _assert_bitwise(got, want, what):
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    bad = (got != want).any(1).nonzero().flatten().tolist()
    assert not bad, (what, "frames differ:", bad[:10], float((got - want).abs().max()))


# ---------------------------------------------------------------------------------------------------------------------
# 1. bitwise evaluate_sequence, 2. a sequence shorter than the lag
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
def test_tracker_is_bitwise_evaluate_sequence(precision, seq):
    from geomapnet_b200.data import DeviceDataset
    from geomapnet_b200.inference import Predictor, evaluate_sequence
    fr, frames, poses, vo = seq
    model = _model(precision)
    for T, skip, fc in CONFIGS:
        ds = DeviceDataset(fr, MEAN, STD, poses=poses, steps=T, skip=skip, vo_poses=vo)
        for B in (1, 8, 32):
            pr = Predictor(model, max_batch=B)
            want = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, **SIG)["pred7"]
            loc, trk = _tracker(pr, T, skip, fc)
            got = _track(trk, frames, vo, _chunks(L_SEQ, B))
            _assert_bitwise(got, want, (precision, T, skip, fc, B))
            trk.close(); loc.close(); pr.close()
        ds.close()


def test_a_sequence_shorter_than_the_lag_comes_out_of_flush(seq):
    from geomapnet_b200.data import DeviceDataset
    from geomapnet_b200.inference import Predictor, evaluate_sequence
    fr, frames, poses, vo = seq
    T, skip, fc, L = 7, 3, True, 6                        # lag 9
    pr = Predictor(_model("bf16"), max_batch=4)
    ds = DeviceDataset(fr[:L], MEAN, STD, poses=poses[:L], steps=T, skip=skip, vo_poses=vo[:L])
    want = evaluate_sequence(pr, ds, POSE_M, POSE_S, fc, **SIG)["pred7"]
    loc, trk = _tracker(pr, T, skip, fc)
    for lo, n in ((0, 4), (4, 2)):
        first, p = trk(frames[lo:lo + n], vo[lo:lo + n])
        assert first == 0 and p.shape == (0, 7)
    first, got = trk.flush()
    assert first == 0
    _assert_bitwise(got, want, "shorter than the lag")
    trk.close(); loc.close(); pr.close(); ds.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. any call sizes, 4. dropout
# ---------------------------------------------------------------------------------------------------------------------
SIZES = [1, 8, 3, 13, 5, 8, 2, 1, 7]                      # 13 > max_batch: two chunks


@pytest.mark.parametrize("T,skip,fc", CONFIGS)
def test_varying_call_sizes_equal_the_composition_of_those_calls(seq, T, skip, fc):
    from geomapnet_b200.inference import Predictor
    _, frames, _, vo = seq
    pr = Predictor(_model("bf16"), max_batch=8)
    loc, trk = _tracker(pr, T, skip, fc)
    got = _track(trk, frames, vo, SIZES)
    _assert_bitwise(got, _composition(pr, frames, vo, SIZES, T, skip, fc), (T, skip, fc))
    # without pose_m / pose_s the translations stay normalised
    plain, trk2 = _tracker(pr, T, skip, fc, metric=False)
    _assert_bitwise(_track(trk2, frames, vo, SIZES), _composition(pr, frames, vo, SIZES, T, skip, fc, metric=False),
                    "normalised")
    trk.close(); trk2.close(); loc.close(); plain.close(); pr.close()


def test_dropout_windows_reuse_each_frames_one_draw(seq):
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.inference import Predictor
    _, frames, _, vo = seq
    T, skip, fc = 4, 5, False
    pa = Predictor(_model("bf16", seed=3, droprate=0.5), max_batch=8)
    pb = Predictor(_model("bf16", seed=3, droprate=0.5), max_batch=8)
    pb.seed = pa.seed
    loc, trk = _tracker(pa, T, skip, fc)
    got = _track(trk, frames, vo, SIZES)
    _assert_bitwise(got, _composition(pb, frames, vo, SIZES, T, skip, fc), "droprate 0.5")
    # the counters end equal: the next forward of either draws the same mask
    pipe = ImagePipeline(MEAN, STD)
    from geomapnet_b200.inference import post
    f = frames[:3]
    assert torch.equal(loc(f), post(pb(pipe(f)), POSE_M, POSE_S))
    trk.close(); loc.close(); pa.close(); pb.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. reset / flush, refresh, fp8
# ---------------------------------------------------------------------------------------------------------------------
def test_reset_and_flush_start_a_new_sequence(seq):
    from geomapnet_b200.inference import Predictor
    _, frames, _, vo = seq
    T, skip, fc = 7, 3, True
    pr = Predictor(_model("bf16"), max_batch=8)
    loc, trk = _tracker(pr, T, skip, fc)
    _, fresh = _tracker(pr, T, skip, fc)
    a, b = frames[40:80], vo[40:80]
    want = _track(fresh, a, b, _chunks(40, 8))
    trk(frames[:21], vo[:21])                             # an abandoned sequence
    trk.reset()
    assert trk.seen == 0
    _assert_bitwise(_track(trk, a, b, _chunks(40, 8)), want, "after reset")
    _assert_bitwise(_track(trk, a, b, _chunks(40, 8)), want, "after flush")
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
    before = _track(trk, frames, vo, sizes)
    opt = Optimizer(params=model.parameters(), method="adam", base_lr=1e-2, weight_decay=0.0)
    model.train()
    x = torch.randn(2, 2, 3, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    out = model(x.requires_grad_(True))
    opt.learner.zero_grad()
    out.square().sum().backward()
    opt.learner.step()
    assert torch.equal(_track(trk, frames, vo, sizes), before)      # frozen until refresh
    pr.refresh()
    after = _track(trk, frames, vo, sizes)
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
    _assert_bitwise(_track(trk, frames, vo, sizes), _composition(pr, frames, vo, sizes, T, skip, fc), "fp8")
    trk.close(); loc.close(); pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. launches and captures; input forms
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
        trk(frames[lo:lo + B], vo[lo:lo + B])
        c1 = lib.mapnet_launch_count()
        assert c1 - c0 == (2 + 43) + (2 + 43 + 3), (B, c1 - c0)
        lo += B
    n_graphs = len(trk._graphs)
    assert n_graphs == 2
    c1 = lib.mapnet_launch_count()
    for B in (4, 1, 4, 4, 1):
        trk(frames[lo:lo + B], vo[lo:lo + B])
        lo += B
    trk(frames[lo:lo + 9], vo[lo:lo + 9])                  # chunks of 4, 4 and 1
    assert lib.mapnet_launch_count() == c1 and len(trk._graphs) == n_graphs
    trk.close(); loc.close(); pr.close()


def test_host_frames_arrays_and_single_frames_agree(seq):
    from geomapnet_b200.inference import Predictor
    fr, frames, _, vo = seq
    pr = Predictor(_model("bf16"), max_batch=4)
    loc, trk = _tracker(pr, 3, 2, False)
    want = _track(trk, frames, vo, [4, 4, 4])
    got = []
    for i in range(12):                                   # one [H,W,3] frame and one [6] VO pose per call
        f = fr[i] if i % 3 == 0 else (torch.from_numpy(fr[i]) if i % 3 == 1 else frames[i])
        v = vo[i].astype(np.float64) if i % 2 else torch.from_numpy(vo[i])
        got.append(trk(f, v)[1])
    got.append(trk.flush()[1])
    _assert_bitwise(torch.cat(got), want, "single frames")
    trk.close(); loc.close(); pr.close()
