"""GPU tests of Monte-Carlo dropout sampling (Predictor.sample, Localizer.sample, mapnet_infer_sample[_frames]).

The contract is bitwise: draw s of a sample call is what the (s+1)-th of S consecutive ordinary forwards of the same
frames returns, and afterwards the dropout counter stands where those S forwards leave it.  Each check runs on twin
Predictors (or Localizers) of one model: A samples, B runs the forwards, both warmed up alike so that their counters
start in step.  The float64 statistics are checked against numpy over the returned draws."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CHESS_MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]
CHESS_STD = [float(np.sqrt(v)) for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
POSE_M, POSE_S = [0.5, -1.25, 2.0], [1.5, 0.75, 2.5]
H, W = 64, 96
# frames per call -> MapNet window shape (L, T): B = 1, 33 and 64 run 32 K-splits of 64, B = 160 16 splits of 128
MAPNET_LT = {1: (1, 1), 33: (11, 3), 64: (16, 4), 160: (32, 5)}


def _bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int64)


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _twins(kind, precision, max_batch, seed=5, calib=None):
    """two Predictors of one model with dropout 0.5"""
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    model, _ = make_product_model(weights.make_state(seed), kind, "bf16" if precision == "fp8" else precision,
                                  droprate=0.5)
    kw = dict(precision="fp8", calibration=calib) if precision == "fp8" else {}
    return Predictor(model, max_batch=max_batch, **kw), Predictor(model, max_batch=max_batch, **kw)


def _x(kind, n, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (n, 3, H, W) if kind == "posenet" else MAPNET_LT[n] + (3, H, W)
    return torch.randn(shape, generator=g).cuda()


def _check_stats(out, S):
    """mean / cov / t_std / q_std_deg against numpy float64 over the returned draws"""
    smp = out["samples"].reshape(-1, S, 6).double().cpu().numpy()
    mean = out["mean"].reshape(-1, 6).cpu().numpy()
    cov = out["cov"].reshape(-1, 6, 6).cpu().numpy()
    for b in range(smp.shape[0]):
        scale = max(np.abs(smp[b]).max(), 1e-30)
        assert np.abs(mean[b] - smp[b].mean(0)).max() <= 1e-13 * scale, b
        want = np.cov(smp[b].T, ddof=1)
        assert np.abs(cov[b] - want).max() <= 1e-13 * max(np.abs(want).max(), 1e-300), b
    tr_t = np.trace(cov[:, :3, :3], axis1=1, axis2=2)
    tr_q = np.trace(cov[:, 3:, 3:], axis1=1, axis2=2)
    np.testing.assert_allclose(out["t_std"].reshape(-1).cpu().numpy(), np.sqrt(tr_t), rtol=1e-13)
    np.testing.assert_allclose(out["q_std_deg"].reshape(-1).cpu().numpy(), 2 * np.sqrt(tr_q) * 180 / np.pi, rtol=1e-13)


# ---------------------------------------------------------------------------------------------------------------------
# 1. draws are bitwise S consecutive forwards, across the split-K plans, precisions and model shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["posenet", "mapnet"])
@pytest.mark.parametrize("precision", ["bf16", "tc_split", "fp8"])
def test_draws_are_bitwise_s_consecutive_forwards(precision, kind):
    calib = torch.randn(8, 3, H, W, generator=torch.Generator().manual_seed(3)).cuda()
    A, B = _twins(kind, precision, 256, calib=calib)
    for n in (1, 33, 64, 160):
        x = _x(kind, n, n)
        assert _same_bits(A(x), B(x))                  # warm-up: both counters step alike
        for S in (2, 7, 32):
            out = A.sample(x, S, keep_samples=True)
            lead = tuple(x.shape[:-3])
            assert tuple(out["samples"].shape) == lead + (S, 6) and out["samples"].dtype == torch.float32
            assert tuple(out["mean"].shape) == lead + (6,) and out["mean"].dtype == torch.float64
            assert tuple(out["cov"].shape) == lead + (6, 6) and tuple(out["t_std"].shape) == lead
            for s in range(S):
                want = B(x)
                assert _same_bits(out["samples"][..., s, :], want), (precision, kind, n, S, s)
            assert _same_bits(A(x), B(x)), (precision, kind, n, S, "counters out of step")
            _check_stats(out, S)
            if S == 7:
                assert not torch.equal(out["samples"][..., 0, :], out["samples"][..., 1, :])
    A.close(); B.close()


def test_inputs_longer_than_max_batch_take_s_steps_per_chunk():
    A, B = _twins("posenet", "bf16", 4)
    x = _x("posenet", 33, 1)[:10]                   # chunks of 4, 4 and 2 frames
    assert _same_bits(A(x), B(x))
    S = 5
    out = A.sample(x, S, keep_samples=True)
    for lo in range(0, 10, 4):
        chunk = x[lo:lo + 4]
        for s in range(S):
            assert _same_bits(out["samples"][lo:lo + 4, s], B(chunk)), (lo, s)
    assert _same_bits(A(x), B(x))
    _check_stats(out, S)
    assert "samples" not in A.sample(x, S)
    A.close(); B.close()


def test_repeated_calls_on_fresh_twins_give_identical_bits():
    x = _x("mapnet", 33, 2)
    outs = []
    for _ in range(2):
        A, B = _twins("mapnet", "tc_split", 64, seed=7)
        A(x)
        outs.append([A.sample(x, 32, keep_samples=True), A.sample(x, 9)])
        A.close(); B.close()
    for a, b in zip(outs[0], outs[1]):
        assert a.keys() == b.keys()
        for k in a:
            assert _same_bits(a[k], b[k]), k


def test_engine_host_step_and_null_samples():
    """an explicit step leaves the counter alone and gives draw s = the forward at step + s; samples = NULL gives the
    same mean / cov"""
    A, _ = _twins("posenet", "bf16", 64)
    x = _x("posenet", 33, 4).contiguous()
    eng = A._engine(H, W)
    n, S = x.shape[0], 6
    smp = torch.empty(n, S, 6, device="cuda")
    m1, m2 = torch.empty(n, 6, dtype=torch.float64, device="cuda"), torch.empty(n, 6, dtype=torch.float64, device="cuda")
    c1, c2 = torch.empty(n, 6, 6, dtype=torch.float64, device="cuda"), torch.empty(n, 6, 6, dtype=torch.float64, device="cuda")
    eng.sample(x, S, 0.5, A.seed, smp, m1, c1, step=11)
    eng.sample(x, S, 0.5, A.seed, None, m2, c2, step=11)
    pred = torch.empty(n, 6, device="cuda")
    for s in range(S):
        eng.forward(x, pred, 0.5, A.seed, step=11 + s)
        assert _same_bits(smp[:, s], pred), s
    assert _same_bits(m1, m2) and _same_bits(c1, c2)
    # the device counter was never touched: the first counted forward uses step 0, as on a fresh engine
    eng.forward(x, pred, 0.5, A.seed)
    want = torch.empty_like(pred)
    eng.forward(x, want, 0.5, A.seed, step=0)
    assert _same_bits(pred, want)
    A.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. argument errors of the C entry points, before any launch
# ---------------------------------------------------------------------------------------------------------------------
def test_engine_refuses_bad_arguments_before_any_launch():
    from geomapnet_b200 import _lib
    L = _lib.lib()
    A, _ = _twins("posenet", "bf16", 4)
    eng, eng2 = A._engine(H, W), A._engine(256, 341)
    torch.cuda.synchronize()
    x = torch.zeros(4, 3, H, W, device="cuda")
    m = torch.empty(8, 6, dtype=torch.float64, device="cuda")
    c = torch.empty(8, 6, 6, dtype=torch.float64, device="cuda")
    n0 = L.mapnet_launch_count()
    for B, S, p, msg in ((4, 1, 0.5, b"draws"), (4, 1025, 0.5, b"draws"), (4, 8, 0.0, b"droprate"),
                         (4, 8, 1.0, b"droprate"), (5, 8, 0.5, b"batch"), (0, 8, 0.5, b"batch")):
        assert L.mapnet_infer_sample(eng.h, x.data_ptr(), B, S, p, 0, 0, None, m.data_ptr(), c.data_ptr(),
                                     _lib.stream_ptr()) != 0
        assert msg in L.mapnet_last_error(), (B, S, p, L.mapnet_last_error())
    assert L.mapnet_infer_sample(eng.h, x.data_ptr(), 4, 8, 0.5, 0, 0, None, None, c.data_ptr(), _lib.stream_ptr()) != 0
    pre = ctypes.c_void_p()
    _lib.check(L.mapnet_preprocess_create(ctypes.byref(pre), 48, 64, 256, 4), "mapnet_preprocess_create")
    fp = ctypes.POINTER(ctypes.c_float)
    mean3, std3 = np.float32(CHESS_MEAN), np.float32(CHESS_STD)
    f = torch.zeros(4, 48, 64, 3, dtype=torch.uint8, device="cuda")
    # pre resizes to 256x341, the engine takes 64x96
    assert L.mapnet_infer_sample_frames(eng.h, pre, f.data_ptr(), 4, mean3.ctypes.data_as(fp), std3.ctypes.data_as(fp),
                                        8, 0.5, 0, 0, None, m.data_ptr(), c.data_ptr(), _lib.stream_ptr()) != 0
    assert b"resizes to 256x341" in L.mapnet_last_error()
    assert L.mapnet_infer_sample_frames(eng2.h, pre, f.data_ptr(), 4, mean3.ctypes.data_as(fp), std3.ctypes.data_as(fp),
                                        1, 0.5, 0, 0, None, m.data_ptr(), c.data_ptr(), _lib.stream_ptr()) != 0
    assert b"draws" in L.mapnet_last_error()
    L.mapnet_preprocess_destroy(pre)
    assert L.mapnet_launch_count() == n0
    A.close()
    with pytest.raises(RuntimeError, match="closed"):
        A.sample(x, 8)


def test_fp8_sample_refuses_frames_of_another_size():
    calib = torch.randn(4, 3, H, W, generator=torch.Generator().manual_seed(3)).cuda()
    A, B = _twins("posenet", "fp8", 4, calib=calib)
    with pytest.raises(ValueError, match="calibrated at %dx%d" % (H, W)):
        A.sample(torch.zeros(2, 3, H, W + 32, device="cuda"), 8)
    A.close(); B.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. one graph replay per chunk, no library call on replay
# ---------------------------------------------------------------------------------------------------------------------
def test_one_graph_replay_per_chunk(monkeypatch):
    from geomapnet_b200 import _lib
    L = _lib.lib()
    A, B = _twins("posenet", "bf16", 4)
    x = _x("posenet", 33, 6)[:10]
    A.sample(x, 8)                                  # captures (4, H, W, 8) and (2, H, W, 8)
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda g: (replays.append(g), real(g))[1])
    c0 = L.mapnet_launch_count()
    A.sample(x, 8)
    assert len(replays) == 3 and L.mapnet_launch_count() == c0
    monkeypatch.undo()
    A.close(); B.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. Localizer.sample
# ---------------------------------------------------------------------------------------------------------------------
def _qexp(v):
    n = np.linalg.norm(v, axis=-1, keepdims=True)
    safe = np.where(n > 0, n, 1.0)
    return np.concatenate([np.where(n > 0, np.cos(n), 1.0), np.where(n > 0, np.sin(n) / safe, 0.0) * v], -1)


@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
def test_localizer_draws_are_bitwise_s_localizer_calls(precision):
    from geomapnet_b200.inference import Localizer
    pa, pb = _twins("posenet", precision, 4, seed=9)
    la = Localizer(pa, CHESS_MEAN, CHESS_STD, pose_m=POSE_M, pose_s=POSE_S)
    lb = Localizer(pb, CHESS_MEAN, CHESS_STD, pose_m=POSE_M, pose_s=POSE_S)
    g = torch.Generator().manual_seed(12)
    frames = torch.randint(0, 256, (6, 48, 64, 3), dtype=torch.uint8, generator=g)
    for n in (3, 6):                                # one chunk; two chunks of max_batch = 4
        f = frames[:n]
        assert _same_bits(la(f), lb(f))             # warm-up: both counters step alike
        S = 7
        out = la.sample(f, S, keep_samples=True)
        assert tuple(out["pose7"].shape) == (n, 7) and tuple(out["cov"].shape) == (n, 6, 6)
        assert tuple(out["samples"].shape) == (n, S, 6)
        for lo in range(0, n, 4):
            fc = f[lo:lo + 4]
            for s in range(S):
                lb(fc)
                pred6 = lb._graphs[(fc.shape[0], 48, 64)][3]
                assert _same_bits(out["samples"][lo:lo + 4, s], pred6), (precision, n, lo, s)
        assert _same_bits(la(f), lb(f))
        smp = out["samples"].double().cpu().numpy()
        mean = smp.mean(1)
        cov = np.stack([np.cov(smp[b].T, ddof=1) for b in range(n)])
        d = np.array(POSE_S + [1.0, 1.0, 1.0])
        pose7 = np.concatenate([mean[:, :3] * d[:3] + np.array(POSE_M), _qexp(mean[:, 3:])], -1)
        covm = d[None, :, None] * cov * d[None, None, :]
        got7, gotc = out["pose7"].cpu().numpy(), out["cov"].cpu().numpy()
        assert np.abs(got7 - pose7).max() <= 1e-13 * np.abs(pose7).max()
        assert np.abs(gotc - covm).max() <= 1e-13 * np.abs(covm).max()
        np.testing.assert_allclose(out["t_std"].cpu().numpy(), np.sqrt(np.trace(covm[:, :3, :3], axis1=1, axis2=2)),
                                   rtol=1e-13)
        np.testing.assert_allclose(out["q_std_deg"].cpu().numpy(),
                                   2 * np.sqrt(np.trace(covm[:, 3:, 3:], axis1=1, axis2=2)) * 180 / np.pi, rtol=1e-13)
    one = la.sample(frames[0].numpy(), 4)
    assert tuple(one["pose7"].shape) == (7,) and tuple(one["cov"].shape) == (6, 6) and "samples" not in one
    la.close(); lb.close(); pa.close(); pb.close()
