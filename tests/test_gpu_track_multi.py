"""GPU tests of inference.MultiTracker and mapnet_track_multi_* (csrc/loader.cu): every stream's poses bit for bit
those of single-stream mapnet_track_* handles fed that stream's rows, and of the composition of the same Predictor
calls with mapnet_eval_windows, pgo and the un-normalisation, split by stream; flush and reset of one stream leave the
others alone, a non-positive-definite window marks its own stream only, MultiTracker(n_streams=1) is Tracker, dropout
draws each frame once, and each chunk is one graph replay of the engine's launches plus three tracking launches."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]
STD = [float(np.sqrt(v)) for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
POSE_M, POSE_S = [0.5, -1.25, 2.0], [1.5, 0.75, 2.5]
SIG = dict(sax=1.0, saq=0.5, srx=20.0, srq=20.0)
CONFIGS = [(3, 2, False), (4, 5, False), (7, 3, True)]          # (steps, skip, vo_fc)
H_IN, W_IN = 480, 640


def _model(precision, seed=5, droprate=0.0):
    from oracle import weights
    from helpers import make_product_model
    model, _ = make_product_model(weights.make_state(seed), "mapnet", precision, droprate=droprate)
    return model


def _assert_bitwise(got, want, what):
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    bad = (got != want).any(1).nonzero().flatten().tolist()
    assert not bad, (what, "rows differ:", bad[:10], float((got - want).abs().max()))


def _schedule(rng, K, n_calls, max_b, absent=()):
    """random interleavings: per call 1 .. max_b stream ids, repeats allowed, `absent` streams never used"""
    live = [s for s in range(K) if s not in absent]
    return [rng.choice(live, int(rng.integers(1, max_b + 1))).astype(np.int64) for _ in range(n_calls)]


# ---------------------------------------------------------------------------------------------------------------------
# 1. the C ABI against single-stream handles
# ---------------------------------------------------------------------------------------------------------------------
class _Handles(object):
    """one mapnet_track_multi_t of K streams and K mapnet_track_t of the same arguments"""

    def __init__(self, K, T, skip, fc, mb, metric):
        from geomapnet_b200 import _lib
        self.L, self.K, self.mb = _lib.lib(), K, mb
        self.lag = (T - 1 - T // 2) * skip
        sig = (ctypes.c_double * 4)(SIG["sax"], SIG["saq"], SIG["srx"], SIG["srq"])
        m3 = (ctypes.c_double * 3)(*POSE_M) if metric else None
        s3 = (ctypes.c_double * 3)(*POSE_S) if metric else None
        self.multi = ctypes.c_void_p()
        _lib.check(self.L.mapnet_track_multi_create(ctypes.byref(self.multi), K, T, skip, int(fc), mb, sig, m3, s3),
                   "mapnet_track_multi_create")
        self.single = []
        for _ in range(K):
            h = ctypes.c_void_p()
            _lib.check(self.L.mapnet_track_create(ctypes.byref(h), T, skip, int(fc), mb, sig, m3, s3),
                       "mapnet_track_create")
            self.single.append(h)
        self.seen = np.zeros(K, dtype=np.int64)

    def step(self, pred6, vo6, ids, now):
        """one call of the multi handle and, per stream present, one call of its single handle; returns
        (multi rows, single rows in the same order, multi now7, single now7 in the same order)"""
        from geomapnet_b200 import _lib
        from geomapnet_b200.inference import _stream_records
        B = ids.shape[0]
        rec, sid, fid = _stream_records(self.seen, ids, self.lag)
        rd = torch.from_numpy(rec).cuda()
        out = torch.full((B, 7), np.nan, dtype=torch.float64, device="cuda")
        now7 = torch.full((B, 7), np.nan, dtype=torch.float64, device="cuda") if now else None
        _lib.check(self.L.mapnet_track_multi_step(self.multi, pred6.data_ptr(), vo6.data_ptr(), rd.data_ptr(), B,
                                                  out.data_ptr(), now7.data_ptr() if now else None, _lib.stream_ptr()),
                   "mapnet_track_multi_step")
        want = torch.empty((sid.shape[0], 7), dtype=torch.float64, device="cuda")
        want_now = torch.empty((B, 7), dtype=torch.float64, device="cuda")
        for s in np.unique(ids):
            rows = np.flatnonzero(ids == s)
            n = rows.shape[0]
            p, v = pred6[rows].contiguous(), vo6[rows].contiguous()
            o = torch.empty((n, 7), dtype=torch.float64, device="cuda")
            if now:
                w = torch.empty((n, 7), dtype=torch.float64, device="cuda")
                _lib.check(self.L.mapnet_track_step_now(self.single[s], p.data_ptr(), v.data_ptr(), n, o.data_ptr(),
                                                        w.data_ptr(), _lib.stream_ptr()), "mapnet_track_step_now")
                want_now[torch.from_numpy(rows).cuda()] = w
            else:
                _lib.check(self.L.mapnet_track_step(self.single[s], p.data_ptr(), v.data_ptr(), n, o.data_ptr(),
                                                    _lib.stream_ptr()), "mapnet_track_step")
            k = int((sid == s).sum())
            want[torch.from_numpy(np.flatnonzero(sid == s)).cuda()] = o[:k]
        self.seen += np.bincount(ids, minlength=self.K)
        return out[:sid.shape[0]], want, now7, (want_now if now else None)

    def flush(self, s):
        from geomapnet_b200 import _lib
        n = int(min(self.lag, self.seen[s]))
        a = torch.empty((max(self.lag, 1), 7), dtype=torch.float64, device="cuda")
        b = torch.empty_like(a)
        _lib.check(self.L.mapnet_track_multi_flush(self.multi, s, a.data_ptr(), _lib.stream_ptr()), "multi flush")
        _lib.check(self.L.mapnet_track_flush(self.single[s], b.data_ptr(), _lib.stream_ptr()), "flush")
        _lib.check(self.L.mapnet_track_multi_reset(self.multi, s, _lib.stream_ptr()), "multi reset")
        _lib.check(self.L.mapnet_track_reset(self.single[s], _lib.stream_ptr()), "reset")
        self.seen[s] = 0
        return a[:n], b[:n]

    def status(self, s):
        seen, failed = ctypes.c_int64(), ctypes.c_int()
        from geomapnet_b200 import _lib
        _lib.check(self.L.mapnet_track_multi_status(self.multi, s, ctypes.byref(seen), ctypes.byref(failed),
                                                    _lib.stream_ptr()), "multi status")
        return seen.value, failed.value

    def close(self):
        torch.cuda.synchronize()
        self.L.mapnet_track_multi_destroy(self.multi)
        for h in self.single:
            self.L.mapnet_track_destroy(h)


@pytest.mark.parametrize("metric", [True, False])
@pytest.mark.parametrize("T,skip,fc", CONFIGS)
def test_c_abi_streams_equal_single_stream_handles(T, skip, fc, metric):
    K, mb = 5, 8
    rng = np.random.default_rng(T * 100 + skip * 10 + int(metric))
    for now in (False, True):
        hs = _Handles(K, T, skip, fc, mb, metric)
        calls = _schedule(rng, K, 30, mb, absent=(4,)) + _schedule(rng, K, 10, mb)
        for c, ids in enumerate(calls):
            B = ids.shape[0]
            pred6 = (torch.randn(B, 6, device="cuda") * 0.3).float()
            vo6 = (torch.randn(B, 6, device="cuda") * 0.3).float()
            got, want, gn, wn = hs.step(pred6, vo6, ids, now)
            _assert_bitwise(got, want, (T, skip, fc, metric, now, c))
            if now:
                _assert_bitwise(gn, wn, ("now7", T, skip, fc, metric, c))
            if c == 17:                                   # flush and reuse stream 2 mid-sequence
                a, b = hs.flush(2)
                _assert_bitwise(a, b, ("flush 2", T, skip, fc))
        for s in range(K):
            assert hs.status(s) == (int(hs.seen[s]), 0)
            a, b = hs.flush(s)
            assert a.shape[0] == b.shape[0]
            _assert_bitwise(a, b, ("final flush", s))
        hs.close()


def test_a_failed_window_marks_only_its_own_stream():
    K, mb, T, skip, fc = 4, 8, 4, 5, False
    hs = _Handles(K, T, skip, fc, mb, True)
    rng = np.random.default_rng(3)
    for c, ids in enumerate(_schedule(rng, K, 12, mb)):
        pred6 = (torch.randn(ids.shape[0], 6, device="cuda") * 0.3).float()
        if c == 5:
            pred6[torch.from_numpy(ids == 1).cuda()] = float("nan")      # NaN poses of stream 1: a numeric status
        hs.step(pred6, (torch.randn(ids.shape[0], 6, device="cuda") * 0.3).float(), ids, c % 2 == 1)
    assert [hs.status(s)[1] for s in range(K)] == [0, 1, 0, 0]
    hs.flush(1)
    assert [hs.status(s)[1] for s in range(K)] == [0, 0, 0, 0]
    hs.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. end to end against the composition, 3. one stream is the Tracker, 4. dropout
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def streams():
    """K = 3 synthetic sequences: uint8 frames [L,480,640,3] and VO-library poses per stream"""
    rng = np.random.default_rng(7)
    out = []
    for k in range(3):
        L = 40
        fr = torch.from_numpy(rng.integers(0, 256, (L, H_IN, W_IN, 3), dtype=np.uint8)).cuda()
        s = np.arange(L)[:, None] / 10.0 + k
        poses = np.concatenate([np.sin(s), np.cos(0.7 * s), 0.1 * s, 0.2 * np.sin(0.3 * s), 0.1 * np.cos(0.5 * s),
                                0.05 * s], 1)
        out.append((fr, (poses + rng.standard_normal(poses.shape) * 0.02).astype(np.float32)))
    return out


def _interleave(streams, sizes, seed):
    """calls of `sizes` frames with random stream ids, each stream's frames in order: [(frames, vo, ids)]"""
    rng = np.random.default_rng(seed)
    pos = [0] * len(streams)
    calls = []
    for n in sizes:
        ids = []
        for _ in range(n):
            live = [s for s in range(len(streams)) if pos[s] < streams[s][0].shape[0]]
            s = int(rng.choice(live))
            ids.append((s, pos[s]))
            pos[s] += 1
        fr = torch.stack([streams[s][0][i] for s, i in ids])
        vo = np.stack([streams[s][1][i] for s, i in ids])
        calls.append((fr, vo, np.array([s for s, _ in ids], dtype=np.int64)))
    return calls


def _windows(pred6, vo, T, skip, fc, last=False, zero_lag=False):
    """eval.py's windows of one stream's per-frame predictions (mapnet_eval_windows), pgo, the middle (or, zero-lag,
    the last) slot of each, un-normalised as _window_errors does"""
    from geomapnet_b200 import _lib
    from geomapnet_b200.inference import pgo
    L = pred6.shape[0]
    lag = (T - 1 - T // 2) * skip
    c = np.arange(L)[:, None] - (lag if zero_lag else 0)
    windows = np.ascontiguousarray(np.clip(c + (np.arange(T)[None] - T // 2) * skip, 0, L - 1), dtype=np.int32)
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
    mid = pgo(pred7, vos7, fc_vos=fc, **SIG)[:, T - 1 if zero_lag else T // 2]
    m = torch.as_tensor(np.asarray(POSE_M, dtype=np.float64), device="cuda")
    s = torch.as_tensor(np.asarray(POSE_S, dtype=np.float64), device="cuda")
    return torch.cat((mid[:, :3] * s + m, mid[:, 3:]), -1)


def _composition(pr, calls, K, T, skip, fc, zero_lag=False):
    """ImagePipeline -> Predictor on the same interleaved batches, split by stream -> _windows per stream"""
    from geomapnet_b200.data import ImagePipeline
    pipe = ImagePipeline(MEAN, STD)
    pred6 = torch.cat([pr(pipe(fr)) for fr, _, _ in calls])
    vo = np.concatenate([v for _, v, _ in calls])
    ids = np.concatenate([i for _, _, i in calls])
    return {s: _windows(pred6[torch.from_numpy(np.flatnonzero(ids == s)).cuda()].contiguous(), vo[ids == s], T, skip,
                        fc, zero_lag=zero_lag) for s in range(K)}


def _run_multi(mt, calls, K, now=False):
    """every stream's poses (lagged with flushes; zero-lag when now) from MultiTracker calls, checked row by row"""
    got = {s: [] for s in range(K)}
    nows = {s: [] for s in range(K)}
    nxt = [0] * K
    for fr, vo, ids in calls:
        if now:
            n7, sid, fid, p = mt.step(fr, vo, ids)
            for s in range(K):
                nows[s].append(n7[torch.from_numpy(ids == s).cuda()])
        else:
            sid, fid, p = mt(fr, vo, list(ids) if len(got[0]) % 2 else torch.from_numpy(ids))
        assert sid.dtype == torch.int64 and fid.dtype == torch.int64 and not sid.is_cuda and p.shape == (sid.shape[0], 7)
        for r in range(sid.shape[0]):
            s = int(sid[r])
            assert int(fid[r]) == nxt[s], (s, int(fid[r]), nxt[s])
            nxt[s] += 1
            got[s].append(p[r:r + 1])
    for s in range(K):
        first, p = mt.flush(s)
        assert first == nxt[s] and mt.seen[s] == 0
        got[s].append(p)
    return {s: torch.cat(v) for s, v in got.items()}, {s: torch.cat(v) for s, v in nows.items()} if now else None


SIZES = [1, 8, 3, 13, 5, 8, 2, 1, 7, 20, 6, 8, 8, 12, 4, 8, 2, 4]          # 120 frames: 13 and 20 split into chunks


@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
def test_each_stream_is_the_composition_of_the_same_predictor_calls(streams, precision):
    from geomapnet_b200.inference import Localizer, MultiTracker, Predictor
    T, skip, fc, K = 7, 3, True, 3
    pr = Predictor(_model(precision), max_batch=8)
    loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
    calls = _interleave(streams, SIZES, 1)
    chunked = [(fr[lo:lo + 8], vo[lo:lo + 8], ids[lo:lo + 8]) for fr, vo, ids in calls for lo in range(0, len(ids), 8)]
    want = _composition(pr, chunked, K, T, skip, fc)
    want_now = _composition(pr, chunked, K, T, skip, fc, zero_lag=True)
    mt = MultiTracker(loc, n_streams=K, steps=T, skip=skip, vo_fc=fc, **SIG)
    got, _ = _run_multi(mt, calls, K)
    for s in range(K):
        _assert_bitwise(got[s], want[s], (precision, "stream", s))
    lagged, now = _run_multi(mt, calls, K, now=True)
    for s in range(K):
        _assert_bitwise(lagged[s], want[s], (precision, "step lagged", s))
        _assert_bitwise(now[s], want_now[s], (precision, "step now7", s))
    mt.close(); loc.close(); pr.close()


def test_one_stream_is_the_tracker(streams):
    from geomapnet_b200.inference import Localizer, MultiTracker, Predictor, Tracker
    fr, vo = streams[0]
    pr = Predictor(_model("bf16"), max_batch=8)
    loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
    for T, skip, fc in CONFIGS:
        mt = MultiTracker(loc, 1, steps=T, skip=skip, vo_fc=fc, **SIG)
        trk = Tracker(loc, steps=T, skip=skip, vo_fc=fc, **SIG)
        lo = 0
        for n in (1, 8, 3, 13, 5):
            f, v = fr[lo:lo + n], vo[lo:lo + n]
            sid, fid, p = mt(f, v, [0] * n)
            first, q = trk(f, v)
            assert (sid == 0).all() and fid.tolist() == list(range(first, first + q.shape[0]))
            _assert_bitwise(p, q, (T, skip, fc, lo))
            n7, sid, fid, p = mt.step(f, v, np.zeros(n, dtype=np.int32))
            m7, first, q = trk.step(f, v)
            _assert_bitwise(n7, m7, ("now7", T, skip, fc, lo))
            _assert_bitwise(p, q, ("step", T, skip, fc, lo))
            lo += n
        (a, p), (b, q) = mt.flush(0), trk.flush()
        assert a == b
        _assert_bitwise(p, q, ("flush", T, skip, fc))
        mt.close(); trk.close()
    loc.close(); pr.close()


def test_dropout_draws_each_frame_once(streams):
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.inference import Localizer, MultiTracker, Predictor, post
    T, skip, fc, K = 4, 5, False, 3
    pa = Predictor(_model("bf16", seed=3, droprate=0.5), max_batch=8)
    pb = Predictor(_model("bf16", seed=3, droprate=0.5), max_batch=8)
    pb.seed = pa.seed
    loc = Localizer(pa, MEAN, STD, POSE_M, POSE_S)
    mt = MultiTracker(loc, K, steps=T, skip=skip, vo_fc=fc, **SIG)
    calls = _interleave(streams, [8, 3, 8, 8, 1, 8, 5, 8], 2)
    got, _ = _run_multi(mt, calls, K)
    want = _composition(pb, calls, K, T, skip, fc)
    for s in range(K):
        _assert_bitwise(got[s], want[s], ("droprate 0.5", s))
    f = streams[0][0][:3]
    assert torch.equal(loc(f), post(pb(ImagePipeline(MEAN, STD)(f)), POSE_M, POSE_S))   # the counters end equal
    mt.close(); loc.close(); pa.close(); pb.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. launches and captures
# ---------------------------------------------------------------------------------------------------------------------
def test_one_replay_of_the_engine_and_three_tracking_launches_per_chunk(streams):
    """2 preprocess + 43 engine launches in the eager run before the capture, the same 45 + gather, k_pgo and emit in
    the capture; a replay makes no library call, and a shape met before makes no new capture"""
    from geomapnet_b200 import _lib
    from geomapnet_b200.inference import Localizer, MultiTracker, Predictor
    fr, vo = streams[0]
    lib = _lib.lib()
    pr = Predictor(_model("bf16"), max_batch=4)
    loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
    mt = MultiTracker(loc, 3, steps=4, skip=5, **SIG)
    pr._engine(256, 341)
    lo = 0
    for B in (1, 4):
        c0 = lib.mapnet_launch_count()
        mt(fr[lo:lo + B], vo[lo:lo + B], [lo % 3] * B)
        assert lib.mapnet_launch_count() - c0 == (2 + 43) + (2 + 43 + 3), B
        lo += B
    c0 = lib.mapnet_launch_count()
    mt.step(fr[lo:lo + 4], vo[lo:lo + 4], [0, 1, 2, 0])
    assert lib.mapnet_launch_count() - c0 == (2 + 43) + (2 + 43 + 3)
    lo += 4
    n_graphs = (len(mt._graphs), len(mt._now_graphs))
    assert n_graphs == (2, 1)
    c1 = lib.mapnet_launch_count()
    for B in (4, 1, 4):
        mt(fr[lo:lo + B], vo[lo:lo + B], [2] * B)
        if B == 4:
            mt.step(fr[lo:lo + B], vo[lo:lo + B], [1, 1, 0, 1])
        lo += B
    mt(fr[lo:lo + 9], vo[lo:lo + 9], [0, 1, 2] * 3)                     # chunks of 4, 4 and 1
    assert lib.mapnet_launch_count() == c1 and (len(mt._graphs), len(mt._now_graphs)) == n_graphs
    mt.close(); loc.close(); pr.close()
