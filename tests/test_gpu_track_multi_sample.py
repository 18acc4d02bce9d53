"""GPU tests of inference.SampledMultiTracker and mapnet_track_multi_sample_* (csrc/loader.cu): every stream's rows
(lagged, zero-lag and flushed) bit for bit those of single-stream mapnet_track_sample_t handles fed that stream's
rows, a non-positive-definite factor or a NaN mean marks its own stream only, the Python class against a twin
Predictor's sampled engine run on the same chunks and split by stream, one stream is the SampledTracker, flush and
reset of one stream leave the others alone, and each chunk is one graph replay of the sampled engine plus three
tracking launches."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]
STD = [float(np.sqrt(v)) for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
POSE_M, POSE_S = [0.5, -1.25, 2.0], [1.5, 0.75, 2.5]
SIG = dict(sax=1e-3, saq=1e-3, srx=20.0, srq=20.0)
S = 16
ROW = 45
CONFIGS = [(3, 2, False), (4, 5, False), (7, 3, True), (16, 1, True)]         # (steps, skip, vo_fc)
H_IN, W_IN = 480, 640


def _model(precision="bf16", seed=5, droprate=0.5):
    from oracle import weights
    from helpers import make_product_model
    model, _ = make_product_model(weights.make_state(seed), "mapnet", precision, droprate=droprate)
    return model


def _assert_bitwise(got, want, what):
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    bad = (got != want).any(1).nonzero().flatten().tolist()
    assert not bad, (what, "rows differ:", bad[:10], float((got - want).abs().max()))


def _rows(est):
    """an est dict as output rows [n,45]"""
    return torch.cat((est["pose7"], est["cov"].reshape(-1, 36), est["t_std"][:, None], est["q_std_deg"][:, None]), 1)


def _schedule(rng, K, n_calls, max_b, absent=()):
    """random interleavings: per call 1 .. max_b stream ids, repeats allowed, `absent` streams never used"""
    live = [s for s in range(K) if s not in absent]
    return [rng.choice(live, int(rng.integers(1, max_b + 1))).astype(np.int64) for _ in range(n_calls)]


def _draw_stats(rng, B):
    """means like the existing tests' poses and positive-definite covariances at the magnitudes of dropout draws"""
    mean = torch.from_numpy(rng.standard_normal((B, 6)) * 0.3).cuda()
    d = np.array([0.05] * 3 + [0.01] * 3)
    A = rng.standard_normal((B, 6, 6))
    cov = d[None, :, None] * (A @ A.transpose(0, 2, 1) / 6.0 + 0.1 * np.eye(6)) * d[None, None, :]
    return mean, torch.from_numpy(cov).cuda()


def _sig():
    return (ctypes.c_double * 4)(SIG["sax"], SIG["saq"], SIG["srx"], SIG["srq"])


class _Singles(object):
    """K mapnet_track_sample_t handles of the same arguments: the per-stream composition of a multi-stream call"""

    def __init__(self, K, T, skip, fc, mb, metric):
        from geomapnet_b200 import _lib
        self.L, self.K = _lib.lib(), K
        self.lag = (T - 1 - T // 2) * skip
        m3 = (ctypes.c_double * 3)(*POSE_M) if metric else None
        s3 = (ctypes.c_double * 3)(*POSE_S) if metric else None
        self.hs = []
        for _ in range(K):
            h = ctypes.c_void_p()
            _lib.check(self.L.mapnet_track_sample_create(ctypes.byref(h), T, skip, int(fc), mb, _sig(), m3, s3),
                       "mapnet_track_sample_create")
            self.hs.append(h)
        self.seen = np.zeros(K, dtype=np.int64)

    def step(self, mean, cov, vo6, ids, now):
        """(rows [n,45] in the multi call's out order, now rows [B,45] in call order or None)"""
        from geomapnet_b200 import _lib
        from geomapnet_b200.inference import _stream_records
        B = ids.shape[0]
        _, sid, _ = _stream_records(self.seen, ids, self.lag)
        want = torch.empty((sid.shape[0], ROW), dtype=torch.float64, device="cuda")
        want_now = torch.empty((B, ROW), dtype=torch.float64, device="cuda")
        for s in np.unique(ids):
            rows = np.flatnonzero(ids == s)
            n = rows.shape[0]
            ix = torch.from_numpy(rows).cuda()
            m, c, v = mean[ix].contiguous(), cov[ix].contiguous(), vo6[ix].contiguous()
            o = torch.empty((n, ROW), dtype=torch.float64, device="cuda")
            if now:
                w = torch.empty((n, ROW), dtype=torch.float64, device="cuda")
                _lib.check(self.L.mapnet_track_sample_step_now(self.hs[s], m.data_ptr(), c.data_ptr(), v.data_ptr(), n,
                                                               o.data_ptr(), w.data_ptr(), _lib.stream_ptr()),
                           "mapnet_track_sample_step_now")
                want_now[ix] = w
            else:
                _lib.check(self.L.mapnet_track_sample_step(self.hs[s], m.data_ptr(), c.data_ptr(), v.data_ptr(), n,
                                                           o.data_ptr(), _lib.stream_ptr()), "mapnet_track_sample_step")
            k = int((sid == s).sum())
            want[torch.from_numpy(np.flatnonzero(sid == s)).cuda()] = o[:k]
        self.seen += np.bincount(ids, minlength=self.K)
        return want, (want_now if now else None)

    def flush(self, s):
        from geomapnet_b200 import _lib
        n = int(min(self.lag, self.seen[s]))
        b = torch.empty((max(self.lag, 1), ROW), dtype=torch.float64, device="cuda")
        _lib.check(self.L.mapnet_track_sample_flush(self.hs[s], b.data_ptr(), _lib.stream_ptr()), "flush")
        _lib.check(self.L.mapnet_track_sample_reset(self.hs[s], _lib.stream_ptr()), "reset")
        self.seen[s] = 0
        return b[:n]

    def close(self):
        torch.cuda.synchronize()
        for h in self.hs:
            self.L.mapnet_track_sample_destroy(h)


class _Multi(object):
    """one mapnet_track_multi_sample_t of K streams, called through the C ABI"""

    def __init__(self, K, T, skip, fc, mb, metric):
        from geomapnet_b200 import _lib
        self.L, self.K = _lib.lib(), K
        self.lag = (T - 1 - T // 2) * skip
        m3 = (ctypes.c_double * 3)(*POSE_M) if metric else None
        s3 = (ctypes.c_double * 3)(*POSE_S) if metric else None
        self.h = ctypes.c_void_p()
        _lib.check(self.L.mapnet_track_multi_sample_create(ctypes.byref(self.h), K, T, skip, int(fc), mb, _sig(), m3,
                                                           s3), "mapnet_track_multi_sample_create")
        self.seen = np.zeros(K, dtype=np.int64)

    def step(self, mean, cov, vo6, ids, now):
        from geomapnet_b200 import _lib
        from geomapnet_b200.inference import _stream_records
        B = ids.shape[0]
        rec, sid, _ = _stream_records(self.seen, ids, self.lag)
        rd = torch.from_numpy(rec).cuda()
        out = torch.full((B, ROW), np.nan, dtype=torch.float64, device="cuda")
        nw = torch.full((B, ROW), np.nan, dtype=torch.float64, device="cuda") if now else None
        _lib.check(self.L.mapnet_track_multi_sample_step(self.h, mean.data_ptr(), cov.data_ptr(), vo6.data_ptr(),
                                                         rd.data_ptr(), B, out.data_ptr(),
                                                         nw.data_ptr() if now else None, _lib.stream_ptr()),
                   "mapnet_track_multi_sample_step")
        self.seen += np.bincount(ids, minlength=self.K)
        return out[:sid.shape[0]], nw

    def flush(self, s):
        from geomapnet_b200 import _lib
        n = int(min(self.lag, self.seen[s]))
        a = torch.empty((max(self.lag, 1), ROW), dtype=torch.float64, device="cuda")
        _lib.check(self.L.mapnet_track_multi_sample_flush(self.h, s, a.data_ptr(), _lib.stream_ptr()), "multi flush")
        _lib.check(self.L.mapnet_track_multi_sample_reset(self.h, s, _lib.stream_ptr()), "multi reset")
        self.seen[s] = 0
        return a[:n]

    def status(self, s):
        from geomapnet_b200 import _lib
        seen, failed = ctypes.c_int64(), ctypes.c_int()
        _lib.check(self.L.mapnet_track_multi_sample_status(self.h, s, ctypes.byref(seen), ctypes.byref(failed),
                                                           _lib.stream_ptr()), "multi status")
        return seen.value, failed.value

    def close(self):
        torch.cuda.synchronize()
        self.L.mapnet_track_multi_sample_destroy(self.h)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the C ABI against single-stream handles, 2. failure isolation
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", [True, False])
@pytest.mark.parametrize("T,skip,fc", CONFIGS)
def test_c_abi_streams_equal_single_stream_handles(T, skip, fc, metric):
    K, mb = 5, 8
    rng = np.random.default_rng(T * 100 + skip * 10 + int(metric))
    multi, singles = _Multi(K, T, skip, fc, mb, metric), _Singles(K, T, skip, fc, mb, metric)
    calls = _schedule(rng, K, 30, mb, absent=(4,)) + _schedule(rng, K, 12, mb)
    for c, ids in enumerate(calls):
        B = ids.shape[0]
        now = c % 3 == 1                                  # zero-lag steps mixed with calls on the same sequences
        mean, cov = _draw_stats(rng, B)
        vo6 = (torch.randn(B, 6, device="cuda") * 0.3).float()
        got, gn = multi.step(mean, cov, vo6, ids, now)
        want, wn = singles.step(mean, cov, vo6, ids, now)
        _assert_bitwise(got, want, (T, skip, fc, metric, now, c))
        if now:
            _assert_bitwise(gn, wn, ("now", T, skip, fc, metric, c))
        if c in (17, 29):                                 # flush and reuse single streams mid-sequence
            s = 2 if c == 17 else 0
            _assert_bitwise(multi.flush(s), singles.flush(s), ("flush", s, c, T, skip, fc))
    for s in range(K):
        assert multi.status(s) == (int(multi.seen[s]), 0)
        n = min(multi.lag, int(multi.seen[s]))
        a, b = multi.flush(s), singles.flush(s)
        assert a.shape[0] == n
        _assert_bitwise(a, b, ("final flush", s))
    multi.close(); singles.close()


def test_a_bad_factor_or_a_nan_mean_marks_only_its_own_stream():
    K, mb, T, skip, fc = 4, 8, 4, 5, False
    multi, singles = _Multi(K, T, skip, fc, mb, True), _Singles(K, T, skip, fc, mb, True)
    rng = np.random.default_rng(3)
    calls = _schedule(rng, K, 14, mb)
    calls[5] = calls[9] = np.array([0, 1, 2, 3, 1], dtype=np.int64)
    for c, ids in enumerate(calls):
        B = ids.shape[0]
        mean, cov = _draw_stats(rng, B)
        if c == 5:
            cov[torch.from_numpy(ids == 1).cuda()] = -torch.eye(6, dtype=torch.float64, device="cuda")  # S7 not PD
        if c == 9:
            mean[torch.from_numpy(ids == 3).cuda()] = float("nan")
        vo6 = (torch.randn(B, 6, device="cuda") * 0.3).float()
        # odd calls are zero-lag steps: each solves the window that ends at its frames, the bad ones included
        got, gn = multi.step(mean, cov, vo6, ids, c % 2 == 1)
        want, wn = singles.step(mean, cov, vo6, ids, c % 2 == 1)
        keep = torch.from_numpy(~np.isin(_rec_streams(singles, ids, got.shape[0]), [1, 3])).cuda()
        _assert_bitwise(got[keep], want[keep], ("healthy streams", c))
        if gn is not None:
            ok = torch.from_numpy(~np.isin(ids, [1, 3])).cuda()
            _assert_bitwise(gn[ok], wn[ok], ("healthy now", c))
    assert [multi.status(s)[1] for s in range(K)] == [0, 1, 0, 1]
    for s in (0, 2):
        _assert_bitwise(multi.flush(s), singles.flush(s), ("flush", s))
    multi.flush(1)
    assert [multi.status(s)[1] for s in range(K)] == [0, 0, 0, 1]
    multi.close(); singles.close()


def _rec_streams(singles, ids, n):
    """the stream of each of a call's n completed rows (the call's seen counts are already advanced)"""
    from geomapnet_b200.inference import _stream_records
    before = singles.seen - np.bincount(ids, minlength=singles.K)
    return _stream_records(before, ids, singles.lag)[1][:n]


def test_flush_raises_for_its_own_stream_only():
    """SampledMultiTracker.flush(s) raises np.linalg.LinAlgError for the stream whose factor was not positive
    definite, after resetting it, and not for the others"""
    from geomapnet_b200 import _lib
    from geomapnet_b200.inference import Localizer, Predictor, SampledMultiTracker, _stream_records
    pr = Predictor(_model(), max_batch=8)
    loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
    smt = SampledMultiTracker(loc, S, 3, steps=4, skip=5, **SIG)
    h, L = smt._handle(), _lib.lib()
    rng = np.random.default_rng(9)
    for c in range(6):                                    # drive the handle with chosen draw statistics
        ids = np.array([0, 1, 2, 1], dtype=np.int64)
        mean, cov = _draw_stats(rng, 4)
        if c == 2:
            cov[1] = -torch.eye(6, dtype=torch.float64, device="cuda")
        vo6 = (torch.randn(4, 6, device="cuda") * 0.3).float()
        rec = torch.from_numpy(_stream_records(smt.seen, ids, smt.lag)[0]).cuda()
        out = torch.empty((4, ROW), dtype=torch.float64, device="cuda")
        _lib.check(L.mapnet_track_multi_sample_step(h, mean.data_ptr(), cov.data_ptr(), vo6.data_ptr(), rec.data_ptr(),
                                                    4, out.data_ptr(), None, _lib.stream_ptr()), "step")
        smt.seen += np.bincount(ids, minlength=3)
    first, est = smt.flush(0)
    assert first == 1 and est["pose7"].shape == (5, 7) and est["cov"].shape == (5, 6, 6)
    with pytest.raises(np.linalg.LinAlgError, match="stream 1"):
        smt.flush(1)
    assert smt.seen.tolist() == [0, 0, 6]
    smt.flush(1)                                          # reset by the flush that raised
    smt.flush(2)
    smt.close(); loc.close(); pr.close()


def test_step_flush_and_status_refuse_bad_arguments_without_a_launch():
    from geomapnet_b200 import _lib
    L = _lib.lib()
    multi = _Multi(3, 4, 2, False, 4, False)
    p = torch.zeros(64, dtype=torch.float64, device="cuda")
    q = p.data_ptr()
    n0 = L.mapnet_launch_count()
    for args in [(None, q, q, q, 1, q, None), (q, None, q, q, 1, q, None), (q, q, None, q, 1, q, None),
                 (q, q, q, None, 1, q, None), (q, q, q, q, 1, None, q)]:
        assert L.mapnet_track_multi_sample_step(multi.h, *args, None) != 0
        assert b"null argument" in L.mapnet_last_error()
    for B in (0, -1, 5):
        assert L.mapnet_track_multi_sample_step(multi.h, q, q, q, q, B, q, None, None) != 0
        assert b"outside [1, max_batch=4]" in L.mapnet_last_error()
    for s in (-1, 3):
        assert L.mapnet_track_multi_sample_flush(multi.h, s, q, None) != 0
        assert b"outside [0, 3)" in L.mapnet_last_error()
        assert L.mapnet_track_multi_sample_status(multi.h, s, None, None, None) != 0
        assert b"outside [0, 3)" in L.mapnet_last_error()
    assert L.mapnet_track_multi_sample_flush(multi.h, 0, None, None) != 0
    assert L.mapnet_track_multi_sample_reset(multi.h, 3, None) != 0 and b"outside [-1, 3)" in L.mapnet_last_error()
    assert L.mapnet_launch_count() == n0
    multi.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. Python against the composition, 4. one stream is the SampledTracker, 5. per-stream flush and reset
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


def _pair(precision="bf16", max_batch=8):
    """two Predictors of one dropout model with equal seeds and counters: A tracks, B composes"""
    from geomapnet_b200.inference import Predictor
    model = _model(precision)
    pa, pb = Predictor(model, max_batch=max_batch), Predictor(model, max_batch=max_batch)
    pa.seed = pb.seed = 20261018
    return pa, pb


def _twin_draws(lb, fb):
    """the normalised mean [B,6] and cov [B,6,6] of Localizer.sample's engine on one chunk (its graph's buffers)"""
    graph, xs, o = lb._sample_graph(fb, S)
    xs.copy_(fb)
    graph.replay()
    return o["mean"].clone(), o["cov6"].clone()


SIZES = [1, 8, 3, 13, 5, 8, 2, 1, 7, 20, 6, 8, 8, 12, 4, 8, 2, 4]          # 120 frames: 13 and 20 split into chunks


@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
def test_each_stream_is_the_composition_of_the_twin_sampled_engine(streams, precision):
    from geomapnet_b200.inference import Localizer, SampledMultiTracker
    T, skip, fc, K, mb = 7, 3, True, 3, 8
    pa, pb = _pair(precision, mb)
    la, lb = Localizer(pa, MEAN, STD, POSE_M, POSE_S), Localizer(pb, MEAN, STD)
    smt = SampledMultiTracker(la, S, K, steps=T, skip=skip, vo_fc=fc, **SIG)
    singles = _Singles(K, T, skip, fc, mb, True)
    for c, (fr, vo, ids) in enumerate(_interleave(streams, SIZES, 1)):
        now = c % 3 == 2
        if now:
            nw, sid, fid, est = smt.step(fr, vo, ids)
        else:
            sid, fid, est = smt(fr, vo, list(ids) if c % 2 else torch.from_numpy(ids))
        assert sid.dtype == torch.int64 and not sid.is_cuda and est["pose7"].shape == (sid.shape[0], 7)
        want, want_now = [], []
        for lo in range(0, ids.shape[0], mb):             # the twin runs the tracker's chunks
            mean, cov = _twin_draws(lb, fr[lo:lo + mb])
            w, wn = singles.step(mean, cov, torch.from_numpy(vo[lo:lo + mb]).cuda(), ids[lo:lo + mb], now)
            want.append(w)
            want_now.append(wn)
        _assert_bitwise(_rows(est), torch.cat(want), (precision, "call", c))
        if now:
            _assert_bitwise(_rows(nw), torch.cat(want_now), (precision, "now", c))
        if c == 9:
            first, est = smt.flush(1)
            _assert_bitwise(_rows(est), singles.flush(1), (precision, "flush 1"))
    for s in range(K):
        first, est = smt.flush(s)
        assert smt.seen[s] == 0
        _assert_bitwise(_rows(est), singles.flush(s), (precision, "final flush", s))
    singles.close(); smt.close(); la.close(); lb.close(); pa.close(); pb.close()


def test_one_stream_is_the_sampled_tracker(streams):
    from geomapnet_b200.inference import Localizer, SampledMultiTracker, SampledTracker
    fr, vo = streams[0]
    pa, pb = _pair()
    la, lb = Localizer(pa, MEAN, STD, POSE_M, POSE_S), Localizer(pb, MEAN, STD, POSE_M, POSE_S)
    for T, skip, fc in CONFIGS[:3]:
        smt = SampledMultiTracker(la, S, 1, steps=T, skip=skip, vo_fc=fc, **SIG)
        st = SampledTracker(lb, S, steps=T, skip=skip, vo_fc=fc, **SIG)
        lo = 0
        for n in (1, 8, 3, 13, 5):
            f, v = fr[lo:lo + n], vo[lo:lo + n]
            sid, fid, p = smt(f, v, [0] * n)
            first, q = st(f, v)
            assert (sid == 0).all() and fid.tolist() == list(range(first, first + q["pose7"].shape[0]))
            _assert_bitwise(_rows(p), _rows(q), (T, skip, fc, lo))
            nw, sid, fid, p = smt.step(f, v, np.zeros(n, dtype=np.int32))
            mw, first, q = st.step(f, v)
            _assert_bitwise(_rows(nw), _rows(mw), ("now", T, skip, fc, lo))
            _assert_bitwise(_rows(p), _rows(q), ("step", T, skip, fc, lo))
            lo += n
        (a, p), (b, q) = smt.flush(0), st.flush()
        assert a == b
        _assert_bitwise(_rows(p), _rows(q), ("flush", T, skip, fc))
        smt.close(); st.close()
    f = fr[:3]
    assert torch.equal(la(f), lb(f))                      # the dropout counters end where the SampledTracker's do
    la.close(); lb.close(); pa.close(); pb.close()


def test_flush_and_reset_of_one_stream_leave_the_others_alone(streams):
    from geomapnet_b200.inference import Localizer, SampledMultiTracker
    T, skip, fc, K = 4, 5, False, 3
    pa, pb = _pair()
    la, lb = Localizer(pa, MEAN, STD, POSE_M, POSE_S), Localizer(pb, MEAN, STD, POSE_M, POSE_S)
    a = SampledMultiTracker(la, S, K, steps=T, skip=skip, vo_fc=fc, **SIG)
    b = SampledMultiTracker(lb, S, K, steps=T, skip=skip, vo_fc=fc, **SIG)
    for c, (fr, vo, ids) in enumerate(_interleave(streams, [8, 5, 8, 8, 3, 8, 6, 8, 8, 4], 3)):
        if c == 3:
            a.flush(1)                                    # stream 1 of A restarts; B's goes on
        if c == 5:
            a.reset(2)
        sa, fa, ea = a(fr, vo, ids)
        sb, fb, eb = b(fr, vo, ids)
        keep_a, keep_b = (sa == 0).cuda(), (sb == 0).cuda()
        assert torch.equal(fa[sa == 0], fb[sb == 0])
        _assert_bitwise(_rows(ea)[keep_a], _rows(eb)[keep_b], ("stream 0", c))
        if c < 3:
            _assert_bitwise(_rows(ea), _rows(eb), ("before", c))
    assert a.seen[0] == b.seen[0] and a.seen[1] < b.seen[1] and a.seen[2] < b.seen[2]
    _assert_bitwise(_rows(a.flush(0)[1]), _rows(b.flush(0)[1]), "flush 0")
    a.close(); b.close(); la.close(); lb.close(); pa.close(); pb.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. launches and captures
# ---------------------------------------------------------------------------------------------------------------------
def test_one_replay_of_the_sampled_engine_and_three_tracking_launches_per_chunk(streams):
    from geomapnet_b200 import _lib
    from geomapnet_b200.inference import Localizer, SampledMultiTracker
    fr, vo = streams[0]
    lib = _lib.lib()
    pa, pb = _pair(max_batch=4)
    la, lb = Localizer(pa, MEAN, STD, POSE_M, POSE_S), Localizer(pb, MEAN, STD, POSE_M, POSE_S)
    smt = SampledMultiTracker(la, S, 3, steps=4, skip=5, **SIG)
    for loc in (la, lb):
        loc.predictor._engine(256, 341)
        loc._plan(H_IN, W_IN)
    c0 = lib.mapnet_launch_count()
    lb.sample(fr[:4], S)                                  # the sampled engine's launches: eager run + capture
    n_sample = (lib.mapnet_launch_count() - c0) // 2 - 1  # minus mapnet_sample_post
    la.sample(fr[:4], S)                                  # the same dropout steps on A
    lo = 4
    for B in (1, 4):
        c0 = lib.mapnet_launch_count()
        smt(fr[lo:lo + B], vo[lo:lo + B], [lo % 3] * B)
        assert lib.mapnet_launch_count() - c0 == n_sample + (n_sample + 3), (B, lib.mapnet_launch_count() - c0)
        lb.sample(fr[lo:lo + B], S)                       # the twin takes the same dropout steps
        lo += B
    h = smt._handle()
    for s in range(3):                                    # the eager runs advanced no stream
        seen = ctypes.c_int64()
        _lib.check(lib.mapnet_track_multi_sample_status(h, s, ctypes.byref(seen), None, _lib.stream_ptr()), "status")
        assert seen.value == smt.seen[s]
    c0 = lib.mapnet_launch_count()
    smt.step(fr[lo:lo + 4], vo[lo:lo + 4], [0, 1, 2, 0])
    assert lib.mapnet_launch_count() - c0 == n_sample + (n_sample + 3)
    lb.sample(fr[lo:lo + 4], S)
    lo += 4
    c1 = lib.mapnet_launch_count()
    smt(fr[lo:lo + 9], vo[lo:lo + 9], [0, 1, 2] * 3)      # chunks of 4, 4 and 1: replays only
    assert lib.mapnet_launch_count() == c1 and (len(smt._graphs), len(smt._now_graphs)) == (2, 1)
    lb.sample(fr[lo:lo + 9], S)
    assert torch.equal(la(fr[:3]), lb(fr[:3]))            # the dropout counters end equal: no eager run advanced it
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        smt(fr[:4], vo[:4], [2, 1, 0, 2])
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    for k in ("k_track_multi_gather<mapnet::SampleFactor>", "k_pgo_cov", "k_track_multi_emit<mapnet::SampleFactor>"):
        assert sum(k in n for n in names) == 1, (k, names)
    smt.close(); la.close(); lb.close(); pa.close(); pb.close()
