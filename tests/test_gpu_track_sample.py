"""GPU tests of the covariance-weighted pose graph (k_pgo_cov, common.pgo.optimize_pose_windows_cov) and of
inference.SampledTracker: the kernel against the numpy oracle of test_track_sample_host on random windows, against
k_pgo's exact solve with the reference's factors, the posterior against the per-frame Monte-Carlo covariance when the
relative factors are switched off, bitwise determinism, the tracker against the composition of Predictor.sample,
eval.py's windows and optimize_pose_windows_cov, and one graph replay of the sampled engine plus three tracking
launches per chunk."""
import math

import numpy as np
import pytest
import torch

from test_track_sample_host import factor, optimize_cov, random_window
from oracle import pgo_oracle as po

pytestmark = pytest.mark.gpu

MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]
STD = [float(np.sqrt(v)) for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
POSE_M, POSE_S = [0.5, -1.25, 2.0], [1.5, 0.75, 2.5]
SIG = dict(sax=1e-3, saq=1e-3, srx=20.0, srq=20.0)
S = 16
L_SEQ, H_IN, W_IN = 61, 480, 640
CONFIGS = [(3, 2, False), (4, 5, False), (7, 3, True)]          # (steps, skip, vo_fc)


def _rel(got, want):
    got, want = np.asarray(got), np.asarray(want)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300))


# ---------------------------------------------------------------------------------------------------------------------
# 1-4. the kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,fc", [(2, False), (3, False), (3, True), (7, False), (7, True), (16, False), (16, True)])
def test_kernel_matches_the_numpy_oracle(N, fc):
    from geomapnet_b200.common.pgo import optimize_pose_windows_cov
    rng = np.random.default_rng(N * 2 + fc)
    W = {2: 60, 3: 60, 7: 40, 16: 12}[N]
    wins = [random_window(rng, N, fc) for _ in range(W)]
    P, C, V = (np.stack([w[k] for w in wins]) for k in range(3))
    got_p, got_c = optimize_pose_windows_cov(torch.from_numpy(P).cuda(), C, V, fc_vos=fc, srx=0.5, srq=0.2)
    got_p, got_c = got_p.cpu().numpy(), got_c.cpu().numpy()
    for w in range(W):
        want_p, want_c = optimize_cov(P[w], C[w], V[w], fc, 0.5, 0.2)
        assert _rel(got_p[w], want_p) < 1e-10, (w, _rel(got_p[w], want_p))
        assert _rel(got_c[w], want_c) < 1e-8, (w, _rel(got_c[w], want_c))
    # determinism: the same call again is bit for bit the same
    again_p, again_c = optimize_pose_windows_cov(torch.from_numpy(P).cuda(), C, V, fc_vos=fc, srx=0.5, srq=0.2)
    assert np.array_equal(again_p.cpu().numpy(), got_p) and np.array_equal(again_c.cpu().numpy(), got_c)


@pytest.mark.parametrize("N,fc", [(3, False), (7, True), (16, False)])
def test_reference_factors_give_the_exact_solve_of_k_pgo(N, fc):
    from geomapnet_b200.common.pgo import optimize_pose_windows, optimize_pose_windows_cov
    rng = np.random.default_rng(40 + N)
    wins = [random_window(rng, N, fc) for _ in range(20)]
    P, V = np.stack([w[0] for w in wins]), np.stack([w[2] for w in wins])
    sax, saq, srx, srq = 0.4, 0.1, 2.0, 3.0
    C = np.broadcast_to(np.diag([sax] * 3 + [saq] * 4), (20, N, 7, 7)).copy()
    got, _ = optimize_pose_windows_cov(torch.from_numpy(P).cuda(), C, V, fc_vos=fc, srx=srx, srq=srq)
    want = optimize_pose_windows(torch.from_numpy(P).cuda(), V, fc, sax, saq, srx, srq, exact_solve=True)
    assert float((got - want).abs().max()) < 1e-12


def test_not_positive_definite_raises():
    from geomapnet_b200.common.pgo import optimize_pose_windows_cov
    rng = np.random.default_rng(1)
    P, C, V = random_window(rng, 3, False)
    C[1] = -np.eye(7)
    with pytest.raises(np.linalg.LinAlgError):
        optimize_pose_windows_cov(torch.from_numpy(P[None]).cuda(), C[None], V[None])


# ---------------------------------------------------------------------------------------------------------------------
# helpers for the tracker
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def seq():
    rng = np.random.default_rng(7)
    fr = rng.integers(0, 256, (L_SEQ, H_IN, W_IN, 3), dtype=np.uint8)
    s = np.arange(L_SEQ)[:, None] / 10.0
    t = np.concatenate([np.sin(s), np.cos(0.7 * s), 0.1 * s], 1)
    lq = np.concatenate([0.2 * np.sin(0.3 * s), 0.1 * np.cos(0.5 * s), 0.05 * s], 1)
    vo = (np.concatenate([t, lq], 1) + rng.standard_normal((L_SEQ, 6)) * 0.02).astype(np.float32)
    return torch.from_numpy(fr).cuda(), vo


def _model(seed=5, droprate=0.5, precision="bf16"):
    from oracle import weights
    from helpers import make_product_model
    model, _ = make_product_model(weights.make_state(seed), "mapnet", precision, droprate=droprate)
    return model


def _pair(max_batch, precision=None, calib=None, seed=5):
    """two Predictors of one model with equal seeds and counters: A tracks, B composes"""
    from geomapnet_b200.inference import Predictor
    model = _model(seed)
    kw = dict(precision=precision, calibration=calib) if precision else {}
    pa, pb = Predictor(model, max_batch=max_batch, **kw), Predictor(model, max_batch=max_batch, **kw)
    pa.seed = pb.seed = 20261018                          # the model's default is torch.initial_seed(), new every run
    return pa, pb


def _tracker(pr, T, skip, fc, metric=True):
    from geomapnet_b200.inference import Localizer, SampledTracker
    loc = Localizer(pr, MEAN, STD, *((POSE_M, POSE_S) if metric else ()))
    return loc, SampledTracker(loc, S, steps=T, skip=skip, vo_fc=fc, **SIG)


def _draws(pb, frames, sizes):
    """the normalised mean [L,6] and cov [L,6,6] of each frame's draws, one Predictor.sample per call size"""
    from geomapnet_b200.data import ImagePipeline
    pipe = ImagePipeline(MEAN, STD)
    los = np.cumsum([0] + list(sizes))
    outs = [pb.sample(pipe(frames[a:b]), S) for a, b in zip(los[:-1], los[1:])]
    return (torch.cat([o["mean"] for o in outs]).cpu().numpy(), torch.cat([o["cov"] for o in outs]).cpu().numpy())


def _factors(mean, cov, sax, saq):
    """(p [n,7], S7 [n,7,7]) on the device, as the tracker forms them (mapnet_test_sample_factor)"""
    from geomapnet_b200 import _lib
    n = mean.shape[0]
    md, cd = torch.as_tensor(mean).cuda().contiguous(), torch.as_tensor(cov).cuda().contiguous()
    p7 = torch.empty((n, 7), dtype=torch.float64, device="cuda")
    s7 = torch.empty((n, 7, 7), dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().mapnet_test_sample_factor(md.data_ptr(), cd.data_ptr(), n, sax, saq, p7.data_ptr(),
                                                    s7.data_ptr(), _lib.stream_ptr()), "mapnet_test_sample_factor")
    return p7, s7


def _solve(mean, cov, vo, T, skip, fc, centres, last, keep, metric=True):
    """eval.py's windows of the given centres (slots clipped at 0 and last), each frame's p and S7 (checked against the
    numpy oracle in test_device_factors_match_the_oracle), optimize_pose_windows_cov; slot `keep` of each, as the
    tracker emits it: dict(pose7, cov, t_std, q_std_deg)"""
    from geomapnet_b200.common.pgo import optimize_pose_windows_cov
    from geomapnet_b200 import _lib
    n = mean.shape[0]
    p7, s7 = _factors(mean, cov, SIG["sax"], SIG["saq"])
    idx = np.array([[min(max(c + (k - T // 2) * skip, 0), last) for k in range(T)] for c in centres], dtype=np.int32)
    pairs = po.edges(T, fc)
    vo_rows = np.ascontiguousarray(idx[:, np.asarray(pairs)], dtype=np.int32)
    W, E = idx.shape[0], len(pairs)
    vo_dev = torch.as_tensor(vo[:n]).cuda().contiguous()
    dummy = torch.zeros((n, 6), dtype=torch.float32, device="cuda")
    w7, t7 = (torch.empty((W, T, 7), dtype=torch.float64, device="cuda") for _ in range(2))
    vos7 = torch.empty((W, E, 7), dtype=torch.float64, device="cuda")
    flat = np.ascontiguousarray(idx.reshape(-1))
    _lib.check(_lib.lib().mapnet_eval_windows(dummy.data_ptr(), n, dummy.data_ptr(), vo_dev.data_ptr(), n,
                                              flat.ctypes.data, flat.ctypes.data, W * T, vo_rows.ctypes.data, W * E,
                                              w7.data_ptr(), t7.data_ptr(), vos7.data_ptr(), _lib.stream_ptr()),
               "mapnet_eval_windows")
    ix = torch.from_numpy(idx.astype(np.int64)).cuda()
    z, cv = optimize_pose_windows_cov(p7[ix], s7[ix], vos7, fc_vos=fc, srx=SIG["srx"], srq=SIG["srq"])
    z, cv = z[:, keep], cv[:, keep]
    d = torch.tensor(list(POSE_S) + [1.0] * 3 if metric else [1.0] * 6, dtype=torch.float64, device="cuda")
    if metric:
        m = torch.tensor(POSE_M, dtype=torch.float64, device="cuda")
        z = torch.cat((z[:, :3] * d[:3] + m, z[:, 3:]), -1)
    cv = d[:, None] * cv * d[None, :]
    tt = cv[:, 0, 0] + cv[:, 1, 1] + cv[:, 2, 2]
    tq = cv[:, 3, 3] + cv[:, 4, 4] + cv[:, 5, 5]
    return dict(pose7=z, cov=cv, t_std=tt.sqrt(), q_std_deg=2.0 * tq.sqrt() * (180.0 / math.pi))


def _assert_close(got, want, what):
    for k, tol in (("pose7", 1e-12), ("cov", 1e-9), ("t_std", 1e-9), ("q_std_deg", 1e-9)):
        assert got[k].shape == want[k].shape, (what, k, tuple(got[k].shape), tuple(want[k].shape))
        if got[k].numel():
            r = _rel(got[k].cpu().numpy(), want[k].cpu().numpy())
            assert r < tol, (what, k, r)


def _track(st, frames, vo, sizes, now=False):
    """every estimate of the sequence (calls or steps of `sizes` frames, then flush), and the zero-lag rows"""
    outs, nows, nxt, lo = [], [], 0, 0
    for n in sizes:
        if now:
            nw, first, est = st.step(frames[lo:lo + n], vo[lo:lo + n])
            nows.append(nw)
        else:
            first, est = st(frames[lo:lo + n], vo[lo:lo + n])
        assert first == nxt and est["pose7"].shape[0] == max(lo + n - st.lag, 0) - max(lo - st.lag, 0)
        outs.append(est)
        nxt += est["pose7"].shape[0]
        lo += n
    first, est = st.flush()
    assert first == nxt and nxt + est["pose7"].shape[0] == lo and st.seen == 0
    outs.append(est)
    cat = lambda ds: {k: torch.cat([d[k] for d in ds]) for k in ds[0]}
    return cat(outs), (cat(nows) if now else None)


def _chunks(L, B):
    return [min(B, L - lo) for lo in range(0, L, B)]


def test_device_factors_match_the_oracle():
    """the tracker's p and S7 (mapnet_test_sample_factor): p bit for bit mapnet_sample_post's pose7 without pose
    statistics, S7 the numpy oracle's factor() to rounding, across |v| from 0 to 2.5"""
    from geomapnet_b200 import _lib
    rng = np.random.default_rng(5)
    ns = [0.0, 1e-12, 1e-9, 1e-6, 1e-3, 0.0999, 0.1, 0.1001, 0.5, 1.0, 2.0, 2.5]
    mean = rng.standard_normal((len(ns), 6)) * 3.0
    for k, n in enumerate(ns):
        mean[k, 3:] *= n / np.linalg.norm(mean[k, 3:])
    A = rng.standard_normal((len(ns), 6, 6)) * 0.1
    cov = A @ A.transpose(0, 2, 1)
    cov[0] = 0.0                                          # no spread: S7 is the floors alone
    p7, s7 = _factors(mean, cov, 1e-3, 2e-3)
    post7 = torch.empty_like(p7)
    ts = torch.empty(len(ns), dtype=torch.float64, device="cuda")
    qs = torch.empty_like(ts)
    md, cd = torch.from_numpy(mean).cuda(), torch.from_numpy(cov).cuda()
    _lib.check(_lib.lib().mapnet_sample_post(md.data_ptr(), cd.data_ptr(), len(ns), None, None, post7.data_ptr(), None,
                                             ts.data_ptr(), qs.data_ptr(), _lib.stream_ptr()), "mapnet_sample_post")
    assert torch.equal(p7, post7)
    p7, s7 = p7.cpu().numpy(), s7.cpu().numpy()
    for k in range(len(ns)):
        want_p, want_s = factor(mean[k], cov[k], 1e-3, 2e-3)
        assert _rel(p7[k], want_p) < 1e-15, (ns[k], _rel(p7[k], want_p))
        assert _rel(s7[k], want_s) < 1e-13, (ns[k], _rel(s7[k], want_s))
    assert np.array_equal(s7[0], np.diag([1e-3] * 3 + [2e-3] * 4))


# ---------------------------------------------------------------------------------------------------------------------
# 3. decoupling: the posterior is the frame's own Monte-Carlo covariance
# ---------------------------------------------------------------------------------------------------------------------
def test_decoupled_posterior_is_the_per_frame_monte_carlo_covariance(seq):
    from geomapnet_b200.common.pgo import optimize_pose_windows_cov
    from geomapnet_b200.inference import Localizer
    frames, _ = seq
    pa, _ = _pair(8)
    loc = Localizer(pa, MEAN, STD)
    out = loc.sample(frames[:16], S)
    cov = out["cov"].cpu().numpy()
    pose7 = out["pose7"].cpu().numpy()
    T = 4
    P = pose7.reshape(4, T, 7)
    # the normalised mean log q from pose7: the draws' mean is qlog of its quaternion
    from test_track_sample_host import qlog
    mu = np.concatenate((pose7[:, :3], np.stack([qlog(q) for q in pose7[:, 3:]])), 1)
    C = np.stack([factor(mu[f], cov[f], 1e-9, 1e-9)[1] for f in range(16)]).reshape(4, T, 7, 7)
    # VOs equal to the poses' own relative transforms: the relative factors start at zero residual
    V = np.stack([[np.concatenate((po.rotate_vector(w[k + 1, :3] - w[k, :3], po.qinverse(w[k, 3:])),
                                   po.qmult(po.qinverse(w[k, 3:]), w[k + 1, 3:]))) for k in range(T - 1)] for w in P])
    z, cv = optimize_pose_windows_cov(torch.from_numpy(P).cuda(), C, V, srx=1e12, srq=1e12)
    assert float((z.reshape(16, 7) - out["pose7"]).abs().max()) < 1e-9
    cv = cv.reshape(16, 6, 6)
    for f in range(16):
        err = float(torch.linalg.norm(cv[f] - out["cov"][f]) / torch.linalg.norm(out["cov"][f]))
        assert err < 1e-4, (f, err)
    loc.close(); pa.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. the tracker against the composition
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 8, 32])
def test_tracker_equals_the_composition(seq, B):
    frames, vo = seq
    for T, skip, fc in (CONFIGS if B == 8 else CONFIGS[-1:]):
        pa, pb = _pair(B)
        loc, st = _tracker(pa, T, skip, fc)
        sizes = _chunks(L_SEQ, B)
        got, _ = _track(st, frames, vo, sizes)
        mean, cov = _draws(pb, frames, sizes)
        want = _solve(mean, cov, vo, T, skip, fc, range(L_SEQ), L_SEQ - 1, T // 2)
        _assert_close(got, want, (B, T, skip, fc))
        st.close(); loc.close(); pa.close(); pb.close()


def test_steps_mixed_with_calls_and_zero_lag_rows(seq):
    frames, vo = seq
    T, skip, fc = 7, 3, True
    pa, pb = _pair(8)
    loc, st = _tracker(pa, T, skip, fc)
    sizes = [3, 8, 8, 5, 8, 8, 8, 8, 5]
    outs, nows, lo = [], [], 0
    for k, n in enumerate(sizes):                         # steps and calls alternate on one sequence
        if k % 2:
            nw, first, est = st.step(frames[lo:lo + n], vo[lo:lo + n])
            nows.append((lo, nw))
        else:
            first, est = st(frames[lo:lo + n], vo[lo:lo + n])
        outs.append(est)
        lo += n
    outs.append(st.flush()[1])
    mean, cov = _draws(pb, frames, sizes)
    want = _solve(mean, cov, vo, T, skip, fc, range(lo), lo - 1, T // 2)
    _assert_close({k: torch.cat([d[k] for d in outs]) for k in outs[0]}, want, "mixed")
    for a, nw in nows:                                    # the window that ends at each frame: its last slot
        fs = list(range(a, a + nw["pose7"].shape[0]))
        wn = _solve(mean[:fs[-1] + 1], cov[:fs[-1] + 1], vo, T, skip, fc, [f - st.lag for f in fs], fs[-1], T - 1)
        # slots of a zero-lag window never pass its own frame, so clipping at the step's last frame is the same
        _assert_close(nw, wn, ("now", a))
    st.close(); loc.close(); pa.close(); pb.close()


def test_short_sequence_reset_refresh_and_normalised_output(seq):
    from geomapnet_b200.common.optimizer import Optimizer
    frames, vo = seq
    T, skip, fc = 4, 5, False
    pa, pb = _pair(8, seed=9)
    loc, st = _tracker(pa, T, skip, fc, metric=False)
    short = [5]                                           # shorter than the lag of 10: everything comes from flush
    got, _ = _track(st, frames, vo, short)
    assert got["pose7"].shape[0] == 5
    mean, cov = _draws(pb, frames, short)
    _assert_close(got, _solve(mean, cov, vo, T, skip, fc, range(5), 4, T // 2, metric=False), "short")
    st(frames[:13], vo[:13])                              # an abandoned sequence
    st.reset()
    assert st.seen == 0
    _draws(pb, frames, [8, 5])                            # keep the counters equal
    model = pa.model
    # a small step: a large one leaves this dropout model's draws so spread that its windows are not positive definite
    opt = Optimizer(params=model.parameters(), method="adam", base_lr=1e-4, weight_decay=0.0)
    model.train()
    x = torch.randn(2, 2, 3, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    model(x).square().sum().backward()
    opt.learner.step()
    pa.refresh(); pb.refresh()
    sizes = _chunks(30, 8)
    got, _ = _track(st, frames, vo, sizes)
    mean, cov = _draws(pb, frames, sizes)
    _assert_close(got, _solve(mean, cov, vo, T, skip, fc, range(30), 29, T // 2, metric=False), "refreshed")
    st.close()
    with pytest.raises(ValueError, match="closed"):
        st(frames[:1], vo[:1])
    loc.close(); pa.close(); pb.close()


def test_fp8_predictor(seq):
    from geomapnet_b200.data import ImagePipeline
    frames, vo = seq
    T, skip, fc = 7, 3, True
    pa, pb = _pair(8, "fp8", ImagePipeline(MEAN, STD)(frames[:8]))
    loc, st = _tracker(pa, T, skip, fc)
    sizes = _chunks(40, 8)
    got, _ = _track(st, frames, vo, sizes)
    mean, cov = _draws(pb, frames, sizes)
    _assert_close(got, _solve(mean, cov, vo, T, skip, fc, range(40), 39, T // 2), "fp8")
    st.close(); loc.close(); pa.close(); pb.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. launches
# ---------------------------------------------------------------------------------------------------------------------
def test_one_replay_of_the_sampled_engine_and_three_tracking_launches_per_chunk(seq):
    from geomapnet_b200 import _lib
    frames, vo = seq
    lib = _lib.lib()
    pa, _ = _pair(4)
    loc, st = _tracker(pa, 4, 5, False)
    pa._engine(256, 341)
    loc._plan(H_IN, W_IN)
    c0 = lib.mapnet_launch_count()
    loc.sample(frames[:4], S)                             # the sampled engine's launches: eager run + capture
    n_sample = (lib.mapnet_launch_count() - c0) // 2 - 1  # minus mapnet_sample_post
    lo = 4
    for B in (1, 4):
        c0 = lib.mapnet_launch_count()
        st(frames[lo:lo + B], vo[lo:lo + B])
        assert lib.mapnet_launch_count() - c0 == n_sample + (n_sample + 3), (B, lib.mapnet_launch_count() - c0)
        lo += B
    c1 = lib.mapnet_launch_count()
    st(frames[lo:lo + 9], vo[lo:lo + 9])                  # chunks of 4, 4 and 1: replays only
    assert lib.mapnet_launch_count() == c1 and len(st._graphs) == 2
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        st(frames[:4], vo[:4])
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    for k in ("k_track_gather<mapnet::SampleFactor>", "k_pgo_cov", "k_track_emit<mapnet::SampleFactor>"):
        assert sum(k in n for n in names) == 1, (k, names)
    st.close(); loc.close(); pa.close()
