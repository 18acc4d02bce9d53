"""GPU run of inference.evaluate_sequence (scripts/eval.py's loop over a device-resident sequence): equal to
evaluate_tuples on the same windows assembled by DeviceLoader(shuffle=False), each distinct frame through the engine
once (droprate 0) or every window's frames in window order (droprate > 0), against a float64 restatement of eval.py's
post-processing and PGO, and the VOs of csrc/loader.cu k_eval_windows against calc_vos_safe / calc_vos_safe_fc."""
import ctypes
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

L_SEQ, H_IN, W_IN, STEPS, SKIP = 50, 120, 160, 3, 2
STATS = (np.array([0.45, 0.5, 0.55]), np.array([0.22, 0.25, 0.2]))
POSE_M, POSE_S = np.array([0.5, 1.0, -1.0]), np.array([2.0, 3.0, 1.5])
SIG = dict(sax=1.0, saq=0.5, srx=0.3, srq=0.2)


def _seq(L, seed):
    rng = np.random.default_rng(seed)
    fr = (rng.random((L, H_IN, W_IN, 3)) * 256).astype(np.uint8)
    t = rng.standard_normal((L, 3)).cumsum(0) * 0.2
    v = rng.standard_normal((L, 3))
    v = v / np.linalg.norm(v, axis=1, keepdims=True) * (rng.random((L, 1)) - 0.5) * math.pi
    poses = np.concatenate([t, v], 1).astype(np.float32)
    vo = (poses + rng.standard_normal(poses.shape) * 0.05).astype(np.float32)      # the VO library's own estimates
    return fr, poses, vo


def _dataset(steps, vo_poses=None, seed=1):
    from geomapnet_b200.data import DeviceDataset
    fr, poses, vo = _seq(L_SEQ, seed)
    return DeviceDataset(fr, STATS[0], STATS[1], poses=poses, steps=steps, skip=SKIP, size=96, max_batch=L_SEQ,
                         chunk=16, vo_poses=vo if vo_poses else None), poses, vo


def _windows(ds):
    """x [L,T,3,H,W], targ6 [L,T,6] from DeviceLoader(shuffle=False), as the reference's DataLoader draws them"""
    from geomapnet_b200.data import DeviceLoader
    xs, ts = [], []
    for x, t in DeviceLoader(ds, 8, shuffle=False):
        xs.append(x.clone()); ts.append(t.clone())
    x, t = torch.cat(xs), torch.cat(ts)
    if ds.steps is None:
        x, t = x.unsqueeze(1), t.unsqueeze(1)
    return x, t


def _device_vos7(ds, vo_fc):
    """the windows' VOs through the loader's MFOnline path (k_loader_assemble's calc_vo_logq_safe) and post()"""
    from geomapnet_b200 import _lib
    from geomapnet_b200.inference import post
    rows = ds.eval_tables(vo_fc=vo_fc)["vo_rows"]
    L, E = rows.shape[:2]
    flat = np.ascontiguousarray(rows.reshape(-1, 2), dtype=np.int32)
    out = torch.empty(flat.shape[0], 6, device="cuda")
    x = torch.empty(1, 3, ds.Ho, ds.Wo, device="cuda")
    idx = np.zeros(1, np.int32)
    fp = ctypes.POINTER(ctypes.c_float)
    step = ds.max_batch * ds.targ_per_item
    for lo in range(0, flat.shape[0], step):
        part = np.ascontiguousarray(flat[lo:lo + step])
        _lib.check(_lib.lib().mapnet_frame_cache_assemble(
            ds.h, 1, idx.ctypes.data, None, ds.vo_poses.data_ptr(), ds.vo_poses.shape[0], part.ctypes.data,
            part.shape[0], ds.mean.ctypes.data_as(fp), ds.std.ctypes.data_as(fp), x.data_ptr(),
            out[lo:lo + part.shape[0]].data_ptr(), _lib.stream_ptr()), "assemble")
    return post(out).view(L, E, 7)


def _count_frames(ds):
    seen = []
    orig = ds.assemble_frames

    def counting(frames, x_out):
        seen.append(len(frames))
        return orig(frames, x_out)
    ds.assemble_frames = counting
    return seen


def _model(kind, precision, droprate=0.0):
    from oracle import weights
    from helpers import make_product_model
    st = weights.make_state(7)
    model, _ = make_product_model(st, kind, precision, droprate=droprate)
    return model, st


CASES = [("posenet", None, False), ("posenet", STEPS, True), ("mapnet", STEPS, False), ("mapnet", STEPS, True)]


@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
@pytest.mark.parametrize("kind,steps,use_pgo", CASES, ids=["posenet_single", "posenet_mf_pgo", "mapnet", "mapnet_pgo"])
def test_equals_evaluate_tuples_on_loader_windows(kind, steps, use_pgo, precision):
    from geomapnet_b200.inference import Predictor, evaluate_sequence, evaluate_tuples
    model, _ = _model(kind, precision)
    ds, poses, _ = _dataset(steps, vo_poses=use_pgo)
    pr = Predictor(model, max_batch=16)
    seen = _count_frames(ds)
    got = evaluate_sequence(pr, ds, POSE_M, POSE_S, **SIG)
    n_unique = len(np.unique(ds.eval_tables()["windows"]))
    assert got["n_frames"] == n_unique == sum(seen)            # each distinct frame through the engine once
    x, targ = _windows(ds)
    vos7 = _device_vos7(ds, False) if use_pgo else None
    ref = evaluate_tuples(pr, x, targ, vos7, POSE_M, POSE_S, **SIG)
    for k in ("pred7", "targ7", "t_err", "q_err"):
        assert got[k].shape == ref[k].shape and torch.equal(got[k], ref[k]), k
    pr.close(); ds.close()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_live_model(precision):
    """a live bf16 model runs a temporary Predictor (bitwise that of Predictor(model)); an fp32 one its eval forward"""
    from geomapnet_b200.inference import Predictor, evaluate_sequence, evaluate_tuples
    model, _ = _model("mapnet", precision)
    ds, _, _ = _dataset(STEPS, vo_poses=True)
    got = evaluate_sequence(model, ds, POSE_M, POSE_S, **SIG)
    assert model.training                                      # the mode is restored
    x, targ = _windows(ds)
    vos7 = _device_vos7(ds, False)
    if precision == "bf16":
        pr = Predictor(model)
        ref = evaluate_tuples(pr, x, targ, vos7, POSE_M, POSE_S, **SIG)
        assert all(torch.equal(got[k], ref[k]) for k in ("pred7", "targ7", "t_err", "q_err"))
        pr.close()
    else:
        ref = evaluate_tuples(model, x, targ, vos7, POSE_M, POSE_S, batch=8, **SIG)
        # the fp32 engine's per-frame arithmetic may depend on the batch's tile plan: the live-path bound
        assert float((got["pred7"] - ref["pred7"]).abs().max() / ref["pred7"].abs().max()) <= 2e-5
        assert torch.equal(got["targ7"], ref["targ7"])
    ds.close()


def test_dropout_windows_in_window_order():
    """droprate > 0: one forward per window, in window order, so the masks are those of a fresh Predictor (same seed)
    called window by window, as the reference's loop calls the model"""
    from geomapnet_b200.inference import Predictor, evaluate_sequence, post
    model, _ = _model("mapnet", "tc_split", droprate=0.5)
    ds, _, _ = _dataset(STEPS)
    pr = Predictor(model, max_batch=8)
    seen = _count_frames(ds)
    got = evaluate_sequence(pr, ds, POSE_M, POSE_S)
    assert got["n_frames"] == L_SEQ * STEPS and seen == [STEPS] * L_SEQ
    x, targ = _windows(ds)
    fresh = Predictor(model, max_batch=8)
    out6 = torch.cat([fresh(x[w:w + 1]) for w in range(L_SEQ)])
    p, t = post(out6, POSE_M, POSE_S), post(targ, POSE_M, POSE_S)
    assert torch.equal(got["pred7"], p[:, STEPS // 2]) and torch.equal(got["targ7"], t[:, STEPS // 2])
    again = evaluate_sequence(Predictor(model, max_batch=8), ds, POSE_M, POSE_S)
    assert torch.equal(again["pred7"], got["pred7"])
    pr.close(); fresh.close(); ds.close()


def _np_qexp(v):
    n = np.linalg.norm(v)
    return np.hstack((np.cos(n), np.sinc(n / np.pi) * v))


def _np_calc_vo_safe(p0, p1):
    """common/pose_utils.py:219-232 restated in float64"""
    def qmult(a, b):
        s = a[0] * b[0] - a[1:] @ b[1:]
        v = a[0] * b[1:] + b[0] * a[1:] + np.cross(a[1:], b[1:])
        q = np.concatenate([[s], v])
        return q / np.linalg.norm(q)

    def rot(t, q):
        b = np.cross(q[1:], t)
        return t + 2 * q[0] * b + 2 * np.cross(q[1:], b)

    p0, p1 = p0.astype(np.float64), p1.astype(np.float64)
    q0, q1 = _np_qexp(p0[3:]), _np_qexp(p1[3:])
    q0i = np.concatenate([[q0[0]], -q0[1:]])
    q = qmult(q0i, q1)
    lq = np.zeros(3) if not q[1:].any() else np.arccos(q[0]) * q[1:] / np.linalg.norm(q[1:])
    return np.concatenate([rot(p1[:3] - p0[:3], q0i), lq])


@pytest.mark.parametrize("vo_fc", [False, True])
def test_matches_float64_restatement(vo_fc):
    """oracle eval forward of every frame, then eval.py:147-199 in numpy with the reference's VOs (calc_vos_safe /
    calc_vos_safe_fc of the VO poses) and pgo_oracle, at test_gpu_inference.py's tolerances"""
    from oracle import mapnet_oracle as O, pgo_oracle as P
    from geomapnet_b200.inference import Predictor, evaluate_sequence
    model, st = _model("mapnet", "tc_split")
    ds, poses, vo = _dataset(STEPS, vo_poses=True)
    pr = Predictor(model, max_batch=16)
    got = evaluate_sequence(pr, ds, POSE_M, POSE_S, vo_fc=vo_fc, **SIG)
    x, _ = _windows(ds)
    out6 = pr(x).double().cpu()
    with torch.no_grad():
        stc = {k: (v.double() if v.is_floating_point() else v).cuda() for k, v in st.items()}
        ref6 = O.mapnet_forward(stc, x.double(), training=False).cpu()
    assert float((out6 - ref6).abs().max() / ref6.abs().max()) <= 3e-4
    win = ds.eval_tables()["windows"]
    exp_pred, exp_targ = [], []
    for w in range(L_SEQ):
        o = out6[w].numpy()
        o7 = np.hstack((o[:, :3], np.asarray([_np_qexp(p[3:]) for p in o])))
        t = poses[win[w]].astype(np.float64)
        t7 = np.hstack((t[:, :3], np.asarray([_np_qexp(p[3:]) for p in t])))
        pairs = [(i, j) for i in range(STEPS) for j in range(i + 1, STEPS)] if vo_fc else \
            [(i, i + 1) for i in range(STEPS - 1)]
        v6 = np.stack([_np_calc_vo_safe(vo[win[w, i]], vo[win[w, j]]) for i, j in pairs])
        v7 = np.hstack((v6[:, :3], np.asarray([_np_qexp(p[3:]) for p in v6])))
        o7 = P.optimize_poses(o7, v7, fc_vos=vo_fc, **SIG)
        o7[:, :3] = o7[:, :3] * POSE_S + POSE_M
        t7[:, :3] = t7[:, :3] * POSE_S + POSE_M
        exp_pred.append(o7[STEPS // 2]); exp_targ.append(t7[STEPS // 2])
    exp_pred, exp_targ = np.stack(exp_pred), np.stack(exp_targ)
    ep = np.abs(got["pred7"].cpu().numpy() - exp_pred).max() / np.abs(exp_pred).max()
    et = np.abs(got["targ7"].cpu().numpy() - exp_targ).max()
    print("vo_fc=%s: pred7 rel err %.2e, targ7 abs err %.2e" % (vo_fc, ep, et))
    assert ep <= 2e-5 and et <= 1e-6
    t_ref = np.linalg.norm(exp_pred[:, :3] - exp_targ[:, :3], axis=1)
    assert np.abs(got["t_err"].cpu().numpy() - t_ref).max() <= 1e-3 * t_ref.max()
    pr.close(); ds.close()


def test_vo_windows_match_calc_vos_safe():
    """k_eval_windows' VOs against calc_vos_safe / calc_vos_safe_fc restated in float64 (float32 on the device)"""
    from geomapnet_b200 import _lib
    ds, poses, vo = _dataset(STEPS, vo_poses=True)
    for vo_fc in (False, True):
        tab = ds.eval_tables(vo_fc=vo_fc)
        L, E = tab["vo_rows"].shape[:2]
        F = tab["frames"].shape[0]
        pred6 = torch.zeros(F, 6, device="cuda")
        p7 = torch.empty(L, STEPS, 7, dtype=torch.float64, device="cuda")
        t7, v7 = torch.empty_like(p7), torch.empty(L, E, 7, dtype=torch.float64, device="cuda")
        _lib.check(_lib.lib().mapnet_eval_windows(
            pred6.data_ptr(), F, ds.poses.data_ptr(), ds.vo_poses.data_ptr(), ds.poses.shape[0],
            tab["windows"].ctypes.data, tab["slots"].ctypes.data, L * STEPS, tab["vo_rows"].ctypes.data, L * E,
            p7.data_ptr(), t7.data_ptr(), v7.data_ptr(), _lib.stream_ptr()), "mapnet_eval_windows")
        got = v7.cpu().numpy()
        win = tab["windows"]
        pairs = [(i, j) for i in range(STEPS) for j in range(i + 1, STEPS)] if vo_fc else \
            [(i, i + 1) for i in range(STEPS - 1)]
        exp = np.stack([np.stack([_np_calc_vo_safe(vo[win[w, i]], vo[win[w, j]]) for i, j in pairs])
                        for w in range(L)])
        exp7 = np.concatenate([exp[..., :3], np.stack([[_np_qexp(p[3:]) for p in r] for r in exp])], -1)
        rel = (np.abs(got - exp7) / np.maximum(np.abs(exp7), 1.0)).max()
        print("vo_fc=%s: VO err / max(|vo|, 1) %.2e" % (vo_fc, rel))
        assert rel <= 2e-6
        assert np.array_equal(t7[:, :, :3].cpu().numpy(), poses[win][..., :3].astype(np.float64))
    # bad index tables fail before any launch
    lc = _lib.lib().mapnet_launch_count()
    bad = tab["vo_rows"].copy()
    bad[3, 0, 1] = ds.poses.shape[0]
    assert _lib.lib().mapnet_eval_windows(
        pred6.data_ptr(), F, ds.poses.data_ptr(), ds.vo_poses.data_ptr(), ds.poses.shape[0], tab["windows"].ctypes.data,
        tab["slots"].ctypes.data, L * STEPS, bad.ctypes.data, L * E, p7.data_ptr(), t7.data_ptr(), v7.data_ptr(),
        _lib.stream_ptr()) != 0
    assert b"outside" in _lib.lib().mapnet_last_error()
    assert _lib.lib().mapnet_launch_count() == lc
    ds.close()
