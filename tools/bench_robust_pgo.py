"""Cauchy-weighted pose graphs on the H100: what robust_c costs per launch and per tracker call, and what it buys on a
synthetic trajectory with gross outliers.

    python tools/bench_robust_pgo.py [--rounds 5] [--pgo-iters 1000] [--iters 100] [--frames 2000] [--out FILE]

Arms alternate plain / robust inside each of `--rounds` rounds; medians are reported.
  pgo        one k_pgo (the trackers' literal solve, flags 0) and one k_pgo_cov launch at RobotCar's geometry (T = 7,
             vo_fc), 1 and 64 windows, plain against robust_c = 2 (CUDA events over --pgo-iters launches)
  per_call   Tracker and SampledTracker (S = 32) calls at B = 1, past the lag, plain against robust_c = 2 (CUDA events
             over --iters calls); the frames, model and RobotCar PGO geometry of tools/bench_track_sample.py
  accuracy   a seeded synthetic trajectory of --frames poses: absolute poses with Gaussian noise (0.1 in translation,
             0.02 rad in rotation) and 5 % gross outliers (2.0 in translation, 0.5 rad), VO of the true relative poses
             with small noise; every frame's T = 7 fc window solved on the GPU in float64 (one launch per arm) and its
             middle slot scored against the truth: median and 95th-percentile translation and rotation error of no
             PGO, plain PGO and robust PGO at c in {1, 2, 4}, with the literal (flags 0) and the exact step.  Synthetic
             data: not a real-data accuracy.
The card's name, power limit and clocks are read in the same run.  Prints one JSON line (and writes it to --out).  No
CPU fallback: without a GPU it exits.
"""
import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_track import MEAN, STD, POSE_M, POSE_S, H_IN, W_IN, T, SKIP, FC  # noqa: E402

S = 32
C = 2.0
SIG = dict(sax=1.0, saq=1.0, srx=20.0, srq=20.0)
SSIG = dict(sax=1e-4, saq=1e-4, srx=20.0, srq=20.0)


def _qmul(a, b):
    import numpy as np
    w1, x1, y1, z1 = np.moveaxis(a, -1, 0)
    w2, x2, y2, z2 = np.moveaxis(b, -1, 0)
    return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1)


def _qexp(v):
    import numpy as np
    n = np.linalg.norm(v, axis=-1, keepdims=True)
    sc = np.where(n > 0, np.sin(n) / np.where(n > 0, n, 1.0), 1.0)
    return np.concatenate((np.cos(n), sc * v), -1)


def _qinv(q):
    return q * [1.0, -1.0, -1.0, -1.0]


def _rotate(v, q):
    import numpy as np
    p = np.concatenate((np.zeros(v.shape[:-1] + (1,)), v), -1)
    return _qmul(_qmul(q, p), _qinv(q))[..., 1:]


def synthetic(n, seed=0):
    """(truth [n,7], predictions [n,7], vo_rows of every frame's fc window [n,E,7], windows [n,T] int, outlier mask)"""
    import numpy as np
    rng = np.random.default_rng(seed)
    s = np.arange(n)[:, None] / 20.0
    t = np.concatenate([10 * np.sin(0.2 * s), 10 * np.cos(0.13 * s), 0.5 * s], 1)
    q = _qexp(np.concatenate([0.2 * np.sin(0.3 * s), 0.1 * np.cos(0.5 * s), 0.3 * s], 1))
    truth = np.concatenate((t, q), 1)
    pt = t + rng.standard_normal((n, 3)) * 0.1
    pq = _qmul(q, _qexp(rng.standard_normal((n, 3)) * 0.01))             # 0.02 rad: a log q step of 0.01
    out = rng.random(n) < 0.05
    d = rng.standard_normal((n, 3))
    pt[out] += 2.0 * d[out] / np.linalg.norm(d[out], axis=1, keepdims=True)
    a = rng.standard_normal((n, 3))
    pq[out] = _qmul(pq[out], _qexp(0.25 * a[out] / np.linalg.norm(a[out], axis=1, keepdims=True)))
    pred = np.concatenate((pt, pq), 1)
    windows = np.clip(np.arange(n)[:, None] + np.arange(T)[None] - T // 2, 0, n - 1)
    pairs = [(i, j) for i in range(T) for j in range(i + 1, T)]
    ia, ib = windows[:, [p[0] for p in pairs]], windows[:, [p[1] for p in pairs]]
    vt = _rotate(t[ib] - t[ia], _qinv(q[ia])) + rng.standard_normal(ia.shape + (3,)) * 0.01
    vq = _qmul(_qmul(_qinv(q[ia]), q[ib]), _qexp(rng.standard_normal(ia.shape + (3,)) * 0.001))
    return truth, pred, np.concatenate((vt, vq), -1), windows, out


def errors(p, truth):
    import numpy as np
    te = np.linalg.norm(p[:, :3] - truth[:, :3], axis=1)
    qn = p[:, 3:] / np.linalg.norm(p[:, 3:], axis=1, keepdims=True)
    qe = 2 * np.degrees(np.arccos(np.clip(np.abs((qn * truth[:, 3:]).sum(1)), 0.0, 1.0)))
    return {"t_median": round(float(np.median(te)), 5), "t_p95": round(float(np.percentile(te, 95)), 5),
            "q_median_deg": round(float(np.median(qe)), 5), "q_p95_deg": round(float(np.percentile(qe, 95)), 5)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--pgo-iters", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_robust_pgo.json"))
    a = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_robust_pgo: no CUDA device")
    from bench_infer import card, events_ms
    from geomapnet_b200 import _lib
    from geomapnet_b200.common.pgo import optimize_pose_windows, optimize_pose_windows_cov
    from geomapnet_b200.data import resize_output_size
    from geomapnet_b200.inference import Localizer, Predictor, SampledTracker, Tracker
    from geomapnet_b200.models.posenet import PoseNet
    L = _lib.lib()
    E = T * (T - 1) // 2
    res = {"what": "Cauchy-weighted absolute factors (robust_c) against the plain pose graph: k_pgo / k_pgo_cov "
                   "launches at T = 7 vo_fc for 1 and 64 windows, Tracker / SampledTracker calls at B = 1, and "
                   "accuracy on a seeded synthetic trajectory with 5 % gross outliers (float64, synthetic: not a "
                   "real-data accuracy)",
           "card": card(), "robust_c": C, "steps": T, "vo_fc": FC, "rounds": a.rounds, "pgo_iters": a.pgo_iters,
           "iters": a.iters}

    # ---- 1. one launch, 1 and 64 windows
    f64 = dict(dtype=torch.float64, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(5)
    stat = torch.zeros(1, dtype=torch.int32, device="cuda")
    pgo_ms, pgo_rounds = {}, {}
    for W in (1, 64):
        w7 = torch.randn(W, T, 7, generator=g, **f64) * 0.01
        w7[..., 3] += 1.0
        v7 = torch.randn(W, E, 7, generator=g, **f64) * 0.01
        v7[..., 3] += 1.0
        c7 = torch.diag(torch.tensor([1e-2] * 3 + [1e-3] * 4, dtype=torch.float64)).expand(W, T, 7, 7).contiguous().cuda()
        o7, oc, ow = torch.empty_like(w7), torch.empty((W, T, 6, 6), **f64), torch.empty((W, T), **f64)
        arms = {
            "k_pgo": lambda: L.mapnet_pgo_optimize(w7.data_ptr(), v7.data_ptr(), o7.data_ptr(), W, T, 1, 1e-2, 1e-3,
                                                   20.0, 20.0, 10, 0, stat.data_ptr(), _lib.stream_ptr()),
            "k_pgo_robust": lambda: L.mapnet_pgo_optimize_robust(w7.data_ptr(), v7.data_ptr(), o7.data_ptr(), W, T, 1,
                                                                 1e-2, 1e-3, 20.0, 20.0, 10, 0, C, ow.data_ptr(),
                                                                 stat.data_ptr(), _lib.stream_ptr()),
            "k_pgo_cov": lambda: L.mapnet_pgo_optimize_cov(w7.data_ptr(), c7.data_ptr(), v7.data_ptr(), o7.data_ptr(),
                                                           oc.data_ptr(), W, T, 1, 20.0, 20.0, 10, stat.data_ptr(),
                                                           _lib.stream_ptr()),
            "k_pgo_cov_robust": lambda: L.mapnet_pgo_optimize_cov_robust(
                w7.data_ptr(), c7.data_ptr(), v7.data_ptr(), o7.data_ptr(), oc.data_ptr(), W, T, 1, 20.0, 20.0, 10, C,
                ow.data_ptr(), stat.data_ptr(), _lib.stream_ptr())}
        for fn in arms.values():
            for _ in range(10):
                assert fn() == 0, L.mapnet_last_error()
        t = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                t[k].append(events_ms(fn, a.pgo_iters))
        pgo_ms["windows_%d" % W] = {k: round(statistics.median(v), 5) for k, v in t.items()}
        pgo_rounds["windows_%d" % W] = {k: [round(x, 5) for x in v] for k, v in t.items()}
    assert int(stat.item()) == 0
    res["pgo_launch_ms"], res["pgo_launch_rounds"] = pgo_ms, pgo_rounds
    print(json.dumps(pgo_ms), file=sys.stderr)

    # ---- 2. tracker calls at B = 1
    Ho, Wo = resize_output_size(H_IN, W_IN)
    lag = (T - 1 - T // 2) * SKIP
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False, precision="bf16",
                  seed=7).cuda()
    with torch.no_grad():
        net.train()
        for _ in range(3):
            net(torch.randn(16, 3, Ho, Wo, device="cuda"))
    net.eval()
    n_frames = a.iters + lag + 64
    gf = torch.Generator(device="cuda").manual_seed(11)
    frames = torch.randint(0, 256, (n_frames, H_IN, W_IN, 3), dtype=torch.uint8, device="cuda", generator=gf)
    rng = np.random.default_rng(3)
    s = np.arange(n_frames)[:, None] / 50.0
    poses = np.concatenate([np.sin(s), np.cos(0.7 * s), 0.1 * s, 0.2 * np.sin(0.3 * s), 0.1 * np.cos(0.5 * s),
                            0.05 * s], 1).astype(np.float32)
    vo_dev = torch.from_numpy((poses + rng.standard_normal(poses.shape) * 0.02).astype(np.float32)).cuda()
    with torch.no_grad():
        pr = Predictor(net, max_batch=1)
        loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
        trackers = {"tracker": Tracker(loc, steps=T, skip=SKIP, vo_fc=FC, **SIG),
                    "tracker_robust": Tracker(loc, steps=T, skip=SKIP, vo_fc=FC, robust_c=C, **SIG),
                    "sampled": SampledTracker(loc, S, steps=T, skip=SKIP, vo_fc=FC, **SSIG),
                    "sampled_robust": SampledTracker(loc, S, steps=T, skip=SKIP, vo_fc=FC, robust_c=C, **SSIG)}
        pos = {k: 0 for k in trackers}

        def arm(k):
            def call():
                i = pos[k] % n_frames
                pos[k] += 1
                return trackers[k](frames[i:i + 1], vo_dev[i:i + 1])
            return call
        arms = {k: arm(k) for k in trackers}
        for _ in range(lag + 1):                          # past the lag: every call emits a pose
            for fn in arms.values():
                fn()
        torch.cuda.synchronize()
        t = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                t[k].append(events_ms(fn, a.iters))
        res["per_call_b1_ms"] = {k: round(statistics.median(v), 4) for k, v in t.items()}
        res["per_call_b1_rounds"] = {k: [round(x, 4) for x in v] for k, v in t.items()}
        for trk in trackers.values():
            trk.close()
        loc.close(); pr.close()
    print(json.dumps(res["per_call_b1_ms"]), file=sys.stderr)

    # ---- 3. accuracy on a synthetic trajectory with outliers
    truth, pred, vos, windows, out = synthetic(a.frames)
    p7 = torch.from_numpy(np.ascontiguousarray(pred[windows])).cuda()
    v7 = torch.from_numpy(np.ascontiguousarray(vos)).cuda()
    sig = dict(sax=0.1 ** 2, saq=0.01 ** 2, srx=0.01 ** 2, srq=0.001 ** 2)
    acc = {"frames": a.frames, "outliers": int(out.sum()), "sigmas": sig, "no_pgo": errors(pred, truth)}
    for step, exact in (("literal", False), ("exact", True)):
        for c in (None, 1.0, 2.0, 4.0):
            name = "%s_%s" % ("plain" if c is None else "robust_c%g" % c, step)
            try:
                r = optimize_pose_windows(p7, v7, fc_vos=True, exact_solve=exact, robust_c=c, **sig)
            except np.linalg.LinAlgError:
                acc[name] = "a window's normal matrix was not positive definite"
                continue
            o = (r if c is None else r[0])[:, T // 2].cpu().numpy()
            acc[name] = errors(o, truth)
            acc[name]["outlier_frames"] = errors(o[out], truth[out])
            if c is not None:
                w = r[1][:, T // 2].cpu().numpy()
                acc[name]["w_median_inliers"] = round(float(np.median(w[~out])), 4)
                acc[name]["w_median_outliers"] = round(float(np.median(w[out])), 4)
    acc["no_pgo"]["outlier_frames"] = errors(pred[out], truth[out])
    # the covariance graph with fixed S7 = diag(sax I3, saq I4) (the sampled trackers' floors alone), exact step
    s7 = torch.diag(torch.tensor([sig["sax"]] * 3 + [sig["saq"]] * 4, dtype=torch.float64)).expand(
        a.frames, T, 7, 7).contiguous().cuda()
    for c in (None, 1.0, 2.0, 4.0):
        name = "%s_cov" % ("plain" if c is None else "robust_c%g" % c)
        try:
            r = optimize_pose_windows_cov(p7, s7, v7, fc_vos=True, srx=sig["srx"], srq=sig["srq"], robust_c=c)
        except np.linalg.LinAlgError:
            acc[name] = "a window's normal matrix was not positive definite"
            continue
        o = r[0][:, T // 2].cpu().numpy()
        acc[name] = errors(o, truth)
        acc[name]["outlier_frames"] = errors(o[out], truth[out])
    res["accuracy_synthetic"] = acc
    print(json.dumps(acc), file=sys.stderr)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
