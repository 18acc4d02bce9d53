"""Monte-Carlo evaluation of a labelled sequence on the H100: inference.evaluate_sequence(samples=32) against a
SampledTracker over the same frames, the same loop written by hand, and evaluate_sequence without samples.

    python tools/bench_eval_sample.py [--frames 2000] [--rounds 5] [--out FILE]

Workload: --frames synthetic 480x640 uint8 frames in a DeviceDataset (cached at Resize(256)), a smooth trajectory as
the targets and noisy VO-library poses, a bf16 MapNet at droprate 0.5, S = 32 draws per frame, RobotCar's PGO
geometry (steps 7, skip 10, vo_fc, srx = srq = 20) with sax = saq = 1e-4.  Arms, alternating inside each of --rounds
rounds, medians reported (host clock around a synchronised whole sequence):
  eval_sample  evaluate_sequence(samples=32): Predictor(max_batch=64), all windows, covariances and calibration scores
  tracker      SampledTracker at B = 64 over the same frames (uint8 on the device) and VO poses, flush included
  hand         Predictor.sample per chunk of 64 (ImagePipeline inputs, prepared once outside the timing), the windows
               in numpy, the factors and VOs with torch ops,
               optimize_pose_windows_cov (which reads its status back), the calibration scores in torch
  eval_point   evaluate_sequence without samples on the same model (one window per forward: eval.py's dropout loop)
The first two arms use twin Predictors (same model, seed and call sequence), and whether their poses are bitwise equal
is recorded every round.  The card's name, power limit and clocks are read in the same run.  Prints one JSON line (and
writes it to --out).  No CPU fallback: without a GPU it exits.
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

from bench_track import MEAN, STD, POSE_M, POSE_S, H_IN, W_IN, T, SKIP, FC, host_ms  # noqa: E402

S = 32
B = 64
SIG = dict(sax=1e-4, saq=1e-4, srx=20.0, srq=20.0)


def _qexp(v):
    import torch
    n = torch.linalg.norm(v, dim=-1, keepdim=True)
    return torch.cat((torch.cos(n), torch.where(n > 0, torch.sin(n) / n, torch.ones_like(n)) * v), -1)


def _qlog(q):
    import torch
    u = q[..., 1:]
    s = torch.linalg.norm(u, dim=-1, keepdim=True)
    a = torch.acos(q[..., :1].clamp(-1.0, 1.0))
    return torch.where(s > 0, a * u / s, torch.zeros_like(u))


def _qmul(a, b):
    import torch
    w = a[..., 0] * b[..., 0] - (a[..., 1:] * b[..., 1:]).sum(-1)
    v = a[..., :1] * b[..., 1:] + b[..., :1] * a[..., 1:] + torch.linalg.cross(a[..., 1:], b[..., 1:])
    return torch.cat((w[..., None], v), -1)


def _rotate(t, q):
    import torch
    b = torch.linalg.cross(q[..., 1:], t)
    return t + 2 * q[..., :1] * b + 2 * torch.linalg.cross(q[..., 1:], b)


def hand(pr, x, vo6, targ6, pairs, dev):
    """the sampled evaluation written by hand around Predictor.sample: returns (pose7 [L,7], cov [L,6,6], u [L,3])"""
    import numpy as np
    import torch
    from geomapnet_b200.common.pgo import optimize_pose_windows_cov
    f64 = dict(dtype=torch.float64, device=dev)
    n = x.shape[0]                                        # eval.py's windows, clipped at the sequence's ends
    windows = np.clip(np.arange(n)[:, None] + (np.arange(T) - T // 2)[None] * SKIP, 0, n - 1)
    mean, cov = [], []
    for lo in range(0, x.shape[0], B):
        o = pr.sample(x[lo:lo + B], S)
        mean.append(o["mean"]); cov.append(o["cov"])
    mean, cov = torch.cat(mean), torch.cat(cov)
    w = torch.from_numpy(windows).to(dev).long()
    v = mean[:, 3:]                                       # the factors: p = (mu_t, qexp(mu_v)), S7 = A Sigma A' + floors
    n = torch.linalg.norm(v, dim=-1)[:, None, None]
    sc, g = torch.sin(n) / n, (n * torch.cos(n) - torch.sin(n)) / n ** 3
    A = torch.zeros((mean.shape[0], 7, 6), **f64)
    A[:, :3, :3] = torch.eye(3, **f64)
    A[:, 3, 3:] = -sc[:, 0] * v
    A[:, 4:, 3:] = sc * torch.eye(3, **f64) + g * v[:, :, None] * v[:, None, :]
    floor = torch.diag(torch.tensor([SIG["sax"]] * 3 + [SIG["saq"]] * 4, **f64))
    S7 = A @ cov @ A.transpose(1, 2) + floor
    p7 = torch.cat((mean[:, :3], _qexp(v)), -1)
    vp = vo6.double()                                     # the VOs: calc_vos_safe(_fc) of the VO-library poses
    i, j = w[:, pairs[:, 0]], w[:, pairs[:, 1]]
    qi, qj = _qexp(vp[i, 3:]), _qexp(vp[j, 3:])
    qinv = torch.cat((qi[..., :1], -qi[..., 1:]), -1)
    q = _qmul(qinv, qj)
    q = q / torch.linalg.norm(q, dim=-1, keepdim=True)
    vos7 = torch.cat((_rotate(vp[j, :3] - vp[i, :3], qinv), _qexp(_qlog(q))), -1)
    z, cv = optimize_pose_windows_cov(p7[w], S7[w], vos7, fc_vos=FC, srx=SIG["srx"], srq=SIG["srq"])
    d = torch.tensor(POSE_S + [1.0] * 3, **f64)
    z, cv = z[:, T // 2], d[:, None] * cv[:, T // 2] * d[None, :]
    pose7 = torch.cat((z[:, :3] * d[:3] + torch.tensor(POSE_M, **f64), z[:, 3:]), -1)
    tg = targ6[w[:, T // 2]].double()                     # the calibration scores
    targ7 = torch.cat((tg[:, :3] * d[:3] + torch.tensor(POSE_M, **f64), _qexp(tg[:, 3:])), -1)
    sg = torch.where((pose7[:, 3:] * targ7[:, 3:]).sum(-1, keepdim=True) < 0, -1.0, 1.0)
    e = torch.cat((pose7[:, :3] - targ7[:, :3], _qlog(pose7[:, 3:]) - _qlog(sg * targ7[:, 3:])), -1)

    def d2(C, x):
        Lc, _ = torch.linalg.cholesky_ex(C)
        y = torch.linalg.solve_triangular(Lc, x[..., None], upper=False)
        return (y[..., 0] ** 2).sum(-1)
    d6, dt, dq = d2(cv, e), d2(cv[:, :3, :3], e[:, :3]), d2(cv[:, 3:, 3:], e[:, 3:])
    f3 = lambda x: torch.erf(torch.sqrt(0.5 * x)) - torch.sqrt(2 * x / math.pi) * torch.exp(-0.5 * x)
    u = torch.stack((1 - torch.exp(-0.5 * d6) * (1 + 0.5 * d6 + 0.125 * d6 ** 2), f3(dt), f3(dq)), -1)
    return pose7, cv, u


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_eval_sample.json"))
    a = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_eval_sample: no CUDA device")
    from bench_infer import card
    from geomapnet_b200.data import DeviceDataset, ImagePipeline
    from geomapnet_b200.inference import Localizer, Predictor, SampledTracker, evaluate_sequence
    from geomapnet_b200.models.posenet import MapNet, PoseNet
    F = a.frames
    res = {"what": "Monte-Carlo evaluation of a labelled sequence: %d synthetic 480x640 frames, bf16 MapNet droprate "
                   "0.5, S = 32, RobotCar PGO geometry (steps 7, skip 10, vo_fc, srx 20, srq 20) with sax = saq = "
                   "1e-4; evaluate_sequence(samples=32) against SampledTracker at B = 64 (flush included), the loop "
                   "written by hand and evaluate_sequence without samples; host clock per synchronised sequence" % F,
           "card": card(), "frames": F, "frame": [H_IN, W_IN], "steps": T, "skip": SKIP, "vo_fc": FC, "S": S,
           "max_batch": B, "droprate": 0.5, "sigmas": SIG, "rounds": a.rounds}
    torch.manual_seed(7)
    model = MapNet(PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False,
                           precision="bf16", seed=7)).cuda()
    rng = np.random.default_rng(3)
    fr = rng.integers(0, 256, (F, H_IN, W_IN, 3), dtype=np.uint8)
    s = np.arange(F)[:, None] / 50.0
    poses = np.concatenate([np.sin(s), np.cos(0.7 * s), 0.1 * s, 0.2 * np.sin(0.3 * s), 0.1 * np.cos(0.5 * s),
                            0.05 * s], 1).astype(np.float32)
    vo = (poses + rng.standard_normal(poses.shape) * 0.02).astype(np.float32)
    ds = DeviceDataset(fr, MEAN, STD, poses=poses, steps=T, skip=SKIP, vo_poses=vo)
    frames = torch.from_numpy(fr).cuda()
    del fr
    vo_dev, targ_dev = torch.from_numpy(vo).cuda(), torch.from_numpy(poses).cuda()
    pairs = np.array([(i, j) for i in range(T) for j in range(i + 1, T)] if FC else [(i, i + 1) for i in range(T - 1)])
    x = ImagePipeline(MEAN, STD)(frames)                  # the hand-written arm's engine inputs, prepared once

    with torch.no_grad():
        pa, pb, ph, pp = (Predictor(model, max_batch=B) for _ in range(4))
        for p in (pa, pb, ph, pp):
            p.seed = 20261018
        loc = Localizer(pb, MEAN, STD, POSE_M, POSE_S)
        st = SampledTracker(loc, S, steps=T, skip=SKIP, vo_fc=FC, **SIG)
        out = {}

        def eval_sample():
            out["eval"] = evaluate_sequence(pa, ds, POSE_M, POSE_S, FC, samples=S, **SIG)

        def tracker():
            ests = []
            for lo in range(0, F, B):
                ests.append(st(frames[lo:lo + B], vo_dev[lo:lo + B])[1])
            ests.append(st.flush()[1])
            out["tracker"] = torch.cat([e["pose7"] for e in ests])

        def hand_arm():
            out["hand"] = hand(ph, x, vo_dev, targ_dev, pairs, ph.device)

        def eval_point():
            out["point"] = evaluate_sequence(pp, ds, POSE_M, POSE_S, FC, **SIG)

        arms = {"eval_sample": eval_sample, "tracker": tracker, "hand": hand_arm, "eval_point": eval_point}
        for fn in arms.values():                          # warm-up: graphs, plans, the pipeline's slots
            fn()
        t = {k: [] for k in arms}
        equal = []
        for _ in range(a.rounds):
            for k, fn in arms.items():
                t[k].append(host_ms(fn))
            equal.append(bool(torch.equal(out["eval"]["pred7"], out["tracker"])))
        med = {k: statistics.median(v) for k, v in t.items()}
        ev = out["eval"]
        hp, hc, hu = out["hand"]
        res["ms"] = {k: round(v, 2) for k, v in med.items()}
        res["ms_rounds"] = {k: [round(v, 2) for v in vs] for k, vs in t.items()}
        res["frames_per_s"] = {k: round(F / v * 1e3, 1) for k, v in med.items()}
        res["hand_over_eval_sample"] = round(med["hand"] / med["eval_sample"], 3)
        res["tracker_over_eval_sample"] = round(med["tracker"] / med["eval_sample"], 3)
        res["eval_sample_poses_bitwise_tracker"] = equal
        res["hand_vs_eval_sample_max_rel"] = {
            "pose7": float((hp - ev["pred7"]).abs().max() / ev["pred7"].abs().max()),
            "cov": float((hc - ev["cov"]).abs().max() / ev["cov"].abs().max()),
            "u": float((hu - ev["u"]).abs().max())}
        res["coverage_of_this_synthetic_run"] = {str(p): [round(float(v), 4) for v in (ev["u"] <= p).double().mean(0)]
                                                 for p in (0.5, 0.9, 0.95, 0.99)}
        st.close(); loc.close()
        for p in (pa, pb, ph, pp):
            p.close()
    ds.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
