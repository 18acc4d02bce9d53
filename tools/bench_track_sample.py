"""Monte-Carlo tracking on the H100: inference.SampledTracker against Tracker, Localizer.sample alone and the same loop
written by hand, one k_pgo_cov launch against one k_pgo launch, and throughput at B = 64.

    python tools/bench_track_sample.py [--iters 100] [--rounds 5] [--frames 2000] [--pgo-iters 1000] [--out FILE]

The frames, trajectory, VO poses and model of tools/bench_track.py, with droprate 0.5 (a bf16 PoseNet), S = 32 draws
per frame and RobotCar's PGO geometry (steps 7, skip 10, vo_fc, srx 20, srq 20; lag 30 frames) with absolute floors
sax = saq = 1e-4, below the sampled variances.  Arms, alternating inside each of `--rounds` rounds, medians reported:
  per call at B = 1 (CUDA events over --iters consecutive calls, past the lag):
    sampled    SampledTracker(frame, vo)                          one graph replay
    tracker    Tracker(frame, vo) (one draw, fixed sax / saq = 1)  one graph replay
    sample     Localizer.sample(frame, 32) alone
    glue       Localizer.sample without pose stats, a device history of p, S7 and VO pose7, the window and its VOs
               rebuilt with torch ops, optimize_pose_windows_cov (which reads its status back), D scaling
  pgo          one k_pgo_cov and one k_pgo launch (exact solve) on one T = 7 fc window (CUDA events, --pgo-iters)
  throughput   --frames frames at B = 64: SampledTracker in calls of 64 and flush() (host clock, synchronised)
Kernels per call are counted with torch.profiler in a pass of its own.  The card's name, power limit and clocks are read
in the same run.  Prints one JSON line (and writes it to --out).  No CPU fallback: without a GPU it exits.
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

from bench_track import MEAN, STD, POSE_M, POSE_S, H_IN, W_IN, T, SKIP, FC, host_ms, kernels_per_call  # noqa: E402

S = 32
SIG = dict(sax=1e-4, saq=1e-4, srx=20.0, srq=20.0)


class Glue(object):
    """the sampled tracker written by hand around Localizer.sample (normalised translations)"""

    def __init__(self, loc, ring):
        import torch
        from bench_track import Glue as G
        self.loc, self.R, self.seen = loc, ring, 0
        self.lag = (T - 1 - T // 2) * SKIP
        self._vos = G(loc, T, SKIP, FC, ring)._vos
        dev = loc.predictor.device
        f64 = dict(dtype=torch.float64, device=dev)
        self.p = torch.zeros((ring, 7), **f64)
        self.c = torch.zeros((ring, 7, 7), **f64)
        self.vo = torch.zeros((ring, 7), **f64)
        self.d = torch.tensor(POSE_S + [1.0] * 3, **f64)
        self.m = torch.tensor(POSE_M, **f64)
        self.floor = torch.diag(torch.tensor([SIG["sax"]] * 3 + [SIG["saq"]] * 4, **f64))

    def _s7(self, q, cov):
        import torch
        u = q[1:]
        s = torch.linalg.norm(u)
        v = torch.atan2(s, q[0]) * u / s                 # the mean log q
        n = torch.linalg.norm(v)
        sc, g = torch.sin(n) / n, (n * torch.cos(n) - torch.sin(n)) / n ** 3
        A = torch.zeros((7, 6), dtype=cov.dtype, device=cov.device)
        A[:3, :3] = torch.eye(3, dtype=cov.dtype, device=cov.device)
        A[3, 3:] = -sc * v
        A[4:, 3:] = sc * torch.eye(3, dtype=cov.dtype, device=cov.device) + g * torch.outer(v, v)
        return A @ cov @ A.T + self.floor

    def __call__(self, frame, vo6):
        import torch
        from geomapnet_b200.common.pgo import optimize_pose_windows_cov
        from geomapnet_b200.inference import post
        out = self.loc.sample(frame, S)
        k = self.seen % self.R
        self.p[k] = out["pose7"][0]
        self.c[k] = self._s7(out["pose7"][0, 3:], out["cov"][0])
        self.vo[k] = post(vo6[None])[0]
        self.seen += 1
        c = self.seen - 1 - self.lag
        if c < 0:
            return None
        idx = [min(max(c + (j - T // 2) * SKIP, 0), self.seen - 1) % self.R for j in range(T)]
        z, cv = optimize_pose_windows_cov(self.p[idx][None], self.c[idx][None], self._vos(self.vo[idx])[None], FC,
                                          SIG["srx"], SIG["srq"])
        z, cv = z[0, T // 2], cv[0, T // 2]
        return torch.cat((z[:3] * self.d[:3] + self.m, z[3:])), self.d[:, None] * cv * self.d[None, :]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--pgo-iters", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_track_sample.json"))
    a = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_track_sample: no CUDA device")
    from bench_infer import card, events_ms
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import resize_output_size
    from geomapnet_b200.inference import Localizer, Predictor, SampledTracker, Tracker
    from geomapnet_b200.models.posenet import PoseNet
    L = _lib.lib()
    Ho, Wo = resize_output_size(H_IN, W_IN)
    lag = (T - 1 - T // 2) * SKIP
    res = {"what": "480x640 uint8 frames + VO-library poses -> Monte-Carlo MapNet+PGO poses and covariances, bf16 "
                   "PoseNet droprate 0.5, S = 32, RobotCar PGO geometry (steps 7, skip 10, vo_fc, srx 20, srq 20) with "
                   "sax = saq = 1e-4: per call at B = 1 SampledTracker, Tracker (sax = saq = 1), Localizer.sample alone "
                   "and the loop written by hand; one k_pgo_cov against one k_pgo launch on a T = 7 fc window; "
                   "SampledTracker throughput at B = 64",
           "card": card(), "frame": [H_IN, W_IN], "engine_input": [Ho, Wo], "steps": T, "skip": SKIP, "vo_fc": FC,
           "S": S, "droprate": 0.5, "sigmas": SIG, "lag": lag, "iters": a.iters, "pgo_iters": a.pgo_iters,
           "rounds": a.rounds, "throughput_frames": a.frames}
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False, precision="bf16",
                  seed=7).cuda()
    with torch.no_grad():
        net.train()
        for _ in range(3):
            net(torch.randn(16, 3, Ho, Wo, device="cuda"))
    net.eval()
    n_frames = max(a.frames, a.iters + lag + 64)
    g = torch.Generator(device="cuda").manual_seed(11)
    frames = torch.randint(0, 256, (n_frames, H_IN, W_IN, 3), dtype=torch.uint8, device="cuda", generator=g)
    rng = np.random.default_rng(3)
    s = np.arange(n_frames)[:, None] / 50.0
    poses = np.concatenate([np.sin(s), np.cos(0.7 * s), 0.1 * s, 0.2 * np.sin(0.3 * s), 0.1 * np.cos(0.5 * s),
                            0.05 * s], 1).astype(np.float32)
    vo_dev = torch.from_numpy((poses + rng.standard_normal(poses.shape) * 0.02).astype(np.float32)).cuda()

    with torch.no_grad():
        # ---- per call at B = 1
        pr1 = Predictor(net, max_batch=1)
        loc_m = Localizer(pr1, MEAN, STD, POSE_M, POSE_S)
        loc_n = Localizer(pr1, MEAN, STD)
        st = SampledTracker(loc_m, S, steps=T, skip=SKIP, vo_fc=FC, **SIG)
        trk = Tracker(loc_m, steps=T, skip=SKIP, vo_fc=FC, sax=1.0, saq=1.0, srx=SIG["srx"], srq=SIG["srq"])
        glue = Glue(loc_n, 1 + (T - 1) * SKIP)
        pos = {"sampled": 0, "tracker": 0, "glue": 0}

        def arm(name, fn):
            def call():
                i = pos[name] % n_frames
                pos[name] += 1
                return fn(frames[i:i + 1], vo_dev[i:i + 1])
            return call

        arms = {"sampled": arm("sampled", lambda f, v: st(f, v)), "tracker": arm("tracker", lambda f, v: trk(f, v)),
                "sample": lambda: loc_m.sample(frames[:1], S), "glue": arm("glue", lambda f, v: glue(f, v[0]))}
        loc_m.sample(frames[:1], S)
        c0 = L.mapnet_launch_count()
        arms["sampled"]()                                # eager sampled engine, then its capture + 3 tracking launches
        launches = {"sampled_first_call": L.mapnet_launch_count() - c0}
        for _ in range(lag + 1):                         # past the lag: every call emits a pose
            for k in ("sampled", "tracker", "glue"):
                arms[k]()
        c0 = L.mapnet_launch_count()
        arms["sampled"]()
        launches["sampled_replayed_call"] = L.mapnet_launch_count() - c0
        torch.cuda.synchronize()
        t = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                t[k].append(events_ms(fn, a.iters))
        med = {k: statistics.median(v) for k, v in t.items()}
        res["per_call_b1"] = {"ms": {k: round(v, 4) for k, v in med.items()},
                              "ms_rounds": {k: [round(x, 4) for x in v] for k, v in t.items()},
                              "glue_over_sampled": round(med["glue"] / med["sampled"], 3),
                              "sampled_minus_sample_ms": round(med["sampled"] - med["sample"], 4),
                              "library_launches": launches,
                              "profiled_per_call": {k: kernels_per_call(fn) for k, fn in arms.items()}}
        print(json.dumps(res["per_call_b1"]), file=sys.stderr)

        # ---- one k_pgo_cov and one k_pgo launch, one window of T = 7 with its 21 VOs
        w7 = torch.randn(1, T, 7, dtype=torch.float64, device="cuda") * 0.01
        w7[..., 3] += 1.0
        v7 = torch.randn(1, T * (T - 1) // 2, 7, dtype=torch.float64, device="cuda") * 0.01
        v7[..., 3] += 1.0
        c7 = torch.diag(torch.tensor([1e-2] * 3 + [1e-3] * 4, dtype=torch.float64)).expand(1, T, 7, 7).contiguous().cuda()
        o7, oc = torch.empty_like(w7), torch.empty((1, T, 6, 6), dtype=torch.float64, device="cuda")
        stat = torch.zeros(1, dtype=torch.int32, device="cuda")

        def pgo_cov():
            _lib.check(L.mapnet_pgo_optimize_cov(w7.data_ptr(), c7.data_ptr(), v7.data_ptr(), o7.data_ptr(),
                                                 oc.data_ptr(), 1, T, int(FC), 20.0, 20.0, 10, stat.data_ptr(),
                                                 _lib.stream_ptr()), "pgo_cov")

        def pgo():
            _lib.check(L.mapnet_pgo_optimize(w7.data_ptr(), v7.data_ptr(), o7.data_ptr(), 1, T, int(FC), 1e-2, 1e-3,
                                             20.0, 20.0, 10, 1, stat.data_ptr(), _lib.stream_ptr()), "pgo")
        for _ in range(10):
            pgo_cov(); pgo()
        tp = {"k_pgo_cov": [], "k_pgo": []}
        for _ in range(a.rounds):
            tp["k_pgo_cov"].append(events_ms(pgo_cov, a.pgo_iters))
            tp["k_pgo"].append(events_ms(pgo, a.pgo_iters))
        res["pgo_T7_one_window_ms"] = {k: round(statistics.median(v), 4) for k, v in tp.items()}
        res["pgo_T7_rounds"] = {k: [round(x, 4) for x in v] for k, v in tp.items()}
        print(json.dumps(res["pgo_T7_one_window_ms"]), file=sys.stderr)
        st.close(); trk.close(); loc_m.close(); loc_n.close(); pr1.close()

        # ---- throughput at B = 64
        F = a.frames
        pr = Predictor(net, max_batch=64)
        loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
        st = SampledTracker(loc, S, steps=T, skip=SKIP, vo_fc=FC, **SIG)

        def run():
            for lo in range(0, F, 64):
                st(frames[lo:lo + 64], vo_dev[lo:lo + 64])
            st.flush()
        run()
        tt = [host_ms(run) for _ in range(a.rounds)]
        m = statistics.median(tt)
        res["throughput_b64"] = {"ms": round(m, 3), "ms_rounds": [round(x, 3) for x in tt],
                                 "frames_per_s": round(F / m * 1e3, 1)}
        print(json.dumps(res["throughput_b64"]), file=sys.stderr)
        st.close(); loc.close(); pr.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
