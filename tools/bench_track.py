"""MapNet+PGO on a camera stream on the H100: inference.Tracker against the glue a user writes by hand around a
Localizer, against a Localizer call alone, and against evaluate_sequence over a cached sequence.

    python tools/bench_track.py [--iters 200] [--rounds 5] [--frames 2000] [--pgo-iters 1000] [--out FILE]

Seeded synthetic 480x640 uint8 RGB frames, a smooth trajectory with noisy VO-library poses, and a bf16 PoseNet at
droprate 0 with the running statistics of a few training-mode batches.  RobotCar's PGO settings
(pgo_inference_RobotCar.ini: steps 7, skip 10, vo_fc, sax 1, saq 1, srx 20, srq 20; lag 30 frames).  Arms, alternating
inside each of `--rounds` rounds, medians reported:
  per call at B = 1 (CUDA events over --iters consecutive calls, the stream already past its lag):
    tracker    Tracker(frame, vo)                                   one graph replay
    glue       Localizer without pose stats, a device history of pose7 and VO pose7, the window and its VOs rebuilt
               with torch ops, inference.pgo (which reads its status back: one host synchronisation), un-normalised
    localizer  Localizer(frame) alone: what PGO adds on top of localisation
  pgo_T7       one k_pgo launch on one window of 7 poses with 21 VOs (mapnet_pgo_optimize; CUDA events, --pgo-iters)
  throughput   (host clock, ending in a synchronisation) --frames frames at B = 64: the Tracker in calls of 64 frames
               and flush(), against evaluate_sequence on a DeviceDataset of the same frames (its build not counted)
Kernels per call are counted with torch.profiler (CUDA activities) over 10 calls of each per-call arm, in a pass of
their own.  The card's name, power limit and clocks are read in the same run.  Prints one JSON line (and writes it to
--out).  No CPU fallback: without a GPU it exits.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]    # 7Scenes chess stats.txt
STD = [v ** 0.5 for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
POSE_M, POSE_S = [0.5, -1.25, 2.0], [1.5, 0.75, 2.5]
H_IN, W_IN = 480, 640
T, SKIP, FC = 7, 10, True
SIG = dict(sax=1.0, saq=1.0, srx=20.0, srq=20.0)


def host_ms(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


class Glue(object):
    """MapNet+PGO written by hand around a Localizer that keeps the normalised translations"""

    def __init__(self, loc, T, skip, fc, ring):
        import torch
        self.loc, self.T, self.skip, self.R = loc, T, skip, ring
        self.lag = (T - 1 - T // 2) * skip
        self.pairs = [(i, j) for i in range(T) for j in range(i + 1, T)] if fc else [(i, i + 1) for i in range(T - 1)]
        self.fc, self.seen = fc, 0
        dev = loc.predictor.device
        self.hist = torch.zeros((ring, 7), dtype=torch.float64, device=dev)
        self.vo = torch.zeros((ring, 7), dtype=torch.float64, device=dev)
        self.m = torch.tensor(POSE_M, dtype=torch.float64, device=dev)
        self.s = torch.tensor(POSE_S, dtype=torch.float64, device=dev)

    @staticmethod
    def _qmul(a, b):
        from geomapnet_b200.common.pgo import _qmult
        return _qmult(a, b)

    def _vos(self, v7):
        import torch
        a, b = v7[[p[0] for p in self.pairs]], v7[[p[1] for p in self.pairs]]
        qa_inv = torch.cat((a[:, 3:4], -a[:, 4:]), 1)
        d = torch.cat((torch.zeros_like(a[:, :1]), b[:, :3] - a[:, :3]), 1)
        t = self._qmul(self._qmul(qa_inv, d), a[:, 3:])[:, 1:]
        q = self._qmul(qa_inv, b[:, 3:])
        q = torch.where(q[:, :1] < 0, -q, q)
        return torch.cat((t, q), 1)

    def __call__(self, frame, vo6):
        import torch
        from geomapnet_b200.inference import pgo, post
        k = self.seen % self.R
        self.hist[k] = self.loc(frame)[0]
        self.vo[k] = post(vo6.view(1, 6))[0]
        self.seen += 1
        c = self.seen - 1 - self.lag
        if c < 0:
            return None
        idx = [min(max(c + (s - self.T // 2) * self.skip, 0), self.seen - 1) % self.R for s in range(self.T)]
        ix = torch.tensor(idx, device=self.hist.device)
        w, v = self.hist[ix], self.vo[ix]
        mid = pgo(w[None], self._vos(v)[None], fc_vos=self.fc, **SIG)[0, self.T // 2]
        return torch.cat((mid[:3] * self.s + self.m, mid[3:]))


def kernels_per_call(fn, n=10):
    import torch
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    kern = [e for e in ev if not e.name.startswith("Memcpy") and not e.name.startswith("Memset")]
    return {"kernels": round(len(kern) / n, 2), "copies_and_sets": round((len(ev) - len(kern)) / n, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--pgo-iters", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_track.json"))
    a = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_track: no CUDA device")
    from bench_infer import card, events_ms
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import DeviceDataset, resize_output_size
    from geomapnet_b200.inference import Localizer, Predictor, Tracker, evaluate_sequence
    from geomapnet_b200.models.posenet import PoseNet
    L = _lib.lib()
    Ho, Wo = resize_output_size(H_IN, W_IN)
    lag = (T - 1 - T // 2) * SKIP
    res = {"what": "480x640 uint8 frames + VO-library poses -> MapNet+PGO poses, bf16 PoseNet droprate 0, RobotCar PGO "
                   "settings (steps 7, skip 10, vo_fc, sax 1, saq 1, srx 20, srq 20): per call at B = 1 the Tracker, "
                   "hand-written glue around a Localizer, and a Localizer call alone; one k_pgo launch on one T = 7 "
                   "window; throughput of the Tracker at B = 64 against evaluate_sequence",
           "card": card(), "frame": [H_IN, W_IN], "engine_input": [Ho, Wo], "steps": T, "skip": SKIP, "vo_fc": FC,
           "sigmas": SIG, "lag": lag, "iters": a.iters, "pgo_iters": a.pgo_iters, "rounds": a.rounds,
           "throughput_frames": a.frames}
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False, precision="bf16",
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
    vo = (poses + rng.standard_normal(poses.shape) * 0.02).astype(np.float32)
    vo_dev = torch.from_numpy(vo).cuda()

    # ---- per call at B = 1
    pr1 = Predictor(net, max_batch=1)
    loc_m = Localizer(pr1, MEAN, STD, POSE_M, POSE_S)
    loc_n = Localizer(pr1, MEAN, STD)
    trk = Tracker(loc_m, steps=T, skip=SKIP, vo_fc=FC, **SIG)
    glue = Glue(loc_n, T, SKIP, FC, ring=1 + (T - 1) * SKIP)
    with torch.no_grad():
        pos = {"tracker": 0, "glue": 0}

        def arm(name, fn):
            def call():
                i = pos[name] % n_frames
                pos[name] += 1
                return fn(frames[i:i + 1], vo_dev[i:i + 1])
            return call

        arms = {"tracker": arm("tracker", lambda f, v: trk(f, v)), "glue": arm("glue", lambda f, v: glue(f, v[0])),
                "localizer": lambda: loc_m(frames[:1])}
        loc_m(frames[:1])                                # the Localizer's engine, plan and graph
        _, xs, _, pred = loc_m._graph(frames[:1])
        c0 = L.mapnet_launch_count()
        loc_m._forward(pr1._engine(Ho, Wo), loc_m._plan(H_IN, W_IN), xs, pred, 0.0)
        fwd = L.mapnet_launch_count() - c0
        c0 = L.mapnet_launch_count()
        arms["tracker"]()                                # an eager forward, then the capture of forward + tracking
        launches = {"tracker": L.mapnet_launch_count() - c0 - fwd, "localizer": fwd + 1}
        for _ in range(lag + 1):                         # past the lag: every call emits a pose
            arms["tracker"](); arms["glue"]()
        torch.cuda.synchronize()
        t = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                t[k].append(events_ms(fn, a.iters))
        med = {k: statistics.median(v) for k, v in t.items()}
        res["per_call_b1"] = {"ms": {k: round(v, 4) for k, v in med.items()},
                              "ms_rounds": {k: [round(x, 4) for x in v] for k, v in t.items()},
                              "glue_over_tracker": round(med["glue"] / med["tracker"], 3),
                              "tracker_minus_localizer_ms": round(med["tracker"] - med["localizer"], 4),
                              "library_launches_per_call": launches,
                              "profiled_per_call": {k: kernels_per_call(fn) for k, fn in arms.items()}}
        print(json.dumps(res["per_call_b1"]), file=sys.stderr)

        # ---- one k_pgo launch, one window of T = 7 (the glue's last window)
        w7 = torch.randn(1, T, 7, dtype=torch.float64, device="cuda") * 0.01
        w7[..., 3] += 1.0
        v7 = torch.randn(1, T * (T - 1) // 2, 7, dtype=torch.float64, device="cuda") * 0.01
        v7[..., 3] += 1.0
        o7, st = torch.empty_like(w7), torch.zeros(1, dtype=torch.int32, device="cuda")

        def pgo_launch():
            _lib.check(L.mapnet_pgo_optimize(w7.data_ptr(), v7.data_ptr(), o7.data_ptr(), 1, T, int(FC), 1.0, 1.0,
                                             20.0, 20.0, 10, 0, st.data_ptr(), _lib.stream_ptr()), "pgo")
        for _ in range(10):
            pgo_launch()
        tp = [events_ms(pgo_launch, a.pgo_iters) for _ in range(a.rounds)]
        res["pgo_T7_one_window_ms"] = round(statistics.median(tp), 4)
        res["pgo_T7_rounds"] = [round(x, 4) for x in tp]
        trk.close(); loc_m.close(); loc_n.close(); pr1.close()

        # ---- throughput at B = 64
        F = a.frames
        pr = Predictor(net, max_batch=64)
        loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
        trk = Tracker(loc, steps=T, skip=SKIP, vo_fc=FC, **SIG)
        ds = DeviceDataset(frames[:F], MEAN, STD, poses=poses[:F], steps=T, skip=SKIP, vo_poses=vo[:F])
        out = {}

        def run_tracker():
            ps = [trk(frames[lo:lo + 64], vo_dev[lo:lo + 64])[1] for lo in range(0, F, 64)]
            out["tracker"] = torch.cat(ps + [trk.flush()[1]])

        def run_eval():
            out["eval"] = evaluate_sequence(pr, ds, POSE_M, POSE_S, FC, **SIG)["pred7"]
        run_tracker(); run_eval()
        tt = {"tracker": [], "evaluate_sequence": []}
        for _ in range(a.rounds):
            tt["tracker"].append(host_ms(run_tracker))
            tt["evaluate_sequence"].append(host_ms(run_eval))
        mt = {k: statistics.median(v) for k, v in tt.items()}
        res["throughput_b64"] = {"ms": {k: round(v, 3) for k, v in mt.items()},
                                 "ms_rounds": {k: [round(x, 3) for x in v] for k, v in tt.items()},
                                 "frames_per_s": {k: round(F / v * 1e3, 1) for k, v in mt.items()},
                                 "tracker_over_evaluate_sequence": round(mt["evaluate_sequence"] / mt["tracker"], 3),
                                 "tracker_equals_evaluate_sequence_bitwise": bool(torch.equal(out["tracker"],
                                                                                              out["eval"]))}
        print(json.dumps(res["throughput_b64"]), file=sys.stderr)
        trk.close(); loc.close(); pr.close(); ds.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
