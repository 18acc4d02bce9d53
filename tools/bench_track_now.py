"""Zero-lag MapNet+PGO poses on the H100: Tracker.step against a lagged Tracker call, against the zero-lag glue a user
writes by hand around a Localizer, and against evaluate_sequence(zero_lag=True) over a cached sequence.

    python tools/bench_track_now.py [--iters 200] [--rounds 5] [--frames 2000] [--out FILE]

tools/bench_track.py's workload: seeded synthetic 480x640 uint8 RGB frames, a smooth trajectory with noisy VO-library
poses, a bf16 PoseNet at droprate 0 with the running statistics of a few training-mode batches, and RobotCar's PGO
settings (pgo_inference_RobotCar.ini: steps 7, skip 10, vo_fc, sax 1, saq 1, srx 20, srq 20; lag 30 frames).  Arms,
alternating inside each of `--rounds` rounds, medians reported:
  per call at B = 1 (CUDA events), past the lag (--iters consecutive calls) and within the first lag frames of a
  sequence (the lag calls after a reset, every round starting a new sequence):
    step       Tracker.step(frame, vo): the zero-lag pose and whatever the lagged output emits; one graph replay
    call       Tracker(frame, vo): the lagged output alone; one graph replay
    glue       Localizer without pose stats, a device history of pose7 and VO pose7, the window that ends at the frame
               and its VOs rebuilt with torch ops, inference.pgo (which reads its status back: one host
               synchronisation), slot steps-1 un-normalised
  throughput   (host clock, ending in a synchronisation) --frames frames at B = 64: Tracker.step and Tracker calls in
               chunks of 64 frames then flush(), against evaluate_sequence(zero_lag=True) on a DeviceDataset of the same
               frames (its build not counted); flags say whether step's zero-lag poses are bitwise evaluate_sequence's
               and whether its lagged poses are bitwise the calls'
The card's name, power limit and clocks are read in the same run.  Prints one JSON line (and writes it to --out).  No
CPU fallback: without a GPU it exits.
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

from bench_track import FC, H_IN, MEAN, POSE_M, POSE_S, SIG, SKIP, STD, T, W_IN, Glue, host_ms   # noqa: E402


class NowGlue(Glue):
    """Glue's history and VOs, but the window that ends at the newest frame (clipped at 0) and its last slot"""

    def __call__(self, frame, vo6):
        import torch
        from geomapnet_b200.inference import pgo, post
        k = self.seen % self.R
        self.hist[k] = self.loc(frame)[0]
        self.vo[k] = post(vo6.view(1, 6))[0]
        self.seen += 1
        c = self.seen - 1 - self.lag
        idx = [max(c + (s - self.T // 2) * self.skip, 0) % self.R for s in range(self.T)]
        ix = torch.tensor(idx, device=self.hist.device)
        w, v = self.hist[ix], self.vo[ix]
        last = pgo(w[None], self._vos(v)[None], fc_vos=self.fc, **SIG)[0, self.T - 1]
        return torch.cat((last[:3] * self.s + self.m, last[3:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_track_now.json"))
    a = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_track_now: no CUDA device")
    from bench_infer import card, events_ms
    from geomapnet_b200.data import DeviceDataset, resize_output_size
    from geomapnet_b200.inference import Localizer, Predictor, Tracker, evaluate_sequence
    from geomapnet_b200.models.posenet import PoseNet
    Ho, Wo = resize_output_size(H_IN, W_IN)
    lag = (T - 1 - T // 2) * SKIP
    res = {"what": "480x640 uint8 frames + VO-library poses -> zero-lag MapNet+PGO poses (the last slot of the window "
                   "that ends at each frame), bf16 PoseNet droprate 0, RobotCar PGO settings (steps 7, skip 10, vo_fc, "
                   "sax 1, saq 1, srx 20, srq 20): per call at B = 1 Tracker.step, a lagged Tracker call and "
                   "hand-written zero-lag glue around a Localizer, past the lag and within the first lag frames; "
                   "throughput at B = 64 of step, calls and evaluate_sequence(zero_lag=True)",
           "card": card(), "frame": [H_IN, W_IN], "engine_input": [Ho, Wo], "steps": T, "skip": SKIP, "vo_fc": FC,
           "sigmas": SIG, "lag": lag, "iters": a.iters, "rounds": a.rounds, "throughput_frames": a.frames}
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
    trk_s = Tracker(loc_m, steps=T, skip=SKIP, vo_fc=FC, **SIG)
    trk_c = Tracker(loc_m, steps=T, skip=SKIP, vo_fc=FC, **SIG)
    glue = NowGlue(loc_n, T, SKIP, FC, ring=1 + (T - 1) * SKIP)
    with torch.no_grad():
        pos = {"step": 0, "call": 0, "glue": 0}
        fns = {"step": lambda f, v: trk_s.step(f, v), "call": lambda f, v: trk_c(f, v), "glue": lambda f, v: glue(f, v[0])}
        restart = {"step": trk_s.reset, "call": trk_c.reset, "glue": lambda: setattr(glue, "seen", 0)}

        def arm(name):
            def call():
                i = pos[name] % n_frames
                pos[name] += 1
                return fns[name](frames[i:i + 1], vo_dev[i:i + 1])
            return call

        arms = {k: arm(k) for k in fns}
        for fn in arms.values():                         # engine, plans, graphs; then past the lag
            for _ in range(lag + 1):
                fn()
        torch.cuda.synchronize()
        past = {k: [] for k in arms}
        warm = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                past[k].append(events_ms(fn, a.iters))
            for k, fn in arms.items():                   # a new sequence: its first lag frames
                restart[k]()
                pos[k] = 0
                warm[k].append(events_ms(fn, lag))
                for _ in range(a.iters):                 # back past the lag for the next round
                    fn()
        # a step and a call on the same frames give the same lagged poses
        trk_s.reset(); trk_c.reset()
        same = True
        for i in range(lag + 8):
            now, f1, p1 = trk_s.step(frames[i:i + 1], vo_dev[i:i + 1])
            f2, p2 = trk_c(frames[i:i + 1], vo_dev[i:i + 1])
            same = same and f1 == f2 and torch.equal(p1, p2)
        mp = {k: statistics.median(v) for k, v in past.items()}
        mw = {k: statistics.median(v) for k, v in warm.items()}
        res["per_call_b1"] = {
            "past_lag_ms": {k: round(v, 4) for k, v in mp.items()},
            "past_lag_ms_rounds": {k: [round(x, 4) for x in v] for k, v in past.items()},
            "first_lag_frames_ms": {k: round(v, 4) for k, v in mw.items()},
            "first_lag_frames_ms_rounds": {k: [round(x, 4) for x in v] for k, v in warm.items()},
            "step_minus_call_past_lag_ms": round(mp["step"] - mp["call"], 4),
            "step_minus_call_first_lag_frames_ms": round(mw["step"] - mw["call"], 4),
            "glue_over_step_past_lag": round(mp["glue"] / mp["step"], 3),
            "step_and_call_lagged_poses_bitwise": bool(same)}
        print(json.dumps(res["per_call_b1"]), file=sys.stderr)
        trk_s.close(); trk_c.close(); loc_m.close(); loc_n.close(); pr1.close()

        # ---- throughput at B = 64
        F = a.frames
        pr = Predictor(net, max_batch=64)
        loc = Localizer(pr, MEAN, STD, POSE_M, POSE_S)
        trk = Tracker(loc, steps=T, skip=SKIP, vo_fc=FC, **SIG)
        ds = DeviceDataset(frames[:F], MEAN, STD, poses=poses[:F], steps=T, skip=SKIP, vo_poses=vo[:F])
        out = {}

        def run_step():
            r = [trk.step(frames[lo:lo + 64], vo_dev[lo:lo + 64]) for lo in range(0, F, 64)]
            out["step_now"] = torch.cat([x[0] for x in r])
            out["step_lagged"] = torch.cat([x[2] for x in r] + [trk.flush()[1]])

        def run_call():
            ps = [trk(frames[lo:lo + 64], vo_dev[lo:lo + 64])[1] for lo in range(0, F, 64)]
            out["call"] = torch.cat(ps + [trk.flush()[1]])

        def run_eval():
            out["eval"] = evaluate_sequence(pr, ds, POSE_M, POSE_S, FC, zero_lag=True, **SIG)["pred7"]
        run_step(); run_call(); run_eval()
        tt = {"step": [], "call": [], "evaluate_sequence_zero_lag": []}
        for _ in range(a.rounds):
            tt["step"].append(host_ms(run_step))
            tt["call"].append(host_ms(run_call))
            tt["evaluate_sequence_zero_lag"].append(host_ms(run_eval))
        mt = {k: statistics.median(v) for k, v in tt.items()}
        res["throughput_b64"] = {
            "ms": {k: round(v, 3) for k, v in mt.items()},
            "ms_rounds": {k: [round(x, 3) for x in v] for k, v in tt.items()},
            "frames_per_s": {k: round(F / v * 1e3, 1) for k, v in mt.items()},
            "step_over_evaluate_sequence_zero_lag": round(mt["evaluate_sequence_zero_lag"] / mt["step"], 3),
            "step_zero_lag_equals_evaluate_sequence_bitwise": bool(torch.equal(out["step_now"], out["eval"])),
            "step_lagged_equals_call_bitwise": bool(torch.equal(out["step_lagged"], out["call"]))}
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
