"""Many camera streams with Monte-Carlo dropout on the H100: one SampledMultiTracker call per tick against K
SampledTrackers called once each per tick.

    python tools/bench_track_multi_sample.py [--rounds 5] [--streams 1,8,64] [--out FILE]

tools/bench_track_multi.py's workload with tools/bench_track_sample.py's sampling: seeded synthetic 480x640 uint8 RGB
frames, smooth trajectories with noisy VO-library poses, a bf16 PoseNet at droprate 0.5 with the running statistics of
a few training-mode batches, S = 32 draws per frame, and RobotCar's PGO geometry (steps 7, skip 10, vo_fc, srx 20,
srq 20; lag 30 frames) with absolute floors sax = saq = 1e-4.  Each of K streams brings one frame per tick.  Arms, per
K, alternating inside each of `--rounds` rounds, medians reported:
    multi_call     SampledMultiTracker(frames [K], vo [K], streams 0 .. K-1): one graph replay (a sampled engine batch
                   of K frames, one k_pgo_cov launch of K windows)
    multi_step     SampledMultiTracker.step of the same: zero-lag estimates as well
    trackers_call  K SampledTrackers, each called with its stream's frame: K graph replays at B = 1
The SampledMultiTracker runs a Predictor of max_batch 64, the SampledTrackers one of max_batch 1 (what a one-camera
deployment runs), both snapshots of the same network.  Every arm is past the lag on every stream before it is timed; a
measurement is CUDA events around `iters` consecutive ticks (max(20, 256 // K)).  Library launches per call are counted
with mapnet_launch_count (the capture of a new shape, and a replay).  After timing, a fresh sequence of lag + 16 ticks
checks that the SampledMultiTracker's lagged (with flushes) and zero-lag estimates are bit for bit those of K
mapnet_track_sample_t handles fed each stream's per-frame draw statistics (the mean and covariance the tick's sampled
engine wrote, read from the graph's buffers).  The card's name, power limit and clocks are read in the same run.
Prints one JSON line (and writes it to --out).  No CPU fallback: without a GPU it exits.
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_track import FC, H_IN, MEAN, POSE_M, POSE_S, SKIP, STD, T, W_IN   # noqa: E402
from bench_track_sample import S, SIG                                      # noqa: E402


class Composition(object):
    """K mapnet_track_sample_t handles of the tracker's arguments, fed one stream's draw statistics each"""

    def __init__(self, K):
        from geomapnet_b200 import _lib
        self.L, self.hs = _lib.lib(), []
        sig = (ctypes.c_double * 4)(SIG["sax"], SIG["saq"], SIG["srx"], SIG["srq"])
        m3, s3 = (ctypes.c_double * 3)(*POSE_M), (ctypes.c_double * 3)(*POSE_S)
        for _ in range(K):
            h = ctypes.c_void_p()
            _lib.check(self.L.mapnet_track_sample_create(ctypes.byref(h), T, SKIP, int(FC), 1, sig, m3, s3),
                       "mapnet_track_sample_create")
            self.hs.append(h)

    def step(self, k, mean, cov, vo, now):
        """stream k's frame: (rows [n,45], now row [1,45] or None)"""
        import torch
        from geomapnet_b200 import _lib
        out = torch.empty((1, _lib.TRACK_SAMPLE_ROW), dtype=torch.float64, device="cuda")
        nw = torch.empty_like(out)
        if now:
            _lib.check(self.L.mapnet_track_sample_step_now(self.hs[k], mean.data_ptr(), cov.data_ptr(), vo.data_ptr(),
                                                           1, out.data_ptr(), nw.data_ptr(), _lib.stream_ptr()),
                       "mapnet_track_sample_step_now")
        else:
            _lib.check(self.L.mapnet_track_sample_step(self.hs[k], mean.data_ptr(), cov.data_ptr(), vo.data_ptr(), 1,
                                                       out.data_ptr(), _lib.stream_ptr()), "mapnet_track_sample_step")
        return out, (nw if now else None)

    def flush(self, k, lag, seen):
        import torch
        from geomapnet_b200 import _lib
        out = torch.empty((lag, _lib.TRACK_SAMPLE_ROW), dtype=torch.float64, device="cuda")
        _lib.check(self.L.mapnet_track_sample_flush(self.hs[k], out.data_ptr(), _lib.stream_ptr()), "flush")
        _lib.check(self.L.mapnet_track_sample_reset(self.hs[k], _lib.stream_ptr()), "reset")
        return out[:min(lag, seen)]

    def close(self):
        import torch
        torch.cuda.synchronize()
        for h in self.hs:
            self.L.mapnet_track_sample_destroy(h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--streams", default="1,8,64")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_track_multi_sample.json"))
    a = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_track_multi_sample: no CUDA device")
    from bench_infer import card, events_ms
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import resize_output_size
    from geomapnet_b200.inference import Localizer, Predictor, SampledMultiTracker, SampledTracker
    from geomapnet_b200.models.posenet import PoseNet
    Ho, Wo = resize_output_size(H_IN, W_IN)
    lag = (T - 1 - T // 2) * SKIP
    Ks = [int(k) for k in a.streams.split(",")]
    res = {"what": "K camera streams of 480x640 uint8 frames + VO-library poses, one frame per stream per tick -> "
                   "Monte-Carlo MapNet+PGO poses and covariances, bf16 PoseNet droprate 0.5, S = 32, RobotCar PGO "
                   "geometry (steps 7, skip 10, vo_fc, srx 20, srq 20) with sax = saq = 1e-4: one SampledMultiTracker "
                   "call per tick (Predictor max_batch 64) against K SampledTrackers called once each (Predictor "
                   "max_batch 1), and SampledMultiTracker.step, past the lag",
           "card": card(), "frame": [H_IN, W_IN], "engine_input": [Ho, Wo], "steps": T, "skip": SKIP, "vo_fc": FC,
           "S": S, "droprate": 0.5, "sigmas": SIG, "lag": lag, "rounds": a.rounds, "streams": Ks, "per_k": {}}
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False, precision="bf16",
                  seed=7).cuda()
    with torch.no_grad():
        net.train()
        for _ in range(3):
            net(torch.randn(16, 3, Ho, Wo, device="cuda"))
    net.eval()
    n_pool = 512
    g = torch.Generator(device="cuda").manual_seed(11)
    frames = torch.randint(0, 256, (n_pool, H_IN, W_IN, 3), dtype=torch.uint8, device="cuda", generator=g)
    rng = np.random.default_rng(3)
    s = np.arange(n_pool)[:, None] / 50.0
    poses = np.concatenate([np.sin(s), np.cos(0.7 * s), 0.1 * s, 0.2 * np.sin(0.3 * s), 0.1 * np.cos(0.5 * s),
                            0.05 * s], 1).astype(np.float32)
    vo_dev = torch.from_numpy((poses + rng.standard_normal(poses.shape) * 0.02).astype(np.float32)).cuda()
    L = _lib.lib()
    pr64, pr1 = Predictor(net, max_batch=64), Predictor(net, max_batch=1)
    loc64 = Localizer(pr64, MEAN, STD, POSE_M, POSE_S)
    loc1 = Localizer(pr1, MEAN, STD, POSE_M, POSE_S)

    def tick_ids(K, t):
        """the pool frame of each stream at tick t: stream k walks the pool from its own offset"""
        return (np.arange(K) * 37 + t) % n_pool

    with torch.no_grad():
        for K in Ks:
            iters = max(20, 256 // K)
            mts = {"call": SampledMultiTracker(loc64, S, K, steps=T, skip=SKIP, vo_fc=FC, **SIG),
                   "step": SampledMultiTracker(loc64, S, K, steps=T, skip=SKIP, vo_fc=FC, **SIG)}
            trks = [SampledTracker(loc1, S, steps=T, skip=SKIP, vo_fc=FC, **SIG) for _ in range(K)]
            ids_k = torch.arange(K)
            pool_ix = [torch.from_numpy(tick_ids(K, t)).cuda() for t in range(n_pool)]
            pos = {}

            def arm(name, mode):
                pos[name] = 0

                def call():
                    ix = pool_ix[pos[name] % n_pool]
                    pos[name] += 1
                    f, v = frames[ix], vo_dev[ix]
                    if mode == "call":
                        return mts["call"](f, v, ids_k)
                    if mode == "step":
                        return mts["step"].step(f, v, ids_k)
                    for k, trk in enumerate(trks):
                        trk(f[k:k + 1], v[k:k + 1])
                return call

            arms = {"multi_call": arm("multi_call", "call"), "multi_step": arm("multi_step", "step"),
                    "trackers_call": arm("trackers_call", "trackers")}
            loc64.sample(frames[:K], S); loc1.sample(frames[:1], S)      # the engines and plans
            torch.cuda.synchronize()
            launches = {}
            for name, fn in arms.items():                 # the first call captures; then past the lag
                c0 = L.mapnet_launch_count()
                fn()
                first = L.mapnet_launch_count() - c0
                c0 = L.mapnet_launch_count()
                fn()
                launches[name] = {"first_call": first, "replayed_call": L.mapnet_launch_count() - c0}
                for _ in range(lag):
                    fn()
            torch.cuda.synchronize()
            tt = {k: [] for k in arms}
            for _ in range(a.rounds):
                for name, fn in arms.items():
                    tt[name].append(events_ms(fn, iters))
            med = {k: statistics.median(v) for k, v in tt.items()}

            # bitwise: a fresh sequence of lag + 16 ticks on every stream against K single-stream handles fed the
            # draw statistics each tick's sampled engine wrote
            V = lag + 16
            same = True
            for mode in ("call", "step"):
                mt = mts[mode]
                mt.reset()
                comp = Composition(K)
                got = {k: [] for k in range(K)}
                want = {k: [] for k in range(K)}
                for t in range(V):
                    ix = torch.from_numpy(tick_ids(K, t)).cuda()
                    f, v = frames[ix], vo_dev[ix]
                    if mode == "call":
                        sid, fid, est = mt(f, v, ids_k)
                    else:
                        now, sid, fid, est = mt.step(f, v, ids_k)
                    mean, cov = (x.clone() for x in mt._graph(f, mode == "step")[5][1:])
                    for r in range(sid.shape[0]):
                        got[int(sid[r])].append(est["pose7"][r:r + 1])
                        got[int(sid[r])].append(est["cov"][r:r + 1].reshape(1, 36))
                    for k in range(K):
                        rows, nw = comp.step(k, mean[k:k + 1], cov[k:k + 1], v[k:k + 1], mode == "step")
                        if rows.shape[0] and t >= lag:
                            want[k].append(rows[:, :7])
                            want[k].append(rows[:, 7:43])
                        if mode == "step":
                            same = same and torch.equal(torch.cat((now["pose7"][k], now["cov"][k].reshape(36),
                                                                   now["t_std"][k:k + 1], now["q_std_deg"][k:k + 1])),
                                                        nw[0])
                for k in range(K):
                    first, est = mt.flush(k)
                    rows = comp.flush(k, lag, V)
                    got[k] += [est["pose7"], est["cov"].reshape(-1, 36)]
                    want[k] += [rows[:, :7], rows[:, 7:43]]
                comp.close()
                same = same and all(torch.equal(torch.cat([x.reshape(-1) for x in got[k]]),
                                                torch.cat([x.reshape(-1) for x in want[k]])) for k in range(K))
            res["per_k"][str(K)] = {
                "iters": iters,
                "ms_per_tick": {k: round(v, 4) for k, v in med.items()},
                "ms_per_tick_rounds": {k: [round(x, 4) for x in v] for k, v in tt.items()},
                "frames_per_s": {k: round(K / v * 1e3, 1) for k, v in med.items()},
                "trackers_over_multi": round(med["trackers_call"] / med["multi_call"], 2),
                "step_over_call": round(med["multi_step"] / med["multi_call"], 3),
                "library_launches": launches,
                "multi_equals_composition_bitwise": bool(same)}
            print(json.dumps({K: res["per_k"][str(K)]["ms_per_tick"], "bitwise": bool(same)}), file=sys.stderr)
            for mt in mts.values():
                mt.close()
            for trk in trks:
                trk.close()
    loc64.close(); loc1.close(); pr64.close(); pr1.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
