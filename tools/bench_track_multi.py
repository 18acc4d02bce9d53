"""Many camera streams on the H100: one MultiTracker call per tick against K Trackers called once each per tick.

    python tools/bench_track_multi.py [--rounds 5] [--streams 1,8,64] [--out FILE]

tools/bench_track.py's workload: seeded synthetic 480x640 uint8 RGB frames, smooth trajectories with noisy VO-library
poses, a bf16 PoseNet at droprate 0 with the running statistics of a few training-mode batches, and RobotCar's PGO
settings (pgo_inference_RobotCar.ini: steps 7, skip 10, vo_fc, sax 1, saq 1, srx 20, srq 20; lag 30 frames).  Each of
K streams brings one frame per tick.  Arms, per K, alternating inside each of `--rounds` rounds, medians reported:
    multi_call     MultiTracker(frames [K], vo [K], streams 0 .. K-1): one graph replay (engine batch of K frames)
    multi_step     MultiTracker.step of the same: zero-lag poses as well
    trackers_call  K Trackers, each called with its stream's frame: K graph replays at B = 1
    trackers_step  K Trackers' step
The MultiTracker runs a Predictor of max_batch 64, the Trackers one of max_batch 1 (what a one-camera deployment
runs), both snapshots of the same network.  Every arm is past the lag on every stream before it is timed; a
measurement is CUDA events around `iters` consecutive ticks (max(20, 256 // K)).  Library launches per call are counted
with mapnet_launch_count (the capture of a new shape, and a replay).  After timing, a fresh sequence of lag + 16 ticks
checks that MultiTracker's lagged (with flushes) and zero-lag poses are bit for bit the per-stream composition of the
same Predictor calls with mapnet_eval_windows, pgo and the un-normalisation.  The card's name, power limit and clocks
are read in the same run.  Prints one JSON line (and writes it to --out).  No CPU fallback: without a GPU it exits.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_track import FC, H_IN, MEAN, POSE_M, POSE_S, SIG, SKIP, STD, T, W_IN   # noqa: E402


def composition(pr, frames, vo, ids_per_tick, K, zero_lag):
    """per stream: Predictor(ImagePipeline(tick frames)) split by stream, eval.py's windows (mapnet_eval_windows),
    pgo, the middle (zero-lag: last) slot, un-normalised"""
    import numpy as np
    import torch
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.inference import pgo
    pipe = ImagePipeline(MEAN, STD)
    pred = torch.stack([pr(pipe(frames[ix])) for ix in ids_per_tick], 1)       # [K, ticks, 6]
    vos = np.stack([vo[ix] for ix in ids_per_tick], 1)
    lag = (T - 1 - T // 2) * SKIP
    m = torch.as_tensor(np.asarray(POSE_M, dtype=np.float64), device="cuda")
    s = torch.as_tensor(np.asarray(POSE_S, dtype=np.float64), device="cuda")
    pairs = [(i, j) for i in range(T) for j in range(i + 1, T)] if FC else [(i, i + 1) for i in range(T - 1)]
    out = []
    for k in range(K):
        p6, L = pred[k].contiguous(), pred.shape[1]
        c = np.arange(L)[:, None] - (lag if zero_lag else 0)
        win = np.ascontiguousarray(np.clip(c + (np.arange(T)[None] - T // 2) * SKIP, 0, L - 1), dtype=np.int32)
        rows = np.ascontiguousarray(win[:, np.asarray(pairs)], dtype=np.int32)
        E = rows.shape[1]
        v = torch.from_numpy(np.ascontiguousarray(vos[k])).cuda()
        p7 = torch.empty((L, T, 7), dtype=torch.float64, device="cuda")
        t7, v7 = torch.empty_like(p7), torch.empty((L, E, 7), dtype=torch.float64, device="cuda")
        _lib.check(_lib.lib().mapnet_eval_windows(p6.data_ptr(), L, p6.data_ptr(), v.data_ptr(), L, win.ctypes.data,
                                                  win.ctypes.data, L * T, rows.ctypes.data, L * E, p7.data_ptr(),
                                                  t7.data_ptr(), v7.data_ptr(), _lib.stream_ptr()), "eval_windows")
        mid = pgo(p7, v7, fc_vos=FC, **SIG)[:, T - 1 if zero_lag else T // 2]
        out.append(torch.cat((mid[:, :3] * s + m, mid[:, 3:]), -1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--streams", default="1,8,64")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_track_multi.json"))
    a = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_track_multi: no CUDA device")
    from bench_infer import card, events_ms
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import resize_output_size
    from geomapnet_b200.inference import Localizer, MultiTracker, Predictor, Tracker
    from geomapnet_b200.models.posenet import PoseNet
    Ho, Wo = resize_output_size(H_IN, W_IN)
    lag = (T - 1 - T // 2) * SKIP
    Ks = [int(k) for k in a.streams.split(",")]
    res = {"what": "K camera streams of 480x640 uint8 frames + VO-library poses, one frame per stream per tick -> "
                   "MapNet+PGO poses, bf16 PoseNet droprate 0, RobotCar PGO settings (steps 7, skip 10, vo_fc, sax 1, "
                   "saq 1, srx 20, srq 20): one MultiTracker call per tick (Predictor max_batch 64) against K "
                   "Trackers called once each (Predictor max_batch 1), __call__ and step, past the lag",
           "card": card(), "frame": [H_IN, W_IN], "engine_input": [Ho, Wo], "steps": T, "skip": SKIP, "vo_fc": FC,
           "sigmas": SIG, "lag": lag, "rounds": a.rounds, "streams": Ks, "per_k": {}}
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False, precision="bf16",
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
    vo = (poses + rng.standard_normal(poses.shape) * 0.02).astype(np.float32)
    vo_dev = torch.from_numpy(vo).cuda()
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
            mts = {"call": MultiTracker(loc64, K, steps=T, skip=SKIP, vo_fc=FC, **SIG),
                   "step": MultiTracker(loc64, K, steps=T, skip=SKIP, vo_fc=FC, **SIG)}
            trks = {m: [Tracker(loc1, steps=T, skip=SKIP, vo_fc=FC, **SIG) for _ in range(K)] for m in mts}
            ids_k = torch.arange(K)
            pool_ix = [torch.from_numpy(tick_ids(K, t)).cuda() for t in range(n_pool)]
            pos = {}

            def arm(name, mode, multi):
                pos[name] = 0

                def call():
                    ix = pool_ix[pos[name] % n_pool]
                    pos[name] += 1
                    f, v = frames[ix], vo_dev[ix]
                    if multi:
                        mt = mts[mode]
                        return mt(f, v, ids_k) if mode == "call" else mt.step(f, v, ids_k)
                    for k, trk in enumerate(trks[mode]):
                        trk(f[k:k + 1], v[k:k + 1]) if mode == "call" else trk.step(f[k:k + 1], v[k:k + 1])
                return call

            arms = {"multi_call": arm("multi_call", "call", True), "multi_step": arm("multi_step", "step", True),
                    "trackers_call": arm("trackers_call", "call", False),
                    "trackers_step": arm("trackers_step", "step", False)}
            loc64(frames[:K]); loc1(frames[:1])           # the engines and plans
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

            # bitwise: a fresh sequence of lag + 16 ticks on every stream against the composition
            V = lag + 16
            ticks = [torch.from_numpy(tick_ids(K, t)).cuda() for t in range(V)]
            same = True
            for mode in ("call", "step"):
                mt = mts[mode]
                mt.reset()
                got = {k: [] for k in range(K)}
                nows = []
                for t in range(V):
                    f, v = frames[ticks[t]], vo_dev[ticks[t]]
                    if mode == "call":
                        sid, fid, p = mt(f, v, ids_k)
                    else:
                        now7, sid, fid, p = mt.step(f, v, ids_k)
                        nows.append(now7)
                    for r in range(sid.shape[0]):
                        got[int(sid[r])].append(p[r:r + 1])
                for k in range(K):
                    got[k].append(mt.flush(k)[1])
                want = composition(pr64, frames, vo, [tk.cpu().numpy() for tk in ticks], K, False)
                same = same and all(torch.equal(torch.cat(got[k]), want[k]) for k in range(K))
                if mode == "step":
                    now_all = torch.stack(nows, 1)                  # [K, V, 7]
                    want_now = composition(pr64, frames, vo, [tk.cpu().numpy() for tk in ticks], K, True)
                    same = same and all(torch.equal(now_all[k], want_now[k]) for k in range(K))
            res["per_k"][str(K)] = {
                "iters": iters,
                "ms_per_tick": {k: round(v, 4) for k, v in med.items()},
                "ms_per_tick_rounds": {k: [round(x, 4) for x in v] for k, v in tt.items()},
                "frames_per_s": {k: round(K / v * 1e3, 1) for k, v in med.items()},
                "trackers_over_multi": {"call": round(med["trackers_call"] / med["multi_call"], 2),
                                        "step": round(med["trackers_step"] / med["multi_step"], 2)},
                "library_launches": launches,
                "multi_equals_composition_bitwise": bool(same)}
            print(json.dumps({K: res["per_k"][str(K)]["ms_per_tick"]}), file=sys.stderr)
            for mt in mts.values():
                mt.close()
            for ts in trks.values():
                for trk in ts:
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
