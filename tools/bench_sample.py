"""Monte-Carlo dropout poses on the H100: S dropout draws per frame from one trunk forward (Predictor.sample,
Localizer.sample) against S ordinary calls.

    python tools/bench_sample.py [--sizes 1,64] [--draws 8,32] [--iters 20] [--warmup 3] [--rounds 5] [--out FILE]

A bf16 PoseNet at droprate 0.5 with the running statistics of a few training-mode batches, and seeded synthetic 480x640
uint8 RGB frames (7Scenes size; Resize(256) -> 256x341; the Predictor arms take them through ImagePipeline once, up
front).  Arms, alternating inside each of `--rounds` rounds, medians reported (CUDA events around --iters calls):
  one     pr(x)                          one ordinary forward
  sample  pr.sample(x, S)                one trunk forward + S head draws + float64 statistics
  loop    S calls pr(x)                  what sampling costs without this feature
  lsample loc.sample(frames, S)          the same from camera frames, metric pose and covariance
  lloop   S calls loc(frames)
Library launches per call are counted with mapnet_launch_count around one eager run of each call's launches; graph
replays per call are 1 for sample / lsample and S for the loops.  Each run also records whether the draws equal the
loop's poses bit for bit (on twin Predictors whose dropout counters start in step).  The card's name, power limit
and clocks are read in the same run.  Prints one JSON line (and writes it to --out).  No CPU fallback: without a GPU
it exits.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]    # 7Scenes chess stats.txt
STD = [v ** 0.5 for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
H_IN, W_IN = 480, 640


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,64")
    ap.add_argument("--draws", default="8,32")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_sample.json"))
    a = ap.parse_args()
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_sample: no CUDA device")
    from bench_infer import card, events_ms
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import ImagePipeline, resize_output_size
    from geomapnet_b200.inference import Localizer, Predictor
    from geomapnet_b200.models.posenet import PoseNet
    L = _lib.lib()
    sizes = [int(s) for s in a.sizes.split(",") if s]
    draws = [int(s) for s in a.draws.split(",") if s]
    mb = max(sizes)
    Ho, Wo = resize_output_size(H_IN, W_IN)
    res = {"what": "480x640 uint8 frames, bf16 PoseNet droprate 0.5: S Monte-Carlo dropout draws per frame from one "
                   "trunk forward (sample) against S ordinary calls (loop), for Predictor and Localizer",
           "card": card(), "frame": [H_IN, W_IN], "engine_input": [Ho, Wo], "iters": a.iters, "warmup": a.warmup,
           "rounds": a.rounds, "runs": []}
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False, precision="bf16",
                  seed=7).cuda()
    with torch.no_grad():
        net.train()
        for _ in range(3):
            net(torch.randn(16, 3, Ho, Wo, device="cuda"))
    net.eval()
    g = torch.Generator().manual_seed(11)
    frames = torch.randint(0, 256, (mb, H_IN, W_IN, 3), dtype=torch.uint8, generator=g).cuda()
    x_all = ImagePipeline(MEAN, STD)(frames)
    pr = Predictor(net, max_batch=mb)
    loc = Localizer(pr, MEAN, STD)
    eng = pr._engine(Ho, Wo)
    for B in sizes:
        x, f = x_all[:B], frames[:B]
        with torch.no_grad():
            pr(x), loc(f)                                # the ordinary graphs of this shape
            for S in draws:
                # bitwise: the draws are S ordinary calls of a twin Predictor whose dropout counter is in step
                p1, p2 = Predictor(net, max_batch=B), Predictor(net, max_batch=B)
                p1(x), p2(x)
                out = p1.sample(x, S, keep_samples=True)
                bitwise = all(torch.equal(out["samples"][:, s], p2(x)) for s in range(S))
                p1.close(), p2.close()
                # library launches of one eager run of each call
                smp = torch.empty(B, S, 6, device="cuda")
                m6 = torch.empty(B, 6, dtype=torch.float64, device="cuda")
                c6 = torch.empty(B, 6, 6, dtype=torch.float64, device="cuda")
                pred = torch.empty(B, 6, device="cuda")
                c0 = L.mapnet_launch_count()
                eng.forward(x.contiguous(), pred, pr.droprate, pr.seed, step=0)
                c1 = L.mapnet_launch_count()
                eng.sample(x.contiguous(), S, pr.droprate, pr.seed, smp, m6, c6, step=0)
                c2 = L.mapnet_launch_count()
                arms = {"one": lambda: pr(x),
                        "sample": lambda: pr.sample(x, S),
                        "loop": lambda: [pr(x) for _ in range(S)],
                        "lsample": lambda: loc.sample(f, S),
                        "lloop": lambda: [loc(f) for _ in range(S)]}
                for fn in arms.values():
                    for _ in range(a.warmup):
                        fn()
                torch.cuda.synchronize()
                t = {k: [] for k in arms}
                for _ in range(a.rounds):
                    for k, fn in arms.items():
                        t[k].append(events_ms(fn, a.iters))
                med = {k: statistics.median(v) for k, v in t.items()}
                run = {"precision": "bf16", "B": B, "S": S,
                       "ms": {k: round(v, 4) for k, v in med.items()},
                       "sample_over_one": round(med["sample"] / med["one"], 3),
                       "loop_over_sample": round(med["loop"] / med["sample"], 2),
                       "lloop_over_lsample": round(med["lloop"] / med["lsample"], 2),
                       # sample: the engine's launches and mapnet_sample_post's one
                       "launches_per_call": {"forward": int(c1 - c0), "sample": int(c2 - c1) + 1,
                                             "loop": S * int(c1 - c0)},
                       "graph_replays_per_call": {"sample": 1, "loop": S},
                       "draws_equal_loop_bitwise": bool(bitwise),
                       "ms_rounds": {k: [round(v, 4) for v in vs] for k, vs in t.items()}}
                res["runs"].append(run)
                print(json.dumps(run), file=sys.stderr)
    loc.close()
    pr.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
