"""Eval-mode inference on the H100: the live path (model.eval() under no_grad, eager) against the Predictor (frozen
snapshot, BatchNorm / residual / ReLU in the conv epilogues, CUDA-graph replay).

    python tools/bench_infer.py [--sizes 1,8,64,256] [--iters 50] [--warmup 10] [--rounds 5] [--out FILE]

PoseNet at 256x256, droprate 0 (deterministic outputs, so the two arms can be compared), precisions bf16 and tc_split.
For every batch size the two arms alternate in `--rounds` rounds of `--iters` calls each, timed with CUDA events after
`--warmup` calls; the median round is reported as ms per call, images/s and the fraction of the 989 TFLOP/s dense
bf16 data-sheet peak that the conv FLOPs (9.5693 GFLOP per image forward) would take.  Launches per call are counted by
mapnet_launch_count around one eager call of each arm; the max relative difference between the arms' outputs is taken
on the same input.  The card's name, power limit and clocks are read in the same run.  Prints one JSON line (and
writes it to --out).  No CPU fallback: without a GPU it exits.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_FLOPS = 989e12            # H100 SXM data sheet, dense bf16
CONV_FLOP_PER_IMAGE = 9.5693e9  # 2 x conv MACs of one 256x256 forward (oracle.mapnet_oracle.conv_macs_per_image)


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        out["nvidia_smi"] = r.stdout.strip()
    except Exception as e:          # the query is informative only
        out["nvidia_smi"] = "unavailable (%s)" % e
    return out


def events_ms(fn, n):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,256")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_infer.json"))
    a = ap.parse_args()
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_infer: no CUDA device")
    from geomapnet_b200 import _lib
    from geomapnet_b200.models.posenet import PoseNet
    from geomapnet_b200.inference import Predictor
    L = _lib.lib()
    sizes = [int(s) for s in a.sizes.split(",")]
    H = W = 256
    res = {"what": "posenet eval forward, 256x256, droprate 0: live model.eval() (eager) vs Predictor (graph replay)",
           "card": card(), "conv_gflop_per_image": CONV_FLOP_PER_IMAGE / 1e9, "peak_tflops": PEAK_FLOPS / 1e12,
           "iters": a.iters, "warmup": a.warmup, "rounds": a.rounds, "runs": []}
    for precision in ("bf16", "tc_split"):
        torch.manual_seed(7)
        net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False, precision=precision,
                      seed=7).cuda()
        # running statistics of a few training-mode batches: activations normalised as in a trained net
        with torch.no_grad():
            net.train()
            for i in range(3):
                net(torch.randn(16, 3, H, W, device="cuda"))
        net.eval()
        pr = Predictor(net, max_batch=max(sizes))
        for B in sizes:
            x = torch.randn(B, 3, H, W, device="cuda")
            with torch.no_grad():
                live_fn = lambda: net(x)
                c0 = L.mapnet_launch_count(); ref = live_fn(); torch.cuda.synchronize()
                live_launches = int(L.mapnet_launch_count() - c0)
                out = pr(x)
                eng = pr._engine(H, W)
                tmp = torch.empty(B, 6, device="cuda")
                c0 = L.mapnet_launch_count(); eng.forward(x, tmp, 0.0, 0); torch.cuda.synchronize()
                pr_launches = int(L.mapnet_launch_count() - c0)
                diff = float((out.double() - ref.double()).abs().max() / ref.double().abs().max())
                pr_fn = lambda: pr(x)
                for _ in range(a.warmup):
                    live_fn(); pr_fn()
                t_live, t_pr = [], []
                for _ in range(a.rounds):
                    t_live.append(events_ms(live_fn, a.iters))
                    t_pr.append(events_ms(pr_fn, a.iters))
            ml, mp = statistics.median(t_live), statistics.median(t_pr)
            flop = CONV_FLOP_PER_IMAGE * B
            run = {"precision": precision, "B": B,
                   "live_ms": round(ml, 4), "predictor_ms": round(mp, 4), "speedup": round(ml / mp, 3),
                   "live_img_s": round(B / ml * 1e3, 1), "predictor_img_s": round(B / mp * 1e3, 1),
                   "live_conv_flop_frac": round(flop / (ml * 1e-3) / PEAK_FLOPS, 4),
                   "predictor_conv_flop_frac": round(flop / (mp * 1e-3) / PEAK_FLOPS, 4),
                   "live_launches": live_launches, "predictor_launches": pr_launches,
                   "max_rel_diff": float("%.3e" % diff),
                   "live_ms_rounds": [round(t, 4) for t in t_live], "predictor_ms_rounds": [round(t, 4) for t in t_pr]}
            res["runs"].append(run)
            print(json.dumps(run), file=sys.stderr)
        pr.close()
        del net
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
