"""fp8 against bf16 inference on the H100: two Predictors of the same PoseNet, alternating in the same run.

    python tools/bench_infer_fp8.py [--sizes 1,8,64,256] [--iters 50] [--warmup 10] [--rounds 5] [--out FILE]

PoseNet at 256x256, droprate 0, a 'bf16' model with the running statistics of a few training-mode batches.  The fp8
Predictor is calibrated on 64 frames from the same distribution.  For every batch size the two Predictors alternate in
`--rounds` rounds of `--iters` graph-replayed calls each, timed with CUDA events after `--warmup` calls; the median
round is reported as ms per call and images/s, and the conv FLOPs (9.5693 GFLOP per image) over that time as a fraction
of both the dense bf16 (989 TFLOP/s) and the dense FP8 (1,979 TFLOP/s) data-sheet rates -- an end-to-end figure of the
whole call, not a kernel's share of peak.  On the same input, the max relative difference of the fp8 output from the
bf16 Predictor and from the fp32 eval forward of the model (model.eval(), fp32 precision copy).  The card's name, power
limit and clocks are read in the same run.  Prints one JSON line (and writes it to --out).  No CPU fallback.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_infer import CONV_FLOP_PER_IMAGE, card, events_ms   # noqa: E402

PEAK_BF16 = 989e12     # H100 SXM data sheet, dense
PEAK_FP8 = 1979e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,256")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_infer_fp8.json"))
    a = ap.parse_args()
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_infer_fp8: no CUDA device")
    from geomapnet_b200 import _lib
    from geomapnet_b200.models.posenet import PoseNet
    from geomapnet_b200.inference import Predictor
    L = _lib.lib()
    sizes = [int(s) for s in a.sizes.split(",")]
    H = W = 256
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False, precision="bf16", seed=7).cuda()
    with torch.no_grad():
        net.train()
        for _ in range(3):
            net(torch.randn(16, 3, H, W, device="cuda"))
    net.eval()
    # the fp32 eval forward of the same weights and running statistics: the reference the drift is measured against
    ref_net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False, precision="fp32",
                      seed=7).cuda()
    ref_net.load_state_dict(net.state_dict())
    ref_net.eval()
    calib = torch.randn(64, 3, H, W, device="cuda")
    mb = max(sizes)
    pr16 = Predictor(net, max_batch=mb)
    pr8 = Predictor(net, max_batch=mb, precision="fp8", calibration=calib)
    res = {"what": "posenet eval forward, 256x256, droprate 0: fp8 Predictor vs bf16 Predictor (graph replay, "
                   "alternating rounds); fp8 calibrated on 64 frames",
           "card": card(), "conv_gflop_per_image": CONV_FLOP_PER_IMAGE / 1e9, "peak_tflops_bf16": PEAK_BF16 / 1e12,
           "peak_tflops_fp8": PEAK_FP8 / 1e12, "iters": a.iters, "warmup": a.warmup, "rounds": a.rounds,
           "act_scales": pr8.act_scales, "runs": []}
    for B in sizes:
        x = torch.randn(B, 3, H, W, device="cuda")
        with torch.no_grad():
            o8, o16 = pr8(x), pr16(x)
            ref = torch.cat([ref_net(x[i:i + 64]) for i in range(0, B, 64)])
            c0 = L.mapnet_launch_count(); pr8._engine(H, W).forward(x[:min(B, mb)], torch.empty(B, 6, device="cuda"), 0.0, 0)
            torch.cuda.synchronize()
            launches = int(L.mapnet_launch_count() - c0)
            rel = lambda p, q: float((p.double() - q.double()).abs().max() / q.double().abs().max())
            f8_fn, bf_fn = (lambda: pr8(x)), (lambda: pr16(x))
            for _ in range(a.warmup):
                f8_fn(); bf_fn()
            t8, t16 = [], []
            for _ in range(a.rounds):
                t8.append(events_ms(f8_fn, a.iters))
                t16.append(events_ms(bf_fn, a.iters))
        m8, m16 = statistics.median(t8), statistics.median(t16)
        flop = CONV_FLOP_PER_IMAGE * B
        run = {"B": B, "fp8_ms": round(m8, 4), "bf16_ms": round(m16, 4), "speedup": round(m16 / m8, 3),
               "fp8_img_s": round(B / m8 * 1e3, 1), "bf16_img_s": round(B / m16 * 1e3, 1),
               "fp8_conv_flop_frac_of_bf16_peak": round(flop / (m8 * 1e-3) / PEAK_BF16, 4),
               "fp8_conv_flop_frac_of_fp8_peak": round(flop / (m8 * 1e-3) / PEAK_FP8, 4),
               "bf16_conv_flop_frac_of_bf16_peak": round(flop / (m16 * 1e-3) / PEAK_BF16, 4),
               "fp8_launches": launches,
               "fp8_vs_bf16_max_rel_diff": float("%.3e" % rel(o8, o16)),
               "fp8_vs_fp32_max_rel_diff": float("%.3e" % rel(o8, ref)),
               "bf16_vs_fp32_max_rel_diff": float("%.3e" % rel(o16, ref)),
               "fp8_ms_rounds": [round(t, 4) for t in t8], "bf16_ms_rounds": [round(t, 4) for t in t16]}
        res["runs"].append(run)
        print(json.dumps(run), file=sys.stderr)
    pr8.close(); pr16.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
