"""Camera frames to metric poses on the H100: inference.Localizer (one graph: resize, Normalize into the stem operand,
the engine, pose post-processing) against the three-call chain it replaces and against the reference's host-side input.

    python tools/bench_localize.py [--sizes 1,8,64] [--fp8-sizes 1,64] [--iters 50] [--ref-iters 3] [--warmup 5]
                                   [--rounds 5] [--out FILE]

Seeded synthetic 480x640 uint8 RGB frames (7Scenes size; Resize(256) -> 256x341) and a bf16 PoseNet at droprate 0 with
the running statistics of a few training-mode batches; the fp8 runs use a Predictor(precision='fp8') of the same model,
calibrated on the preprocessed frames.  Arms, alternating inside each of `--rounds` rounds, medians reported:
  a  Localizer(frames) from a CUDA frame batch                              (CUDA events, --iters calls)
  b  post(Predictor(ImagePipeline(frames)))                                 (CUDA events, --iters calls)
  c  a and b from a pinned host frame batch, ending in a host copy of the poses   (host clock, --iters calls)
  d  the reference's input side: Pillow Resize(256) + torchvision ToTensor / Normalize per frame on the host, then
     Predictor and post, ending in a host copy                              (host clock, --ref-iters calls)
Launches per call are counted with mapnet_launch_count around one eager run of each chain.  The preprocessing bytes
per frame are computed here from the shapes (algorithmic: each tensor written once and read once), not measured.
The card's name, power limit and clocks are read in the same run.  Prints one JSON line (and writes it to --out).
No CPU fallback: without a GPU it exits.
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
H_IN, W_IN = 480, 640


def preprocess_bytes(Hin, Win, size=256, operand_elt=2):
    """algorithmic bytes per frame of the input side, from the shapes: (today, fused)"""
    from geomapnet_b200.data import resize_output_size
    Ho, Wo = resize_output_size(Hin, Win, size)
    hc, wc = (Ho - 1) // 2 + 1, (Wo - 1) // 2 + 1
    frame = Hin * Win * 3                               # uint8 input, read once
    inter = Hin * Wo * 3                                # uint8 after the horizontal pass, written and read
    image = Ho * Wo * 3 * 4                             # float32 NCHW after Normalize, written and read
    operand = (hc + 3) * ((wc + 6) // 4 * 4) * 16 * operand_elt    # space-to-depth stem operand, written
    return {"frame": frame, "intermediate_u8": inter, "float32_image": image, "stem_operand": operand,
            "chain": frame + 2 * inter + 2 * image + operand, "fused": frame + 2 * inter + operand}


def host_ms(fn, n):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64")
    ap.add_argument("--fp8-sizes", default="1,64")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--ref-iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_localize.json"))
    a = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    import torchvision.transforms as T
    from PIL import Image
    if not torch.cuda.is_available():
        sys.exit("bench_localize: no CUDA device")
    from bench_infer import card, events_ms
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import ImagePipeline, resize_output_size
    from geomapnet_b200.inference import Localizer, Predictor, post
    from geomapnet_b200.models.posenet import PoseNet
    L = _lib.lib()
    sizes = [int(s) for s in a.sizes.split(",") if s]
    f8_sizes = [int(s) for s in a.fp8_sizes.split(",") if s]
    mb = max(sizes + f8_sizes)
    Ho, Wo = resize_output_size(H_IN, W_IN)
    res = {"what": "480x640 uint8 frames -> float64 poses, PoseNet droprate 0: Localizer (a) vs the three-call chain "
                   "(b), both from pinned host frames with a host copy of the poses (c), and Pillow/torchvision host "
                   "preprocessing + Predictor + post (d)",
           "card": card(), "frame": [H_IN, W_IN], "engine_input": [Ho, Wo],
           "preprocess_bytes_per_frame": preprocess_bytes(H_IN, W_IN),
           "iters": a.iters, "ref_iters": a.ref_iters, "warmup": a.warmup, "rounds": a.rounds, "runs": []}
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False, precision="bf16",
                  seed=7).cuda()
    with torch.no_grad():
        net.train()
        for _ in range(3):
            net(torch.randn(16, 3, Ho, Wo, device="cuda"))
    net.eval()
    g = torch.Generator().manual_seed(11)
    frames_host = torch.randint(0, 256, (mb, H_IN, W_IN, 3), dtype=torch.uint8, generator=g).pin_memory()
    frames_dev = frames_host.cuda()
    pipe = ImagePipeline(MEAN, STD)
    ref_tf = T.Compose([T.Resize(256), T.ToTensor(), T.Normalize(MEAN, STD)])
    arrays = [frames_host[i].numpy() for i in range(mb)]
    for precision, bs in (("bf16", sizes), ("fp8", f8_sizes)):
        if not bs:
            continue
        if precision == "fp8":
            pr = Predictor(net, max_batch=mb, precision="fp8", calibration=pipe(frames_dev[:8]))
        else:
            pr = Predictor(net, max_batch=mb)
        loc = Localizer(pr, MEAN, STD)
        eng = pr._engine(Ho, Wo)
        for B in bs:
            fd, fh = frames_dev[:B], frames_host[:B]
            with torch.no_grad():
                arm_a = lambda: loc(fd)
                arm_b = lambda: post(pr(pipe(fd)))
                arm_ca = lambda: loc(fh).cpu()
                arm_cb = lambda: post(pr(pipe(fh.cuda(non_blocking=True)))).cpu()
                arm_d = lambda: post(pr(torch.stack([ref_tf(Image.fromarray(arrays[i])) for i in range(B)])
                                        .cuda())).cpu()
                out_a, out_b, out_d = arm_a(), arm_b(), arm_d()
                # launches of one eager run of each chain (a replays a graph of exactly these launches)
                _, xs, out7, pred6 = loc._graph(fd)
                c0 = L.mapnet_launch_count()
                loc._launch(eng, loc._plan(H_IN, W_IN), xs, pred6, out7, 0.0)
                c1 = L.mapnet_launch_count()
                x = pipe(fd)
                tmp = torch.empty(B, 6, device="cuda")
                eng.forward(x, tmp, 0.0, 0)
                post(tmp)
                c2 = L.mapnet_launch_count()
                torch.cuda.synchronize()
                for _ in range(a.warmup):
                    arm_a(); arm_b(); arm_ca(); arm_cb()
                arm_d()
                t = {k: [] for k in ("a", "b", "c_a", "c_b", "d")}
                for _ in range(a.rounds):
                    t["a"].append(events_ms(arm_a, a.iters))
                    t["b"].append(events_ms(arm_b, a.iters))
                    t["c_a"].append(host_ms(arm_ca, a.iters))
                    t["c_b"].append(host_ms(arm_cb, a.iters))
                    t["d"].append(host_ms(arm_d, a.ref_iters))
            med = {k: statistics.median(v) for k, v in t.items()}
            run = {"precision": precision, "B": B,
                   "ms": {k: round(v, 4) for k, v in med.items()},
                   "frames_per_s": {k: round(B / v * 1e3, 1) for k, v in med.items()},
                   "speedup_a_over_b": round(med["b"] / med["a"], 3),
                   "speedup_c": round(med["c_b"] / med["c_a"], 3),
                   "launches_per_call": {"localizer": int(c1 - c0), "chain": int(c2 - c1)},
                   "a_equals_b_bitwise": bool(torch.equal(out_a, out_b)),
                   "d_equals_b_bitwise": bool(torch.equal(out_d.to(out_b.device), out_b)),
                   "ms_rounds": {k: [round(x, 4) for x in v] for k, v in t.items()}}
            res["runs"].append(run)
            print(json.dumps(run), file=sys.stderr)
        loc.close()
        pr.close()
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
