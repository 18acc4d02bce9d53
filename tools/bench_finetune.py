"""Fine-tuning step time on the H100: the graphed posenet_bs64 training step with the lower layers frozen.

    python tools/bench_finetune.py [--iters 20] [--warmup 5] [--rounds 5] [--out FILE]

posenet_bs64 as bench.py runs it (B = 64 at 256x256, bf16, Adam with weight decay, learnable criterion scalars, one
GraphedTrainStep per arm), with requires_grad_(False) on every parameter below the arm's first trainable layer:
  all          -- nothing frozen (the full step)
  from_layer2  -- stem and layer1 frozen
  from_layer3  -- stem, layer1 and layer2 frozen
  layer4_head  -- only layer4 and the pose head (feature_extractor.fc, fc_xyz, fc_wpqr) train
  head_only    -- only the pose head trains
Each arm has its own model and optimizer (a captured optimizer step belongs to the set of parameters it updates).  The
arms alternate within each of `--rounds` rounds of `--iters` replays, timed with CUDA events after `--warmup` replays; the
median round is reported, next to the conv FLOPs the arm's backward schedule computes (forward + the wgrads of trainable
convs + the dgrads the skipping rule keeps) as a share of the full step's.  The card's name, power limit and clocks are
read in the same run.  Prints one JSON line (and writes it to --out).  No CPU fallback.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_infer import card, events_ms   # noqa: E402

FE = "feature_extractor."
HEAD = (FE + "fc.", "fc_xyz.", "fc_wpqr.")
ARMS = (
    ("all", lambda n: True),
    ("from_layer2", lambda n: not n.startswith((FE + "conv1.", FE + "bn1.", FE + "layer1."))),
    ("from_layer3", lambda n: not n.startswith((FE + "conv1.", FE + "bn1.", FE + "layer1.", FE + "layer2."))),
    ("layer4_head", lambda n: n.startswith(HEAD + (FE + "layer4.",))),
    ("head_only", lambda n: n.startswith(HEAD)),
)
STAGES = ((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2))


def conv_gflop(train, H=256, W=256):
    """(forward, wgrad, dgrad) conv GFLOP per image of one training step when the parameters `train(name)` selects need
    a gradient: the backward stops at the lowest block with a trainable conv or BatchNorm (the stem when conv1 / bn1
    trains), that block computes no input gradient unless the stem trains, and a wgrad runs for a trainable weight."""
    def out(n, k, s, p):
        return (n + 2 * p - k) // s + 1
    h, w = out(H, 7, 2, 3), out(W, 7, 2, 3)
    stem = 2.0 * h * w * 64 * 3 * 49
    h, w = out(h, 3, 2, 1), out(w, 3, 2, 1)
    blocks, inpl = [], 64          # [(prefix, [(conv name, flops)])]
    for li, (planes, nblk, stride) in enumerate(STAGES):
        for b in range(nblk):
            s = stride if b == 0 else 1
            h2, w2 = out(h, 3, s, 1), out(w, 3, s, 1)
            pre = "%slayer%d.%d." % (FE, li + 1, b)
            convs = [("conv1", 2.0 * h2 * w2 * planes * inpl * 9), ("conv2", 2.0 * h2 * w2 * planes * planes * 9)]
            if s != 1 or inpl != planes:
                convs.append(("downsample.0", 2.0 * h2 * w2 * planes * inpl))
            blocks.append((pre, convs))
            h, w, inpl = h2, w2, planes

    def block_trains(pre, convs):
        bns = ["bn1", "bn2"] + (["downsample.1"] if len(convs) == 3 else [])
        return (any(train(pre + c + ".weight") for c, _ in convs)
                or any(train(pre + b + s) for b in bns for s in (".weight", ".bias")))
    stem_trains = any(train(FE + p) for p in ("conv1.weight", "bn1.weight", "bn1.bias"))
    lo = -1 if stem_trains else next((i for i, b in enumerate(blocks) if block_trains(*b)), len(blocks))
    fwd = stem + sum(f for _, convs in blocks for _, f in convs)
    wgrad = stem if train(FE + "conv1.weight") else 0.0
    dgrad = 0.0
    for bi, (pre, convs) in enumerate(blocks):
        wgrad += sum(f for c, f in convs if train(pre + c + ".weight"))
        if bi >= max(lo, 0):
            dgrad += convs[1][1] + (sum(f for c, f in convs if c != "conv2") if bi > lo else 0.0)
    return fwd * 1e-9, wgrad * 1e-9, dgrad * 1e-9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_finetune.json"))
    a = ap.parse_args()
    import torch
    import torchvision
    if not torch.cuda.is_available():
        sys.exit("bench_finetune: no CUDA device")
    from geomapnet_b200.models.posenet import PoseNet
    from geomapnet_b200.common.criterion import PoseNetCriterion
    from geomapnet_b200.common.optimizer import Optimizer
    from geomapnet_b200.graph import GraphedTrainStep
    from oracle import weights, mapnet_oracle as O
    B, H, W = 64, 256, 256
    full = conv_gflop(lambda n: True, H, W)
    assert abs(sum(full) - O.train_flops_per_image(H, W) * 1e-9) < 1e-6 * sum(full)
    x, t = weights.make_inputs(dict(kind="posenet", N=B, H=H, W=W), 1000)
    x, t = x.cuda(), t.cuda()
    arms = []
    for name, train in ARMS:
        torch.manual_seed(7)
        net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False, precision="bf16",
                      seed=7).cuda()
        crit = PoseNetCriterion(sax=0.0, saq=-3.0, learn_beta=True).cuda()
        n_train = 0
        for pn, p in net.named_parameters():
            p.requires_grad_(bool(train(pn)))
            n_train += p.numel() if p.requires_grad else 0
        opt = Optimizer(params=[{"params": net.parameters()}, {"params": list(crit.parameters())}], method="adam",
                        base_lr=1e-4, weight_decay=5e-4)
        net.train()
        step = GraphedTrainStep(net, crit, opt, x, t, warmup=2)
        gf = conv_gflop(train, H, W)
        arms.append(dict(name=name, step=step, net=net, n_train=n_train, gf=gf))
    for arm in arms:
        for _ in range(a.warmup):
            arm["step"].replay()
    times = {arm["name"]: [] for arm in arms}
    for _ in range(a.rounds):
        for arm in arms:
            times[arm["name"]].append(events_ms(arm["step"].replay, a.iters))
    base = statistics.median(times["all"])
    res = {"what": "posenet_bs64 graphed training step (B=64, 256x256, bf16, Adam + weight decay, droprate 0.5) with the "
                   "layers below each arm's first trainable one frozen (requires_grad_(False)); arms alternate in "
                   "every round, median of rounds",
           "card": card(), "B": B, "H": H, "W": W, "iters": a.iters, "warmup": a.warmup, "rounds": a.rounds,
           "full_conv_gflop_per_image": round(sum(full), 4), "arms": []}
    for arm in arms:
        m = statistics.median(times[arm["name"]])
        fwd, wg, dg = arm["gf"]
        res["arms"].append({
            "arm": arm["name"], "ms": round(m, 4), "img_s": round(B / m * 1e3, 1), "time_share": round(m / base, 3),
            "conv_gflop_per_image": {"fwd": round(fwd, 3), "wgrad": round(wg, 3), "dgrad": round(dg, 3),
                                     "total": round(fwd + wg + dg, 3)},
            "conv_flop_share": round((fwd + wg + dg) / sum(full), 3),
            "trainable_params": arm["n_train"], "kernels_per_step": arm["step"].kernels_per_step,
            "ms_rounds": [round(v, 4) for v in times[arm["name"]]]})
        print(json.dumps(res["arms"][-1]), file=sys.stderr)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
