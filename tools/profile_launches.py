"""Launch list of ONE eager posenet_bs64 training step (B = 64, 256x256, bf16), recorded with torch.profiler's CUDA
activity trace: one row per kernel in start order, `index,kernel,dur_ns`, the input of tools/stage_table.py.

    python tools/profile_launches.py profiles/h100_launches_raw.csv

Two warm-up steps run first (arena, tensor maps, plans); the recorded step is the third.  Kernel names are cut to
`name<template args>` (no `void`, namespace or parameter list).  Durations under the profiler are those of an eager
step: compare stages with each other, not with the CUDA-graph step time of bench.py."""
import csv
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torchvision
    from torch.profiler import ProfilerActivity, profile
    from geomapnet_b200.models.posenet import PoseNet
    from geomapnet_b200.common.criterion import PoseNetCriterion
    from geomapnet_b200.common.optimizer import Optimizer
    from oracle import weights
    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False, precision="bf16", seed=7).cuda()
    crit = PoseNetCriterion(sax=0.0, saq=-3.0, learn_beta=True).cuda()
    opt = Optimizer([{"params": net.parameters()}, {"params": list(crit.parameters())}], "adam", 1e-4, 5e-4)
    net.train()
    x, t = weights.make_inputs(dict(kind="posenet", N=64, T=1, H=256, W=256), 1000)
    x, t = x.cuda(), t.cuda()

    def step():
        loss = crit(net(x), t)
        opt.learner.zero_grad()
        loss.backward()
        opt.learner.step()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    rows = []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or e.name.startswith(("Memcpy", "Memset")):
            continue
        name = re.sub(r"\(.*", "", e.name)
        name = re.sub(r"^void ", "", name).replace("mapnet::", "")
        rows.append((e.time_range.start, name, int(round(e.time_range.elapsed_us() * 1000))))
    rows.sort(key=lambda r: r[0])
    with open(sys.argv[1], "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["index", "kernel", "dur_ns"])
        for i, (_, name, ns) in enumerate(rows):
            w.writerow([i, name, ns])
    print("%d kernels -> %s" % (len(rows), sys.argv[1]))


if __name__ == "__main__":
    main()
