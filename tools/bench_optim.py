"""Fused SGD / RMSprop on the H100: the optimizer step alone and the whole CUDA-graph training step.

    python tools/bench_optim.py [--steps 200] [--warmup 10] [--rounds 5] [--train-steps 30] [--out FILE]

Prints one JSON line (and writes it to --out).

* Optimizer step alone, on the PoseNet parameter set (the flat buffer of 22 347 590 parameters plus padding, one run,
  and the criterion's sax / saq group) with the gradients of one backward pass.  For each configuration the fused
  step is captured once in a CUDA graph and replayed `--steps` times between CUDA events (kernel time: the step's
  launches without Python); the same step called eagerly and torch.optim.SGD / RMSprop (foreach) with
  clip_grad_norm_ are timed the same way, eagerly (host launch cost included).  Algorithmic bytes per parameter:
  SGD 12 (20 with momentum), RMSprop 20 (28 with momentum or centered, 36 with both), +4 with the clip (the norm
  reads the gradient once more); fraction of the 3.35 TB/s H100 SXM data-sheet bandwidth.
* Whole step: GraphedTrainStep images/s at posenet_bs64 (bf16, droprate 0.5) with adam, sgd (momentum 0.9) and
  rmsprop, in `--rounds` alternating rounds of `--train-steps` replays each; the median round is reported.

The card's name and power limit are read in the same run.  No CPU fallback: without a GPU it exits.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet
CONFIGS = [("sgd", dict(momentum=0.0)), ("sgd", dict(momentum=0.9)), ("sgd", dict(momentum=0.9, nesterov=True)),
           ("rmsprop", dict()), ("rmsprop", dict(momentum=0.9)), ("rmsprop", dict(momentum=0.9, centered=True))]


def bytes_per_param(method, kw, clip):
    if method == "sgd":
        b = 20 if kw.get("momentum", 0.0) else 12
    else:
        b = 20 + 8 * (kw.get("momentum", 0.0) > 0) + 8 * bool(kw.get("centered", False))
    return b + (4 if clip else 0)


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        out["nvidia_smi"] = r.stdout.strip()
    except Exception as e:          # the query is informative only
        out["nvidia_smi"] = "unavailable (%s)" % e
    return out


def make_posenet(N, H, W, precision="bf16", droprate=0.5):
    import torch
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet
    from geomapnet_b200.common.criterion import PoseNetCriterion
    torch.manual_seed(7)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=droprate, pretrained=False, precision=precision,
                  seed=7)
    crit = PoseNetCriterion(sax=0.0, saq=-3.0, learn_beta=True)
    net.cuda(); crit.cuda(); net.train()
    return net, crit


def events_ms(fn, n):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def graphed(fn, warmup):
    import torch
    cur = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        for _ in range(warmup):
            fn()
    cur.wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def bench_step_alone(args):
    import torch
    from geomapnet_b200.common.optimizer import FusedRMSprop, FusedSGD
    from oracle import weights
    net, crit = make_posenet(2, 64, 64)
    x, t = weights.make_inputs(dict(kind="posenet", N=2, H=64, W=64), 3)
    loss = crit(net(x.cuda()), t.cuda())
    loss.backward()
    del loss
    model_params = list(net.parameters())
    crit_params = list(crit.parameters())
    n_model = sum(p.numel() for p in model_params)
    n_all = n_model + sum(p.numel() for p in crit_params)
    flat, _ = net.flat_parameters()
    rows = []
    for method, kw in CONFIGS:
        for clip in (0.0, 5.0):
            groups = [{"params": model_params}, {"params": crit_params}]
            cls, tcls = (FusedSGD, torch.optim.SGD) if method == "sgd" else (FusedRMSprop, torch.optim.RMSprop)
            fused = cls(groups, lr=1e-6, weight_decay=5e-4, **kw)

            def fstep():
                fused.step(max_grad_norm=clip)
            g = graphed(fstep, args.warmup)
            for _ in range(args.warmup):
                g.replay()
            ms_graph = events_ms(g.replay, args.steps)
            ms_eager = events_ms(fstep, args.steps)
            del g
            ref = tcls([{"params": model_params}, {"params": crit_params}], lr=1e-6, weight_decay=5e-4, foreach=True,
                       **kw)

            def tstep():
                if clip:
                    torch.nn.utils.clip_grad_norm_(model_params, clip, foreach=True)
                ref.step()
            for _ in range(args.warmup):
                tstep()
            ms_torch = events_ms(tstep, args.steps)
            if clip:            # torch's clip scaled the gradients in place: put the backward's values back
                net.zero_grad(set_to_none=True); crit.zero_grad(set_to_none=True)
                loss = crit(net(x.cuda()), t.cuda())
                loss.backward()
                del loss
            bpp = bytes_per_param(method, kw, clip)
            nbytes = bpp * n_all
            rows.append({"method": method, "config": dict(kw, clip=clip), "bytes_per_param": bpp,
                         "algorithmic_MB": nbytes / 1e6,
                         "fused_graph_ms": ms_graph, "fused_graph_GBps": nbytes / (ms_graph * 1e-3) / 1e9,
                         "fused_graph_frac_of_3p35TBps": nbytes / (ms_graph * 1e-3) / HBM_BYTES_PER_S,
                         "fused_eager_ms": ms_eager, "torch_foreach_eager_ms": ms_torch,
                         "torch_over_fused_graph": ms_torch / ms_graph})
            print("%-8s %-40s %6.1f MB  fused graph %.4f ms (%.0f%% of 3.35 TB/s)  fused eager %.4f ms  "
                  "torch foreach %.4f ms" % (method, dict(kw, clip=clip), nbytes / 1e6, ms_graph,
                                             100 * rows[-1]["fused_graph_frac_of_3p35TBps"], ms_eager, ms_torch),
                  file=sys.stderr, flush=True)
            del fused, ref
    assert bool(torch.isfinite(flat).all())
    return {"n_params": n_all, "n_model_params": n_model, "flat_numel_padded": int(flat.numel()), "rows": rows}


def bench_whole_step(args):
    import torch
    from geomapnet_b200.common.optimizer import Optimizer
    from geomapnet_b200.graph import GraphedTrainStep
    from oracle import weights
    cfg = dict(kind="posenet", N=64, H=256, W=256)
    batches = [weights.make_inputs(cfg, 1000 + i) for i in range(4)]
    batches = [(x.cuda(), t.cuda()) for x, t in batches]
    arms = {}
    for method in ("adam", "sgd", "rmsprop"):
        net, crit = make_posenet(64, 256, 256)
        groups = [{"params": net.parameters()}, {"params": list(crit.parameters())}]
        kw = dict(momentum=0.9, lr_decay=0.1, lr_stepvalues=[60, 80]) if method == "sgd" else {}
        opt = Optimizer(groups, method, 1e-4, 5e-4, **kw)
        g = GraphedTrainStep(net, crit, opt, batches[0][0], batches[0][1], warmup=2)
        for i in range(5):
            g(*batches[i % 4])
        arms[method] = (net, crit, opt, g)
    torch.cuda.synchronize()
    rates = {m: [] for m in arms}
    losses = {}
    for r in range(args.rounds):
        for m, (net, crit, opt, g) in arms.items():
            i = [0]

            def one():
                g(*batches[i[0] % 4]); i[0] += 1
            ms = events_ms(one, args.train_steps)
            rates[m].append(cfg["N"] / (ms * 1e-3))
            losses[m] = float(g.loss)
    out = {}
    for m in arms:
        out[m] = {"images_per_s_median": statistics.median(rates[m]), "images_per_s_rounds": rates[m],
                  "ms_per_step_median": 1e3 * cfg["N"] / statistics.median(rates[m]), "last_loss": losses[m]}
        print("posenet_bs64 graphed %-8s %.0f img/s (rounds %s)" % (m, out[m]["images_per_s_median"],
                                                                    ["%.0f" % v for v in rates[m]]),
              file=sys.stderr, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--train-steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.steps < 100:
        raise SystemExit("bench_optim.py: --steps must be at least 100")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim.py: no CUDA device (no CPU fallback)")
    line = {"tool": "tools/bench_optim.py", "card": card(), "torch": torch.__version__,
            "steps": args.steps, "warmup": args.warmup,
            "step_alone": bench_step_alone(args),
            "whole_step": {"workload": "posenet_bs64", "precision": "bf16", "droprate": 0.5, "rounds": args.rounds,
                           "train_steps_per_round": args.train_steps, "arms": bench_whole_step(args)}}
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
