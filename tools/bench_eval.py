"""Evaluation throughput on the H100: scripts/eval.py's loop over a whole sequence, three ways.

    python tools/bench_eval.py [--frames 1000] [--rounds 2] [--out FILE]

A synthetic 480x640 uint8 sequence of --frames frames (poses drawn from a seed), a bf16 MapNet (ResNet-34, droprate 0),
MF windows with steps=3, skip=10 (one window per frame, no_duplicates=False, as eval.py builds them), no pose-graph
optimisation.  The arms alternate within each of --rounds rounds; each is timed end to end with a host clock that ends in
a device synchronise, and the median round is reported:
  reference   -- eval.py's loop: MF-style windows from torch.utils.data.DataLoader(num_workers=5, batch_size=1) with
                 Pillow Resize(256) + torchvision ToTensor / Normalize, the live model's eval forward on each window,
                 its output copied to the host and qexp'd with numpy per pose;
  tuples      -- inference.evaluate_tuples(Predictor) on windows [L,3,3,256,341] built once on the host beforehand
                 (pinned memory; the build is not timed);
  sequence    -- inference.evaluate_sequence(Predictor, DeviceDataset): each distinct frame through the engine once,
                 the windows rebuilt on the device (the cache is filled once beforehand; ingest_s is that fill).
Frames/s is sequence frames (one window each) per second.  cnn_frames counts the frames each arm pushes through the
network (counted, not timed).  The card's name, power limit and clocks are read in the same run.  Prints one JSON line
(and writes it to --out).  No CPU fallback.
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

from bench_infer import card   # noqa: E402

STEPS, SKIP, H_IN, W_IN = 3, 10, 480, 640
STATS = ([0.45, 0.5, 0.55], [0.22, 0.25, 0.2])


class _RefMF(object):
    """composite.py MF.__getitem__ without VOs over a frame array, with scripts/eval.py's transforms"""

    def __init__(self, fr, poses):
        import torchvision.transforms as T
        self.fr, self.poses = fr, poses
        self.tf = T.Compose([T.Resize(256), T.ToTensor(), T.Normalize(mean=STATS[0], std=STATS[1])])

    def __len__(self):
        return self.fr.shape[0]

    def __getitem__(self, i):
        import torch
        from PIL import Image
        from geomapnet_b200.data import tuples
        idx = tuples.mf_indices(i, self.fr.shape[0], STEPS, SKIP)
        return (torch.stack([self.tf(Image.fromarray(self.fr[j])) for j in idx]),
                torch.from_numpy(self.poses[idx]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_eval.json"))
    args = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    from geomapnet_b200.data import DeviceDataset
    from geomapnet_b200.inference import Predictor, evaluate_sequence, evaluate_tuples
    from geomapnet_b200.models.posenet import PoseNet, MapNet
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval needs a CUDA device")
    torch.cuda.set_device(0)
    L = args.frames
    rng = np.random.default_rng(0)
    fr = (rng.random((L, H_IN, W_IN, 3)) * 256).astype(np.uint8)
    v = rng.standard_normal((L, 3)) * 0.3
    poses = np.concatenate([rng.standard_normal((L, 3)).cumsum(0), v], 1).astype(np.float32)
    torch.manual_seed(0)
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False, precision="bf16")
    model = MapNet(net).cuda().eval()
    pr = Predictor(model, max_batch=64)
    counts = {"reference": 0, "tuples": 0, "sequence": 0}
    run0 = pr._run

    def counted_run(xb):
        counts[arm_now[0]] += xb.shape[0]
        return run0(xb)
    pr._run = counted_run
    arm_now = [None]

    # the device cache (untimed fill)
    t0 = time.perf_counter()
    ds = DeviceDataset(fr, STATS[0], STATS[1], poses=poses, steps=STEPS, skip=SKIP, max_batch=64)
    ingest_s = time.perf_counter() - t0
    asm0 = ds.assemble_frames

    def counted_asm(frames, x_out):
        counts["sequence"] += len(frames)
        return asm0(frames, x_out)
    ds.assemble_frames = counted_asm
    # the host windows of the tuples arm (untimed build, pinned)
    ref_ds = _RefMF(fr, poses)
    t0 = time.perf_counter()
    dl = torch.utils.data.DataLoader(ref_ds, batch_size=16, shuffle=False, num_workers=5)
    xs, ts = zip(*[(x, t) for x, t in dl])
    x_host = torch.cat(xs).pin_memory()
    targ_host = torch.cat(ts)
    del xs, ts
    build_s = time.perf_counter() - t0

    def arm_reference():
        loader = torch.utils.data.DataLoader(ref_ds, batch_size=1, shuffle=False, num_workers=5, pin_memory=True)
        out = np.zeros((L, 7))
        with torch.no_grad():
            for i, (data, target) in enumerate(loader):
                o = model(data.cuda(non_blocking=True))
                counts["reference"] += o.shape[0] * o.shape[1]
                o = o.cpu().numpy().reshape(-1, 6)
                q = [np.hstack((np.cos(np.linalg.norm(p[3:])), np.sinc(np.linalg.norm(p[3:]) / np.pi) * p[3:]))
                     for p in o]
                out[i] = np.hstack((o[:, :3], np.asarray(q)))[STEPS // 2]
        return out

    def arm_tuples():
        return evaluate_tuples(pr, x_host, targ_host)

    def arm_sequence():
        return evaluate_sequence(pr, ds)

    arms = (("reference", arm_reference), ("tuples", arm_tuples), ("sequence", arm_sequence))
    for name, fn in arms:                   # warm-up: graphs, worker start-up paths, the engine's plans
        if name != "reference":
            arm_now[0] = name
            fn()
    torch.cuda.synchronize()
    for k in counts:
        counts[k] = 0
    times = {name: [] for name, _ in arms}
    results = {}
    for _ in range(args.rounds):
        for name, fn in arms:
            arm_now[0] = name
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            results[name] = fn()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
    a, b = results["tuples"], results["sequence"]
    same = all(torch.equal(a[k], b[k]) for k in ("pred7", "targ7", "t_err", "q_err"))
    ref_mid = torch.as_tensor(results["reference"])
    res = {"bench": "eval", "card": card(), "frame_hw": [H_IN, W_IN], "input_hw": [ds.Ho, ds.Wo], "frames": L,
           "model": "mapnet resnet34 bf16 droprate 0", "steps": STEPS, "skip": SKIP, "pgo": False,
           "rounds": args.rounds, "ingest_s": round(ingest_s, 2), "host_window_build_s": round(build_s, 2),
           "unique_frames": int(b["n_frames"]), "tuples_equal_sequence": bool(same),
           "reference_vs_sequence_pred7_max_abs": float((ref_mid - b["pred7"].cpu()).abs().max())}
    for name, _ in arms:
        med = statistics.median(times[name])
        res[name] = {"s": round(med, 3), "frames_per_s": round(L / med, 1),
                     "cnn_frames": counts[name] // args.rounds, "rounds_s": [round(t, 3) for t in times[name]]}
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
