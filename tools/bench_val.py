"""Validation-pass throughput on the H100: the val pass of Trainer.train_val (common/train.py:214-250) as mapnet.ini runs
it (do_val = yes, batch_size 20, shuffle, dropout 0.5, color_jitter 0.7 -- the val set uses the training transform),
four ways.

    python tools/bench_val.py [--frames 2000] [--rounds 5] [--ref-batches 20] [--out FILE]

A synthetic 480x640 uint8 sequence of --frames frames (poses drawn from a seed), MF(steps=3, skip=10) items, one per
frame, batch 20, shuffle on, MapNetCriterion() (all four sigma 0), a bf16 MapNet (ResNet-34).  The arms alternate within
each of --rounds rounds; each is timed end to end with a host clock that ends in a device synchronise, and the median
round is reported:
  validate_unique  -- inference.validate(Predictor) with droprate 0 and no ColorJitter: each distinct frame of the pass
                      through the engine once, all batch losses in one launch;
  validate_batches -- inference.validate(Predictor) with droprate 0.5 and ColorJitter 0.7: each jittered batch
                      assembled straight into a graph input and run on its own;
  loop_device      -- the reference's loop restated (step_feedfwd(train=False): the live model's eval forward, the
                      criterion, loss.item() per batch) on DeviceLoader batches, the settings of validate_batches;
  loop_reference   -- the same loop fed by DataLoader(num_workers=5, pin_memory=True) with Pillow Resize(256) +
                      torchvision ColorJitter / ToTensor / Normalize, as tools/bench_eval.py restates the reference.
                      It runs the first --ref-batches batches of the pass only (Pillow is slow); its rate is over those.
Frames/s is items (one window of 3 frames each) per second.  cnn_frames counts the frames each arm pushes through the
network in one pass (counted, not timed).  The card's name, power limit and clocks are read in the same run.  Prints one
JSON line (and writes it to --out).  No CPU fallback.
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

STEPS, SKIP, H_IN, W_IN, BATCH, CJ, DROP = 3, 10, 480, 640, 20, 0.7, 0.5
STATS = ([0.45, 0.5, 0.55], [0.22, 0.25, 0.2])


class _RefMF(object):
    """composite.py MF.__getitem__ without VOs over a frame array, with scripts/train.py's transforms"""

    def __init__(self, fr, poses):
        import torchvision.transforms as T
        self.fr, self.poses = fr, poses
        self.tf = T.Compose([T.Resize(256), T.ColorJitter(brightness=CJ, contrast=CJ, saturation=CJ, hue=0.5),
                             T.ToTensor(), T.Normalize(mean=STATS[0], std=STATS[1])])

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
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ref-batches", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_val.json"))
    args = ap.parse_args()
    import numpy as np
    import torch
    import torchvision
    from geomapnet_b200.common.criterion import MapNetCriterion
    from geomapnet_b200.data import DeviceDataset, DeviceLoader
    from geomapnet_b200.inference import Predictor, validate
    from geomapnet_b200.models.posenet import PoseNet, MapNet
    if not torch.cuda.is_available():
        raise SystemExit("bench_val needs a CUDA device")
    torch.cuda.set_device(0)
    L = args.frames
    rng = np.random.default_rng(0)
    fr = rng.integers(0, 256, (L, H_IN, W_IN, 3), dtype=np.uint8)
    v = rng.standard_normal((L, 3)) * 0.3
    poses = np.concatenate([rng.standard_normal((L, 3)).cumsum(0), v], 1).astype(np.float32)
    torch.manual_seed(0)
    models = {}
    for drop in (0.0, DROP):
        net = PoseNet(torchvision.models.resnet34(weights=None), droprate=drop, pretrained=False, precision="bf16")
        if drop:
            net.load_state_dict(models[0.0].mapnet.state_dict())
        models[drop] = MapNet(net).cuda()
    crit = MapNetCriterion().cuda()
    counts = {}
    arm_now = [None]
    prs = {drop: Predictor(m, max_batch=64) for drop, m in models.items()}
    t0 = time.perf_counter()
    ds_plain = DeviceDataset(fr, STATS[0], STATS[1], poses=poses, steps=STEPS, skip=SKIP, max_batch=BATCH)
    ds_jit = DeviceDataset(fr, STATS[0], STATS[1], poses=poses, steps=STEPS, skip=SKIP, max_batch=BATCH, color_jitter=CJ)
    ingest_s = time.perf_counter() - t0
    for ds in (ds_plain, ds_jit):
        asm0, asmb0 = ds.assemble_frames, ds.assemble

        def counted_asm(frames, x_out, asm0=asm0):
            counts[arm_now[0]] = counts.get(arm_now[0], 0) + len(frames)
            return asm0(frames, x_out)

        def counted_asmb(batch, x_out, targ_out, asmb0=asmb0):
            counts[arm_now[0]] = counts.get(arm_now[0], 0) + len(batch[0])
            return asmb0(batch, x_out, targ_out)
        ds.assemble_frames, ds.assemble = counted_asm, counted_asmb
    loader_plain, loader_jit = DeviceLoader(ds_plain, BATCH, shuffle=True), DeviceLoader(ds_jit, BATCH, shuffle=True)
    ref_ds = _RefMF(fr, poses)
    live = models[DROP]
    n_ref = min(args.ref_batches * BATCH, L)

    def arm_validate_unique():
        return validate(prs[0.0], loader_plain, crit)[0]

    def arm_validate_batches():
        return validate(prs[DROP], loader_jit, crit)[0]

    def loop(batches):
        live.eval()
        losses = []
        with torch.no_grad():
            for data, target in batches:
                out = live(data.cuda(non_blocking=True))
                if arm_now[0] == "loop_reference":          # the device arms count their assembled frames
                    counts[arm_now[0]] = counts.get(arm_now[0], 0) + out.shape[0] * out.shape[1]
                losses.append(crit(out, target.cuda(non_blocking=True)).item())
        live.train()
        return sum(losses) / len(losses)

    def arm_loop_device():
        return loop(loader_jit)

    def arm_loop_reference():
        sub = torch.utils.data.Subset(ref_ds, range(n_ref))
        return loop(torch.utils.data.DataLoader(sub, batch_size=BATCH, shuffle=True, num_workers=5, pin_memory=True))

    arms = (("validate_unique", arm_validate_unique), ("validate_batches", arm_validate_batches),
            ("loop_device", arm_loop_device), ("loop_reference", arm_loop_reference))
    for name, fn in arms[:3]:               # warm-up: graphs, the engines' plans, the live trunk's arena
        arm_now[0] = name
        fn()
    torch.cuda.synchronize()
    counts.clear()
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
    items = {"validate_unique": L, "validate_batches": L, "loop_device": L, "loop_reference": n_ref}
    res = {"bench": "val", "card": card(), "frame_hw": [H_IN, W_IN], "input_hw": [ds_plain.Ho, ds_plain.Wo],
           "frames": L, "model": "mapnet resnet34 bf16", "steps": STEPS, "skip": SKIP, "batch": BATCH,
           "criterion": "MapNetCriterion() (sigmas 0)", "rounds": args.rounds, "ingest_s": round(ingest_s, 2),
           "val_loss": {k: round(v, 6) for k, v in results.items()}}
    for name, _ in arms:
        med = statistics.median(times[name])
        res[name] = {"items": items[name], "s": round(med, 3), "frames_per_s": round(items[name] / med, 1),
                     "cnn_frames": counts.get(name, 0) // args.rounds, "rounds_s": [round(t, 3) for t in times[name]]}
    res["validate_unique"]["settings"] = "droprate 0, no ColorJitter"
    for name in ("validate_batches", "loop_device", "loop_reference"):
        res[name]["settings"] = "droprate %.1f, ColorJitter %.1f" % (DROP, CJ)
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
