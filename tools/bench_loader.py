"""Training from a device-resident dataset on the H100: what the input side costs the graphed training step.

    python tools/bench_loader.py [--frames 1630] [--rounds 3] [--ref-batches 6] [--out FILE]

Synthetic seeded 7Scenes-size frames (480x640 RGB uint8 -> Resize(256) -> 256x341), ColorJitter 0.7 with hue 0.5 as
in the reference configs, bf16 trunk.  Workloads: posenet batch 64; MapNet steps 3, skip 10, batch 32 (96 frames per
step); MFOnline steps 5, skip 10, batch 16 (160 frames).  The frame count leaves a partial last batch.  Arms, alternated
in `--rounds` rounds (median reported):
  * fixed  -- GraphedTrainStep replayed on one batch already in its static buffers (the step alone);
  * epoch  -- geomapnet_b200.graph.train_epoch over a DeviceLoader: a full epoch, last partial batch included, each
              batch assembled on the GPU while the previous step's optimizer graph runs;
  * torch_dataloader (posenet only) -- the reference's input side: torch.utils.data.DataLoader(num_workers=5) with
              Pillow Resize / ColorJitter and torchvision ToTensor / Normalize, each batch copied into the same graphed
              step; `--ref-batches` batches after two warm-up batches.
Also the assembly kernel alone (CUDA events over 50 calls of a full batch) and its algorithmic bytes per batch (uint8
frames read, twice with ColorJitter, float32 NCHW written) over the 3.35 TB/s HBM3 data-sheet bandwidth.  The card's
name, power limit and the host CPU count are read in the same run.  Prints one JSON line (and writes it to --out).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet
CJ = 0.7


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "host_cpus": os.cpu_count()}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        out["nvidia_smi"] = r.stdout.strip()
    except Exception as e:          # the query is informative only
        out["nvidia_smi"] = "unavailable (%s)" % e
    return out


def frames(L, seed):
    import numpy as np
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (8, 480, 640, 3), dtype=np.uint8)
    out = np.empty((L, 480, 640, 3), np.uint8)
    for i in range(L):                  # smooth drift over a few textures: cheap to generate, not constant
        out[i] = np.roll(base[i % 8], i, axis=1)
    poses = rng.standard_normal((L, 6)).astype(np.float32) * 0.3
    return out, poses


class _RefSet(object):
    """scripts/train.py's transform stack on uint8 frames (posenet layout), for torch.utils.data.DataLoader."""

    def __init__(self, fr, poses, stats):
        import torchvision.transforms as T
        self.fr, self.poses = fr, poses
        self.tf = T.Compose([T.Resize(256), T.ColorJitter(brightness=CJ, contrast=CJ, saturation=CJ, hue=0.5),
                             T.ToTensor(), T.Normalize(mean=stats[0], std=stats[1])])

    def __len__(self):
        return self.fr.shape[0]

    def __getitem__(self, i):
        import torch
        from PIL import Image
        return self.tf(Image.fromarray(self.fr[i])), torch.from_numpy(self.poses[i])


def workload(kind, fr, poses, vfr, vposes, args, out):
    import numpy as np
    import torch
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet, MapNet
    from geomapnet_b200.common import criterion as C
    from geomapnet_b200.common.optimizer import Optimizer
    from geomapnet_b200.data import DeviceDataset, DeviceLoader
    from geomapnet_b200.graph import GraphedTrainStep, train_epoch
    stats = ([0.5, 0.45, 0.4], [0.25, 0.24, 0.26])
    if kind == "posenet":
        bs, kw = 64, dict()
    elif kind == "mapnet":
        bs, kw = 32, dict(steps=3, skip=10)
    else:
        bs, kw = 16, dict(steps=5, skip=10, online=True, val_frames=vfr, val_poses=vposes)
    torch.manual_seed(0)
    np.random.seed(0)
    t0 = time.time()
    ds = DeviceDataset(fr, stats[0], stats[1], poses=poses, color_jitter=CJ, max_batch=bs, **kw)
    torch.cuda.synchronize()
    ingest_s = time.time() - t0
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False)
    model = (net if kind == "posenet" else MapNet(net)).cuda()
    sv = dict(sax=0.0, saq=-3.0, learn_beta=True)
    if kind == "posenet":
        crit = C.PoseNetCriterion(**sv)
    elif kind == "mapnet":
        crit = C.MapNetCriterion(srx=0.0, srq=-3.0, learn_gamma=True, **sv)
    else:
        crit = C.MapNetOnlineCriterion(srx=0.0, srq=-3.0, learn_gamma=True, **sv)
    crit = crit.cuda()
    opt = Optimizer([{"params": model.parameters()}, {"params": list(crit.parameters())}], "adam", 1e-4, 5e-4)
    model.train()
    loader = DeviceLoader(ds, bs, shuffle=True)
    nsteps = len(loader)
    frames_per_step = bs * ds.frames_per_item
    total_frames = len(ds) * ds.frames_per_item
    steps = {}
    train_epoch(loader, model, crit, opt, steps=steps)          # captures + warm-up epoch
    fixed = steps[bs]
    # assembly kernel alone: a full batch, CUDA events
    batch = ds.example(bs)
    jit = next(loader.batches())[1]                             # real ColorJitter records of one batch
    batch = (batch[0], jit, batch[2], batch[3])
    xs, ts = ds.batch_shapes(bs)
    xb, tb = torch.empty(xs, device="cuda"), torch.empty(ts, device="cuda")
    for _ in range(5):
        ds.assemble(batch, xb, tb)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        ds.assemble(batch, xb, tb)
    e1.record()
    torch.cuda.synchronize()
    asm_ms = e0.elapsed_time(e1) / 50
    npix = ds.Ho * ds.Wo
    nimg = frames_per_step
    asm_bytes = nimg * (npix * 3 * 2 + npix * 3 * 4) + tb.numel() * 4
    ref = None
    if kind == "posenet" and args.ref_batches > 0:
        ref = torch.utils.data.DataLoader(_RefSet(fr, poses, stats), batch_size=bs, shuffle=True, num_workers=5,
                                          pin_memory=True)
    arms = {"fixed_ms_per_step": [], "epoch_ms_per_step": [], "epoch_img_per_s": []}
    if ref is not None:
        arms["torch_dataloader_ms_per_step"] = []
    for _ in range(args.rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(nsteps):
            fixed.replay()
        torch.cuda.synchronize()
        arms["fixed_ms_per_step"].append((time.perf_counter() - t0) * 1e3 / nsteps)
        t0 = time.perf_counter()
        losses = train_epoch(loader, model, crit, opt, steps=steps)
        dt = time.perf_counter() - t0
        assert len(losses) == nsteps and all(v == v for v in losses)
        arms["epoch_ms_per_step"].append(dt * 1e3 / nsteps)
        arms["epoch_img_per_s"].append(total_frames / dt)
        if ref is not None:
            it = iter(ref)
            for _ in range(2):
                x, t = next(it)
                fixed(x.cuda(non_blocking=True), t.cuda(non_blocking=True))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.ref_batches):
                x, t = next(it)
                fixed(x.cuda(non_blocking=True), t.cuda(non_blocking=True))
            torch.cuda.synchronize()
            arms["torch_dataloader_ms_per_step"].append((time.perf_counter() - t0) * 1e3 / args.ref_batches)
            del it
    res = {k: round(statistics.median(v), 3) for k, v in arms.items()}
    res.update(batch=bs, frames_per_step=frames_per_step, steps_per_epoch=nsteps, items=len(ds),
               last_batch=len(ds) % bs, frames_in_cache=ds.L + ds.Lv, cache_mb=round((ds.L + ds.Lv) * npix * 3 / 1e6, 1),
               ingest_s=round(ingest_s, 2), input_hw=[ds.Ho, ds.Wo],
               fixed_img_per_s=round(frames_per_step / res["fixed_ms_per_step"] * 1e3, 1),
               epoch_over_fixed=round(res["epoch_ms_per_step"] / res["fixed_ms_per_step"], 4),
               assemble_ms=round(asm_ms, 4), assemble_mb_per_batch=round(asm_bytes / 1e6, 2),
               assemble_frac_of_hbm_peak=round(asm_bytes / (asm_ms * 1e-3) / HBM_BYTES_PER_S, 3),
               rounds={k: [round(x, 3) for x in v] for k, v in arms.items()})
    if ref is not None:
        res["torch_dataloader_img_per_s"] = round(bs / res["torch_dataloader_ms_per_step"] * 1e3, 1)
    out[kind] = res
    del steps, fixed, loader
    ds.close()
    torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1630)
    ap.add_argument("--val-frames", type=int, default=400)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ref-batches", type=int, default=6)
    ap.add_argument("--workloads", default="posenet,mapnet,online")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_loader: no CUDA device (there is no CPU fallback)")
    fr, poses = frames(args.frames, 1)
    vfr, vposes = frames(args.val_frames, 2)
    out = {"bench": "loader", "card": card(), "frame_hw": [480, 640], "color_jitter": CJ, "precision": "bf16"}
    for kind in args.workloads.split(","):
        workload(kind, fr, poses, vfr, vposes, args, out)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
