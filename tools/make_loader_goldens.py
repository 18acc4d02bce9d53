"""Regenerate tests/golden/loader.npz from the reference (build container only: needs the reference tree).

    python tools/make_loader_goldens.py

* ``calc_vos_safe``: the reference's common/pose_utils.py:276-288 on seeded pose tuples (the VO targets of MFOnline's
  validation half).
* The host-side stream of ``DataLoader(MF(...), batch_size, shuffle=True, num_workers=0)`` under fixed torch / numpy
  seeds: item order, ``variable_skip`` gaps and the ColorJitter parameters each frame's transform draws.  MF is driven
  by the reference's own ``get_indices`` source (oracle.make_goldens._reference_mf_get_indices) and its __getitem__
  order (dataset_loaders/composite.py:77-97: indices, then one transform per frame); each frame goes through the real
  torchvision ColorJitter of scripts/train.py:121-124, whose ``get_params`` result is recorded.
"""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from oracle.make_goldens import _reference_mf_get_indices  # noqa: E402

# MF stream: 23 frames, steps 3, skip 4, variable_skip, batch 5 (last batch partial), color_jitter 0.7
STREAM = dict(L=23, steps=3, skip=4, batch=5, cj=0.7, torch_seed=1234, np_seed=77, epochs=2)


def vos_golden(out):
    pu = ref_loader.load().pose_utils
    g = torch.Generator().manual_seed(5)
    N, T = 16, 5
    t = torch.randn(N, T, 3, generator=g)
    v = torch.randn(N, T, 3, generator=g)
    v = v / v.norm(dim=2, keepdim=True) * ((torch.rand(N, T, 1, generator=g) - 0.5) * math.pi)
    poses = torch.cat([t, v], 2).float()
    poses[0, 1, 3:] = 0                       # a zero rotation (qexp at the origin)
    poses[1, 2] = poses[1, 1]                 # two equal poses (zero VO, qlog of the identity)
    out["vos_poses"] = poses.numpy()
    out["vos_safe"] = pu.calc_vos_safe(poses).numpy()


def stream_golden(out):
    import torchvision.transforms as TV
    from PIL import Image
    ref_get_indices = _reference_mf_get_indices()
    rec = {"items": [], "frames": [], "jitter": []}
    cj = STREAM["cj"]
    jitter = TV.ColorJitter(brightness=cj, contrast=cj, saturation=cj, hue=0.5)
    orig = TV.ColorJitter.get_params

    def logged(*a, **k):
        r = orig(*a, **k)
        fn_idx, b, c, s, h = r
        rec["jitter"].append([float(fn_idx[i]) for i in range(4)] + [b, c, s, h])
        return r

    TV.ColorJitter.get_params = staticmethod(logged)
    img = Image.fromarray(np.zeros((4, 4, 3), np.uint8))

    class Frames(torch.utils.data.Dataset):
        def __len__(self):
            return STREAM["L"]

        def __getitem__(self, i):
            jitter(img)
            return torch.zeros(1), torch.zeros(6)

    class MF(torch.utils.data.Dataset):
        def __init__(self):
            self.steps, self.skip, self.variable_skip, self.no_duplicates = STREAM["steps"], STREAM["skip"], True, False
            self.dset = Frames()

        def get_indices(self, index):
            return ref_get_indices(self, index)

        def __getitem__(self, index):
            idx = self.get_indices(index)
            rec["items"].append(index)
            rec["frames"].append(list(idx))
            clip = [self.dset[i] for i in idx]
            return torch.stack([c[0] for c in clip]), torch.stack([c[1] for c in clip])

        def __len__(self):
            return len(self.dset)

    try:
        torch.manual_seed(STREAM["torch_seed"])
        np.random.seed(STREAM["np_seed"])
        dl = torch.utils.data.DataLoader(MF(), batch_size=STREAM["batch"], shuffle=True, num_workers=0)
        sizes = []
        for _ in range(STREAM["epochs"]):
            for x, _t in dl:
                sizes.append(x.shape[0])
    finally:
        TV.ColorJitter.get_params = orig
    for k, v in STREAM.items():
        out["stream_" + k] = np.array(v)
    out["stream_items"] = np.array(rec["items"], np.int64)
    out["stream_frames"] = np.array(rec["frames"], np.int64)
    out["stream_jitter"] = np.array(rec["jitter"], np.float64)
    out["stream_batch_sizes"] = np.array(sizes, np.int64)


def main():
    if not ref_loader.available():
        sys.exit("reference tree not available")
    out = {}
    vos_golden(out)
    stream_golden(out)
    path = os.path.join(ROOT, "tests", "golden", "loader.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %s" % (path, sorted(out)))


if __name__ == "__main__":
    main()
