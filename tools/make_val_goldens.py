"""Regenerate tests/golden/validate.npz from the reference (build container only: needs the reference tree).

    python tools/make_val_goldens.py

What the reference's validation loop (common/train.py:214-250) draws from its val_loader, ``DataLoader(val_set,
batch_size, shuffle, num_workers=0)`` over a single-frame set (SevenScenes / RobotCar: one frame per index) or
``MF(steps, skip, variable_skip)`` (MF driven by the reference's own ``get_indices`` source,
oracle.make_goldens._reference_mf_get_indices, in its __getitem__ order: indices, then one transform per frame):

* per case, the frames of every item in loader order, the batch sizes (the last one partial), and the torch and numpy
  RNG states the pass leaves behind.  Every frame goes through the real torchvision ColorJitter of
  scripts/train.py:121-124 when the case has one;
* Trainer.train_val's interleaving over two epochs (validation pass, then the training epoch, both MF with
  variable_skip and ColorJitter, shuffle on): the frames of every item and every frame's ColorJitter draw, in the
  order the reference consumes them.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from oracle.make_goldens import _reference_mf_get_indices  # noqa: E402

SEED_TORCH, SEED_NP = 4321, 99
# name: (frames, steps or None, skip, variable_skip, batch, shuffle, color_jitter)
CASES = {
    "posenet_shuffle": (23, None, 1, False, 5, True, 0.7),
    "posenet_ordered": (23, None, 1, False, 5, False, 0.0),
    "mf_vs_shuffle": (23, 3, 4, True, 5, True, 0.7),
    "mf_vs_ordered": (23, 3, 4, True, 5, False, 0.0),
    "mf_shuffle": (19, 3, 2, False, 4, True, 0.0),
}
# Trainer.train_val: (val frames, train frames, steps, skip, batch, color_jitter, epochs)
INTERLEAVE = (17, 23, 3, 4, 5, 0.7, 2)


def _datasets(rec):
    import torchvision.transforms as TV
    from PIL import Image
    ref_get_indices = _reference_mf_get_indices()
    img = Image.fromarray(np.zeros((4, 4, 3), np.uint8))

    class Frames(torch.utils.data.Dataset):
        """one frame per index, through the transform stack's ColorJitter when there is one"""
        def __init__(self, L, cj, tag):
            self.L, self.tag = L, tag
            self.jitter = TV.ColorJitter(brightness=cj, contrast=cj, saturation=cj, hue=0.5) if cj > 0 else None

        def __len__(self):
            return self.L

        def __getitem__(self, i):
            if self.jitter is not None:
                rec["tag"] = self.tag
                self.jitter(img)
            return torch.zeros(1), torch.zeros(6)

    class Single(Frames):
        def __getitem__(self, i):
            rec["items"].append((self.tag, [i]))
            return Frames.__getitem__(self, i)

    class MF(torch.utils.data.Dataset):
        def __init__(self, L, steps, skip, variable_skip, cj, tag):
            self.steps, self.skip, self.variable_skip, self.no_duplicates = steps, skip, variable_skip, False
            self.dset, self.tag = Frames(L, cj, tag), tag

        def get_indices(self, index):
            return ref_get_indices(self, index)

        def __getitem__(self, index):
            idx = self.get_indices(index)
            rec["items"].append((self.tag, [int(i) for i in idx]))
            clip = [self.dset[i] for i in idx]
            return torch.stack([c[0] for c in clip]), torch.stack([c[1] for c in clip])

        def __len__(self):
            return len(self.dset)

    def make(L, steps, skip, variable_skip, cj, tag):
        return Single(L, cj, tag) if steps is None else MF(L, steps, skip, variable_skip, cj, tag)
    return make


def main():
    if not ref_loader.available():
        sys.exit("reference tree not available")
    import torchvision.transforms as TV
    rec = {"items": [], "jitter": []}
    orig = TV.ColorJitter.get_params

    def logged(*a, **k):
        r = orig(*a, **k)
        fn_idx, b, c, s, h = r
        rec["jitter"].append([rec["tag"]] + [float(fn_idx[i]) for i in range(4)] + [b, c, s, h])
        return r

    TV.ColorJitter.get_params = staticmethod(logged)
    make = _datasets(rec)
    out = {"seed_torch": np.array(SEED_TORCH), "seed_np": np.array(SEED_NP)}
    try:
        for name, (L, steps, skip, vs, bs, shuffle, cj) in CASES.items():
            rec["items"], rec["jitter"] = [], []
            torch.manual_seed(SEED_TORCH)
            np.random.seed(SEED_NP)
            dl = torch.utils.data.DataLoader(make(L, steps, skip, vs, cj, 0), batch_size=bs, shuffle=shuffle,
                                             num_workers=0)
            sizes = [x.shape[0] for x, _ in dl]
            st = np.random.get_state()
            out[name + "_case"] = np.array([L, -1 if steps is None else steps, skip, int(vs), bs, int(shuffle)])
            out[name + "_cj"] = np.array(cj)
            out[name + "_frames"] = np.array([f for _, f in rec["items"]], np.int64)
            out[name + "_sizes"] = np.array(sizes, np.int64)
            out[name + "_torch_state"] = torch.get_rng_state().numpy()
            out[name + "_np_mt"] = np.asarray(st[1])
            out[name + "_np_pos"] = np.array(st[2])
        # common/train.py:212-300: per epoch the validation pass (epoch % val_freq == 0, val_freq 1), then the epoch
        Lv, Lt, steps, skip, bs, cj, epochs = INTERLEAVE
        rec["items"], rec["jitter"] = [], []
        torch.manual_seed(SEED_TORCH)
        np.random.seed(SEED_NP)
        val = torch.utils.data.DataLoader(make(Lv, steps, skip, True, cj, 0), batch_size=bs, shuffle=True, num_workers=0)
        train = torch.utils.data.DataLoader(make(Lt, steps, skip, True, cj, 1), batch_size=bs, shuffle=True,
                                            num_workers=0)
        for _ in range(epochs):
            for _b in val:
                pass
            for _b in train:
                pass
        out["interleave_case"] = np.array(INTERLEAVE[:5] + (INTERLEAVE[6],))
        out["interleave_cj"] = np.array(cj)
        out["interleave_tags"] = np.array([t for t, _ in rec["items"]], np.int64)
        out["interleave_frames"] = np.array([f for _, f in rec["items"]], np.int64)
        out["interleave_jitter"] = np.array(rec["jitter"], np.float64)
    finally:
        TV.ColorJitter.get_params = orig
    path = os.path.join(ROOT, "tests", "golden", "validate.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %s" % (path, sorted(out)))


if __name__ == "__main__":
    main()
