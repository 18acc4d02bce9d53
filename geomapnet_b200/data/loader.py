"""Training from a device-resident dataset: frames resized once into HBM, every batch assembled on the GPU.

The reference builds each batch with ``DataLoader(dataset, batch_size, shuffle, num_workers)`` (common/train.py:180-188)
and a per-image Pillow / torchvision transform stack (scripts/train.py:119-128).  Here:

* ``DeviceDataset`` keeps the ``Resize(256)`` output of every frame in device memory (the resize is deterministic and
  comes before ColorJitter, so caching it changes no value) with the pose table next to it, in the three layouts
  scripts/train.py builds: single frames (posenet: SevenScenes / RobotCar), ``MF(steps, skip, variable_skip)`` and
  ``MFOnline(gps_mode)`` (dataset_loaders/composite.py);
* ``DeviceLoader`` draws what the reference's ``DataLoader(dataset, batch_size, shuffle, num_workers=0)`` draws, in the
  same order -- the RandomSampler permutation from the global torch RNG, per item in sampler order the np.random gaps
  of ``variable_skip``, per frame in load order (MFOnline: training frames, then validation frames) one ColorJitter
  draw -- and keeps the last partial batch.  The order of ``num_workers > 0`` (per-worker RNG streams) is not
  reproduced;
* each batch is one kernel launch (two with ColorJitter) that gathers the frames, applies the jitter, ToTensor and
  Normalize, writes float32 NCHW into a given buffer and gathers the targets (MFOnline's validation VOs are computed
  on the device, calc_vos_safe).  Results are bit-identical to Pillow + torchvision on the CPU
  (tests/test_gpu_loader.py).
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from . import tuples
from .preprocess import ColorJitterSampler, resize_output_size

__all__ = ["ItemLayout", "DeviceDataset", "DeviceLoader", "host_batches"]


def _frames_and_poses(src, poses):
    """uint8 [L,H,W,3] array / tensor + poses, or a reference-style dataset built with transform=None whose
    __getitem__ returns (decoded PIL image, target): each frame is decoded once."""
    if torch.is_tensor(src) or isinstance(src, np.ndarray):
        return src, poses
    imgs, ps = [], []
    for i in range(len(src)):
        img, p = src[i]
        imgs.append(np.asarray(img, dtype=np.uint8))
        ps.append(np.asarray(p, dtype=np.float32).reshape(6))
    return np.stack(imgs), (np.stack(ps) if poses is None else poses)


class ItemLayout(object):
    """The host side of the three dataset layouts: item count, the frames and target rows of an item, the random
    draws the reference makes for it.  Needs no GPU; DeviceDataset adds the device cache."""

    def __init__(self, n_frames, steps=None, skip=1, variable_skip=False, online=False, n_val_frames=0, gps_mode=False,
                 color_jitter=0.0):
        self.steps, self.skip, self.variable_skip = steps, int(skip), bool(variable_skip)
        self.online, self.gps_mode = bool(online), bool(gps_mode)
        self.L, self.Lv = int(n_frames), (int(n_val_frames) if online else 0)
        if online and steps is None:
            raise ValueError("MFOnline needs steps")
        if steps is not None and (int(steps) < 1 or self.skip < 1):
            raise ValueError("steps and skip must be >= 1")
        if len(self) < 1:
            raise ValueError("the dataset has no items")
        cj = float(color_jitter)
        self.jitter = ColorJitterSampler(cj, cj, cj, 0.5) if cj > 0 else None
        self.frames_per_item = 1 if steps is None else (2 * steps if online else steps)
        self.targ_per_item = 1 if steps is None else (steps if not online else
                                                      (2 * steps if gps_mode else 2 * steps - 1))

    # ------------------------------------------------------- host-side items
    def __len__(self):
        if self.steps is None:
            return self.L
        if self.online:
            return tuples.mfonline_len(self.Lv, self.steps, self.skip)
        return tuples.mf_len(self.L, self.steps, self.skip)

    def item(self, index):
        """The host part of the reference's __getitem__(index), with its random draws in the same order:
        -> (cache frame numbers int32 [F], ColorJitter records uint8 [F,32] or None, target rows int32 [R,2])."""
        index = int(index)
        if not 0 <= index < len(self):
            raise IndexError("item %d outside [0, %d)" % (index, len(self)))
        if self.steps is None:
            fr = np.array([index], dtype=np.int64)
            rows = np.array([[index, -1]])
            jit = self.jitter.sample(1) if self.jitter is not None else None
            return fr.astype(np.int32), jit, rows.astype(np.int32)
        T = self.steps
        if not self.online:
            fr = tuples.mf_indices(index, self.L, T, self.skip, False, self.variable_skip)
            jit = self.jitter.sample(T) if self.jitter is not None else None
            rows = np.stack([fr, -np.ones_like(fr)], 1)
            return fr.astype(np.int32), jit, rows.astype(np.int32)
        # MFOnline (composite.py:117-126): training tuple (np gaps, then its frames' jitter), then validation tuple
        tr = tuples.mf_indices(index % tuples.mf_len(self.L, T, self.skip, False), self.L, T, self.skip, False,
                               self.variable_skip)
        jt = self.jitter.sample(T) if self.jitter is not None else None
        va = tuples.mf_indices(index % tuples.mf_len(self.Lv, T, self.skip, True), self.Lv, T, self.skip, True,
                               self.variable_skip) + self.L
        jv = self.jitter.sample(T) if self.jitter is not None else None
        rows = [[f, -1] for f in tr]
        if self.gps_mode:
            rows += [[f, -1] for f in va]                                  # real absolute poses
        else:
            rows += [[va[i], va[i + 1]] for i in range(T - 1)]             # calc_vos_safe of the real poses
        jit = torch.cat([jt, jv]) if jt is not None else None
        return np.concatenate([tr, va]).astype(np.int32), jit, np.asarray(rows, dtype=np.int32)

    def collate(self, items):
        """A list of item() results -> one batch record (frame numbers, jitter records, target rows, N)."""
        fr = np.ascontiguousarray(np.concatenate([it[0] for it in items]), dtype=np.int32)
        jit = None
        if self.jitter is not None:
            jit = np.ascontiguousarray(torch.cat([it[1] for it in items]).numpy())
        rows = np.ascontiguousarray(np.concatenate([it[2] for it in items]), dtype=np.int32)
        return fr, jit, rows, len(items)

    def eval_tables(self, unique=True, vo_fc=False):
        """The windows scripts/eval.py evaluates: one per item, in index order, as DataLoader(shuffle=False) draws them
        (with variable_skip, np.random is consumed as in the reference's loop).  Returns host int32 tables:
          windows [L,T]   the frame of every window slot (T = 1 for single frames);
          frames [F]      the frames that go through the network, in that order;
          slots [L,T]     the row of `frames` whose prediction fills each window slot;
          vo_rows [L,E,2] the frame pairs of each window's VOs: consecutive slots (calc_vos_safe, E = T-1) or every
                          pair i<j in row-major order (vo_fc: calc_vos_safe_fc, E = T(T-1)/2).
        unique=True: every distinct frame once, in frame order.  unique=False: every window's frames in window order
        (frames = windows.ravel()), what a network that draws dropout masks at eval needs to see."""
        if self.online or self.jitter is not None:
            raise ValueError("evaluation windows need a single-frame or MF layout without ColorJitter")
        windows = np.stack([self.item(i)[0] for i in range(len(self))]).astype(np.int32)
        L, T = windows.shape
        if unique:
            frames, inv = np.unique(windows, return_inverse=True)
            slots = inv.reshape(L, T)
        else:
            frames, slots = windows.reshape(-1), np.arange(L * T).reshape(L, T)
        pairs = [(i, j) for i in range(T) for j in range(i + 1, T)] if vo_fc else [(i, i + 1) for i in range(T - 1)]
        pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
        vo_rows = windows[:, pairs] if len(pairs) else np.zeros((L, 0, 2), np.int32)
        return dict(windows=windows, frames=np.ascontiguousarray(frames, dtype=np.int32),
                    slots=np.ascontiguousarray(slots, dtype=np.int32), vo_rows=np.ascontiguousarray(vo_rows, dtype=np.int32))

    def val_tables(self, batch_size, shuffle=True, unique=True):
        """One validation pass (common/train.py:214-250) as DataLoader(dataset, batch_size, shuffle, num_workers=0) draws
        it: the batch records of host_batches, drawn in full (the global torch and numpy RNG streams advance as in the
        reference's loop), and host int32 tables over the items of the pass in loader order:
          batch_items [n_batches+1]  item offset of each batch (the last batch may be partial);
          targ_rows [I,T]            the pose row of every window slot (T = 1 for single frames);
          frames [F]                 the frames that go through the network, in that order;
          pred_rows [I,T]            the row of `frames` whose prediction fills each window slot.
        unique=True: every distinct frame of the pass once, in frame order.  unique=False: every item's frames in loader
        order (pred_rows is the identity), what a forward that draws dropout masks or a jittered batch needs."""
        if self.online:
            raise ValueError("validation passes need a single-frame or MF layout (MFOnline never validates)")
        batches = list(host_batches(self, batch_size, shuffle))
        T = self.frames_per_item
        items = np.cumsum([0] + [b[3] for b in batches]).astype(np.int32)
        fr = np.concatenate([b[0] for b in batches]).astype(np.int32)
        targ = np.concatenate([b[2][:, 0] for b in batches]).astype(np.int32).reshape(-1, T)
        if unique:
            frames, inv = np.unique(fr, return_inverse=True)
        else:
            frames, inv = fr, np.arange(fr.shape[0])
        return dict(batches=batches, batch_items=items, targ_rows=np.ascontiguousarray(targ),
                    frames=np.ascontiguousarray(frames, dtype=np.int32),
                    pred_rows=np.ascontiguousarray(inv.reshape(-1, T), dtype=np.int32))

    def example(self, n):
        """A batch record of items 0, 1, ... (n of them) that makes no random draw (fixed skips, no ColorJitter): an
        input for warm-up and capture that leaves the RNG streams where the reference's loop has them."""
        jit, vs = self.jitter, self.variable_skip
        self.jitter, self.variable_skip = None, False
        try:
            return self.collate([self.item(i % len(self)) for i in range(n)])
        finally:
            self.jitter, self.variable_skip = jit, vs


class DeviceDataset(ItemLayout):
    def __init__(self, frames, mean, std, poses=None, color_jitter=0.0, steps=None, skip=1, variable_skip=False,
                 online=False, val_frames=None, val_poses=None, gps_mode=False, size=256, max_batch=64, chunk=64,
                 device=None, vo_poses=None):
        """frames: uint8 [L,H,W,3] (RGB, numpy or torch) or a reference-style dataset (see _frames_and_poses); poses:
        [L,6] float32 targets.  mean / std: as handed to transforms.Normalize.  color_jitter: the ColorJitter of
        scripts/train.py:121-124 (brightness = contrast = saturation = color_jitter, hue = 0.5) when > 0.
        steps=None: single frames (posenet); steps=T: MF(steps, skip, variable_skip) tuples; online=True: MFOnline,
        with the validation sequence val_frames and its VO-library ("real") poses val_poses, gps_mode as the reference.
        max_batch: the largest batch (in items) assemble() takes.  vo_poses: [L,6] float32, the VO-library ("real")
        pose of every frame, from which evaluation derives the windows' VOs as MF(real=True, include_vos=True) does
        (dataset_loaders/composite.py:47-97; the poses stay the targets, as its gt_dset's)."""
        frames, poses = _frames_and_poses(frames, poses)
        if online:
            val_frames, val_poses = _frames_and_poses(val_frames, val_poses)
        seqs = [(frames, poses)] + ([(val_frames, val_poses)] if online else [])
        shapes = set()
        for f, p in seqs:
            if f.dtype not in (np.uint8, torch.uint8) or f.ndim != 4 or f.shape[3] != 3:
                raise ValueError("expected uint8 frames [L,H,W,3], got %s %s" % (f.dtype, tuple(f.shape)))
            if p is None or tuple(np.shape(p)) != (f.shape[0], 6):
                raise ValueError("expected poses [%d,6], got %s" % (f.shape[0], None if p is None else np.shape(p)))
            shapes.add(tuple(f.shape[1:3]))
        if len(shapes) != 1:
            raise ValueError("all frames must have one size, got %s" % sorted(shapes))
        if vo_poses is not None:
            if online:
                raise ValueError("vo_poses are for evaluation windows; MFOnline takes its VO poses as val_poses")
            if tuple(np.shape(vo_poses)) != (frames.shape[0], 6):
                raise ValueError("expected vo_poses [%d,6], got %s" % (frames.shape[0], np.shape(vo_poses)))
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise RuntimeError("geomapnet_b200.data.DeviceDataset has no CPU path: device must be CUDA")
        self.H, self.W = shapes.pop()
        self.size = int(size)
        self.Ho, self.Wo = resize_output_size(self.H, self.W, size)
        ItemLayout.__init__(self, frames.shape[0], steps, skip, variable_skip, online,
                            val_frames.shape[0] if online else 0, gps_mode, color_jitter)
        self.mean = np.asarray(mean, dtype=np.float64).astype(np.float32).reshape(3).copy()
        self.std = np.asarray(std, dtype=np.float64).astype(np.float32).reshape(3).copy()
        if not (self.std > 0).all():
            raise ValueError("std must be positive, got %s" % (self.std,))
        self.poses = torch.as_tensor(np.concatenate([np.asarray(p, dtype=np.float32) for _, p in seqs]),
                                     dtype=torch.float32).to(self.device).contiguous()
        self.vo_poses = None if vo_poses is None else torch.as_tensor(
            np.asarray(vo_poses, dtype=np.float32)).to(self.device).contiguous()
        # the cache: every frame resized once, in chunks (training sequence first, then the validation sequence)
        self.max_batch = int(max_batch)
        if self.max_batch < 1:
            raise ValueError("max_batch must be >= 1")
        self.h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().mapnet_frame_cache_create(
                ctypes.byref(self.h), self.L + self.Lv, self.H, self.W, self.size, int(chunk),
                self.max_batch * self.frames_per_item, self.max_batch * self.targ_per_item), "mapnet_frame_cache_create")
            first = 0
            for f, _ in seqs:
                for lo in range(0, f.shape[0], int(chunk)):
                    part = torch.as_tensor(f[lo:lo + int(chunk)]).to(self.device).contiguous()
                    _lib.check(_lib.lib().mapnet_frame_cache_ingest(self.h, part.data_ptr(), first + lo, part.shape[0],
                                                                    _lib.stream_ptr()), "mapnet_frame_cache_ingest")
                first += f.shape[0]
            torch.cuda.current_stream(self.device).synchronize()

    def close(self):
        if self.h:
            _lib.lib().mapnet_frame_cache_destroy(self.h)
            self.h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def batch_shapes(self, n):
        """(input shape, target shape) of a batch of n items, as the model and criterion take them."""
        img = (3, self.Ho, self.Wo)
        if self.steps is None:
            return (n,) + img, (n, 6)
        return (n, self.frames_per_item) + img, (n, self.targ_per_item, 6)

    # ------------------------------------------------------------ assembly
    def assemble(self, batch, x_out, targ_out):
        """Assembles one collate() record into the float32 CUDA tensors x_out / targ_out (batch_shapes(N)), on the
        current stream: one launch, two with ColorJitter."""
        fr, jit, rows, n = batch
        xs, ts = self.batch_shapes(n)
        for t, shp, nm in ((x_out, xs, "x_out"), (targ_out, ts, "targ_out")):
            if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
                    and tuple(t.shape) == shp and t.device == self.device):
                raise ValueError("%s must be a contiguous float32 tensor %s on %s" % (nm, shp, self.device))
        fp = ctypes.POINTER(ctypes.c_float)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().mapnet_frame_cache_assemble(
                self.h, fr.shape[0], fr.ctypes.data, jit.ctypes.data if jit is not None else None, self.poses.data_ptr(),
                self.poses.shape[0], rows.ctypes.data, rows.shape[0], self.mean.ctypes.data_as(fp),
                self.std.ctypes.data_as(fp), x_out.data_ptr(), targ_out.data_ptr(), _lib.stream_ptr()),
                "mapnet_frame_cache_assemble")


    def assemble_frames(self, frames, x_out):
        """Frames `frames` (host int32 [n], n <= max_batch * frames_per_item) of the cache into the float32 CUDA tensor
        x_out [n,3,Ho,Wo] (ToTensor + Normalize, no ColorJitter), on the current stream: one launch."""
        fr = np.ascontiguousarray(frames, dtype=np.int32)
        n = fr.shape[0]
        if not (torch.is_tensor(x_out) and x_out.is_cuda and x_out.dtype == torch.float32 and x_out.is_contiguous()
                and tuple(x_out.shape) == (n, 3, self.Ho, self.Wo) and x_out.device == self.device):
            raise ValueError("x_out must be a contiguous float32 tensor %s on %s" % ((n, 3, self.Ho, self.Wo), self.device))
        fp = ctypes.POINTER(ctypes.c_float)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().mapnet_frame_cache_assemble(
                self.h, n, fr.ctypes.data, None, None, 0, None, 0, self.mean.ctypes.data_as(fp),
                self.std.ctypes.data_as(fp), x_out.data_ptr(), None, _lib.stream_ptr()), "mapnet_frame_cache_assemble")


class _Items(torch.utils.data.Dataset):
    def __init__(self, ds):
        self.ds = ds

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, i):
        return self.ds.item(i)


def host_batches(layout, batch_size, shuffle=True):
    """The host-side stream of DataLoader(dataset, batch_size, shuffle, num_workers=0) over a layout: one collate()
    record per batch, drawn lazily.  It is torch's own DataLoader over the host part of each item, so the global torch
    and numpy RNG streams advance exactly as in the reference's loop."""
    return iter(torch.utils.data.DataLoader(_Items(layout), batch_size=int(batch_size), shuffle=bool(shuffle),
                                            num_workers=0, collate_fn=layout.collate))


class DeviceLoader(object):
    """DataLoader(dataset, batch_size, shuffle, num_workers=0) over a DeviceDataset: yields device (x, targ) batches,
    the last one partial.  The sampling is torch's own DataLoader over the host part of each item, so the global torch
    and numpy RNG streams advance exactly as in the reference's loop.  The next batch is assembled on a side stream
    while the caller works on the current one; a yielded batch stays valid until the next one is requested."""

    def __init__(self, dataset, batch_size, shuffle=True):
        self.dataset, self.batch_size, self.shuffle = dataset, int(batch_size), bool(shuffle)
        if not 1 <= self.batch_size <= dataset.max_batch:
            raise ValueError("batch_size must be in [1, dataset.max_batch=%d]" % dataset.max_batch)
        self._bufs = None

    def __len__(self):
        return (len(self.dataset) + self.batch_size - 1) // self.batch_size

    def batches(self):
        """The host-side stream: one collate() record per batch, drawn lazily in the reference's order."""
        return host_batches(self.dataset, self.batch_size, self.shuffle)

    def __iter__(self):
        ds, dev = self.dataset, self.dataset.device
        if self._bufs is None:
            xs, ts = ds.batch_shapes(self.batch_size)
            self._bufs = [(torch.empty(xs, device=dev), torch.empty(ts, device=dev)) for _ in range(2)]
            self._side = torch.cuda.Stream(dev)
            self._ready = [torch.cuda.Event() for _ in range(2)]
            self._free = [torch.cuda.Event() for _ in range(2)]

        def launch(batch, slot):
            x, t = self._bufs[slot]
            n = batch[3]
            self._side.wait_event(self._free[slot])           # the consumer of the slot's previous batch is done
            with torch.cuda.stream(self._side):
                ds.assemble(batch, x[:n], t[:n])
            self._ready[slot].record(self._side)
            return n

        it = self.batches()
        first = next(it, None)
        if first is None:
            return
        slot, n = 0, launch(first, 0)
        while True:
            nxt = next(it, None)
            nn = launch(nxt, 1 - slot) if nxt is not None else 0
            cur = torch.cuda.current_stream(dev)
            cur.wait_event(self._ready[slot])
            x, t = self._bufs[slot]
            yield x[:n], t[:n]
            self._free[slot].record(torch.cuda.current_stream(dev))
            if nxt is None:
                return
            slot, n = 1 - slot, nn
