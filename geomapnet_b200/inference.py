"""Batched inference + pose-graph optimisation: the evaluation loop of the reference on the GPU.

Host-side mirror of /root/reference/scripts/eval.py:137-199.  The reference runs batch size 1 ("batch_size MUST be 1",
:136-138), moves every prediction to numpy, applies qexp per pose in Python, optionally runs a dense numpy PGO per
frame and keeps the middle prediction of each tuple.  Here: ``predict`` runs the eval-mode forward in batches of tuples
through the same fprop engines as training (BatchNorm running statistics, no dropout at eval -- see note), ``post`` does
qexp + un-normalisation for all poses in one launch, ``pgo`` optimises all windows in one launch (csrc/pgo.cu), and
``pose_errors`` gives the translation / rotation errors eval.py prints (:193-199).  ``evaluate_sequence`` runs the
whole loop from a device-resident sequence (data.DeviceDataset), each distinct frame through the network once, and
``validate`` the trainer's validation pass (common/train.py:214-250) over a data.DeviceLoader.

Note on dropout: models/posenet.py:68-69 calls F.dropout without ``training=``, so the reference drops features at eval
time too whenever droprate > 0; scripts/eval.py builds the model with the ini's dropout.  ``predict`` follows the
module (geomapnet_b200.models.PoseNet keeps that behaviour); pass a model built with droprate=0 for deterministic poses.
"""
import contextlib
import ctypes

import numpy as np
import torch

from . import _lib
from .common.pgo import check_robust_c, optimize_pose_windows
from .data.loader import SidePipeline

__all__ = ["Predictor", "Localizer", "Tracker", "MultiTracker", "SampledTracker", "predict", "post", "pgo", "pose_errors", "evaluate_tuples", "evaluate_sequence", "validate"]


class Predictor(object):
    """Frozen eval-mode predictor of a PoseNet or MapNet: a snapshot of its weights and BatchNorm running statistics,
    run by the inference engine (csrc/infer.cu) with BatchNorm, residual and ReLU fused into the conv epilogues.

        pr = Predictor(model, max_batch=64)
        poses = pr(x)       # [L,3,H,W] -> [L,6];  [L,T,3,H,W] -> [L,T,6];  max_batch frames per engine call
        pr.refresh()        # take a new snapshot of the model's current parameters / running statistics
        mc = pr.sample(x, 32)   # droprate > 0: mean [L,6] / cov [L,6,6] of 32 dropout draws per frame, one trunk forward
        pr.close()

    Training the model afterwards does not change the predictor's output until ``refresh()``.  Precision, droprate and
    seed follow the model ('bf16' or 'tc_split' only).  Every distinct (B, H, W) is captured into a CUDA graph on its first
    call and replayed after that.  With droprate > 0 the masks follow the engine's own step counter (as the model's
    dropout, the reference's F.dropout is active at eval).

    ``precision='fp8'`` (for a 'bf16' or 'tc_split' model) runs every conv but the stem on e4m3 operands: the weights get
    a power-of-two scale per output channel, every activation tensor one power-of-two scale taken from ``calibration``
    frames ([L,3,H,W] or [L,T,3,H,W] on the GPU, L*T <= max_batch).  The engine is fixed to the calibration frames' (H, W);
    ``refresh()`` re-packs the weights and re-calibrates on a device copy of the frames, in place.  ``act_scales`` lists
    the scales (pool output, then each block's h and output)."""

    def __init__(self, model, max_batch=64, precision=None, calibration=None):
        net = model.mapnet if hasattr(model, "mapnet") else model
        if net.precision not in ("bf16", "tc_split"):
            raise ValueError("Predictor supports the precisions 'bf16' and 'tc_split' (the model uses %r)" % net.precision)
        if int(max_batch) < 1:
            raise ValueError("max_batch must be >= 1")
        if precision not in (None, "fp8"):
            raise ValueError("Predictor precision must be None (the model's) or 'fp8', got %r" % (precision,))
        self.model, self.net, self.max_batch = model, net, int(max_batch)
        self.precision, self.droprate, self.seed = precision or net.precision, float(net.droprate), net._seed
        self.device = torch.device("cuda", torch.cuda.current_device())
        self._calib = None      # fp8: device copy of the calibration frames [N,3,H,W]
        if self.precision == "fp8":
            if calibration is None:
                raise ValueError("precision='fp8' needs calibration frames ([L,3,H,W] or [L,T,3,H,W] on the GPU)")
            c = calibration
            if not c.is_cuda or c.dim() not in (4, 5) or c.shape[-3] != 3:
                raise ValueError("calibration must be a CUDA tensor [L,3,H,W] or [L,T,3,H,W], got %s on %s"
                                 % (tuple(c.shape), c.device))
            frames = c.reshape(-1, *c.shape[-3:])
            if not 1 <= frames.shape[0] <= self.max_batch:
                raise ValueError("%d calibration frames: need 1 .. max_batch=%d" % (frames.shape[0], self.max_batch))
            self._calib = frames.detach().to(self.device, torch.float32).contiguous().clone()
        elif calibration is not None:
            raise ValueError("calibration frames are only used with precision='fp8'")
        self._engines = {}      # (H, W) -> _lib.Infer
        self._graphs = {}       # (B, H, W) -> (CUDAGraph, static input, static output)
        self._sample_graphs = {}    # (B, H, W, S) -> (CUDAGraph, static input, static outputs)
        self._params = self._bufs = None
        self.refresh()
        if self._calib is not None:
            self._engine(*self._calib.shape[-2:])

    def refresh(self):
        """Snapshot the model's current parameters and running statistics into every engine of this predictor."""
        net = self.net
        if not net._is_flat(self.device):
            net._reflatten(self.device)
        with torch.no_grad():
            self._params = net._flat.detach().clone()
            self._bufs = net._bufs.detach().clone()
        with torch.cuda.device(self.device):
            for eng in self._engines.values():
                eng.load(self._params, self._bufs)      # in place: the captured graphs read the engines' own buffers
                if self._calib is not None:
                    eng.calibrate(self._calib)
        torch.cuda.current_stream(self.device).synchronize()

    @property
    def act_scales(self):
        """fp8: the 33 activation scales of the current snapshot, in schedule order"""
        if self._calib is None:
            raise RuntimeError("act_scales: only an fp8 Predictor has activation scales")
        return self._engine(*self._calib.shape[-2:]).act_scales()

    def _engine(self, H, W):
        eng = self._engines.get((H, W))
        if eng is None:
            with torch.cuda.device(self.device):
                eng = _lib.Infer(self.max_batch, H, W, self.net.feat_dim, self.precision)
                eng.load(self._params, self._bufs)
                if self._calib is not None:
                    eng.calibrate(self._calib)
            self._engines[(H, W)] = eng
        return eng

    def _graph(self, B, H, W, xb=None, slot=0, warm_droprate=None):
        """(CUDA graph, static input [B,3,H,W], static output [B,6]) of one batch shape, captured on first use after an
        eager run on xb (zeros when None).  slot > 0: a further graph of the same shape with its own input buffer.
        warm_droprate: the droprate of that eager run (default the predictor's; 0 leaves the dropout counter alone)."""
        key = (B, H, W) if slot == 0 else (B, H, W, slot)
        g = self._graphs.get(key)
        if g is None:
            eng = self._engine(H, W)
            xs = torch.zeros((B, 3, H, W), dtype=torch.float32, device=self.device)
            ps = torch.empty((B, 6), dtype=torch.float32, device=self.device)
            if xb is not None:
                xs.copy_(xb)
            cur = torch.cuda.current_stream(self.device)
            side = torch.cuda.Stream(self.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):        # eager run first: tile plans, tensor maps, kernel attributes
                eng.forward(xs, ps, self.droprate if warm_droprate is None else warm_droprate, self.seed)
            cur.wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                eng.forward(xs, ps, self.droprate, self.seed)
            g = self._graphs[key] = (graph, xs, ps)
        return g

    def _check_frames(self, H, W):
        """raises unless the predictor is open and takes frames of H x W (an fp8 one only its calibration size)"""
        if self._params is None:
            raise RuntimeError("Predictor is closed")
        if self._calib is not None and (H, W) != tuple(self._calib.shape[-2:]):
            raise ValueError("this fp8 Predictor was calibrated at %dx%d, got frames of %dx%d"
                             % (self._calib.shape[-2], self._calib.shape[-1], H, W))

    def _run(self, xb):
        """pred [B,6] for frames xb [B,3,H,W] (B <= max_batch): graph replay, captured on the first call of a shape."""
        graph, xs, ps = self._graph(xb.shape[0], xb.shape[2], xb.shape[3], xb)
        xs.copy_(xb)
        graph.replay()
        return ps.clone()

    def _frames(self, x):
        """float32 frames [N,3,H,W] of an input [L,3,H,W] or [L,T,3,H,W]; raises on anything this predictor cannot run"""
        if not x.is_cuda:
            raise RuntimeError("geomapnet_b200.inference.Predictor has no CPU path: input must be a CUDA tensor "
                               "(got %s)" % x.device)
        if x.dim() not in (4, 5) or x.shape[-3] != 3:
            raise ValueError("expected input [L,3,H,W] or [L,T,3,H,W], got %s" % (tuple(x.shape),))
        if x.shape[0] < 1 or (x.dim() == 5 and x.shape[1] < 1):
            raise ValueError("empty batch")
        self._check_frames(x.shape[-2], x.shape[-1])
        frames = x.reshape(-1, *x.shape[-3:])
        return frames if frames.dtype == torch.float32 else frames.float()

    @torch.no_grad()
    def __call__(self, x):
        frames = self._frames(x)
        with torch.cuda.device(self.device):
            outs = [self._run(frames[i:i + self.max_batch]) for i in range(0, frames.shape[0], self.max_batch)]
        out = torch.cat(outs, 0)
        return out.view(*x.shape[:-3], 6)

    def _sample_graph(self, B, H, W, S, slot=0):
        """(CUDA graph, static input [B,3,H,W], static outputs) of S dropout draws per frame for one batch shape,
        captured after an eager run at an explicit dropout step, which leaves the engine's dropout counter alone.
        slot > 0: a further graph of the same shape with its own input and output buffers."""
        key = (B, H, W, S) if slot == 0 else (B, H, W, S, slot)
        g = self._sample_graphs.get(key)
        if g is None:
            eng, dev, L = self._engine(H, W), self.device, _lib.lib()
            xs = torch.zeros((B, 3, H, W), dtype=torch.float32, device=dev)
            o = _sample_outputs(B, S, dev)

            def launch(step):
                eng.sample(xs, S, self.droprate, self.seed, o["samples"], o["mean"], o["cov"], step)
                _lib.check(L.mapnet_sample_post(o["mean"].data_ptr(), o["cov"].data_ptr(), B, None, None, None, None,
                                                o["t_std"].data_ptr(), o["q_std_deg"].data_ptr(), _lib.stream_ptr()),
                           "mapnet_sample_post")

            cur = torch.cuda.current_stream(dev)
            side = torch.cuda.Stream(dev)
            side.wait_stream(cur)
            with torch.cuda.stream(side):        # eager run first: tile plans, tensor maps, kernel attributes
                launch(0)
            cur.wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                launch(_lib.UINT64_MAX)
            g = self._sample_graphs[key] = (graph, xs, o)
        return g

    @torch.no_grad()
    def sample(self, x, S, keep_samples=False):
        """Monte-Carlo dropout: S dropout draws of every frame's pose from one trunk forward.  x as for ``__call__``
        ([L,3,H,W] or [L,T,3,H,W] on the GPU).  Returns dict(mean [...,6] float64, cov [...,6,6] float64 (two-pass,
        divisor S - 1), t_std [...] = sqrt(trace of the translation block) in the model's normalised units, q_std_deg
        [...] = 2 sqrt(trace of the log q block) in degrees, and samples [...,S,6] float32 when keep_samples).

        Only the head differs between draws, so the trunk and the fc product run once per frame and one kernel forms
        the S masks and products (csrc/head.cu, k_head_draws).  Draw s is bit for bit what the (s+1)-th of S calls
        ``self(x)`` returns on the same frames, and the dropout counter ends where those S calls leave it.  Inputs of
        more than max_batch frames run in chunks of max_batch; each chunk takes S consecutive dropout steps, in chunk
        order (as S calls on the first chunk, then S calls on the next).  One graph per (B, H, W, S), replayed once per
        chunk.  2 <= S <= 1024; a model without dropout (droprate == 0) has nothing to sample and raises ValueError."""
        S = _check_draws(S, self.droprate)
        frames = self._frames(x)
        n, H, W, mb = frames.shape[0], frames.shape[2], frames.shape[3], self.max_batch
        out = _sample_outputs(n, S, self.device, keep_samples)
        with torch.cuda.device(self.device):
            for lo in range(0, n, mb):
                fb = frames[lo:lo + mb]
                graph, xs, o = self._sample_graph(fb.shape[0], H, W, S)
                xs.copy_(fb)
                graph.replay()
                for k, v in out.items():
                    v[lo:lo + fb.shape[0]].copy_(o[k])
        lead = tuple(x.shape[:-3])
        return {k: v.view(*(lead + tuple(v.shape[1:]))) for k, v in out.items()}

    def close(self):
        self._graphs.clear()
        self._sample_graphs.clear()
        for eng in self._engines.values():
            eng.close()
        self._engines.clear()
        self._params = self._bufs = self._calib = None


def _check_draws(S, droprate):
    """S as an int in [2, MAX_SAMPLE_DRAWS]; raises when there is no dropout to sample"""
    if isinstance(S, bool) or not isinstance(S, (int, np.integer)) or not 2 <= S <= _lib.MAX_SAMPLE_DRAWS:
        raise ValueError("S must be an int in [2, %d], got %r" % (_lib.MAX_SAMPLE_DRAWS, S))
    if not droprate > 0:
        raise ValueError("sample: the model has no dropout (droprate == 0), so every draw is the same pose")
    return int(S)


def _sample_outputs(n, S, dev, keep_samples=True):
    """the device outputs of n frames' S-draw Monte-Carlo statistics"""
    f64 = dict(dtype=torch.float64, device=dev)
    out = dict(mean=torch.empty((n, 6), **f64), cov=torch.empty((n, 6, 6), **f64), t_std=torch.empty(n, **f64),
               q_std_deg=torch.empty(n, **f64))
    if keep_samples:
        out["samples"] = torch.empty((n, S, 6), dtype=torch.float32, device=dev)
    return out


@torch.no_grad()
def predict(model, x, batch=64):
    """model(x) in eval mode, `batch` leading entries at a time.  x: [L,3,H,W] (PoseNet) or [L,T,3,H,W] (MapNet), on the
    GPU or pinned host memory.  Returns float32 [L,6] / [L,T,6] on the device.  `model` may be a Predictor, which runs
    its snapshot in chunks of its own max_batch frames."""
    if isinstance(model, Predictor):
        return model(x if x.is_cuda else x.cuda(non_blocking=True))
    was_training = model.training
    model.eval()
    outs = []
    try:
        for i in range(0, x.shape[0], batch):
            xb = x[i:i + batch]
            if not xb.is_cuda:
                xb = xb.cuda(non_blocking=True)
            outs.append(model(xb).float())
    finally:
        model.train(was_training)
    return torch.cat(outs, 0)


def post(pred6, pose_m=None, pose_s=None):
    """eval.py:163-181: (t, log q) -> (t * pose_s + pose_m, qexp(log q)) for every pose; [..., 6] float32 -> [..., 7] float64."""
    p = pred6.detach().float().contiguous()
    if not p.is_cuda:
        raise RuntimeError("geomapnet_b200.inference has no CPU path: predictions must be CUDA tensors")
    n = p.numel() // 6
    out = torch.empty(p.shape[:-1] + (7,), dtype=torch.float64, device=p.device)
    m = s = None
    if pose_m is not None:
        m = (ctypes.c_double * 3)(*[float(v) for v in np.asarray(pose_m).reshape(3)])
        s = (ctypes.c_double * 3)(*[float(v) for v in np.asarray(pose_s).reshape(3)])
    with torch.cuda.device(p.device):
        _lib.check(_lib.lib().mapnet_pose_post(p.data_ptr(), out.data_ptr(), n, m, s, _lib.stream_ptr()), "mapnet_pose_post")
    return out


class Localizer(object):
    """Camera frames in, metric poses out: Resize(size) + ToTensor + Normalize(mean, std), the Predictor's snapshot and
    ``post`` in one CUDA graph per batch shape.

        loc = Localizer(predictor, mean, std, pose_m=None, pose_s=None, size=256)
        poses = loc(frames)     # uint8 [L,H,W,3] or [H,W,3] (RGB, as PIL decodes), a CUDA or host tensor or an ndarray
                                # -> float64 [L,7] (or [7]) on the device: (t * pose_s + pose_m, qexp(log q))
        mc = loc.sample(frames, 32)     # droprate > 0: metric mean pose7 [L,7] and cov [L,6,6] of 32 dropout draws
        loc.close()

    ``loc(frames)`` is bit for bit ``post(predictor(ImagePipeline(mean, std, size)(frames.cuda())), pose_m, pose_s)``,
    but the normalised image is written straight into the engine's stem operand (csrc/preprocess.cu,
    k_pre_resize_v_s2d) instead of going through a float32 tensor, and the whole call replays one graph: the horizontal
    resize, that fused pass, the engine from the stem conv on and the pose post-processing.  The snapshot, ``refresh()``,
    precision (bf16, tc_split or fp8), ``max_batch`` and the dropout counter are the predictor's: the Localizer runs the
    predictor's own engines, so with droprate > 0 the masks follow the same sequence of engine calls as calling the
    predictor does.  An fp8 predictor takes only frames that resize to its calibration size.  Each distinct (B, H, W)
    is captured after one eager run, as Predictor's graphs are; longer inputs run in chunks of max_batch frames.
    mean / std are rounded to float32 as ImagePipeline rounds them; pose_m / pose_s (pose_stats.txt) may be left out
    together, which keeps the normalised translations."""

    def __init__(self, predictor, mean, std, pose_m=None, pose_s=None, size=256):
        if not isinstance(predictor, Predictor):
            raise TypeError("Localizer wraps a geomapnet_b200.inference.Predictor, got %s" % type(predictor).__name__)
        self.mean = np.asarray(mean, dtype=np.float64).astype(np.float32).reshape(3).copy()
        self.std = np.asarray(std, dtype=np.float64).astype(np.float32).reshape(3).copy()
        if not (self.std > 0).all():
            raise ValueError("std must be positive, got %s" % (self.std,))
        if (pose_m is None) != (pose_s is None):
            raise ValueError("pose_m and pose_s go together (pose_stats.txt rows 0 and 1), or neither is given")
        self._m = self._s = None
        if pose_m is not None:
            self._m = (ctypes.c_double * 3)(*[float(v) for v in np.asarray(pose_m).reshape(3)])
            self._s = (ctypes.c_double * 3)(*[float(v) for v in np.asarray(pose_s).reshape(3)])
        self.predictor, self.size = predictor, int(size)
        self._plans = {}        # (H_in, W_in) -> mapnet_preprocess_t of max_batch frames
        self._graphs = {}       # (B, H_in, W_in) -> (CUDAGraph, static uint8 input, static float64 output, pred6)
        self._warm = set()      # engine shapes (B, H', W') whose eager run has drawn a dropout mask
        self._sample_graphs = {}    # (B, H_in, W_in, S) -> (CUDAGraph, static uint8 input, static outputs)
        self._open = True

    def _resized(self, H, W):
        """the (H, W) the engine sees for frames of H x W: torchvision's Resize(size)"""
        from .data.preprocess import resize_output_size
        return resize_output_size(H, W, self.size)

    def _plan(self, H, W):
        h = self._plans.get((H, W))
        if h is None:
            h = ctypes.c_void_p()
            _lib.check(_lib.lib().mapnet_preprocess_create(ctypes.byref(h), H, W, self.size, self.predictor.max_batch),
                       "mapnet_preprocess_create")
            self._plans[(H, W)] = h
        return h

    def _forward(self, eng, pre, xs, pred, droprate):
        """the engine's launches on the current stream: frames xs -> pred [B,6]"""
        fp = ctypes.POINTER(ctypes.c_float)
        _lib.check(_lib.lib().mapnet_infer_forward_frames(
            eng.h, pre, xs.data_ptr(), xs.shape[0], self.mean.ctypes.data_as(fp), self.std.ctypes.data_as(fp),
            droprate, int(self.predictor.seed), _lib.UINT64_MAX, pred.data_ptr(), _lib.stream_ptr()),
            "mapnet_infer_forward_frames")

    def _post(self, pred, out):
        _lib.check(_lib.lib().mapnet_pose_post(pred.data_ptr(), out.data_ptr(), pred.shape[0], self._m, self._s,
                                               _lib.stream_ptr()), "mapnet_pose_post")

    def _launch(self, eng, pre, xs, pred, out, droprate):
        """the call's library launches on the current stream: frames xs -> pred [B,6] -> out [B,7]"""
        self._forward(eng, pre, xs, pred, droprate)
        self._post(pred, out)

    def _capture(self, fb, tail, eager_tail=True):
        """(CUDA graph, static uint8 input, static pred6 [B,6]) of frames shaped like fb: the engine's forward, then
        tail(pred6)'s launches.  Captured after an eager run of the forward (and of tail when eager_tail): tile plans,
        tensor maps, kernel attributes.  That eager run draws a dropout mask only where calling the predictor would run
        one: the first time this Localizer or the predictor meets the engine shape (B, H', W'), so frame sizes that
        resize alike share one draw."""
        B, H, W = fb.shape[:3]
        pr = self.predictor
        Ho, Wo = self._resized(H, W)
        eng, pre = pr._engine(Ho, Wo), self._plan(H, W)
        new_shape = (B, Ho, Wo) not in pr._graphs and (B, Ho, Wo) not in self._warm
        self._warm.add((B, Ho, Wo))
        xs = torch.empty((B, H, W, 3), dtype=torch.uint8, device=pr.device)
        pred = torch.empty((B, 6), dtype=torch.float32, device=pr.device)
        xs.copy_(fb)
        cur = torch.cuda.current_stream(pr.device)
        side = torch.cuda.Stream(pr.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            self._forward(eng, pre, xs, pred, pr.droprate if new_shape else 0.0)
            if eager_tail:
                tail(pred)
        cur.wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._forward(eng, pre, xs, pred, pr.droprate)
            tail(pred)
        return graph, xs, pred

    def _graph(self, fb):
        """(CUDA graph, static input, static output, static pred6) of frames shaped like fb (see _capture)"""
        B, H, W = fb.shape[:3]
        g = self._graphs.get((B, H, W))
        if g is None:
            out = torch.empty((B, 7), dtype=torch.float64, device=self.predictor.device)
            graph, xs, pred = self._capture(fb, lambda pred: self._post(pred, out))
            g = self._graphs[(B, H, W)] = (graph, xs, out, pred)
        return g

    def _run(self, fb):
        graph, xs, out, _ = self._graph(fb)
        xs.copy_(fb, non_blocking=True)
        graph.replay()
        return out.clone()

    def _frames(self, frames):
        """(contiguous uint8 frames [L,H,W,3], whether a single [H,W,3] frame was given); raises on anything this
        Localizer cannot run"""
        if not self._open or self.predictor._params is None:
            raise ValueError("Localizer is closed" if not self._open else "the Localizer's Predictor is closed")
        if isinstance(frames, np.ndarray):
            if frames.dtype != np.uint8:
                raise ValueError("expected uint8 frames, got %s" % frames.dtype)
            frames = torch.from_numpy(np.ascontiguousarray(frames))
        if not torch.is_tensor(frames) or frames.dtype != torch.uint8:
            raise ValueError("expected uint8 frames, got %s" % getattr(frames, "dtype", type(frames).__name__))
        if frames.dim() not in (3, 4) or frames.shape[-1] != 3:
            raise ValueError("expected RGB frames [L,H,W,3] or [H,W,3], got %s" % (tuple(frames.shape),))
        single = frames.dim() == 3
        x = frames.unsqueeze(0) if single else frames
        if x.shape[0] < 1 or x.shape[1] < 1 or x.shape[2] < 1:
            raise ValueError("empty batch: frames of shape %s" % (tuple(frames.shape),))
        self.predictor._check_frames(*self._resized(x.shape[1], x.shape[2]))
        return x.contiguous(), single

    @torch.no_grad()
    def __call__(self, frames):
        x, single = self._frames(frames)
        mb = self.predictor.max_batch
        with torch.cuda.device(self.predictor.device):
            outs = [self._run(x[i:i + mb]) for i in range(0, x.shape[0], mb)]
        out = outs[0] if len(outs) == 1 else torch.cat(outs, 0)
        return out[0] if single else out

    def _sample_launch(self, eng, pre, xs, o, S, step):
        """the sample call's library launches on the current stream: frames xs -> S draws -> float64 metric post"""
        pr, L, B = self.predictor, _lib.lib(), xs.shape[0]
        fp = ctypes.POINTER(ctypes.c_float)
        _lib.check(L.mapnet_infer_sample_frames(eng.h, pre, xs.data_ptr(), B, self.mean.ctypes.data_as(fp),
                                                self.std.ctypes.data_as(fp), S, pr.droprate, int(pr.seed), step,
                                                o["samples"].data_ptr(), o["mean"].data_ptr(), o["cov6"].data_ptr(),
                                                _lib.stream_ptr()), "mapnet_infer_sample_frames")
        _lib.check(L.mapnet_sample_post(o["mean"].data_ptr(), o["cov6"].data_ptr(), B, self._m, self._s,
                                        o["pose7"].data_ptr(), o["cov"].data_ptr(), o["t_std"].data_ptr(),
                                        o["q_std_deg"].data_ptr(), _lib.stream_ptr()), "mapnet_sample_post")

    def _sample_graph(self, fb, S):
        """(CUDA graph, static input, static outputs) of S draws per frame for frames shaped like fb, captured after an
        eager run at an explicit dropout step (the dropout counter is left alone)"""
        B, H, W = fb.shape[:3]
        g = self._sample_graphs.get((B, H, W, S))
        if g is None:
            pr = self.predictor
            eng, pre = pr._engine(*self._resized(H, W)), self._plan(H, W)
            xs = torch.empty((B, H, W, 3), dtype=torch.uint8, device=pr.device)
            xs.copy_(fb)
            o = _sample_outputs(B, S, pr.device)
            o["cov6"] = torch.empty_like(o["cov"])
            o["pose7"] = torch.empty((B, 7), dtype=torch.float64, device=pr.device)
            cur = torch.cuda.current_stream(pr.device)
            side = torch.cuda.Stream(pr.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):        # eager run first: tile plans, tensor maps, kernel attributes
                self._sample_launch(eng, pre, xs, o, S, 0)
            cur.wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._sample_launch(eng, pre, xs, o, S, _lib.UINT64_MAX)
            g = self._sample_graphs[(B, H, W, S)] = (graph, xs, o)
        return g

    @torch.no_grad()
    def sample(self, frames, S, keep_samples=False):
        """Monte-Carlo dropout poses: S dropout draws of every frame's pose from one trunk forward, in metric units.
        frames as for ``__call__``.  Returns dict(pose7 [L,7] float64 = (mean_t * pose_s + pose_m, qexp(mean log q)),
        cov [L,6,6] float64 = D cov D with D = diag(pose_s, 1, 1, 1) (translation block in metres, log q block
        unscaled), t_std [L] = sqrt(trace of the translation block), q_std_deg [L] = 2 sqrt(trace of the log q block)
        in degrees, and samples [L,S,6] float32 -- the draws in the model's normalised units -- when keep_samples); a
        single [H,W,3] frame drops the leading L.  Without pose_m / pose_s, D is the identity.

        Draw s is bit for bit what the (s+1)-th of S calls ``self(frames)`` draws (Predictor.sample); the Localizer
        shares the predictor's engines and dropout counter as ``__call__`` does, and longer inputs run in chunks of
        max_batch frames, each taking S consecutive dropout steps.  Each chunk replays one graph: the resize, the fused
        stem operand, the engine, the draws and the float64 post step.  2 <= S <= 1024; a model without dropout raises
        ValueError."""
        x, single = self._frames(frames)
        pr = self.predictor
        S = _check_draws(S, pr.droprate)
        n, mb = x.shape[0], pr.max_batch
        out = _sample_outputs(n, S, pr.device, keep_samples)
        del out["mean"]                                 # the normalised mean: pose7 is what a caller of loc uses
        out["pose7"] = torch.empty((n, 7), dtype=torch.float64, device=pr.device)
        with torch.cuda.device(pr.device):
            for lo in range(0, n, mb):
                fb = x[lo:lo + mb]
                graph, xs, o = self._sample_graph(fb, S)
                xs.copy_(fb, non_blocking=True)
                graph.replay()
                for k, v in out.items():
                    v[lo:lo + fb.shape[0]].copy_(o[k])
        return {k: v[0] for k, v in out.items()} if single else out

    def close(self):
        """Free the graphs and preprocess plans (the predictor stays open)."""
        if self._graphs or self._plans:
            torch.cuda.current_stream(self.predictor.device).synchronize()
        self._graphs.clear()
        self._sample_graphs.clear()
        for h in self._plans.values():
            _lib.lib().mapnet_preprocess_destroy(h)
        self._plans.clear()
        self._open = False


def _first_pending(seen, lag):
    """the first frame whose window is not complete after `seen` frames (csrc/track_core.h, first_pending)"""
    return max(seen - lag, 0)


def _int_arg(v, name, lo, hi=None):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < lo or (hi is not None and v > hi):
        raise ValueError("%s must be an int in [%d, %s], got %r" % (name, lo, "inf" if hi is None else hi, v))
    return int(v)


class Tracker(object):
    """MapNet+PGO on a camera stream: scripts/eval.py's pose-graph optimisation (--pose_graph) over frames as they
    arrive, from a Localizer.

        loc = Localizer(Predictor(model, max_batch=8), mean, std, pose_m, pose_s)
        trk = Tracker(loc, steps=7, skip=10, vo_fc=True, sax=1, saq=1, srx=20, srq=20)    # pgo_inference_RobotCar.ini
        first, pose7 = trk(frames, vo_poses)    # uint8 [B,H,W,3] or [H,W,3] as loc takes them; float32 [B,6] or [6]
                                                # -> frames first .. first+n-1 whose windows completed: float64 [n,7]
        now7, first, pose7 = trk.step(frames, vo_poses)     # also each given frame's zero-lag pose: float64 [B,7]
        first, pose7 = trk.flush()              # the last min(lag, seen) frames; starts a new sequence
        trk.reset(); trk.lag; trk.close()

    The window of frame i is eval.py's MF(steps, skip, real=True, include_vos=True): slot k holds frame
    clip(i + (k - steps//2) * skip, 0, L-1); its VOs are calc_vos_safe of the VO-library poses of consecutive slots (or
    calc_vos_safe_fc of every pair i<j when vo_fc); PGO runs on the normalised translations (10 iterations, the
    reference's literal linear solve, covariances sax, saq, srx, srq) and the middle slot, un-normalised with the
    Localizer's pose_m / pose_s (kept normalised without them), is frame i's pose.  Frame i's window is complete once
    frame i + lag has arrived, lag = (steps - 1 - steps//2) * skip (30 frames at RobotCar's steps=7, skip=10; 450 at
    7Scenes' skip=150): a fixed-lag smoother, faithful to eval.py.  flush() emits the last frames with their windows
    clipped at the last frame seen, as eval.py clips them at the sequence's end.  vo_poses: the VO library's per-frame
    poses in the dataset's normalisation ((t - pose_m) / pose_s, log q), as DeviceDataset(vo_poses=) takes them; any
    real floating dtype, rounded to float32 as DeviceDataset rounds them.

    step() is the zero-lag output for live use: besides what the call emits, each frame f it brings gets the last slot
    of the optimised window that ends at f -- frame (f - lag)'s window, slots below 0 clipped at 0 during the first lag
    frames -- in the call that brings it.  That is the window a call solves anyway once f >= lag, so a step costs what
    a call costs past the lag, and one window more per frame before it.  evaluate_sequence(..., zero_lag=True) is its
    offline counterpart on a labelled sequence.  Calls and steps share the sequence, so they may be mixed.

    With droprate == 0 the poses are bit for bit evaluate_sequence's on a DeviceDataset of the same frames, when the
    Predictor runs the same chunks.  With droprate > 0 every frame goes through the network once and every window that
    holds it reuses that draw, where eval.py draws each window's frames anew: the poses are what eval.py's windows of
    exactly those per-frame draws give.  Engines, snapshot, refresh(), precision and dropout counter are the
    Localizer's predictor's.  Each chunk of max_batch frames replays one CUDA graph, captured per (B, H, W) after an
    eager forward as the Localizer captures: mapnet_infer_forward_frames, then three tracking launches (csrc/loader.cu:
    gather the windows from device rings of recent poses, k_pgo, emit), with the frame counter in device memory; a
    call never waits for the device.  The host counts frames too, so the frames a call emits follow from the call
    sizes.  A window whose normal matrix is not positive definite (where scipy's cholesky raises) is reported by
    flush(), which raises np.linalg.LinAlgError after resetting.

    robust_c=c (a finite number > 0, in sigmas) gives every window's absolute factors the Cauchy loss of scale c
    (common.pgo.optimize_pose_windows(robust_c=c)): a frame whose prediction is far off -- glare, occlusion -- is
    down-weighted in each window that holds it instead of pulling on all of them.  The output formats, launches and
    chunking stay; the poses are bit for bit evaluate_sequence(..., robust_c=c)'s.  A bad robust_c raises ValueError
    here, before anything is launched."""

    _API = "mapnet_track"       # the handle's C calls: _API + "_create", "_step", "_step_now", "_flush", ...
    _ROW = 7                    # doubles per output row

    def __init__(self, localizer, steps, skip=1, vo_fc=False, sax=1.0, saq=1.0, srx=1.0, srq=1.0, robust_c=None):
        if not isinstance(localizer, Localizer):
            raise TypeError("Tracker wraps a geomapnet_b200.inference.Localizer, got %s" % type(localizer).__name__)
        self.steps = _int_arg(steps, "steps", 2, _lib.MAX_TRACK_STEPS)
        self.skip = _int_arg(skip, "skip", 1)
        self.sigmas = [float(v) for v in (sax, saq, srx, srq)]
        if not all(v > 0 for v in self.sigmas):
            raise ValueError("sax, saq, srx, srq must be positive, got %s" % (self.sigmas,))
        self.robust_c = check_robust_c(robust_c)
        self.loc, self.vo_fc = localizer, bool(vo_fc)
        self.lag = (self.steps - 1 - self.steps // 2) * self.skip
        self.seen = 0           # frames of the current sequence, mirrored on the device
        self._graphs = {}       # (B, H, W) -> (CUDAGraph, static uint8 input, vo [B,6], out [B,_ROW], engine outputs)
        self._now_graphs = {}   # the same for step(), with now [B,_ROW] last
        self.h = ctypes.c_void_p()      # mapnet_track_t, created with the first call
        self._open = True

    def _check_open(self):
        name = type(self).__name__
        if not self._open:
            raise ValueError("%s is closed" % name)
        if not self.loc._open or self.loc.predictor._params is None:
            raise ValueError("the %s's %s is closed" % (name, "Localizer" if not self.loc._open else "Predictor"))

    def _vo(self, vo_poses, n, single):
        """vo_poses as a tensor [n,6] of a real floating dtype; raises on anything else"""
        v = torch.from_numpy(np.ascontiguousarray(vo_poses)) if isinstance(vo_poses, np.ndarray) else vo_poses
        if not torch.is_tensor(v) or v.dtype not in (torch.float16, torch.bfloat16, torch.float32, torch.float64):
            raise ValueError("vo_poses must be a float tensor or array, got %s" % getattr(v, "dtype", type(v).__name__))
        want = (6,) if single else (n, 6)
        if tuple(v.shape) != want:
            raise ValueError("vo_poses must be %s for %s, got %s" % (
                list(want), "one [H,W,3] frame" if single else "%d frames" % n, tuple(v.shape)))
        return v.reshape(n, 6)

    @staticmethod
    def _est(rows):
        """what a caller gets for output rows [n, _ROW]: pose7 itself"""
        return rows

    def _capture(self, fb, track):
        """(CUDA graph, static uint8 input, engine outputs) of frames shaped like fb: the Localizer's engine, then
        track(*engine outputs)'s launches"""
        return self.loc._capture(fb, track, eager_tail=False)  # the eager run must not advance the stream

    def _handle(self):
        if not self.h:
            pr = self.loc.predictor
            sig = (ctypes.c_double * 4)(*self.sigmas)
            _lib.check(getattr(_lib.lib(), self._API + "_create")(ctypes.byref(self.h), self.steps, self.skip,
                                                                  int(self.vo_fc), pr.max_batch, sig, self.loc._m,
                                                                  self.loc._s), self._API + "_create")
            self._set_robust()
        return self.h

    def _set_robust(self):
        """the new handle's Cauchy scale, before its first step (nothing is launched)"""
        if self.robust_c is not None:
            _lib.check(getattr(_lib.lib(), self._API + "_set_robust")(self.h, self.robust_c), self._API + "_set_robust")

    def _graph(self, fb, now=False):
        B, H, W = fb.shape[:3]
        graphs = self._now_graphs if now else self._graphs
        g = graphs.get((B, H, W))
        if g is None:
            dev, h = self.loc.predictor.device, self._handle()
            vs = torch.zeros((B, 6), dtype=torch.float32, device=dev)
            out = torch.empty((B, self._ROW), dtype=torch.float64, device=dev)
            nows = (torch.empty((B, self._ROW), dtype=torch.float64, device=dev),) if now else ()
            name = self._API + ("_step_now" if now else "_step")

            def track(*ins):
                _lib.check(getattr(_lib.lib(), name)(h, *[t.data_ptr() for t in ins], vs.data_ptr(), B, out.data_ptr(),
                                                     *[t.data_ptr() for t in nows], _lib.stream_ptr()), name)

            graph, xs, ins = self._capture(fb, track)
            g = (graph, xs, vs, out, ins) + nows        # every buffer the graph reads stays alive
            graphs[(B, H, W)] = g
        return g

    def _run(self, frames, vo_poses, now):
        """(first, rows [n,_ROW], now rows [B,_ROW] or None): the chunks of max_batch frames, one graph replay each"""
        self._check_open()
        x, single = self.loc._frames(frames)
        vo = self._vo(vo_poses, x.shape[0], single)
        pr = self.loc.predictor
        mb, first = pr.max_batch, _first_pending(self.seen, self.lag)
        outs, nows = [], []
        with torch.cuda.device(pr.device):
            for lo in range(0, x.shape[0], mb):
                fb = x[lo:lo + mb]
                g = self._graph(fb, now)
                graph, xs, vs, out = g[:4]
                xs.copy_(fb, non_blocking=True)
                vs.copy_(vo[lo:lo + mb], non_blocking=True)
                graph.replay()
                n = _first_pending(self.seen + fb.shape[0], self.lag) - _first_pending(self.seen, self.lag)
                self.seen += fb.shape[0]
                outs.append(out[:n].clone())
                if now:
                    nows.append(g[5].clone())
        cat = lambda ts: ts[0] if len(ts) == 1 else torch.cat(ts, 0)
        return first, cat(outs), (cat(nows) if now else None)

    @torch.no_grad()
    def __call__(self, frames, vo_poses):
        """-> (first, pose7 float64 [n,7] on the device): the frames first .. first+n-1 whose windows this call
        completed, n = max(seen + B - lag, 0) - max(seen - lag, 0) for the B frames given"""
        first, rows, _ = self._run(frames, vo_poses, False)
        return first, self._est(rows)

    @torch.no_grad()
    def step(self, frames, vo_poses):
        """-> (now7 float64 [B,7] on the device, first, pose7 [n,7]): row b of now7 is the zero-lag pose of the b-th
        frame given, f = seen + b: slot steps-1 of the optimised window that ends at f (frame (f - lag)'s window,
        clipped at 0), un-normalised as pose7; (first, pose7) is what self(frames, vo_poses) returns.  Takes what
        __call__ takes; each chunk replays a graph of its own, the same three tracking launches."""
        first, rows, nows = self._run(frames, vo_poses, True)
        return self._est(nows), first, self._est(rows)

    @torch.no_grad()
    def flush(self):
        """-> (first, pose7 [n,7]): the last n = min(lag, seen) frames, their windows clipped at the last frame seen.
        Synchronises, starts a new sequence, and raises np.linalg.LinAlgError if a window of the sequence that ended
        was not positive definite."""
        self._check_open()
        pr = self.loc.predictor
        first = _first_pending(self.seen, self.lag)
        n, failed = self.seen - first, ctypes.c_int(0)
        with torch.cuda.device(pr.device):
            out = torch.empty((max(self.lag, 1), self._ROW), dtype=torch.float64, device=pr.device)
            if self.h:
                L = _lib.lib()
                _lib.check(getattr(L, self._API + "_flush")(self.h, out.data_ptr(), _lib.stream_ptr()),
                           self._API + "_flush")
                _lib.check(getattr(L, self._API + "_status")(self.h, None, ctypes.byref(failed), _lib.stream_ptr()),
                           self._API + "_status")
        self.reset()
        if failed.value:
            raise np.linalg.LinAlgError("pose graph: the normal matrix of a window of the sequence is not positive "
                                        "definite")
        return first, self._est(out[:n])

    def reset(self):
        """Start a new sequence: the next frame is frame 0 (stream-ordered)."""
        self._check_open()
        if self.h:
            with torch.cuda.device(self.loc.predictor.device):
                _lib.check(getattr(_lib.lib(), self._API + "_reset")(self.h, _lib.stream_ptr()), self._API + "_reset")
        self.seen = 0

    def close(self):
        """Free the graphs and the device state (the Localizer and its predictor stay open)."""
        if self.h:
            torch.cuda.current_stream(self.loc.predictor.device).synchronize()
            self._graphs.clear()
            self._now_graphs.clear()
            getattr(_lib.lib(), self._API + "_destroy")(self.h)
            self.h = ctypes.c_void_p()
        self._open = False


def _sampled_capture(loc, S, fb, track):
    """(CUDA graph, static uint8 input [B,H,W,3], (draws [B,S,6], mean [B,6], cov [B,6,6])) of frames shaped like fb:
    the Localizer's sampled engine (mapnet_infer_sample_frames: S draws per frame, their normalised float64 mean and
    covariance) at the device dropout counter, then track(mean, cov)'s launches.  Captured after an eager run of the
    engine alone at an explicit dropout step, so building the graph advances neither the dropout counter nor any
    tracked sequence."""
    B, H, W = fb.shape[:3]
    pr, L = loc.predictor, _lib.lib()
    dev = pr.device
    eng, pre = pr._engine(*loc._resized(H, W)), loc._plan(H, W)
    f64 = dict(dtype=torch.float64, device=dev)
    xs = torch.empty((B, H, W, 3), dtype=torch.uint8, device=dev)
    xs.copy_(fb)
    smp = torch.empty((B, S, 6), dtype=torch.float32, device=dev)
    mean, cov = torch.empty((B, 6), **f64), torch.empty((B, 6, 6), **f64)
    fp = ctypes.POINTER(ctypes.c_float)

    def sample(step):
        _lib.check(L.mapnet_infer_sample_frames(eng.h, pre, xs.data_ptr(), B, loc.mean.ctypes.data_as(fp),
                                                loc.std.ctypes.data_as(fp), S, pr.droprate, int(pr.seed), step,
                                                smp.data_ptr(), mean.data_ptr(), cov.data_ptr(), _lib.stream_ptr()),
                   "mapnet_infer_sample_frames")

    cur = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(cur)
    with torch.cuda.stream(side):        # eager run first, at an explicit dropout step: no state advances
        sample(0)
    cur.wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sample(_lib.UINT64_MAX)
        track(mean, cov)
    return graph, xs, (smp, mean, cov)


class SampledTracker(Tracker):
    """Tracker with Monte-Carlo dropout: each frame's S dropout draws weigh its pose in the pose graph, and every
    tracked pose comes with a covariance.

        st = SampledTracker(loc, S=32, steps=7, skip=10, vo_fc=True, sax=1e-4, saq=1e-4, srx=20, srq=20)
        first, est = st(frames, vo_poses)       # est = dict(pose7 [n,7], cov [n,6,6], t_std [n], q_std_deg [n])
        now, first, est = st.step(frames, vo_poses)     # now: the same dict, each given frame's zero-lag estimate
        first, est = st.flush(); st.reset(); st.close(); st.lag; st.seen

    Frames, VO poses, windows, lag, chunking and errors are Tracker's.  Per frame f, the S draws (Localizer.sample's,
    in the model's normalised units) give a mean (mu_t, mu_v) and a covariance Sigma_f [6,6].  Its absolute pose is
    p_f = (mu_t, qexp(mu_v)) (bit for bit Localizer.sample's pose7 without pose statistics), and its factor covariance
        S7_f = A Sigma_f A' + diag(sax, sax, sax, saq, saq, saq, saq),  A = blockdiag(I3, d qexp(v) / dv at mu_v).
    The absolute factor of slot k holding frame f has residual C^-1 (z_k - p_f), S7_f = C C'; the relative factors
    (srx, srq), state and manifold update are the Tracker's, and each of the 10 iterations takes the exact Gauss-Newton
    step (not eval.py's literal solve, whose end point has no posterior).  A window's posterior is the inverse of its
    normal matrix at the returned state; slot k's 6 x 6 block, mapped to (t, log q), is cov_k, comparable with
    Localizer.sample's cov.  est per emitted frame: pose7 (slot steps//2, un-normalised as Tracker's), cov = D cov_k D
    with D = diag(pose_s, 1, 1, 1), t_std = sqrt(trace of its translation block), q_std_deg = 2 sqrt(trace of its log q
    block) in degrees -- Localizer.sample's statistics.  All float64 on the device.

    sax and saq keep the reference's meaning, the variance floor of the absolute factors (normalised units).  The
    sampled covariance is added to them, so it matters only where the floors sit below the sampled variances: at the
    reference's default of 1, the floors dominate and the weights barely move.

    Each chunk of max_batch frames replays one CUDA graph, captured per (B, H, W): the Localizer's sampled engine
    launches at the device dropout counter (S consecutive dropout steps per chunk, as Localizer.sample takes them), then
    three tracking launches (csrc/loader.cu, mapnet_track_sample_*: gather, k_pgo_cov, emit).  The eager run before the
    capture uses an explicit dropout step and runs no tracking launch, so it advances neither the dropout counter nor
    the sequence.  Engines, snapshot, refresh(), precision and dropout counter are the Localizer's predictor's.  S as
    Localizer.sample takes it: 2 <= S <= 1024, and a model without dropout raises ValueError.  robust_c as Tracker's, on
    the whitened residual C^-1 (z - p): a frame that is wrong and confident (small Sigma_f) is down-weighted too, and
    each posterior is taken with the weights at the returned state."""

    _API = "mapnet_track_sample"
    _ROW = _lib.TRACK_SAMPLE_ROW

    def __init__(self, localizer, S, steps, skip=1, vo_fc=False, sax=1.0, saq=1.0, srx=1.0, srq=1.0, robust_c=None):
        super(SampledTracker, self).__init__(localizer, steps, skip, vo_fc, sax, saq, srx, srq, robust_c)
        self.S = _check_draws(S, localizer.predictor.droprate)

    @staticmethod
    def _est(rows):
        """the est dict of output rows [n,45]"""
        return dict(pose7=rows[:, :7].contiguous(), cov=rows[:, 7:43].reshape(-1, 6, 6).contiguous(),
                    t_std=rows[:, 43].contiguous(), q_std_deg=rows[:, 44].contiguous())

    def _capture(self, fb, track):
        return _sampled_capture(self.loc, self.S, fb, track)


def _stream_records(seen, streams, lag):
    """The records of one chunk of a multi-stream call (mapnet_track_multi_step's rec): streams int64 [B], the stream
    of each frame in call order; seen int64 [n_streams], each stream's frames before the chunk.  Returns (rec int32
    [B,6], sid int64 [n], fid int64 [n]): a completed window per frame f >= lag of its stream, that of frame f - lag,
    in call order.  Adding np.bincount(streams) to seen gives the counts after the chunk."""
    B = streams.shape[0]
    order = np.argsort(streams, kind="stable")
    srt = streams[order]
    rank = np.empty(B, np.int64)
    rank[order] = np.arange(B) - np.searchsorted(srt, srt, side="left")
    count = np.bincount(streams, minlength=seen.shape[0])[streams]
    frame = seen[streams] + rank
    if B and frame.max() >= 2 ** 31:
        raise ValueError("a stream reached frame 2^31; flush or reset it")
    done = np.flatnonzero(frame >= lag)
    rec = np.full((B, 6), -1, dtype=np.int32)
    rec[:, 0], rec[:, 1], rec[:, 2], rec[:, 3] = streams, rank, count, frame
    rec[done, 4] = np.arange(done.shape[0])
    rec[:done.shape[0], 5] = done
    return rec, streams[done], frame[done] - lag


def _stream_chunks(seen, streams, lag, max_batch):
    """Yields (lo, rec, sid, fid) for each chunk of max_batch frames of a multi-stream call (_stream_records), and
    advances seen (int64 [n_streams], in place) by the chunk's frames once the caller has run it."""
    for lo in range(0, streams.shape[0], max_batch):
        sb = streams[lo:lo + max_batch]
        rec, sid, fid = _stream_records(seen, sb, lag)
        yield (lo, rec, sid, fid)
        seen += np.bincount(sb, minlength=seen.shape[0])


class MultiTracker(Tracker):
    """Tracker for n_streams independent camera streams that share one Localizer: the frames of any streams go through
    the engine as one batch, and one set of tracking launches serves all of them.

        mt = MultiTracker(loc, n_streams=64, steps=7, skip=10, vo_fc=True, sax=1, saq=1, srx=20, srq=20)
        sid, fid, pose7 = mt(frames, vo_poses, streams)     # frames / vo_poses as Tracker takes them; streams: B ints
        now7, sid, fid, pose7 = mt.step(frames, vo_poses, streams)
        first, pose7 = mt.flush(s)          # stream s alone: its last min(lag, seen[s]) frames; starts a new sequence
        mt.reset(); mt.reset(s); mt.seen; mt.lag; mt.close()

    streams gives each frame's stream, an int in [0, n_streams): a list, an ndarray or a CPU integer tensor (an int for
    one [H,W,3] frame).  A stream may appear several times in a call, its frames in call order; streams absent from a
    call are untouched.  Each stream is tracked exactly as a Tracker of the same arguments tracks it: its poses are bit
    for bit what a Tracker fed that stream's frames in order gives (with droprate > 0, from the same per-frame draws).
    (sid, fid, pose7) are the windows the call completes, one row per given frame f >= lag of its stream, for frame
    f - lag of stream sid, in call order; sid and fid are int64 CPU tensors the host knows without waiting for the
    device, pose7 is float64 [n,7] on the device.  step's now7 [B,7] is each given frame's zero-lag pose
    (Tracker.step), in the order given.  seen is each stream's frame count (int64 [n_streams]).

    A call of more than max_batch frames runs in chunks of max_batch, in order, one graph replay each: the engine's
    launches and three tracking launches (csrc/loader.cu, mapnet_track_multi_*), captured per (B, H, W) as Tracker
    captures; the per-frame records (stream, rank, counts, frame index, output row) are built on the host from its own
    counts and copied in with the frames.  All frames of a call share one H x W.  A window whose normal matrix is not
    positive definite marks its own stream only: flush(s) raises np.linalg.LinAlgError for stream s after resetting
    it.  robust_c as Tracker's, for every stream."""

    _API = "mapnet_track_multi"

    def __init__(self, localizer, n_streams, steps, skip=1, vo_fc=False, sax=1.0, saq=1.0, srx=1.0, srq=1.0,
                 robust_c=None):
        super(MultiTracker, self).__init__(localizer, steps, skip, vo_fc, sax, saq, srx, srq, robust_c)
        self.n_streams = _int_arg(n_streams, "n_streams", 1, _lib.MAX_TRACK_STREAMS)
        self.seen = np.zeros(self.n_streams, dtype=np.int64)    # frames of each stream's sequence, mirrored on the device

    def _handle(self):
        if not self.h:
            pr = self.loc.predictor
            sig = (ctypes.c_double * 4)(*self.sigmas)
            _lib.check(getattr(_lib.lib(), self._API + "_create")(ctypes.byref(self.h), self.n_streams, self.steps,
                                                                  self.skip, int(self.vo_fc), pr.max_batch, sig,
                                                                  self.loc._m, self.loc._s), self._API + "_create")
            self._set_robust()
        return self.h

    def _stream_ids(self, streams, B, single):
        """streams as int64 [B]; raises on anything that is not B ints in [0, n_streams)"""
        if torch.is_tensor(streams):
            if streams.device.type != "cpu":
                raise ValueError("streams must be a list, an ndarray or a CPU integer tensor, got a tensor on %s"
                                 % streams.device)
            streams = streams.numpy()
        ids = np.asarray(streams)
        if ids.dtype.kind not in "iu":
            raise ValueError("stream ids must be integers, got %s" % ids.dtype)
        if ids.ndim == 0 and single:
            ids = ids.reshape(1)
        if ids.ndim != 1 or ids.shape[0] != B:
            raise ValueError("streams must hold one id per frame: %d, got shape %s" % (B, tuple(ids.shape)))
        if B and (ids.min() < 0 or ids.max() >= self.n_streams):
            raise ValueError("stream ids must be in [0, %d), got %d .. %d" % (self.n_streams, ids.min(), ids.max()))
        return ids.astype(np.int64)

    def _graph(self, fb, now=False):
        B, H, W = fb.shape[:3]
        graphs = self._now_graphs if now else self._graphs
        g = graphs.get((B, H, W))
        if g is None:
            dev, h, name = self.loc.predictor.device, self._handle(), self._API + "_step"
            vs = torch.zeros((B, 6), dtype=torch.float32, device=dev)
            rs = torch.zeros((B, 6), dtype=torch.int32, device=dev)
            out = torch.empty((B, self._ROW), dtype=torch.float64, device=dev)
            nowb = torch.empty((B, self._ROW), dtype=torch.float64, device=dev) if now else None

            def track(*ins):
                _lib.check(getattr(_lib.lib(), name)(h, *[t.data_ptr() for t in ins], vs.data_ptr(), rs.data_ptr(), B,
                                                     out.data_ptr(), nowb.data_ptr() if now else None,
                                                     _lib.stream_ptr()), name)

            graph, xs, ins = self._capture(fb, track)
            g = graphs[(B, H, W)] = (graph, xs, vs, rs, out, ins, nowb)     # every buffer the graph reads stays alive
        return g

    def _run(self, frames, vo_poses, streams, now):
        """(sid [n], fid [n], rows [n,_ROW], now rows [B,_ROW] or None): the chunks of max_batch frames, one graph
        replay each"""
        self._check_open()
        x, single = self.loc._frames(frames)
        vo = self._vo(vo_poses, x.shape[0], single)
        ids = self._stream_ids(streams, x.shape[0], single)
        pr = self.loc.predictor
        mb = pr.max_batch
        sids, fids, outs, nows = [], [], [], []
        with torch.cuda.device(pr.device):
            for lo, rec, sid, fid in _stream_chunks(self.seen, ids, self.lag, mb):
                fb = x[lo:lo + mb]
                graph, xs, vs, rs, out, _, now7 = self._graph(fb, now)
                xs.copy_(fb, non_blocking=True)
                vs.copy_(vo[lo:lo + mb], non_blocking=True)
                rs.copy_(torch.from_numpy(rec), non_blocking=True)
                graph.replay()
                sids.append(torch.from_numpy(sid))
                fids.append(torch.from_numpy(fid))
                outs.append(out[:sid.shape[0]].clone())
                if now:
                    nows.append(now7.clone())
        cat = lambda ts: ts[0] if len(ts) == 1 else torch.cat(ts, 0)
        return cat(sids), cat(fids), cat(outs), (cat(nows) if now else None)

    @torch.no_grad()
    def __call__(self, frames, vo_poses, streams):
        """-> (sid int64 [n], fid int64 [n], pose7 float64 [n,7] on the device): the windows this call completes"""
        sid, fid, rows, _ = self._run(frames, vo_poses, streams, False)
        return sid, fid, self._est(rows)

    @torch.no_grad()
    def step(self, frames, vo_poses, streams):
        """-> (now7 float64 [B,7] on the device, sid, fid, pose7): row b of now7 is the zero-lag pose of the b-th frame
        given, as Tracker.step defines it for that frame's stream; (sid, fid, pose7) is what __call__ returns"""
        sid, fid, rows, nows = self._run(frames, vo_poses, streams, True)
        return self._est(nows), sid, fid, self._est(rows)

    @torch.no_grad()
    def flush(self, s):
        """-> (first, pose7 [n,7]): stream s's last n = min(lag, seen[s]) frames, their windows clipped at its last
        frame.  Synchronises, starts a new sequence on stream s alone, and raises np.linalg.LinAlgError if a window of
        stream s's sequence that ended was not positive definite."""
        self._check_open()
        s = _int_arg(s, "stream", 0, self.n_streams - 1)
        pr = self.loc.predictor
        first = _first_pending(int(self.seen[s]), self.lag)
        n, failed = int(self.seen[s]) - first, ctypes.c_int(0)
        with torch.cuda.device(pr.device):
            out = torch.empty((max(self.lag, 1), self._ROW), dtype=torch.float64, device=pr.device)
            if self.h:
                L = _lib.lib()
                _lib.check(getattr(L, self._API + "_flush")(self.h, s, out.data_ptr(), _lib.stream_ptr()),
                           self._API + "_flush")
                _lib.check(getattr(L, self._API + "_status")(self.h, s, None, ctypes.byref(failed), _lib.stream_ptr()),
                           self._API + "_status")
        self.reset(s)
        if failed.value:
            raise np.linalg.LinAlgError("pose graph: the normal matrix of a window of stream %d's sequence is not "
                                        "positive definite" % s)
        return first, self._est(out[:n])

    def reset(self, s=None):
        """Start a new sequence on stream s, or on every stream when s is None (stream-ordered)."""
        self._check_open()
        s = -1 if s is None else _int_arg(s, "stream", 0, self.n_streams - 1)
        if self.h:
            with torch.cuda.device(self.loc.predictor.device):
                _lib.check(getattr(_lib.lib(), self._API + "_reset")(self.h, s, _lib.stream_ptr()),
                           self._API + "_reset")
        if s < 0:
            self.seen[:] = 0
        else:
            self.seen[s] = 0


class SampledMultiTracker(MultiTracker):
    """MultiTracker with Monte-Carlo dropout: n_streams camera streams share one Localizer, each frame's S dropout
    draws weigh its pose in its stream's pose graph, and every tracked pose comes with a covariance.

        smt = SampledMultiTracker(loc, S=32, n_streams=64, steps=7, skip=10, vo_fc=True, sax=1e-4, saq=1e-4, srx=20,
                                  srq=20)
        sid, fid, est = smt(frames, vo_poses, streams)  # est = dict(pose7 [n,7], cov [n,6,6], t_std [n], q_std_deg [n])
        now, sid, fid, est = smt.step(frames, vo_poses, streams)    # now: the same dict, one zero-lag row per frame
        first, est = smt.flush(s)       # stream s alone: its last min(lag, seen[s]) frames; starts a new sequence
        smt.reset(); smt.reset(s); smt.seen; smt.lag; smt.close()

    Frames, VO poses, stream ids, the rows a call returns and their order, chunking, flush and reset are MultiTracker's;
    the factor model, sax / saq, S and the est dict are SampledTracker's.  Each stream is tracked exactly as a
    SampledTracker of the same arguments tracks it, given the same per-frame draws: a stream's estimates are bit for
    bit those of a SampledTracker fed that stream's frames' means and covariances in order.  They are not those of a
    SampledTracker fed the same frames, because dropout draws a frame's masks by its row in the engine batch (and by
    the chunk's dropout steps), and a frame's row in a batch of many streams is not its row in a one-stream batch.

    A call of more than max_batch frames runs in chunks of max_batch, in order, one CUDA graph replay each, captured per
    (B, H, W): the Localizer's sampled engine launches at the device dropout counter (S consecutive dropout steps per
    chunk, as SampledTracker takes them), then three tracking launches (csrc/loader.cu, mapnet_track_multi_sample_*:
    gather, k_pgo_cov, emit) for all of the chunk's streams.  The per-frame records are built on the host and copied in
    with the frames.  The eager run before a capture uses an explicit dropout step and makes no tracking launch, so it
    advances neither the dropout counter nor any stream.  A window whose normal matrix or one of whose frames' factor
    covariances is not positive definite marks its own stream only: flush(s) raises np.linalg.LinAlgError for stream s
    after resetting it.  robust_c as SampledTracker's, for every stream."""

    _API = "mapnet_track_multi_sample"
    _ROW = SampledTracker._ROW
    _est = staticmethod(SampledTracker._est)
    _capture = SampledTracker._capture

    def __init__(self, localizer, S, n_streams, steps, skip=1, vo_fc=False, sax=1.0, saq=1.0, srx=1.0, srq=1.0,
                 robust_c=None):
        super(SampledMultiTracker, self).__init__(localizer, n_streams, steps, skip, vo_fc, sax, saq, srx, srq,
                                                  robust_c)
        self.S = _check_draws(S, localizer.predictor.droprate)


def pgo(pred7, vos7, sax=1.0, saq=1.0, srx=1.0, srq=1.0, fc_vos=False, robust_c=None):
    """eval.py:172-178 for all windows at once: pred7 [W,N,7], vos7 [W,N-1,7] -> [W,N,7]; with robust_c, (poses,
    w [W,N]) of the Cauchy-weighted graph (optimize_pose_windows)"""
    return optimize_pose_windows(pred7, vos7, fc_vos=fc_vos, sax=sax, saq=saq, srx=srx, srq=srq, robust_c=robust_c)


def pose_errors(pred7, targ7):
    """eval.py:80-81,193-199: per pose ||t_pred - t_gt|| and the quaternion angular error in degrees
    (common/pose_utils.py:358-368).  Returns (t_err [L], q_err_deg [L]) float64 on the device."""
    p, t = pred7.double(), targ7.double().to(pred7.device)
    t_err = (p[..., :3] - t[..., :3]).norm(dim=-1)
    d = (p[..., 3:] * t[..., 3:]).sum(-1).abs().clamp(-1.0, 1.0)
    return t_err, 2.0 * torch.acos(d) * 180.0 / np.pi


def evaluate_tuples(model, x, targ6, vos7=None, pose_m=None, pose_s=None, batch=32, **sigmas):
    """The whole loop of eval.py:147-199 for a MapNet: x [L,T,3,H,W], targ6 [L,T,6] (log-q targets), vos7 [L,T-1,7]
    or None (no PGO).  Keeps the middle prediction of every tuple.  Returns dict(pred7 [L,7], targ7 [L,7], t_err, q_err)."""
    out6 = predict(model, x, batch)                     # [L,T,6]
    pred = post(out6)                                   # normalised translations, as PGO sees them (eval.py:172-178)
    targ = post(targ6.to(out6.device))
    if vos7 is not None:
        pred = pgo(pred, vos7.to(out6.device), **sigmas)
    return _window_errors(pred, targ, pose_m, pose_s)


def _window_errors(pred, targ, pose_m, pose_s, last=False):
    """eval.py:180-199 on windows pred7, targ7 [L,T,7]: translations un-normalised with pose_m / pose_s (when given),
    the middle pose of every window (the last one when `last`: zero-lag windows) and its errors.  Returns
    dict(pred7 [L,7], targ7 [L,7], t_err, q_err)."""
    if pose_m is not None:
        m = torch.as_tensor(np.asarray(pose_m, dtype=np.float64), device=pred.device)
        s = torch.as_tensor(np.asarray(pose_s, dtype=np.float64), device=pred.device)
        pred = torch.cat((pred[..., :3] * s + m, pred[..., 3:]), -1)
        targ = torch.cat((targ[..., :3] * s + m, targ[..., 3:]), -1)
    mid = pred.shape[1] - 1 if last else pred.shape[1] // 2     # eval.py:183-185 (py2 integer division)
    p_mid, t_mid = pred[:, mid], targ[:, mid]
    t_err, q_err = pose_errors(p_mid, t_mid)
    return dict(pred7=p_mid, targ7=t_mid, t_err=t_err, q_err=q_err)


def _frame_runners(pr, net, keys, H, W, dev, quiet=()):
    """{(frames, slot): (static input [n,3,H,W], run(), static output [n,6])} for keys [(n, slot)], created in that
    order: Predictor graphs, or the live eval forward of `net` on plain buffers when there is no Predictor.  The graphs
    of `quiet` keys are captured after an eager run without dropout, which leaves the engine's dropout counter alone."""
    runners = {}
    for n, s in keys:
        if pr is not None:
            graph, xs, ps = pr._graph(n, H, W, slot=s, warm_droprate=0.0 if (n, s) in quiet else None)
            runners[(n, s)] = (xs, graph.replay, ps)
        else:
            xs = torch.empty((n, 3, H, W), dtype=torch.float32, device=dev)
            ps = torch.empty((n, 6), dtype=torch.float32, device=dev)
            runners[(n, s)] = (xs, (lambda xs=xs, ps=ps: ps.copy_(net(xs))), ps)
    return runners


def _model_for(model, ds, what):
    """(Predictor or None, network, device) of a model or Predictor that runs over the DeviceDataset ds"""
    pr = model if isinstance(model, Predictor) else None
    net = pr.net if pr is not None else (model.mapnet if hasattr(model, "mapnet") else model)
    dev = pr.device if pr is not None else next(net.parameters()).device
    if dev != ds.device:
        raise RuntimeError("geomapnet_b200.inference.%s has no CPU path: the model is on %s and the dataset on %s; both "
                           "must be on one CUDA device" % (what, dev, ds.device))
    if pr is not None:
        pr._check_frames(ds.Ho, ds.Wo)
    return pr, net, dev


@contextlib.contextmanager
def _eval_pass(model, pr, net, dev, max_batch):
    """The body of an evaluation pass on dev with the network in eval mode.  Yields the Predictor that runs it: pr, or
    for a live bf16 / tc_split model a temporary one of max_batch frames, closed at the end; None for any other live
    model, which runs its own eval forward.  The network's training flag is restored at the end."""
    own = pr is None and net.precision in ("bf16", "tc_split")
    if own:
        pr = Predictor(model, max_batch=max_batch)
    was_training = net.training
    net.eval()
    try:
        with torch.cuda.device(dev):
            yield pr
    finally:
        net.train(was_training)
        if own:
            torch.cuda.current_stream(dev).synchronize()     # the temporary engines are freed once their work is done
            pr.close()


def _predict_frames(pr, net, ds, frames, B, n_slots, dev):
    """pred [F,6] of the cache frames `frames` (host int32 [F]), B frames per forward, in order.  With two slots the
    next chunk is assembled on a side stream while this one runs; with one the forwards follow each other."""
    F = frames.shape[0]
    chunks = [(lo, min(lo + B, F)) for lo in range(0, F, B)]
    n_slots = n_slots if len(chunks) > 1 else 1
    keys = [(hi - lo, k % n_slots) for k, (lo, hi) in enumerate(chunks)]
    runners = _frame_runners(pr, net, [(n, s) for n in sorted({n for n, _ in keys}) for s in range(n_slots)],
                             ds.Ho, ds.Wo, dev)
    pipe = SidePipeline(dev)
    pred6 = torch.empty((F, 6), dtype=torch.float32, device=dev)

    def fill(k):
        lo, hi = chunks[k]
        pipe.fill(keys[k], lambda: ds.assemble_frames(frames[lo:hi], runners[keys[k]][0]))

    fill(0)
    for k, (lo, hi) in enumerate(chunks):
        _, run, out = runners[keys[k]]
        pipe.take(keys[k])
        run()
        pipe.read(keys[k]).record(torch.cuda.current_stream(dev))
        pred6[lo:hi].copy_(out)
        if k + 1 < len(chunks):
            fill(k + 1)
    return pred6


def _predict_batches(pr, net, ds, batches, droprate, dev):
    """(pred [I*T,6], targ [I*T,6]) of a pass's batch records, in order: each batch is assembled, with its ColorJitter
    records, straight into the input of its forward on a side stream (two slots) while the previous batch runs.

    With dropout the masks follow the Predictor's own sequence of forwards, and that sequence is the one calling the
    Predictor batch by batch makes: a batch size met for the first time costs one eager forward, before its first
    replay.  The graphs of the second slot are captured without touching the dropout counter, and the eager forward
    of a new size that is not the first batch's is run just before that size's first replay."""
    T, H, W = ds.frames_per_item, ds.Ho, ds.Wo
    sizes = [b[3] * T for b in batches]
    n_slots = 2 if len(batches) > 1 else 1
    keys = [(n, k % n_slots) for k, n in enumerate(sizes)]
    order = list(dict.fromkeys([(n, 0) for n in sizes] + keys))      # each size's own graph first, as the Predictor
    counted = pr is not None and droprate > 0
    new = {n for n in sizes if (n, H, W) not in pr._graphs} if counted else set()
    runners = _frame_runners(pr, net, order, H, W, dev, quiet=set(order[1:]) if counted else ())
    pending = new - {sizes[0]}          # the eager forwards still to run, one per new size
    I = sum(b[3] for b in batches)
    pred = torch.empty((I * T, 6), dtype=torch.float32, device=dev)
    targ = torch.empty((I * T, 6), dtype=torch.float32, device=dev)
    pipe = SidePipeline(dev)
    rows = np.cumsum([0] + sizes)

    def fill(k):
        xs_shape, t_shape = ds.batch_shapes(batches[k][3])
        pipe.fill(keys[k], lambda: ds.assemble(batches[k], runners[keys[k]][0].view(xs_shape),
                                               targ[rows[k]:rows[k + 1]].view(t_shape)))

    fill(0)
    for k in range(len(batches)):
        xs, run, out = runners[keys[k]]
        pipe.take(keys[k])
        if sizes[k] in pending:
            pending.discard(sizes[k])
            pr._engine(H, W).forward(xs, out, pr.droprate, pr.seed)
        run()
        pipe.read(keys[k]).record(torch.cuda.current_stream(dev))
        pred[rows[k]:rows[k + 1]].copy_(out)
        if k + 1 < len(batches):
            fill(k + 1)
    return pred, targ


def _sample_frames(pr, ds, frames, S, dev):
    """(mean [F,6], cov [F,36]) float64 of the S dropout draws of each cache frame `frames` (host int32 [F]): chunks of
    the Predictor's max_batch frames in order, each taking S consecutive dropout steps, as Predictor.sample on those
    chunks.  The next chunk is assembled on a side stream (a second graph slot) while this one runs; a chunk larger
    than the dataset's assembly is assembled in parts."""
    F, B, cap = frames.shape[0], pr.max_batch, ds.max_batch * ds.frames_per_item
    chunks = [(lo, min(lo + B, F)) for lo in range(0, F, B)]
    n_slots = 2 if len(chunks) > 1 else 1
    keys = [(hi - lo, k % n_slots) for k, (lo, hi) in enumerate(chunks)]
    graphs = {key: pr._sample_graph(key[0], ds.Ho, ds.Wo, S, slot=key[1]) for key in dict.fromkeys(keys)}
    pipe = SidePipeline(dev)
    mean = torch.empty((F, 6), dtype=torch.float64, device=dev)
    cov = torch.empty((F, 36), dtype=torch.float64, device=dev)

    def fill(k):
        lo, hi = chunks[k]
        xs = graphs[keys[k]][1]
        pipe.fill(keys[k], lambda: [ds.assemble_frames(frames[a:min(a + cap, hi)], xs[a - lo:min(a + cap, hi) - lo])
                                    for a in range(lo, hi, cap)])

    fill(0)
    for k, (lo, hi) in enumerate(chunks):
        graph, _, o = graphs[keys[k]]
        pipe.take(keys[k])
        graph.replay()
        pipe.read(keys[k]).record(torch.cuda.current_stream(dev))
        mean[lo:hi].copy_(o["mean"])
        cov[lo:hi].copy_(o["cov"].view(-1, 36))
        if k + 1 < len(chunks):
            fill(k + 1)
    return mean, cov


def _evaluate_sampled(pr, ds, S, vo, vo_fc, zero_lag, pose_m, pose_s, sig, dev, robust_c=None):
    """evaluate_sequence(samples=S) once the arguments are checked: the draws of every frame, then one gather, one
    k_pgo_cov and one emit (with VO poses) or one emit, and one host synchronisation for the PGO status"""
    L_lib = _lib.lib()
    # every frame of the sequence is the kept slot of its own window (the middle slot's offset is 0, and a zero-lag
    # window ends at its frame), so the draws are queued first and the host builds the window tables after them
    frames = np.arange(ds.L, dtype=np.int32)
    mean, cov = _sample_frames(pr, ds, frames, S, dev)
    tab = ds.eval_tables(unique=True, vo_fc=vo_fc, zero_lag=zero_lag)
    if not np.array_equal(tab["frames"], frames):
        raise RuntimeError("evaluate_sequence: the windows do not hold every frame of the sequence")
    windows, slots = tab["windows"], tab["slots"]
    L, T = windows.shape
    F = frames.shape[0]
    keep = T - 1 if zero_lag else T // 2
    f64 = dict(dtype=torch.float64, device=dev)
    opt7 = post36 = status = None
    if vo:
        E = tab["vo_rows"].shape[1]
        p7, s7 = torch.empty((L * T, 7), **f64), torch.empty((L * T, 49), **f64)
        vos7, opt7, post36 = torch.empty((L * E, 7), **f64), torch.empty((L * T, 7), **f64), torch.empty((L * T, 36), **f64)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        _lib.check(L_lib.mapnet_eval_sample_windows(
            mean.data_ptr(), cov.data_ptr(), F, sig["sax"], sig["saq"], ds.vo_poses.data_ptr(), ds.poses.shape[0],
            slots.ctypes.data, L * T, tab["vo_rows"].ctypes.data, L * E, p7.data_ptr(), s7.data_ptr(), vos7.data_ptr(),
            _lib.stream_ptr()), "mapnet_eval_sample_windows")
        if robust_c is None:
            _lib.check(L_lib.mapnet_pgo_optimize_cov(p7.data_ptr(), s7.data_ptr(), vos7.data_ptr(), opt7.data_ptr(),
                                                     post36.data_ptr(), L, T, 1 if vo_fc else 0, sig["srx"], sig["srq"],
                                                     10, status.data_ptr(), _lib.stream_ptr()), "mapnet_pgo_optimize_cov")
        else:
            w = torch.empty((L, T), **f64)
            _lib.check(L_lib.mapnet_pgo_optimize_cov_robust(
                p7.data_ptr(), s7.data_ptr(), vos7.data_ptr(), opt7.data_ptr(), post36.data_ptr(), L, T,
                1 if vo_fc else 0, sig["srx"], sig["srq"], 10, robust_c, w.data_ptr(), status.data_ptr(),
                _lib.stream_ptr()), "mapnet_pgo_optimize_cov_robust")
    m = s = None
    if pose_m is not None:
        m = (ctypes.c_double * 3)(*[float(v) for v in np.asarray(pose_m).reshape(3)])
        s = (ctypes.c_double * 3)(*[float(v) for v in np.asarray(pose_s).reshape(3)])
    out = torch.empty((L, SampledTracker._ROW), **f64)
    targ7, d2, u, nll = torch.empty((L, 7), **f64), torch.empty((L, 3), **f64), torch.empty((L, 3), **f64), \
        torch.empty(L, **f64)
    frame_k = np.ascontiguousarray(windows[:, keep])
    slot_k = np.ascontiguousarray(slots[:, keep])
    _lib.check(L_lib.mapnet_eval_sample_emit(
        mean.data_ptr(), cov.data_ptr(), F, opt7.data_ptr() if vo else None, post36.data_ptr() if vo else None, T, keep,
        ds.poses.data_ptr(), ds.poses.shape[0], frame_k.ctypes.data, slot_k.ctypes.data, L, m, s, out.data_ptr(),
        targ7.data_ptr(), d2.data_ptr(), u.data_ptr(), nll.data_ptr(), _lib.stream_ptr()), "mapnet_eval_sample_emit")
    if vo and int(status.item()) != 0:                      # the sequence's one host synchronisation
        raise np.linalg.LinAlgError("pose graph: the normal matrix of a window of the sequence is not positive definite")
    est = SampledTracker._est(out)
    t_err, q_err = pose_errors(est["pose7"], targ7)
    res = dict(pred7=est["pose7"], targ7=targ7, t_err=t_err, q_err=q_err, n_frames=F, cov=est["cov"],
               t_std=est["t_std"], q_std_deg=est["q_std_deg"], d2=d2, u=u, nll=nll)
    if robust_c is not None:
        res["w"] = w[:, keep].contiguous()
    return res


@torch.no_grad()
def evaluate_sequence(model, dataset, pose_m=None, pose_s=None, vo_fc=False, zero_lag=False, samples=None,
                      robust_c=None, **sigmas):
    """The whole loop of scripts/eval.py:117-199 over a device-resident sequence: the windows of MF(steps, skip,
    variable_skip, no_duplicates=False) -- or single frames when dataset.steps is None -- one per frame index, in index
    order.  Returns what evaluate_tuples returns (pred7 [L,7], targ7 [L,7], t_err, q_err: the middle frame of each
    window) and n_frames, the number of frames that went through the network.

    zero_lag=True evaluates the pose a live tracker has for each frame when it arrives (Tracker.step): item i's window
    is the one that ends at frame i, MF.get_indices(i - lag) with lag = (steps - 1 - steps//2) * skip, and its last
    slot is kept.  It needs dataset.steps and fixed skips (no variable_skip), else ValueError before any launch.

    model: a PoseNet / MapNet or a Predictor (any precision).  A live model whose precision a Predictor supports is
    run by a temporary Predictor; any other runs its own eval forward.  dataset: a DeviceDataset without ColorJitter;
    its poses are the targets.  With dataset.vo_poses, each window's VOs (calc_vos_safe of the VO-library poses, or
    calc_vos_safe_fc when vo_fc) drive the pose-graph optimisation, with the covariances `sigmas` (sax, saq, srx, srq).

    In eval mode BatchNorm uses running statistics, so a frame's pose does not depend on the rest of its window:
    with droprate == 0 every distinct frame goes through the network once, in chunks of the Predictor's max_batch,
    and the windows are rebuilt from the per-frame poses.  With droprate > 0 (the reference's dropout is active at
    eval) each window's frames go through the network together, one window per forward, as in the reference's loop.
    Chunk k+1 is assembled on a side stream while chunk k runs.  variable_skip draws from np.random as the
    reference's DataLoader(shuffle=False) does.

    samples=S (an int, 2 <= S <= 1024; the model must have dropout) evaluates Monte-Carlo dropout, SampledTracker's
    model, on the labelled sequence.  Every distinct frame goes through the sampled engine once, in frame order, in
    chunks of the Predictor's max_batch frames, each chunk taking S consecutive dropout steps (Predictor.sample on
    those chunks).  Each frame's S draws are shared by every window that holds it, as the sampled trackers share them,
    where eval.py would draw each window's frames anew: with the same chunks, seed and dropout counter the estimates
    are bit for bit those of a SampledTracker fed the same frames (its step() rows under zero_lag).  With
    dataset.vo_poses each window slot gets the frame's factor (mean pose, S7 = A Sigma A' + the floors sax / saq) and
    all windows are solved in one covariance-weighted PGO launch (srx / srq); the kept slot's posterior is the
    estimate.  Without VO poses each item's estimate is its frame's own sampled mean and covariance.  The result
    adds, per item, SampledTracker's cov [L,6,6] (D cov D with D = diag(pose_s, 1, 1, 1)), t_std and q_std_deg, and
    the calibration of that covariance against the target: d2 [L,3], the squared Mahalanobis distances of the error
    (t^ - t, qlog(q^) - qlog(sign(q^.q) q)) over all 6 DoF, the translation block and the log q block; u [L,3], their
    chi-square CDFs (6, 3 and 3 degrees of freedom), each uniform on [0, 1] for a calibrated model, so the coverage at
    level p is (u <= p).mean(0); and nll [L], the 6-DoF Gaussian negative log-likelihood.  A covariance (block) that is
    not positive definite gives NaN there: without PGO the 6-DoF column always is for S <= 6, since S draws span at
    most S - 1 dimensions.  A window whose normal matrix (or a slot's S7) is not positive definite raises
    np.linalg.LinAlgError.  The model is a Predictor of any precision or a live bf16 / tc_split model (run by a
    temporary Predictor); a live model without a sampled engine raises ValueError.  Launches past the per-chunk
    assembly and engine replay: one gather, one k_pgo_cov and one emit (one emit without VO poses), and one host
    synchronisation.

    robust_c=c (a finite number > 0, in sigmas; needs dataset.vo_poses) gives the absolute factors of every window the
    Cauchy loss of scale c (common.pgo: optimize_pose_windows / optimize_pose_windows_cov with robust_c), on the point
    path and with samples, zero_lag and variable skips alike, and the result gains w [L], the final weight of each
    item's kept slot: near 1 for a frame its window agrees with, near 0 for one it overrules.  The trackers given the
    same robust_c produce these poses bit for bit.  A bad robust_c raises ValueError before anything is launched."""
    from .data.loader import DeviceDataset
    robust_c = check_robust_c(robust_c)
    ds = dataset
    if not isinstance(ds, DeviceDataset):
        raise TypeError("evaluate_sequence needs a geomapnet_b200.data.DeviceDataset, got %s" % type(ds).__name__)
    if ds.jitter is not None:
        raise ValueError("evaluate_sequence: the dataset applies ColorJitter; build it with color_jitter=0")
    if ds.online:
        raise ValueError("evaluate_sequence: MFOnline datasets are not evaluation sequences")
    if not ds.h:
        raise RuntimeError("evaluate_sequence: the dataset is closed")
    if zero_lag and (ds.steps is None or ds.variable_skip):
        raise ValueError("evaluate_sequence: zero_lag needs a windowed dataset (steps) with fixed skips; got %s" %
                         ("single frames" if ds.steps is None else "variable_skip"))
    pr, net, dev = _model_for(model, ds, "evaluate_sequence")
    vo = ds.vo_poses is not None
    T = 1 if ds.steps is None else ds.steps
    if vo and T < 2:
        raise ValueError("pose-graph optimisation needs windows of >= 2 frames (dataset.steps)")
    if vo_fc and not vo:
        raise ValueError("vo_fc: the dataset has no vo_poses")
    if robust_c is not None and not vo:
        raise ValueError("robust_c weighs the absolute factors of a pose graph: the dataset has no vo_poses")
    droprate = pr.droprate if pr is not None else float(net.droprate)
    cap = ds.max_batch * ds.frames_per_item                  # frames the dataset's cache assembles per call
    if samples is not None:
        S = _check_draws(samples, droprate)
        if pr is None and net.precision not in ("bf16", "tc_split"):
            raise ValueError("evaluate_sequence: samples needs a Predictor or a bf16 / tc_split model (a %s model has "
                             "no sampled engine)" % net.precision)
        sig = dict(sax=1.0, saq=1.0, srx=1.0, srq=1.0)
        for k, v in sigmas.items():
            if k not in sig:
                raise TypeError("evaluate_sequence: unknown covariance %r (sax, saq, srx, srq)" % k)
            sig[k] = float(v)
        if not all(v > 0 for v in sig.values()):
            raise ValueError("sax, saq, srx, srq must be positive, got %s" % (sig,))
        with _eval_pass(model, pr, net, dev, min(64, cap)) as pr:
            return _evaluate_sampled(pr, ds, S, vo, vo_fc, zero_lag, pose_m, pose_s, sig, dev, robust_c)
    B = min(pr.max_batch if pr is not None else 64, cap)
    if droprate > 0:
        if B < T:
            raise ValueError("droprate > 0 runs one window of %d frames per forward; max_batch allows %d" % (T, B))
        B = T
    tab = ds.eval_tables(unique=droprate == 0, vo_fc=vo_fc, zero_lag=zero_lag)
    frames, L = tab["frames"], tab["windows"].shape[0]
    F = frames.shape[0]
    with _eval_pass(model, pr, net, dev, min(64, cap)) as pr:
        # two input buffers, so that the next chunk is assembled while this one runs; one when the forward draws
        # dropout masks, which then follow the Predictor's own sequence of forwards
        pred6 = _predict_frames(pr, net, ds, frames, B, 2 if droprate == 0 else 1, dev)
        E = tab["vo_rows"].shape[1]
        pred7 = torch.empty((L, T, 7), dtype=torch.float64, device=dev)
        targ7 = torch.empty_like(pred7)
        vos7 = torch.empty((L, E, 7), dtype=torch.float64, device=dev) if vo else None
        _lib.check(_lib.lib().mapnet_eval_windows(
            pred6.data_ptr(), F, ds.poses.data_ptr(), ds.vo_poses.data_ptr() if vo else None, ds.poses.shape[0],
            tab["windows"].ctypes.data, tab["slots"].ctypes.data, L * T,
            tab["vo_rows"].ctypes.data if vo else None, L * E if vo else 0, pred7.data_ptr(), targ7.data_ptr(),
            vos7.data_ptr() if vo else None, _lib.stream_ptr()), "mapnet_eval_windows")
        if robust_c is None:
            out = _window_errors(pgo(pred7, vos7, fc_vos=vo_fc, **sigmas) if vo else pred7, targ7, pose_m, pose_s,
                                 last=zero_lag)
        else:
            opt, w = pgo(pred7, vos7, fc_vos=vo_fc, robust_c=robust_c, **sigmas)
            out = _window_errors(opt, targ7, pose_m, pose_s, last=zero_lag)
            out["w"] = w[:, T - 1 if zero_lag else T // 2].contiguous()
    return dict(out, n_frames=F)


@torch.no_grad()
def validate(model, loader, criterion):
    """The validation pass of common/train.py:214-250 over a DeviceLoader: every batch of DataLoader(val_set,
    batch_size, shuffle) through the eval-mode model and `criterion`.  Returns (avg, losses): the per-batch losses as
    floats in batch order and their plain mean, the reference's AverageMeter.avg (the last, partial batch weighs as
    much as any other).  The batch records are drawn with loader.batches(), so the torch and numpy RNG streams advance
    as the reference's DataLoader advances them (sampler permutation, ColorJitter, variable_skip).

    model: a PoseNet / MapNet or a Predictor, handled as evaluate_sequence handles it; the model's training flag is
    left as it was.  loader: over a single-frame or MF DeviceDataset.  criterion: PoseNetCriterion for single frames,
    MapNetCriterion for MF tuples; its sax, saq, srx, srq are read on the device (scripts/train.py default-constructs
    the validation criterion, all four 0).

    With droprate == 0 and no ColorJitter each distinct frame of the pass goes through the network once (a frame's
    eval-mode pose does not depend on the other frames of its batch).  Otherwise each batch is assembled with its
    jitter records straight into a forward input and run on its own, in batch order; dropout masks then follow the
    Predictor's sequence of forwards as when it is called batch by batch.  All batch losses come from one
    mapnet_batch_losses launch, bit for bit what the criterion returns per batch, and the pass synchronises with the
    host once, at its end."""
    from .common.criterion import MapNetCriterion, PoseNetCriterion
    from .data.loader import DeviceLoader
    if not isinstance(loader, DeviceLoader):
        raise TypeError("validate needs a geomapnet_b200.data.DeviceLoader, got %s" % type(loader).__name__)
    ds = loader.dataset
    if ds.online:
        raise ValueError("validate: MFOnline datasets are not validated (scripts/train.py builds no val_set for them)")
    mode = "posenet" if isinstance(criterion, PoseNetCriterion) else ("mapnet" if isinstance(criterion, MapNetCriterion)
                                                                     else None)
    if mode is None or (mode == "posenet") != (ds.steps is None):
        raise ValueError("validate: a %s does not fit the dataset's %s; use PoseNetCriterion for single frames and "
                         "MapNetCriterion for MF tuples" % (type(criterion).__name__,
                                                            "single frames" if ds.steps is None else "MF tuples"))
    if not ds.h:
        raise RuntimeError("validate: the dataset is closed")
    pr, net, dev = _model_for(model, ds, "validate")
    droprate = pr.droprate if pr is not None else float(net.droprate)
    unique = droprate == 0 and ds.jitter is None
    T = ds.frames_per_item
    per_batch = loader.batch_size * T
    if not unique and pr is not None and per_batch > pr.max_batch:
        raise ValueError("with dropout or ColorJitter one batch of %d frames runs per forward; the Predictor's "
                         "max_batch allows %d" % (per_batch, pr.max_batch))
    cap = ds.max_batch * T                                   # frames the dataset's cache assembles per call
    tab = ds.val_tables(loader.batch_size, loader.shuffle, unique)
    n_batches = len(tab["batches"])
    with _eval_pass(model, pr, net, dev, min(64, cap) if unique else max(64, per_batch)) as pr:
        zero = torch.zeros(1, dtype=torch.float32, device=dev)
        s4 = torch.cat([getattr(criterion, k).detach().float().to(dev).reshape(1) if hasattr(criterion, k) else zero
                        for k in ("sax", "saq", "srx", "srq")])
        if unique:
            pred = _predict_frames(pr, net, ds, tab["frames"], min(pr.max_batch if pr is not None else 64, cap), 2, dev)
            targ, pred_rows, targ_rows = ds.poses, tab["pred_rows"], tab["targ_rows"]
        else:
            pred, targ = _predict_batches(pr, net, ds, tab["batches"], droprate, dev)
            pred_rows = targ_rows = tab["pred_rows"]           # the identity: pred and targ are in loader order
        out = torch.empty(n_batches, dtype=torch.float32, device=dev)
        _lib.check(_lib.lib().mapnet_batch_losses(
            _lib.LOSS_MODE[mode], pred.data_ptr(), pred.shape[0], targ.data_ptr(), targ.shape[0],
            pred_rows.ctypes.data, targ_rows.ctypes.data, T, tab["batch_items"].ctypes.data, n_batches,
            s4.data_ptr(), out.data_ptr(), _lib.stream_ptr()), "mapnet_batch_losses")
        losses = out.cpu().tolist()                             # the pass's one host synchronisation
    return sum(losses) / len(losses), losses
