"""Batched inference + pose-graph optimisation: the evaluation loop of the reference on the GPU.

Host-side mirror of /root/reference/scripts/eval.py:137-199.  The reference runs batch size 1 ("batch_size MUST be 1",
:136-138), moves every prediction to numpy, applies qexp per pose in Python, optionally runs a dense numpy PGO per
frame and keeps the middle prediction of each tuple.  Here: ``predict`` runs the eval-mode forward in batches of tuples
through the same fprop engines as training (BatchNorm running statistics, no dropout at eval -- see note), ``post`` does
qexp + un-normalisation for all poses in one launch, ``pgo`` optimises all windows in one launch (csrc/pgo.cu), and
``pose_errors`` gives the translation / rotation errors eval.py prints (:193-199).

Note on dropout: models/posenet.py:68-69 calls F.dropout without ``training=``, so the reference drops features at eval
time too whenever droprate > 0; scripts/eval.py builds the model with the ini's dropout.  ``predict`` follows the
module (geomapnet_b200.models.PoseNet keeps that behaviour); pass a model built with droprate=0 for deterministic poses.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .common.pgo import optimize_pose_windows

__all__ = ["Predictor", "predict", "post", "pgo", "pose_errors", "evaluate_tuples"]


class Predictor(object):
    """Frozen eval-mode predictor of a PoseNet or MapNet: a snapshot of its weights and BatchNorm running statistics,
    run by the inference engine (csrc/infer.cu) with BatchNorm, residual and ReLU fused into the conv epilogues.

        pr = Predictor(model, max_batch=64)
        poses = pr(x)       # [L,3,H,W] -> [L,6];  [L,T,3,H,W] -> [L,T,6];  max_batch frames per engine call
        pr.refresh()        # take a new snapshot of the model's current parameters / running statistics
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

    def _run(self, xb):
        """pred [B,6] for frames xb [B,3,H,W] (B <= max_batch): graph replay, captured on the first call of a shape."""
        B, _, H, W = xb.shape
        key = (B, H, W)
        g = self._graphs.get(key)
        if g is None:
            eng = self._engine(H, W)
            xs = torch.empty((B, 3, H, W), dtype=torch.float32, device=self.device)
            ps = torch.empty((B, 6), dtype=torch.float32, device=self.device)
            xs.copy_(xb)
            cur = torch.cuda.current_stream(self.device)
            side = torch.cuda.Stream(self.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):        # eager run first: tile plans, tensor maps, kernel attributes
                eng.forward(xs, ps, self.droprate, self.seed)
            cur.wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                eng.forward(xs, ps, self.droprate, self.seed)
            g = self._graphs[key] = (graph, xs, ps)
        graph, xs, ps = g
        xs.copy_(xb)
        graph.replay()
        return ps.clone()

    @torch.no_grad()
    def __call__(self, x):
        if not x.is_cuda:
            raise RuntimeError("geomapnet_b200.inference.Predictor has no CPU path: input must be a CUDA tensor "
                               "(got %s)" % x.device)
        if x.dim() not in (4, 5) or x.shape[-3] != 3:
            raise ValueError("expected input [L,3,H,W] or [L,T,3,H,W], got %s" % (tuple(x.shape),))
        if x.shape[0] < 1 or (x.dim() == 5 and x.shape[1] < 1):
            raise ValueError("empty batch")
        if self._params is None:
            raise RuntimeError("Predictor is closed")
        if self._calib is not None and tuple(x.shape[-2:]) != tuple(self._calib.shape[-2:]):
            raise ValueError("this fp8 Predictor was calibrated at %dx%d, got frames of %dx%d"
                             % (self._calib.shape[-2], self._calib.shape[-1], x.shape[-2], x.shape[-1]))
        frames = x.reshape(-1, *x.shape[-3:])
        if frames.dtype != torch.float32:
            frames = frames.float()
        with torch.cuda.device(self.device):
            outs = [self._run(frames[i:i + self.max_batch]) for i in range(0, frames.shape[0], self.max_batch)]
        out = torch.cat(outs, 0)
        return out.view(*x.shape[:-3], 6)

    def close(self):
        self._graphs.clear()
        for eng in self._engines.values():
            eng.close()
        self._engines.clear()
        self._params = self._bufs = self._calib = None


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


def pgo(pred7, vos7, sax=1.0, saq=1.0, srx=1.0, srq=1.0, fc_vos=False):
    """eval.py:172-178 for all windows at once: pred7 [W,N,7], vos7 [W,N-1,7] -> [W,N,7]"""
    return optimize_pose_windows(pred7, vos7, fc_vos=fc_vos, sax=sax, saq=saq, srx=srx, srq=srq)


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
    T = out6.shape[1]
    pred = post(out6)                                   # normalised translations, as PGO sees them (eval.py:172-178)
    targ = post(targ6.to(out6.device))
    if vos7 is not None:
        pred = pgo(pred, vos7.to(out6.device), **sigmas)
    if pose_m is not None:
        m = torch.as_tensor(np.asarray(pose_m, dtype=np.float64), device=pred.device)
        s = torch.as_tensor(np.asarray(pose_s, dtype=np.float64), device=pred.device)
        pred = torch.cat((pred[..., :3] * s + m, pred[..., 3:]), -1)
        targ = torch.cat((targ[..., :3] * s + m, targ[..., 3:]), -1)
    mid = T // 2                                        # eval.py:183-185 (py2 integer division)
    p_mid, t_mid = pred[:, mid], targ[:, mid]
    t_err, q_err = pose_errors(p_mid, t_mid)
    return dict(pred7=p_mid, targ7=t_mid, t_err=t_err, q_err=q_err)
