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
import ctypes

import numpy as np
import torch

from . import _lib
from .common.pgo import optimize_pose_windows

__all__ = ["Predictor", "predict", "post", "pgo", "pose_errors", "evaluate_tuples", "evaluate_sequence", "validate"]


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

    def _run(self, xb):
        """pred [B,6] for frames xb [B,3,H,W] (B <= max_batch): graph replay, captured on the first call of a shape."""
        graph, xs, ps = self._graph(xb.shape[0], xb.shape[2], xb.shape[3], xb)
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
    if pr is not None and pr._params is None:
        raise RuntimeError("Predictor is closed")
    if pr is not None and pr._calib is not None and tuple(pr._calib.shape[-2:]) != (ds.Ho, ds.Wo):
        raise ValueError("this fp8 Predictor was calibrated at %dx%d, the dataset's frames are %dx%d"
                         % (pr._calib.shape[-2], pr._calib.shape[-1], ds.Ho, ds.Wo))
    return pr, net, dev


def _predict_frames(pr, net, ds, frames, B, n_slots, dev):
    """pred [F,6] of the cache frames `frames` (host int32 [F]), B frames per forward, in order.  With two slots the
    next chunk is assembled on a side stream while this one runs; with one the forwards follow each other."""
    F = frames.shape[0]
    chunks = [(lo, min(lo + B, F)) for lo in range(0, F, B)]
    n_slots = n_slots if len(chunks) > 1 else 1
    runners = _frame_runners(pr, net, [(n, s) for n in sorted({hi - lo for lo, hi in chunks}) for s in range(n_slots)],
                             ds.Ho, ds.Wo, dev)
    cur = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(cur)
    read = {k: torch.cuda.Event() for k in runners}
    ready = torch.cuda.Event()
    pred6 = torch.empty((F, 6), dtype=torch.float32, device=dev)

    def launch(k):
        lo, hi = chunks[k]
        key = (hi - lo, k % n_slots)
        side.wait_event(read[key])                   # the previous forward from this buffer has read it
        with torch.cuda.stream(side):
            ds.assemble_frames(frames[lo:hi], runners[key][0])
        ready.record(side)
        return key

    key = launch(0)
    for k in range(len(chunks)):
        cur.wait_event(ready)
        _, run, out = runners[key]
        run()
        read[key].record(cur)
        lo, hi = chunks[k]
        pred6[lo:hi].copy_(out)
        if k + 1 < len(chunks):
            key = launch(k + 1)
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
    cur = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(cur)
    read = {k: torch.cuda.Event() for k in runners}
    ready = torch.cuda.Event()
    rows = np.cumsum([0] + sizes)

    def launch(k):
        n = batches[k][3]
        xs_shape, t_shape = ds.batch_shapes(n)
        side.wait_event(read[keys[k]])
        with torch.cuda.stream(side):
            ds.assemble(batches[k], runners[keys[k]][0].view(xs_shape), targ[rows[k]:rows[k + 1]].view(t_shape))
        ready.record(side)

    launch(0)
    for k in range(len(batches)):
        cur.wait_event(ready)
        xs, run, out = runners[keys[k]]
        if sizes[k] in pending:
            pending.discard(sizes[k])
            pr._engine(H, W).forward(xs, out, pr.droprate, pr.seed)
        run()
        read[keys[k]].record(cur)
        pred[rows[k]:rows[k + 1]].copy_(out)
        if k + 1 < len(batches):
            launch(k + 1)
    return pred, targ


@torch.no_grad()
def evaluate_sequence(model, dataset, pose_m=None, pose_s=None, vo_fc=False, **sigmas):
    """The whole loop of scripts/eval.py:117-199 over a device-resident sequence: the windows of MF(steps, skip,
    variable_skip, no_duplicates=False) -- or single frames when dataset.steps is None -- one per frame index, in index
    order.  Returns what evaluate_tuples returns (pred7 [L,7], targ7 [L,7], t_err, q_err: the middle frame of each
    window) and n_frames, the number of frames that went through the network.

    model: a PoseNet / MapNet or a Predictor (any precision).  A live model whose precision a Predictor supports is
    run by a temporary Predictor; any other runs its own eval forward.  dataset: a DeviceDataset without ColorJitter;
    its poses are the targets.  With dataset.vo_poses, each window's VOs (calc_vos_safe of the VO-library poses, or
    calc_vos_safe_fc when vo_fc) drive the pose-graph optimisation, with the covariances `sigmas` (sax, saq, srx, srq).

    In eval mode BatchNorm uses running statistics, so a frame's pose does not depend on the rest of its window:
    with droprate == 0 every distinct frame goes through the network once, in chunks of the Predictor's max_batch,
    and the windows are rebuilt from the per-frame poses.  With droprate > 0 (the reference's dropout is active at
    eval) each window's frames go through the network together, one window per forward, as in the reference's loop.
    Chunk k+1 is assembled on a side stream while chunk k runs.  variable_skip draws from np.random as the
    reference's DataLoader(shuffle=False) does."""
    from .data.loader import DeviceDataset
    ds = dataset
    if not isinstance(ds, DeviceDataset):
        raise TypeError("evaluate_sequence needs a geomapnet_b200.data.DeviceDataset, got %s" % type(ds).__name__)
    if ds.jitter is not None:
        raise ValueError("evaluate_sequence: the dataset applies ColorJitter; build it with color_jitter=0")
    if ds.online:
        raise ValueError("evaluate_sequence: MFOnline datasets are not evaluation sequences")
    if not ds.h:
        raise RuntimeError("evaluate_sequence: the dataset is closed")
    pr, net, dev = _model_for(model, ds, "evaluate_sequence")
    vo = ds.vo_poses is not None
    T = 1 if ds.steps is None else ds.steps
    if vo and T < 2:
        raise ValueError("pose-graph optimisation needs windows of >= 2 frames (dataset.steps)")
    if vo_fc and not vo:
        raise ValueError("vo_fc: the dataset has no vo_poses")
    droprate = pr.droprate if pr is not None else float(net.droprate)
    cap = ds.max_batch * ds.frames_per_item                  # frames the dataset's cache assembles per call
    own = pr is None and net.precision in ("bf16", "tc_split")
    B = min(pr.max_batch if pr is not None else 64, cap)
    if droprate > 0:
        if B < T:
            raise ValueError("droprate > 0 runs one window of %d frames per forward; max_batch allows %d" % (T, B))
        B = T
    tab = ds.eval_tables(unique=droprate == 0, vo_fc=vo_fc)
    frames, L = tab["frames"], tab["windows"].shape[0]
    F = frames.shape[0]
    if own:
        pr = Predictor(model, max_batch=min(64, cap))
    was_training = net.training
    net.eval()
    try:
        with torch.cuda.device(dev):
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
            pred, targ = pred7, targ7
            if vo:
                pred = pgo(pred, vos7, fc_vos=vo_fc, **sigmas)
            if pose_m is not None:       # eval.py:180-181, as evaluate_tuples
                m = torch.as_tensor(np.asarray(pose_m, dtype=np.float64), device=dev)
                s = torch.as_tensor(np.asarray(pose_s, dtype=np.float64), device=dev)
                pred = torch.cat((pred[..., :3] * s + m, pred[..., 3:]), -1)
                targ = torch.cat((targ[..., :3] * s + m, targ[..., 3:]), -1)
            mid = T // 2
            p_mid, t_mid = pred[:, mid], targ[:, mid]
            t_err, q_err = pose_errors(p_mid, t_mid)
    finally:
        net.train(was_training)
        if own:
            torch.cuda.current_stream(dev).synchronize()     # the temporary engines are freed once their work is done
            pr.close()
    return dict(pred7=p_mid, targ7=t_mid, t_err=t_err, q_err=q_err, n_frames=F)


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
    own = pr is None and net.precision in ("bf16", "tc_split")
    tab = ds.val_tables(loader.batch_size, loader.shuffle, unique)
    n_batches = len(tab["batches"])
    if own:
        pr = Predictor(model, max_batch=min(64, cap) if unique else max(64, per_batch))
    was_training = net.training
    net.eval()
    try:
        with torch.cuda.device(dev):
            zero = torch.zeros(1, dtype=torch.float32, device=dev)
            s4 = torch.cat([getattr(criterion, k).detach().float().to(dev).reshape(1) if hasattr(criterion, k) else zero
                            for k in ("sax", "saq", "srx", "srq")])
            if unique:
                pred = _predict_frames(pr, net, ds, tab["frames"], min(pr.max_batch if pr is not None else 64, cap), 2,
                                       dev)
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
    finally:
        net.train(was_training)
        if own:
            torch.cuda.current_stream(dev).synchronize()     # the temporary engines are freed once their work is done
            pr.close()
    return sum(losses) / len(losses), losses
