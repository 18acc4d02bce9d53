"""CUDA-graph capture of the training step (common/train.py:339-361).

The step is ~200 short kernel launches; replaying it as two CUDA graphs removes the
host launch cost and most of the inter-kernel gaps.  Graph 1 =
forward + criterion + zero_grad + backward, graph 2 = [clip +] the optimizer step (Adam, SGD or RMSprop).  Data parallel: the
whole-buffer allreduce of FlatDataParallel sits between the two graphs (default).  With
FlatDataParallel(overlap=True) the three slice allreduces issued from the backward-part hook
are captured INSIDE graph 1, on a side stream that forks from and joins the capturing stream,
and only the 16-byte reduce of the criterion scalars stays eager between the graphs (measured
gain at 2 GPUs: 0.3 %, see geomapnet_b200/ddp.py).

    step = GraphedTrainStep(model, criterion, optimizer, x_example, targ_example)
    loss = step(x, targ)            # x, targ: CUDA tensors (copied into static buffers)
    step.out                        # the step's prediction (a static buffer, overwritten by the next replay)

Build it before (or without) keeping tensors of an earlier eager step alive: a live `loss` from a step that ran on the
default stream pins the parameters' AccumulateGrad nodes to that stream and the capture then fails with
cudaErrorStreamCaptureImplicit (torch: "delete all references to the autograd graph").

Everything captured is the same product code that runs eagerly (the reference-facing
modules and the C ABI underneath); counters that change per step (Adam bias
correction, SGD's first step, dropout offset) live in device memory so replays stay correct,
and so does the SGD / RMSprop learning rate: a schedule (Optimizer.adjust_lr / mult_lr) changes
param_groups on the host, and each call writes a changed rate to the device before graph 2 replays.
"""
import torch

__all__ = ["GraphedTrainStep", "train_val"]


class GraphedTrainStep(object):
    def __init__(self, model, criterion, optimizer, x_example, targ_example, dp=None, max_grad_norm=0.0,
                 warmup=3):
        self.model, self.criterion, self.dp = model, criterion, dp
        self.learner = optimizer.learner if hasattr(optimizer, "learner") else optimizer
        self.max_grad_norm = float(max_grad_norm or 0.0)
        self.posenet = model.mapnet if hasattr(model, "mapnet") else model
        self.posenet._graph_rng = True
        dev = x_example.device
        self.x = torch.empty_like(x_example)
        self.t = torch.empty_like(targ_example)
        self.x.copy_(x_example); self.t.copy_(targ_example)
        self.scale = 1.0 / dp.world if dp is not None else 1.0
        snap = self._snapshot()
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):       # builds arenas, tensor maps, optimizer plans
                self._fwd_bwd()
                if dp is not None:
                    dp.allreduce_grads()
                self._opt()
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        from . import _lib
        lc = _lib.lib().mapnet_launch_count()
        # graph 1 holds the backward schedule of the parameters that train now (frozen ones get no gradient)
        self.trainable = self.posenet.trainable_mask()
        self.g1 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g1):
            self.loss = self._fwd_bwd()
        self.g2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g2):
            self._opt()
        self.kernels_per_step = int(_lib.lib().mapnet_launch_count() - lc)   # library kernels in the two graphs
        # the capture passes ran the host-side counters once each without executing kernels
        self._fix_host_counters()
        # construction must not train: put parameters, BN buffers, criterion scalars and the
        # optimizer moments / step counters back to what they were before the warm-up steps
        self._restore(snap)

    def _snapshot(self):
        snap = {"model": {k: v.detach().clone() for k, v in self.model.state_dict().items()},
                "crit": {k: v.detach().clone() for k, v in self.criterion.state_dict().items()},
                "opt": {}}
        for p, st in self.learner.state.items():
            snap["opt"][p] = {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in st.items()}
        return snap

    def _restore(self, snap):
        with torch.no_grad():
            sd = self.model.state_dict()
            for k, v in snap["model"].items():
                sd[k].copy_(v)
            cd = self.criterion.state_dict()
            for k, v in snap["crit"].items():
                cd[k].copy_(v)
            # every tensor of the optimizer state (Adam moments, SGD / RMSprop momentum buffers, square_avg,
            # grad_avg, step): the snapshot's value, or zero for a slot the warm-up created
            for p, st in self.learner.state.items():
                old = snap["opt"].get(p) or {}
                for k, v in st.items():
                    if torch.is_tensor(v):
                        if torch.is_tensor(old.get(k)):
                            v.copy_(old[k])
                        else:
                            v.zero_()
            if hasattr(self.learner, "_runs"):
                # the fused learners' device step counters and their host mirrors
                for key, runs in self.learner._runs.values():
                    for r in runs:
                        step0 = self.learner._host_step(snap["opt"].get(r["params"][0]) or {})
                        self.learner._set_host_step(r, step0)
                        r["step_dev"].fill_(step0)
        torch.cuda.synchronize()

    def _fwd_bwd(self):
        out = self.model(self.x)
        self.out = out.detach()
        loss = self.criterion(out, self.t)
        self.learner.zero_grad()
        loss.backward()
        if self.dp is not None and getattr(self.dp, "overlap", False):
            self.dp.join_slices()         # the side stream's NCCL work joins the (capturing) stream here
        return loss.detach()

    def _opt(self):
        self.learner.step(grad_scale=self.scale, max_grad_norm=self.max_grad_norm)

    def _fix_host_counters(self):
        # capture executed Python bookkeeping (host step mirrors) but launched nothing
        if hasattr(self.learner, "advance_host_step"):
            self.learner.advance_host_step(-1)

    def check_trainable(self):
        if self.posenet.trainable_mask() != self.trainable:
            raise RuntimeError("GraphedTrainStep: requires_grad of the model's parameters changed since the step was "
                               "captured; the graph would replay the old backward schedule.  Build a new "
                               "GraphedTrainStep for the new set of trainable parameters.")

    def __call__(self, x, targ):
        self.x.copy_(x, non_blocking=True)
        self.t.copy_(targ, non_blocking=True)
        return self.replay()

    def replay(self, inputs_read=None):
        """One step on what self.x / self.t hold.  inputs_read: a torch.cuda.Event recorded once the step no longer
        reads them (after graph 1), so the next batch can be written there while the optimizer runs."""
        self.check_trainable()
        self.g1.replay()
        if inputs_read is not None:
            inputs_read.record()
        if self.dp is not None:
            self.dp.allreduce_grads(slices_in_graph=getattr(self.dp, "overlap", False))
        if hasattr(self.learner, "sync_lr"):
            self.learner.sync_lr()        # the captured SGD / RMSprop launches read the rate from device memory
        self.g2.replay()
        if hasattr(self.learner, "advance_host_step"):
            self.learner.advance_host_step(1)
        return self.loss


def train_epoch(loader, model, criterion, optimizer, max_grad_norm=0.0, steps=None):
    """One epoch of a geomapnet_b200.data.DeviceLoader through CUDA graphs, last partial batch included
    (common/train.py:276-300 with step_feedfwd).  One GraphedTrainStep per distinct batch size, built before the
    first step and full size first, so that the trunk's arena never grows under a captured graph.  Each batch is
    assembled on a side stream straight into the static input of the step that takes it, while the previous step's
    optimizer graph runs.  steps: a dict {batch size: GraphedTrainStep} kept by the caller to reuse the captures in
    later epochs (filled on first use).  Returns the per-step losses as floats (one device sync, at the end)."""
    from .data.loader import SidePipeline
    ds = loader.dataset
    dev = ds.device
    steps = {} if steps is None else steps
    sizes = [loader.batch_size]
    last = len(ds) % loader.batch_size
    if last:
        sizes.append(last)
    for n in sizes:
        if n not in steps:
            xs, ts = ds.batch_shapes(n)
            x0, t0 = torch.empty(xs, device=dev), torch.empty(ts, device=dev)
            ds.assemble(ds.example(n), x0, t0)
            steps[n] = GraphedTrainStep(model, criterion, optimizer, x0, t0, max_grad_norm=max_grad_norm)
    for st in steps.values():      # captures kept from an earlier epoch: before any batch is assembled
        st.check_trainable()
    pipe = SidePipeline(dev)          # one buffer per batch size: the static inputs of its step
    losses = []

    def fill(batch):
        st = steps[batch[3]]
        pipe.fill(batch[3], lambda: ds.assemble(batch, st.x, st.t))
        return batch[3]

    it = loader.batches()
    b = next(it, None)
    n = fill(b) if b is not None else None
    while n is not None:
        pipe.take(n)
        steps[n].replay(inputs_read=pipe.read(n))
        losses.append(steps[n].loss.clone())
        b = next(it, None)
        n = fill(b) if b is not None else None
    return [float(v) for v in torch.stack(losses).cpu()] if losses else []


def train_val(model, train_loader, val_loader, train_criterion, val_criterion, optimizer, n_epochs, val_freq, snapshot,
              logdir, max_grad_norm=0.0, start_epoch=0):
    """Trainer.train_val (common/train.py:212-317) over DeviceLoaders, in the reference's order.  For each epoch from
    start_epoch: validate (inference.validate) when epoch % val_freq == 0 or it is the last epoch, unless val_loader is
    None (do_val = no); save a checkpoint (common.checkpoint.save_checkpoint, with train_criterion) when
    epoch % snapshot == 0; optimizer.adjust_lr(epoch); one train_epoch.  Then a final checkpoint at n_epochs.

    One Predictor of the model (bf16 / tc_split) serves every validation pass, refreshed before each; any other model
    runs its own eval forward.  The train_epoch captures are kept across epochs.  Returns {"val": {epoch: avg loss},
    "train": {epoch: [per-step losses]}} and prints nothing."""
    from .common.checkpoint import save_checkpoint
    from .inference import Predictor, validate
    net = model.mapnet if hasattr(model, "mapnet") else model
    pr = Predictor(model) if val_loader is not None and net.precision in ("bf16", "tc_split") else None
    steps, out = {}, {"val": {}, "train": {}}
    try:
        for epoch in range(int(start_epoch), int(n_epochs)):
            if val_loader is not None and (epoch % val_freq == 0 or epoch == n_epochs - 1):
                if pr is not None:
                    pr.refresh()
                out["val"][epoch] = validate(pr if pr is not None else model, val_loader, val_criterion)[0]
            if epoch % snapshot == 0:
                save_checkpoint(logdir, epoch, model, optimizer, train_criterion)
            optimizer.adjust_lr(epoch)
            model.train()
            out["train"][epoch] = train_epoch(train_loader, model, train_criterion, optimizer,
                                              max_grad_norm=max_grad_norm, steps=steps)
        save_checkpoint(logdir, int(n_epochs), model, optimizer, train_criterion)
    finally:
        if pr is not None:
            pr.close()
    return out
