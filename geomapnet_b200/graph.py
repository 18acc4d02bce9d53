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

__all__ = ["GraphedTrainStep"]


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

    def __call__(self, x, targ):
        self.x.copy_(x, non_blocking=True)
        self.t.copy_(targ, non_blocking=True)
        self.g1.replay()
        if self.dp is not None:
            self.dp.allreduce_grads(slices_in_graph=getattr(self.dp, "overlap", False))
        if hasattr(self.learner, "sync_lr"):
            self.learner.sync_lr()        # the captured SGD / RMSprop launches read the rate from device memory
        self.g2.replay()
        if hasattr(self.learner, "advance_host_step"):
            self.learner.advance_host_step(1)
        return self.loss
