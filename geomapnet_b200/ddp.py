"""Plain data parallel over the GPUs of one box: one process per GPU, the flat
gradient buffer sum-reduced over NCCL (NVLink 5 / NVSwitch) -- as ONE allreduce
after the backward pass (default), or as three slices issued from inside it.

The reference is single-GPU (common/train.py:193-196); this is the multi-GPU
row of SURVEY.md section 8e.  Tuples (the N dimension of [N,T,3,H,W]) are sharded
across ranks, never the T frames of a tuple: the relative-pose loss only
couples frames inside a tuple (common/criterion.py:94-105).  BatchNorm
statistics stay per-rank (no SyncBN), as when running the reference at the
local batch size.  Equal local batches => mean of local L1 means == global L1
mean, so averaged gradients equal the single-process gradient.

Overlap (overlap=True, MAPNET_DDP_OVERLAP=1): the backward pass finishes the
gradients back to front.  The library runs it in three parts
(mapnet_backward_part: head + layer4 = 64 % of the 89.4 MB after ~20 % of the
backward FLOPs, then layer3, then the rest) and calls back after each one; the
callback enqueues that slice's allreduce on a side stream, so that only the
last 5 MB slice would be exposed.  Whether that hides the NVLink time depends on
the SMs NCCL gets (not measured on H100).  The backward's kernels leave NCCL's CTAs little room: the
conv engines hold every SM with a persistent CTA of ~200 KB shared memory, the
element-wise kernels fill every SM's 2048 thread slots, and programmatic
dependent launch keeps the next kernel's CTAs queued ahead.  Hiding the
collective needs SMs reserved for it (or copy-engine collectives); until then the
default is the single allreduce, which is also the simplest thing to capture
around (no NCCL work inside the CUDA graph).

All functions work on any device/backend (gloo on CPU in the tests).
"""
import torch
import torch.distributed as dist

__all__ = ["shard_tuples", "allreduce_flat_", "FlatDataParallel"]


def shard_tuples(x, rank, world):
    """Rank r takes tuples [r*n, (r+1)*n) of the leading dimension (must divide evenly)."""
    N = x.shape[0]
    if N % world != 0:
        raise ValueError("global batch %d is not divisible by world size %d" % (N, world))
    n = N // world
    return x[rank * n:(rank + 1) * n]


def allreduce_flat_(flat_grad, extra_grads=(), group=None, average=False):
    """Sum-allreduce of ``flat_grad`` plus the (tiny) ``extra_grads`` tensors (criterion scalars
    sax/saq/srx/srq), in place; returns the world size.  The extras travel as ONE packed tensor in a second,
    16-byte collective (they are produced by a different autograd node than the flat buffer, so they cannot be
    assumed to sit in it).  With average=False the caller folds 1/world into the optimizer step
    (FusedAdam grad_scale)."""
    world = dist.get_world_size(group)
    dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    extras = [g for g in extra_grads if g is not None]
    if extras:
        packed = torch.cat([g.reshape(-1).to(flat_grad.dtype) for g in extras])
        dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=group)
        off = 0
        for g in extras:
            g.copy_(packed[off:off + g.numel()].view_as(g))
            off += g.numel()
    if average:
        flat_grad.mul_(1.0 / world)
        for g in extras:
            g.mul_(1.0 / world)
    return world


class FlatDataParallel(object):
    """Wraps a geomapnet_b200 PoseNet/MapNet (+ criterion) for data-parallel steps.

        dp = FlatDataParallel(model, criterion)       # then dp.broadcast_parameters() once
        loss = criterion(model(x_local), targ_local); loss.backward()   # slices are reduced WHILE this runs
        scale = dp.allreduce_grads()                  # joins the side stream (+ the scalars); returns 1/world
        optimizer.learner.step(grad_scale=scale)

    The step(grad_scale=...) call works with all three of the package's learners (Optimizer 'adam', 'sgd' and
    'rmsprop': FusedAdam, FusedSGD, FusedRMSprop), which fold the 1/world scale into their fused update.

    overlap=False (default): one allreduce of the whole buffer inside allreduce_grads(); overlap=True: three slices
    reduced from the backward-part hook on a side stream (see the module docstring for what was measured).
    """

    def __init__(self, model, criterion=None, group=None, broadcast=True, overlap=False):
        self.model = model
        self.posenet = model.mapnet if hasattr(model, "mapnet") else model
        self.criterion = criterion
        self.group = group
        self.world = dist.get_world_size(group)
        self._broadcast_pending = broadcast
        self.overlap = bool(overlap)
        self._side = None
        self._parts_done = 0
        self._slice_group = group
        if self.overlap:
            self.posenet._grad_part_hook = self._on_part
            # The slice allreduces run WHILE the backward's conv kernels fill every SM (persistent CTAs, ~200 KB of
            # shared memory each): on a normal-priority stream NCCL's CTAs only get placed when a conv kernel drains
            # (measured at N=2: 5.678 vs 5.674 ms/step with and without the hook).  A separate NCCL communicator on
            # HIGH-PRIORITY streams is the documented way to get them placed first; measured: 5.340 vs 5.355 ms.
            if dist.get_backend(group) == "nccl" and self.world > 1:
                try:
                    opts = dist.ProcessGroupNCCL.Options(is_high_priority_stream=True)
                    ranks = dist.get_process_group_ranks(group) if group is not None else None
                    self._slice_group = dist.new_group(ranks=ranks, backend="nccl", pg_options=opts)
                except Exception:                       # older torch: keep the default communicator
                    self._slice_group = group

    def close(self):
        if getattr(self.posenet, "_grad_part_hook", None) == self._on_part:
            self.posenet._grad_part_hook = None

    def broadcast_parameters(self):
        flat, _ = self.posenet.flat_parameters()
        dist.broadcast(flat, src=0, group=self.group)
        dist.broadcast(self.posenet._bufs, src=0, group=self.group)
        if self.criterion is not None:
            for p in self.criterion.parameters():
                dist.broadcast(p.data, src=0, group=self.group)
        self._broadcast_pending = False

    # -- overlap machinery -----------------------------------------------------------------------------------
    def _side_stream(self, device):
        if device.type != "cuda":
            return None
        if self._side is None or self._side.device != device:
            self._side = torch.cuda.Stream(device, priority=-1)
        return self._side

    def _on_part(self, part, grad_slice):
        """Called by PoseNet._run_backward right after backward part `part` was enqueued: its slice of the flat
        gradient buffer is final once the compute stream reaches this point."""
        if self._broadcast_pending:
            raise RuntimeError("call broadcast_parameters() once after the model is on its device")
        side = self._side_stream(grad_slice.device)
        if side is None:                         # CPU tensors (gloo tests): no streams, reduce in place now
            dist.all_reduce(grad_slice, op=dist.ReduceOp.SUM, group=self._slice_group)
        else:
            side.wait_stream(torch.cuda.current_stream(grad_slice.device))
            with torch.cuda.stream(side):
                dist.all_reduce(grad_slice, op=dist.ReduceOp.SUM, group=self._slice_group)
        self._parts_done = part + 1

    def _criterion_grads(self):
        if self.criterion is None:
            return []
        return [p.grad for p in self.criterion.parameters() if p.requires_grad and p.grad is not None]

    def join_slices(self):
        """Make the compute stream wait for the slice allreduces issued from the backward-part hook."""
        if self._side is not None:
            torch.cuda.current_stream(self._side.device).wait_stream(self._side)

    def allreduce_grads(self, slices_in_graph=False):
        """slices_in_graph: the three slice allreduces were captured into the CUDA graph that just replayed (and joined
        there): only the criterion scalars remain."""
        if slices_in_graph:
            self._parts_done = 3
        if self._broadcast_pending:
            raise RuntimeError("call broadcast_parameters() once after the model is on its device")
        _, gflat = self.posenet.flat_parameters()
        if gflat is None:
            raise RuntimeError("no gradient buffer: run backward() first")
        # the buffer this reduces must be the one the optimizer reads through p.grad (gradient accumulation or
        # zero_grad(set_to_none=False) make autograd accumulate into a DIFFERENT tensor than the last backward wrote)
        g0 = self.posenet._param_list[0].grad
        if g0 is None or not (gflat.data_ptr() <= g0.data_ptr() < gflat.data_ptr() + gflat.numel() * gflat.element_size()):
            raise RuntimeError("FlatDataParallel: parameter .grad does not alias the flat gradient buffer of the last "
                               "backward (gradient accumulation is not supported: call zero_grad() -- set_to_none=True -- "
                               "before every backward)")
        extras = self._criterion_grads()
        if self.overlap and self._parts_done == 3:
            self._parts_done = 0
            side = self._side_stream(gflat.device)
            if extras:
                packed = torch.cat([g.reshape(-1).float() for g in extras])
                if side is not None:
                    side.wait_stream(torch.cuda.current_stream(gflat.device))
                    with torch.cuda.stream(side):
                        dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=self.group)
                else:
                    dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=self.group)
            if side is not None:
                torch.cuda.current_stream(gflat.device).wait_stream(side)
            if extras:
                off = 0
                for g in extras:
                    g.copy_(packed[off:off + g.numel()].view_as(g))
                    off += g.numel()
        else:
            self._parts_done = 0
            allreduce_flat_(gflat, extras, group=self.group, average=False)
        return 1.0 / self.world
