"""Optimizer wrapper with the reference's surface + flat-buffer fused Adam, SGD and RMSprop.

Mirror of /root/reference/common/optimizer.py:8-47 (``Optimizer(params, method,
base_lr, weight_decay, **kwargs)``, ``.learner``, ``.adjust_lr``, ``.mult_lr``).
``method='adam'`` builds ``FusedAdam``: one CUDA launch per contiguous run of
parameters (the whole PoseNet is one run -- its parameters are views of one flat
buffer) instead of ~10 pointwise launches x 114 tensors (SURVEY.md section 8f-1).
``FusedAdam`` is a torch.optim.Optimizer: param_groups / state_dict() have
torch.optim.Adam's structure (step, exp_avg, exp_avg_sq per parameter) so
common/train.py:167-176,202 (checkpoint resume) keeps working.
``method='sgd'`` / ``'rmsprop'`` build ``FusedSGD`` / ``FusedRMSprop``: subclasses of
torch.optim.SGD / RMSprop (their constructor checks, defaults and state_dict() format)
whose step() runs one launch per run as well, takes the same grad_scale / max_grad_norm
arguments as FusedAdam's, and reads the learning rate from device memory, so the SGD
schedule (adjust_lr) reaches a replayed CUDA graph (geomapnet_b200/graph.py).
"""
import bisect
import ctypes

import torch
import torch.optim as optim

from .. import _lib

__all__ = ["Optimizer", "FusedAdam", "FusedSGD", "FusedRMSprop"]

_PAD = 64  # alignment padding (floats) between parameters in the flat buffer


def _dense(p):
    """Every element of p's memory span belongs to p exactly once (elementwise kernels may sweep the span)."""
    return p.is_contiguous() or (p.dim() == 4 and p.is_contiguous(memory_format=torch.channels_last))


def _fusable(p):
    """A parameter the flat-buffer kernels take: dense fp32 on the GPU, its gradient in the same strides."""
    return p.is_cuda and p.dtype == torch.float32 and _dense(p) and p.grad.stride() == p.stride()


class _FlatRuns(object):
    """Contiguous-run planning and the fused step's bookkeeping, shared by the fused learners (a mixin placed before
    the torch.optim class).  A learner names the per-parameter state buffers its configuration uses in `_slots`;
    every slot is one flat buffer per run, bound into `self.state` as views in each parameter's own element order."""

    _KEEPS_STEP = True      # state["step"] is part of the method's state_dict (Adam, RMSprop; not SGD)

    def _init_runs(self):
        self._runs = {}
        self._scratch = None

    def _slots(self, group):
        """[(state key, run field)] of the state buffers `group`'s configuration uses."""
        raise NotImplementedError

    def _host_step(self, st):
        """Steps already taken according to one parameter's state: where the device step counter starts."""
        return int(float(st["step"])) if "step" in st else 0

    def _set_host_step(self, r, n):
        r["step_host"] = n
        if self._KEEPS_STEP:
            t = torch.tensor(float(n))
            for p in r["params"]:
                self.state[p]["step"] = t

    def _plan(self, gi, params):
        """Contiguous runs of the group's parameters (one launch each) with their state buffers.

        The plan is keyed on the RUN STRUCTURE -- which parameters sit in which run, i.e. parameter addresses and the
        relative placement of their gradients -- not on absolute gradient addresses: a free-standing parameter (the
        criterion's sax / saq / srx / srq) gets a freshly allocated .grad from autograd every step, and the launch
        takes the gradient pointer of the day anyway.  Keyed on absolute gradient addresses the plan was rebuilt on
        every such step; harmless eagerly (state and step are carried over) but not while a CUDA graph is being
        captured: the rebuild's allocations, zero fills, state copies and the step-counter fill were captured with
        the step and replayed each time, resetting those parameters' optimizer state on every replay
        (tests/test_gpu_graph.py: criterion scalars 0.38 lr off after 4 replays)."""
        slots = tuple(self._slots(self.param_groups[gi]))
        order = sorted(params, key=lambda p: p.data_ptr())
        runs, cur = [], None
        for p in order:
            if cur is not None:
                last = cur["params"][-1]
                gap = (p.data_ptr() - (last.data_ptr() + last.numel() * 4)) // 4
                # a gap is swept by the kernels: only tolerated inside ONE storage on both sides (the flat
                # PoseNet buffers, whose padding the package zero-fills) -- never caching-allocator slack
                # between separately allocated tensors, which may hold stale NaN / Inf
                one_storage = (p.untyped_storage().data_ptr() == last.untyped_storage().data_ptr() and
                               p.grad.untyped_storage().data_ptr() == last.grad.untyped_storage().data_ptr())
                same = (p.device == last.device and (gap == 0 or (0 < gap < _PAD and one_storage)) and
                        (p.data_ptr() - last.data_ptr()) == (p.grad.data_ptr() - last.grad.data_ptr()))
                if same:
                    cur["params"].append(p)
                    continue
            cur = {"params": [p]}
            runs.append(cur)
        key = (slots, tuple(tuple(q.data_ptr() for q in r["params"]) for r in runs))
        cached = self._runs.get(gi)
        if cached is not None and cached[0] == key:
            # still valid only while the state's buffers ARE the run buffers (load_state_dict replaces them)
            def bound(r):
                if not slots:
                    return True
                t = self.state[r["params"][0]].get(slots[0][0])
                return t is not None and t.data_ptr() == r[slots[0][1]].data_ptr()
            if all(bound(r) for r in cached[1]):
                return cached[1]
        for r in runs:
            first, last = r["params"][0], r["params"][-1]
            r["n"] = (last.data_ptr() + last.numel() * 4 - first.data_ptr()) // 4
            step0 = self._host_step(self.state.get(first, {}))    # before the buffers are bound (SGD reads them)
            bufs = {field: torch.zeros(r["n"], dtype=torch.float32, device=first.device) for _, field in slots}
            # (SGD without momentum has no per-parameter state at all, as in torch)
            for p in (r["params"] if slots or self._KEEPS_STEP else ()):
                off = (p.data_ptr() - first.data_ptr()) // 4
                st = self.state[p]
                for k, field in slots:
                    # state in the parameter's own element order (channels_last for the KRSC conv weights)
                    view = torch.as_strided(bufs[field], tuple(p.shape), p.stride(), off)
                    if st.get(k) is not None:      # resumed / re-planned: keep the values
                        view.copy_(st[k].to(p.device))
                    st[k] = view
                if self._KEEPS_STEP and "step" not in st:
                    st["step"] = torch.tensor(0.0)
            r.update(bufs)
            # device-side step counter (keeps captured CUDA graphs correct on replay)
            r["step_host"] = step0
            r["step_dev"] = torch.full((1,), step0, dtype=torch.int32, device=first.device)
        self._runs[gi] = (key, runs)
        return runs

    def _fused_groups(self, clip_groups):
        """[(group index, group, parameters with gradients, clipped)]; None when some parameter is not one the kernels
        take (see _fusable)."""
        out = []
        for gi, group in enumerate(self.param_groups):
            params = [p for p in group["params"] if p.grad is not None]
            if not params:
                continue
            if not all(_fusable(p) for p in params):
                return None
            out.append((gi, group, params, clip_groups is None or gi in clip_groups))
        return out

    def _fused_step(self, groups, grad_scale, max_grad_norm, launch):
        """One launch per run: launch(L, group, gi, run, sqnorm pointer or None, stream).  With max_grad_norm > 0 the
        squared norm of the clipped groups' gradients is summed first (mapnet_sqnorm, one launch per run)."""
        L = _lib.lib()
        groups = [(gi, group, self._plan(gi, params), clipped) for gi, group, params, clipped in groups]
        dev = groups[0][2][0]["params"][0].device
        sq_ptr = None
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            if max_grad_norm and max_grad_norm > 0.0:
                if self._scratch is None or self._scratch.device != dev:
                    self._scratch = torch.zeros(2048, dtype=torch.float32, device=dev)
                total = self._scratch[1024:1025]
                total.zero_()
                part = self._scratch[1025:1026]
                for gi, group, runs, clipped in groups:
                    if not clipped:
                        continue
                    for r in runs:
                        g0 = r["params"][0].grad
                        _lib.check(L.mapnet_sqnorm(g0.data_ptr(), r["n"], self._scratch.data_ptr(),
                                                   part.data_ptr(), st), "mapnet_sqnorm")
                        total += part
                sq_ptr = total.data_ptr()
            for gi, group, runs, clipped in groups:
                for r in runs:
                    self._set_host_step(r, r["step_host"] + 1)
                    launch(L, group, gi, r, ctypes.c_void_p(sq_ptr) if (sq_ptr and clipped) else None, st)

    def advance_host_step(self, n=1):
        """After replaying a captured graph that contains step(): the device counters advanced,
        bring the host mirrors (state['step'], used by state_dict()) in line."""
        for key, runs in self._runs.values():
            for r in runs:
                self._set_host_step(r, r["step_host"] + n)


class FusedAdam(_FlatRuns, optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        if lr < 0 or eps < 0 or not (0 <= betas[0] < 1) or not (0 <= betas[1] < 1) or weight_decay < 0:
            raise ValueError("invalid Adam hyper-parameter")
        super(FusedAdam, self).__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._init_runs()

    def _slots(self, group):
        return (("exp_avg", "m"), ("exp_avg_sq", "v"))

    @torch.no_grad()
    def step(self, closure=None, grad_scale=1.0, max_grad_norm=0.0, clip_groups=(0,)):
        """grad_scale multiplies every gradient first (1/world_size after a sum-allreduce);
        max_grad_norm > 0 applies clip_grad_norm_ (fused) to the param groups listed in `clip_groups` --
        the norm is taken over those groups only and only they are scaled.  Default: group 0, the model
        (common/train.py:357-358 clips model.parameters(); the criterion's sax/saq/srx/srq groups of
        scripts/train.py:104-110 are neither counted nor scaled).  clip_groups=None: every group."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        groups = self._fused_groups(clip_groups)
        if groups is None:
            raise RuntimeError("FusedAdam needs dense fp32 CUDA parameters with gradients in the same strides "
                               "(contiguous, or channels_last views of a flat buffer; no CPU path)")
        if not groups:
            return loss

        def launch(L, group, gi, r, sq, st):
            b1, b2 = group["betas"]
            p0 = r["params"][0]
            _lib.check(L.mapnet_adam_step_dev(
                p0.data_ptr(), p0.grad.data_ptr(), r["m"].data_ptr(), r["v"].data_ptr(), r["n"],
                float(group["lr"]), float(b1), float(b2), float(group["eps"]),
                float(group["weight_decay"]), r["step_dev"].data_ptr(), float(grad_scale),
                sq, float(max_grad_norm or 0.0), st), "mapnet_adam_step_dev")
        self._fused_step(groups, grad_scale, max_grad_norm, launch)
        return loss


class _DeviceLrFlatRuns(_FlatRuns):
    """Fused learners whose kernels read the learning rate from device memory (one float per param group), so that
    a schedule written into param_groups on the host reaches a replayed CUDA graph.

    Everything the kernels do not take keeps torch's own step: parameters that are not dense fp32 CUDA tensors,
    maximize=True, differentiable=True and a tensor-valued lr.  There grad_scale and the clip are applied to the
    gradients in place with torch ops, then the parent class steps."""

    _NAME = None

    def _init_runs(self):
        super(_DeviceLrFlatRuns, self)._init_runs()
        self._lr_dev, self._lr_synced = {}, {}

    def sync_lr(self):
        """Write each group's host rate into its device float when it changed since the last sync.  step() calls
        this first; call it before replaying a graph that contains step() (GraphedTrainStep does).  Never captured:
        a rate that changed while a graph is being captured is an error."""
        for gi, t in self._lr_dev.items():
            lr = self.param_groups[gi]["lr"]
            if torch.is_tensor(lr) or lr == self._lr_synced[gi]:
                continue
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("%s: the learning rate changed while a CUDA graph is being captured" % self._NAME)
            t.fill_(float(lr))
            self._lr_synced[gi] = lr

    def _lr_ptr(self, gi, group, dev):
        t = self._lr_dev.get(gi)
        if t is None or t.device != dev:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("%s: take one eager step before capturing step() in a CUDA graph (the device "
                                   "learning rate is allocated and written there)" % self._NAME)
            t = torch.full((1,), float(group["lr"]), dtype=torch.float32, device=dev)
            self._lr_dev[gi], self._lr_synced[gi] = t, group["lr"]
        return t.data_ptr()

    def _kernel_takes(self, group):
        return not (group.get("maximize") or group.get("differentiable") or torch.is_tensor(group["lr"]))

    def _torch_step(self, grad_scale, max_grad_norm, clip_groups):
        if grad_scale != 1.0:
            for group in self.param_groups:
                for p in group["params"]:
                    if p.grad is not None:
                        p.grad.mul_(grad_scale)
        if max_grad_norm and max_grad_norm > 0.0:
            clipped = [p for gi, group in enumerate(self.param_groups) if clip_groups is None or gi in clip_groups
                       for p in group["params"] if p.grad is not None]
            torch.nn.utils.clip_grad_norm_(clipped, max_grad_norm)
        super(_DeviceLrFlatRuns, self).step()

    def _step(self, closure, grad_scale, max_grad_norm, clip_groups, launch):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        groups = self._fused_groups(clip_groups)
        if groups is None or not all(self._kernel_takes(group) for _, group, _, _ in groups):
            self._torch_step(grad_scale, max_grad_norm, clip_groups)
            return loss
        if not groups:
            return loss
        self.sync_lr()
        self._fused_step(groups, grad_scale, max_grad_norm, launch)
        return loss


class FusedSGD(_DeviceLrFlatRuns, optim.SGD):
    """torch.optim.SGD whose step() runs k_sgd (geomapnet_b200/csrc/optim.cu) once per contiguous run of parameters.
    step(closure=None, grad_scale=1.0, max_grad_norm=0.0, clip_groups=(0,)) as FusedAdam.step."""

    _KEEPS_STEP = False
    _NAME = "FusedSGD"

    def __init__(self, params, *args, **kwargs):
        super(FusedSGD, self).__init__(params, *args, **kwargs)
        self._init_runs()

    def _slots(self, group):
        return (("momentum_buffer", "buf"),) if group["momentum"] != 0 else ()

    def _host_step(self, st):
        # SGD keeps no step count; only the first step differs (it initialises the momentum buffer), and a
        # momentum buffer in the state -- stepped or loaded -- means it has been taken
        return 1 if st.get("momentum_buffer") is not None else 0

    @torch.no_grad()
    def step(self, closure=None, grad_scale=1.0, max_grad_norm=0.0, clip_groups=(0,)):
        def launch(L, group, gi, r, sq, st):
            p0 = r["params"][0]
            _lib.check(L.mapnet_sgd_step_dev(
                p0.data_ptr(), p0.grad.data_ptr(), r["buf"].data_ptr() if "buf" in r else None, r["n"],
                self._lr_ptr(gi, group, p0.device), float(group["momentum"]), float(group["dampening"]),
                float(group["weight_decay"]), int(bool(group["nesterov"])), r["step_dev"].data_ptr(),
                float(grad_scale), sq, float(max_grad_norm or 0.0), st), "mapnet_sgd_step_dev")
        return self._step(closure, grad_scale, max_grad_norm, clip_groups, launch)


class FusedRMSprop(_DeviceLrFlatRuns, optim.RMSprop):
    """torch.optim.RMSprop whose step() runs k_rmsprop (geomapnet_b200/csrc/optim.cu) once per contiguous run of
    parameters.  step(closure=None, grad_scale=1.0, max_grad_norm=0.0, clip_groups=(0,)) as FusedAdam.step."""

    _NAME = "FusedRMSprop"

    def __init__(self, params, *args, **kwargs):
        super(FusedRMSprop, self).__init__(params, *args, **kwargs)
        self._init_runs()

    def _slots(self, group):
        slots = [("square_avg", "sq")]
        if group["momentum"] > 0:
            slots.append(("momentum_buffer", "buf"))
        if group["centered"]:
            slots.append(("grad_avg", "ga"))
        return slots

    @torch.no_grad()
    def step(self, closure=None, grad_scale=1.0, max_grad_norm=0.0, clip_groups=(0,)):
        def launch(L, group, gi, r, sq, st):
            p0 = r["params"][0]
            _lib.check(L.mapnet_rmsprop_step_dev(
                p0.data_ptr(), p0.grad.data_ptr(), r["sq"].data_ptr(), r["ga"].data_ptr() if "ga" in r else None,
                r["buf"].data_ptr() if "buf" in r else None, r["n"], self._lr_ptr(gi, group, p0.device),
                float(group["alpha"]), float(group["eps"]), float(group["weight_decay"]), float(group["momentum"]),
                r["step_dev"].data_ptr(), float(grad_scale), sq, float(max_grad_norm or 0.0), st),
                "mapnet_rmsprop_step_dev")
        return self._step(closure, grad_scale, max_grad_norm, clip_groups, launch)


class Optimizer:
    """Learner + learning-rate schedule behind the reference's wrapper surface
    (``Optimizer(params, method, base_lr, weight_decay, **kwargs)``, ``.learner``, ``.adjust_lr(epoch)``,
    ``.mult_lr(f)`` -- what /root/reference/common/train.py:128,281,359 and scripts/train.py:112 use).
    'adam', 'sgd' and 'rmsprop' are the fused flat-buffer learners above.  Only SGD has a schedule: the rate drops
    by ``lr_decay`` at every epoch listed in ``lr_stepvalues``."""

    _LEARNERS = {"sgd": FusedSGD, "adam": FusedAdam, "rmsprop": FusedRMSprop}

    def __init__(self, params, method, base_lr, weight_decay, **kwargs):
        if method not in self._LEARNERS:
            raise NotImplementedError(method)
        self.method, self.base_lr = method, base_lr
        if method == "sgd":
            self.lr_decay = kwargs.pop("lr_decay")
            self.lr_stepvalues = sorted(kwargs.pop("lr_stepvalues"))
        self.learner = self._LEARNERS[method](params, lr=base_lr, weight_decay=weight_decay, **kwargs)

    def _each_group(self, fn):
        for group in self.learner.param_groups:
            group["lr"] = fn(group["lr"])

    def adjust_lr(self, epoch):
        """Rate for `epoch`; written into every param group when there is a schedule (SGD)."""
        if self.method != "sgd":
            return self.base_lr
        drops = bisect.bisect_right(self.lr_stepvalues, epoch)      # step values already reached
        lr = self.base_lr * self.lr_decay ** drops
        self._each_group(lambda _: lr)
        return lr

    def mult_lr(self, f):
        self._each_group(lambda lr: lr * f)
