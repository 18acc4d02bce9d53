"""H100-native PoseNet / MapNet behind the reference's nn.Module surface.

Host-side mirror of /root/reference/models/posenet.py (PoseNet :36-73, MapNet
:75-97, filter_hook :28-34): same constructor signatures, same parameter /
state_dict key names and order (``feature_extractor.conv1.weight`` first; 222
entries), same initialisation RNG consumption -- but ``forward`` runs the
hand-written sm_90a kernels through the C ABI (include/mapnet_b200.h) instead
of a torchvision/cuDNN autograd graph, and the backward is one explicit call
(no autograd inside the trunk).  PyTorch owns all parameter / gradient storage
so torch.optim, clip_grad_norm_, state_dict, torch.save keep working
(SURVEY.md section 8b).  No CPU path: tensors must be CUDA.
"""
import os

import torch
import torch.nn as nn

from .. import _lib

__all__ = ["PoseNet", "MapNet", "filter_hook"]

_DEFAULT_PRECISION = os.environ.get("GEOMAPNET_B200_PRECISION", "bf16")


def filter_hook(m, g_in, g_out):
    """Kept for API parity with models/posenet.py:28-34 (NaN -> 0 on grad_input).
    The fused backward applies this filter itself when filter_nans=True."""
    g_filtered = []
    for g in g_in:
        g = g.clone()
        g[g != g] = 0
        g_filtered.append(g)
    return tuple(g_filtered)


class _Node(nn.Module):
    """Parameter container mirroring the reference's module tree (names only)."""

    def forward(self, *a, **k):
        raise RuntimeError("geomapnet_b200: the trunk runs as one fused CUDA step; "
                           "sub-modules are parameter containers and cannot be called")


class _TrunkFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, net, x, *params):
        pred = net._run_forward(x)
        ctx.net = net
        ctx.fwd_id = net._fwd_id
        return pred

    @staticmethod
    def backward(ctx, dpred):
        net = ctx.net
        if ctx.fwd_id != net._fwd_id:
            raise RuntimeError("geomapnet_b200: backward() must follow the forward() it belongs to "
                               "(activations of one step are kept in a static arena)")
        # needs_input_grad: each parameter's requires_grad at forward time.  Frozen parameters get no gradient, and the
        # trunk skips their weight gradients and every input gradient below the lowest layer that trains.
        grads = net._run_backward(dpred, ctx.needs_input_grad[2:])
        return (None, None) + tuple(grads)


class PoseNet(nn.Module):
    def __init__(self, feature_extractor, droprate=0.5, pretrained=True, feat_dim=2048, filter_nans=False,
                 precision=None, seed=None):
        """feature_extractor: a torchvision-style ResNet-34 object.  It is NEVER run:
        only ``.fc.in_features`` is read and its state_dict harvested as initial trunk
        weights (scripts/train.py:76-78).  precision: 'bf16' (wgmma tensor cores, bf16 operands,
        default), 'tc_split' (the same engines on fp16 hi/lo operand planes: 1e-4 parity on tensor cores),
        'fp32' (strict-parity CUDA-core path) or 'bf16_simt' (cross-check)."""
        super(PoseNet, self).__init__()
        self.droprate = droprate
        self.feat_dim = feat_dim
        self.filter_nans = bool(filter_nans)
        self.precision = precision or _DEFAULT_PRECISION
        if self.precision not in _lib.PREC:
            raise ValueError("precision must be one of %s" % sorted(_lib.PREC))
        fe_out_planes = feature_extractor.fc.in_features
        if fe_out_planes != 512:
            raise NotImplementedError("geomapnet_b200 implements the ResNet-34 trunk (fc.in_features=512), got %d"
                                      % fe_out_planes)

        spec = _lib.Trunk(0, 64, 64, feat_dim, self.precision)      # spec-only handle, no device needed
        self._table, self._n_params, self._n_bufs = spec.table()
        self._krsc = spec.layouts()       # conv weights stored [Co][KH][KW][Ci] in the flat buffers (channels_last views)
        spec.close()
        self._n_nbt = sum(1 for e in self._table if e[1] == 2)
        self._flat = torch.zeros(self._n_params, dtype=torch.float32)
        self._bufs = torch.zeros(self._n_bufs, dtype=torch.float32)
        self._nbt = torch.zeros(self._n_nbt, dtype=torch.int64)
        self._build_tree()

        # ---- weights: harvest the extractor, then initialise as models/posenet.py:45-63 does
        src = feature_extractor.state_dict()
        with torch.no_grad():
            for name, kind, shape, off in self._table:
                if not name.startswith("feature_extractor.") or name.startswith("feature_extractor.fc."):
                    continue
                key = name[len("feature_extractor."):]
                if key not in src or tuple(src[key].shape) != tuple(shape):
                    raise NotImplementedError(
                        "feature_extractor is not a ResNet-34 (BasicBlock [3,4,6,3]): key %s %s" %
                        (key, "missing" if key not in src else "has shape %s, want %s" % (tuple(src[key].shape), shape)))
                self._entry_tensor(name).copy_(src[key].detach().to("cpu"))
            # same RNG consumption as the reference constructor: three nn.Linear are
            # created (posenet.py:46,48,49) before the kaiming initialisation
            tmp_fc = nn.Linear(fe_out_planes, feat_dim)
            tmp_xyz = nn.Linear(feat_dim, 3)
            tmp_wpqr = nn.Linear(feat_dim, 3)
            for nm, lin in (("feature_extractor.fc", tmp_fc), ("fc_xyz", tmp_xyz), ("fc_wpqr", tmp_wpqr)):
                self._entry_tensor(nm + ".weight").copy_(lin.weight)
                self._entry_tensor(nm + ".bias").copy_(lin.bias)
            if pretrained:
                init_names = ["feature_extractor.fc", "fc_xyz", "fc_wpqr"]
            else:
                init_names = [n[:-len(".weight")] for n, k, s, o in self._table
                              if k == 0 and n.endswith(".weight") and len(s) in (2, 4)]
            for nm in init_names:
                w = self._entry_tensor(nm + ".weight")
                tmp = torch.empty(tuple(w.shape))     # contiguous: the same RNG draw -> element mapping as the reference's
                nn.init.kaiming_normal_(tmp)          # nn.init on its contiguous parameters (channels_last views differ)
                w.copy_(tmp)
                if (nm + ".bias") in self._by_name:
                    nn.init.constant_(self._entry_tensor(nm + ".bias"), 0)
        self._trunks = {}
        self._gflat = [None, None]
        self._gsel = 0
        self._fwd_id = 0
        self._step = 0
        self._seed = int(seed) if seed is not None else int(torch.initial_seed() & 0x7FFFFFFFFFFFFFFF)
        self._last_shape = None
        self._graph_rng = False      # True: dropout counter lives on the device (CUDA-graph capture)
        self._grad_part_hook = None  # callable(part, flat_grad_slice) set by ddp.FlatDataParallel (overlapped allreduce)

    # ------------------------------------------------------------------ tree
    def _build_tree(self):
        self._by_name = {}
        self._param_list = []
        for idx, (name, kind, shape, off) in enumerate(self._table):
            parts = name.split(".")
            mod = self
            for p in parts[:-1]:
                if p not in mod._modules:
                    mod.add_module(p, _Node())
                mod = mod._modules[p]
            n = 1
            for s in shape:
                n *= s
            if kind == 0:
                t = nn.Parameter(self._pview(self._flat, name, off, n, shape))
                mod.register_parameter(parts[-1], t)
                self._param_list.append(t)
            elif kind == 1:
                t = self._bufs[off:off + n].view(shape)
                mod.register_buffer(parts[-1], t)
            else:
                t = self._nbt[off:off + 1].view(())
                mod.register_buffer(parts[-1], t)
            self._by_name[name] = (mod, parts[-1], kind, shape, off, n)

    def _pview(self, flat, name, off, n, shape):
        """The entry's tensor as a view of a flat buffer.  Conv weights (all but the stem) are stored in the order the
        wgmma engines read and accumulate them, [Co][KH][KW][Ci] (mapnet_param_layout == 1): the view has the
        reference's [Co,Ci,KH,KW] shape with torch.channels_last strides, so indexing, state_dict(), load_state_dict()
        and optimizers see the same tensor as in the reference while no kernel ever transposes a weight or a gradient."""
        if name in self._krsc:
            co, ci, kh, kw = shape
            return flat[off:off + n].view(co, kh, kw, ci).permute(0, 3, 1, 2)
        return flat[off:off + n].view(shape)

    def _entry_tensor(self, name):
        mod, leaf, kind, shape, off, n = self._by_name[name]
        return mod._parameters[leaf].data if kind == 0 else mod._buffers[leaf]

    def _is_flat(self, device):
        if self._flat.device != device:
            return False
        es = self._flat.element_size()
        first, last = self._table[0], None
        for e in self._table:
            if e[1] == 0:
                last = e
        for e in (first, last):
            if self._entry_tensor(e[0]).data_ptr() != self._flat.data_ptr() + e[3] * es:
                return False
        for e in self._table:
            if e[1] == 1:
                if self._entry_tensor(e[0]).data_ptr() != self._bufs.data_ptr() + e[3] * es:
                    return False
                break
        return True

    def _reflatten(self, device):
        """(Re)binds every parameter / buffer to a view of one flat device tensor.
        nn.Module.cuda()/to() give each tensor its own storage; the kernels want one
        flat buffer (single allreduce, single fused Adam)."""
        with torch.no_grad():
            flat = torch.zeros(self._n_params, dtype=torch.float32, device=device)
            bufs = torch.zeros(self._n_bufs, dtype=torch.float32, device=device)
            nbt = torch.zeros(self._n_nbt, dtype=torch.int64, device=device)
            for name, kind, shape, off in self._table:
                mod, leaf, _, _, _, n = self._by_name[name]
                if kind == 0:
                    p = mod._parameters[leaf]
                    v = self._pview(flat, name, off, n, shape)
                    v.copy_(p.data.to(device=device, dtype=torch.float32))
                    p.data = v
                    p.grad = None
                elif kind == 1:
                    v = bufs[off:off + n].view(shape)
                    v.copy_(mod._buffers[leaf].to(device=device, dtype=torch.float32))
                    mod._buffers[leaf] = v
                else:
                    v = nbt[off:off + 1].view(())
                    v.copy_(mod._buffers[leaf].to(device=device))
                    mod._buffers[leaf] = v
            self._flat, self._bufs, self._nbt = flat, bufs, nbt
            self._gflat = [None, None]

    def _trunk(self, device, B, H, W):
        key = (device.index, H, W)
        t = self._trunks.get(key)
        if t is None or t.max_B < B:
            if t is not None:
                t.close()
            with torch.cuda.device(device):
                t = _lib.Trunk(B, H, W, self.feat_dim, self.precision)
            self._trunks[key] = t
        return t

    # --------------------------------------------------------------- forward
    def forward(self, x):
        if not x.is_cuda:
            raise RuntimeError("geomapnet_b200.PoseNet has no CPU path: input must be a CUDA tensor "
                               "(got %s)" % x.device)
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("expected input [N,3,H,W], got %s" % (tuple(x.shape),))
        if x.shape[0] < 1:
            raise ValueError("empty batch")
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in self._param_list)
        if need_grad and not self.training:
            raise NotImplementedError("geomapnet_b200: backward through eval-mode BatchNorm is not implemented; "
                                      "call model.train() or wrap in torch.no_grad()")
        if need_grad:
            return _TrunkFn.apply(self, x, *self._param_list)
        return self._run_forward(x)

    def _run_forward(self, x):
        xd = x.detach()
        if xd.dtype != torch.float32 or not xd.is_contiguous():
            xd = xd.contiguous().float()
        B, _, H, W = xd.shape
        dev = xd.device
        if not self._is_flat(dev):
            self._reflatten(dev)
        trunk = self._trunk(dev, B, H, W)
        pred = torch.empty(B, 6, dtype=torch.float32, device=dev)
        training = 1 if self.training else 0
        # F.dropout(x, p) at posenet.py:69 passes no `training=`; with the torch this
        # container (and the oracle) runs, that default is True: dropout is active
        # whenever droprate > 0, also under eval().
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().mapnet_forward(
                trunk.h, xd.data_ptr(), self._flat.data_ptr(), self._bufs.data_ptr(), B, training,
                float(self.droprate), self._seed, 0xFFFFFFFFFFFFFFFF if self._graph_rng else self._step,
                pred.data_ptr(), _lib.stream_ptr()),
                "mapnet_forward")
        if training:
            self._nbt += 1
        self._step += 1
        self._fwd_id += 1
        self._last_shape = (dev, B, H, W)
        return pred

    def trainable_mask(self):
        """One flag per parameter, in parameter-table order (= self.parameters()): its requires_grad."""
        return tuple(bool(p.requires_grad) for p in self._param_list)

    def _run_backward(self, dpred, needs):
        dev, B, H, W = self._last_shape
        trunk = self._trunks[(dev.index, H, W)]
        dpred = dpred.contiguous().float()
        trunk.set_trainable(needs)
        # two flat gradient buffers: never write into the one p.grad currently aliases
        sel = self._gsel
        g0 = next((p.grad for p, n in zip(self._param_list, needs) if n), None)
        for cand in (sel, 1 - sel):
            buf = self._gflat[cand]
            if buf is None or buf.device != dev:
                buf = torch.zeros(self._n_params, dtype=torch.float32, device=dev)
                self._gflat[cand] = buf
            if g0 is None or not (buf.data_ptr() <= g0.data_ptr() < buf.data_ptr() + buf.numel() * 4):
                sel = cand
                break
        gbuf = self._gflat[sel]
        self._gsel = sel
        hook = self._grad_part_hook
        with torch.cuda.device(dev):
            if hook is None:
                _lib.check(_lib.lib().mapnet_backward(trunk.h, dpred.data_ptr(), self._flat.data_ptr(),
                                                      gbuf.data_ptr(), 1 if self.filter_nans else 0,
                                                      _lib.stream_ptr()), "mapnet_backward")
            else:
                # data parallel: the pass runs in three parts; after each one the hook may start reducing that part's
                # (final) slice of the flat gradient buffer on another stream while the next part computes
                ranges = trunk.grad_part_ranges()
                for part in range(3):
                    _lib.check(_lib.lib().mapnet_backward_part(trunk.h, part, dpred.data_ptr(), self._flat.data_ptr(),
                                                               gbuf.data_ptr(), 1 if self.filter_nans else 0,
                                                               _lib.stream_ptr()), "mapnet_backward_part")
                    lo, hi = ranges[part]
                    hook(part, gbuf[lo:hi])
        self.last_grad_flat = gbuf
        out = []
        for name, kind, shape, off in self._table:
            if kind == 0:
                n = self._by_name[name][5]
                out.append(self._pview(gbuf, name, off, n, shape) if needs[len(out)] else None)
        return out

    # ------------------------------------------------------- flat-buffer API
    def flat_parameters(self):
        """(flat fp32 parameter tensor, flat gradient tensor of the last backward or None)."""
        return self._flat, getattr(self, "last_grad_flat", None)


class MapNet(nn.Module):
    """models/posenet.py:75-97: folds the T frames of each tuple into the batch."""

    def __init__(self, mapnet):
        super(MapNet, self).__init__()
        self.mapnet = mapnet

    def forward(self, x):
        s = x.size()
        x = x.view(-1, *s[2:])
        poses = self.mapnet(x)
        poses = poses.view(s[0], s[1], -1)
        return poses
