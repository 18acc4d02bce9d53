"""Frozen parameters (requires_grad_(False)) on the H100: the backward pass skips their work and matches torch semantics.

For seven freeze patterns in bf16, tc_split and fp32:
  * the gradients of the parameters that train equal those of a full backward of the same forward, within the spread of
    two full backwards (0 in practice: the wgrad split-K reduction has a fixed order);
  * frozen parameters get .grad None and exact zeros in the flat gradient buffer;
  * the dgrad / wgrad conv launches are those the skipping rule predicts from the parameter table;
and, separately: the default mask is the old schedule (bitwise, same launch count), a CUDA-graph step of a partly frozen
model follows the eager steps, changing requires_grad after capture makes replay() raise, and the three backward parts
compose to the masked one-call backward."""
import ctypes
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

PRECS = ("bf16", "tc_split", "fp32")
CFGS = {"tiny": dict(kind="posenet", N=4, H=64, W=64), "b8_256": dict(kind="posenet", N=8, H=256, W=256)}
FE = "feature_extractor."
HEAD = (FE + "fc.", "fc_xyz.", "fc_wpqr.")


def _head(n):
    return n.startswith(HEAD)


PATTERNS = {
    "a_head": _head,
    "b_layer4_head": lambda n: _head(n) or n.startswith(FE + "layer4."),
    "c_layer3.1_up": lambda n: (_head(n) or n.startswith(FE + "layer4.")
                                or any(n.startswith(FE + "layer3.%d." % i) for i in range(1, 6))),
    "d_bn_affine": lambda n: re.search(r"\.(bn\d|downsample\.1)\.(weight|bias)$", n) is not None,
    "e_layer2.1.conv2": lambda n: n == FE + "layer2.1.conv2.weight",
    "f_stem": lambda n: n.startswith((FE + "conv1.", FE + "bn1.")),
    "g_all_but_layer1": lambda n: not n.startswith(FE + "layer1."),
}


def expected_conv_launches(names, mask, fold):
    """(dgrad, wgrad) conv launches of one masked backward: the pass stops at the lowest block with a trainable conv or
    BatchNorm (the stem, when conv1 / bn1 trains); that block computes no input gradient unless the stem trains; a conv's
    wgrad runs when its weight trains.  fold: a stride-2 block's downsample dgrad rides in its conv1 dgrad launch."""
    tr = [n for n, m in zip(names, mask) if m]
    blocks = sorted({re.match(r"feature_extractor\.layer(\d)\.(\d)\.", n).groups() for n in names
                     if re.match(r"feature_extractor\.layer\d\.\d\.", n)}, key=lambda b: (int(b[0]), int(b[1])))
    pre = ["%slayer%s.%s." % (FE, l, b) for l, b in blocks]
    lo = len(blocks)
    for bi in reversed(range(len(blocks))):
        if any(n.startswith(pre[bi]) for n in tr):
            lo = bi
    if any(n.startswith((FE + "conv1.", FE + "bn1.")) for n in tr):
        lo = -1
    dgrad = 0
    for bi in range(max(lo, 0), len(blocks)):
        ds = any(n.startswith(pre[bi] + "downsample.") for n in names)
        dgrad += 1 + ((2 if ds and not fold else 1) if bi > lo else 0)
    wgrad = sum(1 for n in tr if re.search(r"(conv\d|downsample\.0)\.weight$", n))
    return dgrad, wgrad


class Rig(object):
    """One model of one precision / input size, and the step the tests repeat on it."""

    def __init__(self, precision, cfg):
        from oracle import weights
        from helpers import make_product_model
        self.state = weights.make_state(7)
        self.model, self.net = make_product_model(self.state, "posenet", precision)
        self.model.train()
        x, _ = weights.make_inputs(cfg, 11)
        self.x = x.cuda()
        g = torch.Generator().manual_seed(5)
        self.w = torch.randn(cfg["N"], 6, generator=g).cuda()        # d loss / d pred
        self.names = [nm for nm, _ in self.net.named_parameters()]
        self.slices = []
        for name, kind, shape, off in self.net._table:
            if kind == 0:
                self.slices.append((off, self.net._by_name[name][5]))
        self.HW = (cfg["H"], cfg["W"])
        self.full = (True,) * len(self.names)
        ln = self.profiled(self.full)
        # the wgmma bf16 path folds the 3 downsample dgrads into conv1's launch
        self.fold = (ln[1] == 32)
        assert ln[1:] == list(expected_conv_launches(self.names, self.full, self.fold)), ln

    def mask(self, pattern):
        return tuple(bool(PATTERNS[pattern](n)) for n in self.names)

    def step(self, mask):
        for p, m in zip(self.net._param_list, mask):
            p.requires_grad_(m)
            p.grad = None
        out = self.model(self.x)
        (out * self.w).sum().backward()
        torch.cuda.synchronize()
        return out.detach().clone(), self.net.flat_parameters()[1].clone(), [p.grad for p in self.net._param_list]

    def profiled(self, mask):
        from geomapnet_b200 import _lib
        L = _lib.lib()
        trunk = self.net._trunks[(0,) + self.HW] if (0,) + self.HW in self.net._trunks else None
        if trunk is None:
            self.step(mask)             # creates the handle
            trunk = self.net._trunks[(0,) + self.HW]
        _lib.check(L.mapnet_profile(trunk.h, 1), "mapnet_profile")
        try:
            self.step(mask)
            ms, fl, ln = (ctypes.c_double * 3)(), (ctypes.c_double * 3)(), (ctypes.c_int * 3)()
            _lib.check(L.mapnet_profile_read(trunk.h, ms, fl, ln), "mapnet_profile_read")
        finally:
            L.mapnet_profile(trunk.h, 0)
        return list(ln)


_RIGS = {}


def rig(precision, cfg):
    key = (precision, cfg)
    if key not in _RIGS:
        _RIGS.clear()           # one model at a time on the device
        _RIGS[key] = Rig(precision, CFGS[cfg])
    return _RIGS[key]


@pytest.mark.parametrize("pattern", list(PATTERNS))      # the first decorator varies fastest: one model per
@pytest.mark.parametrize("cfg", list(CFGS))              # (precision, size)
@pytest.mark.parametrize("precision", PRECS)
def test_masked_backward(precision, cfg, pattern):
    r = rig(precision, cfg)
    mask = r.mask(pattern)
    assert any(mask) and not all(mask)
    pred1, full1, _ = r.step(r.full)
    pred2, full2, _ = r.step(r.full)
    pred, g, grads = r.step(mask)
    assert torch.equal(pred, pred1) and torch.equal(pred1, pred2)
    spread, err = 0.0, 0.0
    for (off, n), m, gr, name in zip(r.slices, mask, grads, r.names):
        if m:
            assert gr is not None, name
            spread = max(spread, float((full1[off:off + n] - full2[off:off + n]).abs().max()))
            err = max(err, float((g[off:off + n] - full1[off:off + n]).abs().max()))
            assert float(g[off:off + n].abs().max()) > 0, name          # really computed
        else:
            assert gr is None, name
            assert not bool(g[off:off + n].any()), "%s: frozen entry of the flat gradient is not 0" % name
    assert err <= spread, (pattern, err, spread)
    ln = r.profiled(mask)
    want = expected_conv_launches(r.names, mask, r.fold)
    assert tuple(ln[1:]) == want, (pattern, ln, want)
    if pattern == "a_head":
        assert want == (0, 0)


@pytest.mark.parametrize("precision", PRECS)
def test_default_mask_is_the_full_schedule(precision):
    """A handle whose mask was set to something else and back to all ones runs exactly what a handle whose mask was never
    set runs: same launches, bitwise the same outputs."""
    from geomapnet_b200 import _lib
    L = _lib.lib()
    r = rig(precision, "tiny")
    B, H, W = r.x.shape[0], r.HW[0], r.HW[1]
    flat = r.net._flat
    n = len(r.names)
    res = []
    for touched in (False, True):
        t = _lib.Trunk(B, H, W, r.net.feat_dim, precision)
        try:
            if touched:
                for m in (r.mask("c_layer3.1_up"), r.full):
                    buf = (ctypes.c_uint8 * n)(*[int(v) for v in m])
                    _lib.check(L.mapnet_trunk_set_trainable(t.h, buf, n), "mapnet_trunk_set_trainable")
            out = []
            for _ in range(2):
                bufs = r.net._bufs.clone()
                pred = torch.empty(B, 6, device="cuda")
                gr = torch.full((flat.numel(),), 7.0, device="cuda")
                c0 = L.mapnet_launch_count()
                _lib.check(L.mapnet_forward(t.h, r.x.data_ptr(), flat.data_ptr(), bufs.data_ptr(), B, 1, 0.0, 3, 0,
                                            pred.data_ptr(), _lib.stream_ptr()), "mapnet_forward")
                _lib.check(L.mapnet_backward(t.h, r.w.data_ptr(), flat.data_ptr(), gr.data_ptr(), 0, _lib.stream_ptr()),
                           "mapnet_backward")
                torch.cuda.synchronize()
                out.append((int(L.mapnet_launch_count() - c0), pred, gr, bufs))
            res.append(out)
        finally:
            t.close()
    for (c0, p0, g0, b0), (c1, p1, g1, b1) in zip(*res):
        assert c0 == c1
        assert torch.equal(p0, p1) and torch.equal(g0, g1) and torch.equal(b0, b1)


@pytest.mark.parametrize("precision", PRECS)
def test_backward_parts_compose(precision):
    """mapnet_backward_part 0, 1, 2 (the data-parallel overlap path) under a mask give the one-call masked gradients."""
    r = rig(precision, "b8_256")
    mask = r.mask("c_layer3.1_up")
    _, g1, _ = r.step(mask)
    _, g2, _ = r.step(mask)
    spread = float((g1 - g2).abs().max())
    parts = []
    r.net._grad_part_hook = lambda part, sl: parts.append(part)
    try:
        _, gp, grads = r.step(mask)
    finally:
        r.net._grad_part_hook = None
    assert parts == [0, 1, 2]
    assert float((gp - g1).abs().max()) <= spread
    assert all((gr is None) == (not m) for gr, m in zip(grads, mask))


def _train(precision, graphed, batches, mask, lr):
    from oracle import weights
    from helpers import make_product_model, make_product_criterion
    from geomapnet_b200.common.optimizer import Optimizer
    from geomapnet_b200.graph import GraphedTrainStep
    st = weights.make_state(7)
    model, net = make_product_model(st, "posenet", precision)
    crit = make_product_criterion("posenet", learn=False)
    for p, m in zip(net._param_list, mask):
        p.requires_grad_(m)
    opt = Optimizer([{"params": model.parameters()}], "adam", lr, 5e-4)
    model.train()
    g = None
    if graphed:
        x0, t0 = batches[0]
        g = GraphedTrainStep(model, crit, opt, x0.cuda(), t0.cuda(), warmup=2)
        for x, t in batches:
            g(x.cuda(), t.cuda())
    else:
        for x, t in batches:
            loss = crit(model(x.cuda()), t.cuda())
            opt.learner.zero_grad()
            loss.backward()
            opt.learner.step()
    torch.cuda.synchronize()
    return st, {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}, net, g, batches


def test_graphed_training_with_frozen_layers():
    """Five CUDA-graph steps of a model whose layers below layer4 are frozen (FusedAdam, weight decay) follow five eager
    steps; frozen weights stay bitwise unchanged in both, while the running statistics of every BatchNorm, frozen or
    not, keep following the forward (training mode) as in torch.  Changing requires_grad afterwards makes replay() raise."""
    from oracle import weights
    cfg = CFGS["b8_256"]
    batches = [weights.make_inputs(cfg, 30 + i) for i in range(5)]
    lr = 1e-5
    from geomapnet_b200 import _lib
    spec = _lib.Trunk(0, 64, 64, 2048, "bf16")
    names = [e[0] for e in spec.table()[0] if e[1] == 0]
    spec.close()
    mask = tuple(bool(PATTERNS["b_layer4_head"](nm)) for nm in names)
    runs = [_train("bf16", graphed, batches, mask, lr) for graphed in (False, True)]
    (st, se, _, _, _), (_, sg, net, g, _) = runs
    frozen = [nm for nm, m in zip(names, mask) if not m]
    trained = [nm for nm, m in zip(names, mask) if m]
    for nm in frozen:
        assert torch.equal(se[nm], st[nm]) and torch.equal(sg[nm], st[nm]), nm
    stats = [k for k in se if k.endswith(("running_mean", "running_var"))]
    frozen_stats = [k for k in stats if k.startswith(FE) and not k.startswith(FE + "layer4.")]
    assert frozen_stats

    def mean_dev(u, v, keys):
        return sum(float((u[k] - v[k]).abs().sum()) for k in keys) / sum(u[k].numel() for k in keys)

    moved, dev = mean_dev(se, st, trained), mean_dev(se, sg, trained)
    bmoved, bdev = mean_dev(se, st, frozen_stats), mean_dev(se, sg, frozen_stats)
    print("frozen-layer graph-vs-eager: trained parameters moved %.3e, graph/eager %.3e; frozen BN statistics moved "
          "%.3e, graph/eager %.3e" % (moved, dev, bmoved, bdev))
    assert moved > 1.5 * lr
    assert dev <= 0.05 * moved, (moved, dev)
    assert bmoved > 0 and bdev <= 0.02 * bmoved, (bmoved, bdev)
    for k in se:
        if not se[k].dtype.is_floating_point:
            assert torch.equal(se[k], sg[k]), k               # num_batches_tracked
    # the captured schedule belongs to the mask at capture
    x, t = batches[0]
    net.fc_xyz.weight.requires_grad_(False)
    with pytest.raises(RuntimeError, match="requires_grad"):
        g(x.cuda(), t.cuda())
    net.fc_xyz.weight.requires_grad_(True)
    w = dict(net.named_parameters())[FE + "layer3.0.conv1.weight"]
    w.requires_grad_(True)
    with pytest.raises(RuntimeError, match="requires_grad"):
        g.replay()
    w.requires_grad_(False)
    g(x.cuda(), t.cuda())                                     # the capture's mask again: replays
    torch.cuda.synchronize()
