"""FusedSGD / FusedRMSprop on the GPU: the kernels against torch.optim's single-tensor arithmetic, the fused scale and
clip, checkpoint interchange with torch in both directions, one step of the product model, CUDA-graph replay that
follows the learning-rate schedule, and the data-parallel step (the reference's common/optimizer.py:16-27 methods)."""
import copy
import os
import socket
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SGD_TOL = dict(rtol=1e-6, atol=1e-7)
RMS_TOL = dict(rtol=2e-5, atol=1e-6)

# momentum x dampening x nesterov x weight decay, the combinations torch accepts (nesterov: momentum > 0, dampening 0)
SGD_CASES = [dict(momentum=m, dampening=d, nesterov=n, weight_decay=wd)
             for m in (0.0, 0.9) for d in (0.0, 0.1) for n in (False, True) for wd in (0.0, 5e-4)
             if not (n and (m == 0.0 or d != 0.0))]
RMS_CASES = [dict(momentum=m, centered=c, weight_decay=wd) for m in (0.0, 0.9) for c in (False, True) for wd in (0.0, 5e-4)]


def _case_id(kw):
    return "-".join("%s%s" % (k[:4], v) for k, v in kw.items())


def _layout(seed):
    """The layout of test_fused_adam_matches_torch_adam -- one flat buffer with gaps, a 1-element tensor and an
    unaligned tail -- plus a free-standing parameter at an address that is not 16-byte aligned (scalar path).
    Returns (fused parameters, torch parameters, setter of identical gradients)."""
    torch.manual_seed(seed)
    flat = torch.randn(10240, device="cuda")
    shapes = [(100, 50), (4999,), (1,)]
    offs = [0, 5056, 10112]
    loose = torch.randn(8, device="cuda")[1:]                  # 4 bytes past an allocation: not 16-byte aligned
    ps = [torch.nn.Parameter(flat[o:o + int(np.prod(s))].view(s)) for s, o in zip(shapes, offs)]
    ps.append(torch.nn.Parameter(loose))
    qs = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    gflat = torch.zeros_like(flat)
    gloose = torch.zeros(8, device="cuda")[1:]

    def set_grads(scale=1.0):
        # the padding between the parameters stays zero, as in the product's flat gradient buffer (the clip's norm
        # sweeps the whole run)
        g = torch.zeros_like(flat)
        for s, o in zip(shapes, offs):
            n = int(np.prod(s))
            g[o:o + n] = torch.randn(n, device="cuda") * scale
        gl = torch.randn(7, device="cuda") * scale
        gflat.copy_(g); gloose.copy_(gl)
        for i, (s, o) in enumerate(zip(shapes, offs)):
            n = int(np.prod(s))
            ps[i].grad = gflat[o:o + n].view(s)
            qs[i].grad = g[o:o + n].view(s).clone()
        ps[3].grad = gloose
        qs[3].grad = gl.clone()
    return ps, qs, set_grads


def _assert_close(ps, qs, a, b, keys, tol):
    """Parameters within `tol`; state buffers within `tol` with atol relative to the buffer's largest element (an
    RMSprop momentum buffer sums d/avg terms of magnitude ~10, whose last-bit rounding is ~1e-6 absolute)."""
    for p, q in zip(ps, qs):
        torch.testing.assert_close(p.detach(), q.detach(), **tol)
        for k in keys:
            if k in b.state[q]:
                want = b.state[q][k]
                scale = max(1.0, float(want.abs().max()))
                torch.testing.assert_close(a.state[p][k], want, rtol=tol["rtol"], atol=tol["atol"] * scale, msg=k)


@pytest.mark.parametrize("kw", SGD_CASES, ids=_case_id)
def test_fused_sgd_matches_torch_sgd(kw):
    from geomapnet_b200.common.optimizer import FusedSGD
    ps, qs, set_grads = _layout(0)
    a = FusedSGD(ps, lr=1e-2, **kw)
    b = torch.optim.SGD(qs, lr=1e-2, foreach=False, **kw)
    for it in range(5):
        set_grads()
        a.step(); b.step()
    _assert_close(ps, qs, a, b, ["momentum_buffer"], SGD_TOL)
    assert ("momentum_buffer" in a.state[ps[0]]) == (kw["momentum"] != 0)


@pytest.mark.parametrize("kw", RMS_CASES, ids=_case_id)
def test_fused_rmsprop_matches_torch_rmsprop(kw):
    from geomapnet_b200.common.optimizer import FusedRMSprop
    ps, qs, set_grads = _layout(1)
    a = FusedRMSprop(ps, lr=1e-2, **kw)
    b = torch.optim.RMSprop(qs, lr=1e-2, foreach=False, **kw)
    for it in range(5):
        set_grads()
        a.step(); b.step()
    _assert_close(ps, qs, a, b, ["square_avg", "momentum_buffer", "grad_avg"], RMS_TOL)
    assert float(a.state[ps[0]]["step"]) == 5.0
    assert set(a.state_dict()["state"][0]) == set(b.state_dict()["state"][0])


@pytest.mark.parametrize("method", ["sgd", "rmsprop"])
def test_scale_and_clip_on_group_zero(method):
    """step(grad_scale=0.5, max_grad_norm=5.0) with two groups == torch after scaling every gradient, clipping group 0
    (the model, common/train.py:357-358) and stepping; group 1 is neither counted nor scaled by the clip."""
    from geomapnet_b200.common.optimizer import FusedRMSprop, FusedSGD
    ps, qs, set_grads = _layout(2)
    if method == "sgd":
        kw, tol = dict(lr=1e-2, momentum=0.9, nesterov=True, weight_decay=5e-4), SGD_TOL
        a, b = FusedSGD([{"params": ps[:3]}, {"params": ps[3:]}], **kw), torch.optim.SGD(
            [{"params": qs[:3]}, {"params": qs[3:]}], foreach=False, **kw)
    else:
        kw, tol = dict(lr=1e-2, momentum=0.9, centered=True, weight_decay=5e-4), RMS_TOL
        a, b = FusedRMSprop([{"params": ps[:3]}, {"params": ps[3:]}], **kw), torch.optim.RMSprop(
            [{"params": qs[:3]}, {"params": qs[3:]}], foreach=False, **kw)
    for it in range(3):
        set_grads(scale=3.0)
        a.step(grad_scale=0.5, max_grad_norm=5.0)
        with torch.no_grad():
            for q in qs:
                q.grad.mul_(0.5)
        norm = torch.nn.utils.clip_grad_norm_(qs[:3], 5.0)
        assert float(norm) > 5.0                                  # the clip is active
        b.step()
    _assert_close(ps, qs, a, b, ["momentum_buffer", "square_avg", "grad_avg"], tol)


class _Holder(torch.nn.Module):
    def __init__(self, params):
        super(_Holder, self).__init__()
        self.ps = torch.nn.ParameterList(params)


@pytest.mark.parametrize("method", ["sgd", "rmsprop"])
def test_checkpoint_interchange_with_torch(method, tmp_path):
    """Two torch steps -> state_dict -> deepcopy -> Fused*.load_state_dict -> two fused steps == four torch steps, and
    the fused state dict loads back into torch; once more through save_checkpoint / load_checkpoint(resume_optim)."""
    from geomapnet_b200.common.checkpoint import load_checkpoint, save_checkpoint
    from geomapnet_b200.common.optimizer import FusedRMSprop, FusedSGD
    if method == "sgd":       # dampening: the first fused step after a resume must NOT re-initialise the buffer
        fused_cls, torch_cls, kw, tol = FusedSGD, torch.optim.SGD, dict(lr=1e-2, momentum=0.9, dampening=0.1), SGD_TOL
        keys = ["momentum_buffer"]
    else:
        fused_cls, torch_cls, kw, tol = (FusedRMSprop, torch.optim.RMSprop,
                                         dict(lr=1e-2, momentum=0.9, centered=True), RMS_TOL)
        keys = ["square_avg", "momentum_buffer", "grad_avg"]
    ps, qs, set_grads = _layout(3)
    rs = [torch.nn.Parameter(q.detach().clone()) for q in qs]     # the torch-only run of four steps
    b = torch_cls(qs, foreach=False, **kw)
    ref = torch_cls(rs, foreach=False, **kw)

    def grads():
        set_grads()
        for r, q in zip(rs, qs):
            r.grad = q.grad.clone()
    for it in range(2):
        grads(); b.step(); ref.step()
    with torch.no_grad():
        for p, q in zip(ps, qs):
            p.copy_(q)
    a = fused_cls(ps, **kw)
    a.load_state_dict(copy.deepcopy(b.state_dict()))
    for it in range(2):
        grads(); a.step(); ref.step()
    _assert_close(ps, rs, a, ref, keys, tol)
    # ... and back: the fused state dict into torch, one more step each
    back = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    c = torch_cls(back, foreach=False, **kw)
    c.load_state_dict(copy.deepcopy(a.state_dict()))
    grads()
    for p, q in zip(back, rs):
        p.grad = q.grad.clone()
    c.step(); ref.step()
    _assert_close(back, rs, c, ref, keys, tol)
    # through the checkpoint files of common/train.py:198-204 / 160-177
    model = _Holder(ps)
    fname = save_checkpoint(str(tmp_path), 4, model, a, torch.nn.Module())
    ps2 = [torch.nn.Parameter(torch.zeros_like(p)) for p in ps]
    a2 = fused_cls(ps2, **kw)
    assert load_checkpoint(fname, _Holder(ps2), a2, torch.nn.Module(), resume_optim=True) == 4
    grads()
    for p2, p in zip(ps2, ps):
        p2.grad = p.grad.detach().clone()
    a.step(); a2.step()
    _assert_close(ps2, ps, a2, a, keys, tol)


def test_product_model_one_eager_sgd_step():
    """Optimizer('sgd') on the product PoseNet (channels_last conv weights, padded flat buffer, free-standing criterion
    scalars) against a plain torch.optim.SGD on an identical model, from identical gradients (two steps: the first
    initialises the momentum buffers, the second decays them)."""
    from oracle import weights
    from helpers import make_product_model, make_product_criterion
    from geomapnet_b200.common.optimizer import FusedSGD, Optimizer
    st = weights.make_state(7)
    x, t = weights.make_inputs(dict(kind="posenet", N=4, H=64, W=64), 7)
    sides = []
    for _ in range(2):
        model, net = make_product_model(st, "posenet", "fp32")
        crit = make_product_criterion("posenet", learn=True)
        model.train()
        loss = crit(model(x.cuda()), t.cuda())
        loss.backward()
        sides.append((model, net, crit))
    (ma, na, ca), (mb, nb, cb) = sides
    with torch.no_grad():
        for pa, pb in zip(list(na.parameters()) + list(ca.parameters()), list(nb.parameters()) + list(cb.parameters())):
            pb.grad.copy_(pa.grad)
    kw = dict(momentum=0.9, weight_decay=5e-4)
    opt = Optimizer([{"params": ma.parameters()}, {"params": list(ca.parameters())}], "sgd", 1e-2, lr_decay=0.1,
                    lr_stepvalues=[60, 80], **kw)
    assert isinstance(opt.learner, FusedSGD)
    ref = torch.optim.SGD([{"params": mb.parameters()}, {"params": list(cb.parameters())}], lr=1e-2, **kw)
    for _ in range(2):
        opt.learner.step(); ref.step()
    conv = dict(na.named_parameters())["feature_extractor.layer1.0.conv1.weight"]
    assert conv.is_contiguous(memory_format=torch.channels_last) and not conv.is_contiguous()
    assert len(opt.learner._runs[0][1]) == 1                     # the whole model is one run (one launch)
    for (n, pa), pb in zip(na.named_parameters(), nb.parameters()):
        torch.testing.assert_close(pa.detach(), pb.detach(), rtol=1e-6, atol=1e-7, msg=n)
        torch.testing.assert_close(opt.learner.state[pa]["momentum_buffer"], ref.state[pb]["momentum_buffer"],
                                   rtol=1e-6, atol=1e-7, msg=n)
    for pa, pb in zip(ca.parameters(), cb.parameters()):
        torch.testing.assert_close(pa.detach(), pb.detach(), rtol=1e-6, atol=1e-7)
    flat, _ = na.flat_parameters()
    assert bool(torch.isfinite(flat).all())


def _graph_setup(method, lr):
    from oracle import weights
    from helpers import make_product_model, make_product_criterion
    from geomapnet_b200.common.optimizer import Optimizer
    st = weights.make_state(7)
    model, net = make_product_model(st, "mapnet", "fp32")
    crit = make_product_criterion("mapnet")
    groups = [{"params": model.parameters()}, {"params": list(crit.parameters())}]
    if method == "sgd":
        opt = Optimizer(groups, "sgd", lr, 5e-4, momentum=0.9, lr_decay=0.1, lr_stepvalues=[1])
    else:
        opt = Optimizer(groups, "rmsprop", lr, 5e-4, momentum=0.9)
    model.train()
    return st, model, net, crit, opt


def test_graphed_sgd_follows_the_schedule():
    """GraphedTrainStep with Optimizer('sgd', momentum=0.9, lr_decay=0.1, lr_stepvalues=[1]) against the eager step
    over four batches with adjust_lr(0), adjust_lr(0), adjust_lr(1), adjust_lr(1): a rate frozen at its capture value
    would make the last two steps ten times too long.  Same mean-deviation criteria as test_graphed_step_matches_eager."""
    from oracle import weights
    from geomapnet_b200.graph import GraphedTrainStep
    cfg = dict(kind="mapnet", N=2, T=3, H=64, W=64)
    batches = [weights.make_inputs(cfg, 20 + i) for i in range(4)]
    epochs = [0, 0, 1, 1]
    lr = 1e-4
    finals = []
    for use_graph in (False, False, True):
        st, model, net, crit, opt = _graph_setup("sgd", lr)
        losses = []
        if use_graph:
            x0, t0 = batches[0]
            g = GraphedTrainStep(model, crit, opt, x0.cuda(), t0.cuda(), max_grad_norm=5.0, warmup=2)
            for k, v in net.state_dict().items():
                assert torch.equal(v.cpu(), st[k]), "GraphedTrainStep construction changed %s" % k
            # the optimizer state is as before the warm-up: no momentum yet, the next step is the first
            for p, s in opt.learner.state.items():
                assert float(s["momentum_buffer"].abs().max()) == 0.0
            for key, runs in opt.learner._runs.values():
                for r in runs:
                    assert r["step_host"] == 0 and int(r["step_dev"].item()) == 0
            for (x, t), ep in zip(batches, epochs):
                opt.adjust_lr(ep)
                losses.append(float(g(x.cuda(), t.cuda())))
        else:
            for (x, t), ep in zip(batches, epochs):
                opt.adjust_lr(ep)
                out = model(x.cuda()); loss = crit(out, t.cuda())
                opt.learner.zero_grad(); loss.backward(); opt.learner.step(max_grad_norm=5.0)
                losses.append(float(loss.detach()))
        torch.cuda.synchronize()
        assert abs(opt.learner.param_groups[0]["lr"] - lr * 0.1) < 1e-15
        finals.append((losses, {k: v.detach().cpu().clone() for k, v in net.state_dict().items()},
                       [float(p.detach()) for p in crit.parameters()], st))
    (la, sa, ca, st), (l2, s2, c2, _), (lb, sb, cb, _) = finals
    assert abs(la[0] - lb[0]) <= 1e-6 * abs(la[0])
    pkeys = [k for k in sa if sa[k].dtype.is_floating_point and not k.endswith(("running_mean", "running_var"))]
    bkeys = [k for k in sa if k.endswith(("running_mean", "running_var"))]

    def mean_dev(u, v, keys):
        return sum(float((u[k] - v[k]).abs().sum()) for k in keys) / sum(u[k].numel() for k in keys)

    moved = mean_dev(sa, st, pkeys)
    noise, dev = mean_dev(sa, s2, pkeys), mean_dev(sa, sb, pkeys)
    bmoved, bdev = mean_dev(sa, st, bkeys), mean_dev(sa, sb, bkeys)
    lg = max(abs(a - b) / abs(a) for a, b in zip(la, lb))
    print("graphed SGD vs eager: parameters moved %.3e; mean deviation eager/eager %.3e, graph/eager %.3e; "
          "BN buffers moved %.3e, graph/eager %.3e; loss deviation %.2e" % (moved, noise, dev, bmoved, bdev, lg))
    assert moved > 0.0
    assert dev <= 0.05 * moved, (moved, noise, dev)
    assert bdev <= 0.02 * bmoved, (bmoved, bdev)
    assert lg <= 2e-3, (la, l2, lb)
    from helpers import SVALS
    for a, b, a0 in zip(ca, cb, [SVALS[k] for k in ("sax", "saq", "srx", "srq")]):
        assert abs(a - b) <= 0.05 * abs(a - a0) + 1e-9, (ca, cb)


@pytest.mark.parametrize("method", ["sgd", "rmsprop"])
def test_graph_reads_the_device_rate(method):
    """After mult_lr(0.0) one replay leaves every parameter bit-identical while the BatchNorm running statistics still
    move: the captured launch reads the rate the host wrote after capture."""
    from oracle import weights
    from geomapnet_b200.graph import GraphedTrainStep
    cfg = dict(kind="mapnet", N=2, T=3, H=64, W=64)
    (x0, t0), (x1, t1) = [weights.make_inputs(cfg, 30 + i) for i in range(2)]
    st, model, net, crit, opt = _graph_setup(method, 1e-4)
    g = GraphedTrainStep(model, crit, opt, x0.cuda(), t0.cuda(), warmup=2)
    g(x0.cuda(), t0.cuda())
    torch.cuda.synchronize()
    moved = {k: v.detach().clone() for k, v in net.state_dict().items()}
    assert any(not torch.equal(moved[k], st[k].cuda()) for k in moved if k.endswith("weight"))   # a real step
    crit0 = [p.detach().clone() for p in crit.parameters()]
    opt.mult_lr(0.0)
    g(x1.cuda(), t1.cuda())
    torch.cuda.synchronize()
    after = net.state_dict()
    bn_moved = False
    for k, v in after.items():
        if k.endswith(("running_mean", "running_var")):
            bn_moved = bn_moved or not torch.equal(v, moved[k])
        elif v.dtype.is_floating_point:
            assert torch.equal(v, moved[k]), k
    assert bn_moved
    for p, q in zip(crit.parameters(), crit0):
        assert torch.equal(p.detach(), q)


# ---------------------------------------------------------------------------------------------------------------------
# data parallel: FlatDataParallel + FusedSGD.step(grad_scale=1/world) == one process stepping on the mean gradient
# ---------------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _ddp_worker(rank, world, port, q):
    try:
        q.put((rank, _ddp_body(rank, world, port)))
    except Exception:                            # report instead of leaving the peer waiting in a collective
        import traceback
        traceback.print_exc()
        sys.stderr.flush()
        q.put((rank, False))
        os._exit(1)


def _ddp_body(rank, world, port):
    import torch.distributed as dist
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from oracle import weights
    from helpers import make_product_model, make_product_criterion
    from geomapnet_b200.common.optimizer import FusedSGD, Optimizer
    from geomapnet_b200.ddp import FlatDataParallel, shard_tuples
    st = weights.make_state(7)
    cfg = dict(kind="mapnet", N=4, T=3, H=64, W=64)
    x, targ = weights.make_inputs(cfg, 7)
    xs, ts = shard_tuples(x, rank, world).cuda(), shard_tuples(targ, rank, world).cuda()
    model, net = make_product_model(st, "mapnet", "fp32")
    crit = make_product_criterion("mapnet")
    kw = dict(momentum=0.9, weight_decay=5e-4)
    opt = Optimizer([{"params": model.parameters()}, {"params": list(crit.parameters())}], "sgd", 1e-2,
                    lr_decay=0.1, lr_stepvalues=[60], **kw)
    ok = isinstance(opt.learner, FusedSGD)
    model.train()
    model(xs)
    dp = FlatDataParallel(model, crit)
    dp.broadcast_parameters()
    flat, _ = net.flat_parameters()
    before = flat.clone()
    crit_before = [p.detach().clone() for p in crit.parameters()]
    loss = crit(model(xs), ts)
    opt.learner.zero_grad()
    loss.backward()
    _, g = net.flat_parameters()
    local = [g.clone()] + [p.grad.clone() for p in crit.parameters()]
    gathered = []
    for t in local:
        parts = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(parts, t)
        gathered.append(parts)
    scale = dp.allreduce_grads()
    opt.learner.step(grad_scale=scale)
    # one process stepping on the mean gradient: torch.optim.SGD over the whole flat buffer and the criterion scalars
    refs = []
    for start, parts in zip([before] + crit_before, gathered):
        r = torch.nn.Parameter(start.clone())
        r.grad = sum(parts) / world
        refs.append(r)
    ref = torch.optim.SGD([{"params": refs[:1]}, {"params": refs[1:]}], lr=1e-2, foreach=False, **kw)
    ref.step()
    for got, want in zip([flat] + [p.detach() for p in crit.parameters()], refs):
        ok = ok and bool(torch.allclose(got, want.detach(), rtol=1e-6, atol=1e-7))
    after = flat.clone(); dist.broadcast(after, src=0)
    ok = ok and torch.equal(flat, after)           # replicas stay in lock-step
    torch.cuda.synchronize()
    dist.destroy_process_group()
    return bool(ok)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_fused_sgd_data_parallel_nccl_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = []
    try:
        while len(res) < 2:
            res.append(q.get(timeout=180))
            if not res[-1][1]:
                break
    finally:
        for p in procs:
            p.join(5 if (res and not res[-1][1]) else 60)
            if p.is_alive():
                p.kill()                         # exactly the processes started above
    assert sorted(res) == [(0, True), (1, True)]
