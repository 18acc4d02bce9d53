"""FusedSGD / FusedRMSprop host logic that needs no GPU: the wrapper builds them, torch's constructor checks still
apply, CPU parameters keep torch's own step (with grad_scale and the clip applied first), and the run planner shared
with FusedAdam binds the method's state buffers as views in each parameter's element order."""
import copy

import pytest
import torch

from geomapnet_b200.common.optimizer import FusedRMSprop, FusedSGD, Optimizer


@pytest.fixture(scope="module")
def built():
    from geomapnet_b200 import build
    return build.build(verbose=False)


def test_wrapper_builds_fused_sgd_and_rmsprop(built):
    p = [torch.nn.Parameter(torch.zeros(3))]
    s = Optimizer(params=p, method="sgd", base_lr=0.1, weight_decay=5e-4, lr_decay=0.1, lr_stepvalues=[60, 80],
                  momentum=0.9)
    assert isinstance(s.learner, FusedSGD) and isinstance(s.learner, torch.optim.SGD)
    assert s.learner.param_groups[0]["momentum"] == 0.9 and s.learner.param_groups[0]["weight_decay"] == 5e-4
    assert abs(s.adjust_lr(80) - 0.001) < 1e-12 and abs(s.learner.param_groups[0]["lr"] - 0.001) < 1e-12
    r = Optimizer(params=p, method="rmsprop", base_lr=1e-3, weight_decay=0.0, alpha=0.9, centered=True)
    assert isinstance(r.learner, FusedRMSprop) and isinstance(r.learner, torch.optim.RMSprop)
    assert r.learner.param_groups[0]["alpha"] == 0.9 and r.learner.param_groups[0]["centered"]
    assert r.adjust_lr(100) == 1e-3 and r.learner.param_groups[0]["lr"] == 1e-3      # no schedule but SGD's


def test_torch_constructor_checks_still_raise(built):
    p = [torch.nn.Parameter(torch.zeros(3))]
    with pytest.raises(ValueError):
        FusedSGD(p, lr=0.1, momentum=0.9, dampening=0.1, nesterov=True)
    with pytest.raises(ValueError):
        FusedSGD(p, lr=0.1, momentum=0.0, nesterov=True)
    with pytest.raises(ValueError):
        FusedSGD(p, lr=-0.1)
    with pytest.raises(ValueError):
        FusedRMSprop(p, lr=1e-3, alpha=-0.5)
    with pytest.raises(ValueError):
        FusedRMSprop(p, lr=1e-3, momentum=-0.1)
    with pytest.raises(ValueError):
        Optimizer(params=p, method="sgd", base_lr=0.1, weight_decay=0.0, lr_decay=0.1, lr_stepvalues=[1],
                  momentum=0.0, nesterov=True)


CPU_CASES = [(FusedSGD, torch.optim.SGD, dict(lr=0.1, momentum=0.9, nesterov=True, weight_decay=5e-4)),
             (FusedSGD, torch.optim.SGD, dict(lr=0.1, momentum=0.9, dampening=0.1)),
             (FusedSGD, torch.optim.SGD, dict(lr=0.1)),
             (FusedRMSprop, torch.optim.RMSprop, dict(lr=1e-2, momentum=0.9, centered=True, weight_decay=5e-4)),
             (FusedRMSprop, torch.optim.RMSprop, dict(lr=1e-2))]


@pytest.mark.parametrize("fused_cls,torch_cls,kw", CPU_CASES)
def test_cpu_parameters_keep_torch_step_with_scale_and_clip(built, fused_cls, torch_cls, kw):
    """CPU tensors are not what the kernels take: step(grad_scale, max_grad_norm) scales the gradients, clips group 0
    (the model) and then runs torch's own step -- bit for bit what the caller would have written by hand."""
    torch.manual_seed(3)
    w = [torch.randn(40, 7), torch.randn(13)]
    s = [torch.randn(1), torch.randn(1)]
    ps = [torch.nn.Parameter(t.clone()) for t in w + s]
    qs = [torch.nn.Parameter(t.clone()) for t in w + s]
    a = fused_cls([{"params": ps[:2]}, {"params": ps[2:]}], **kw)
    b = torch_cls([{"params": qs[:2]}, {"params": qs[2:]}], **kw)
    for it in range(3):
        grads = [torch.randn_like(t) * 4 for t in w + s]
        for p, q, g in zip(ps, qs, grads):
            p.grad = g.clone(); q.grad = g.clone()
        a.step(grad_scale=0.5, max_grad_norm=1.0)
        with torch.no_grad():
            for q in qs:
                q.grad.mul_(0.5)
        torch.nn.utils.clip_grad_norm_(qs[:2], 1.0)
        b.step()
        for p, q in zip(ps, qs):
            assert torch.equal(p, q), it
    sa, sb = a.state_dict(), b.state_dict()
    assert sa["param_groups"] == sb["param_groups"]
    for i in sb["state"]:
        assert set(sa["state"][i]) == set(sb["state"][i])
        for k, v in sb["state"][i].items():
            assert torch.equal(sa["state"][i][k], v), (i, k)


def _conv_layout_params():
    """Two parameters of one flat buffer, a 4-D conv weight in channels_last strides (the KRSC layout the trunk stores)
    and a bias after a 4-float gap, with gradients in the same positions of a second buffer."""
    Co, Ci, K = 4, 3, 3
    n_w = Co * Ci * K * K
    flat, gflat = torch.zeros(n_w + 4 + 8), torch.zeros(n_w + 4 + 8)

    def conv(buf):
        return buf[:n_w].view(Co, K, K, Ci).permute(0, 3, 1, 2)
    w = torch.nn.Parameter(conv(flat)); b = torch.nn.Parameter(flat[n_w + 4:])
    w.grad = conv(gflat); b.grad = gflat[n_w + 4:]
    assert w.is_contiguous(memory_format=torch.channels_last) and not w.is_contiguous()
    return w, b, n_w


@pytest.mark.parametrize("cls,kw,slots", [
    (FusedSGD, dict(lr=0.1, momentum=0.9), [("momentum_buffer", "buf")]),
    (FusedRMSprop, dict(lr=1e-2, momentum=0.9, centered=True),
     [("square_avg", "sq"), ("momentum_buffer", "buf"), ("grad_avg", "ga")])])
def test_planner_binds_state_views_in_parameter_order(built, cls, kw, slots):
    w, b, n_w = _conv_layout_params()
    opt = cls([w, b], **kw)
    runs = opt._plan(0, [w, b])
    assert len(runs) == 1 and runs[0]["n"] == n_w + 4 + 8
    r = runs[0]
    assert r["step_host"] == 0 and opt._plan(0, [w, b]) is runs
    for k, field in slots:
        sw, sb = opt.state[w][k], opt.state[b][k]
        assert sw.shape == w.shape and sw.stride() == w.stride()          # channels_last, as the parameter
        assert sw.data_ptr() == r[field].data_ptr() and sb.data_ptr() == r[field].data_ptr() + (n_w + 4) * 4
    # a value written through the state view lands where the parameter's own element sits in the flat buffer
    k0, f0 = slots[0]
    with torch.no_grad():
        for k, _ in slots:
            opt.state[w][k].copy_(torch.arange(w.numel(), dtype=torch.float32).view(4, 3, 3, 3) + 1)
            opt.state[b][k].fill_(-2.0)
        flat_w = w.detach().clone()
        flat_w.copy_(opt.state[w][k0])
    assert torch.equal(r[f0][:n_w], flat_w.permute(0, 2, 3, 1).reshape(-1))
    assert float(r[f0][n_w:n_w + 4].abs().sum()) == 0.0                      # the gap stays zero
    if cls is FusedRMSprop:
        opt.state[w]["step"] = opt.state[b]["step"] = torch.tensor(3.0)
    # load_state_dict (torch.load of a checkpoint) replaces the state tensors: re-planned, values carried over
    sd = copy.deepcopy(opt.state_dict())
    opt.load_state_dict(sd)
    assert opt.state[w][k0].data_ptr() != r[f0].data_ptr()
    r2 = opt._plan(0, [w, b])[0]
    assert r2 is not r
    for k, field in slots:
        assert opt.state[w][k].data_ptr() == r2[field].data_ptr() and opt.state[w][k].stride() == w.stride()
        assert torch.equal(opt.state[w][k], torch.arange(w.numel(), dtype=torch.float32).view(4, 3, 3, 3) + 1), k
        assert float(opt.state[b][k].sum()) == -2.0 * b.numel()
    # SGD keeps no step count: a momentum buffer in the loaded state means the first step has been taken
    assert r2["step_host"] == (1 if cls is FusedSGD else 3)
    assert ("step" in opt.state[w]) == (cls is FusedRMSprop)


def test_sgd_without_momentum_has_no_state(built):
    w, b, _ = _conv_layout_params()
    opt = FusedSGD([w, b], lr=0.1)
    runs = opt._plan(0, [w, b])
    assert len(runs) == 1 and "buf" not in runs[0]
    assert len(opt.state) == 0 or all(len(st) == 0 for st in opt.state.values())
    assert opt.state_dict()["state"] == {}
