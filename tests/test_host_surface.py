"""Host-side logic that needs no GPU: the drop-in surface (state_dict keys, parameter
order, init RNG parity), the C ABI (library loads, exports every symbol the header
declares), loud failure without CUDA, flat-buffer plumbing."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from geomapnet_b200 import build
    return build.build(verbose=False)


def test_cabi_exports_every_declared_symbol(built):
    hdr = open(os.path.join(ROOT, "include", "mapnet_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = sorted(set(re.findall(r"\b(mapnet_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 15
    L = ctypes.CDLL(built)
    for name in declared:
        assert hasattr(L, name), "libmapnet_b200.so does not export %s" % name
    from geomapnet_b200 import _lib
    assert sorted(_lib.EXPORTED) == declared
    assert _lib.lib().mapnet_abi_version() == 2


def test_spec_table_matches_reference_module(built, golden_dir):
    from geomapnet_b200 import _lib
    t = _lib.Trunk(0, 256, 256, 2048, "bf16")
    table, n_params, n_bufs = t.table()
    t.close()
    keys = np.load(os.path.join(golden_dir, "keys.npz"))
    assert [e[0] for e in table] == list(keys["posenet_state_keys"])
    assert sum(int(np.prod(e[2])) for e in table if e[1] == 0) == int(keys["n_params"]) == 22347590
    offs = [(e[3], int(np.prod(e[2]))) for e in table if e[1] == 0]
    for (o1, n1), (o2, _) in zip(offs, offs[1:]):
        assert o2 >= o1 + n1 and o2 % 64 == 0 and o2 - (o1 + n1) < 64      # padded, non-overlapping
    assert n_params >= offs[-1][0] + offs[-1][1]


def _model(pretrained=False, seed=7):
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet
    torch.manual_seed(seed)
    fe = torchvision.models.resnet34(weights=None)
    return PoseNet(fe, droprate=0.0, pretrained=pretrained), fe


def test_state_dict_and_parameter_order(built, golden_dir):
    from geomapnet_b200.models.posenet import MapNet
    m, _ = _model()
    keys = np.load(os.path.join(golden_dir, "keys.npz"))
    assert list(m.state_dict().keys()) == list(keys["posenet_state_keys"])
    assert [n for n, _ in m.named_parameters()] == list(keys["posenet_param_names"])
    assert [repr(tuple(p.shape)) for _, p in m.named_parameters()] == list(keys["posenet_param_shapes"])
    assert list(MapNet(m).state_dict().keys()) == list(keys["mapnet_state_keys"])
    # common/train.py:22-53 prefix logic reads the first names
    assert next(iter(m.state_dict().keys())) == "feature_extractor.conv1.weight"


def test_weights_harvested_and_roundtrip(built):
    m, fe = _model(pretrained=True)
    sd = m.state_dict()
    fsd = fe.state_dict()
    assert torch.equal(sd["feature_extractor.layer3.2.conv1.weight"], fsd["layer3.2.conv1.weight"])
    assert torch.equal(sd["feature_extractor.bn1.running_var"], fsd["bn1.running_var"])
    assert float(sd["fc_xyz.bias"].abs().max()) == 0.0          # posenet.py:62-63
    from oracle import weights
    st = weights.make_state(5)
    m.load_state_dict(st)
    for k, v in m.state_dict().items():
        assert torch.equal(v, st[k]), k
    # parameters are views of one flat buffer (single allreduce / fused Adam)
    flat, _ = m.flat_parameters()
    p = dict(m.named_parameters())["feature_extractor.layer1.0.conv1.weight"]
    assert flat.data_ptr() <= p.data_ptr() < flat.data_ptr() + flat.numel() * 4


def test_init_rng_parity_with_reference(built, golden_dir):
    """After torch.manual_seed(11) the product PoseNet initialises exactly like the reference PoseNet
    (models/posenet.py:50-66), without and with `pretrained`: same keys, and per tensor the same sum and the same
    values at a fixed stride, as recorded from the reference class in tests/golden/live_reference.npz."""
    L = np.load(os.path.join(golden_dir, "live_reference.npz"))
    for pretrained in (False, True):
        tag = "init_pre%d_" % int(pretrained)
        m, _ = _model(pretrained=pretrained, seed=11)
        sd = m.state_dict()
        keys = [str(k) for k in L[tag + "keys"]]
        assert list(sd.keys()) == keys, pretrained
        for i, k in enumerate(keys):
            v = sd[k].detach().cpu()
            ref_sum = float(L[tag + "sum"][i])
            assert abs(float(v.double().sum()) - ref_sum) <= 1e-12 * max(1.0, abs(ref_sum)), (pretrained, k)
            sample = v.flatten()[::int(L[tag + "stride"][i])].numpy()
            assert np.array_equal(sample, L[tag + "%d" % i]), (pretrained, k)


def test_no_cpu_fallback(built):
    from geomapnet_b200.common.criterion import PoseNetCriterion, MapNetCriterion
    from geomapnet_b200 import _lib
    m, _ = _model()
    with pytest.raises(RuntimeError):
        m(torch.zeros(2, 3, 64, 64))
    with pytest.raises(RuntimeError):
        PoseNetCriterion()(torch.zeros(2, 6), torch.zeros(2, 6))
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MapNetLibError):
            _lib.Trunk(4, 64, 64, 2048, "bf16")        # a real handle needs a device
    with pytest.raises(NotImplementedError):
        MapNetCriterion(t_loss_fn=torch.nn.MSELoss())


def test_rejects_non_resnet34(built):
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet
    with pytest.raises(NotImplementedError):
        PoseNet(torchvision.models.resnet18(weights=None), pretrained=False)
    with pytest.raises(NotImplementedError):
        PoseNet(torchvision.models.resnet50(weights=None), pretrained=False)


def test_criterion_surface(built):
    from geomapnet_b200.common.criterion import PoseNetCriterion, MapNetCriterion, MapNetOnlineCriterion
    c = MapNetOnlineCriterion(sax=0.0, saq=-3.0, srx=0.0, srq=-3.0, learn_beta=True, learn_gamma=False, gps_mode=True)
    names = [n for n, _ in c.named_parameters()]
    assert names == ["sax", "saq", "srx", "srq"]
    assert c.sax.requires_grad and not c.srx.requires_grad and c.gps_mode
    assert [n for n, _ in PoseNetCriterion().named_parameters()] == ["sax", "saq"]
    assert list(MapNetCriterion().state_dict().keys()) == ["sax", "saq", "srx", "srq"]


def test_optimizer_wrapper_surface(built):
    from geomapnet_b200.common.optimizer import Optimizer, FusedAdam
    p = [torch.nn.Parameter(torch.zeros(3))]
    o = Optimizer(params=p, method="adam", base_lr=1e-4, weight_decay=5e-4)
    assert isinstance(o.learner, FusedAdam) and o.adjust_lr(10) == 1e-4
    s = Optimizer(params=p, method="sgd", base_lr=0.1, weight_decay=0.0, lr_decay=0.1, lr_stepvalues=[60, 80], momentum=0.9)
    assert abs(s.adjust_lr(70) - 0.01) < 1e-12 and abs(s.learner.param_groups[0]["lr"] - 0.01) < 1e-12
    p[0].grad = torch.zeros(3)
    with pytest.raises(RuntimeError):
        o.learner.step()             # CPU tensors: no CPU path


def test_fused_adam_plan_is_keyed_on_run_structure(built):
    """FusedAdam._plan (host logic, no kernels): the run structure and the moment buffers must survive a change of
    the ABSOLUTE gradient addresses of free-standing parameters (autograd hands the criterion scalars a fresh .grad
    every step) -- a rebuild during CUDA-graph capture would be replayed with the step and reset their Adam state --
    and must be rebuilt, keeping the moments, when load_state_dict replaces the state tensors."""
    from geomapnet_b200.common.optimizer import FusedAdam
    flat = torch.zeros(64 + 64 + 8)
    gflat = torch.zeros_like(flat)
    a = torch.nn.Parameter(flat[0:60].view(6, 10)); b = torch.nn.Parameter(flat[64:72])     # 4-float gap: one run
    s1 = torch.nn.Parameter(torch.zeros(1)); s2 = torch.nn.Parameter(torch.zeros(1))
    a.grad = gflat[0:60].view(6, 10); b.grad = gflat[64:72]
    s1.grad = torch.ones(1); s2.grad = torch.ones(1)
    opt = FusedAdam([{"params": [a, b]}, {"params": [s1, s2]}], lr=1e-3)
    r0 = opt._plan(0, [a, b]); r1 = opt._plan(1, [s1, s2])
    assert len(r0) == 1 and r0[0]["n"] == 72 and [p is q for p, q in zip(r0[0]["params"], (a, b))] == [True, True]
    assert len(r1) == 2 and all(r["n"] == 1 for r in r1)
    m_ptrs = [r["m"].data_ptr() for r in r1]
    opt.state[s1]["exp_avg"].fill_(0.25)                       # pretend a step happened
    keep = [s1.grad, s2.grad]                                   # keep the old tensors alive: new addresses guaranteed
    s1.grad = torch.full((1,), 2.0); s2.grad = torch.full((1,), 3.0)
    assert s1.grad.data_ptr() != keep[0].data_ptr()
    r1b = opt._plan(1, [s1, s2])
    assert r1b is r1 and [r["m"].data_ptr() for r in r1b] == m_ptrs
    assert opt._plan(0, [a, b]) is r0
    # a different gradient LAYOUT of a multi-parameter run does change the structure (b's grad no longer follows a's)
    b.grad = torch.zeros(8)
    r0b = opt._plan(0, [a, b])
    assert r0b is not r0 and len(r0b) == 2
    # load_state_dict replaces the state tensors: rebuilt, moments carried over
    import copy
    sd = copy.deepcopy(opt.state_dict())                        # what torch.load of a checkpoint hands over
    opt.load_state_dict(sd)
    assert opt.state[s1]["exp_avg"].data_ptr() not in m_ptrs
    r1c = opt._plan(1, [s1, s2])
    assert r1c is not r1
    assert float(opt.state[s1]["exp_avg"]) == 0.25
    assert opt.state[s1]["exp_avg"].data_ptr() in [r["m"].data_ptr() for r in r1c]
