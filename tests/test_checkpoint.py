"""Checkpoint interchange with the reference (SURVEY.md section 8 row f4): the dict written by
common/train.py:198-204 and the prefix logic of common/train.py:22-53, exercised on CPU between the
REFERENCE's own modules (when the reference tree is present) / a torchvision-built stand-in and the
product modules.  No kernels run here: the product modules are parameter containers on CPU."""
import os

import pytest
import torch
import torchvision

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from geomapnet_b200 import build
    return build.build(verbose=False)


def _product(seed=3, pretrained=False):
    from geomapnet_b200.models.posenet import PoseNet
    torch.manual_seed(seed)
    return PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=pretrained)


def _reference_like_state(seed=9):
    """A PoseNet state dict produced by the reference's own class when the tree is present, else by the
    oracle's weight generator, checked against the reference's recorded key order and shapes (same 222 keys)."""
    from oracle import ref_loader, weights
    if ref_loader.available():
        ns = ref_loader.load()
        torch.manual_seed(seed)
        r = ns.PoseNet(torchvision.models.resnet34(weights=None), droprate=0.5, pretrained=False)
        with torch.no_grad():
            for k, v in r.state_dict().items():          # make running stats / counters non-trivial
                if k.endswith("running_mean"):
                    v.normal_()
                elif k.endswith("running_var"):
                    v.uniform_(0.5, 2.0)
                elif k.endswith("num_batches_tracked"):
                    v.fill_(17)
        return {k: v.clone() for k, v in r.state_dict().items()}, "reference class"
    # without the reference tree: the oracle's generator, held to the reference PoseNet's recorded state_dict layout
    import numpy as np
    st = weights.make_state(seed)
    L = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live_reference.npz"))
    layout = {str(k).replace("mapnet.", "", 1): str(sh) for k, sh in zip(L["mapnet_state_keys"], L["mapnet_state_shapes"])}
    assert list(st.keys()) == list(layout.keys())
    for k, v in st.items():
        assert repr(tuple(v.shape)) == layout[k], k
    return st, "oracle weights"


def test_reference_checkpoint_loads_into_posenet_and_mapnet(built, tmp_path):
    from geomapnet_b200.models.posenet import MapNet
    from geomapnet_b200.common.checkpoint import load_checkpoint
    sd, src = _reference_like_state()
    # the file the reference's Trainer writes (common/train.py:198-204); its optimizer entry is torch.optim.Adam's
    f = str(tmp_path / "epoch_005.pth.tar")
    torch.save({"epoch": 5, "model_state_dict": sd, "optim_state_dict": {"state": {}, "param_groups": []},
                "criterion_state_dict": {"sax": torch.Tensor([0.0]), "saq": torch.Tensor([-3.0])}}, f)
    m = _product()
    assert load_checkpoint(f, m) == 0                     # weights only: epoch is not resumed (train.py:167)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), (src, k)
    # PoseNet checkpoint -> MapNet wrapper: model names carry 'mapnet.' (scripts/eval.py:72-88)
    mm = MapNet(_product(seed=4))
    load_checkpoint(f, mm)
    for k, v in mm.state_dict().items():
        assert k.startswith("mapnet.") and torch.equal(v, sd[k[len("mapnet."):]]), k
    # the flat parameter buffer really holds the loaded values (what the kernels read)
    flat, _ = mm.mapnet.flat_parameters()
    w = sd["feature_extractor.layer2.0.downsample.0.weight"]
    p = dict(mm.named_parameters())["mapnet.feature_extractor.layer2.0.downsample.0.weight"]
    off = (p.data_ptr() - flat.data_ptr()) // 4
    assert torch.equal(flat[off:off + w.numel()].view(w.shape), w)


def test_prefixed_and_legacy_state_dicts(built):
    from geomapnet_b200.models.posenet import MapNet
    from geomapnet_b200.common.checkpoint import load_state_dict
    sd, _ = _reference_like_state(seed=10)
    # MapNet / DataParallel checkpoint ('mapnet.' / 'module.' prefixes) -> bare PoseNet (state_prefix branch)
    for prefix in ("mapnet.", "module."):
        m = _product()
        load_state_dict(m, {prefix + k: v for k, v in sd.items()})
        for k, v in m.state_dict().items():
            assert torch.equal(v, sd[k]), (prefix, k)
    # checkpoints written before BatchNorm tracked num_batches_tracked (torch < 0.4.1): zeros are supplied
    legacy = {k: v for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    assert len(legacy) == len(sd) - 36
    mm = MapNet(_product())
    load_state_dict(mm, legacy)
    out = mm.state_dict()
    for k, v in out.items():
        if k.endswith("num_batches_tracked"):
            assert int(v) == 0
        else:
            assert torch.equal(v, sd[k[len("mapnet."):]]), k
    # unrelated first key: the reference raises KeyError (train.py:38-41)
    with pytest.raises(KeyError):
        load_state_dict(_product(), {"encoder.stem.weight": torch.zeros(1)})


def test_product_checkpoint_loads_into_reference_class(built, tmp_path, golden_dir):
    """The other direction: a checkpoint saved from the product modules is a valid reference checkpoint -- it has the
    state_dict layout the reference MapNet's strict load_state_dict checks (the same 222 names, the same shapes) and
    its criterion's keys, as recorded from the reference classes in tests/golden/live_reference.npz."""
    import numpy as np
    from geomapnet_b200.common.checkpoint import save_checkpoint
    from geomapnet_b200.common.criterion import MapNetCriterion
    from geomapnet_b200.models.posenet import MapNet
    L = np.load(os.path.join(golden_dir, "live_reference.npz"))
    m = MapNet(_product(seed=21))
    crit = MapNetCriterion(sax=0.0, saq=-3.0, srx=0.0, srq=-3.0, learn_beta=True, learn_gamma=True)
    opt = torch.optim.Adam(list(m.parameters()) + list(crit.parameters()), lr=1e-4)
    f = save_checkpoint(str(tmp_path), 12, m, opt, crit)
    assert os.path.basename(f) == "epoch_012.pth.tar"
    ck = torch.load(f, map_location="cpu", weights_only=False)
    assert sorted(ck.keys()) == ["criterion_state_dict", "epoch", "model_state_dict", "optim_state_dict"]
    msd = ck["model_state_dict"]
    keys = [str(k) for k in L["mapnet_state_keys"]]
    assert len(keys) == 222 and sorted(msd.keys()) == sorted(keys)
    for k, shape in zip(keys, L["mapnet_state_shapes"]):
        assert repr(tuple(msd[k].shape)) == str(shape), k
        assert torch.equal(msd[k], m.state_dict()[k]), k
    ckeys = [str(k) for k in L["mapnet_criterion_state_keys"]]
    assert sorted(ck["criterion_state_dict"].keys()) == sorted(ckeys)
    assert [float(ck["criterion_state_dict"][k]) for k in ckeys] == [float(p.detach()) for p in crit.parameters()]


def test_resume_restores_optimizer_epoch_and_criterion(built, tmp_path):
    """common/train.py:160-177 with resume_optim: Adam moments / step, epoch, criterion scalars; criterion
    parameters missing from an older checkpoint default to 0.0."""
    from geomapnet_b200.common.checkpoint import save_checkpoint, load_checkpoint
    from geomapnet_b200.common.criterion import PoseNetCriterion, MapNetCriterion
    lin = torch.nn.Linear(4, 3)
    crit = PoseNetCriterion(sax=0.25, saq=-3.0, learn_beta=True)
    opt = torch.optim.Adam(list(lin.parameters()) + list(crit.parameters()), lr=1e-3, weight_decay=5e-4)
    (lin(torch.ones(2, 4)).sum() + sum(p.sum() for p in crit.parameters())).backward()
    opt.step()
    f = save_checkpoint(str(tmp_path), 7, lin, opt, crit)
    lin2 = torch.nn.Linear(4, 3)
    crit2 = MapNetCriterion(sax=9.0, saq=9.0, srx=9.0, srq=9.0, learn_beta=True, learn_gamma=True)
    opt2 = torch.optim.Adam(list(lin2.parameters()) + list(crit2.parameters())[:2], lr=1e-3, weight_decay=5e-4)
    assert load_checkpoint(f, lin2, opt2, crit2, resume_optim=True) == 7
    assert torch.equal(lin2.weight, lin.weight)
    s1, s2 = opt.state_dict()["state"], opt2.state_dict()["state"]
    assert torch.equal(s2[0]["exp_avg"], s1[0]["exp_avg"]) and float(s2[0]["step"]) == 1.0
    got = {k: float(v) for k, v in crit2.state_dict().items()}
    want = {k: float(v) for k, v in crit.state_dict().items()}       # sax, saq after the Adam step above
    assert abs(want["sax"] - 0.25) > 1e-5                            # (the step really moved them)
    assert got == {"sax": want["sax"], "saq": want["saq"], "srx": 0.0, "srq": 0.0}
    with pytest.raises(IOError):
        load_checkpoint(str(tmp_path / "missing.pth.tar"), lin2)
