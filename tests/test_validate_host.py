"""Host side of inference.validate and graph.train_val: the batch tables of a validation pass equal what the reference's
DataLoader yields over its single-frame / MF validation sets and leave the torch and numpy RNG streams where it leaves
them (tests/golden/validate.npz, tools/make_val_goldens.py); Trainer.train_val's validation-then-training draw order;
argument errors of mapnet_batch_losses and validate before any launch.  No GPU needed."""
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ["posenet_shuffle", "posenet_ordered", "mf_vs_shuffle", "mf_vs_ordered", "mf_shuffle"]


def _golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "validate.npz"))


def _seed(g):
    torch.manual_seed(int(g["seed_torch"]))
    np.random.seed(int(g["seed_np"]))


def _layout(g, name):
    from geomapnet_b200.data import ItemLayout
    L, steps, skip, vs, bs, shuffle = (int(v) for v in g[name + "_case"])
    lay = ItemLayout(L, steps=None if steps < 0 else steps, skip=skip, variable_skip=bool(vs),
                     color_jitter=float(g[name + "_cj"]))
    return lay, bs, bool(shuffle)


@pytest.mark.parametrize("unique", [True, False])
@pytest.mark.parametrize("name", CASES)
def test_val_tables_equal_reference_dataloader(name, unique):
    g = _golden()
    lay, bs, shuffle = _layout(g, name)
    _seed(g)
    tab = lay.val_tables(bs, shuffle, unique)
    ref = g[name + "_frames"].astype(np.int32)            # [I,T]: every item's frames, loader order
    sizes = g[name + "_sizes"]
    assert sizes[-1] < bs                                  # a partial last batch
    assert tab["batch_items"].tolist() == [0] + np.cumsum(sizes).tolist()
    assert [b[3] for b in tab["batches"]] == sizes.tolist()
    assert np.array_equal(tab["targ_rows"], ref)          # single frames / MF: the targets are the frames' poses
    if unique:
        assert np.array_equal(tab["frames"], np.unique(ref))
    else:
        assert np.array_equal(tab["frames"], ref.reshape(-1))
        assert np.array_equal(tab["pred_rows"], np.arange(ref.size).reshape(ref.shape))
    assert np.array_equal(tab["frames"][tab["pred_rows"]], ref)
    for k in ("batch_items", "targ_rows", "frames", "pred_rows"):
        assert tab[k].dtype == np.int32 and tab[k].flags.c_contiguous, k
    # the RNG streams the pass leaves behind: sampler permutation, ColorJitter, variable_skip
    assert np.array_equal(torch.get_rng_state().numpy(), g[name + "_torch_state"])
    st = np.random.get_state()
    assert np.array_equal(st[1], g[name + "_np_mt"]) and st[2] == int(g[name + "_np_pos"])


def test_train_val_draw_order_equals_reference():
    """two epochs of graph.train_val's host draws (every epoch validates: validation pass, then the training epoch)
    against Trainer.train_val over the reference's DataLoaders: each item's frames and each frame's ColorJitter draw"""
    from geomapnet_b200.data import ItemLayout, host_batches
    g = _golden()
    Lv, Lt, steps, skip, bs, epochs = (int(v) for v in g["interleave_case"])
    cj = float(g["interleave_cj"])
    val = ItemLayout(Lv, steps=steps, skip=skip, variable_skip=True, color_jitter=cj)
    train = ItemLayout(Lt, steps=steps, skip=skip, variable_skip=True, color_jitter=cj)
    _seed(g)
    tags, frames, jit = [], [], []
    for _ in range(epochs):
        for tag, batches in ((0, val.val_tables(bs, True, False)["batches"]), (1, list(host_batches(train, bs, True)))):
            for fr, j, _rows, n in batches:
                tags += [tag] * n
                frames.append(fr.reshape(n, steps))
                jit.append(np.ascontiguousarray(j).view(np.int32).reshape(-1, 8))
    assert tags == g["interleave_tags"].tolist()
    assert np.array_equal(np.concatenate(frames), g["interleave_frames"])
    rec, gj = np.concatenate(jit), g["interleave_jitter"]
    assert np.array_equal(gj[:, 0], np.repeat(g["interleave_tags"], steps))
    assert np.array_equal(rec[:, :4], gj[:, 1:5].astype(np.int32))
    assert np.array_equal(rec[:, 4:].copy().view(np.float32), gj[:, 5:].astype(np.float32))


def test_mfonline_has_no_validation_tables():
    from geomapnet_b200.data import ItemLayout
    with pytest.raises(ValueError, match="MFOnline"):
        ItemLayout(30, steps=3, skip=2, online=True, n_val_frames=12).val_tables(4)


def _tables(I=7, T=3, sizes=(3, 3, 1)):
    items = np.cumsum([0] + list(sizes)).astype(np.int32)
    rows = np.arange(I * T, dtype=np.int32)
    return rows, rows.copy(), items


def test_batch_losses_checks_arguments_before_any_launch():
    from geomapnet_b200 import _lib
    L = _lib.lib()
    lc = L.mapnet_launch_count()
    pr, tr, items = _tables()
    buf = torch.zeros(64)           # host memory: every table check comes first
    p = buf.data_ptr()

    def call(mode=1, n_pred=21, n_targ=21, prow=pr, trow=tr, T=3, it=items, nb=3, ptr=p):
        return L.mapnet_batch_losses(mode, ptr, n_pred, ptr, n_targ, prow.ctypes.data, trow.ctypes.data, T,
                                     it.ctypes.data, nb, ptr, ptr, None)

    bad = pr.copy(); bad[5] = 21
    neg = tr.copy(); neg[0] = -1
    cases = [
        (dict(mode=2), b"only posenet"), (dict(mode=3), b"only posenet"), (dict(mode=0), b"posenet mode wants T = 1"),
        (dict(T=0), b"T = 0"), (dict(nb=0), b"bad count"), (dict(n_pred=0), b"bad count"),
        (dict(it=np.array([1, 3, 6, 7], np.int32)), b"batch_items[0]"),
        (dict(it=np.array([0, 3, 3, 7], np.int32)), b"batch 1 is empty"),
        (dict(it=np.array([0, 4, 3, 7], np.int32)), b"batch 1 is empty"),
        (dict(prow=bad), b"row 5"), (dict(trow=neg), b"row 0"), (dict(n_targ=20), b"row 20"),
        (dict(ptr=None), b"null argument"),
        (dict(), b"device memory"),
    ]
    for kw, msg in cases:
        assert call(**kw) != 0, kw
        assert msg in L.mapnet_last_error(), (kw, L.mapnet_last_error())
    assert "mapnet_batch_losses" in _lib.EXPORTED
    assert L.mapnet_launch_count() == lc


def test_validate_rejects_bad_arguments_before_drawing():
    import torchvision
    from geomapnet_b200.common.criterion import MapNetCriterion, MapNetOnlineCriterion, PoseNetCriterion
    from geomapnet_b200.data import DeviceDataset, DeviceLoader, ItemLayout
    from geomapnet_b200.inference import validate
    from geomapnet_b200.models.posenet import PoseNet, MapNet

    def stub(**kw):             # the host part of a DeviceDataset, with no cache behind it
        ds = DeviceDataset.__new__(DeviceDataset)
        ItemLayout.__init__(ds, 9, **kw)
        ds.device, ds.h, ds.vo_poses, ds.max_batch = torch.device("cuda", 0), None, None, 4
        return ds

    model = MapNet(PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False))    # on the CPU
    np.random.seed(0)
    torch.manual_seed(0)
    np_state, t_state = np.random.get_state()[1].copy(), torch.get_rng_state()
    with pytest.raises(TypeError, match="DeviceLoader"):
        validate(model, [], MapNetCriterion())
    with pytest.raises(ValueError, match="MFOnline"):
        validate(model, DeviceLoader(stub(steps=3, skip=2, online=True, n_val_frames=6), 4), MapNetCriterion())
    with pytest.raises(ValueError, match="PoseNetCriterion for single frames"):
        validate(model, DeviceLoader(stub(steps=3, variable_skip=True), 4), PoseNetCriterion())
    with pytest.raises(ValueError, match="MapNetCriterion for MF"):
        validate(model, DeviceLoader(stub(), 4), MapNetCriterion())
    with pytest.raises(ValueError, match="MapNetOnlineCriterion"):
        validate(model, DeviceLoader(stub(steps=3), 4), MapNetOnlineCriterion())
    with pytest.raises(RuntimeError, match="closed"):
        validate(model, DeviceLoader(stub(steps=3), 4), MapNetCriterion())
    ds = stub(steps=3, variable_skip=True, color_jitter=0.5)
    ds.h = object()
    with pytest.raises(RuntimeError, match="no CPU path"):
        validate(model, DeviceLoader(ds, 4), MapNetCriterion())
    ds.h = None
    # nothing was drawn
    assert np.array_equal(np.random.get_state()[1], np_state) and torch.equal(torch.get_rng_state(), t_state)
