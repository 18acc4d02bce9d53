"""Host side of inference.evaluate_sequence: the evaluation window table equals the reference's MF.get_indices (run
from its source when the reference tree is present) and leaves np.random where the reference's loop leaves it, the
unique-frame / slot tables rebuild every window, the VO pair tables give the reference's calc_vos_safe /
calc_vos_safe_fc, and bad input fails before any launch.  No GPU needed."""
import ast
import os
import types

import numpy as np
import pytest
import torch

from oracle import ref_loader


def _reference_get_indices():
    """dataset_loaders/composite.py MF.get_indices, executed from the reference's source.  Python 2 under Python 3,
    as oracle/ref_loader.py does for criterion.py: `len(offsets) / 2` and `self.steps/2` are py2 integer divisions
    and `np.int` (removed from numpy) is the platform int64; the text is otherwise verbatim."""
    path = os.path.join(ref_loader.REF_ROOT, "dataset_loaders", "composite.py")
    src = open(path).read()
    tree = ast.parse(src)
    mf = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "MF")
    fn = next(n for n in mf.body if isinstance(n, ast.FunctionDef) and n.name == "get_indices")
    text = "\n".join(src.splitlines()[fn.lineno - 1:fn.end_lineno])
    text = __import__("textwrap").dedent(text)
    for a, b in (("len(offsets) / 2", "len(offsets) // 2"), ("self.steps/2", "self.steps//2"),
                 ("astype(np.int)", "astype(np.int64)")):
        assert a in text
        text = text.replace(a, b)
    ns = {"np": np}
    exec(compile(text, path, "exec"), ns)
    return ns["get_indices"]


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
@pytest.mark.parametrize("variable_skip", [False, True])
@pytest.mark.parametrize("steps,skip", [(3, 10), (5, 2), (4, 3)])
def test_window_table_equals_reference_get_indices(steps, skip, variable_skip):
    from geomapnet_b200.data import ItemLayout
    get_indices = _reference_get_indices()
    L = 40
    me = types.SimpleNamespace(steps=steps, skip=skip, variable_skip=variable_skip, no_duplicates=False,
                               dset=range(L))
    np.random.seed(3)
    ref = np.stack([get_indices(me, i) for i in range(L)])     # eval.py: DataLoader(shuffle=False), item by item
    ref_state = np.random.get_state()
    np.random.seed(3)
    got = ItemLayout(L, steps=steps, skip=skip, variable_skip=variable_skip).eval_tables()["windows"]
    assert np.array_equal(got, ref)
    st = np.random.get_state()
    assert st[2] == ref_state[2] and np.array_equal(st[1], ref_state[1])


@pytest.mark.parametrize("steps,skip,vs", [(None, 1, False), (3, 2, False), (3, 10, True), (5, 3, True)])
def test_unique_and_slot_tables_rebuild_every_window(steps, skip, vs):
    from geomapnet_b200.data import ItemLayout
    lay = ItemLayout(37, steps=steps, skip=skip, variable_skip=vs)
    np.random.seed(5)
    u = lay.eval_tables(unique=True)
    np.random.seed(5)
    d = lay.eval_tables(unique=False)
    assert np.array_equal(u["windows"], d["windows"])
    T = 1 if steps is None else steps
    assert u["windows"].shape == (37, T) and u["windows"].dtype == np.int32
    assert np.array_equal(u["frames"], np.unique(u["windows"]))           # each distinct frame once, in frame order
    assert np.array_equal(u["frames"][u["slots"]], u["windows"])
    assert np.array_equal(d["frames"], d["windows"].reshape(-1))          # window order
    assert np.array_equal(d["slots"], np.arange(37 * T).reshape(37, T))
    assert np.array_equal(d["frames"][d["slots"]], d["windows"])
    for t in (u, d):
        assert all(a.dtype == np.int32 and a.flags.c_contiguous for a in t.values())


def _vos_from_rows(vo_poses, rows):
    """the VOs k_eval_windows computes, per row pair (a, b): calc_vo_logq_safe(vo_poses[a], vo_poses[b]), float64"""
    def qexp(l):
        n = np.linalg.norm(l)
        return np.concatenate([[np.cos(n)], np.sinc(n / np.pi) * l])

    def vo(p0, p1):
        q0, q1 = qexp(p0[3:]), qexp(p1[3:])
        q0i = np.concatenate([[q0[0]], -q0[1:]])
        s = q0i[0] * q1[0] - q0i[1:] @ q1[1:]
        v = q0i[0] * q1[1:] + q1[0] * q0i[1:] + np.cross(q0i[1:], q1[1:])
        q = np.concatenate([[s], v]) / np.linalg.norm(np.concatenate([[s], v]))
        b = np.cross(q0i[1:], p1[:3] - p0[:3])
        t = p1[:3] - p0[:3] + 2 * q0i[0] * b + 2 * np.cross(q0i[1:], b)
        lq = np.zeros(3) if not q[1:].any() else np.arccos(q[0]) * q[1:] / np.linalg.norm(q[1:])   # qlog (:307-317)
        return np.concatenate([t, lq])
    p = vo_poses.astype(np.float64)
    return np.stack([np.stack([vo(p[a], p[b]) for a, b in w]) for w in rows])


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
@pytest.mark.parametrize("vo_fc", [False, True])
def test_vo_rows_give_reference_calc_vos_safe(vo_fc):
    from geomapnet_b200.data import ItemLayout
    pu = ref_loader.load().pose_utils
    rng = np.random.default_rng(2)
    L, T = 30, 4
    v = rng.standard_normal((L, 3))
    v = v / np.linalg.norm(v, axis=1, keepdims=True) * (rng.random((L, 1)) - 0.5) * np.pi
    vo_poses = np.concatenate([rng.standard_normal((L, 3)).cumsum(0), v], 1).astype(np.float32)
    tab = ItemLayout(L, steps=T, skip=3).eval_tables(vo_fc=vo_fc)
    assert tab["vo_rows"].shape == (L, T * (T - 1) // 2 if vo_fc else T - 1, 2)
    f = pu.calc_vos_safe_fc if vo_fc else pu.calc_vos_safe
    ref = f(torch.from_numpy(vo_poses[tab["windows"]])).numpy()          # MF(real=True, include_vos=True)
    got = _vos_from_rows(vo_poses, tab["vo_rows"])
    assert np.abs(got - ref).max() / max(1.0, np.abs(ref).max()) <= 2e-6


def test_bad_input_fails_before_any_launch():
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import DeviceDataset, ItemLayout
    from geomapnet_b200.inference import evaluate_sequence
    lc = _lib.lib().mapnet_launch_count()
    fr = np.zeros((6, 16, 16, 3), np.uint8)
    po = np.zeros((6, 6), np.float32)
    with pytest.raises(ValueError, match="vo_poses"):
        DeviceDataset(fr, [0.5] * 3, [0.2] * 3, poses=po, steps=3, vo_poses=np.zeros((5, 6), np.float32), device="cuda")
    with pytest.raises(ValueError, match="vo_poses"):
        DeviceDataset(fr, [0.5] * 3, [0.2] * 3, poses=po, steps=3, online=True, val_frames=fr, val_poses=po,
                      vo_poses=po, device="cuda")
    with pytest.raises(RuntimeError, match="no CPU path"):
        DeviceDataset(fr, [0.5] * 3, [0.2] * 3, poses=po, steps=3, vo_poses=po, device="cpu")
    with pytest.raises(ValueError, match="ColorJitter"):
        ItemLayout(6, steps=3, color_jitter=0.5).eval_tables()
    with pytest.raises(TypeError, match="DeviceDataset"):
        evaluate_sequence(None, ItemLayout(6, steps=3))

    def stub(**kw):             # the host part of a DeviceDataset, with no cache behind it
        ds = DeviceDataset.__new__(DeviceDataset)
        ItemLayout.__init__(ds, 6, **kw)
        ds.device, ds.h, ds.vo_poses = torch.device("cuda", 0), None, None
        return ds
    with pytest.raises(ValueError, match="ColorJitter"):
        evaluate_sequence(None, stub(steps=3, color_jitter=0.4))
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet, MapNet
    model = MapNet(PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False))    # on the CPU
    ds = stub(steps=3)
    ds.h = object()
    np.random.seed(0)
    state = np.random.get_state()[1].copy()
    with pytest.raises(RuntimeError, match="no CPU path"):
        evaluate_sequence(model, ds)
    assert np.array_equal(np.random.get_state()[1], state)        # no window was drawn
    ds.h = None
    assert _lib.lib().mapnet_launch_count() == lc
