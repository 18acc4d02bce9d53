"""GPU run of the device-resident loader (geomapnet_b200/data/loader.py, csrc/preprocess.cu k_loader_assemble):
batches bit-identical to Pillow + torchvision applied on the CPU to the same frames with the same draws, exact
targets, device VO targets against the reference's calc_vos_safe (tests/golden/loader.npz), a graphed epoch with a
ragged last batch against eager steps, and the per-batch-size plan cache under a captured graph."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CJ = 0.7


def _seq(L, H, W, seed):
    rng = np.random.default_rng(seed)
    fr = (rng.random((L, H, W, 3)) * 256).astype(np.uint8)
    fr[1, : H // 3] = 255
    fr[2 % L, :, : W // 4] = 0
    t = rng.standard_normal((L, 3))
    v = rng.standard_normal((L, 3))
    v = v / np.linalg.norm(v, axis=1, keepdims=True) * (rng.random((L, 1)) - 0.5) * math.pi
    return fr, np.concatenate([t, v], 1).astype(np.float32)


def _np_calc_vo_safe(p0, p1):
    """common/pose_utils.py:276-288 restated in float64 (the test tolerance covers the float32 rounding)."""
    def qexp(l):
        n = np.linalg.norm(l)
        return np.concatenate([[np.cos(n)], np.sinc(n / np.pi) * l])

    def qmult(a, b):
        s = a[0] * b[0] - a[1:] @ b[1:]
        v = a[0] * b[1:] + b[0] * a[1:] + np.cross(a[1:], b[1:])
        q = np.concatenate([[s], v])
        return q / np.linalg.norm(q)

    def rot(t, q):
        b = np.cross(q[1:], t)
        return t + 2 * q[0] * b + 2 * np.cross(q[1:], b)

    q0, q1 = qexp(p0[3:].astype(np.float64)), qexp(p1[3:].astype(np.float64))
    q0i = np.concatenate([[q0[0]], -q0[1:]])
    t = rot((p1[:3] - p0[:3]).astype(np.float64), q0i)
    q = qmult(q0i, q1)
    lq = np.zeros(3) if not q[1:].any() else np.arccos(q[0]) * q[1:] / np.linalg.norm(q[1:])
    return np.concatenate([t, lq])


def _reference_batches(kind, seqs, stats, bs, seed, steps=3, skip=2, variable_skip=False, gps=False):
    """The reference's loop on the CPU: DataLoader(dataset, bs, shuffle=True, num_workers=0) over a dataset whose
    __getitem__ follows dataset_loaders/composite.py (posenet: one frame; MF: get_indices then one transform per
    frame; MFOnline: the training tuple, then the validation tuple) with scripts/train.py:119-128's transforms."""
    from PIL import Image
    import torchvision.transforms as T
    from geomapnet_b200.data import tuples
    tf = T.Compose([T.Resize(256), T.ColorJitter(brightness=CJ, contrast=CJ, saturation=CJ, hue=0.5), T.ToTensor(),
                    T.Normalize(mean=stats[0], std=np.sqrt(stats[1]))])
    (fr, po), val = seqs[0], (seqs[1] if len(seqs) > 1 else None)
    L = fr.shape[0]

    def load(f, idx):
        return torch.stack([tf(Image.fromarray(f[i])) for i in idx])

    class DS(torch.utils.data.Dataset):
        def __len__(self):
            if kind == "posenet":
                return L
            if kind == "mf":
                return L
            return tuples.mfonline_len(val[0].shape[0], steps, skip)

        def __getitem__(self, i):
            if kind == "posenet":
                return load(fr, [i])[0], torch.from_numpy(po[i])
            if kind == "mf":
                idx = tuples.mf_indices(i, L, steps, skip, False, variable_skip)
                return load(fr, idx), torch.from_numpy(po[idx])
            tr = tuples.mf_indices(i % L, L, steps, skip, False, variable_skip)
            xi = load(fr, tr)
            Lv = val[0].shape[0]
            va = tuples.mf_indices(i % tuples.mf_len(Lv, steps, skip, True), Lv, steps, skip, True, variable_skip)
            xv = load(val[0], va)
            rp = val[1][va]
            vt = rp if gps else np.stack([_np_calc_vo_safe(rp[k], rp[k + 1]) for k in range(steps - 1)])
            return torch.cat([xi, xv]), torch.cat([torch.from_numpy(po[tr]), torch.from_numpy(vt.astype(np.float32))])

    torch.manual_seed(seed)
    np.random.seed(seed)
    return list(torch.utils.data.DataLoader(DS(), batch_size=bs, shuffle=True, num_workers=0))


@pytest.mark.parametrize("kind,variable_skip,gps", [("posenet", False, False), ("mf", False, False), ("mf", True, False),
                                                    ("online", True, False), ("online", False, True)])
def test_device_batches_bit_equal_pillow_torchvision(kind, variable_skip, gps):
    from geomapnet_b200.data import DeviceDataset, DeviceLoader
    fr, po = _seq(9, 90, 120, 3)
    val = _seq(9, 90, 120, 4) if kind == "online" else None     # 5 tuples: batches 4, 1
    stats = np.array([[0.45, 0.5, 0.55], [0.05, 0.06, 0.04]])
    bs, seed, steps, skip = 4, 11, 3, 2
    seqs = [(fr, po)] + ([val] if val else [])
    ref = _reference_batches(kind, seqs, stats, bs, seed, steps, skip, variable_skip, gps)
    ds = DeviceDataset(fr, stats[0], np.sqrt(stats[1]), poses=po, color_jitter=CJ,
                       steps=None if kind == "posenet" else steps, skip=skip, variable_skip=variable_skip,
                       online=kind == "online", val_frames=val[0] if val else None, val_poses=val[1] if val else None,
                       gps_mode=gps, max_batch=bs, chunk=4)
    torch.manual_seed(seed)
    np.random.seed(seed)
    got = [(x.cpu().numpy(), t.cpu().numpy()) for x, t in DeviceLoader(ds, bs, shuffle=True)]
    assert [g[0].shape[0] for g in got] == [r[0].shape[0] for r in ref] and ref[-1][0].shape[0] < bs     # ragged
    for (gx, gt), (rx, rt) in zip(got, ref):
        rx, rt = rx.numpy(), rt.numpy()
        assert gx.shape == rx.shape and np.array_equal(gx.view(np.uint32), rx.view(np.uint32))
        if kind == "online" and not gps:
            T = steps
            assert np.array_equal(gt[:, :T], rt[:, :T])
            assert np.abs(gt[:, T:] - rt[:, T:]).max() <= 2e-5
        else:
            assert np.array_equal(gt, rt)
    # the same draws again: identical device batches (nothing depends on what ran before)
    torch.manual_seed(seed)
    np.random.seed(seed)
    again = [(x.cpu().numpy(), t.cpu().numpy()) for x, t in DeviceLoader(ds, bs, shuffle=True)]
    assert all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(again, got))
    ds.close()


def test_device_vo_targets_match_reference_calc_vos_safe():
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import DeviceDataset
    g = np.load(os.path.join(ROOT, "tests", "golden", "loader.npz"))
    poses, vos = g["vos_poses"], g["vos_safe"]
    N, T = poses.shape[:2]
    flat = poses.reshape(N * T, 6)
    ds = DeviceDataset(np.zeros((N * T, 32, 32, 3), np.uint8), [0.5] * 3, [0.25] * 3, poses=flat, size=32,
                       max_batch=N * T)
    rows = np.array([[n * T + k, n * T + k + 1] for n in range(N) for k in range(T - 1)], np.int32)
    x = torch.empty(1, 3, 32, 32, device="cuda")
    out = torch.empty(rows.shape[0], 6, device="cuda")
    idx = np.zeros(1, np.int32)
    fp = ctypes.POINTER(ctypes.c_float)
    _lib.check(_lib.lib().mapnet_frame_cache_assemble(
        ds.h, 1, idx.ctypes.data, None, ds.poses.data_ptr(), N * T, rows.ctypes.data, rows.shape[0],
        ds.mean.ctypes.data_as(fp), ds.std.ctypes.data_as(fp), x.data_ptr(), out.data_ptr(), _lib.stream_ptr()),
        "assemble")
    got = out.cpu().numpy().reshape(N, T - 1, 6)
    # float32 on both sides (loader.cu is built without contracted multiply-adds; sinf / cosf still round differently
    # from numpy): the bound is relative to max(|VO|, 1) -- translations here reach ~4, where a float32 ulp is 4.8e-7
    err = np.abs(got - vos).max()
    rel = (np.abs(got - vos) / np.maximum(np.abs(vos), 1.0)).max()
    print("device calc_vos_safe vs reference: max abs err %.2e, max err / max(|vo|, 1) %.2e" % (err, rel))
    assert rel <= 1e-6
    # argument errors: no launch
    lc = _lib.lib().mapnet_launch_count()
    bad = rows.copy()
    bad[3, 1] = N * T
    with pytest.raises(_lib.MapNetLibError, match="target row 3"):
        _lib.check(_lib.lib().mapnet_frame_cache_assemble(
            ds.h, 1, idx.ctypes.data, None, ds.poses.data_ptr(), N * T, bad.ctypes.data, bad.shape[0],
            ds.mean.ctypes.data_as(fp), ds.std.ctypes.data_as(fp), x.data_ptr(), out.data_ptr(), _lib.stream_ptr()), "a")
    oob = np.array([N * T], np.int32)
    with pytest.raises(_lib.MapNetLibError, match="frame_index"):
        _lib.check(_lib.lib().mapnet_frame_cache_assemble(
            ds.h, 1, oob.ctypes.data, None, ds.poses.data_ptr(), N * T, rows.ctypes.data, rows.shape[0],
            ds.mean.ctypes.data_as(fp), ds.std.ctypes.data_as(fp), x.data_ptr(), out.data_ptr(), _lib.stream_ptr()), "a")
    host = torch.empty(1, 3, 32, 32)
    with pytest.raises(_lib.MapNetLibError, match="device memory"):
        _lib.check(_lib.lib().mapnet_frame_cache_assemble(
            ds.h, 1, idx.ctypes.data, None, ds.poses.data_ptr(), N * T, rows.ctypes.data, rows.shape[0],
            ds.mean.ctypes.data_as(fp), ds.std.ctypes.data_as(fp), host.data_ptr(), out.data_ptr(), _lib.stream_ptr()), "a")
    assert _lib.lib().mapnet_launch_count() == lc
    ds.close()


def test_graphed_epoch_with_ragged_batch_matches_eager_steps():
    """Two epochs of MF tuples (11 items, batch 4: sizes 4, 4, 3) through train_epoch against eager steps on the same
    batches, with the tolerances of tests/test_gpu_graph.py (the captures are reused in the second epoch)."""
    from oracle import weights
    from helpers import make_product_model, make_product_criterion
    from geomapnet_b200.common.optimizer import Optimizer
    from geomapnet_b200.data import DeviceDataset, DeviceLoader
    from geomapnet_b200.graph import train_epoch
    fr, po = _seq(11, 48, 64, 5)
    st = weights.make_state(7)
    lr = 1e-5
    finals = []
    for use_graph in (False, False, True):
        model, net = make_product_model(st, "mapnet", "fp32")
        crit = make_product_criterion("mapnet")
        opt = Optimizer([{"params": model.parameters()}, {"params": list(crit.parameters())}], "adam", lr, 5e-4)
        model.train()
        ds = DeviceDataset(fr, [0.4, 0.5, 0.6], [0.2, 0.25, 0.3], poses=po, color_jitter=CJ, steps=3, skip=2,
                           variable_skip=True, size=64, max_batch=4)
        loader = DeviceLoader(ds, 4, shuffle=True)
        torch.manual_seed(3)
        np.random.seed(3)
        losses, steps = [], {}
        for _ in range(2):
            if use_graph:
                losses += train_epoch(loader, model, crit, opt, max_grad_norm=5.0, steps=steps)
            else:
                for x, t in loader:
                    out = model(x)
                    loss = crit(out, t)
                    opt.learner.zero_grad(); loss.backward(); opt.learner.step(max_grad_norm=5.0)
                    losses.append(float(loss.detach()))
        if use_graph:
            assert sorted(steps) == [3, 4]
        torch.cuda.synchronize()
        finals.append((losses, {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}))
        ds.close()
    (la, sa), (l2, s2), (lb, sb) = finals
    assert len(la) == len(lb) == 6
    pkeys = [k for k in sa if sa[k].dtype.is_floating_point and not k.endswith(("running_mean", "running_var"))]

    def mean_dev(u, v, keys):
        return sum(float((u[k] - v[k]).abs().sum()) for k in keys) / sum(u[k].numel() for k in keys)

    moved, noise, dev = mean_dev(sa, st, pkeys), mean_dev(sa, s2, pkeys), mean_dev(sa, sb, pkeys)
    lg = max(abs(a - b) / abs(a) for a, b in zip(la, lb))
    print("graphed epoch vs eager: moved %.3e, eager/eager %.3e, graph/eager %.3e, loss dev %.2e" % (moved, noise, dev, lg))
    assert abs(la[0] - lb[0]) <= 1e-6 * abs(la[0])
    assert moved > 1.5 * lr
    assert dev <= 0.05 * moved, (moved, noise, dev)
    assert lg <= 2e-3, (la, lb)
    for k in sa:
        if not sa[k].dtype.is_floating_point:
            assert torch.equal(sa[k], sb[k]), k


def test_plan_cache_keeps_a_captured_graph_valid_across_batch_sizes():
    """Capture at B = 64, run an eager training forward + backward at B = 50 on the same trunk, replay at B = 64: the
    replay equals one with no call in between (the B = 50 call used to free the captured plans' split-K workspaces)."""
    from oracle import weights
    from helpers import make_product_model, make_product_criterion
    from geomapnet_b200.common.optimizer import Optimizer
    from geomapnet_b200.graph import GraphedTrainStep
    st = weights.make_state(7)
    g = torch.Generator().manual_seed(9)
    xs = [torch.randn(64, 3, 64, 64, generator=g).cuda() for _ in range(2)]
    ts = [torch.cat([torch.randn(64, 3, generator=g), 0.3 * torch.randn(64, 3, generator=g)], 1).cuda() for _ in range(2)]
    x50 = torch.randn(50, 3, 64, 64, generator=g).cuda()
    t50 = torch.cat([torch.randn(50, 3, generator=g), 0.3 * torch.randn(50, 3, generator=g)], 1).cuda()
    res = []
    for between in (True, False):
        model, net = make_product_model(st, "posenet", "bf16")
        crit = make_product_criterion("posenet")
        opt = Optimizer([{"params": model.parameters()}, {"params": list(crit.parameters())}], "adam", 1e-4, 5e-4)
        model.train()
        step = GraphedTrainStep(model, crit, opt, xs[0], ts[0], max_grad_norm=5.0)
        step(xs[0], ts[0])
        if between:
            loss = crit(model(x50), t50)
            loss.backward()
            del loss
        loss = float(step(xs[1], ts[1]))
        torch.cuda.synchronize()
        sd = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()
              if v.dtype.is_floating_point and not k.endswith(("running_mean", "running_var"))}
        res.append((loss, step.out.cpu().clone(), sd))
        del step
    (l1, o1, s1), (l2, o2, s2) = res
    assert l1 == l2
    assert torch.equal(o1, o2)
    for k in s1:
        assert torch.equal(s1[k], s2[k]), k
