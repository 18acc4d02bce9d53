"""Host side of the device-resident loader (geomapnet_b200/data/loader.py): the random stream it draws equals the
reference DataLoader's (tests/golden/loader.npz, tools/make_loader_goldens.py), and bad arguments fail before any
launch.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "loader.npz"))


def test_host_stream_equals_reference_dataloader():
    """DataLoader(MF(steps 3, skip 4, variable_skip), batch 5, shuffle=True, num_workers=0) with ColorJitter 0.7 over
    two epochs: the item order, the variable_skip gaps (as frame numbers) and every frame's ColorJitter draw, in the
    order the reference consumes them, and the partial last batch of each epoch."""
    from geomapnet_b200.data import ItemLayout, host_batches
    g = _golden()
    lay = ItemLayout(int(g["stream_L"]), steps=int(g["stream_steps"]), skip=int(g["stream_skip"]), variable_skip=True,
                     color_jitter=float(g["stream_cj"]))
    torch.manual_seed(int(g["stream_torch_seed"]))
    np.random.seed(int(g["stream_np_seed"]))
    frames, jit, sizes = [], [], []
    for _ in range(int(g["stream_epochs"])):
        for fr, j, rows, n in host_batches(lay, int(g["stream_batch"]), shuffle=True):
            frames.append(fr.reshape(n, -1))
            jit.append(j)
            sizes.append(n)
            assert np.array_equal(rows[:, 0], fr) and (rows[:, 1] == -1).all()       # MF targets: the frames' poses
    assert sizes == g["stream_batch_sizes"].tolist()
    assert np.array_equal(np.concatenate(frames), g["stream_frames"])
    rec = np.ascontiguousarray(np.concatenate(jit)).view(np.int32).reshape(-1, 8)
    order = rec[:, :4]
    fac = rec[:, 4:].copy().view(np.float32)
    gj = g["stream_jitter"]
    assert np.array_equal(order, gj[:, :4].astype(np.int32))
    assert np.array_equal(fac, gj[:, 4:].astype(np.float32))


def test_item_layouts_and_target_rows():
    from geomapnet_b200.data import ItemLayout
    from geomapnet_b200.data import tuples
    pn = ItemLayout(7)
    assert len(pn) == 7
    fr, j, rows, n = pn.collate([pn.item(3), pn.item(6)])
    assert fr.tolist() == [3, 6] and j is None and rows.tolist() == [[3, -1], [6, -1]] and n == 2
    on = ItemLayout(30, steps=3, skip=2, online=True, n_val_frames=12)
    assert len(on) == tuples.mfonline_len(12, 3, 2) == 8
    fr, _, rows = on.item(5)
    tr, va = tuples.mfonline_indices(5, 30, 12, 3, 2)
    assert fr.tolist() == tr.tolist() + (va + 30).tolist()
    assert rows.tolist() == [[f, -1] for f in tr] + [[30 + va[0], 30 + va[1]], [30 + va[1], 30 + va[2]]]
    gps = ItemLayout(30, steps=3, skip=2, online=True, n_val_frames=12, gps_mode=True)
    assert gps.item(5)[2].tolist() == [[f, -1] for f in tr] + [[30 + f, -1] for f in va]
    assert (on.frames_per_item, on.targ_per_item, gps.targ_per_item) == (6, 5, 6)
    # example() makes no random draw
    vs = ItemLayout(20, steps=3, skip=4, variable_skip=True, color_jitter=0.5)
    s0, n0 = torch.get_rng_state(), np.random.get_state()[2]
    vs.example(4)
    assert torch.equal(torch.get_rng_state(), s0) and np.random.get_state()[2] == n0
    for bad in (dict(n_frames=5, online=True), dict(n_frames=5, steps=0), dict(n_frames=0)):
        with pytest.raises(ValueError):
            ItemLayout(**bad)
    with pytest.raises(IndexError):
        pn.item(7)


def test_frame_cache_abi_checks_arguments_before_any_launch():
    from geomapnet_b200 import _lib
    L = _lib.lib()
    h = ctypes.c_void_p()
    assert L.mapnet_frame_cache_create(ctypes.byref(h), 0, 480, 640, 256, 8, 8, 8) != 0
    assert b"bad argument" in L.mapnet_last_error()
    assert L.mapnet_frame_cache_create(None, 10, 480, 640, 256, 8, 8, 8) != 0
    lc = L.mapnet_launch_count()
    idx = np.zeros(4, np.int32)
    m = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    assert L.mapnet_frame_cache_ingest(None, None, 0, 1, None) != 0
    assert b"null argument" in L.mapnet_last_error()
    assert L.mapnet_frame_cache_assemble(None, 4, idx.ctypes.data, None, None, 0, None, 0, m, m, None, None, None) != 0
    assert b"null argument" in L.mapnet_last_error()
    assert L.mapnet_frame_cache_destroy(None) == 0
    assert L.mapnet_launch_count() == lc
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MapNetLibError, match="no CUDA device"):
            _lib.check(L.mapnet_frame_cache_create(ctypes.byref(h), 10, 480, 640, 256, 8, 8, 8), "create")


def test_device_dataset_rejects_bad_input_before_touching_the_device():
    from geomapnet_b200.data import DeviceDataset
    f = np.zeros((4, 40, 50, 3), np.uint8)
    p = np.zeros((4, 6), np.float32)
    with pytest.raises(ValueError, match="uint8"):
        DeviceDataset(f.astype(np.float32), [0.5] * 3, [0.2] * 3, poses=p, device="cuda:0")
    with pytest.raises(ValueError, match="poses"):
        DeviceDataset(f, [0.5] * 3, [0.2] * 3, poses=p[:3], device="cuda:0")
    with pytest.raises(RuntimeError, match="no CPU path"):
        DeviceDataset(f, [0.5] * 3, [0.2] * 3, poses=p, device="cpu")
