"""Host-side checks of the zero-lag tracker output (no GPU needed): mapnet_track_step_now is declared, exported and
refuses bad arguments before any launch; eval_tables(zero_lag=True) gives the reference's MF.get_indices(i - lag), and
csrc/track_core.h's zero-lag window arithmetic (compiled for the host) gives the same windows and splits every call's
windows into the warm-up ones and those a lagged step completes; Tracker.step and evaluate_sequence(zero_lag=True)
raise their argument errors before the device is touched."""
import ctypes
import os
import re
import subprocess
import tempfile
import types

import numpy as np
import pytest
import torch

from oracle import ref_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests")
MEAN = [0.5, 0.44, 0.45]
STD = [0.21, 0.23, 0.22]
# (steps, skip, L): lag 0, lag < L, lag > L (every window of the sequence is a warm-up window), RobotCar / 7Scenes
CASES = [(2, 1, 9), (3, 2, 30), (4, 5, 12), (5, 3, 7), (7, 3, 40), (7, 10, 25), (7, 150, 60), (16, 2, 50)]


@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


@pytest.fixture(scope="module")
def ht():
    d = tempfile.mkdtemp(prefix="hosttracknow")
    so = os.path.join(d, "libhosttracknow.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(HERE, "_hosttrack_now.cpp")])
    lib = ctypes.CDLL(so)
    ll, i = ctypes.c_longlong, ctypes.c_int
    for name, args in (("htn_lag", [i, i]), ("htn_slot_frame", [ll, i, i, i, ll]), ("htn_first_pending", [ll, ll]),
                       ("htn_now_first", [ll, ll]), ("htn_now_lead", [ll, ll, ll])):
        getattr(lib, name).restype = ll
        getattr(lib, name).argtypes = args
    return lib


def _stub_predictor():
    """an open Predictor as the Localizer sees it, without an engine: any device use would fail on this host"""
    from geomapnet_b200.inference import Predictor
    pr = Predictor.__new__(Predictor)
    pr.max_batch, pr.droprate, pr.seed, pr.precision = 4, 0.0, 0, "bf16"
    pr.device = torch.device("cuda", 0)
    pr._params = pr._bufs = torch.zeros(1)
    pr._calib = None
    pr._engines, pr._graphs = {}, {}
    return pr


def test_step_now_is_declared_exported_and_refuses_bad_arguments_without_a_launch(L):
    from geomapnet_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mapnet_b200.h")).read(), flags=re.S)
    assert re.search(r"\bmapnet_track_step_now\s*\(", hdr)
    assert "mapnet_track_step_now" in _lib.TRACK_API and "mapnet_track_step_now" in _lib.EXPORTED
    assert len(L.mapnet_track_step_now.argtypes) == 7 and L.mapnet_track_step_now.restype == ctypes.c_int
    n0 = L.mapnet_launch_count()
    p = ctypes.c_void_p(16)                     # never dereferenced: every call below fails its checks first
    assert L.mapnet_track_step_now(None, p, p, 1, p, p, None) != 0
    assert b"null handle" in L.mapnet_last_error()
    # a handle needs a device.  The pointer checks come before the handle is read, so a dummy one serves here; B
    # outside [1, max_batch] (whose message reads the handle) is checked on a real handle by the GPU tests.
    fake = ctypes.c_void_p(8)
    for args in ((None, p, 1, p, p), (p, None, 1, p, p), (p, p, 1, None, p), (p, p, 1, p, None)):
        assert L.mapnet_track_step_now(fake, *args, None) != 0
        assert b"null argument" in L.mapnet_last_error(), L.mapnet_last_error()
    assert L.mapnet_launch_count() == n0


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
@pytest.mark.parametrize("steps,skip,n", CASES)
def test_zero_lag_windows_equal_reference_get_indices(steps, skip, n):
    from test_eval_sequence_host import _reference_get_indices
    from geomapnet_b200.data import ItemLayout
    get_indices = _reference_get_indices()
    lag = (steps - 1 - steps // 2) * skip
    me = types.SimpleNamespace(steps=steps, skip=skip, variable_skip=False, no_duplicates=False, dset=range(n))
    ref = np.stack([get_indices(me, i - lag) for i in range(n)])
    tab = ItemLayout(n, steps=steps, skip=skip).eval_tables(zero_lag=True)
    assert np.array_equal(tab["windows"], ref)
    assert np.array_equal(tab["windows"][:, -1], np.arange(n))          # window i ends at frame i
    u = ItemLayout(n, steps=steps, skip=skip).eval_tables(unique=True, zero_lag=True)
    assert np.array_equal(u["frames"][u["slots"]], ref)
    nu = ItemLayout(n, steps=steps, skip=skip).eval_tables(unique=False, zero_lag=True)
    assert np.array_equal(nu["frames"][nu["slots"]], ref)


@pytest.mark.parametrize("steps,skip,n", CASES)
def test_track_core_zero_lag_windows_are_eval_tables_zero_lag(ht, steps, skip, n):
    """every split of a sequence into calls: window w of a call is eval_tables(zero_lag)'s window of frame seen + w,
    and the windows from now_lead on are the ones a lagged step completes, in order"""
    from geomapnet_b200.data import ItemLayout
    for fc in (False, True):
        want = ItemLayout(n, steps=steps, skip=skip).eval_tables(zero_lag=True, vo_fc=fc)
        assert want["vo_rows"].shape[1] == (steps * (steps - 1) // 2 if fc else steps - 1)
    want = want["windows"]
    lag = ht.htn_lag(steps, skip)
    rng = np.random.default_rng(steps * 1000 + skip)
    for trial in range(20):
        seen = 0
        while seen < n:
            b = min(int(rng.integers(1, 2 * lag + 3)), n - seen)
            c0 = ht.htn_now_first(seen, lag)
            assert c0 == seen - lag
            got = [[ht.htn_slot_frame(c0 + w, k, steps, skip, seen + b - 1) for k in range(steps)] for w in range(b)]
            assert got == want[seen:seen + b].tolist(), (seen, b)
            lead = ht.htn_now_lead(seen, b, lag)
            assert lead == sum(1 for w in range(b) if c0 + w < 0)       # the windows whose centre is negative
            a, e = ht.htn_first_pending(seen, lag), ht.htn_first_pending(seen + b, lag)
            assert list(range(c0 + lead, c0 + b)) == list(range(a, e))
            seen += b


def test_step_and_zero_lag_evaluation_argument_errors_before_any_launch(L):
    from geomapnet_b200.data import DeviceDataset, ItemLayout
    from geomapnet_b200.inference import Localizer, Tracker, evaluate_sequence
    pr = _stub_predictor()
    loc = Localizer(pr, MEAN, STD)
    n0 = L.mapnet_launch_count()
    trk = Tracker(loc, 7, skip=10, vo_fc=True)
    f2 = torch.zeros(2, 48, 64, 3, dtype=torch.uint8)
    bad = [
        (f2, torch.zeros(3, 6), "vo_poses must be \\[2, 6\\]"),
        (f2[0], torch.zeros(1, 6), "vo_poses must be \\[6\\]"),
        (f2, torch.zeros(2, 6, dtype=torch.int32), "float"),
        (f2, np.zeros((2, 6), dtype=np.int64), "float"),
        (torch.zeros(2, 48, 64, 3), torch.zeros(2, 6), "uint8"),
        (torch.zeros(0, 48, 64, 3, dtype=torch.uint8), torch.zeros(0, 6), "empty"),
        (torch.zeros(2, 48, 64, 4, dtype=torch.uint8), torch.zeros(2, 6), "RGB"),
    ]
    for frames, vo, msg in bad:
        with pytest.raises(ValueError, match=msg):
            trk.step(frames, vo)
    assert trk.seen == 0 and not trk.h and not trk._now_graphs
    trk.close()
    with pytest.raises(ValueError, match="Tracker is closed"):
        trk.step(f2, torch.zeros(2, 6))
    trk = Tracker(loc, 3)
    pr._params = None                                     # what Predictor.close() leaves
    with pytest.raises(ValueError, match="Predictor is closed"):
        trk.step(f2, torch.zeros(2, 6))
    pr._params = torch.zeros(1)
    loc.close()
    with pytest.raises(ValueError, match="Localizer is closed"):
        trk.step(f2, torch.zeros(2, 6))

    def stub(**kw):             # the host part of a DeviceDataset, with no cache behind it
        ds = DeviceDataset.__new__(DeviceDataset)
        ItemLayout.__init__(ds, 6, **kw)
        ds.device, ds.h, ds.vo_poses = torch.device("cuda", 0), object(), None
        return ds
    np.random.seed(0)
    state = np.random.get_state()[1].copy()
    for kw, msg in ((dict(), "single frames"), (dict(steps=3, skip=2, variable_skip=True), "variable_skip")):
        with pytest.raises(ValueError, match="zero_lag needs a windowed dataset.*" + msg):
            evaluate_sequence(pr, stub(**kw), zero_lag=True)
        with pytest.raises(ValueError, match="fixed skips"):
            ItemLayout(6, **kw).eval_tables(zero_lag=True)
    assert np.array_equal(np.random.get_state()[1], state)        # no window was drawn
    assert L.mapnet_launch_count() == n0


def _quoted(v):
    return ("%.4f" % v).rstrip("0").rstrip(".")


def test_readme_quotes_the_committed_zero_lag_evidence():
    """README quotes profiles/h100_bench_track_now.json, which records the card it was measured on"""
    import json
    with open(os.path.join(ROOT, "profiles", "h100_bench_track_now.json")) as f:
        d = json.loads(f.read())
    assert "H100" in d["card"]["name"] and "W" in d["card"]["nvidia_smi"]
    assert (d["steps"], d["skip"], d["vo_fc"], d["lag"], d["throughput_frames"]) == (7, 10, True, 30, 2000)
    pc, tp = d["per_call_b1"], d["throughput_b64"]
    assert pc["step_and_call_lagged_poses_bitwise"]
    assert tp["step_zero_lag_equals_evaluate_sequence_bitwise"] and tp["step_lagged_equals_call_bitwise"]
    readme = open(os.path.join(ROOT, "README.md")).read()
    for v in (pc["past_lag_ms"]["step"], pc["past_lag_ms"]["call"], pc["past_lag_ms"]["glue"],
              pc["first_lag_frames_ms"]["step"], pc["first_lag_frames_ms"]["call"],
              pc["step_minus_call_first_lag_frames_ms"]):
        assert _quoted(v) in readme, v
    assert "%.2f" % pc["glue_over_step_past_lag"] in readme
    assert "%.2f" % tp["step_over_evaluate_sequence_zero_lag"] in readme
    for k in ("step", "call", "evaluate_sequence_zero_lag"):
        assert "%d %03d" % divmod(round(tp["frames_per_s"][k]), 1000) in readme, k
