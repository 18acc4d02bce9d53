"""Host-side checks of inference.Tracker and mapnet_track_* (no GPU needed): the entry points are declared, exported
and refuse bad arguments before any launch, every Tracker argument error is raised before the device is touched, the
window arithmetic of csrc/track_core.h (compiled for the host) is data/tuples.py's mf_indices and eval_tables' VO
pairs, the un-normalisation rounds as torch's float64 multiply-then-add, and the frames emitted by any sequence of call
sizes tile the sequence once, in order."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests")
MEAN = [0.5, 0.44, 0.45]
STD = [0.21, 0.23, 0.22]


@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


@pytest.fixture(scope="module")
def ht():
    d = tempfile.mkdtemp(prefix="hosttrack")
    so = os.path.join(d, "libhosttrack.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                           os.path.join(HERE, "_hosttrack.cpp")])
    lib = ctypes.CDLL(so)
    ll, i = ctypes.c_longlong, ctypes.c_int
    lib.ht_lag.restype = lib.ht_ring_frames.restype = lib.ht_slot_frame.restype = lib.ht_first_pending.restype = ll
    lib.ht_lag.argtypes = [i, i]
    lib.ht_ring_frames.argtypes = [i, i, i]
    lib.ht_slot_frame.argtypes = [ll, i, i, i, ll]
    lib.ht_first_pending.argtypes = [ll, ll]
    lib.ht_vo_pair.argtypes = [i, i, i, ctypes.POINTER(i), ctypes.POINTER(i)]
    lib.ht_unnormalize.argtypes = [ctypes.c_void_p] * 3 + [ll, ctypes.c_void_p]
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


def test_entry_points_are_declared_exported_and_refuse_bad_arguments_without_a_launch(L):
    from geomapnet_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mapnet_b200.h")).read(), flags=re.S)
    for name in _lib.TRACK_API:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in _lib.EXPORTED and hasattr(L, name)
    n0 = L.mapnet_launch_count()
    out = ctypes.c_void_p()
    sig = (ctypes.c_double * 4)(1.0, 1.0, 1.0, 1.0)
    m3 = (ctypes.c_double * 3)(0.0, 0.0, 0.0)
    for T, skip, mb, s, pm, ps, msg in [
            (1, 1, 4, sig, None, None, b"outside [2, 16]"), (17, 1, 4, sig, None, None, b"outside [2, 16]"),
            (3, 0, 4, sig, None, None, b"must be >= 1"), (3, 1, 0, sig, None, None, b"must be >= 1"),
            (3, 1, 4, (ctypes.c_double * 4)(1.0, 0.0, 1.0, 1.0), None, None, b"positive"),
            (3, 1, 4, sig, m3, None, b"go together"), (3, 1, 4, None, None, None, b"null argument")]:
        assert L.mapnet_track_create(ctypes.byref(out), T, skip, 0, mb, s, pm, ps) != 0, (T, skip, mb)
        assert msg in L.mapnet_last_error(), (msg, L.mapnet_last_error())
        assert not out.value
    for rc in (L.mapnet_track_step(None, None, None, 1, None, None), L.mapnet_track_flush(None, None, None),
               L.mapnet_track_reset(None, None), L.mapnet_track_status(None, None, None, None)):
        assert rc != 0 and b"null handle" in L.mapnet_last_error()
    assert L.mapnet_track_destroy(None) == 0
    assert L.mapnet_launch_count() == n0


def test_tracker_argument_errors_before_any_launch(L):
    from geomapnet_b200.inference import Localizer, Tracker
    pr = _stub_predictor()
    loc = Localizer(pr, MEAN, STD)
    n0 = L.mapnet_launch_count()
    for obj in (pr, None, "loc"):
        with pytest.raises(TypeError, match="Localizer"):
            Tracker(obj, 3)
    for steps in (1, 17, 0, 2.0, True, "3"):
        with pytest.raises(ValueError, match="steps"):
            Tracker(loc, steps)
    for skip in (0, -1, 1.5):
        with pytest.raises(ValueError, match="skip"):
            Tracker(loc, 3, skip=skip)
    with pytest.raises(ValueError, match="positive"):
        Tracker(loc, 3, srx=0.0)
    trk = Tracker(loc, 7, skip=10, vo_fc=True)
    assert trk.lag == 30 and trk.seen == 0
    assert Tracker(loc, 7, skip=150).lag == 450 and Tracker(loc, 2, skip=5).lag == 0 and Tracker(loc, 4, 5).lag == 5
    f2 = torch.zeros(2, 48, 64, 3, dtype=torch.uint8)
    bad = [
        (f2, torch.zeros(3, 6), "vo_poses must be \\[2, 6\\]"),           # count differs
        (f2, torch.zeros(2, 7), "vo_poses must be \\[2, 6\\]"),
        (f2, torch.zeros(12), "vo_poses must be \\[2, 6\\]"),
        (f2[0], torch.zeros(1, 6), "vo_poses must be \\[6\\]"),            # one [H,W,3] frame takes one [6] pose
        (f2, torch.zeros(2, 6, dtype=torch.int32), "float"),
        (f2, np.zeros((2, 6), dtype=np.int64), "float"),
        (f2, [[0.0] * 6] * 2, "float"),
        (f2, torch.zeros(2, 6, dtype=torch.complex64), "float"),
        (torch.zeros(2, 48, 64, 3), torch.zeros(2, 6), "uint8"),
        (torch.zeros(0, 48, 64, 3, dtype=torch.uint8), torch.zeros(0, 6), "empty"),
        (torch.zeros(2, 48, 64, 4, dtype=torch.uint8), torch.zeros(2, 6), "RGB"),
    ]
    for frames, vo, msg in bad:
        with pytest.raises(ValueError, match=msg):
            trk(frames, vo)
    trk.close()
    for call in (lambda: trk(f2, torch.zeros(2, 6)), trk.flush, trk.reset):
        with pytest.raises(ValueError, match="Tracker is closed"):
            call()
    trk = Tracker(loc, 3)
    loc.close()
    with pytest.raises(ValueError, match="Localizer is closed"):
        trk(f2, torch.zeros(2, 6))
    trk = Tracker(Localizer(pr, MEAN, STD), 3)
    pr._params = None                                     # what Predictor.close() leaves
    with pytest.raises(ValueError, match="Predictor is closed"):
        trk(f2, torch.zeros(2, 6))
    with pytest.raises(ValueError, match="Predictor is closed"):
        trk.flush()
    assert L.mapnet_launch_count() == n0


def test_slot_clipping_is_mf_indices(ht):
    from geomapnet_b200.data.tuples import mf_indices, mf_offsets
    rng = np.random.default_rng(0)
    cases = [(T, skip, L) for T in range(2, 17) for skip in (1, 2, 3, 10, 150) for L in (1, 2, 7, 50, 500)]
    for T, skip, L in cases:
        lag = ht.ht_lag(T, skip)
        assert lag == int(mf_offsets(T, skip)[-1]) and lag >= 0, (T, skip)
        assert ht.ht_ring_frames(8, T, skip) == 8 + (T - 1) * skip
        idx = set(rng.integers(0, L, 12).tolist()) | {0, L - 1}
        for i in idx:
            want = mf_indices(i, L, T, skip)
            got = [ht.ht_slot_frame(i, k, T, skip, L - 1) for k in range(T)]
            assert got == want.tolist(), (i, L, T, skip, got, want)
            if i + lag <= L - 1:                          # a window complete before the end needs no end clipping
                assert [ht.ht_slot_frame(i, k, T, skip, i + lag) for k in range(T)] == want.tolist()


@pytest.mark.parametrize("fc", [False, True])
def test_vo_pairs_are_eval_tables_pairs(ht, fc):
    from geomapnet_b200.data.loader import ItemLayout
    i, j = ctypes.c_int(), ctypes.c_int()
    for T in range(2, 17):
        rows = ItemLayout(3 * T, steps=T, skip=1).eval_tables(vo_fc=fc)["vo_rows"][T]     # window of frame T: slots T-T//2 ..
        E = rows.shape[0]
        assert E == (T * (T - 1) // 2 if fc else T - 1)
        got = []
        for e in range(E):
            ht.ht_vo_pair(e, T, int(fc), ctypes.byref(i), ctypes.byref(j))
            got.append((i.value, j.value))
        base = T - T // 2
        assert got == [(int(a) - base, int(b) - base) for a, b in rows], (T, fc)


def test_unnormalize_rounds_as_torch_multiply_then_add(ht):
    rng = np.random.default_rng(3)
    t = rng.standard_normal(3 * 4096) * np.exp(rng.uniform(-20, 20, 3 * 4096))
    s = np.array([1.5, 0.7512345678901234, 3.3e-3])
    m = np.array([0.5, -1.25e3, 2.0e-5])
    out = np.empty_like(t)
    ht.ht_unnormalize(t.ctypes.data, s.ctypes.data, m.ctypes.data, t.size, out.ctypes.data)
    want = (torch.from_numpy(t).view(-1, 3) * torch.from_numpy(s) + torch.from_numpy(m)).reshape(-1).numpy()
    assert np.array_equal(out, want)


def test_emitted_ranges_tile_the_sequence_once_in_order(ht):
    from geomapnet_b200.inference import _first_pending
    rng = np.random.default_rng(1)
    for trial in range(300):
        T, skip = int(rng.integers(2, 17)), int(rng.integers(1, 40))
        lag = ht.ht_lag(T, skip)
        seen, emitted = 0, []
        for _ in range(int(rng.integers(0, 30))):
            n = int(rng.integers(1, 70))
            a, b = _first_pending(seen, lag), _first_pending(seen + n, lag)
            assert (a, b) == (ht.ht_first_pending(seen, lag), ht.ht_first_pending(seen + n, lag))
            assert 0 <= b - a <= n
            emitted += range(a, b)
            seen += n
        emitted += range(_first_pending(seen, lag), seen)  # flush
        assert emitted == list(range(seen)), (T, skip, trial)
        assert seen - _first_pending(seen, lag) == min(lag, seen)


def _quoted(v):
    return ("%.4f" % v).rstrip("0").rstrip(".")


def test_documents_quote_the_committed_track_evidence():
    """README / DESIGN quote profiles/h100_bench_track.json, which records the card it was measured on"""
    import json
    with open(os.path.join(ROOT, "profiles", "h100_bench_track.json")) as f:
        d = json.loads(f.read())
    assert "H100" in d["card"]["name"] and "W" in d["card"]["nvidia_smi"]
    assert (d["steps"], d["skip"], d["vo_fc"], d["lag"]) == (7, 10, True, 30)
    pc, tp = d["per_call_b1"], d["throughput_b64"]
    assert pc["library_launches_per_call"] == {"tracker": 48, "localizer": 46}
    assert tp["tracker_equals_evaluate_sequence_bitwise"]
    readme = open(os.path.join(ROOT, "README.md")).read()
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    for doc in (readme, design):
        for v in (pc["ms"]["tracker"], pc["ms"]["glue"], pc["ms"]["localizer"], d["pgo_T7_one_window_ms"]):
            assert _quoted(v) in doc, v
        assert "%.2f" % pc["glue_over_tracker"] in doc and "%.2f" % tp["tracker_over_evaluate_sequence"] in doc
        for k in ("tracker", "evaluate_sequence"):
            assert "%d %03d" % divmod(round(tp["frames_per_s"][k]), 1000) in doc, k
