"""Host-side checks of inference.SampledMultiTracker and mapnet_track_multi_sample_* (no GPU needed): the entry points
are declared, exported and refuse bad arguments before any launch, every SampledMultiTracker argument error is raised
before the device is touched, and the documents quote the committed multi-stream Monte-Carlo evidence."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

from test_track_host import _stub_predictor      # an open Predictor without an engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MEAN = [0.5, 0.44, 0.45]
STD = [0.21, 0.23, 0.22]


@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


def test_entry_points_are_declared_exported_and_refuse_bad_arguments_without_a_launch(L):
    from geomapnet_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mapnet_b200.h")).read(), flags=re.S)
    for name in _lib.TRACK_MULTI_SAMPLE_API:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in _lib.EXPORTED and hasattr(L, name)
    n0 = L.mapnet_launch_count()
    out = ctypes.c_void_p()
    sig = (ctypes.c_double * 4)(1.0, 1.0, 1.0, 1.0)
    m3 = (ctypes.c_double * 3)(0.0, 0.0, 0.0)
    for K, T, skip, mb, s, pm, ps, msg in [
            (0, 3, 1, 4, sig, None, None, b"streams outside [1, 65536]"),
            (65537, 3, 1, 4, sig, None, None, b"streams outside [1, 65536]"),
            (-1, 3, 1, 4, sig, None, None, b"streams outside"),
            (2, 1, 1, 4, sig, None, None, b"outside [2, 16]"), (2, 17, 1, 4, sig, None, None, b"outside [2, 16]"),
            (2, 3, 0, 4, sig, None, None, b"must be >= 1"), (2, 3, 1, 0, sig, None, None, b"must be >= 1"),
            (2, 3, 1, -3, sig, None, None, b"must be >= 1"),
            (2, 3, 1, 4, (ctypes.c_double * 4)(0.0, 1.0, 1.0, 1.0), None, None, b"positive"),
            (2, 3, 1, 4, (ctypes.c_double * 4)(1.0, -1.0, 1.0, 1.0), None, None, b"positive"),
            (2, 3, 1, 4, (ctypes.c_double * 4)(1.0, 1.0, 1.0, 0.0), None, None, b"positive"),
            (2, 3, 1, 4, sig, m3, None, b"go together"), (2, 3, 1, 4, sig, None, m3, b"go together"),
            (2, 3, 1, 4, None, None, None, b"null argument")]:
        assert L.mapnet_track_multi_sample_create(ctypes.byref(out), K, T, skip, 0, mb, s, pm, ps) != 0, (K, T, mb)
        assert msg in L.mapnet_last_error(), (msg, L.mapnet_last_error())
        assert b"track_multi_sample_create" in L.mapnet_last_error()
        assert not out.value
    assert L.mapnet_track_multi_sample_create(None, 2, 3, 1, 0, 4, sig, None, None) != 0
    assert b"null argument" in L.mapnet_last_error()
    p = ctypes.c_void_p(16)
    for rc in (L.mapnet_track_multi_sample_step(None, p, p, p, p, 1, p, None, None),
               L.mapnet_track_multi_sample_flush(None, 0, p, None), L.mapnet_track_multi_sample_reset(None, 0, None),
               L.mapnet_track_multi_sample_status(None, 0, None, None, None)):
        assert rc != 0 and b"null handle" in L.mapnet_last_error()
    assert L.mapnet_track_multi_sample_destroy(None) == 0
    assert L.mapnet_launch_count() == n0


def test_sampled_multitracker_argument_errors_before_any_launch(L):
    from geomapnet_b200.inference import Localizer, MultiTracker, SampledMultiTracker
    pr = _stub_predictor()
    loc = Localizer(pr, MEAN, STD)
    n0 = L.mapnet_launch_count()
    with pytest.raises(ValueError, match="no dropout"):
        SampledMultiTracker(loc, 8, 2, 3)                 # droprate 0
    pr.droprate = 0.5
    for obj in (pr, None):
        with pytest.raises(TypeError, match="Localizer"):
            SampledMultiTracker(obj, 8, 2, 3)
    for S in (1, 0, 1025, 2.0, True, "8"):
        with pytest.raises(ValueError, match="S must be"):
            SampledMultiTracker(loc, S, 2, 3)
    for K in (0, -1, 65537, 2.0, True, "2"):
        with pytest.raises(ValueError, match="n_streams"):
            SampledMultiTracker(loc, 8, K, 3)
    for steps in (1, 17):
        with pytest.raises(ValueError, match="steps"):
            SampledMultiTracker(loc, 8, 2, steps)
    for k in ("sax", "saq", "srx", "srq"):
        with pytest.raises(ValueError, match="positive"):
            SampledMultiTracker(loc, 8, 2, 3, **{k: 0.0})
    smt = SampledMultiTracker(loc, 8, 4, 7, skip=10, vo_fc=True, sax=1e-4, saq=1e-4, srx=20, srq=20)
    assert isinstance(smt, MultiTracker) and smt.lag == 30 and smt.n_streams == 4 and smt.S == 8
    assert smt.seen.dtype == np.int64 and smt.seen.tolist() == [0, 0, 0, 0]
    f2, v2 = torch.zeros(2, 48, 64, 3, dtype=torch.uint8), torch.zeros(2, 6)
    bad = [
        (f2, v2, [0, 4], "in \\[0, 4\\)"),                                   # out of range
        (f2, v2, [-1, 0], "in \\[0, 4\\)"),
        (f2, v2, np.array([3, 9]), "in \\[0, 4\\)"),
        (f2, v2, [0.0, 1.0], "integers"),                                    # a float dtype
        (f2, v2, np.array([0.0, 1.0], dtype=np.float32), "integers"),
        (f2, v2, torch.tensor([0.0, 1.0]), "integers"),
        (f2, v2, [0], "one id per frame: 2"),                                # wrong count
        (f2, v2, [0, 1, 2], "one id per frame: 2"),
        (f2, v2, 1, "one id per frame: 2"),
        (f2, torch.zeros(3, 6), [0, 1], "vo_poses must be \\[2, 6\\]"),     # VO shape mismatch
        (f2, torch.zeros(2, 7), [0, 1], "vo_poses must be \\[2, 6\\]"),
        (f2[0], torch.zeros(1, 6), 0, "vo_poses must be \\[6\\]"),
        (f2, torch.zeros(2, 6, dtype=torch.int32), [0, 1], "float"),
        (torch.zeros(2, 48, 64, 3), v2, [0, 1], "uint8"),
    ]
    bad.append((f2, v2, torch.tensor([0, 1], device="meta"), "CPU integer tensor"))          # a device tensor
    if torch.cuda.is_available():
        bad.append((f2, v2, torch.tensor([0, 1], device="cuda"), "CPU integer tensor"))     # a CUDA tensor
    for frames, vo, streams, msg in bad:
        for call in (smt, smt.step):
            with pytest.raises(ValueError, match=msg):
                call(frames, vo, streams)
    for s in (-1, 4, 1.0, None, True):
        with pytest.raises(ValueError, match="stream"):
            smt.flush(s)
    for s in (-1, 4, 2.0):
        with pytest.raises(ValueError, match="stream"):
            smt.reset(s)
    smt.reset(2); smt.reset()                             # no handle yet: host counts only
    assert smt.seen.tolist() == [0, 0, 0, 0]
    smt.close()
    for call in (lambda: smt(f2, v2, [0, 1]), lambda: smt.flush(0), smt.reset):
        with pytest.raises(ValueError, match="SampledMultiTracker is closed"):
            call()
    smt = SampledMultiTracker(loc, 8, 2, 3)
    pr._params = None
    for call in (lambda: smt(f2, v2, [0, 1]), lambda: smt.step(f2, v2, [0, 1]), lambda: smt.flush(0)):
        with pytest.raises(ValueError, match="Predictor is closed"):
            call()
    assert L.mapnet_launch_count() == n0


def _quoted(v):
    return ("%.4f" % v).rstrip("0").rstrip(".")


def test_documents_quote_the_committed_multi_stream_sampled_evidence():
    """README / DESIGN / INTEGRATION quote profiles/h100_bench_track_multi_sample.json, which records the card it was
    measured on and that the timed estimates were bitwise the per-stream composition"""
    with open(os.path.join(ROOT, "profiles", "h100_bench_track_multi_sample.json")) as f:
        d = json.loads(f.read())
    assert "H100" in d["card"]["name"] and "W" in d["card"]["nvidia_smi"]
    assert (d["steps"], d["skip"], d["vo_fc"], d["lag"], d["streams"], d["S"], d["droprate"]) == \
        (7, 10, True, 30, [1, 8, 64], 32, 0.5)
    assert d["sigmas"] == {"sax": 1e-4, "saq": 1e-4, "srx": 20.0, "srq": 20.0}
    for k, r in d["per_k"].items():
        assert r["multi_equals_composition_bitwise"], k
        for arm in ("multi_call", "multi_step", "trackers_call"):
            assert r["library_launches"][arm]["replayed_call"] == 0, (k, arm)
    readme = open(os.path.join(ROOT, "README.md")).read()
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    integration = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    p64, p8, p1 = d["per_k"]["64"], d["per_k"]["8"], d["per_k"]["1"]
    for doc in (readme, design):
        assert "h100_bench_track_multi_sample.json" in doc and "700 W" in doc
        for r in (p64, p8):
            for arm in ("multi_call", "trackers_call"):
                assert _quoted(r["ms_per_tick"][arm]) in doc, arm
            assert "%.2f×" % r["trackers_over_multi"] in doc
    for v in (p1["ms_per_tick"]["multi_call"], p1["ms_per_tick"]["trackers_call"], p64["ms_per_tick"]["multi_step"]):
        assert _quoted(v) in readme, v
    assert "SampledMultiTracker" in integration and "h100_bench_track_multi_sample.json" in integration
