"""Host-side checks of inference.MultiTracker and mapnet_track_multi_* (no GPU needed): the entry points are declared,
exported and refuse bad arguments before any launch, every MultiTracker argument error is raised before the device is
touched, the host record builder emits exactly the frames K independent single-stream trackers would emit, in call
order, over random interleavings and chunkings with mid-sequence flushes, and the documents quote the committed
multi-stream evidence."""
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
    for name in _lib.TRACK_MULTI_API:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in _lib.EXPORTED and hasattr(L, name)
    assert "#define MAPNET_TRACK_MAX_STREAMS %d" % _lib.MAX_TRACK_STREAMS in hdr
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
            (2, 3, 1, 4, (ctypes.c_double * 4)(1.0, 0.0, 1.0, 1.0), None, None, b"positive"),
            (2, 3, 1, 4, sig, m3, None, b"go together"), (2, 3, 1, 4, None, None, None, b"null argument")]:
        assert L.mapnet_track_multi_create(ctypes.byref(out), K, T, skip, 0, mb, s, pm, ps) != 0, (K, T, skip, mb)
        assert msg in L.mapnet_last_error(), (msg, L.mapnet_last_error())
        assert b"track_multi_create" in L.mapnet_last_error()
        assert not out.value
    for rc in (L.mapnet_track_multi_step(None, None, None, None, 1, None, None, None),
               L.mapnet_track_multi_flush(None, 0, None, None), L.mapnet_track_multi_reset(None, 0, None),
               L.mapnet_track_multi_status(None, 0, None, None, None)):
        assert rc != 0 and b"null handle" in L.mapnet_last_error()
    assert L.mapnet_track_multi_destroy(None) == 0
    assert L.mapnet_launch_count() == n0


def test_multitracker_argument_errors_before_any_launch(L):
    from geomapnet_b200.inference import Localizer, MultiTracker, Tracker
    pr = _stub_predictor()
    loc = Localizer(pr, MEAN, STD)
    n0 = L.mapnet_launch_count()
    with pytest.raises(TypeError, match="Localizer"):
        MultiTracker(pr, 2, 3)
    for K in (0, -1, 65537, 2.0, True, "2"):
        with pytest.raises(ValueError, match="n_streams"):
            MultiTracker(loc, K, 3)
    for steps in (1, 17):
        with pytest.raises(ValueError, match="steps"):
            MultiTracker(loc, 2, steps)
    mt = MultiTracker(loc, 4, 7, skip=10, vo_fc=True)
    assert isinstance(mt, Tracker) and mt.lag == 30 and mt.n_streams == 4
    assert mt.seen.dtype == np.int64 and mt.seen.tolist() == [0, 0, 0, 0]
    f2, v2 = torch.zeros(2, 48, 64, 3, dtype=torch.uint8), torch.zeros(2, 6)
    bad = [
        (f2, v2, [0, 4], "in \\[0, 4\\)"),                                   # out of range
        (f2, v2, [-1, 0], "in \\[0, 4\\)"),                                  # negative
        (f2, v2, np.array([3, 9]), "in \\[0, 4\\)"),
        (f2, v2, torch.tensor([0, 5]), "in \\[0, 4\\)"),
        (f2, v2, [0.0, 1.0], "integers"),                                    # non-integer
        (f2, v2, [0, 1.5], "integers"),
        (f2, v2, torch.tensor([0.0, 1.0]), "integers"),
        (f2, v2, np.array([True, False]), "integers"),
        (f2, v2, ["0", "1"], "integers"),
        (f2, v2, [0], "one id per frame: 2"),                                # len(streams) != B
        (f2, v2, [0, 1, 2], "one id per frame: 2"),
        (f2, v2, np.zeros((1, 2), dtype=np.int64), "one id per frame: 2"),
        (f2, v2, 1, "one id per frame: 2"),
        (f2, torch.zeros(3, 6), [0, 1], "vo_poses must be \\[2, 6\\]"),     # VO shape mismatch
        (f2, torch.zeros(2, 7), [0, 1], "vo_poses must be \\[2, 6\\]"),
        (f2[0], torch.zeros(1, 6), 0, "vo_poses must be \\[6\\]"),
        (f2, torch.zeros(2, 6, dtype=torch.int32), [0, 1], "float"),
        (torch.zeros(2, 48, 64, 3), v2, [0, 1], "uint8"),
    ]
    for frames, vo, streams, msg in bad:
        for call in (mt, mt.step):
            with pytest.raises(ValueError, match=msg):
                call(frames, vo, streams)
    for s in (-1, 4, 1.0, None, True):
        with pytest.raises(ValueError, match="stream"):
            mt.flush(s)
    for s in (-1, 4, 2.0):
        with pytest.raises(ValueError, match="stream"):
            mt.reset(s)
    mt.reset(2); mt.reset()                               # no handle yet: host counts only
    assert mt.seen.tolist() == [0, 0, 0, 0]
    mt.close()
    for call in (lambda: mt(f2, v2, [0, 1]), lambda: mt.flush(0), mt.reset):
        with pytest.raises(ValueError, match="MultiTracker is closed"):
            call()
    mt = MultiTracker(loc, 2, 3)
    loc.close()
    with pytest.raises(ValueError, match="Localizer is closed"):
        mt(f2, v2, [0, 1])
    mt = MultiTracker(Localizer(pr, MEAN, STD), 2, 3)
    pr._params = None
    for call in (lambda: mt(f2, v2, [0, 1]), lambda: mt.step(f2, v2, [0, 1]), lambda: mt.flush(0)):
        with pytest.raises(ValueError, match="Predictor is closed"):
            call()
    assert L.mapnet_launch_count() == n0


def _single_model(seen, s, lag):
    """the frames a single-stream tracker emits when frame seen[s] of stream s arrives (its _first_pending counters)"""
    from geomapnet_b200.inference import _first_pending
    return list(range(_first_pending(seen[s], lag), _first_pending(seen[s] + 1, lag)))


def _check_records(rec, ids, seen_before, lag):
    """the fields of one chunk's records, from their definition in include/mapnet_b200.h"""
    B = ids.shape[0]
    assert rec.dtype == np.int32 and rec.shape == (B, 6)
    assert rec[:, 0].tolist() == ids.tolist()
    for b in range(B):
        s = ids[b]
        same = np.flatnonzero(ids == s)
        assert rec[b, 1] == np.flatnonzero(same == b)[0] and rec[b, 2] == same.shape[0]
        assert rec[b, 3] == seen_before[s] + rec[b, 1]
    rows = [b for b in range(B) if rec[b, 3] >= lag]
    assert rec[:, 4].tolist() == [rows.index(b) if b in rows else -1 for b in range(B)]
    assert rec[:, 5].tolist() == rows + [-1] * (B - len(rows))


@pytest.mark.parametrize("seed", range(6))
def test_records_emit_what_independent_single_trackers_emit(seed):
    from geomapnet_b200.inference import _first_pending, _stream_chunks
    rng = np.random.default_rng(seed)
    for trial in range(40):
        K = int(rng.integers(1, 9))
        T, skip = int(rng.integers(2, 17)), int(rng.integers(1, 12))
        lag = (T - 1 - T // 2) * skip
        mb = int(rng.integers(1, 17))
        idle = set(rng.choice(K, int(rng.integers(0, K)), replace=False).tolist()) if K > 1 else set()
        live = [s for s in range(K) if s not in idle]
        seen = np.zeros(K, dtype=np.int64)             # the MultiTracker's host counts
        model = [0] * K                                # K single trackers' counts
        emitted = {s: [] for s in range(K)}
        for _ in range(int(rng.integers(1, 25))):
            if rng.random() < 0.15:                    # flush one stream mid-sequence
                s = int(rng.integers(0, K))
                first = _first_pending(int(seen[s]), lag)
                emitted[s] += range(first, int(seen[s]))
                assert emitted[s] == list(range(int(seen[s]))), (seed, trial, s)
                emitted[s] = []
                seen[s] = model[s] = 0
                continue
            n = int(rng.integers(1, 3 * mb + 1))
            ids = rng.choice(live, n).astype(np.int64)
            want = []
            for s in ids:                              # K independent trackers, frames in call order
                want += [(int(s), f) for f in _single_model(model, s, lag)]
                model[s] += 1
            got = []
            for lo, rec, sid, fid in _stream_chunks(seen, ids, lag, mb):
                chunk = ids[lo:lo + mb]
                assert lo % mb == 0 and chunk.shape[0] <= mb
                _check_records(rec, chunk, seen.copy(), lag)
                assert sid.dtype == np.int64 and fid.dtype == np.int64
                got += list(zip(sid.tolist(), fid.tolist()))
            assert got == want, (seed, trial)
            assert seen.tolist() == model
            for s, f in got:
                emitted[s].append(f)
            for s in idle:
                assert seen[s] == 0 and not emitted[s]
        for s in range(K):                             # a final flush: each stream's frames tile 0 .. seen-1 once
            emitted[s] += range(_first_pending(int(seen[s]), lag), int(seen[s]))
            assert emitted[s] == list(range(int(seen[s]))), (seed, trial, s)


def test_a_chunk_that_fails_leaves_the_counts_alone():
    from geomapnet_b200.inference import _stream_chunks
    seen = np.zeros(3, dtype=np.int64)
    ids = np.array([0, 1, 2, 0, 1, 2, 0], dtype=np.int64)
    it = _stream_chunks(seen, ids, 2, 4)
    next(it)
    assert seen.tolist() == [0, 0, 0]                 # advanced only once the chunk has run
    next(it)
    assert seen.tolist() == [2, 1, 1]
    assert list(it) == [] and seen.tolist() == [3, 2, 2]


def _quoted(v):
    return ("%.4f" % v).rstrip("0").rstrip(".")


def test_documents_quote_the_committed_multi_stream_evidence():
    """README / DESIGN quote profiles/h100_bench_track_multi.json, which records the card it was measured on"""
    with open(os.path.join(ROOT, "profiles", "h100_bench_track_multi.json")) as f:
        d = json.loads(f.read())
    assert "H100" in d["card"]["name"] and "W" in d["card"]["nvidia_smi"]
    assert (d["steps"], d["skip"], d["vo_fc"], d["lag"], d["streams"]) == (7, 10, True, 30, [1, 8, 64])
    for k, r in d["per_k"].items():
        assert r["multi_equals_composition_bitwise"], k
        for arm in ("multi_call", "multi_step"):
            assert r["library_launches"][arm] == {"first_call": 45 + 48, "replayed_call": 0}
        assert r["library_launches"]["trackers_call"] == {"first_call": int(k) * 93, "replayed_call": 0}
    readme = open(os.path.join(ROOT, "README.md")).read()
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    p64, p8 = d["per_k"]["64"], d["per_k"]["8"]
    for doc in (readme, design):
        assert "h100_bench_track_multi.json" in doc and "700 W" in doc
        for r in (p64, p8):
            for arm in ("multi_call", "trackers_call"):
                assert _quoted(r["ms_per_tick"][arm]) in doc, arm
            assert "%.2f×" % r["trackers_over_multi"]["call"] in doc
    p1 = d["per_k"]["1"]
    for v in (p1["ms_per_tick"]["multi_call"], p1["ms_per_tick"]["trackers_call"], p64["ms_per_tick"]["multi_step"]):
        assert _quoted(v) in readme, v
    for arm in ("multi_call", "trackers_call"):
        assert "%d %03d" % divmod(round(p64["frames_per_s"][arm]), 1000) in readme or \
            "%d frames/s" % round(p64["frames_per_s"][arm]) in readme, arm
