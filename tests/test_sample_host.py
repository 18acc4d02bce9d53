"""Host-side checks of Monte-Carlo dropout sampling (no GPU needed): Predictor.sample and Localizer.sample refuse every
bad argument before the device is touched, the new C entry points are declared, exported and refuse null handles, and
the split-K plan that mapnet_infer_sample reproduces is the plan launch_small_gemm has always run."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHESS_MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]
CHESS_STD = [float(np.sqrt(v)) for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
NEW = ("mapnet_infer_sample", "mapnet_infer_sample_frames", "mapnet_sample_post", "mapnet_test_small_gemm_plan")


@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


def _stub_predictor(droprate=0.5, calib_hw=None):
    """an open Predictor as sample() sees it, without an engine: any device use would fail on this host"""
    from geomapnet_b200.inference import Predictor
    pr = Predictor.__new__(Predictor)
    pr.max_batch, pr.droprate, pr.seed, pr.precision = 4, droprate, 0, "bf16" if calib_hw is None else "fp8"
    pr.device = torch.device("cuda", 0)
    pr._params = pr._bufs = torch.zeros(1)
    pr._calib = None if calib_hw is None else torch.zeros(1, 3, *calib_hw)
    pr._engines, pr._graphs, pr._sample_graphs = {}, {}, {}
    return pr


def test_new_entry_points_are_declared_exported_and_refuse_null_handles(L):
    import ctypes
    from geomapnet_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mapnet_b200.h")).read(), flags=re.S)
    for name in NEW:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in _lib.EXPORTED and hasattr(L, name)
    n0 = L.mapnet_launch_count()
    assert L.mapnet_infer_sample(None, None, 1, 8, 0.5, 0, 0, None, None, None, None) != 0
    assert b"null handle" in L.mapnet_last_error()
    assert L.mapnet_infer_sample_frames(None, None, None, 1, None, None, 8, 0.5, 0, 0, None, None, None, None) != 0
    assert b"null handle" in L.mapnet_last_error()
    assert L.mapnet_sample_post(None, None, 1, None, None, None, None, None, None, None) != 0
    assert b"bad argument" in L.mapnet_last_error()
    s, k = ctypes.c_int(), ctypes.c_int()
    assert L.mapnet_test_small_gemm_plan(0, 0, 3, 2048, ctypes.byref(s), ctypes.byref(k)) != 0
    assert L.mapnet_launch_count() == n0


def _plan_before_the_refactor(epi, M, N, K, n_sms=132):
    """launch_small_gemm's split-K plan as it was written inline before small_gemm_split_plan: (splits, kchunk)"""
    gx, gy = -(-N // 32), -(-M // 32)
    kchunk, z = K, 1
    if epi == 0 and gx * gy < n_sms // 2 and K >= 256:
        splits = min(n_sms // (gx * gy), K // 64)
        if splits > 1:
            kchunk = ((K + splits - 1) // splits + 63) // 64 * 64
            z = -(-K // kchunk)
    return z, kchunk


def test_split_plan_is_the_plan_launch_small_gemm_ran(L):
    import ctypes
    s, k = ctypes.c_int(), ctypes.c_int()
    cases = [(0, B, 3, 2048) for B in range(1, 513)]                       # the head's feat_dim -> 3 products
    cases += [(0, B, 3, K) for B in (1, 7, 64, 100, 300, 2100) for K in (8, 255, 256, 1000, 4096)]
    cases += [(epi, B, 2048, 512) for epi in (0, 1, 2) for B in (1, 64, 256)]
    for epi, M, N, K in cases:
        assert L.mapnet_test_small_gemm_plan(epi, M, N, K, ctypes.byref(s), ctypes.byref(k)) == 0
        assert (s.value, k.value) == _plan_before_the_refactor(epi, M, N, K), (epi, M, N, K)
    # the plans the GPU tests cross: 32 splits of 64 up to B = 128, 16 of 128 up to B = 256
    for B, want in ((1, (32, 64)), (64, (32, 64)), (128, (32, 64)), (129, (16, 128)), (160, (16, 128)),
                    (256, (16, 128)), (257, (11, 192))):
        assert L.mapnet_test_small_gemm_plan(0, B, 3, 2048, ctypes.byref(s), ctypes.byref(k)) == 0
        assert (s.value, k.value) == want, B


def test_predictor_sample_argument_errors_before_any_launch(L):
    pr = _stub_predictor()
    x = torch.zeros(2, 3, 32, 32)
    n0 = L.mapnet_launch_count()
    for S in (1, 0, -3, 1025, 2.5, True, "8", None):
        with pytest.raises(ValueError, match="S must be an int"):
            pr.sample(x, S)
    with pytest.raises(ValueError, match="no dropout"):
        _stub_predictor(droprate=0.0).sample(x, 8)
    with pytest.raises(RuntimeError, match="no CPU path"):              # the draws are checked first, then the input
        pr.sample(x, 8)
    assert L.mapnet_launch_count() == n0


def test_localizer_sample_argument_errors_before_any_launch(L):
    from geomapnet_b200.inference import Localizer
    pr = _stub_predictor()
    loc = Localizer(pr, CHESS_MEAN, CHESS_STD)
    ok = torch.zeros(2, 48, 64, 3, dtype=torch.uint8)
    n0 = L.mapnet_launch_count()
    for S in (1, 1025, 3.0, False):
        with pytest.raises(ValueError, match="S must be an int"):
            loc.sample(ok, S)
    with pytest.raises(ValueError, match="no dropout"):
        Localizer(_stub_predictor(droprate=0.0), CHESS_MEAN, CHESS_STD).sample(ok, 8)
    bad = [
        (torch.zeros(2, 48, 64, 3, dtype=torch.float32), "uint8"),
        (np.zeros((2, 48, 64, 3), dtype=np.int16), "uint8"),
        (torch.zeros(2, 48, 64, dtype=torch.uint8), "RGB"),
        (torch.zeros(2, 48, 64, 4, dtype=torch.uint8), "RGB"),
        (torch.zeros(1, 1, 2, 48, 64, 3, dtype=torch.uint8), "RGB"),
        (torch.zeros(0, 48, 64, 3, dtype=torch.uint8), "empty"),
    ]
    for frames, msg in bad:
        with pytest.raises(ValueError, match=msg):
            loc.sample(frames, 8)
    off = Localizer(_stub_predictor(calib_hw=(256, 342)), CHESS_MEAN, CHESS_STD)
    with pytest.raises(ValueError, match="calibrated at 256x342, got frames of 256x341"):
        off.sample(np.zeros((480, 640, 3), dtype=np.uint8), 8)
    loc.close()
    with pytest.raises(ValueError, match="Localizer is closed"):
        loc.sample(ok, 8)
    loc = Localizer(pr, CHESS_MEAN, CHESS_STD)
    pr._params = None                            # what Predictor.close() leaves
    with pytest.raises(ValueError, match="Predictor is closed"):
        loc.sample(ok, 8)
    assert L.mapnet_launch_count() == n0


def test_documents_quote_the_committed_sample_evidence():
    """README quotes profiles/h100_bench_sample.json, which records the card it was measured on"""
    import json
    with open(os.path.join(ROOT, "profiles", "h100_bench_sample.json")) as f:
        d = json.loads(f.read())
    assert "H100" in d["card"]["name"] and "W" in d["card"]["nvidia_smi"]
    runs = {(r["B"], r["S"]): r for r in d["runs"]}
    assert set(runs) == {(1, 8), (1, 32), (64, 8), (64, 32)}
    readme = open(os.path.join(ROOT, "README.md")).read()
    for r in runs.values():
        assert r["draws_equal_loop_bitwise"] and r["graph_replays_per_call"] == {"sample": 1, "loop": r["S"]}
        assert r["launches_per_call"]["loop"] == r["S"] * r["launches_per_call"]["forward"]
    r1, r64 = runs[(1, 32)], runs[(64, 32)]
    fmt = lambda v: ("%.4f" % v).rstrip("0").rstrip(".")
    for v in (r1["ms"]["sample"], r1["ms"]["one"], r1["ms"]["loop"], r64["ms"]["sample"]):
        assert fmt(v) in readme, v
    for r in (r1, r64):
        assert "%.3f" % r["sample_over_one"] in readme and "%.2f" % r["loop_over_sample"] in readme
        assert "%.2f" % r["lloop_over_lsample"] in readme
    assert "%d library launches" % r1["launches_per_call"]["sample"] in readme
    assert "makes %d." % r1["launches_per_call"]["forward"] in readme
