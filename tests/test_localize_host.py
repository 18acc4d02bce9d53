"""Host-side checks of inference.Localizer and mapnet_infer_forward_frames (no GPU needed): every argument the Localizer
refuses is refused before the device is touched, the new C entry points are declared, exported and refuse bad handles,
and the engine size a frame maps to is torchvision's Resize(256)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHESS_MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]
CHESS_STD = [float(np.sqrt(v)) for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]


@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


def _stub_predictor(calib_hw=None):
    """an open Predictor as the Localizer sees it, without an engine: any device use would fail on this host"""
    from geomapnet_b200.inference import Predictor
    pr = Predictor.__new__(Predictor)
    pr.max_batch, pr.droprate, pr.seed, pr.precision = 4, 0.0, 0, "bf16" if calib_hw is None else "fp8"
    pr.device = torch.device("cuda", 0)
    pr._params = pr._bufs = torch.zeros(1)
    pr._calib = None if calib_hw is None else torch.zeros(1, 3, *calib_hw)
    pr._engines, pr._graphs = {}, {}
    return pr


def test_new_entry_points_are_declared_exported_and_refuse_null_handles(L):
    from geomapnet_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mapnet_b200.h")).read(), flags=re.S)
    for name in ("mapnet_infer_forward_frames", "mapnet_test_stem_operand"):
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert name in _lib.EXPORTED and hasattr(L, name)
    n0 = L.mapnet_launch_count()
    assert L.mapnet_infer_forward_frames(None, None, None, 1, None, None, 0.0, 0, 0, None, None) != 0
    assert b"null handle" in L.mapnet_last_error()
    assert L.mapnet_test_stem_operand(_lib.PREC["fp32"], None, None, None, 1, None, None, None, None) != 0
    assert b"precision" in L.mapnet_last_error()
    assert L.mapnet_test_stem_operand(_lib.PREC["bf16"], None, None, None, 1, None, None, None, None) != 0
    assert L.mapnet_launch_count() == n0


def test_localizer_wraps_only_a_predictor():
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet, MapNet
    from geomapnet_b200.inference import Localizer
    net = PoseNet(torchvision.models.resnet34(weights=None), pretrained=False, precision="bf16")
    for model in (net, MapNet(net), None):
        with pytest.raises(TypeError, match="Predictor"):
            Localizer(model, CHESS_MEAN, CHESS_STD)


def test_localizer_argument_errors_before_any_launch(L):
    from geomapnet_b200.inference import Localizer
    pr = _stub_predictor()
    with pytest.raises(ValueError, match="pose_m and pose_s"):
        Localizer(pr, CHESS_MEAN, CHESS_STD, pose_m=[0.0, 0.0, 0.0])
    with pytest.raises(ValueError, match="pose_m and pose_s"):
        Localizer(pr, CHESS_MEAN, CHESS_STD, pose_s=[1.0, 1.0, 1.0])
    with pytest.raises(ValueError, match="std must be positive"):
        Localizer(pr, CHESS_MEAN, [0.2, 0.0, 0.2])
    loc = Localizer(pr, CHESS_MEAN, CHESS_STD)
    # mean / std rounded to float32 as ImagePipeline rounds them
    assert loc.mean.dtype == np.float32 and loc.mean.tolist() == np.float32(CHESS_MEAN).tolist()
    assert loc.std.tolist() == np.float32(CHESS_STD).tolist()
    n0 = L.mapnet_launch_count()
    bad = [
        (torch.zeros(2, 48, 64, 3, dtype=torch.float32), "uint8"),
        (np.zeros((2, 48, 64, 3), dtype=np.float32), "uint8"),
        (np.zeros((2, 48, 64, 3), dtype=np.int16), "uint8"),
        (torch.zeros(2, 48, 64, dtype=torch.uint8), "RGB"),           # gray
        (torch.zeros(2, 48, 64, 1, dtype=torch.uint8), "RGB"),
        (torch.zeros(2, 48, 64, 4, dtype=torch.uint8), "RGB"),        # RGBA
        (np.zeros((48, 64, 4), dtype=np.uint8), "RGB"),
        (torch.zeros(1, 1, 2, 48, 64, 3, dtype=torch.uint8), "RGB"),
        (torch.zeros(0, 48, 64, 3, dtype=torch.uint8), "empty"),
        (torch.zeros(2, 0, 64, 3, dtype=torch.uint8), "empty"),
        ([[0, 0, 0]], "uint8"),
    ]
    for frames, msg in bad:
        with pytest.raises(ValueError, match=msg):
            loc(frames)
    loc.close()
    with pytest.raises(ValueError, match="closed"):
        loc(torch.zeros(1, 48, 64, 3, dtype=torch.uint8))
    loc = Localizer(pr, CHESS_MEAN, CHESS_STD)
    pr._params = None                            # what Predictor.close() leaves
    with pytest.raises(ValueError, match="Predictor is closed"):
        loc(torch.zeros(1, 48, 64, 3, dtype=torch.uint8))
    assert L.mapnet_launch_count() == n0


@pytest.mark.parametrize("hw", [(480, 640), (960, 1280), (256, 256), (200, 300), (481, 643), (640, 480)],
                         ids=lambda s: "%dx%d" % s)
def test_engine_size_is_torchvision_resize_256(hw):
    """the (H', W') a frame is fed to the engine at is the size torchvision's Resize(256) gives the PIL image, and an
    fp8 predictor calibrated at any other size refuses the frame before a launch"""
    from PIL import Image
    import torchvision.transforms as T
    from geomapnet_b200.inference import Localizer
    H, W = hw
    want = T.Resize(256)(Image.new("RGB", (W, H))).size[::-1]
    loc = Localizer(_stub_predictor(), CHESS_MEAN, CHESS_STD)
    assert loc._resized(H, W) == want, (hw, loc._resized(H, W), want)
    off = Localizer(_stub_predictor(calib_hw=(want[0], want[1] + 1)), CHESS_MEAN, CHESS_STD)
    with pytest.raises(ValueError, match="calibrated at %dx%d, got frames of %dx%d" % (want[0], want[1] + 1, *want)):
        off(np.zeros((H, W, 3), dtype=np.uint8))


def test_documents_quote_the_committed_localize_evidence():
    """README / DESIGN quote profiles/h100_bench_localize.json, which records the card it was measured on"""
    import json
    with open(os.path.join(ROOT, "profiles", "h100_bench_localize.json")) as f:
        d = json.loads(f.read())
    assert "H100" in d["card"]["name"] and "W" in d["card"]["nvidia_smi"]
    assert d["preprocess_bytes_per_frame"]["chain"] == 4736576 and d["preprocess_bytes_per_frame"]["fused"] == 2641472
    runs = {(r["precision"], r["B"]): r for r in d["runs"]}
    readme = open(os.path.join(ROOT, "README.md")).read()
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    for r in runs.values():
        assert r["launches_per_call"] == {"localizer": 46, "chain": 47} and r["a_equals_b_bitwise"]
    b1, b64 = runs[("bf16", 1)], runs[("bf16", 64)]
    fps = "%d %03d" % divmod(round(b64["frames_per_s"]["a"]), 1000)
    for doc in (readme, design):
        for v in (b1["ms"]["a"], b1["ms"]["b"], b1["ms"]["c_a"], b1["ms"]["c_b"]):
            assert ("%.4f" % v).rstrip("0").rstrip(".") in doc, v
        assert fps in doc and "%.2f" % b1["speedup_a_over_b"] in doc
    assert "%.1f frames/s" % b1["frames_per_s"]["d"] in readme
    for key in (("bf16", 8), ("bf16", 64), ("fp8", 1), ("fp8", 64)):
        for arm in ("a", "b"):
            assert ("%.4f" % runs[key]["ms"][arm]).rstrip("0").rstrip(".") in design, (key, arm)
