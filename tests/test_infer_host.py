"""Host-side checks of the eval-mode inference engine (no GPU needed): argument errors arrive before anything is
allocated, the activation arena is what the shapes say, the Predictor refuses the precisions it has no engine for, and
the inference instantiations of the wgmma fprop kernel compile without register spills."""
import ctypes
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


def _arena_from_shapes(B, H, W, elt_z, elt_a, feat_dim=2048):
    """the engine's live set, restated from the ResNet-34 shapes: the stem operand (space-to-depth image), the stem
    conv output, three rotating block tensors (input, h, output; the largest is layer1's) and the downsample output
    (the largest is layer2.0's), plus the head vectors"""
    conv = lambda n, k, s, p: (n + 2 * p - k) // s + 1
    hc, wc = conv(H, 7, 2, 3), conv(W, 7, 2, 3)
    hp, wp = conv(hc, 3, 2, 1), conv(wc, 3, 2, 1)
    wsp = (wc + 6) // 4 * 4
    a0 = (hc + 3) * wsp * 16 * elt_z
    y0 = hc * wc * 64 * elt_a
    act = hp * wp * 64 * elt_z
    h2, w2 = conv(hp, 3, 2, 1), conv(wp, 3, 2, 1)
    ds = h2 * w2 * 128 * elt_a
    head = (512 + 3 * feat_dim) * 4
    return B * (a0 + y0 + 3 * act + ds + head)


def test_arena_bytes_match_the_shapes_and_stay_under_6mb_per_image(L):
    from geomapnet_b200._lib import PREC
    for B in (1, 64):
        got = L.mapnet_infer_arena_bytes(B, 256, 256, PREC["bf16"])
        assert got == _arena_from_shapes(B, 256, 256, 2, 2), got
        assert got / B <= 6e6, got / B
    # strict mode: 4-byte operands (fp16 hi/lo planes) and fp32 conv outputs
    assert L.mapnet_infer_arena_bytes(8, 256, 256, PREC["tc_split"]) == _arena_from_shapes(8, 256, 256, 4, 4)
    # the training trunk's arena at the same shape is several times larger (DESIGN.md section 2: ~20 MB per image)
    print("inference arena at 256x256, bf16: %.2f MB per image" % (L.mapnet_infer_arena_bytes(1, 256, 256, 1) / 1e6))


def test_argument_errors_arrive_before_any_allocation(L):
    from geomapnet_b200._lib import PREC
    for prec in (PREC["fp32"], PREC["bf16_simt"], 7):
        assert L.mapnet_infer_arena_bytes(4, 256, 256, prec) < 0
        assert b"bf16" in L.mapnet_last_error() and b"tc_split" in L.mapnet_last_error()
        h = ctypes.c_void_p()
        # rejected on the argument alone: no device is touched (this test also runs without one)
        assert L.mapnet_infer_create(ctypes.byref(h), 4, 256, 256, 2048, prec) != 0
        assert not h.value
        assert b"precision" in L.mapnet_last_error()
    h = ctypes.c_void_p()
    assert L.mapnet_infer_create(ctypes.byref(h), 0, 256, 256, 2048, PREC["bf16"]) != 0
    assert b"max_B" in L.mapnet_last_error()
    assert L.mapnet_infer_arena_bytes(0, 256, 256, PREC["bf16"]) < 0
    assert L.mapnet_infer_forward(None, None, 1, 0.0, 0, 0, None, None) != 0
    assert L.mapnet_infer_load(None, None, None, None) != 0
    assert L.mapnet_infer_destroy(None) == 0
    # the unit entry point rejects the precisions without an inference epilogue before looking for a device
    assert L.mapnet_test_conv_affine(PREC["fp32"], 1, 8, 8, 64, 64, 3, 1, None, None, None, None, None, 0, None, None) != 0
    assert b"precision" in L.mapnet_last_error()


@pytest.mark.parametrize("precision", ["fp32", "bf16_simt"])
def test_predictor_rejects_precisions_without_an_engine(precision):
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet, MapNet
    from geomapnet_b200.inference import Predictor
    net = PoseNet(torchvision.models.resnet34(weights=None), pretrained=False, precision=precision)
    for model in (net, MapNet(net)):
        with pytest.raises(ValueError, match="'bf16' and 'tc_split'"):
            Predictor(model)


def test_inference_conv_kernels_compile_without_spills(L):
    """ptxas -v of the build: every instantiation of the fprop engine with the inference epilogues
    (k_tc_conv<BN, true>) uses no local memory for spills"""
    logs = glob.glob(os.path.join(ROOT, "geomapnet_b200", "csrc", "_obj", "conv_tc.o.log"))
    assert logs, "build log of conv_tc.cu missing"
    text = open(logs[0]).read()
    found = 0
    for m in re.finditer(r"Compiling entry function '(\w+)'[^\n]*\n(?:[^\n]*\n){0,2}?\s*(\d+) bytes stack frame, "
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", text):
        name = m.group(1)
        if "k_tc_conv" in name and name.endswith("ELb1EEEv14CUtensorMap_stS1_S1_S1_S1_S1_NS_10ConvParamsEPK13__nv_bfloat16PS3_PdNS_6EpiBwdE"):
            found += 1
            assert m.group(3) == "0" and m.group(4) == "0", (name, m.group(0))
    assert found == 2, found        # BN = 64 and 128
