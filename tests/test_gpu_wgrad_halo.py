"""The stride-1 3x3 wgrad halo engine (k_halo_wgrad) against the per-tap engine (k_tc_wgrad), on the GPU.

Both engines keep the same K partition (pixel box, splits, pixel tiles per split) and feed every dW element the same
wgmma k16 steps in the same order, so each halo variant -- 3 filter taps per CTA at N tile 64 or 128, 9 taps at 64 --
must give the per-tap engine's dW bit for bit.  The shapes are every stride-1 3x3 conv of ResNet-34 at B = 64 (the
benchmark) and at a ragged B = 5, which covers one split (layer4: the kernel adds into dW) and many splits (the
reduction pass adds into dW).  dW holds a nonzero gradient before each launch, so the add-into-the-gradient path is
the one checked.  The planner's choice is also checked per element against float64 at the bound
tests/test_gpu_conv_plans.py derives: 2^-23 of the running sum per wgmma instruction (4 per pixel tile), 2^-24 per
split add and 2^-24 for the add onto the prior gradient."""
import ctypes
import json

import pytest
import torch
import torch.nn.functional as F

from geomapnet_b200 import _lib

SHAPES = [("layer1", 64, 64), ("layer2", 32, 128), ("layer3", 16, 256), ("layer4", 8, 512)]
VARIANTS = [(3, 64), (3, 128), (9, 64)]


def describe(B, H, C):
    buf = ctypes.create_string_buffer(1 << 17)
    _lib.check(_lib.lib().mapnet_test_plan_describe(2, B, H, H, C, C, 3, 1, 0, buf, len(buf)), "mapnet_test_plan_describe")
    return json.loads(buf.value.decode())["wgrad"]


def run(taps, bn, x, dy, dw0):
    B, H, W, C = x.shape
    dw = dw0.clone()
    _lib.check(_lib.lib().mapnet_test_wgrad(taps, bn, B, H, W, C, dy.shape[3], 3, 1, x.data_ptr(), dy.data_ptr(),
                                            dw.data_ptr(), 0, None), "mapnet_test_wgrad")
    return dw


def operands(B, H, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, H, C, generator=g, device="cuda").bfloat16()
    dy = torch.randn(B, H, H, C, generator=g, device="cuda").bfloat16()
    dw0 = torch.randn(C, 9, C, generator=g, device="cuda")
    return x, dy, dw0


@pytest.mark.gpu
@pytest.mark.parametrize("B", [64, 5])
@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_halo_variants_equal_the_per_tap_engine_bit_for_bit(shape, B):
    name, H, C = shape
    x, dy, dw0 = operands(B, H, C, 11)
    ref = run(0, 0, x, dy, dw0)
    P = describe(B, H, C)
    ran = 0
    for taps, bn in VARIANTS:
        if C % bn != 0:
            continue
        got = run(taps, bn, x, dy, dw0)
        diff = int((got != ref).sum())
        assert diff == 0, "%s B=%d: %d-tap BN %d differs from the per-tap engine in %d of %d elements (splits %d)" % (
            name, B, taps, bn, diff, got.numel(), P["splits"])
        ran += 1
    assert ran == (2 if C == 64 else 3)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [64, 5])
@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_planned_wgrad_per_element_against_float64(shape, B):
    name, H, C = shape
    x, dy, dw0 = operands(B, H, C, 12)
    got = run(-1, 0, x, dy, dw0).double() - dw0.double()
    P = describe(B, H, C)
    xd = x.permute(0, 3, 1, 2).double()
    dyd = dy.permute(0, 3, 1, 2).double()

    def wgrad(a, b):
        ww = torch.zeros(C, C, 3, 3, dtype=torch.float64, device="cuda", requires_grad=True)
        return torch.autograd.grad(F.conv2d(a, ww, None, 1, 1), ww, b)[0].permute(0, 2, 3, 1).reshape(C, 9, C)

    ref, S = wgrad(xd, dyd), wgrad(xd.abs(), dyd.abs())
    gamma = 4 * P["tiles_per_split"] * 2.0 ** -23 + P["splits"] * 2.0 ** -24
    bound = 2.0 ** -24 * (dw0.double().abs() + S) + (1 + 2.0 ** -24) * gamma * S + 1e-30
    err = (got - ref).abs()
    assert bool((err <= bound).all()), "%s B=%d (%s): %d elements outside the bound, max err/bound %.3g" % (
        name, B, P["engine"], int((err > bound).sum()), float((err / bound).max()))
    print("wgrad-halo %s B=%d engine %s: max err/bound %.3g" % (name, B, P["engine"], float((err / bound).max())))
