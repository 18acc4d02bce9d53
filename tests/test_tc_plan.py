"""Host logic of the tensor-core conv engines, checked WITHOUT a GPU.

`tc_plan_create` (geomapnet_b200/csrc/conv_tc.cu) turns a convolution into tiles, output-parity classes and filter
taps (spatial offset, activation view, K index of the weight slice).  That arithmetic is pure host code; the kernels
only walk it.  Here the plan is exported as JSON
(`mapnet_test_plan_describe`) and REPLAYED on the CPU in float64 exactly as the kernels consume it -- TMA semantics:
out-of-bounds rows read as zero, stride-2 convs read parity views -- and compared with torch's conv2d and its autograd
(the third-party arithmetic the reference calls, reference models/posenet.py:66).  Shapes are fuzzed: odd
sizes, both strides, 1x1 and 3x3, the downsample shortcut folded into the stride-2 dgrad."""
import ctypes
import os
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F


@pytest.fixture(scope="module")
def lib():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


def describe(lib, kind, geom, shortcut=0):
    B, H, W, Ci, Co, k, s = geom
    buf = ctypes.create_string_buffer(1 << 17)
    rc = lib.mapnet_test_plan_describe(kind, B, H, W, Ci, Co, k, s, shortcut, buf, len(buf))
    assert rc == 0, lib.mapnet_last_error()
    return json.loads(buf.value.decode())


def parity_view(x, s, a, b):
    """[B,H,W,C] -> the view a stride-s conv reads through tensor map (a, b)"""
    return x if s == 1 else x[:, a::2, b::2, :]


def gather(v, dh, dw, Hs, Ws):
    """v[n, jh+dh, jw+dw, :] for jh < Hs, jw < Ws, zero outside v (what the TMA box load returns)"""
    B, Hv, Wv, C = v.shape
    out = torch.zeros(B, Hs, Ws, C, dtype=v.dtype)
    h0, h1 = max(0, -dh), min(Hs, Hv - dh)
    w0, w1 = max(0, -dw), min(Ws, Wv - dw)
    if h1 > h0 and w1 > w0:
        out[:, h0:h1, w0:w1, :] = v[:, h0 + dh:h1 + dh, w0 + dw:w1 + dw, :]
    return out


def make_case(geom, seed):
    B, H, W, Ci, Co, k, s = geom
    g = torch.Generator().manual_seed(seed)
    pad = (k - 1) // 2
    x = torch.randn(B, Ci, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(Co, Ci, k, k, generator=g, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(x, w, None, s, pad)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dy)
    nhwc = lambda t: t.detach().permute(0, 2, 3, 1).contiguous()
    return dict(x=nhwc(x), y=nhwc(y), dy=nhwc(dy), dx=nhwc(x.grad), w=w.detach(),
                dw_krsc=w.grad.permute(0, 2, 3, 1).reshape(Co, k * k, Ci).contiguous())


def w_krsc(w):      # [Co][KK*Ci], K index = tap*Ci + ci
    Co, Ci, k, _ = w.shape
    return w.permute(0, 2, 3, 1).reshape(Co, k * k * Ci)


def w_dg(w):        # [Ci][KK*Co], K index = tap*Co + co
    Co, Ci, k, _ = w.shape
    return w.permute(1, 2, 3, 0).reshape(Ci, k * k * Co)


def replay_launches(plan, views, wmats, out_shape):
    """fprop / dgrad through the per-tap engines: every class of every launch"""
    out = torch.full(out_shape, float("nan"), dtype=torch.float64)
    written = torch.zeros(out_shape[:3], dtype=torch.int32)
    for L in plan["launches"]:
        assert L["TW"] * L["TH"] * L["TN"] == 128
        assert L["n_tiles_m"] == L["tiles_w"] * L["tiles_h"] * L["tiles_n"]
        assert L["n_tiles_n"] * plan["BN"] == L["Cout"]
        Cs, os_ = L["Cs"], L["os"]
        for c in L["classes"]:
            Hs, Ws = c["Hs"], c["Ws"]
            # the shared tile grid reaches every pixel of the class
            assert L["tiles_w"] * L["TW"] >= Ws and L["tiles_h"] * L["TH"] >= Hs and L["tiles_n"] * L["TN"] >= L["Nimg"]
            acc = torch.zeros(out_shape[0], Hs, Ws, out_shape[3], dtype=torch.float64)
            for dh, dw, mp, kidx in c["taps"]:
                v = views[mp & 3]
                Wm = wmats[1 if (mp & 4) else 0]
                acc += gather(v, dh, dw, Hs, Ws) @ Wm[:, kidx * Cs:(kidx + 1) * Cs].T
            out[:, c["oa"]::os_, c["ob"]::os_, :][:, :Hs, :Ws, :] = acc
            written[:, c["oa"]::os_, c["ob"]::os_][:, :Hs, :Ws] += 1
    assert int(written.min()) == 1 and int(written.max()) == 1, "output pixels not covered exactly once"
    return out


GEOMS = [(2, 16, 16, 64, 64, 3, 1), (2, 16, 16, 64, 128, 3, 2), (2, 16, 16, 64, 128, 1, 2), (3, 9, 11, 128, 128, 3, 1),
         (2, 18, 22, 64, 128, 3, 2), (1, 8, 8, 128, 256, 3, 2), (1, 12, 10, 128, 64, 1, 1), (3, 17, 13, 64, 128, 3, 2),
         (2, 7, 5, 128, 128, 3, 2), (1, 33, 9, 64, 64, 3, 1), (2, 6, 40, 64, 64, 3, 1), (1, 11, 11, 64, 128, 1, 2)]


@pytest.mark.parametrize("geom", GEOMS)
def test_fprop_plan_replays_to_conv2d(lib, geom):
    c = make_case(geom, 3)
    plan = describe(lib, 0, geom)
    B, H, W, Ci, Co, k, s = geom
    maps = plan["launches"][0]["maps"]
    views = [parity_view(c["x"], s, a, b) for a, b in maps] + [None] * 4
    got = replay_launches(plan, views, [w_krsc(c["w"])], tuple(c["y"].shape))
    assert float((got - c["y"]).abs().max()) < 1e-9 * max(1.0, float(c["y"].abs().max()))


@pytest.mark.parametrize("geom", GEOMS)
def test_dgrad_plan_replays_to_autograd(lib, geom):
    c = make_case(geom, 4)
    plan = describe(lib, 1, geom)
    if geom[6] == 2:
        assert len(plan["launches"]) == 1 and len(plan["launches"][0]["classes"]) == 4     # one launch, four parity classes
        taps = sorted(len(cl["taps"]) for cl in plan["launches"][0]["classes"])
        assert taps == ([1, 2, 2, 4] if geom[5] == 3 else [0, 0, 0, 1])
    got = replay_launches(plan, [c["dy"], None, None, None], [w_dg(c["w"])], tuple(c["dx"].shape))
    assert float((got - c["dx"]).abs().max()) < 1e-9 * max(1.0, float(c["dx"].abs().max()))


@pytest.mark.parametrize("geom", [g for g in GEOMS if g[5] == 3 and g[6] == 2])
def test_dgrad_plan_with_folded_shortcut(lib, geom):
    """conv1 (3x3/s2) dgrad + the block's 1x1/s2 downsample dgrad as the 10th tap of class (0,0)"""
    B, H, W, Ci, Co, k, s = geom
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, Ci, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    w1 = torch.randn(Co, Ci, 3, 3, generator=g, dtype=torch.float64)
    w2 = torch.randn(Co, Ci, 1, 1, generator=g, dtype=torch.float64)
    y1, y2 = F.conv2d(x, w1, None, 2, 1), F.conv2d(x, w2, None, 2, 0)
    dy1 = torch.randn(y1.shape, generator=g, dtype=torch.float64)
    dy2 = torch.randn(y2.shape, generator=g, dtype=torch.float64)
    ((y1 * dy1).sum() + (y2 * dy2).sum()).backward()
    nhwc = lambda t: t.detach().permute(0, 2, 3, 1).contiguous()
    plan = describe(lib, 1, geom, shortcut=1)
    assert plan["shortcut"] == 1
    last = plan["launches"][0]["classes"][-1]
    assert (last["oa"], last["ob"]) == (0, 0) and last["taps"][-1] == [0, 0, 5, 0]      # map 1 | second weight matrix
    got = replay_launches(plan, [nhwc(dy1), nhwc(dy2), None, None], [w_dg(w1), w_dg(w2)], (B, H, W, Ci))
    ref = nhwc(x.grad)
    assert float((got - ref).abs().max()) < 1e-9 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("geom", GEOMS)
def test_wgrad_plan_replays_to_autograd(lib, geom):
    c = make_case(geom, 6)
    B, H, W, Ci, Co, k, s = geom
    plan = describe(lib, 2, geom)
    P = plan["wgrad"]
    assert P["TW"] * P["TH"] * P["TN"] == 64 and P["n_pix_tiles"] == P["tiles_w"] * P["tiles_h"] * P["tiles_n"]
    Ho, Wo = c["dy"].shape[1], c["dy"].shape[2]
    assert P["tiles_w"] * P["TW"] >= Wo and P["tiles_h"] * P["TH"] >= Ho and P["tiles_n"] * P["TN"] >= B
    assert P["splits"] * P["tiles_per_split"] >= P["n_pix_tiles"] and (P["splits"] - 1) * P["tiles_per_split"] < P["n_pix_tiles"]
    assert P["n_chunks"] == k * k * (Ci // 64) and len(P["chunks"]) == P["n_chunks"]
    assert P["n_mtiles"] * 2 >= P["n_chunks"] and P["n_ntiles"] * P["BN"] == Co
    views = [parity_view(c["x"], s, a, b) for a, b in P["maps"]]
    got = torch.full((Co, k * k, Ci), float("nan"), dtype=torch.float64)
    for dh, dw, mp, c0, tap in P["chunks"]:
        xv = gather(views[mp], dh, dw, Ho, Wo)[..., c0:c0 + 64]                    # [B,Ho,Wo,64]
        got[:, tap, c0:c0 + 64] = torch.einsum("nhwo,nhwc->oc", c["dy"], xv)
    assert bool(torch.isfinite(got).all()), "some (tap, channel chunk) of dW is never produced"
    assert float((got - c["dw_krsc"]).abs().max()) < 1e-9 * max(1.0, float(c["dw_krsc"].abs().max()))


def test_resnet34_persistent_plans_at_benchmark_size(lib):
    """The engines the cost model picks for the BASELINE shapes (B = 64, 256x256 input): recorded here so that a
    change of the tile choice shows up in review, and checked for the invariants the kernels rely on."""
    rows = []
    for name, H, Ci, Co, k, s in (("layer1", 64, 64, 64, 3, 1), ("layer2.0.conv1", 64, 64, 128, 3, 2),
                                  ("layer2", 32, 128, 128, 3, 1), ("layer3.0.conv1", 32, 128, 256, 3, 2),
                                  ("layer3", 16, 256, 256, 3, 1), ("layer4.0.conv1", 16, 256, 512, 3, 2),
                                  ("layer4", 8, 512, 512, 3, 1)):
        for kind in (0, 1):
            p = describe(lib, kind, (64, H, H, Ci, Co, k, s), shortcut=1 if (kind == 1 and s == 2) else 0)
            n_out = Co if kind == 0 else Ci
            L = p["launches"][0]
            items = L["n_tiles_m"] * L["n_tiles_n"] * len(L["classes"])
            assert n_out % p["BN"] == 0 and p["BN"] in (64, 128) and len(p["launches"]) == 1
            rows.append((name, "fprop" if kind == 0 else "dgrad", p["BN"], items))
    table = {(r[0], r[1]): r[2:] for r in rows}
    assert table[("layer1", "fprop")][0] == 64
    for r in rows:
        assert r[3] >= 32, r          # enough work items to occupy a good part of the 132 SMs
