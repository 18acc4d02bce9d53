"""Host logic of the wgrad engine choice, checked WITHOUT a GPU.

`tc_plan_create` keeps every wgrad's K partition (pixel box, splits, pixel tiles per split) as the per-tap engine
(k_tc_wgrad) defines it and then picks the engine that runs it: the per-tap engine or, for stride-1 3x3 convs, the halo
engine (k_halo_wgrad) with 3 or 9 filter taps per CTA.  Here the plan (`mapnet_test_plan_describe`) is checked for
the benchmark shapes and fuzzed ones: the engine chosen, the K partition against the per-tap formula, the CTA's halo
against its shared-memory slot, and the halo descriptor arithmetic -- every (filter tap, k16 step, lane row) of a
k-block addresses the halo row of the pixel the per-tap box puts there."""
import ctypes
import json

import pytest

NSM = 132
HALO_MAX = {3: 16384, 9: 28672}         # bytes of a stage's halo slot (halo_max_bytes)


@pytest.fixture(scope="module")
def lib():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


def describe(lib, geom, flags=0):
    B, H, W, Ci, Co, k, s = geom
    buf = ctypes.create_string_buffer(1 << 17)
    assert lib.mapnet_test_plan_describe(2, B, H, W, Ci, Co, k, s, flags, buf, len(buf)) == 0, lib.mapnet_last_error()
    return json.loads(buf.value.decode())["wgrad"]


def cdiv(a, b):
    return -(-a // b)


def per_tap_partition(geom):
    """the per-tap engine's K partition (tc_plan_create, bf16 mode)"""
    B, H, W, Ci, Co, k, s = geom
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    tw = 8
    while tw < Wo and tw < 64:
        tw *= 2
    th = 1
    while tw * th < 64 and th < Ho:
        th *= 2
    tn = max(1, 64 // (tw * th))
    npix = cdiv(Wo, tw) * cdiv(Ho, th) * cdiv(B, tn)
    bn = 128 if Co % 128 == 0 else 64
    units = cdiv(k * k * Ci // 64, 2) * (Co // bn)
    splits = min(max(1, 2 * NSM // units), npix)
    tps = cdiv(npix, splits)
    return dict(TW=tw, TH=th, TN=tn, n_pix_tiles=npix, BN=bn, splits=cdiv(npix, tps), tiles_per_split=tps)


def check_plan(P, geom):
    B, H, W, Ci, Co, k, s = geom
    for key, v in per_tap_partition(geom).items():
        assert P[key] == v, (geom, key, P[key], v)
    E = P["engine"]
    taps, bn = E["taps"], E["BN"]
    if taps == 0:
        assert bn == P["BN"] and E["units"] == P["n_mtiles"] * P["n_ntiles"]
        return E
    assert k == 3 and s == 1 and (taps, bn) in ((3, 64), (3, 128), (9, 64)) and Co % bn == 0
    assert E["units"] == (Ci // 64) * (9 // taps) * (Co // bn) and E["grid"] == E["units"] * P["splits"]
    TW, TH, TN, RW, HR = P["TW"], P["TH"], P["TN"], E["RW"], E["HR"]
    assert RW % 8 == 0 and RW >= TW + 2 and HR == TH + taps // 3 - 1
    assert E["halo_bytes"] == 128 * RW * HR * TN <= HALO_MAX[taps]
    # pixel q of the box (w fastest, then h, then image) under filter tap (r, kw) of the CTA's rows r = 0 .. taps/3 - 1
    halo_row = lambda q, r, kw: ((q // (TW * TH)) * HR + (q // TW) % TH + r) * RW + q % TW + kw
    for r in range(taps // 3):
        for kw in range(3):
            for j in range(4):
                start = E["step_row"][j] + r * RW + kw
                for i in range(16):
                    row = start + (i if i < 8 else E["sbo"] // 128 + i - 8)
                    assert row == halo_row(16 * j + i, r, kw), (geom, r, kw, j, i)
                    assert 0 <= row < RW * HR * TN
    return E


# (name, geometry, expected engine (taps, BN)); B = 64 is posenet_bs64, B = 96 mapnet_n32t3 (32 tuples x 3 frames)
BENCH = [("layer1", (64, 64, 64, 64, 64, 3, 1), (3, 64)), ("layer2", (64, 32, 32, 128, 128, 3, 1), (9, 64)),
         ("layer3", (64, 16, 16, 256, 256, 3, 1), (9, 64)), ("layer4", (64, 8, 8, 512, 512, 3, 1), (3, 128)),
         ("layer1", (96, 64, 64, 64, 64, 3, 1), (3, 64)), ("layer2", (96, 32, 32, 128, 128, 3, 1), (9, 64)),
         ("layer3", (96, 16, 16, 256, 256, 3, 1), (9, 64)), ("layer4", (96, 8, 8, 512, 512, 3, 1), (3, 128)),
         ("layer2.0.conv1", (64, 64, 64, 64, 128, 3, 2), (0, 128)),
         ("layer2.0.downsample", (64, 64, 64, 64, 128, 1, 2), (0, 128)),
         ("layer4.0.conv1", (96, 16, 16, 256, 512, 3, 2), (0, 128))]


@pytest.mark.parametrize("case", BENCH, ids=["%s-B%d" % (c[0], c[1][0]) for c in BENCH])
def test_benchmark_wgrad_engines(lib, case):
    name, geom, want = case
    E = check_plan(describe(lib, geom), geom)
    assert (E["taps"], E["BN"]) == want, (name, geom, E)


FUZZ = [(2, 16, 16, 64, 64, 3, 1), (3, 9, 11, 128, 128, 3, 1), (1, 33, 9, 64, 64, 3, 1), (2, 6, 40, 64, 64, 3, 1),
        (5, 64, 64, 64, 64, 3, 1), (5, 8, 8, 512, 512, 3, 1), (4, 64, 86, 64, 64, 3, 1), (4, 8, 11, 512, 512, 3, 1),
        (1, 3, 5, 128, 256, 3, 1), (7, 1, 1, 64, 64, 3, 1), (2, 16, 16, 64, 128, 3, 2), (1, 12, 10, 128, 64, 1, 1)]


@pytest.mark.parametrize("geom", FUZZ)
def test_fuzzed_wgrad_plans_keep_the_partition(lib, geom):
    check_plan(describe(lib, geom), geom)


def test_strict_mode_keeps_the_per_tap_engine(lib):
    P = describe(lib, (64, 16, 16, 256, 256, 3, 1), flags=2)
    assert P["engine"]["taps"] == 0
