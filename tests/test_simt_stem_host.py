"""Host-only checks of the CUDA-core conv, im2col-stem and im2col-trunk entry points and of tests/test_gpu_simt_stem.py's
case lists (no GPU needed): the exports, every argument error returned before any launch, the limits of
launch_stem_im2col (the patch-matrix row of 192 and the 48 KB of shared memory of a W <= 570 frame), and that the cases still
reach every mode and stem layout, every wgrad split regime of launch_conv_simt_wgrad, a ragged pixel count and the N / K
tails -- so a change of a plan or of a case list cannot quietly drop coverage."""
import ctypes

import pytest

from geomapnet_b200 import _lib

import test_gpu_simt_stem as T

NEW = ("mapnet_test_conv_simt", "mapnet_test_stem_im2col", "mapnet_test_trunk_create")


@pytest.fixture(scope="module")
def lib():
    from geomapnet_b200 import build
    build.build(verbose=False)
    return _lib.lib()


def _err(lib):
    m = lib.mapnet_last_error()
    return m.decode() if m else ""


def test_new_entry_points_are_exported(lib):
    for name in NEW:
        assert name in _lib.EXPORTED
        assert hasattr(lib, name), name


# a non-null placeholder: every call below fails its argument checks before it could dereference one
P = 256
GEOM = (4, 16, 16, 64, 64, 3, 1)


@pytest.mark.parametrize("args,msg", [
    ((1, 0) + GEOM + (P, None, P, None, P), "not a CUDA-core precision"),        # bf16 (tensor cores)
    ((3, 0) + GEOM + (P, None, P, None, P), "not a CUDA-core precision"),        # tc_split
    ((7, 0) + GEOM + (P, None, P, None, P), "precision 7"),
    ((0, 3) + GEOM + (P, None, P, None, P), "kind 3"),
    ((0, -1) + GEOM + (P, None, P, None, P), "kind -1"),
    ((0, 0, 4, 16, 16, 6, 64, 3, 1, P, None, P, None, P), "Ci 6"),
    ((2, 1, 4, 16, 16, 64, 10, 3, 1, P, None, P, None, P), "Co 10"),
    ((0, 0, 4, 16, 16, 64, 64, 5, 1, P, None, P, None, P), "k 5"),
    ((0, 0, 4, 16, 16, 64, 64, 3, 3, P, None, P, None, P), "stride 3"),
    ((0, 0, 0, 16, 16, 64, 64, 3, 1, P, None, P, None, P), "B 0"),
    ((0, 0, 4, 0, 16, 64, 64, 3, 1, P, None, P, None, P), "bad shape"),
    ((0, 0) + GEOM + (None, None, P, None, P), "null argument"),
    ((0, 0) + GEOM + (P, None, None, None, P), "null argument"),                 # fprop without weights
    ((2, 1) + GEOM + (P, None, None, None, P), "null argument"),                 # dgrad without weights
    ((0, 2) + GEOM + (P, None, None, None, P), "null argument"),                 # wgrad without dy
    ((0, 0) + GEOM + (P, None, P, None, None), "null argument"),
    ((0, 0) + GEOM + (P, None, P, P, P), "a residual is a dgrad feature"),
    ((2, 2) + GEOM + (P, P, None, P, P), "a residual is a dgrad feature"),
])
def test_conv_simt_argument_errors_before_any_launch(lib, args, msg):
    n0 = lib.mapnet_launch_count()
    assert lib.mapnet_test_conv_simt(*args, None) != 0
    assert msg in _err(lib), _err(lib)
    assert lib.mapnet_launch_count() == n0


# (precision, B, H, W, x, w, a_out, y, dy, dw, out_scale, host_sums)
STEM = (256, 256, P, P, None, P, P, P, 0.0, None)


@pytest.mark.parametrize("args,msg", [
    ((4, 2) + STEM, "precision 4"),                                              # fp8 has no training stem
    ((-1, 2) + STEM, "precision -1"),
    ((0, 0) + STEM, "bad shape"),
    ((1, 2, 31, 256) + STEM[2:], "bad shape"),
    ((2, 2, 256, 16) + STEM[2:], "bad shape"),
    ((0, 2, 256, 571) + STEM[2:], "image width 571 too large (at most 570)"),
    ((2, 2, 256, 579) + STEM[2:], "image width 579 too large (at most 570)"),
    ((3, 1, 64, 4000) + STEM[2:], "image width 4000 too large"),
    ((0, 2, 256, 256, None, P, None, P, P, P, 0.0, None), "null argument"),
    ((1, 2, 256, 256, P, None, None, P, P, P, 0.0, None), "null argument"),
    ((3, 2, 256, 256, P, P, None, None, P, P, 0.0, None), "null argument"),
    ((0, 2, 256, 256, P, P, None, P, None, P, 0.0, None), "dy and dw_oihw go together"),
    ((1, 2, 256, 256, P, P, None, P, P, None, 0.0, None), "dy and dw_oihw go together"),
    ((1, 2, 256, 256, P, P, None, P, P, P, 0.5, None), "out_scale 0.5"),          # bf16 has no gradient scale
    ((0, 2, 256, 256, P, P, None, P, P, P, 0.5, None), "out_scale 0.5"),
    ((3, 2, 256, 256, P, P, None, P, None, None, 0.5, None), "out_scale 0.5"),   # no wgrad to scale
    ((3, 2, 256, 256, P, P, None, P, P, P, -1.0, None), "out_scale -1"),
    ((3, 2, 256, 256, P, P, None, P, P, P, float("inf"), None), "out_scale inf"),
    ((0, 2, 256, 256, P, P, None, P, P, P, 0.0, P), "tensor-core feature"),      # statistics: tensor-core epilogue
    ((2, 2, 256, 256, P, P, None, P, P, P, 0.0, P), "tensor-core feature"),
])
def test_stem_im2col_argument_errors_before_any_launch(lib, args, msg):
    n0 = lib.mapnet_launch_count()
    assert lib.mapnet_test_stem_im2col(*args, None) != 0
    assert msg in _err(lib), _err(lib)
    assert lib.mapnet_launch_count() == n0


@pytest.mark.parametrize("args,msg", [
    ((8, 256, 256, 2048, 1, 2), "im2col_stem 2"),
    ((8, 256, 256, 2048, 1, -1), "im2col_stem -1"),
    ((8, 256, 256, 2048, 4, 1), "precision 4"),                                  # fp8 is an inference precision
    ((8, 256, 256, 2048, -1, 0), "precision -1"),
    ((8, 31, 256, 2048, 1, 1), "bad shape"),
    ((-1, 256, 256, 2048, 1, 1), "bad shape"),
    ((8, 256, 256, 6, 1, 1), "bad shape"),
    ((8, 256, 256, 2046, 3, 1), "bad shape"),
])
def test_trunk_create_argument_errors_before_any_launch(lib, args, msg):
    h = ctypes.c_void_p(1)
    n0 = lib.mapnet_launch_count()
    assert lib.mapnet_test_trunk_create(ctypes.byref(h), *args) != 0
    assert msg in _err(lib), _err(lib)
    assert not h.value
    assert lib.mapnet_launch_count() == n0
    assert lib.mapnet_test_trunk_create(None, *args) != 0
    assert "null out pointer" in _err(lib)


@pytest.mark.parametrize("precision", ["fp32", "bf16", "bf16_simt", "tc_split"])
def test_spec_only_trunk_has_the_im2col_stem_table(lib, precision):
    """max_B = 0 (no device): the same parameter table as mapnet_trunk_create's, in both stem layouts"""
    ref = _lib.Trunk(0, 256, 341, 2048, precision)
    for stem in (0, 1):
        h = ctypes.c_void_p()
        _lib.check(lib.mapnet_test_trunk_create(ctypes.byref(h), 0, 256, 341, 2048, _lib.PREC[precision], stem),
                   "mapnet_test_trunk_create")
        try:
            assert lib.mapnet_params_numel(h) == lib.mapnet_params_numel(ref.h)
            assert lib.mapnet_param_count(h) == lib.mapnet_param_count(ref.h)
            assert [lib.mapnet_param_layout(h, i) for i in range(lib.mapnet_param_count(h))] == \
                [lib.mapnet_param_layout(ref.h, i) for i in range(lib.mapnet_param_count(ref.h))]
        finally:
            lib.mapnet_trunk_destroy(h)
    ref.close()


def test_im2col_width_limit_is_the_shared_memory_limit():
    smem = lambda W: 21 * (W + 6) * 4 + T.STEM_K * 4          # staged rows + the k -> offset table
    assert smem(T.MAX_IM2COL_W) <= 48 * 1024 < smem(T.MAX_IM2COL_W + 1)
    assert max(W for _, (B, H, W), _ in T.STEM_CASES) == T.MAX_IM2COL_W


def test_conv_cases_reach_every_split_regime_and_tail():
    plans = {name: T.simt_wgrad_plan(geom) for name, geom in T.CONV_CASES}
    # a single split that adds into dW
    assert plans["posenet_bs64.layer4"][0] == 1
    # 50 - 180 splits through the workspace, with a short last split
    assert plans["7scenes_b4.layer1"][:3] == (58, 384, 22016 - 57 * 384)
    assert plans["posenet_bs64.stem_view"][0] == 176
    assert any(p[0] > 100 for p in plans.values())
    assert any(1 < p[0] and p[2] < p[1] for p in plans.values())
    # the kchunk >= 256 clamp
    assert any(p[3] for p in plans.values())
    assert all(p[1] >= 256 and p[1] % 16 == 0 and 0 < p[2] <= p[1] for p in plans.values())
    geoms = [g for _, g in T.CONV_CASES]
    # a ragged pixel count (M not a multiple of the 64-row tile) in fprop / wgrad and in dgrad
    assert any((g[0] * T.out_hw(g)[0] * T.out_hw(g)[1]) % 64 for g in geoms)
    assert any((g[0] * g[1] * g[2]) % 64 for g in geoms)
    # N tails (Co or Ci not a multiple of 64) and K tails (taps * channels not a multiple of 16) on both sides
    assert any(g[4] % 64 for g in geoms) and any(g[3] % 64 for g in geoms)
    assert any((g[5] ** 2 * g[3]) % 16 for g in geoms) and any((g[5] ** 2 * g[4]) % 16 for g in geoms)
    # both strides, both filter sizes, and the model geometries
    assert {(g[5], g[6]) for g in geoms} == {(1, 1), (1, 2), (3, 1), (3, 2)}
    names = {n for n, _ in T.CONV_CASES}
    assert {"posenet_bs64.layer%d" % i for i in range(1, 5)} <= names
    assert {"mapnetpp_n16t10.layer1", "7scenes_b4.layer1", "7scenes_b4.layer3.0.conv1", "7scenes_b4.layer4"} <= names
    assert len(T.CONV_CASES) == len({g for _, g in T.CONV_CASES})


def test_stem_cases_reach_every_mode_and_layout(lib):
    assert set(T.TRAIN_PREC) == set(_lib.PREC)
    frames = {f for _, f, _ in T.STEM_CASES}
    assert (64, 256, 256) in frames and (4, 256, 341) in frames
    assert any(T.stem_hw(H, W)[1] % 2 for _, (B, H, W), _ in T.STEM_CASES)          # odd Wc: stem_fuse off
    for name, (B, H, W), plans in T.STEM_CASES:
        Hc, Wc = T.stem_hw(H, W)
        for prec in ("bf16", "tc_split"):
            assert (T.stem_view_plan(0, B, Hc, Wc, prec), T.stem_view_plan(2, B, Hc, Wc, prec)) == plans[prec], \
                (name, prec)
    # the training steps run on the im2col stem in both tensor-core modes, at a benchmark size in each
    assert {p for p, _ in T.STEP_CASES} == {"bf16", "tc_split"}
    for prec in ("bf16", "tc_split"):
        assert (prec, "posenet_b64_256") in T.STEP_CASES
