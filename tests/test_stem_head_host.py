"""Host-only checks of the stem / head test entry points (no GPU needed): the exports, argument errors returned before
any launch, and that the case list of tests/test_gpu_stem_head.py still reaches the plans that matter -- so a change
of a plan heuristic cannot quietly drop coverage."""
import ctypes

import pytest

from geomapnet_b200 import _lib

import test_gpu_stem_head as T


@pytest.fixture(scope="module")
def lib():
    from geomapnet_b200 import build
    build.build(verbose=False)
    return _lib.lib()


def test_new_entry_points_are_exported(lib):
    for name in ("mapnet_test_stem_ex", "mapnet_test_head"):
        assert name in _lib.EXPORTED
        assert hasattr(lib, name), name


def _err(lib):
    m = lib.mapnet_last_error()
    return m.decode() if m else ""


# a non-null placeholder: every call below fails its argument checks before it could dereference one
P = 256


@pytest.mark.parametrize("args,msg", [
    ((0, 64, 256, 256, P, P, P, None, None, 0.0, None), "precision"),
    ((2, 64, 256, 256, P, P, P, None, None, 0.0, None), "precision"),
    ((1, 0, 256, 256, P, P, P, None, None, 0.0, None), "bad shape"),
    ((1, 4, 31, 256, P, P, P, None, None, 0.0, None), "bad shape"),
    ((1, 4, 256, 256, None, P, P, None, None, 0.0, None), "null argument"),
    ((1, 4, 256, 256, P, P, None, None, None, 0.0, None), "null argument"),
    ((1, 4, 256, 256, P, P, P, P, None, 0.0, None), "go together"),
    ((1, 4, 256, 256, P, P, P, None, P, 0.0, None), "go together"),
    ((1, 4, 256, 256, P, P, P, P, P, 0.25, None), "out_scale"),          # bf16 has no gradient scale
    ((3, 4, 256, 256, P, P, P, None, None, 0.25, None), "out_scale"),    # no wgrad to scale
    ((3, 4, 256, 256, P, P, P, P, P, -1.0, None), "out_scale"),
    ((3, 4, 256, 256, P, P, P, P, P, float("inf"), None), "out_scale"),
])
def test_stem_ex_argument_errors_before_any_launch(lib, args, msg):
    n0 = lib.mapnet_launch_count()
    assert lib.mapnet_test_stem_ex(*args, None) != 0
    assert msg in _err(lib), _err(lib)
    assert lib.mapnet_launch_count() == n0


U64 = _lib.UINT64_MAX
# (B, F, feat, params, droprate, seed, step, stride, ctr, mask, fcpre, hdrop, pred, dpred, filter, dh, dfeat, grads, scale2)
OK = (4, 64, P, P, 0.0, 1, 0, 256, None, None, P, P, P, None, 0, None, None, None, None)


def _with(**kw):
    names = ["B", "F", "feat", "params", "droprate", "seed", "step", "stride", "ctr", "mask", "fcpre", "hdrop", "pred",
             "dpred", "filter", "dh", "dfeat", "grads", "scale2"]
    a = list(OK)
    for k, v in kw.items():
        a[names.index(k)] = v
    return tuple(a)


@pytest.mark.parametrize("args,msg", [
    (_with(B=0), "need B >= 1"),
    (_with(F=6), "multiple of 4"),
    (_with(F=66), "multiple of 4"),
    (_with(feat=None), "null argument"),
    (_with(pred=None), "null argument"),
    (_with(droprate=1.0), "droprate"),
    (_with(droprate=-0.1), "droprate"),
    (_with(droprate=0.5), "dropout needs mask"),                                   # no mask
    (_with(droprate=0.5, mask=P, stride=255), "dropout needs mask"),               # stride < B * F
    (_with(droprate=0.5, mask=P, step=U64), "dropout needs mask"),                 # device counter missing
    (_with(dpred=P), "the backward needs"),
    (_with(dpred=P, dh=P, dfeat=P), "the backward needs"),
    (_with(scale2=P), "gradient scale"),
])
def test_head_argument_errors_before_any_launch(lib, args, msg):
    n0 = lib.mapnet_launch_count()
    assert lib.mapnet_test_head(*args, None) != 0
    assert msg in _err(lib), _err(lib)
    assert lib.mapnet_launch_count() == n0


def test_stem_wgrad_plan_is_described(lib):
    """k == 7 describes the stem's fprop and wgrad, in bf16 and strict mode; the shortcut and fp8 flags stay errors"""
    buf = ctypes.create_string_buffer(1 << 16)
    for kind in (0, 2):
        for flags in (0, 2):
            assert lib.mapnet_test_plan_describe(kind, 64, 256, 256, 3, 64, 7, 2, flags, buf, len(buf)) == 0, _err(lib)
    w = T.stem_plan(2, 64, 256, 256, "bf16")
    assert (w["BN"], w["pix"]) == (64, 64 * 128 * 128 // 64)
    for kind, flags in ((1, 0), (2, 1), (0, 4), (2, 4)):
        assert lib.mapnet_test_plan_describe(kind, 64, 256, 256, 3, 64, 7, 2, flags, buf, len(buf)) != 0, (kind, flags)


def test_case_list_covers_the_plans_that_matter(lib):
    wg = {"bf16": [], "tc_split": []}
    for c in T.STEM_CASES:
        f, w = T.expected_stem_plans(c)
        wg[c[1]].append(w)
        assert f["taps"] * f["Cs"] // 16 == (64 if c[1] == "tc_split" else 16)
    for prec in ("bf16", "tc_split"):
        assert any(w["splits"] > 1 and w["last"] < w["tps"] for w in wg[prec]), \
            "no multi-split stem wgrad with a ragged last split in %s" % prec
    assert any(c[5] for c in T.STEM_CASES), "no coherent stem wgrad"
    assert max(c[2][0] * ((c[2][1] - 1) // 2 + 1) * ((c[2][2] - 1) // 2 + 1) for c in T.STEM_CASES) >= 2 ** 20, \
        "no stem wgrad over >= 1 M pixels"
    assert any(((c[2][2] - 1) // 2 + 1) % 2 == 1 for c in T.STEM_CASES), "no odd stem output width"
    plans = {B: T.head_plans(B) for B in T.HEAD_BATCHES}
    pose = {p["pose"][0] for p in plans.values()}
    dfeat = {p["dfeat"][0] for p in plans.values()}
    assert {32, 16} <= pose, pose
    assert {4, 2, 1} <= dfeat, dfeat
    assert any(p["dWpose"][0] > 1 for p in plans.values()), "no split-K weight-gradient product (M = 3, sak = 6)"
    assert any(B % 32 for B in T.HEAD_BATCHES), "no ragged 32-row tile"
    assert any(p not in (0.0, 0.5) for p in T.DROPRATES), "no keep scale that is not a power of two"
