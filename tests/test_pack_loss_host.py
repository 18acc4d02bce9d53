"""Host-only checks of the weight-pack entry points and of tests/test_gpu_pack_loss.py's case lists (no GPU needed): the
exports, argument errors returned before any launch, the descriptor table's invariants against the parameter table,
and that the cases still reach every precision, both stem layouts, the short row group of every k_pack_weights group
size that occurs and every criterion mode -- so a change of the table or of a case list cannot quietly drop coverage."""
import ctypes

import numpy as np
import pytest

from geomapnet_b200 import _lib

import test_gpu_pack_loss as T


@pytest.fixture(scope="module")
def lib():
    from geomapnet_b200 import build
    build.build(verbose=False)
    return _lib.lib()


def _err(lib):
    m = lib.mapnet_last_error()
    return m.decode() if m else ""


def test_new_entry_points_are_exported(lib):
    for name in ("mapnet_test_weight_table", "mapnet_test_pack_weights"):
        assert name in _lib.EXPORTED
        assert hasattr(lib, name), name


# a non-null placeholder: every call below fails its argument checks before it could dereference one
P = 256


@pytest.mark.parametrize("args,msg", [
    ((5, 0, 256, 256, P, P, P, None), "precision 5"),
    ((-1, 0, 256, 256, P, P, P, None), "precision -1"),
    ((1, 0, 31, 256, P, P, P, None), "H,W>=32"),
    ((1, 0, 256, 16, P, P, P, None), "H,W>=32"),
    ((0, 0, 256, 256, None, P, P, None), "null argument"),
    ((3, 0, 256, 256, P, None, P, None), "null argument"),
    ((1, 0, 256, 256, P, P, None, None), "null argument"),
    ((4, 0, 256, 256, P, P, P, None), "s_w_out"),           # fp8 needs the scales
    ((1, 0, 256, 256, P, P, P, P), "s_w_out"),              # only fp8 has them
    ((4, 1, 256, 256, P, P, P, P), "no im2col stem"),       # the fp8 engine requires the space-to-depth stem
    ((1, 2, 256, 256, P, P, P, None), "im2col_stem 2"),
])
def test_pack_weights_argument_errors_before_any_launch(lib, args, msg):
    n0 = lib.mapnet_launch_count()
    assert lib.mapnet_test_pack_weights(*args, None) != 0
    assert msg in _err(lib), _err(lib)
    assert lib.mapnet_launch_count() == n0


def test_weight_table_argument_errors(lib):
    buf = (ctypes.c_int64 * 512)()
    assert lib.mapnet_test_weight_table(256, 256, 1, 0, buf, 2 + 9 * 36 - 1) != 0
    assert "cap" in _err(lib)
    assert lib.mapnet_test_weight_table(256, 256, 7, 0, buf, 512) != 0
    assert "precision 7" in _err(lib)
    assert lib.mapnet_test_weight_table(256, 256, 4, 1, buf, 512) != 0
    assert "no im2col stem" in _err(lib)
    assert lib.mapnet_test_weight_table(256, 256, 1, 0, None, 512) != 0
    assert lib.mapnet_test_weight_table(256, 256, 1, 0, buf, 2 + 9 * 36) == 0


@pytest.mark.parametrize("frame,mode,stem", T.PACK_CASES)
def test_weight_table_invariants(lib, frame, mode, stem):
    H, W = T.FRAMES[frame]
    T.table_invariants(H, W, mode, stem)


def test_pack_cases_reach_every_mode_and_stem_layout(lib):
    assert {m for _, m, _ in T.PACK_CASES} == set(T.PACK_PREC)
    assert set(T.FRAMES.values()) == {(256, 256), (256, 341)}
    for frame, mode, stem in T.PACK_CASES:
        rows, _ = T.weight_table(*T.FRAMES[frame], mode, stem)
        assert ("s2d" if rows[0][8] else "im2col") == stem
    # every stem layout a precision can run: the CUDA-core modes im2col, the tensor-core training modes both, fp8 s2d
    reached = {(m, s) for _, m, s in T.PACK_CASES}
    assert reached == {("fp32", "im2col"), ("bf16_simt", "im2col"), ("bf16", "s2d"), ("bf16", "im2col"),
                       ("tc_split", "s2d"), ("tc_split", "im2col"), ("fp8", "s2d")}


def test_weight_table_does_not_depend_on_the_frame(lib):
    """the 7Scenes pack cases confirm the packs do not see the frame geometry; they do not test another layout"""
    for mode in T.PACK_PREC:
        assert T.weight_table(256, 256, mode, T.STEM_LAYOUT[mode]) == T.weight_table(256, 341, mode, T.STEM_LAYOUT[mode])


def test_planted_rows_reach_every_short_row_group(lib):
    rows, _ = T.weight_table(256, 256, "bf16")
    groups = {}
    for i, r in enumerate(rows[1:], start=1):
        G = T.pack_group(r[5] * r[6] * r[3])
        groups.setdefault(G, []).append(r[2] % G)
    # layer1: 64 = 9 * 7 + 1, layer2: 128 = 42 * 3 + 2 -- the groups k_pack_weights runs short
    short = {G for G, rest in groups.items() if any(rest)}
    assert short == {3, 7}
    plants = T.plant_rows(rows)
    for G in short:
        hit = [(i, co) for i, co, kind in plants if kind == "edges" and i > 0
               and T.pack_group(rows[i][5] * rows[i][6] * rows[i][3]) == G and co >= rows[i][2] - rows[i][2] % G]
        assert hit, "no edge row in a short group of size %d" % G
    assert {T.pack_group(r[5] * r[6] * r[3]) for i, r in enumerate(rows) if i > 0
            and any(p[0] == i and p[2] == "edges" for p in plants)} >= {1, 3, 7, 8}
    assert any(p[0] == 0 for p in plants)                      # the stem's slab path
    kinds = {k for _, _, k in plants}
    assert kinds >= {"f8_zero", "f8_amax_448", "f8_above_448", "f8_inf", "f8_tiny"}


def test_planted_values_hit_their_edges():
    """the edge values really are the ties / subnormals / saturations the docstring names"""
    v = T.EDGE_VALUES
    assert np.isnan(v).sum() == 1 and np.any(np.signbit(v) & (v == 0))
    assert np.any((np.abs(v) > 0) & (np.abs(v) < np.float32(2.0 ** -126)))          # fp32 subnormals
    assert np.any(np.abs(v) > 65504)
    bf = v[np.isfinite(v)].view(np.uint32)
    assert np.any((bf & 0xFFFF) == 0x8000)                                            # exact bf16 ties
    h = v[np.isfinite(v) & (np.abs(v) < 65504)]
    assert np.any(np.abs(h.astype(np.float64) - h.astype(np.float16).astype(np.float64)) ==
                  np.abs(np.spacing(h.astype(np.float16)).astype(np.float64)) / 2)     # exact fp16 ties
    assert T.f8_pow2_scale(0.0) == 1.0 and T.f8_pow2_scale(np.inf) == 2.0 ** 120
    assert T.f8_pow2_scale(T.F8_AMAX) == 2.0 ** -12
    assert T.f8_pow2_scale(np.nextafter(T.F8_AMAX, np.float32(1))) == 2.0 ** -11
    assert T.f8_pow2_scale(2.0 ** -120) == 2.0 ** -126
    from fp8_emulation import pow2_scale
    for a in (0.0, 1e-30, 2.0 ** -120, float(T.F8_AMAX), 0.3, 448.0, 449.0, 3e38, np.inf):
        assert T.f8_pow2_scale(a) == pow2_scale(a)


def test_criterion_cases_reach_every_mode_and_edge():
    modes = {c[1] for c in T.CRIT_CASES}
    assert modes == set(_lib.LOSS_MODE)
    sizes = {c[2] * c[3] for c in T.CRIT_CASES}
    assert {1, 255, 256, 257, 1024} <= sizes
    for mode, N, Tp in (("posenet", 64, 1), ("mapnet", 32, 3), ("online", 16, 20), ("online_gps", 16, 20)):
        assert {c[4] for c in T.CRIT_CASES if c[1:4] == (mode, N, Tp)} == set(T.S4)
    assert {c[5] for c in T.CRIT_CASES if c[1] == "online"} == {"vo", "large"}
    assert len({c[0] + "." + c[4] for c in T.CRIT_CASES}) == len(T.CRIT_CASES)
    assert len({c[0] for c in T.BATCH_CASES}) == len(T.BATCH_CASES)
    for _, mode, Tb, sizes in T.BATCH_CASES:
        rows = [s * Tb for s in sizes]
        assert max(rows) == T.MAX_BATCH_ROWS - T.MAX_BATCH_ROWS % Tb and any(256 < r < T.MAX_BATCH_ROWS for r in rows)
        assert T.MAX_BATCH_ROWS * 48 <= 200 * 1024 < (T.MAX_BATCH_ROWS + 1) * 48


def test_vo_case_rotations_are_vo_sized():
    """the "vo" regime's relative rotations sit in [1e-3, 1e-2] rad, the "large" ones are of order 1"""
    from oracle import mapnet_oracle as O
    import torch
    for regime, lo, hi in (("vo", 5e-4, 2e-2), ("large", 0.05, 3.2)):
        pred, _ = T.make_crit_inputs("online", 16, 20, regime, 1)
        o = O.calc_vos(torch.from_numpy(pred[:, 10:].astype(np.float64))).numpy()
        th = np.linalg.norm(o[..., 3:], axis=-1)
        assert lo <= th.min() and th.max() <= hi, (regime, th.min(), th.max())


def test_sqnorm_cases_reach_both_paths_and_every_tail():
    """the float4 path with scalar tails of 1, 2 and 3 elements, and the scalar path of an unaligned start; each
    planted head / tail / past-the-end value is thousands of bounds"""
    import inspect
    cases = next(m.args[1] for m in T.test_sqnorm_vs_float64.pytestmark if m.name == "parametrize")
    n_full = 22347712                                   # a multiple of 64, as every params_flat length
    vec_tails = {(n_full - trim) % 4 for start, trim in cases if start % 4 == 0}
    assert vec_tails == {0, 1, 2, 3}
    assert any(start % 4 for start, _ in cases)
    for start, trim in cases:
        buf, n, pos = T.sqnorm_buffer(n_full, start, trim, 0)
        x = buf[start: start + n].astype(np.float64)
        bound = (2 * T.U + n * 2.0 ** -52) * float(x @ x)
        assert {start, start + n - 1, start + n} <= set(pos)
        assert min(float(buf[q]) ** 2 for q in pos) > 1000 * bound
    assert "sqnorm_buffer" in inspect.getsource(T.test_sqnorm_vs_float64)
