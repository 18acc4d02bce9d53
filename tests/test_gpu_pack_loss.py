"""The whole-network weight packs bit for bit, and the fused criterion, the validation pass's batch losses and the clip's
squared norm per element against float64, at the shapes the benchmarks run.

Packs (mapnet_test_pack_weights: the launches Net::forward_t runs per precision, and InferNet::load's fp8 pair, over the
real descriptor table of mapnet_test_weight_table).  The packs are data movement and one rounding, so every packed
element of all 36 convs is compared BIT FOR BIT with a numpy reference built from the table:
  * KRSC: the fp32 copy of params_flat[p_off ...] ([Co][KH][KW][Ci], mapnet_param_layout 1); bf16 is round to nearest
    even of it (bf16_simt rounds and stores the result as fp32).
  * dgrad: w_dg[ci][tap][co] = w_krsc[co][tap][ci]; the stem has none (its range stays unwritten).
  * stem (torch order [64][3][7][7]): the space-to-depth row of 256 (k = kh2*64 + kw2*16 + (pr*2+pc)*3 + c with
    (kh, kw) = (2 kh2 + pr - 1, 2 kw2 + pc - 1), zero in channels 12..15 and in the padding row and column of the 8x8
    kernel) in the tensor-core modes, the im2col row k = (kh*7+kw)*3 + c zero-padded to im2col_k = 192 in the CUDA-core
    modes.
  * tc_split: hi = fp16(clamp(x, +-65504)), lo = fp16(x_c - hi) (a NaN stays NaN in both), element (c, p) of a tap at
    ((c>>3)<<4) + (p<<3) + (c&7), hi in both plane slots of tap t and lo in both of tap KK + t; fprop rows [Co][KK][Ci]
    and dgrad rows [Ci][KK][Co] of the fp32 matrices, the stem as one tap of 256.
  * fp8: s = f8_pow2_scale(max |row|) (NaN ignored, as fmaxf), byte = e4m3 satfinite round-to-nearest-even of
    fp32(x * fp32(1/s)), s at s_w[conv * 512 + co]; the stem packed as bf16.
params_flat is Kaiming-scaled normal values with planted rows: bf16 and fp16 ties (normal and subnormal), fp32
subnormals and -0, |x| > 65504 (tc_split saturation), a NaN, +-inf, and the fp8 rows (zero row: scale 1; amax exactly
448 * 2^-12: m = 0.875 in f8_pow2_scale; one float above it; an infinity: 2^120; amax below 2^-118: clamped to 2^-126).
The edge rows sit in the LAST, short row group of convs of every k_pack_weights group size that leaves one (7 and 3).
Each pack runs twice, over outputs pre-filled with the bytes 0xA5 and 0x5A: every packed byte must be written (it
matches in both runs), and every byte outside the convs' ranges must keep the fill.  Stem layouts: fp32 / bf16_simt
run the im2col stem, bf16 / tc_split / fp8 the space-to-depth stem, and bf16 / tc_split also run the im2col stem they
fall back to when the driver rejects overlapped tensor maps (mapnet_test_pack_weights' im2col_stem).  Frames: 256x256
(the benchmark) and 256x341 (7Scenes).  The descriptors do not depend on the frame size (stem_s2d_geometry sets the same
WeightDesc fields for any frame; tests/test_pack_loss_host.py asserts the tables are equal), so the 7Scenes cases
confirm that no frame geometry leaks into the packs rather than test another layout.

Criterion (mapnet_loss_fwd_bwd, k_loss).  Reference: float64 autograd of oracle.mapnet_oracle.criterion on the same
float32 inputs.  u = 2^-24.  Bounds, per case (printed as max(err / bound)):
  * loss and ds4: each L1 sum S_k is a per-thread chain of at most 3 ceil(N Tp / 256) adds, 5 shuffle levels and the 8
    warp partials, so |fl(S_k) - S_k| <= (3 ceil(N Tp / 256) + 13) u sum|terms| plus the terms' own evaluation error
    e_d (abs: u |d|; mapnet rel: 2u (|p_i+1 - p_i| + |t_i+1 - t_i|) + u |d|, calc_vos_simple's three roundings;
    MapNet++ rel: the VO error below).  finalize: expf (2 ulp = 4u), the division by the count and the product (2u),
    then at most 8 adds of the terms e^-s A + s.
  * dpred, posenet / mapnet / online_gps: a sum of +-c (c = e^-s / count: expf and one division) over at most 3 terms:
    8u per coefficient.  Sign exception: a residual whose float64 value is within its float32 evaluation error e_d
    may take either sign (or 0), so 2c more (the absolute residuals p - t are exact in sign).
  * dpred, MapNet++ (online): the same for the absolute half; each VO pair (p0, p1) adds J^T g with g = c sgn(o - t):
    K_J u sum_m c_m |J_mk| for the float32 evaluation of the pose chain (J = d o / d (p0, p1) in float64), plus
    K_Q u (3 crq) / sin^2(theta) on the log q components of both poses, theta = |o_logq| the pair's relative rotation.
    The forward carries u / sin theta: qlog's acos of an fp32 c = cos(theta) that is off by a few u.  The backward
    carries one more 1 / sin theta: qlog_bwd's acos'(c) = -1/sqrt(1 - c^2) takes 1 - c^2 ~ sin^2 theta from fp32 c
    (relative error ~u / sin^2 theta on a gradient of size 1 / sin theta), and qmult_bwd's normalisation projects that
    q.s component back down by sin theta only, leaving ~u / sin^2 theta per unit of upstream gradient.  (Measured with
    the host shim of loss_core.h: K_Q ~ 0.7 at VO-sized theta; a u / sin theta term would need K ~ 400 there.)  The VO
    residual o - t itself is off by at most e_o = K_T u (|t0| + |t1| + |o_t|) (translation) and K_L u (1 + 1 / sin
    theta) (log q; measured K_T < 4, K_L < 8), the sign-exception window.  K_J = 32: the same host-shim fit, with every
    other term of the bound in place, needs K_J < 8 over the online cases (largest at large rotations).
    What the VO cases pin: at theta = 1e-3 the K_Q term is about 0.7 crq per log-q element, so there the relative-q
    gradient is checked only loosely; the "large" cases (theta of order 1, K_Q term ~1e-6 crq) pin it, and the VO cases
    pin the translation chain, the absolute terms and the sign handling at small residuals.
  The cases run the benchmark shapes (posenet N 64, mapnet N 32 T 3, online / online_gps N 16 T 10 = Tp 20), the
block-stride edges N Tp in {1, 255, 256, 257, 1024} (k_loss: one block of 256 threads), three settings of s4 and, for
MapNet++, VO-sized relative rotations (theta ~ 1e-3 .. 1e-2) and large ones.  dpred is NaN before the launch, so a pose
that no thread visits fails.

mapnet_batch_losses (k_batch_losses): ragged posenet / mapnet batches, one over 256 rows and one at the 200 KB shared
memory limit (4266 rows): every batch's loss is bit for bit mapnet_loss_fwd_bwd on that batch gathered, and within the
loss bound of the float64 reference.

mapnet_sqnorm: over the real flat-gradient length of a product PoseNet, with an aligned start and one 4 bytes off (the
scalar path), a tail that is not a multiple of 4.  Each of the 296 partials is a float64 sum rounded to fp32 once (u of
it), the final float64 sum of the partials rounded once more: |got - ref| <= (2u + n 2^-52) ref.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from geomapnet_b200 import _lib

U = 2.0 ** -24
PACK_PREC = {"fp32": 0, "bf16": 1, "bf16_simt": 2, "tc_split": 3, "fp8": 4}
TRUNK_PREC = {"fp32": "fp32", "bf16": "bf16", "bf16_simt": "bf16_simt", "tc_split": "tc_split", "fp8": "bf16"}
FRAMES = {"bench_256x256": (256, 256), "7scenes_256x341": (256, 341)}
# the stem layout each precision runs: the tensor-core training modes fall back to the im2col stem when the driver
# rejects overlapped tensor maps (net.cu: Net::init), the fp8 engine requires the space-to-depth one
STEM_LAYOUT = {"fp32": "im2col", "bf16_simt": "im2col", "bf16": "s2d", "tc_split": "s2d", "fp8": "s2d"}
PACK_CASES = [(f, m, STEM_LAYOUT[m]) for f in FRAMES for m in PACK_PREC] + \
    [("bench_256x256", m, "im2col") for m in ("bf16", "tc_split")]
FILLS = (0xA5, 0x5A)


def pack_group(n_in):
    """layout.cu: output channels per k_pack_weights block"""
    g = 4096 // max(n_in, 1)
    return min(max(g, 1), 8)


def weight_table(H, W, mode, stem=None):
    """[(p_off, k_off, Co, Ci, Ci_real, KH, KW, im2col_k, s2d)] and wk_total of mapnet_test_weight_table"""
    buf = (ctypes.c_int64 * 512)()
    _lib.check(_lib.lib().mapnet_test_weight_table(H, W, PACK_PREC[mode], int(stem == "im2col"), buf, 512),
               "mapnet_test_weight_table")
    n = buf[0]
    rows = [tuple(int(v) for v in buf[2 + 9 * i: 11 + 9 * i]) for i in range(n)]
    return rows, int(buf[1])


def conv_ne(row):
    """packed elements of one conv's KRSC matrix"""
    _, _, Co, Ci, _, KH, KW, im2col_k, _ = row
    return Co * (im2col_k if im2col_k > 0 else KH * KW * Ci)


def conv_numel(row):
    """elements of one conv's master weight in params_flat"""
    _, _, Co, Ci, Ci_real, KH, KW, im2col_k, _ = row
    return Co * Ci_real * (49 if im2col_k > 0 else KH * KW)


def param_entries(H, W, mode):
    """the trunk's parameter table: [(name, kind, shape, offset, layout)], n_params"""
    t = _lib.Trunk(0, H, W, 2048, TRUNK_PREC[mode])
    try:
        entries, n_params, _ = t.table()
        L = _lib.lib()
        out = [(nm, k, s, o, L.mapnet_param_layout(t.h, i)) for i, (nm, k, s, o) in enumerate(entries)]
    finally:
        t.close()
    return out, n_params


def table_invariants(H, W, mode, stem):
    """the descriptor table against the parameter table and itself; returns (rows, wk_total, n_params).  The parameter
    table is the one tests/test_host_surface.py and tests/test_checkpoint.py pin to models/posenet.py's parameters."""
    rows, wk = weight_table(H, W, mode, stem)
    entries, n_params = param_entries(H, W, mode)
    convs = [e for e in entries if e[1] == 0 and len(e[2]) == 4]
    assert len(rows) == len(convs) == 36
    # p_off: conv i is the i-th 4-d weight of the parameter table, in its order and size
    for r, (nm, _, shape, off, layout) in zip(rows, convs):
        assert r[0] == off, nm
        assert conv_numel(r) == int(np.prod(shape)), nm
        assert r[2] == shape[0] and r[4] == shape[1] and (r[7] > 0 or (r[5], r[6]) == tuple(shape[2:])), nm
        assert layout == (0 if r[7] > 0 else 1), nm          # the stem keeps torch's order, every other conv KRSC
    if stem == "s2d":
        assert rows[0][2:] == (64, 64, 3, 4, 1, 256, 1)
    else:
        assert rows[0][2:] == (64, 192, 3, 1, 1, 192, 0)
    for r in rows[1:]:
        assert r[7] == 0 and r[8] == 0 and r[3] == r[4] and r[5] == r[6] and r[5] in (1, 3)
        assert r[2] % 32 == 0 and r[3] % 32 == 0          # k_transpose_dg's 32 x 32 tiles, the float4 copies
    # every trainable parameter range lies in params_flat, none overlaps, the gaps are the 64-float alignment
    spans = sorted((o, o + int(np.prod(s)) if s else o + 1) for _, k, s, o, _ in entries if k == 0)
    assert spans[0][0] == 0
    for (a0, a1), (b0, _) in zip(spans, spans[1:]):
        assert a1 <= b0 and b0 - a1 < 64 and b0 % 64 == 0
    assert spans[-1][1] <= n_params < spans[-1][1] + 64
    # k_off: the convs' packed matrices tile [0, wk_total) in order, each 512-element aligned
    k = 0
    for r in rows:
        assert r[1] == k
        k += -(-conv_ne(r) // 512) * 512
    assert k == wk
    return rows, wk, n_params


# ---- planted rows ---------------------------------------------------------------------------------------------------
F32_SUB = np.array([1, 0x00012345, 0x807FFFFF], np.uint32).view(np.float32)       # 2^-149, subnormals, -subnormal
EDGE_VALUES = np.concatenate([
    np.array([1 + 2.0 ** -8, -(1 + 3 * 2.0 ** -8), 2.0 ** -126 * (1 + 2.0 ** -8),       # bf16 ties (normal)
              3 * 2.0 ** -134, 2.0 ** -134,                                              # bf16 ties (subnormal)
              1 + 2.0 ** -11, -(1 + 3 * 2.0 ** -11), 3 * 2.0 ** -25, -(2.0 ** -25),      # fp16 ties (normal, subnormal)
              (1 + 2.0 ** -11) * 2.0 ** -14 + 2.0 ** -36,                                 # fp16: lo plane carries a tie
              -0.0, 7.0e4, -1.0e5, 65504.0, 65520.0, np.nan, 1e-40], np.float32),
    F32_SUB]).astype(np.float32)
F8_AMAX = np.float32(448.0 * 2.0 ** -12)


def short_group_rows(rows):
    """{group size G: (conv, first row of its last, short group)} for every G whose convs end in a short group"""
    out = {}
    for i, r in enumerate(rows[1:], start=1):
        G = pack_group(r[5] * r[6] * r[3])
        if r[2] % G:
            out.setdefault(G, (i, r[2] - r[2] % G))
    return out


def plant_rows(rows):
    """[(conv, row, kind)]: the edge rows (one in the stem, one in the last short group of every group size that
    leaves one, one in a G = 1 and one in a G = 8 conv) and the fp8 scale rows (conv 2)"""
    plants = [(0, 5, "edges")]
    for G, (i, r0) in sorted(short_group_rows(rows).items()):
        plants += [(i, co, "edges") for co in sorted({r0, rows[i][2] - 1})]
    g1 = next(i for i, r in enumerate(rows[1:], 1) if pack_group(r[5] * r[6] * r[3]) == 1)
    g8 = next(i for i, r in enumerate(rows[1:], 1) if pack_group(r[5] * r[6] * r[3]) == 8)
    plants += [(g1, rows[g1][2] - 1, "edges"), (g8, 3, "edges")]
    plants += [(2, 0, "f8_zero"), (2, 1, "f8_amax_448"), (2, 2, "f8_above_448"), (2, 3, "f8_inf"), (2, 4, "f8_tiny")]
    return plants


def make_params(rows, n_params, seed=0):
    """Kaiming-scaled normal master weights (other parameters N(0, 0.02)) with the planted rows"""
    g = np.random.default_rng(seed)
    p = (g.standard_normal(n_params) * 0.02).astype(np.float32)
    for r in rows:
        n = conv_numel(r)
        fan_in = n // r[2]
        p[r[0]: r[0] + n] = (g.standard_normal(n) * math.sqrt(2.0 / fan_in)).astype(np.float32)
    for i, co, kind in plant_rows(rows):
        n = conv_numel(rows[i]) // rows[i][2]
        row = p[rows[i][0] + co * n: rows[i][0] + (co + 1) * n]
        if kind == "edges":
            pos = g.choice(n, size=len(EDGE_VALUES), replace=False)
            row[pos] = EDGE_VALUES
        elif kind == "f8_zero":
            row[:] = 0.0
            row[::7] = -0.0
        elif kind in ("f8_amax_448", "f8_above_448"):
            row[:] = np.clip(row, -0.1, 0.1)
            row[n // 2] = F8_AMAX if kind == "f8_amax_448" else np.nextafter(F8_AMAX, np.float32(1))
            row[n // 3] = -F8_AMAX
        elif kind == "f8_inf":
            row[n // 2] = np.inf
            row[n // 5] = -np.inf
        elif kind == "f8_tiny":
            row[:] = (row * 2.0 ** -121).astype(np.float32)       # |x| < 2^-118: normal and subnormal fp32
    return p


# ---- numpy references of the packs ----------------------------------------------------------------------------------
def stem_index(stem):
    """for each k of the stem's packed row: the flat index c*49 + kh*7 + kw into the [3][7][7] slab, or -1"""
    if stem == "s2d":
        idx = np.full(256, -1, np.int64)
        for k in range(256):
            kh2, kw2, ch = k >> 6, (k >> 4) & 3, k & 15
            if ch < 12:
                q, c = ch // 3, ch % 3
                kh, kw = 2 * kh2 + (q >> 1) - 1, 2 * kw2 + (q & 1) - 1
                if 0 <= kh < 7 and 0 <= kw < 7:
                    idx[k] = c * 49 + kh * 7 + kw
        return idx
    idx = np.full(192, -1, np.int64)
    for k in range(147):
        t, c = k // 3, k % 3
        idx[k] = c * 49 + t
    return idx


def bf16_bits(x):
    """round to nearest even fp32 -> bf16 bit patterns (NaN handled by the caller)"""
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def f16_split(x):
    """(hi, lo) fp16 bit patterns of split_f16"""
    c = np.clip(x, np.float32(-65504.0), np.float32(65504.0)).astype(np.float32)
    hi = c.astype(np.float16)
    lo = (c - hi.astype(np.float32)).astype(np.float16)
    return hi.view(np.uint16), lo.view(np.uint16)


def split_layout(hi, lo, R, KK, C):
    """[R][KK][C] hi / lo -> [R][2KK][2C] in the 8-interleaved plane order"""
    h = hi.reshape(R, KK, C // 8, 1, 8)
    l = lo.reshape(R, KK, C // 8, 1, 8)
    out = np.empty((R, 2, KK, C // 8, 2, 8), np.uint16)
    out[:, 0] = h
    out[:, 1] = l
    return out.reshape(-1)


def f8_pow2_scale(amax):
    """common.cuh f8_pow2_scale restated"""
    a = np.float32(amax)
    if not a > 0:
        return np.float32(1.0)
    if not np.isfinite(a):
        return np.float32(2.0 ** 120)
    m, k = np.frexp(a)
    e = k - 9 if m <= np.float32(0.875) else k - 8
    return np.float32(2.0 ** max(int(e), -126))


def e4m3_bytes(x):
    """e4m3 satfinite round-to-nearest-even bytes of float32 values (NaN -> 0x7F / 0xFF)"""
    from fp8_emulation import e4m3_rne_satfinite_numpy
    r = e4m3_rne_satfinite_numpy(x)
    return torch.from_numpy(r).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


class Expect(object):
    """expected contents of one output buffer: element bit patterns where written, a mask of written elements and a
    mask of elements that must be NaN (any payload)"""

    def __init__(self, n, dtype):
        self.ref = np.zeros(n, dtype)
        self.written = np.zeros(n, bool)
        self.nan = np.zeros(n, bool)

    def put(self, off, bits, nan):
        self.ref[off: off + bits.size] = bits
        self.written[off: off + bits.size] = True
        self.nan[off: off + bits.size] = nan


def reference_packs(params, rows, wk, mode, stem):
    """{output name: Expect} for one precision"""
    stem_idx = stem_index(stem)
    k32, d32 = [], []          # per conv: fp32 KRSC matrix [R][KK][C] (rows, KK, C) and dgrad matrix (or None)
    for i, r in enumerate(rows):
        p_off, k_off, Co, Ci, Ci_real, KH, KW, im2col_k, s2d = r
        src = params[p_off: p_off + conv_numel(r)]
        if im2col_k > 0:
            slab = src.reshape(Co, Ci_real * 49)
            m = np.where(stem_idx[None, :] >= 0, slab[:, np.maximum(stem_idx, 0)], np.float32(0)).astype(np.float32)
            k32.append((m.reshape(-1), Co, 1, im2col_k))
            d32.append(None)
        else:
            KK = KH * KW
            k32.append((src, Co, KK, Ci))
            d32.append((np.ascontiguousarray(src.reshape(Co, KK, Ci).transpose(2, 1, 0)).reshape(-1), Ci, KK, Co))
    out = {}
    if mode in ("fp32", "bf16_simt", "bf16"):
        dt = np.uint16 if mode == "bf16" else np.uint32
        for name, mats in (("krsc", k32), ("dg", d32)):
            e = Expect(wk, dt)
            for r, m in zip(rows, mats):
                if m is None:
                    continue
                v = m[0]
                if mode == "fp32":
                    bits = v.view(np.uint32)
                else:
                    b = bf16_bits(v)
                    bits = b if mode == "bf16" else b.astype(np.uint32) << 16
                e.put(r[1], bits, np.isnan(v))
            out[name] = e
    elif mode == "tc_split":
        for name, mats in (("krsc", k32), ("dg", d32)):
            e = Expect(4 * wk, np.uint16)
            for r, m in zip(rows, mats):
                if m is None:
                    continue
                v, R, KK, C = m
                hi, lo = f16_split(v)
                nan = np.isnan(v).reshape(R, KK, C)
                nn = split_layout(nan.reshape(-1).astype(np.uint16), nan.reshape(-1).astype(np.uint16), R, KK, C)
                e.put(4 * r[1], split_layout(hi, lo, R, KK, C), nn.astype(bool))
            out[name] = e
    else:      # fp8
        e8 = Expect(wk, np.uint8)
        sw = Expect(len(rows) * 512, np.uint32)
        for i, r in enumerate(rows[1:], start=1):
            v = k32[i][0].reshape(r[2], -1)
            amax = np.fmax.reduce(np.abs(v), axis=1)
            s = np.array([f8_pow2_scale(a) for a in amax], np.float32)
            inv = (np.float32(1.0) / s).astype(np.float32)
            q = (v * inv[:, None]).astype(np.float32)
            e8.put(r[1], e4m3_bytes(q.reshape(-1)), np.isnan(q.reshape(-1)))
            sw.put(i * 512, s.view(np.uint32), np.zeros(r[2], bool))
        stem = Expect(rows[1][1], np.uint16)
        stem.put(0, bf16_bits(k32[0][0]), np.isnan(k32[0][0]))
        out.update(krsc=e8, dg=stem, s_w=sw)
    return out


def check_expect(name, got, e, fill, fp16=False):
    """got: uint element array of the whole buffer after a launch over the fill byte"""
    fill_val = np.frombuffer(bytes([fill]) * got.dtype.itemsize, got.dtype)[0]
    untouched = ~e.written
    assert np.all(got[untouched] == fill_val), "%s: %d elements written outside the convs' ranges (fill %#x)" % (
        name, int(np.sum(got[untouched] != fill_val)), fill)
    ok = e.written & ~e.nan
    bad = np.flatnonzero(ok & (got != e.ref))
    assert bad.size == 0, "%s: %d elements differ (fill %#x), first at %d: got %#x want %#x" % (
        name, bad.size, fill, bad[0], int(got[bad[0]]), int(e.ref[bad[0]]))
    gn = got[e.nan]
    if got.dtype == np.uint32:
        isn = np.isnan(gn.view(np.float32))
    elif got.dtype == np.uint16:
        isn = ((gn & 0x7C00) == 0x7C00) & ((gn & 0x3FF) != 0) if fp16 else ((gn & 0x7F80) == 0x7F80) & ((gn & 0x7F) != 0)
    else:
        isn = (gn & 0x7F) == 0x7F
    assert np.all(isn), "%s: a NaN input did not stay NaN (fill %#x)" % (name, fill)
    return int(np.sum(e.written))


@pytest.mark.gpu
@pytest.mark.parametrize("frame,mode,stem", PACK_CASES)
def test_whole_network_pack_bit_for_bit(frame, mode, stem):
    H, W = FRAMES[frame]
    rows, wk, n_params = table_invariants(H, W, mode, stem)
    params = make_params(rows, n_params)
    ref = reference_packs(params, rows, wk, mode, stem)
    dev = torch.from_numpy(params).cuda()
    L = _lib.lib()
    for fill in FILLS:
        bufs = {n: torch.full((e.ref.size * e.ref.itemsize,), fill, dtype=torch.uint8, device="cuda")
                for n, e in ref.items()}
        _lib.check(L.mapnet_test_pack_weights(PACK_PREC[mode], int(stem == "im2col"), H, W, dev.data_ptr(),
                                              bufs["krsc"].data_ptr(), bufs["dg"].data_ptr(),
                                              bufs["s_w"].data_ptr() if "s_w" in bufs else None, _lib.stream_ptr()),
                   "mapnet_test_pack_weights")
        torch.cuda.synchronize()
        n = 0
        for name, e in ref.items():
            got = bufs[name].cpu().numpy().view(e.ref.dtype)
            n += check_expect("%s %s %s" % (frame, mode, name), got, e, fill, fp16=(mode == "tc_split"))
    print("pack %s %s: %d elements bit for bit, stem %s" % (frame, mode, n, stem))


# ---- criterion --------------------------------------------------------------------------------------------------------
LOSS_MODE = _lib.LOSS_MODE
S4 = {"s0": (0.0, -3.0, 0.0, -3.0), "s1": (0.3, -2.0, 0.1, -1.5), "s2": (-4.0, 2.0, 3.0, -6.0)}
K_T, K_L, K_J, K_Q = 16.0, 16.0, 32.0, 4.0

# (id, mode, N, Tp, s4 key, rotation regime): "vo" relative rotations of 1e-3 .. 1e-2 rad, "large" of order 1
CRIT_CASES = []
for _s in S4:
    CRIT_CASES += [("posenet_n64", "posenet", 64, 1, _s, "large"), ("mapnet_n32t3", "mapnet", 32, 3, _s, "large"),
                   ("online_n16t10_vo", "online", 16, 20, _s, "vo"), ("online_n16t10_large", "online", 16, 20, _s, "large"),
                   ("online_gps_n16t10", "online_gps", 16, 20, _s, "vo")]
CRIT_CASES += [
    ("posenet_n1", "posenet", 1, 1, "s1", "large"), ("posenet_n255", "posenet", 255, 1, "s2", "large"),
    ("posenet_n256", "posenet", 256, 1, "s0", "large"), ("posenet_n257", "posenet", 257, 1, "s1", "large"),
    ("posenet_n1024", "posenet", 1024, 1, "s2", "large"),
    ("mapnet_n85t3", "mapnet", 85, 3, "s1", "large"), ("mapnet_n128t2", "mapnet", 128, 2, "s2", "large"),
    ("mapnet_n1t257", "mapnet", 1, 257, "s0", "large"), ("mapnet_n256t4", "mapnet", 256, 4, "s1", "large"),
    ("online_n16t8", "online", 16, 16, "s2", "vo"), ("online_n1t128", "online", 1, 256, "s1", "large"),
    ("online_n43t3", "online", 43, 6, "s0", "vo"), ("online_n64t8", "online", 64, 16, "s1", "vo"),
    ("online_gps_n128t1", "online_gps", 128, 2, "s1", "large"), ("online_gps_n1t128", "online_gps", 1, 256, "s2", "vo"),
    ("online_gps_n257t1", "online_gps", 257, 2, "s0", "vo"), ("online_gps_n32t16", "online_gps", 32, 32, "s1", "large"),
]


def _qexp64(l):
    n = np.maximum(np.linalg.norm(l, axis=-1, keepdims=True), 1e-12)
    return np.concatenate([np.cos(n), l * np.sin(n) / n], -1)


def make_crit_inputs(mode, N, Tp, regime, seed):
    """float32 pred [N, Tp, 6] and targ [N, Tt, 6]"""
    g = np.random.default_rng(seed)
    t = np.cumsum(g.standard_normal((N, Tp, 3)) * 0.3, axis=1) + g.standard_normal((N, 1, 3)) * 2.0
    if regime == "vo":
        step = g.standard_normal((N, Tp, 3))
        step *= (g.uniform(1e-3, 1e-2, (N, Tp, 1)) / np.linalg.norm(step, axis=-1, keepdims=True))
        l = np.cumsum(step, axis=1) + g.standard_normal((N, 1, 3)) * 0.3
    else:
        l = g.standard_normal((N, Tp, 3)) * 0.8
    pred = np.concatenate([t, l], -1).astype(np.float32)
    scale = np.array([0.2] * 3 + [0.02 if regime == "large" else 2e-3] * 3)
    if mode in ("posenet", "mapnet"):
        targ = pred + g.standard_normal(pred.shape) * scale
        if mode == "posenet":
            return pred.reshape(N, 6), targ.astype(np.float32).reshape(N, 6)
        return pred, targ.astype(np.float32)
    T = Tp // 2
    targ_abs = pred[:, :T] + g.standard_normal((N, T, 6)) * scale
    if mode == "online_gps":
        targ_v = pred[:, T:] + g.standard_normal((N, T, 6)) * scale
    else:
        from oracle import mapnet_oracle as O
        pv = torch.from_numpy(pred[:, T:].astype(np.float64))
        vo = O.calc_vos(pv).numpy()
        vscale = np.array([0.05] * 3 + [5e-3 if regime == "vo" else 0.02] * 3)
        targ_v = vo + g.standard_normal(vo.shape) * vscale
    return pred, np.concatenate([targ_abs, targ_v], 1).astype(np.float32)


def crit_reference(mode, pred, targ, s4):
    """float64 autograd: loss, dpred, ds4"""
    from oracle import mapnet_oracle as O
    p = torch.from_numpy(pred.astype(np.float64)).requires_grad_(True)
    tt = torch.from_numpy(targ.astype(np.float64))
    sv = [torch.tensor([float(np.float32(v))], dtype=torch.float64, requires_grad=True) for v in s4]
    L = O.criterion(mode, p, tt, dict(sax=sv[0], saq=sv[1], srx=sv[2], srq=sv[3]))
    L.backward()
    ds = [float(v.grad) if v.grad is not None else 0.0 for v in sv]
    return L.item(), p.grad.numpy(), np.array(ds)


def _vo64(p0, p1):
    """float64 calc_vo_logq on rows [P, 6] and its Jacobian |d o / d (p0, p1)| [P, 6, 12]"""
    from oracle import mapnet_oracle as O
    a = torch.from_numpy(p0).requires_grad_(True)
    b = torch.from_numpy(p1).requires_grad_(True)
    o = O.calc_vo_logq(a, b)
    J = np.zeros((p0.shape[0], 6, 12))
    for m in range(6):
        ga, gb = torch.autograd.grad(o[:, m].sum(), (a, b), retain_graph=True)
        J[:, m, :6] = ga.numpy()
        J[:, m, 6:] = gb.numpy()
    return o.detach().numpy(), np.abs(J)


def crit_bounds(mode, pred, targ, s4):
    """(bound on |loss - ref|, bound per ds4 [4], bound per dpred element), from the float32 inputs"""
    N = pred.shape[0]
    P = pred.reshape(N, -1, 6).astype(np.float64)
    Tg = targ.reshape(N, -1, 6).astype(np.float64)
    Tp = P.shape[1]
    s = np.array([np.float32(v) for v in s4], np.float64)
    if mode == "posenet":
        cnt = [3.0 * N, 3.0 * N, 0, 0]
    elif mode == "mapnet":
        cnt = [3.0 * N * Tp] * 2 + [3.0 * N * (Tp - 1)] * 2
    else:
        T = Tp // 2
        cnt = [3.0 * N * T] * 2 + ([3.0 * N * (T - 1)] * 2 if mode == "online" else [2.0 * N * T, 0])
    c = np.array([math.exp(-s[k]) / cnt[k] if cnt[k] else 0.0 for k in range(4)])
    A = np.zeros(4)         # sums of |terms|
    E = np.zeros(4)         # sums of the terms' evaluation errors
    bd = np.zeros_like(P)   # dpred bound
    T_abs = Tp if mode in ("posenet", "mapnet") else Tp // 2
    d = P[:, :T_abs] - Tg[:, :T_abs]
    for k, sl in ((0, slice(0, 3)), (1, slice(3, 6))):
        A[k] += np.abs(d[..., sl]).sum()
        E[k] += U * np.abs(d[..., sl]).sum()
        bd[:, :T_abs, sl] += 8 * U * c[k]
    if mode == "mapnet":
        dv = (P[:, 1:] - P[:, :-1]) - (Tg[:, 1:] - Tg[:, :-1])
        ed = 2 * U * (np.abs(P[:, 1:] - P[:, :-1]) + np.abs(Tg[:, 1:] - Tg[:, :-1]))
        for k, sl in ((2, slice(0, 3)), (3, slice(3, 6))):
            A[k] += np.abs(dv[..., sl]).sum()
            E[k] += (ed[..., sl] + U * np.abs(dv[..., sl])).sum()
            w = c[k] * (8 * U + 2.0 * (np.abs(dv[..., sl]) <= ed[..., sl]))
            bd[:, 1:, sl] += w
            bd[:, :-1, sl] += w
    elif mode == "online_gps":
        dv = P[:, T_abs:, :2] - Tg[:, T_abs:, :2]
        A[2] += np.abs(dv).sum()
        E[2] += U * np.abs(dv).sum()
        bd[:, T_abs:, :2] += 8 * U * c[2]
    elif mode == "online":
        T = T_abs
        p0 = P[:, T:-1].reshape(-1, 6)
        p1 = P[:, T + 1:].reshape(-1, 6)
        o, J = _vo64(p0, p1)
        tv = Tg[:, T:].reshape(-1, 6)
        dv = o - tv
        theta = np.linalg.norm(o[:, 3:], axis=1)
        sinv = 1.0 / np.maximum(np.sin(np.minimum(theta, math.pi - 1e-7)), 1e-7)
        eo = np.zeros_like(o)
        eo[:, :3] = K_T * U * (np.linalg.norm(p0[:, :3], axis=1) + np.linalg.norm(p1[:, :3], axis=1)
                               + np.linalg.norm(o[:, :3], axis=1))[:, None]
        eo[:, 3:] = K_L * U * (1.0 + sinv)[:, None]
        cm = np.array([c[2]] * 3 + [c[3]] * 3)
        A[2] += np.abs(dv[:, :3]).sum()
        A[3] += np.abs(dv[:, 3:]).sum()
        E[2] += eo[:, :3].sum()
        E[3] += eo[:, 3:].sum()
        flip = (np.abs(dv) <= eo) * 2.0 * cm                       # [P, 6]
        pair = K_J * U * np.einsum("pm,pmk->pk", np.broadcast_to(cm, dv.shape), J) + np.einsum("pm,pmk->pk", flip, J)
        pair[:, 3:6] += K_Q * U * 3 * c[3] * (sinv ** 2)[:, None]
        pair[:, 9:12] += K_Q * U * 3 * c[3] * (sinv ** 2)[:, None]
        pair = pair.reshape(N, T - 1, 12)
        bd[:, T:-1] += pair[..., :6]
        bd[:, T + 1:] += pair[..., 6:]
    depth = 3 * -(-N * Tp // 256) + 13
    errS = depth * U * A + E                    # |fl(S_k) - S_k|
    terms = c * A                               # e^-s S / count
    berr = terms * 6 * U + c * errS
    b_loss = berr.sum() + 8 * U * (np.abs(terms).sum() + np.abs(s).sum())
    b_ds = berr + U * np.abs(1.0 - terms)
    return b_loss, b_ds, bd.reshape(pred.shape)


def run_loss(mode, pred, targ, s4):
    N = pred.shape[0]
    Tp = 1 if pred.ndim == 2 else pred.shape[1]
    Tt = 1 if targ.ndim == 2 else targ.shape[1]
    p = torch.from_numpy(pred).cuda()
    t = torch.from_numpy(targ).cuda()
    s = torch.tensor(s4, dtype=torch.float32, device="cuda")
    loss = torch.full((1,), float("nan"), device="cuda")
    dpred = torch.full_like(p, float("nan"))
    ds = torch.full((4,), float("nan"), device="cuda")
    _lib.check(_lib.lib().mapnet_loss_fwd_bwd(LOSS_MODE[mode], p.data_ptr(), t.data_ptr(), N, Tp, Tt, s.data_ptr(),
                                              loss.data_ptr(), dpred.data_ptr(), ds.data_ptr(), _lib.stream_ptr()),
               "mapnet_loss_fwd_bwd")
    return float(loss.cpu()), dpred.cpu().numpy(), ds.cpu().numpy()


def crit_case_inputs(case):
    cid, mode, N, Tp, skey, regime = case
    seed = 1000 + CRIT_CASES.index(case)
    pred, targ = make_crit_inputs(mode, N, Tp, regime, seed)
    return mode, pred, targ, S4[skey]


def check_criterion(got, ref, bounds, mode):
    """max(err / bound) of loss, ds4 and dpred; fails on any excess"""
    (gl, gd, gs), (rl, rd, rs), (bl, bs, bd) = got, ref, bounds
    assert np.all(np.isfinite(gd)), "dpred has NaN: a pose no thread wrote"
    n_s = 2 if mode == "posenet" else (3 if mode == "online_gps" else 4)
    r_loss = abs(gl - rl) / bl
    r_ds = max(abs(gs[k] - rs[k]) / bs[k] for k in range(n_s))
    assert all(gs[k] == 0.0 for k in range(n_s, 4))
    err = np.abs(gd.astype(np.float64) - rd)
    assert np.all(err[bd == 0] == 0), "a gradient the criterion does not reach is not 0"
    r_d = float(np.max(err[bd > 0] / bd[bd > 0]))
    assert r_loss <= 1.0, (gl, rl, bl)
    assert r_ds <= 1.0, (gs, rs, bs)
    assert r_d <= 1.0, r_d
    return r_loss, r_ds, r_d


@pytest.mark.gpu
@pytest.mark.parametrize("case", CRIT_CASES, ids=["%s.%s" % (c[0], c[4]) for c in CRIT_CASES])
def test_fused_criterion_vs_float64(case):
    mode, pred, targ, s4 = crit_case_inputs(case)
    got = run_loss(mode, pred, targ, s4)
    ref = crit_reference(mode, pred, targ, s4)
    r = check_criterion(got, ref, crit_bounds(mode, pred, targ, s4), mode)
    print("criterion %s.%s: max err/bound loss %.3g ds4 %.3g dpred %.3g" % (case[0], case[4], r[0], r[1], r[2]))


# ---- validation batch losses ------------------------------------------------------------------------------------------
MAX_BATCH_ROWS = 200 * 1024 // 48           # mapnet_batch_losses: [rows][6] pred + targ in 200 KB of shared memory
# (id, mode, T, batch sizes in items)
BATCH_CASES = [("posenet_ragged", "posenet", 1, [64, 1, 300, 257, 7, MAX_BATCH_ROWS]),
               ("mapnet_ragged", "mapnet", 3, [32, 2, 86, 1, MAX_BATCH_ROWS // 3, 100])]


@pytest.mark.gpu
@pytest.mark.parametrize("case", BATCH_CASES, ids=[c[0] for c in BATCH_CASES])
@pytest.mark.parametrize("skey", ["s0", "s1"])
def test_batch_losses_bitwise_and_vs_float64(case, skey):
    cid, mode, T, sizes = case
    s4 = S4[skey]
    g = np.random.default_rng(7)
    items = int(sum(sizes))
    n_rows = items * T + 11
    pred, targ = make_crit_inputs("mapnet", 1, n_rows, "large", 11)
    pred, targ = pred[0], targ[0]
    # each item's T rows: a random window of consecutive rows (MapNet: a sequence), stored in permuted order
    starts = g.integers(0, n_rows - T + 1, items)
    rows = (starts[:, None] + np.arange(T)[None, :]).reshape(-1).astype(np.int32)
    pperm = g.permutation(n_rows).astype(np.int32)
    tperm = g.permutation(n_rows).astype(np.int32)
    pstore = np.empty_like(pred)
    tstore = np.empty_like(targ)
    pstore[pperm] = pred
    tstore[tperm] = targ
    prow = pperm[rows]
    trow = tperm[rows]
    bi = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    dp = torch.from_numpy(pstore).cuda()
    dt = torch.from_numpy(tstore).cuda()
    s = torch.tensor(s4, dtype=torch.float32, device="cuda")
    losses = torch.full((len(sizes),), float("nan"), device="cuda")
    I32 = ctypes.POINTER(ctypes.c_int32)
    _lib.check(_lib.lib().mapnet_batch_losses(
        LOSS_MODE[mode], dp.data_ptr(), n_rows, dt.data_ptr(), n_rows, prow.ctypes.data_as(I32),
        trow.ctypes.data_as(I32), T, bi.ctypes.data_as(I32), len(sizes), s.data_ptr(), losses.data_ptr(),
        _lib.stream_ptr()), "mapnet_batch_losses")
    got = losses.cpu().numpy()
    worst = 0.0
    for b in range(len(sizes)):
        r = rows[bi[b] * T: bi[b + 1] * T]
        bp = pred[r].reshape(sizes[b], T, 6)
        bt = targ[r].reshape(sizes[b], T, 6)
        if mode == "posenet":
            bp, bt = bp.reshape(-1, 6), bt.reshape(-1, 6)
        one, _, _ = run_loss(mode, np.ascontiguousarray(bp), np.ascontiguousarray(bt), s4)
        assert np.float32(got[b]).tobytes() == np.float32(one).tobytes(), (b, got[b], one)
        rl, _, _ = crit_reference(mode, bp, bt, s4)
        bl, _, _ = crit_bounds(mode, bp, bt, s4)
        worst = max(worst, abs(float(got[b]) - rl) / bl)
        assert abs(float(got[b]) - rl) <= bl, (b, got[b], rl, bl)
    print("batch_losses %s %s: %d batches bitwise, max err/bound %.3g" % (cid, skey, len(sizes), worst))


# ---- clip norm --------------------------------------------------------------------------------------------------------
def flat_grad_len():
    """the flat gradient length of a product PoseNet (its parameter table's n_params)"""
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet
    net = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False, precision="bf16")
    return int(net._n_params)


def sqnorm_buffer(n_full, start, trim, seed):
    """(buffer, n, planted positions): n_full + 8 float32 values of many magnitudes, the sum taken over
    [start, start + n), n = n_full - trim.  Values far above the bound sit where an edge mistake would land: the first
    element, the last 4 (the vector path's scalar tail is n mod 4 of them), the element just past the end and the one
    just before the start -- so a dropped head or tail, or a read past either end, moves the sum by many bounds."""
    n = n_full - trim
    g = np.random.default_rng(seed)
    buf = (g.standard_normal(n_full + 8) * np.exp(g.uniform(-8, 3, n_full + 8))).astype(np.float32)
    base = float(np.dot(buf.astype(np.float64), buf.astype(np.float64)))
    pos = sorted({start, start + n - 4, start + n - 3, start + n - 2, start + n - 1, start + n} |
                 ({start - 1} if start > 0 else set()))
    for k, q in enumerate(pos):
        buf[q] = np.float32(math.sqrt(1e-3 * base) * (1.0 + k / 8.0) * (-1) ** k)
    return buf, n, pos


@pytest.mark.gpu
@pytest.mark.parametrize("start,trim", [(0, 0), (1, 0), (0, 3), (3, 1), (4, 2), (0, 1), (4, 3)])
def test_sqnorm_vs_float64(start, trim):
    buf, n, pos = sqnorm_buffer(flat_grad_len(), start, trim, start * 10 + trim)
    dev = torch.from_numpy(buf).cuda()
    assert dev.data_ptr() % 16 == 0         # start 0 / 4: the float4 path with its scalar tail; 1 / 3: the scalar path
    scratch = torch.zeros(1024, device="cuda")
    out = torch.full((1,), float("nan"), device="cuda")
    ptr = dev.data_ptr() + 4 * start
    _lib.check(_lib.lib().mapnet_sqnorm(ptr, n, scratch.data_ptr(), out.data_ptr(), _lib.stream_ptr()), "mapnet_sqnorm")
    got = float(out.cpu())
    x = buf[start: start + n].astype(np.float64)
    ref = float(np.dot(x, x))
    bound = (2 * U + n * 2.0 ** -52) * ref
    # each planted square is thousands of bounds: losing one, or reading one outside the range, cannot pass
    assert min(float(buf[q]) ** 2 for q in pos) > 1000 * bound
    print("sqnorm n %d (n mod 4 = %d) start +%d floats: err/bound %.3g" % (n, n % 4, start, abs(got - ref) / bound))
    assert abs(got - ref) <= bound
