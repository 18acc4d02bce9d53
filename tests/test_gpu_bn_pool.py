"""The element-wise kernels of the training step, one launch sequence at a time, against float64.

bn.cu: k_channel_sums (batch statistics and the backward reductions, last-block finalize), k_bn_eval_scale, k_bn_apply,
k_bn_bwd_apply (with and without the lazy finalize of accumulated sums), k_stem_pool, k_stem_pool_bwd[_quad],
k_bn_bwd_finalize_accum; head.cu: k_gap, k_gap_bwd -- through the mapnet_test_bn_* / mapnet_test_stem_pool /
mapnet_test_gap entry points, in every storage mode (fp32, bf16, bf16_simt, tc_split; e4m3 for the inference pool).

The references are float64, computed from the DECODED stored inputs (bf16 through torch, the tc_split hi/lo fp16 planes
decoded here).  Element-wise outputs are checked against the reference with the kernels' own fp32 per-channel parameters
(which are checked against float64 separately), so that a per-channel error and an element-wise error are both seen.

Bounds are per element and derived from the storage formats; u = 2^-24 is fp32's unit roundoff:
 * fp32 arithmetic: an expression of k roundings whose terms have magnitudes summing to T is off by at most k*u*T; the
   apply kernels round at most 3 times per output (scale*y + shift, the residual's own affine map, the add), hence
   e = 2^-22 * T with T = |scale*y| + |shift| + |res| (+ |scale2*y2| + |shift2|).
 * stored fp32: |got - ref| <= e.  Stored bf16 / e4m3: got lies between the format's round-to-nearest-even of ref - e
   and of ref + e (rounding is monotonic; the bracket ends are widened by 2^-23 |ref| for their own conversion to fp32).
   Stored hi/lo fp16 planes: |got - ref| <= e + 2^-22 (|ref| + e) + 2^-25 (the split's absolute error, common.cuh).
 * ReLU gates are evaluated in fp32, so an element whose float64 pre-activation lies within 2^-20 * T of zero (4x the
   arithmetic bound) is ambiguous and either branch is accepted there; fewer than 1e-4 of the elements may be ambiguous.
   Elements whose gate is surely closed must hold exact zeros.
 * per-channel sums accumulated in fp32 over n terms per thread and then over r rows of a block (k_channel_sums, the
   quad pool backward) are off by at most (n + r + 1) * u * sum|terms| (recursive summation; +1 for the product);
   fp64 sums (lazy replicas, fp64 atomics) by far less than 2^-40 * sum|terms|.  From there the finalize formulas are
   propagated to first order (the mean / variance cancellation E[y^2] - m^2 included), plus one fp32 rounding of each
   stored result.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fp8_emulation import quantize_e4m3
from geomapnet_b200 import _lib

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DEV = "cuda"
# rows of the per-BatchNorm state (include/mapnet_b200.h)
GAMMA, BETA, RMEAN, RVAR, MEAN, INVSTD, SCALE, SHIFT, MSCALE, MSHIFT, DGAMMA, DBETA, COEF = range(13)
NROWS = 15
# storage format of (conv outputs / fp32-math tensors, forward conv operands, backward conv operands) per precision
FMT = {"fp32": ("f32", "f32", "f32"), "bf16": ("bf16", "bf16", "bf16"), "bf16_simt": ("bf16", "bf16", "bf16"),
       "tc_split": ("f32", "hsplit", "hsplit")}
PRECS = list(FMT)
NUM_SMS = 132


# ---------------------------------------------------------------------------------------------------------------------
# storage formats
# ---------------------------------------------------------------------------------------------------------------------
def encode(x, fmt):
    """float64 device tensor [..., C] -> (the stored tensor a kernel reads, its decoded float64 value)"""
    if fmt == "f32":
        t = x.float()
        return t, t.double()
    if fmt == "bf16":
        t = x.bfloat16()
        return t, t.double()
    assert fmt == "hsplit"
    xf = x.float()
    hi = xf.half()
    lo = (xf - hi.float()).half()
    lead, C = x.shape[:-1], x.shape[-1]
    t = torch.stack((hi.reshape(*lead, C // 8, 8), lo.reshape(*lead, C // 8, 8)), -2).reshape(*lead, 2 * C)
    return t.contiguous(), hi.double() + lo.double()


def decode(t, fmt):
    if fmt == "hsplit":       # per 8 channels: 8 hi then 8 lo fp16 values (common.cuh, hsplit)
        v = t.reshape(*t.shape[:-1], t.shape[-1] // 16, 2, 8).double()
        return (v[..., 0, :] + v[..., 1, :]).reshape(*t.shape[:-1], t.shape[-1] // 2)
    if fmt == "e4m3":
        return t.view(torch.float8_e4m3fn).double()
    return t.double()


def empty(shape, fmt):
    """an output buffer full of NaN: an element the kernel does not write fails every check"""
    if fmt == "hsplit":
        return torch.full((*shape[:-1], 2 * shape[-1]), float("nan"), dtype=torch.float16, device=DEV)
    if fmt == "e4m3":
        return torch.full(shape, 0x7f, dtype=torch.uint8, device=DEV)      # e4m3 NaN
    return torch.full(shape, float("nan"), dtype=torch.float32 if fmt == "f32" else torch.bfloat16, device=DEV)


def stored_ok(got, ref, e, fmt):
    """got (decoded) is the stored form of a fp32 value within e of ref"""
    if fmt == "f32":
        return (got - ref).abs() <= e
    if fmt == "hsplit":
        return (got - ref).abs() <= e + 2.0 ** -22 * (ref.abs() + e) + 2.0 ** -25
    q = (lambda v: v.float().bfloat16().double()) if fmt == "bf16" else (lambda v: quantize_e4m3(v.float()).double())
    w = e + 2.0 ** -23 * ref.abs()
    return (q(ref - w) <= got) & (got <= q(ref + w))


def relu_ok(got, pre, terms, e, fmt):
    """got = stored relu(pre) computed in fp32; returns (ok mask, ambiguous mask)"""
    amb = pre.abs() <= 2.0 ** -20 * terms
    closed = (pre < 0) & ~amb
    val_ok = stored_ok(got, pre, e, fmt)
    ok = torch.where(closed, got == 0, torch.where(amb, (got == 0) | val_ok, val_ok))
    return ok, amb


def gate_ok(got, val, open_, amb, e, fmt):
    """got = stored (open ? val : 0) with val computed in fp32 (bound e); amb: either branch"""
    val_ok = stored_ok(got, val, e, fmt)
    return torch.where(amb, (got == 0) | val_ok, torch.where(open_, val_ok, got == 0))


def assert_all(ok, what):
    bad = int((~ok).sum())
    assert bad == 0, "%s: %d of %d elements outside the bound" % (what, bad, ok.numel())


def assert_rare(amb, what):
    frac = float(amb.double().mean()) if amb.numel() else 0.0
    assert frac < 1e-4, "%s: %.2e of the elements are ambiguous" % (what, frac)


def assert_close(got, ref, bound, what):
    got = np.asarray(got, dtype=np.float64)
    bad = ~(np.abs(got - ref) <= bound)
    assert not bad.any(), "%s: channels %s got %s ref %s bound %s" % (
        what, np.nonzero(bad)[0][:4], got[bad][:4], ref[bad][:4], np.asarray(bound)[bad][:4])


def rnd(x):
    """one fp32 rounding of a result computed in fp64 (with room for the fp64 arithmetic before it)"""
    return (U + 2.0 ** -40) * np.abs(x)


def ptr(t):
    return t.data_ptr() if t is not None else None


def host(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed), np.random.default_rng(seed)


def activations(M, C, g, rng):
    """conv-output-like [M, C] float64: every 4th channel has |mean| = 3 std (the variance formula E[y^2] - m^2 then
    cancels 90 % of E[y^2]), the others a small offset"""
    std = rng.uniform(0.5, 2.0, C)
    off = np.where(np.arange(C) % 4 == 0, 3.0 * std * rng.choice([-1.0, 1.0], C), 0.3 * rng.standard_normal(C))
    z = torch.randn(M, C, generator=g, device=DEV, dtype=torch.float64)
    return z * torch.tensor(std, device=DEV) + torch.tensor(off, device=DEV)


def bn_params(nbn, C, rng):
    """host state [nbn][15][C]: gamma (a quarter negative), beta, running statistics, scale / shift for source 3,
    gate parameters; the outputs NaN"""
    p = np.full((nbn, NROWS, C), np.nan, dtype=np.float32)
    for b in range(nbn):
        p[b, GAMMA] = rng.uniform(0.5, 1.5, C) * np.where(rng.random(C) < 0.25, -1.0, 1.0)
        p[b, BETA] = rng.standard_normal(C) * 0.5
        p[b, RMEAN] = rng.standard_normal(C) * 0.2
        p[b, RVAR] = rng.uniform(0.5, 2.0, C)
        p[b, SCALE] = rng.uniform(0.3, 1.5, C) * np.where(rng.random(C) < 0.25, -1.0, 1.0)
        p[b, SHIFT] = rng.standard_normal(C) * 0.5
        p[b, MSCALE] = rng.uniform(0.3, 1.5, C)
        p[b, MSHIFT] = rng.standard_normal(C) * 0.5
    return p


def spread(S, nrep, rng):
    """float64 sums S [3][C] as nrep uneven replicas [nrep][3][C]: every third replica is zero, the others are O(|S|)
    and of either sign, the last one makes the total -- dropping or double-counting any non-zero replica moves the total
    by O(|S|)"""
    parts = np.zeros((nrep,) + S.shape)
    for r in range(nrep - 1):
        if r % 3 != 1:
            parts[r] = rng.uniform(-1.0, 1.5, S.shape) * np.abs(S) / 2
    parts[-1] = S - parts[:-1].sum(0)
    return np.ascontiguousarray(parts)


def sums_terms(M, C):
    """fp32 summation length of k_channel_sums: per-thread rows plus the block's rows_par (bn.cu, sums_grid)"""
    rows_par = 256 // (C // 8)
    grid = min(-(-M // (rows_par * 8)), NUM_SMS * 4)
    return -(-M // (grid * rows_par)) + rows_par + 1


# ---------------------------------------------------------------------------------------------------------------------
# per-channel references
# ---------------------------------------------------------------------------------------------------------------------
def check_forward_channels(out, prm, y64, source, what):
    """one BatchNorm's state rows after a forward pass (out) against float64 from its input y64 [M, C]"""
    M = y64.shape[0]
    if source == 3:
        for r in (SCALE, SHIFT, RMEAN, RVAR):
            assert np.array_equal(out[r], prm[r]), what
        return
    gm, bt, rm, rv = (prm[r].astype(np.float64) for r in (GAMMA, BETA, RMEAN, RVAR))
    if source == 2:                               # k_bn_eval_scale: fp32 add, sqrt, division (each rounded once)
        m, var, dmean, is_rel = rm, rv, np.zeros_like(rm), 4 * U
    else:
        s0, s1 = y64.sum(0).cpu().numpy(), (y64 * y64).sum(0).cpu().numpy()
        a0 = y64.abs().sum(0).cpu().numpy()
        m = s0 / M
        var = ((y64 - y64.mean(0)) ** 2).sum(0).cpu().numpy() / M
        K = sums_terms(M, y64.shape[1]) if source == 0 else 2.0 ** -16
        d0, d1 = K * U * a0, K * U * s1
        dm = d0 / M
        dv = d1 / M + 2 * np.abs(m) * dm + dm * dm            # var = s1/M - m^2
        dmean = dm + rnd(m)
        is_rel = 0.5 * dv / (var + 1e-5) + 2 * U              # + the rounding of invstd and the fp64 rsqrt
    invstd = 1.0 / np.sqrt(var + 1e-5)
    sc = gm * invstd
    sh = bt - m * sc
    dis = invstd * is_rel
    dsc = np.abs(gm) * dis + rnd(sc)
    dsh = np.abs(sc) * dmean + np.abs(m) * dsc + 2 * U * (np.abs(m * sc) + np.abs(bt))
    if source == 2:
        assert np.array_equal(out[MEAN], prm[RMEAN]), what
    else:
        assert_close(out[MEAN], m, dmean, what + " mean")
    assert_close(out[INVSTD], invstd, dis, what + " invstd")
    assert_close(out[SCALE], sc, dsc, what + " scale")
    assert_close(out[SHIFT], sh, dsh, what + " shift")
    if source == 2:                               # eval mode leaves the running statistics alone
        assert np.array_equal(out[RMEAN], prm[RMEAN]) and np.array_equal(out[RVAR], prm[RVAR]), what
        return
    unb = M / (M - 1)
    # momentum 0.1 in fp32: 0.9f and 0.1f are off by < 2^-25 relative, two roundings more
    assert_close(out[RMEAN], 0.9 * rm + 0.1 * m, 0.1 * dmean + 2.0 ** -22 * (np.abs(0.9 * rm) + np.abs(0.1 * m)),
                 what + " running_mean")
    assert_close(out[RVAR], 0.9 * rv + 0.1 * var * unb, 0.1 * unb * dv + 2.0 ** -22 * (0.9 * rv + 0.1 * var * unb),
                 what + " running_var")


def check_backward_channels(out, prm, s0, s1, d0, d1, M, what):
    """d gamma, d beta and the dy = A*g + B*y + C coefficients of one BatchNorm from the float64 sums s0 = sum g,
    s1 = sum g*y (off by at most d0, d1 in the kernel) and the forward's fp32 mean / invstd / gamma"""
    mu, is_, gm = (prm[r].astype(np.float64) for r in (MEAN, INVSTD, GAMMA))
    s2 = is_ * (s1 - mu * s0)
    A = gm * is_
    B = -A * is_ * s2 / M
    Cc = -A * s0 / M - B * mu
    d2 = is_ * (d1 + np.abs(mu) * d0)
    dB = np.abs(A * is_ / M) * d2
    dC = np.abs(A / M) * d0 + np.abs(mu) * dB
    assert_close(out[DGAMMA], s2, d2 + rnd(s2), what + " dgamma")
    assert_close(out[DBETA], s0, d0 + rnd(s0), what + " dbeta")
    assert_close(out[COEF], A, rnd(A), what + " A")
    assert_close(out[COEF + 1], B, dB + rnd(B), what + " B")
    assert_close(out[COEF + 2], Cc, dC + rnd(Cc), what + " C")


def dev_rows(out, *rows):
    return [torch.tensor(out[r], dtype=torch.float64, device=DEV) for r in rows]


# ---------------------------------------------------------------------------------------------------------------------
# forward: batch statistics / lazy finalize / eval scale + k_bn_apply
# ---------------------------------------------------------------------------------------------------------------------
SMALL = (33, 128)
# posenet_bs64's layers (M = 64 * H * W), 7Scenes B = 4 (stem-sized layer1, layer4), ragged M
REAL = [(262144, 64), (65536, 128), (16384, 256), (4096, 512), (22016, 64), (352, 512)]
RAGGED = [(2, 64), (33, 512), (4225, 512)]
BENCH = {(262144, 64), (65536, 128)}

FWD_CASES = ([(p, s, r, SMALL) for p in PRECS for s in range(4) for r in range(3)]
             + [(p, s, 2, (4225, 512)) for p in PRECS for s in (0, 1)]
             + [(p, 1, r, sh) for p in ("bf16", "tc_split") for sh in REAL + RAGGED for r in (0, 1, 2)
                if not (sh in BENCH and r == 0)]
             + [(p, 0, 1, (262144, 64)) for p in ("fp32", "bf16_simt")])


def _fwd_id(c):
    return "%s-src%d-res%d-%dx%d" % (c[0], c[1], c[2], c[3][0], c[3][1])


@pytest.mark.parametrize("case", FWD_CASES, ids=_fwd_id)
def test_bn_forward_apply_vs_float64(case):
    prec, source, res_mode, (M, C) = case
    fa, fz, _ = FMT[prec]
    g, rng = gen(M * 7 + C + 13 * source + res_mode)
    nbn = 2 if res_mode == 2 else 1
    relu = 0 if source == 3 else 1
    prm = bn_params(nbn, C, rng)
    y, y64 = encode(activations(M, C, g, rng), fa)
    res = r64 = None
    if res_mode == 1:
        res, r64 = encode(torch.relu(torch.randn(M, C, generator=g, device=DEV, dtype=torch.float64)), fz)
    elif res_mode == 2:
        res, r64 = encode(activations(M, C, g, rng), fa)
    nrep = 8
    sums = None
    if source == 1:                    # the conv epilogue's sums, spread over the 8 replicas of a slot
        sums = np.stack([spread(np.stack([(t.sum(0)).cpu().numpy(), (t * t).sum(0).cpu().numpy(), np.zeros(C)]), nrep, rng)
                         for t in ([y64, r64] if nbn == 2 else [y64])])
    passes = 2 if source == 0 else 1
    out = np.zeros((passes, nbn, NROWS, C), dtype=np.float32)
    z = empty((M, C), fz)
    _lib.check(_lib.lib().mapnet_test_bn_forward(_lib.PREC[prec], res_mode, relu, source, M, C, ptr(y), ptr(res), ptr(z),
                                                 host(prm), host(sums) if sums is not None else None, nrep, host(out),
                                                 _lib.stream_ptr()), "mapnet_test_bn_forward")
    torch.cuda.synchronize()
    what = _fwd_id(case)
    # per-channel results of every pass (source 0: the second reduction on the same accumulators and counter)
    for p in range(passes):
        check_forward_channels(out[p, 0], prm[0], y64, source, "%s pass %d" % (what, p))
        if nbn == 2:
            check_forward_channels(out[p, 1], prm[1], r64, source, "%s pass %d ds" % (what, p))
    sc, sh = dev_rows(out[-1, 0], SCALE, SHIFT)
    pre = y64 * sc + sh
    terms = (y64 * sc).abs() + sh.abs()
    if res_mode == 1:
        pre = pre + r64
        terms = terms + r64.abs()
    elif res_mode == 2:
        sc2, sh2 = dev_rows(out[-1, 1], SCALE, SHIFT)
        pre = pre + (r64 * sc2 + sh2)
        terms = terms + (r64 * sc2).abs() + sh2.abs()
    got = decode(z, fz)
    e = 2.0 ** -22 * terms
    if relu:
        ok, amb = relu_ok(got, pre, terms, e, fz)
        assert_rare(amb, what)
    else:
        ok = stored_ok(got, pre, e, fz)
    assert_all(ok, what + " z")


# ---------------------------------------------------------------------------------------------------------------------
# backward: reductions / lazy finalize + k_bn_bwd_apply
# ---------------------------------------------------------------------------------------------------------------------
BWD_CASES = ([(p, s, gate, ds, go, SMALL) for p in PRECS for s in (0, 1) for gate in (1, 2) for ds in (0, 1) for go in (0, 1)]
             + [(p, s, 0, 0, 0, (4225, 512)) for p in PRECS for s in (0, 1)]
             + [(p, 1, 1, ds, 1 - ds, sh) for p in ("bf16", "tc_split") for sh in REAL + RAGGED for ds in (0, 1)]
             + [(p, 0, 2, 0, 0, (262144, 64)) for p in ("fp32", "bf16_simt")])
GSCALE = {"tc_split": 2.0 ** -3, "fp32": 4.0}       # the strict mode's power-of-two gradient scale; others none


def _bwd_id(c):
    return "%s-src%d-gate%d-ds%d-gout%d-%dx%d" % (c[0], c[1], c[2], c[3], c[4], c[5][0], c[5][1])


@pytest.mark.parametrize("case", BWD_CASES, ids=_bwd_id)
def test_bn_backward_apply_vs_float64(case):
    prec, source, gate, ds, go, (M, C) = case
    fa, fz, fg = FMT[prec]
    g, rng = gen(M * 5 + C + 11 * source + 3 * gate + ds + 2 * go)
    nbn = 2 if ds else 1
    prm = bn_params(nbn, C, rng)
    for b in range(nbn):                           # the forward's statistics
        prm[b, MEAN] = rng.standard_normal(C)
        prm[b, INVSTD] = rng.uniform(0.3, 2.0, C)
    # incoming gradient with a non-zero mean per channel (so that the C coefficient matters)
    dout, d64 = encode(torch.randn(M, C, generator=g, device=DEV, dtype=torch.float64)
                       + torch.tensor(rng.standard_normal(C) * 0.5, device=DEV), fa)
    y, y64 = encode(activations(M, C, g, rng), fa)
    yd = yd64 = None
    if ds:
        yd, yd64 = encode(activations(M, C, g, rng), fa)
    zm = None
    amb = torch.zeros(M, C, dtype=torch.bool, device=DEV)
    if gate == 1:                                  # post-ReLU tensor with stored zeros and -0.0
        zv = torch.relu(torch.randn(M, C, generator=g, device=DEV, dtype=torch.float64))
        negz = (zv == 0) & (torch.rand(M, C, generator=g, device=DEV) < 0.5)
        zv = torch.where(negz, torch.full_like(zv, -0.0), zv)
        zm, z64 = encode(zv, fz)
        open_ = z64 > 0
    elif gate == 2:                                # ReLU gate recomputed from y in fp32
        msc, msh = (torch.tensor(prm[0, r], dtype=torch.float64, device=DEV) for r in (MSCALE, MSHIFT))
        pre = y64 * msc + msh
        amb = pre.abs() <= 2.0 ** -20 * ((y64 * msc).abs() + msh.abs())
        open_ = pre > 0
    else:
        open_ = torch.ones(M, C, dtype=torch.bool, device=DEV)
    g64 = torch.where(open_, d64, torch.zeros_like(d64))
    s0 = g64.sum(0).cpu().numpy()
    s1 = (g64 * y64).sum(0).cpu().numpy()
    s1d = (g64 * yd64).sum(0).cpu().numpy() if ds else np.zeros(C)
    nrep = 32 if (C == 64 and M == 262144) else 8    # the stem's backward slot has 32 replicas, conv slots 8
    sums = spread(np.stack([s0, s1, s1d]), nrep, rng) if source == 1 else None
    gs = GSCALE.get(prec, 0.0)
    dy = empty((M, C), fg)
    dyd = empty((M, C), fg) if ds else None
    gout = empty((M, C), fa) if go else None
    passes = 2 if source == 0 else 1
    out = np.zeros((passes, nbn, NROWS, C), dtype=np.float32)
    _lib.check(_lib.lib().mapnet_test_bn_backward(
        _lib.PREC[prec], source, gate, M, C, ptr(dout), ptr(zm), ptr(y), ptr(yd), ptr(dy), ptr(dyd), ptr(gout), host(prm),
        host(sums) if sums is not None else None, nrep, gs, host(out), _lib.stream_ptr()), "mapnet_test_bn_backward")
    torch.cuda.synchronize()
    what = _bwd_id(case)
    assert_rare(amb, what)
    # sum bounds: fp32 partial sums (source 0) or fp64 replicas (lazy); an ambiguous gate may add or drop its term
    ag = g64.abs()
    amb_g = torch.where(amb, d64.abs(), torch.zeros_like(d64))
    K = sums_terms(M, C) if source == 0 else 2.0 ** -16
    d0 = K * U * ag.sum(0).cpu().numpy() + amb_g.sum(0).cpu().numpy()
    d1 = K * U * (ag * y64.abs()).sum(0).cpu().numpy() + (amb_g * y64.abs()).sum(0).cpu().numpy()
    for p in range(passes):
        check_backward_channels(out[p, 0], prm[0], s0, s1, d0, d1, M, "%s pass %d" % (what, p))
        if ds:
            d1d = K * U * (ag * yd64.abs()).sum(0).cpu().numpy() + (amb_g * yd64.abs()).sum(0).cpu().numpy()
            check_backward_channels(out[p, 1], prm[1], s0, s1d, d0, d1d, M, "%s pass %d ds" % (what, p))
    S = gs if gs > 0 else 1.0
    for b, (yy, t) in enumerate([(y64, dy)] + ([(yd64, dyd)] if ds else [])):
        A, B, Cc = dev_rows(out[-1, b], COEF, COEF + 1, COEF + 2)
        val = S * (A * d64 + B * yy + Cc)
        e = S * 2.0 ** -22 * ((A * d64).abs() + (B * yy).abs() + Cc.abs())
        # closed gate: dy = B*y + C, computed with g = 0
        val_c = S * (B * yy + Cc)
        got = decode(t, fg)
        ok_open = stored_ok(got, val, e, fg)
        ok_closed = stored_ok(got, val_c, e, fg)
        ok = torch.where(amb, ok_open | ok_closed, torch.where(open_, ok_open, ok_closed))
        assert_all(ok, what + (" dyd" if b else " dy"))
    if go:                                         # the gated gradient itself, bit-exact
        got = decode(gout, fa)
        ok = torch.where(amb, (got == d64) | (got == 0), got == g64)
        assert_all(ok, what + " gout")


# ---------------------------------------------------------------------------------------------------------------------
# stem: BatchNorm + ReLU + 3x3/s2/p1 max pool, its backward
# ---------------------------------------------------------------------------------------------------------------------
def pool_windows(v, fill):
    """[B, H, W, C] -> [B, Ho, Wo, C, 9] windows of the 3x3 / stride 2 / pad 1 pool in scan order kh * 3 + kw"""
    x = F.pad(v.permute(0, 3, 1, 2), (1, 1, 1, 1), value=fill)
    w = x.unfold(2, 3, 2).unfold(3, 3, 2)                      # [B, C, Ho, Wo, 3, 3]
    return w.permute(0, 2, 3, 1, 4, 5).reshape(*w.shape[:1], w.shape[2], w.shape[3], w.shape[1], 9)


def plant_ties(y, g, sign):
    """constant patches (exact ties) and patches far below the mean (all-zero windows after the ReLU)"""
    B, H, W, C = y.shape
    n = max(2, B * H * W // 400)
    for k in range(n):
        b = int(torch.randint(B, (1,), generator=g, device=DEV)); h = int(torch.randint(H, (1,), generator=g, device=DEV))
        w = int(torch.randint(W, (1,), generator=g, device=DEV))
        blk = y[b, h:h + 3, w:w + 3]
        if k % 2 == 0:
            blk[...] = y[b, h, w].clone()
        else:
            blk[...] = -sign * (20.0 + torch.rand(blk.shape, generator=g, device=DEV, dtype=torch.float64))
    return y


STEM_SHAPES = [(4, 128, 171), (3, 7, 9), (2, 2, 2), (1, 1, 3), (2, 18, 22)]
STEM_CASES = ([(p, s, sh) for p in PRECS for s in (0, 1, 2) for sh in STEM_SHAPES]
              + [(p, s, (64, 128, 128)) for p in ("bf16", "tc_split") for s in (0, 1)]
              + [("fp8", 3, sh) for sh in ((3, 7, 9), (4, 128, 171))])


def _stem_id(c):
    return "%s-src%d-%dx%dx%d" % (c[0], c[1], *c[2])


@pytest.mark.parametrize("case", STEM_CASES, ids=_stem_id)
def test_stem_pool_and_backward_vs_float64(case):
    prec, source, (B, H, W) = case
    f8 = prec == "fp8"
    fa, fz, fg = ("bf16", "e4m3", None) if f8 else FMT[prec]
    C = 64
    M = B * H * W
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    g, rng = gen(B * 1000 + H * 10 + W + source)
    prm = bn_params(1, C, rng)
    if f8:            # the inference pool: scale = 1 / s (a power of two), shift 0; y = the stem's post-ReLU bf16 output
        prm[0, SCALE] = 0.25
        prm[0, SHIFT] = 0.0
        yv = torch.relu(torch.randn(B, H, W, C, generator=g, device=DEV, dtype=torch.float64) * 60)
        sign = torch.ones(C, dtype=torch.float64, device=DEV)
    else:
        yv = activations(M, C, g, rng).reshape(B, H, W, C)
        sign = torch.tensor(np.sign(prm[0, SCALE] if source == 3 else prm[0, GAMMA]), dtype=torch.float64, device=DEV)
    yv = plant_ties(yv, g, sign)
    y, y64 = encode(yv, fa)
    sums = None
    if source == 1:
        yf = y64.reshape(M, C)
        sums = spread(np.stack([yf.sum(0).cpu().numpy(), (yf * yf).sum(0).cpu().numpy(), np.zeros(C)]), 8, rng)
    even = H % 2 == 0 and W % 2 == 0
    backward = source in (0, 1)
    bsource = 1 if (source == 1 and even) else 0
    z = empty((B, Ho, Wo, C), fz)
    amax = torch.full((B, Ho, Wo, C), 0xff, dtype=torch.uint8, device=DEV)
    dz = d64 = gbuf = dy = None
    if backward:
        dz, d64 = encode(torch.randn(B, Ho, Wo, C, generator=g, device=DEV, dtype=torch.float64), fa)
        gbuf = empty((B, H, W, C), fa)
        dy = empty((B, H, W, C), fg)
    out = np.zeros((NROWS, C), dtype=np.float32)
    _lib.check(_lib.lib().mapnet_test_stem_pool(
        4 if f8 else _lib.PREC[prec], source, bsource, B, H, W, ptr(y), ptr(z), ptr(amax), ptr(dz), ptr(gbuf), ptr(dy),
        host(prm), host(sums) if sums is not None else None, 8, host(out), _lib.stream_ptr()), "mapnet_test_stem_pool")
    torch.cuda.synchronize()
    what = _stem_id(case)
    if not f8:
        check_forward_channels(out, prm[0], y64.reshape(M, C), source, what)
    sc, sh = dev_rows(out, SCALE, SHIFT)
    pre = y64 * sc + sh
    e = 2.0 ** -22 * ((y64 * sc).abs() + sh.abs())
    # every tap's fp32 activation lies in [lo, hi]; padding taps are -inf (never chosen)
    lo = pool_windows(torch.relu(pre - e), -math.inf)
    hi = pool_windows(torch.relu(pre + e), -math.inf)
    a = pool_windows(torch.relu(pre), -math.inf)
    yw = pool_windows(y64, math.nan)
    idx = torch.arange(9, device=DEV)
    amx = a.amax(-1, keepdim=True)
    ref_arg = torch.where(a == amx, idx, 9).amin(-1)                     # torch's rule: the first maximum wins
    got_arg = amax.long()
    lo_best = torch.gather(lo, -1, ref_arg[..., None])
    y_best = torch.gather(yw, -1, ref_arg[..., None])
    hi_best = torch.gather(hi, -1, ref_arg[..., None])
    # a tap is a rival when its fp32 value may reach the winner's unless it is surely equal to it (the same input, or
    # both surely zero after the ReLU) -- then the first-in-scan-order rule decides exactly
    surely_eq = (yw == y_best) | ((hi == 0) & (hi_best == 0))
    cand = (hi >= lo_best) & (hi > -math.inf)
    rival = cand & ~surely_eq & (idx != ref_arg[..., None])
    amb = rival.any(-1)
    assert_rare(amb, what + " argmax")
    got_in_cand = torch.gather(cand, -1, got_arg.clamp(max=8)[..., None])[..., 0] & (got_arg < 9)
    assert_all(torch.where(amb, got_in_cand, got_arg == ref_arg), what + " argmax")
    # pooled value: the stored form of the fp32 window maximum, which lies in [max lo, max hi]
    vlo, vhi = lo.amax(-1), hi.amax(-1)
    got = decode(z, fz)
    mid = (vlo + vhi) / 2
    assert_all(stored_ok(got, mid, (vhi - vlo) / 2, fz), what + " z")
    if not backward:
        return
    # pool / ReLU backward from the kernel's argmax: every window adds dz to its argmax tap, in fp32 (<= 4 windows)
    oh = torch.arange(Ho, device=DEV).view(1, Ho, 1, 1)
    ow = torch.arange(Wo, device=DEV).view(1, 1, Wo, 1)
    ih = 2 * oh - 1 + got_arg // 3
    iw = 2 * ow - 1 + got_arg % 3
    bb = torch.arange(B, device=DEV).view(B, 1, 1, 1)
    cc = torch.arange(C, device=DEV).view(1, 1, 1, C)
    flat = (((bb * H + ih) * W + iw) * C + cc).reshape(-1)
    acc = torch.zeros(M * C, dtype=torch.float64, device=DEV).index_add_(0, flat, d64.reshape(-1)).view(B, H, W, C)
    aab = torch.zeros(M * C, dtype=torch.float64, device=DEV).index_add_(0, flat, d64.abs().reshape(-1)).view(B, H, W, C)
    gate_amb = pre.abs() <= 2.0 ** -20 * ((y64 * sc).abs() + sh.abs())
    assert_rare(gate_amb, what + " gate")
    gg = decode(gbuf, fa)
    assert_all(gate_ok(gg, acc, pre > 0, gate_amb, 3 * U * aab, fa), what + " g")
    # the BatchNorm's sums over the stored g: fused into the quad kernel (even sizes) or a reducing pass
    gf, yf = gg.reshape(M, C), y64.reshape(M, C)
    if even:
        nq = B * (H // 2) * (W // 2) * 8
        grid = min(-(-nq // 256), NUM_SMS * 8)
        K = 4 * -(-nq // (grid * 256)) + 32 + 1
    else:
        K = sums_terms(M, C)
    s0, s1 = gf.sum(0).cpu().numpy(), (gf * yf).sum(0).cpu().numpy()
    d0 = K * U * gf.abs().sum(0).cpu().numpy()
    d1 = K * U * (gf * yf).abs().sum(0).cpu().numpy()
    check_backward_channels(out, out, s0, s1, d0, d1, M, what)
    A, Bc, Cc = dev_rows(out, COEF, COEF + 1, COEF + 2)
    val = A * gf + Bc * yf + Cc
    e = 2.0 ** -22 * ((A * gf).abs() + (Bc * yf).abs() + Cc.abs())
    assert_all(stored_ok(decode(dy, fg).reshape(M, C), val, e, fg), what + " dy")


# ---------------------------------------------------------------------------------------------------------------------
# global average pool and its backward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("HW", [1, 4, 64, 88])
@pytest.mark.parametrize("prec", PRECS)
def test_gap_and_backward_vs_float64(prec, HW):
    fa, fz, _ = FMT[prec]
    B, C = 3, 512
    g, _ = gen(HW + 17)
    z, z64 = encode(torch.relu(torch.randn(B, HW, C, generator=g, device=DEV, dtype=torch.float64)) + 0.5, fz)
    dfeat = torch.randn(B, C, generator=g, device=DEV)
    feat = torch.full((B, C), float("nan"), device=DEV)
    dz = empty((B, HW, C), fa)
    _lib.check(_lib.lib().mapnet_test_gap(_lib.PREC[prec], B, HW, C, ptr(z), ptr(feat), ptr(dfeat), ptr(dz),
                                          _lib.stream_ptr()), "mapnet_test_gap")
    torch.cuda.synchronize()
    # fp32: per-thread sums over ceil(HW / npg) pixels, npg partials (npg = 256 / (C / 8)), times the rounded 1 / HW
    npg = 256 // (C // 8)
    e = (-(-HW // npg) + npg + 2) * U * z64.abs().sum(1) / HW
    assert_all(stored_ok(feat.double(), z64.mean(1), e, "f32"), "%s HW %d feat" % (prec, HW))
    ref = (dfeat.double() / HW)[:, None, :].expand(B, HW, C)
    assert_all(stored_ok(decode(dz, fa), ref, 2 * U * ref.abs(), fa), "%s HW %d dz" % (prec, HW))
