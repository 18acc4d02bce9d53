"""The two ends of the training step -- the tensor-core stem (conv 0) and the pose head -- one launch sequence at a
time, at the shapes the benchmarked workloads run, checked element by element against float64.

Stem (mapnet_test_stem_ex: k_stem_s2d, the mode's weight pack, the 4x1 fprop over the overlapped view of the
space-to-depth image with the BatchNorm-statistics epilogue, the wgrad and k_unpack_wgrads, as Net runs them).  Cases
are posenet_bs64 (B = 64), mapnet_n32t3 (96) and mapnetpp_n16t10 (160) at 256x256, 7Scenes (B = 4, 256x341: Wc = 171
is odd, the space-to-depth rows are padded to Wsp = 176 blocks) and a 97x65 frame whose zero halo reaches both edges; in
strict mode (tc_split) posenet_bs64 and 7Scenes.  Each case states its fprop plan (N tile, work items) and its wgrad
plan (N tile, pixel tiles, splits, pixel tiles per split) and asserts them from mapnet_test_plan_describe (k = 7) before
it launches; `test_case_list_covers_the_plans_that_matter` (host only) checks that the list still reaches them.

Reference.  float64 on the GPU: F.conv2d(x, w, None, 2, 3) and its autograd on the decoded stored operands (bf16 mode:
x and w rounded to bf16, as k_stem_s2d and the weight pack store them; strict mode: the fp32 inputs).  S = the same ops
on |x| and |w| (|x| and |dy| for the wgrad).

Per-element bounds (as tests/test_gpu_conv_plans.py derives them).  |got - ref| <= u_store |ref| + (1 + u_store) gamma S:
  * fprop: the engine runs the stem as 4 taps x 64 channels = 16 wgmma instructions per tile, each truncating its
    fp32 accumulation once (2^-23 relative to the running sum, which is at most S), then the bf16 store rounds (2^-8).
    Strict mode runs 8 taps (hi / lo weight planes) x 128 split channels = 64 instructions, adds 2 * 2^-22 + 2^-44 for
    the hi/lo split of two operands of magnitude in [2^-3, 2^3] (the halo zeros and padded channels split exactly), and
    stores the fp32 accumulator as it is.
  * wgrad: 4 instructions per 64-pixel tile, tiles_per_split tiles, then the splits added in fp32 (2^-24 per add, one
    per split when there are several).  Strict mode adds the split terms and the 3 fp32 adds of the four hi/lo cells;
    its dy is scaled by 2^8 and the engine multiplies by out_scale = 2^-8 (exact).  The gradient is checked in the
    [64,3,7,7] .grad layout, so a padded tap or channel that leaked through k_unpack_wgrads, or a wrong permutation,
    fails.  posenet_bs64 reduces over B*Hc*Wc = 1.05 M pixels; the `coherent` case (non-negative x and dy, running
    sums that only grow) shows how close that truncation chain comes to its bound.
  * BatchNorm statistics: the epilogue's (sum y, sum y^2) per channel against float64 sums of the STORED y, within the
    fp32 chain of the epilogue: 4 rows per lane, 3 shuffle levels, one add per tile of the CTA, 3 adds across the
    epilogue warps, each 2^-24 of the column's sum of |terms|.

Head (mapnet_test_head: head_forward / head_backward, the launch sequences Net's step runs).  F = 2048 and
B in {1, 33, 64, 96, 160, 256, 300}: 33 leaves ragged 32-row tiles, the pose products run 32 K-splits up to B = 96 and
16 at B = 160 and 256, dfeat runs 8 / 4 / 2 / 1 splits, and at B >= 256 the weight-gradient products of fc_xyz /
fc_wpqr (M = 3, K = B, A strided by 6) take the split-K path.  droprate 0, 0.5 and 0.3 (keep scale 1/0.7, not a power
of two), with and without the NaN filter.
  * mask: bitwise against splitmix64 (dropout_mask_at) reimplemented in numpy uint64, at a flat offset step * stride
    above 2^32, and through the device step counter (which must advance by one).
  * products: k_small_gemm is an fmaf chain per K split (plus the bias on split 0) and k_split_sum adds the splits in
    order, so |got - ref| <= gamma_n S with gamma_n = n u / (1 - n u), u = 2^-24, n = kchunk + splits (from
    mapnet_test_small_gemm_plan); k_colsum is a chain of B adds, k_head_dh a 6-term contraction.  One more store
    rounding (u |ref|) where a non-power-of-two keep scale multiplies.  ReLU is 1-Lipschitz, so fcpre near zero needs
    no special case in hdrop.  Each product's reference reads the operands the kernel really read: pred from the
    stored hdrop, the backward from the stored hdrop / dh and the kernel's own gate fcpre > 0.
  * NaN filter (models/posenet.py:28-34 hook semantics, head.cu): a NaN in dpred[b, 3 + j] zeroes row j of dW_wpqr and
    db_wpqr[j] exactly and sends nothing of sample b's rotation half into the trunk; the translation half is untouched.
  * k_grad_scale: exactly 2^(8 - e), e from frexp(max |dpredh|), clamped to 2^+-100; 1 for all zeros, NaN or Inf.

Every output is NaN before the launch, so an element that is never written fails.  Every case prints max(err/bound).
"""
import ctypes
import json
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from geomapnet_b200 import _lib

NSM = 132
U_BF16 = 2.0 ** -8
U_FP32 = 2.0 ** -24
TRUNC = 2.0 ** -23          # one ulp per truncating wgmma accumulation
SPLIT = 2.0 ** -22          # hi/lo fp16 split of one operand
GSCALE = 8                  # strict-mode gradients arrive scaled by 2^GSCALE; the wgrad multiplies by 2^-GSCALE
UINT64_MAX = 0xFFFFFFFFFFFFFFFF

# (id, precision, (B, H, W), fprop plan (BN, items), wgrad plan (BN, pixel tiles, splits, tiles per split), coherent)
STEM_CASES = [
    ("posenet_bs64", "bf16", (64, 256, 256), (64, 8192), (64, 16384, 132, 125), False),
    ("posenet_bs64.coherent", "bf16", (64, 256, 256), (64, 8192), (64, 16384, 132, 125), True),
    ("mapnet_n32t3", "bf16", (96, 256, 256), (64, 12288), (64, 24576, 132, 187), False),
    ("mapnetpp_n16t10", "bf16", (160, 256, 256), (64, 20480), (64, 40960, 132, 311), False),
    ("7scenes_b4", "bf16", (4, 256, 341), (64, 1024), (64, 1536, 128, 12), False),
    ("halo_97x65", "bf16", (3, 97, 65), (64, 75), (64, 147, 74, 2), False),
    ("posenet_bs64", "tc_split", (64, 256, 256), (64, 8192), (128, 16384, 66, 249), False),
    ("7scenes_b4", "tc_split", (4, 256, 341), (64, 1024), (128, 1536, 64, 24), False),
]

HEAD_F = 2048
HEAD_BATCHES = [1, 33, 64, 96, 160, 256, 300]
DROPRATES = [0.0, 0.5, 0.3]


# ------------------------------------------------------------------------------------------------------------------
# plans (host only)
# ------------------------------------------------------------------------------------------------------------------
def stem_plan(kind, B, H, W, precision):
    buf = ctypes.create_string_buffer(1 << 17)
    flags = 2 if precision == "tc_split" else 0
    _lib.check(_lib.lib().mapnet_test_plan_describe(kind, B, H, W, 3, 64, 7, 2, flags, buf, len(buf)),
               "mapnet_test_plan_describe")
    p = json.loads(buf.value.decode())
    if kind == 2:
        P = p["wgrad"]
        return dict(BN=P["BN"], pix=P["n_pix_tiles"], splits=P["splits"], tps=P["tiles_per_split"],
                    last=P["n_pix_tiles"] - (P["splits"] - 1) * P["tiles_per_split"])
    assert len(p["launches"]) == 1
    L = p["launches"][0]
    return dict(BN=p["BN"], items=L["n_tiles_m"] * L["n_tiles_n"], taps=len(L["classes"][0]["taps"]), Cs=L["Cs"])


def expected_stem_plans(case):
    _, prec, (B, H, W), fp, wg, _ = case
    f = stem_plan(0, B, H, W, prec)
    assert (f["BN"], f["items"]) == fp, (case[0], prec, "fprop", f)
    w = stem_plan(2, B, H, W, prec)
    assert (w["BN"], w["pix"], w["splits"], w["tps"]) == wg, (case[0], prec, "wgrad", w)
    return f, w


def gemm_plan(epi, M, N, K):
    sp, kc = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.lib().mapnet_test_small_gemm_plan(epi, M, N, K, ctypes.byref(sp), ctypes.byref(kc)),
               "mapnet_test_small_gemm_plan")
    return sp.value, kc.value


def head_plans(B, Fd=HEAD_F):
    """(splits, kchunk) of every head product at batch B"""
    return dict(fc=gemm_plan(1, B, Fd, 512), pose=gemm_plan(0, B, 3, Fd), dWpose=gemm_plan(0, 3, Fd, B),
                dWfc=gemm_plan(0, Fd, 512, B), dfeat=gemm_plan(0, B, 512, Fd))


# ------------------------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------------------------
def check_elements(what, got, ref, bound):
    """every element within its bound (NaN fails; a zero bound demands an exact result); prints and returns
    max(err / bound)"""
    err = (got - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError("%s: %d of %d elements outside the bound (%d NaN); first at index %s (shape %s): got %r "
                             "ref %r bound %r" % (what, bad.shape[0], got.numel(), int(torch.isnan(got).sum()), i,
                                                  tuple(got.shape), float(got[i]), float(ref[i]), float(bound[i])))
    pos = bound > 0
    ratio = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
    print("stem-head %-58s max err/bound %.3g" % (what, ratio))
    return ratio


def gamma(n):
    return n * U_FP32 / (1.0 - n * U_FP32)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _logu(shape, g, scale=1.0):
    """fp32 values of magnitude in [2^-3, 2^3], random sign: inside fp16's window for the hi/lo split"""
    e = torch.rand(shape, generator=g, device="cuda") * 6.0 - 3.0
    s = torch.where(torch.rand(shape, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    return (s * torch.exp2(e) * scale).float()


def _sum_bound(stored_abs_terms, tiles_per_cta):
    return (4 + 3 + tiles_per_cta + 3 + 1) * U_FP32 * stored_abs_terms + 1e-30


nhwc = lambda t: t.permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------------------------
# stem
# ------------------------------------------------------------------------------------------------------------------
def _stem_wgrad(x, dy):
    ww = torch.zeros((64, 3, 7, 7), dtype=torch.float64, device="cuda", requires_grad=True)
    return torch.autograd.grad(F.conv2d(x, ww, None, 2, 3), ww, dy)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEM_CASES, ids=["%s-%s" % (c[1], c[0]) for c in STEM_CASES])
def test_stem_fprop_statistics_and_wgrad(case):
    name, prec, (B, H, W), _, _, coherent = case
    fplan, wplan = expected_stem_plans(case)
    t0 = time.time()
    strict = prec == "tc_split"
    g = _gen(2000 + STEM_CASES.index(case))
    Hc, Wc = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    if strict:
        x = _logu((B, 3, H, W), g)
        w = _logu((64, 3, 7, 7), g)
        dy = _logu((B, 64, Hc, Wc), g)
        xr, wr, dyr = x.double(), w.double(), dy.double()
        dy_in = (nhwc(dy) * 2.0 ** GSCALE).contiguous()
        out_scale = 2.0 ** -GSCALE
        y = torch.full((B, Hc, Wc, 64), float("nan"), dtype=torch.float32, device="cuda")
    else:
        x = torch.randn((B, 3, H, W), generator=g, device="cuda")
        w = torch.randn((64, 3, 7, 7), generator=g, device="cuda") * (2.0 / 147) ** 0.5
        dy = torch.randn((B, 64, Hc, Wc), generator=g, device="cuda").bfloat16()
        if coherent:
            x, dy = x.abs(), dy.abs()
        xr, wr, dyr = x.bfloat16().double(), w.bfloat16().double(), dy.double()
        dy_in = nhwc(dy).contiguous()
        out_scale = 0.0
        y = torch.full((B, Hc, Wc, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    del dy
    dw = torch.full((64, 3, 7, 7), float("nan"), dtype=torch.float32, device="cuda")
    sums = np.full((2, 64), np.nan, dtype=np.float64)
    _lib.check(_lib.lib().mapnet_test_stem_ex(_lib.PREC[prec], B, H, W, x.data_ptr(), w.data_ptr(), y.data_ptr(),
                                              dy_in.data_ptr(), dw.data_ptr(), float(out_scale),
                                              sums.ctypes.data_as(ctypes.c_void_p), _lib.stream_ptr()),
               "mapnet_test_stem_ex")
    torch.cuda.synchronize()
    del x, w, dy_in
    what = "%s %s %s" % (prec, name, (B, H, W))
    # fprop
    ref = nhwc(F.conv2d(xr, wr, None, 2, 3))
    S = nhwc(F.conv2d(xr.abs(), wr.abs(), None, 2, 3))
    gam = fplan["taps"] * fplan["Cs"] // 16 * TRUNC + (2 * SPLIT + SPLIT ** 2 if strict else 0.0)
    u = 0.0 if strict else U_BF16
    got = y.double()
    del y
    check_elements(what + " fprop", got, ref, u * ref.abs() + (1 + u) * gam * S)
    del ref, S
    # the BatchNorm statistics of the stored y
    st = got.reshape(-1, 64)
    del got
    tpc = math.ceil(fplan["items"] / NSM)
    sums = torch.from_numpy(sums).cuda()
    for j, (terms, n_extra) in enumerate(((st, 0), (st * st, 1))):
        bound = _sum_bound(terms.abs().sum(0), tpc + n_extra)
        err = (sums[j] - terms.sum(0)).abs()
        assert bool((err <= bound).all()), "%s: statistic %d off in channel %d: got %r ref %r bound %r" % (
            what, j, int((err / bound).argmax()), float(sums[j][int((err / bound).argmax())]),
            float(terms.sum(0)[int((err / bound).argmax())]), float(bound[int((err / bound).argmax())]))
        print("stem-head %-58s max err/bound %.3g" % (what + (" sum y" if j == 0 else " sum y^2"),
                                                        float((err / bound).max())))
    del st
    # wgrad in the .grad layout
    ref = _stem_wgrad(xr, dyr)
    S = _stem_wgrad(xr.abs(), dyr.abs())
    gw = 4 * wplan["tps"] * TRUNC + (wplan["splits"] if wplan["splits"] > 1 else 0) * U_FP32
    if strict:
        gw += 2 * SPLIT + SPLIT ** 2 + 3 * U_FP32
    check_elements(what + (" wgrad coherent" if coherent else " wgrad") + " splits %d x %d tiles" % (
        wplan["splits"], wplan["tps"]), dw.double(), ref, (1 + U_FP32) * gw * S)
    print("stem-head %-58s %.1f s" % (what, time.time() - t0))


# ------------------------------------------------------------------------------------------------------------------
# head
# ------------------------------------------------------------------------------------------------------------------
def mask_ref(seed, offset, n, p):
    """dropout_mask_at (head.cu) over flat elements offset .. offset + n - 1, in numpy uint64 / float32"""
    with np.errstate(over="ignore"):
        e = np.arange(n, dtype=np.uint64) + np.uint64(offset)
        z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * (e + np.uint64(1))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    u = (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    keep = np.float32(1.0) / (np.float32(1.0) - np.float32(p))
    return np.where(u >= np.float32(p), keep, np.float32(0.0)).astype(np.float32)


def grad_scale_ref(v):
    """k_grad_scale: S = 2^(8 - e), max|v| = f * 2^e with f in [0.5, 1), e clamped to 8 -+ 100; 1 when max|v| is 0,
    NaN or infinite"""
    m = np.abs(np.asarray(v, dtype=np.float64))
    if not np.isfinite(m).all() or m.max() == 0.0:
        return 1.0
    k = 8 - int(np.frexp(m.max())[1])
    return 2.0 ** max(-100, min(100, k))


def head_params(g, Fd):
    fc_w = torch.randn(Fd, 512, generator=g, device="cuda") * (1.0 / 512) ** 0.5
    fc_b = torch.randn(Fd, generator=g, device="cuda") * 0.1
    xyz_w = torch.randn(3, Fd, generator=g, device="cuda") * (1.0 / Fd) ** 0.5
    xyz_b = torch.randn(3, generator=g, device="cuda") * 0.1
    wpqr_w = torch.randn(3, Fd, generator=g, device="cuda") * (1.0 / Fd) ** 0.5
    wpqr_b = torch.randn(3, generator=g, device="cuda") * 0.1
    return [fc_w, fc_b, xyz_w, xyz_b, wpqr_w, wpqr_b]


def pack(ts):
    return torch.cat([t.reshape(-1) for t in ts]).contiguous()


def unpack(flat, Fd):
    sizes = [(Fd, 512), (Fd,), (3, Fd), (3,), (3, Fd), (3,)]
    out, o = [], 0
    for s in sizes:
        n = int(np.prod(s))
        out.append(flat[o:o + n].view(*s))
        o += n
    return out


def run_head(B, Fd, feat, params, droprate, seed, step, stride, ctr=None, dpred=None, filter_nans=0, scale=False):
    nan = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device="cuda")
    o = dict(mask=nan(B, Fd), fcpre=nan(B, Fd), hdrop=nan(B, Fd), pred=nan(B, 6))
    if dpred is not None:
        o.update(dh=nan(B, Fd), dfeat=nan(B, 512), grads=nan(params.numel()), scale2=nan(2) if scale else None)
    ptr = lambda t: t.data_ptr() if t is not None else None
    _lib.check(_lib.lib().mapnet_test_head(
        B, Fd, feat.data_ptr(), params.data_ptr(), float(droprate), int(seed), int(step), int(stride), ptr(ctr),
        o["mask"].data_ptr(), o["fcpre"].data_ptr(), o["hdrop"].data_ptr(), o["pred"].data_ptr(), ptr(dpred),
        int(filter_nans), ptr(o.get("dh")), ptr(o.get("dfeat")), ptr(o.get("grads")), ptr(o.get("scale2")),
        _lib.stream_ptr()), "mapnet_test_head")
    torch.cuda.synchronize()
    return o


def check_mask(what, got, B, Fd, seed, offset, p):
    ref = torch.from_numpy(mask_ref(seed, offset, B * Fd, p)).view(B, Fd)
    got = got.cpu()
    same = (got.view(torch.int32) == ref.view(torch.int32))
    if not bool(same.all()):
        i = tuple((~same).nonzero()[0].tolist())
        raise AssertionError("%s: mask differs from splitmix64 in %d of %d elements; first at %s: got %r ref %r" % (
            what, int((~same).sum()), B * Fd, i, float(got[i]), float(ref[i])))
    kept = float((ref != 0).double().mean())
    assert abs(kept - (1 - p)) < 0.05, (what, kept)
    print("stem-head %-58s mask bitwise (offset %d, kept %.3f)" % (what, offset, kept))


@pytest.mark.gpu
@pytest.mark.parametrize("filter_nans", [0, 1], ids=["plain", "nanfilter"])
@pytest.mark.parametrize("droprate", DROPRATES, ids=["p%g" % p for p in DROPRATES])
@pytest.mark.parametrize("B", HEAD_BATCHES)
def test_head_forward_and_backward(B, droprate, filter_nans):
    Fd = HEAD_F
    plans = head_plans(B)
    if B == 64 or B == 96:
        assert plans["pose"][0] == 32, plans
    if B == 160:
        assert plans["pose"][0] == 16 and plans["dfeat"][0] == 1, plans
    assert plans["dfeat"][0] == {64: 4, 96: 2}.get(B, plans["dfeat"][0]), plans
    assert (plans["dWpose"][0] > 1) == (B >= 256) and plans["fc"][0] == 1 and plans["dWfc"][0] == 1, plans
    what = "head B %d p %g %s" % (B, droprate, "nanfilter" if filter_nans else "plain")
    g = _gen(3000 + B * 7 + int(droprate * 10) + filter_nans)
    feat = torch.randn(B, 512, generator=g, device="cuda").abs()
    P = head_params(g, Fd)
    params = pack(P)
    max_B = 320
    stride = max_B * Fd
    step = 2 ** 32 // stride + 11                         # flat offset step * stride above 2^32: 64-bit index math
    seed = 0x5EED0000 + B
    dpred = torch.randn(B, 6, generator=g, device="cuda")
    nan_cols, nan_rows = [], []
    if filter_nans:
        nan_at = [(min(1, B - 1), 0), (B - 1, 2)]         # dpred[b, 3 + j]
        for b, j in nan_at:
            dpred[b, 3 + j] = float("nan")
        nan_cols = sorted({j for _, j in nan_at})
        nan_rows = sorted({b for b, _ in nan_at})
    o = run_head(B, Fd, feat, params, droprate, seed, step, stride, dpred=dpred, filter_nans=filter_nans, scale=True)
    fc_w, fc_b, xyz_w, xyz_b, wpqr_w, wpqr_b = (t.double() for t in P)
    fd = feat.double()
    pow2 = droprate in (0.0, 0.5)
    # ---- forward ----
    if droprate > 0:
        check_mask(what, o["mask"], B, Fd, seed, step * stride, droprate)
        mk = o["mask"].double()
    else:
        mk = torch.ones(B, Fd, dtype=torch.float64, device="cuda")
    sp, kc = plans["fc"]
    fref = fd @ fc_w.T + fc_b
    fS = fd.abs() @ fc_w.abs().T + fc_b.abs()
    check_elements(what + " fcpre", o["fcpre"].double(), fref, gamma(kc + sp) * fS)
    href = torch.relu(fref) * mk
    check_elements(what + " hdrop", o["hdrop"].double(), href,
                   mk * gamma(kc + sp) * fS + (0.0 if pow2 else U_FP32) * href.abs())
    h = o["hdrop"].double()
    sp, kc = plans["pose"]
    W6 = torch.cat([xyz_w, wpqr_w]); b6 = torch.cat([xyz_b, wpqr_b])
    check_elements(what + " pred (%d splits)" % sp, o["pred"].double(), h @ W6.T + b6,
                   gamma(kc + sp) * (h.abs() @ W6.abs().T + b6.abs()))
    # ---- backward: the filtered copies of dpred ----
    dp = dpred.double()
    dpw, dph = dp.clone(), dp.clone()
    if filter_nans:
        for j in nan_cols:
            dpw[:, 3 + j] = 0.0
        for b in nan_rows:
            dph[b, 3:] = 0.0
    assert float(o["scale2"][0]) == grad_scale_ref(dph.cpu().numpy()), (what, o["scale2"].tolist())
    assert float(o["scale2"][1]) == 1.0 / float(o["scale2"][0])
    G = unpack(o["grads"], Fd)
    sp, kc = plans["dWpose"]
    gw = gamma(kc + sp)
    check_elements(what + " dW_xyz (%d splits)" % sp, G[2].double(), dpw[:, :3].T @ h, gw * (dpw[:, :3].abs().T @ h.abs()))
    check_elements(what + " dW_wpqr", G[4].double(), dpw[:, 3:].T @ h, gw * (dpw[:, 3:].abs().T @ h.abs()))
    check_elements(what + " db_xyz", G[3].double(), dpw[:, :3].sum(0), gamma(B) * dpw[:, :3].abs().sum(0))
    check_elements(what + " db_wpqr", G[5].double(), dpw[:, 3:].sum(0), gamma(B) * dpw[:, 3:].abs().sum(0))
    for j in nan_cols:        # the hook's semantics, exactly: the whole weight row and the bias get no gradient
        assert bool((G[4][j] == 0).all()) and float(G[5][j]) == 0.0, (what, j)
    gate = (o["fcpre"].double() > 0).double()
    dref = (dph @ W6) * mk * gate
    check_elements(what + " dh", o["dh"].double(), dref,
                   gamma(6) * (dph.abs() @ W6.abs()) * mk * gate + (0.0 if pow2 else U_FP32) * dref.abs())
    for b in nan_rows:        # the rotation half of a filtered sample sends nothing; its translation half is intact
        tr = (dp[b, :3] @ xyz_w) * mk[b] * gate[b]
        tb = gamma(6) * (dp[b, :3].abs() @ xyz_w.abs()) * mk[b] + (0.0 if pow2 else U_FP32) * tr.abs()
        assert bool(((o["dh"][b].double() - tr).abs() <= tb).all()), (what, b)
    dh = o["dh"].double()
    sp, kc = plans["dWfc"]
    check_elements(what + " dW_fc", G[0].double(), dh.T @ fd, gamma(kc + sp) * (dh.abs().T @ fd))
    check_elements(what + " db_fc", G[1].double(), dh.sum(0), gamma(B) * dh.abs().sum(0))
    sp, kc = plans["dfeat"]
    check_elements(what + " dfeat (%d splits)" % sp, o["dfeat"].double(), dh @ fc_w,
                   gamma(kc + sp) * (dh.abs() @ fc_w.abs()))


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.5, 0.3])
def test_dropout_mask_from_the_device_counter(p):
    """step == UINT64_MAX: the mask of flat offset (*ctr) * stride, and *ctr advanced by one"""
    B, Fd = 33, HEAD_F
    g = _gen(41)
    feat = torch.randn(B, 512, generator=g, device="cuda").abs()
    params = pack(head_params(g, Fd))
    stride = 300 * Fd
    c = 2 ** 33 // stride + 5
    ctr = torch.tensor([c], dtype=torch.int64, device="cuda")
    o = run_head(B, Fd, feat, params, p, 1234, UINT64_MAX, stride, ctr=ctr)
    assert int(ctr.item()) == c + 1
    check_mask("device counter p %g" % p, o["mask"], B, Fd, 1234, c * stride, p)


# (id, dpred [B, 6] float32, S): the gradient scale of the strict mode at the edges of k_grad_scale
def _grad_scale_cases():
    B = 5
    z = np.zeros((B, 6), dtype=np.float32)

    def at(v, b=2, k=4, base=None):
        d = (np.full((B, 6), 0.25, dtype=np.float32) if base is None else base).copy()
        d[b, k] = v
        return d
    return [("pow2", at(1.0), 2.0 ** 7), ("pow2_negative", at(-4.0), 2.0 ** 5), ("between", at(0.75), 2.0 ** 8),
            ("translation_half", at(3.0, k=0), 2.0 ** 6),
            ("small", at(2.0 ** -90, base=z), 2.0 ** 97), ("denormal_max", at(2.0 ** -130, base=z), 2.0 ** 100), ("small_clamped", at(2.0 ** -95, base=z), 2.0 ** 100),
            ("large_clamped", at(2.0 ** 120), 2.0 ** -100), ("near_float_max", at(3.2e38), 2.0 ** -100),
            ("zeros", z, 1.0), ("nan", at(float("nan")), 1.0), ("inf", at(float("inf")), 1.0),
            ("minus_inf", at(-float("inf")), 1.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,dpred,S", _grad_scale_cases(), ids=[c[0] for c in _grad_scale_cases()])
def test_grad_scale_edges(name, dpred, S):
    B, Fd = dpred.shape[0], 64
    assert grad_scale_ref(dpred) == S
    g = _gen(43)
    feat = torch.randn(B, 512, generator=g, device="cuda").abs()
    params = pack(head_params(g, Fd))
    o = run_head(B, Fd, feat, params, 0.0, 0, 0, B * Fd, dpred=torch.from_numpy(dpred).cuda(), scale=True)
    got = o["scale2"].cpu().tolist()
    assert got == [S, 1.0 / S], (name, got, S)
