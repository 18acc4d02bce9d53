"""The wgmma conv engines (csrc/conv_tc.cu) one launch at a time, at the tile plans the benchmarked workloads run,
checked element by element against float64.

Cases are the distinct ResNet-34 conv geometries of posenet_bs64 (B = 64, 256x256), a few of mapnet_n32t3 (B = 96)
and mapnetpp_n16t10 (B = 160, layer1: about 39 tiles per persistent CTA) and the 7Scenes 256x341 input (B = 4, ragged
widths 86 / 43 / 22 / 11; layer1 picks the 128x1 pixel box).  Each runs fprop, dgrad and wgrad.  A case states the
plan it expects (N tile BN, work items against the 132 persistent CTAs, wgrad splits and pixel tiles per split) and
asserts it from mapnet_test_plan_describe before launching; `test_case_list_covers_the_benchmark_plans` (host only)
checks that the list as a whole still reaches the plans that matter, so a change of the tile cost model cannot
quietly drop coverage.

Reference.  float64 on the GPU: torch.nn.functional.conv2d and its autograd, on the decoded stored operands (bf16
converts to float64 exactly; strict mode takes the fp32 inputs).  S = sum |a*b| per element comes from the same ops
on |a| and |b|.

Per-element bound.  |got - ref| <= eps_store(|ref|) + (1 + u_store) * gamma * S, with
  * eps_store: round-to-nearest of the stored format.  bf16 keeps 8 significant bits, so half a spacing is
    u_store = 2^-8 relative.  fp32 outputs (strict mode, wgrad) are stored as accumulated, except for one fp32 add of a
    residual or of the prior gradient: 2^-24 of what is added.
  * gamma: the fp32 accumulation chain.  A wgmma instruction adds 16 exact products into the accumulator, and the
    tensor core's fp32 accumulation truncates instead of rounding, so each instruction is allowed one ulp,
    2^-23 relative to the running sum, which is at most S.  fprop / dgrad run K / 16 instructions per tile,
    K = taps * channels (dgrad: the heaviest parity class, plus Cout of a folded shortcut).  wgrad runs 4 per
    64-pixel tile, tiles_per_split of them, and then adds the splits up in fp32 (k_wgrad_reduce, round-to-nearest,
    2^-24 per add).
  * strict mode (tc_split): every operand is cut into fp16 hi + lo planes, x = (hi + lo)(1 + d), |d| <= 2^-22, when
    |x| >= 2^-3 (lo is then normal, or its absolute error 2^-25 is still below 2^-22 |x|); the operands are drawn with
    magnitudes in [2^-3, 2^3].  A product then carries 2 * 2^-22 + 2^-44; the four hi/lo products make K four times
    longer; wgrad sums its four hi/lo accumulator cells with 3 more fp32 adds.  Gradient scales are powers of two, so
    scaling is exact.
The bound is worst-case.  With signed random operands the accumulation error stays far below gamma * S, and the bf16
store rounding carries fprop / dgrad to within a factor of two of their bound.  wgrad stores fp32, so a wgrad case
with non-negative operands (`coherent`), whose running sums grow monotonically, shows how close the truncation chain
comes to its bound.  Every case prints max(err / bound).

Every element is written exactly once: fprop / dgrad outputs are NaN before the launch (the strict dgrad's output
holds its residual, which it reads in place); wgrad outputs hold a nonzero dW0 before the launch, and out - dW0 is
checked, which covers the add-into-the-gradient contract of the single-split store and of k_wgrad_reduce.

The fused epilogues (BatchNorm statistics in fprop; ReLU gate, residual and BatchNorm-backward sums in dgrad; the
folded stride-2 shortcut) run at posenet_bs64 shapes whose plan is BN 128.  Their per-channel sums are checked
against float64 sums of the stored values within the fp32 summation chain: 4 rows per lane, 3 shuffle levels, one add
per tile of the CTA, 3 adds across the epilogue warps, each 2^-24 of the column's sum of |terms|.
"""
import ctypes
import json
import math
import time

import pytest
import torch
import torch.nn.functional as F

from geomapnet_b200 import _lib

NSM = 132
U_BF16 = 2.0 ** -8
U_FP32 = 2.0 ** -24
TRUNC = 2.0 ** -23          # one ulp per truncating wgmma accumulation
SPLIT = 2.0 ** -22          # hi/lo fp16 split of one operand
GSCALE = 8                  # strict-mode gradients arrive scaled by 2^GSCALE; the engines multiply by 2^-GSCALE

# (id, precision, (B, H, W, Ci, Co, k, stride), fprop plan (BN, items), dgrad plan (BN, items, parity classes),
#  wgrad plan (BN, pixel tiles, splits, tiles per split), coherent wgrad operands)
CASES = [
    ("posenet_bs64.layer1", "bf16", (64, 64, 64, 64, 64, 3, 1), (64, 2048), (64, 2048, 1), (64, 4096, 52, 79), False),
    ("posenet_bs64.layer1.coherent", "bf16", (64, 64, 64, 64, 64, 3, 1), None, None, (64, 4096, 52, 79), True),
    ("posenet_bs64.layer2.0.conv1", "bf16", (64, 64, 64, 64, 128, 3, 2), (128, 512), (64, 2048, 4), (128, 1024, 52, 20), False),
    ("posenet_bs64.layer2.0.downsample", "bf16", (64, 64, 64, 64, 128, 1, 2), (128, 512), (64, 2048, 4), (128, 1024, 256, 4), False),
    ("posenet_bs64.layer2", "bf16", (64, 32, 32, 128, 128, 3, 1), (128, 512), (128, 512, 1), (128, 1024, 29, 36), False),
    ("posenet_bs64.layer3.0.conv1", "bf16", (64, 32, 32, 128, 256, 3, 2), (128, 256), (128, 512, 4), (128, 256, 14, 19), False),
    ("posenet_bs64.layer3.0.downsample", "bf16", (64, 32, 32, 128, 256, 1, 2), (128, 256), (128, 512, 4), (128, 256, 128, 2), False),
    ("posenet_bs64.layer3", "bf16", (64, 16, 16, 256, 256, 3, 1), (128, 256), (128, 256, 1), (128, 256, 7, 37), False),
    ("posenet_bs64.layer4.0.conv1", "bf16", (64, 16, 16, 256, 512, 3, 2), (128, 128), (128, 256, 4), (128, 64, 3, 22), False),
    ("posenet_bs64.layer4.0.downsample", "bf16", (64, 16, 16, 256, 512, 1, 2), (128, 128), (128, 256, 4), (128, 64, 32, 2), False),
    ("posenet_bs64.layer4", "bf16", (64, 8, 8, 512, 512, 3, 1), (128, 128), (128, 128, 1), (128, 64, 1, 64), False),
    ("posenet_bs64.layer4.coherent", "bf16", (64, 8, 8, 512, 512, 3, 1), None, None, (128, 64, 1, 64), True),
    ("mapnet_n32t3.layer1", "bf16", (96, 64, 64, 64, 64, 3, 1), (64, 3072), (64, 3072, 1), (64, 6144, 52, 119), False),
    ("mapnet_n32t3.layer4", "bf16", (96, 8, 8, 512, 512, 3, 1), (128, 192), (128, 192, 1), (128, 96, 1, 96), False),
    ("mapnetpp_n16t10.layer1", "bf16", (160, 64, 64, 64, 64, 3, 1), (64, 5120), (64, 5120, 1), (64, 10240, 52, 197), False),
    ("7scenes_b4.layer1", "bf16", (4, 64, 86, 64, 64, 3, 1), (64, 256), (64, 256, 1), (64, 512, 52, 10), False),
    ("7scenes_b4.layer3.0.conv1", "bf16", (4, 32, 43, 128, 256, 3, 2), (64, 64), (64, 128, 4), (128, 32, 11, 3), False),
    ("7scenes_b4.layer4", "bf16", (4, 8, 11, 512, 512, 3, 1), (64, 32), (64, 32, 1), (128, 8, 1, 8), False),
    # strict mode: dgrad with the power-of-two gradient scale and its residual read in place from the output, as the
    # trunk's downsampling blocks run conv_dgrad(conv1, S1, S0, S0); wgrad with the gradient scale
    ("posenet_bs64.layer1", "tc_split", (64, 64, 64, 64, 64, 3, 1), (64, 2048), (64, 2048, 1), (128, 4096, 29, 142), False),
    ("posenet_bs64.layer3", "tc_split", (64, 16, 16, 256, 256, 3, 1), (128, 256), (128, 256, 1), (128, 256, 1, 256), False),
    ("posenet_bs64.layer4.0.conv1", "tc_split", (64, 16, 16, 256, 512, 3, 2), (128, 128), (128, 256, 4), (128, 64, 1, 64), False),
]

# fused-epilogue cases at posenet_bs64 (plans as above: BN 128)
EPI_GEOMS = [("posenet_bs64.layer2", (64, 32, 32, 128, 128, 3, 1)),
             ("posenet_bs64.layer3.0.conv1", (64, 32, 32, 128, 256, 3, 2))]
# the folded shortcut of layer3.0 / layer4.0: (B, H, W, Ci, Co), merged dgrad plan (BN, items)
SHORTCUT_GEOMS = [("posenet_bs64.layer3.0", (64, 32, 32, 128, 256), (128, 512)),
                  ("posenet_bs64.layer4.0", (64, 16, 16, 256, 512), (128, 256))]

KINDS = {"fprop": 0, "dgrad": 1, "wgrad": 2}


def describe(kind, geom, precision="bf16", shortcut=False):
    """the engine's plan of one conv (host only)"""
    buf = ctypes.create_string_buffer(1 << 17)
    flags = (1 if shortcut else 0) | (2 if precision == "tc_split" else 0)
    _lib.check(_lib.lib().mapnet_test_plan_describe(kind, *geom, flags, buf, len(buf)), "mapnet_test_plan_describe")
    return json.loads(buf.value.decode())


def plan_summary(kind, geom, precision="bf16", shortcut=False):
    p = describe(kind, geom, precision, shortcut)
    if kind == 2:
        P = p["wgrad"]
        return dict(BN=P["BN"], pix=P["n_pix_tiles"], splits=P["splits"], tps=P["tiles_per_split"],
                    last=P["n_pix_tiles"] - (P["splits"] - 1) * P["tiles_per_split"])
    assert len(p["launches"]) == 1
    L = p["launches"][0]
    return dict(BN=p["BN"], items=L["n_tiles_m"] * L["n_tiles_n"] * len(L["classes"]), classes=len(L["classes"]),
                box=(L["TW"], L["TH"], L["TN"]), max_taps=max(len(c["taps"]) for c in L["classes"]),
                Cs=L["Cs"])


def expected_plan(case, kind):
    _, prec, geom, fp, dg, wg, _ = case
    s = plan_summary(KINDS[kind], geom, prec)
    if kind == "fprop":
        assert (s["BN"], s["items"]) == fp, (case[0], prec, kind, s)
    elif kind == "dgrad":
        assert (s["BN"], s["items"], s["classes"]) == dg, (case[0], prec, kind, s)
    else:
        assert (s["BN"], s["pix"], s["splits"], s["tps"]) == wg, (case[0], prec, kind, s)
    return s


def test_case_list_covers_the_benchmark_plans():
    """Host only: the case list still reaches the plans the benchmark spends its time in."""
    from geomapnet_b200 import build
    build.build(verbose=False)
    fp, dg, wg = [], [], []
    for c in CASES:
        _, prec, geom, f, d, w, _ = c
        if f is not None:
            fp.append((prec, expected_plan(c, "fprop")))
        if d is not None:
            dg.append((prec, expected_plan(c, "dgrad")))
        wg.append((prec, expected_plan(c, "wgrad")))
    for _, geom in EPI_GEOMS:
        fp.append(("epi", plan_summary(0, geom)))
        dg.append(("epi", plan_summary(1, geom)))
    for _, (B, H, W, Ci, Co), (bn, items) in SHORTCUT_GEOMS:
        s = plan_summary(1, (B, H, W, Ci, Co, 3, 2), shortcut=True)
        assert (s["BN"], s["items"], s["classes"]) == (bn, items, 4)
        dg.append(("shortcut", s))
    bf = lambda rows: [s for p, s in rows if p != "tc_split"]
    assert any(s["BN"] == 128 for s in bf(fp)), "no BN-128 fprop"
    assert any(s["BN"] == 128 for s in bf(dg)), "no BN-128 dgrad"
    assert any(s["items"] >= 3 * NSM for s in bf(fp)) and any(s["items"] >= 3 * NSM for s in bf(dg)), \
        "no fprop / dgrad with >= 3 work items per CTA"
    assert any(s["BN"] == 128 and s["classes"] == 4 for s in bf(dg)), "no merged stride-2 dgrad at BN 128"
    assert any(s["classes"] == 4 and s["BN"] == 128 for p, s in dg if p == "shortcut"), "no folded shortcut at BN 128"
    assert any(s["splits"] == 1 and s["pix"] >= 32 for s in bf(wg)), "no single-split wgrad with >= 32 pixel tiles"
    assert any(s["splits"] > 1 and s["last"] < s["tps"] for s in bf(wg)), "no multi-split wgrad with a ragged last split"
    assert any(s["box"] == (128, 1, 1) for s in bf(fp)) and any(s["box"] == (128, 1, 1) for s in bf(dg)), \
        "no 128x1 pixel box"
    assert any(s["items"] >= 16 * NSM for s in bf(fp)), "no fprop with >= 16 tiles per CTA"
    st = [s for p, s in dg if p == "tc_split"]
    assert any(s["classes"] == 4 for s in st), "no strict stride-2 dgrad (the aliased-residual launch)"
    assert any(s["splits"] == 1 for p, s in wg if p == "tc_split") and \
        any(s["splits"] > 1 for p, s in wg if p == "tc_split"), "strict wgrad: need a single- and a multi-split plan"


# ------------------------------------------------------------------------------------------------------------------
# operands and float64 references (NCHW, on the GPU)
# ------------------------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf16(shape, g, scale=1.0, positive=False):
    t = torch.randn(shape, generator=g, device="cuda")
    if positive:
        t = t.abs()
    return (t * scale).bfloat16().double()


def _logu(shape, g, scale=1.0):
    """fp32 values of magnitude in [2^-3, 2^3] (times a power-of-two scale), random sign: inside fp16's window for
    the hi/lo split"""
    e = torch.rand(shape, generator=g, device="cuda") * 6.0 - 3.0
    s = torch.where(torch.rand(shape, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    return (s * torch.exp2(e) * scale).float().double()


def _dgrad(dy, w, xshape, s, pad):
    xx = torch.zeros(xshape, dtype=torch.float64, device="cuda", requires_grad=True)
    return torch.autograd.grad(F.conv2d(xx, w, None, s, pad), xx, dy)[0]


def _wgrad(x, dy, wshape, s, pad):
    ww = torch.zeros(wshape, dtype=torch.float64, device="cuda", requires_grad=True)
    return torch.autograd.grad(F.conv2d(x, ww, None, s, pad), ww, dy)[0]


def reference(kind, x, w, dy, s, pad):
    """(value, sum |a*b|) per element, float64"""
    if kind == 0:
        return F.conv2d(x, w, None, s, pad), F.conv2d(x.abs(), w.abs(), None, s, pad)
    if kind == 1:
        return _dgrad(dy, w, x.shape, s, pad), _dgrad(dy.abs(), w.abs(), x.shape, s, pad)
    return _wgrad(x, dy, w.shape, s, pad), _wgrad(x.abs(), dy.abs(), w.shape, s, pad)


nhwc = lambda t: t.permute(0, 2, 3, 1)


def check_elements(what, got, ref, bound, max_ratio_floor=None):
    """every element within its bound (NaN fails); prints and returns max(err / bound)"""
    err = (got - ref).abs()
    ok = err <= bound
    ratio = float((err / bound).max()) if bool(ok.all()) else float("inf")
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError("%s: %d of %d elements outside the bound (%d NaN); first at index %s (shape %s): got %r "
                             "ref %r bound %r" % (what, bad.shape[0], got.numel(), int(torch.isnan(got).sum()), i,
                                                  tuple(got.shape), float(got[i]), float(ref[i]), float(bound[i])))
    print("conv-plans %-60s max err/bound %.3g" % (what, ratio))
    return ratio


def _run_ex(prec, kind, geom, in0, in1, wmat, residual, out_scale, out):
    B, H, W, Ci, Co, k, s = geom
    ptr = lambda t: t.data_ptr() if t is not None else None
    _lib.check(_lib.lib().mapnet_test_conv_ex(_lib.PREC[prec], kind, B, H, W, Ci, Co, k, s, ptr(in0), ptr(in1), ptr(wmat),
                                              ptr(residual), float(out_scale), ptr(out), _lib.stream_ptr()),
               "mapnet_test_conv_ex")
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("case,kind", [pytest.param(c, kind, id="%s-%s-%s" % (c[1], c[0], kind)) for c in CASES
                                       for kind, p in (("fprop", c[3]), ("dgrad", c[4]), ("wgrad", c[5])) if p is not None])
def test_conv_engine_at_benchmark_plan(case, kind):
    name, prec, geom, fp, dg, wg, coherent = case
    plan = expected_plan(case, kind)
    t0 = time.time()
    B, H, W, Ci, Co, k, s = geom
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    g = _gen(1000 + CASES.index(case))
    strict = prec == "tc_split"
    kk = KINDS[kind]
    if strict:
        x = _logu((B, Ci, H, W), g)
        w = _logu((Co, Ci, k, k), g)
        dy = _logu((B, Co, Ho, Wo), g)
    else:
        x = _bf16((B, Ci, H, W), g, positive=True)                          # post-ReLU activations
        w = _bf16((Co, Ci, k, k), g, (2.0 / (Ci * k * k)) ** 0.5)
        dy = _bf16((B, Co, Ho, Wo), g, positive=coherent)
    if kk == 0:
        x_in, w_in, dy_in = x, w, None
    elif kk == 1:
        x_in, w_in, dy_in = None, w, dy
    else:
        x_in, w_in, dy_in = x, None, dy
    ref, S = reference(kk, x, w, dy, s, pad)
    del x, w, dy
    act = torch.float32 if strict else torch.bfloat16
    wt = torch.float32 if strict else torch.bfloat16
    gs = 2.0 ** GSCALE if strict else 1.0
    out_scale = 2.0 ** -GSCALE if (strict and kk > 0) else 0.0
    if kk == 0:
        steps = plan["max_taps"] * plan["Cs"] // 16
        gamma = steps * TRUNC + (2 * SPLIT + SPLIT ** 2 if strict else 0.0)
        out = torch.full((B, Ho, Wo, Co), float("nan"), dtype=act, device="cuda")
        _run_ex(prec, 0, geom, nhwc(x_in).contiguous().to(act), None,
                w_in.permute(0, 2, 3, 1).contiguous().to(wt), None, 0.0, out)
        ref, S = nhwc(ref), nhwc(S)
        u = 0.0 if strict else U_BF16          # strict mode stores the fp32 accumulator as it is
        bound = u * ref.abs() + (1 + u) * gamma * S
        got = out.double()
    elif kk == 1:
        steps = plan["max_taps"] * plan["Cs"] // 16
        gamma = steps * TRUNC + (2 * SPLIT + SPLIT ** 2 if strict else 0.0)
        ref, S = nhwc(ref), nhwc(S)
        res = None
        if strict:
            # the residual (the downsample branch's dgrad in the trunk) is read from the output buffer in place
            res = torch.randn(ref.shape, generator=g, device="cuda") * float(ref.std())
            out = res.clone()
            _run_ex(prec, 1, geom, (nhwc(dy_in) * gs).contiguous().to(act), None,
                    w_in.permute(1, 2, 3, 0).contiguous().to(wt), out, out_scale, out)
            res = res.double()
            ref = ref + res
            bound = U_FP32 * (ref.abs() + 2 * res.abs()) + (1 + U_FP32) * gamma * S
        else:
            out = torch.full((B, H, W, Ci), float("nan"), dtype=act, device="cuda")
            _run_ex(prec, 1, geom, nhwc(dy_in).contiguous().to(act), None,
                    w_in.permute(1, 2, 3, 0).contiguous().to(wt), None, 0.0, out)
            bound = U_BF16 * ref.abs() + (1 + U_BF16) * gamma * S
        got = out.double()
        del res
    else:
        # 4 wgmma steps per 64-pixel tile; strict mode: the four hi/lo cells are summed with 3 fp32 adds
        gamma = 4 * plan["tps"] * TRUNC + (plan["splits"] if plan["splits"] > 1 else 0) * U_FP32
        if strict:
            gamma += 2 * SPLIT + SPLIT ** 2 + 3 * U_FP32
        ref, S = ref.permute(0, 2, 3, 1), S.permute(0, 2, 3, 1)                # [Co][k][k][Ci]
        dw0 = (torch.randn(ref.shape, generator=g, device="cuda") * float(ref.std())).float()
        out = dw0.clone()
        _run_ex(prec, 2, geom, nhwc(x_in).contiguous().to(act), (nhwc(dy_in) * gs).contiguous().to(act), None, None,
                out_scale, out)
        dw0 = dw0.double()
        got = out.double() - dw0                                                 # exact in float64
        bound = U_FP32 * (dw0.abs() + ref.abs()) + (1 + U_FP32) * gamma * S
    what = "%s %s %s %s BN%d" % (prec, name, kind, geom, plan["BN"])
    check_elements(what, got, ref, bound)
    print("conv-plans %-60s %.1f s" % (what, time.time() - t0))


# ------------------------------------------------------------------------------------------------------------------
# fused epilogues at BN 128
# ------------------------------------------------------------------------------------------------------------------
def _sum_bound(stored_abs_terms, tiles_per_cta):
    """fp32 chain of the epilogue's column sums: 4 rows per lane, 3 shuffle levels, one add per tile of the CTA, 3
    adds across the four epilogue warps (the fp64 replica atomics add nothing measurable)"""
    return (4 + 3 + tiles_per_cta + 3 + 1) * U_FP32 * stored_abs_terms + 1e-30


def _run_epilogue(kind, geom, in0, wmat, residual, y, zmask, yd, mscale, mshift, out, C):
    import numpy as np
    B, H, W, Ci, Co, k, stride = geom
    sums = np.zeros((3, C), dtype=np.float64)
    ptr = lambda t: t.data_ptr() if t is not None else None
    _lib.check(_lib.lib().mapnet_test_conv_epilogue(
        kind, B, H, W, Ci, Co, k, stride, ptr(in0), ptr(wmat), ptr(residual), ptr(y), ptr(zmask), ptr(yd), ptr(mscale),
        ptr(mshift), ptr(out), sums.ctypes.data_as(ctypes.c_void_p), _lib.stream_ptr()), "mapnet_test_conv_epilogue")
    torch.cuda.synchronize()
    return torch.from_numpy(sums).cuda()


def _check_sums(what, got, ref, bound):
    err = (got - ref).abs()
    assert bool((err <= bound).all()), "%s: channel sums off: max err %g, worst channel %d (got %r ref %r bound %r)" % (
        what, float(err.max()), int((err / bound).argmax()), float(got.flatten()[int((err / bound).argmax())]),
        float(ref.flatten()[int((err / bound).argmax())]), float(bound.flatten()[int((err / bound).argmax())]))
    print("conv-plans %-60s sums max err/bound %.3g" % (what, float((err / bound).max())))


@pytest.mark.gpu
@pytest.mark.parametrize("name,geom", EPI_GEOMS, ids=[e[0] for e in EPI_GEOMS])
def test_fprop_batchnorm_statistics_at_bn128(name, geom):
    B, H, W, Ci, Co, k, s = geom
    plan = plan_summary(0, geom)
    assert plan["BN"] == 128
    pad = (k - 1) // 2
    g = _gen(7)
    x = _bf16((B, Ci, H, W), g, positive=True)
    w = _bf16((Co, Ci, k, k), g, (2.0 / (Ci * k * k)) ** 0.5)
    ref, S = (nhwc(t) for t in reference(0, x, w, None, s, pad))
    out = torch.full(ref.shape, float("nan"), dtype=torch.bfloat16, device="cuda")
    sums = _run_epilogue(0, geom, nhwc(x).contiguous().bfloat16(), w.permute(0, 2, 3, 1).contiguous().bfloat16(),
                         None, None, None, None, None, None, out, Co)
    del x, w
    gamma = plan["max_taps"] * plan["Cs"] // 16 * TRUNC
    got = out.double()
    check_elements("bf16 %s fprop+stats BN128" % name, got, ref, U_BF16 * ref.abs() + (1 + U_BF16) * gamma * S)
    st = got.reshape(-1, Co)
    tpc = math.ceil(plan["items"] / NSM)
    _check_sums("bf16 %s fprop sum" % name, sums[0], st.sum(0), _sum_bound(st.abs().sum(0), tpc))
    _check_sums("bf16 %s fprop sum sq" % name, sums[1], (st * st).sum(0), _sum_bound((st * st).sum(0), tpc + 1))


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["ymask", "zmask_res", "zmask_res_yd"])
@pytest.mark.parametrize("name,geom", EPI_GEOMS, ids=[e[0] for e in EPI_GEOMS])
def test_dgrad_gate_residual_and_batchnorm_sums_at_bn128(name, geom, variant):
    B, H, W, Ci, Co, k, s = geom
    plan = plan_summary(1, geom)
    assert plan["BN"] == 128
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    g = _gen(8)
    w = _bf16((Co, Ci, k, k), g, (2.0 / (Ci * k * k)) ** 0.5)
    dy = _bf16((B, Co, Ho, Wo), g)
    dx, S = (nhwc(t) for t in reference(1, torch.empty(B, Ci, H, W, dtype=torch.float64, device="cuda"), w, dy, s, pad))
    shape = (B, H, W, Ci)
    ybn = torch.randn(shape, generator=g, device="cuda").bfloat16()       # the consumer BatchNorm's input
    ydn = torch.randn(shape, generator=g, device="cuda").bfloat16()
    res = torch.randn(shape, generator=g, device="cuda").bfloat16()
    msc = torch.rand(Ci, generator=g, device="cuda") + 0.5
    msh = torch.randn(Ci, generator=g, device="cuda") * 0.3
    z = torch.relu(torch.randn(shape, generator=g, device="cuda")).bfloat16()
    use_z, use_res, use_yd = variant != "ymask", "res" in variant, variant.endswith("yd")
    out = torch.full(shape, float("nan"), dtype=torch.bfloat16, device="cuda")
    sums = _run_epilogue(1, geom, nhwc(dy).contiguous().bfloat16(), w.permute(1, 2, 3, 0).contiguous().bfloat16(),
                         res if use_res else None, ybn, z if use_z else None, ydn if use_yd else None,
                         None if use_z else msc, None if use_z else msh, out, Ci)
    del w, dy
    gamma = plan["max_taps"] * plan["Cs"] // 16 * TRUNC
    r = res.double() if use_res else torch.zeros_like(dx)
    v = dx + r
    bound = U_BF16 * v.abs() + (1 + U_BF16) * (gamma * S + U_FP32 * (dx.abs() + r.abs() + gamma * S))
    got = out.double()
    if use_z:
        gate, amb = z.double() > 0, torch.zeros(shape, dtype=torch.bool, device="cuda")
    else:
        t = ybn.double() * msc.double() + msh.double()
        gate = t > 0
        amb = t.abs() <= 2.0 ** -20 * (ybn.double().abs() * msc.double() + msh.double().abs())   # either branch
    assert float(amb.double().mean()) < 1e-4
    closed = ~gate & ~amb
    assert bool((got[closed] == 0).all()), "%s %s: a closed gate stored a nonzero" % (name, variant)
    ref = torch.where(gate, v, torch.zeros_like(v))
    ref = torch.where(amb & (got == 0), torch.zeros_like(v), ref)
    ref = torch.where(amb & (got != 0), v, ref)
    check_elements("bf16 %s dgrad %s BN128" % (name, variant), got, ref, bound)
    st = got.reshape(-1, Ci)
    yy, yd2 = ybn.double().reshape(-1, Ci), ydn.double().reshape(-1, Ci)
    tpc = math.ceil(plan["items"] / NSM)
    _check_sums("bf16 %s %s sum g" % (name, variant), sums[0], st.sum(0), _sum_bound(st.abs().sum(0), tpc))
    _check_sums("bf16 %s %s sum g*y" % (name, variant), sums[1], (st * yy).sum(0),
                _sum_bound((st * yy).abs().sum(0), tpc + 1))
    if use_yd:
        _check_sums("bf16 %s %s sum g*yd" % (name, variant), sums[2], (st * yd2).sum(0),
                    _sum_bound((st * yd2).abs().sum(0), tpc + 1))


@pytest.mark.gpu
@pytest.mark.parametrize("name,geom,expect", SHORTCUT_GEOMS, ids=[e[0] for e in SHORTCUT_GEOMS])
def test_folded_shortcut_dgrad_at_bn128(name, geom, expect):
    B, H, W, Ci, Co = geom
    plan = plan_summary(1, (B, H, W, Ci, Co, 3, 2), shortcut=True)
    assert (plan["BN"], plan["items"], plan["classes"]) == expect + (4,)
    g = _gen(9)
    w1 = _bf16((Co, Ci, 3, 3), g, (2.0 / (Ci * 9)) ** 0.5)
    w2 = _bf16((Co, Ci, 1, 1), g, (2.0 / Ci) ** 0.5)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dy1 = _bf16((B, Co, Ho, Wo), g)
    dy2 = _bf16((B, Co, Ho, Wo), g)
    xs = (B, Ci, H, W)
    ref = nhwc(_dgrad(dy1, w1, xs, 2, 1) + _dgrad(dy2, w2, xs, 2, 0))
    S = nhwc(_dgrad(dy1.abs(), w1.abs(), xs, 2, 1) + _dgrad(dy2.abs(), w2.abs(), xs, 2, 0))
    out = torch.full((B, H, W, Ci), float("nan"), dtype=torch.bfloat16, device="cuda")
    d1, d2 = nhwc(dy1).contiguous().bfloat16(), nhwc(dy2).contiguous().bfloat16()        # alive until the call returns
    m1, m2 = w1.permute(1, 2, 3, 0).contiguous().bfloat16(), w2.permute(1, 2, 3, 0).contiguous().bfloat16()
    _lib.check(_lib.lib().mapnet_test_dgrad_shortcut(B, H, W, Ci, Co, d1.data_ptr(), d2.data_ptr(), m1.data_ptr(),
                                                     m2.data_ptr(), out.data_ptr(), _lib.stream_ptr()),
               "mapnet_test_dgrad_shortcut")
    torch.cuda.synchronize()
    gamma = plan["max_taps"] * plan["Cs"] // 16 * TRUNC           # class (0, 0): 4 taps + the shortcut tap
    check_elements("bf16 %s dgrad+shortcut BN128" % name, out.double(), ref, U_BF16 * ref.abs() + (1 + U_BF16) * gamma * S)
