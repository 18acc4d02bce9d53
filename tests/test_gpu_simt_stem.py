"""The CUDA-core conv engines (csrc/conv_simt.cu: every conv of precision fp32 and bf16_simt) and the im2col stem
(k_stem_im2col, the 1x1 GEMM view of the stem over its [B*Hc*Wc][192] patch matrix, k_unpack_wgrads: the stem of the
CUDA-core modes and the fallback stem of the tensor-core modes), one launch sequence at a time, checked element by
element against float64; then the tensor-core training step run on the im2col stem against the reference goldens.

A. CUDA-core engines (mapnet_test_conv_simt, launched as Net::conv_fprop / conv_dgrad / conv_wgrad launch them).
Cases: the distinct ResNet-34 geometries of posenet_bs64 (test_gpu_conv_plans.CASES), mapnetpp_n16t10 layer1
(B = 160), the 7Scenes 256x341 geometries at B = 4 (widths 86 / 43 / 11; layer4's M = 352 is not a multiple of the
64-row tile), the stem's GEMM view at posenet_bs64 and 7Scenes, and tails the engine's contract allows (Ci / Co of 4,
12 and 20: N not a multiple of 64, K not a multiple of 16; a 2x7x5 map at stride 2).  Every case runs fprop, dgrad
with a separate residual and in place (residual == out, as Net::backward_t's conv_dgrad(conv1, S1, S0, S0)), and
wgrad into a nonzero dW0.  The wgrad split plan is replicated on the host (`simt_wgrad_plan`, launch_conv_simt_wgrad's
formula) so the case list provably reaches a single split that adds into dW (posenet_bs64 layer4), split counts of
50 - 180 through the workspace and launch_split_reduce with a short last split (7Scenes layer1: 58 splits of 384 pixels
over 22 016; the stem view: 176), and the kchunk = 256 clamp.

  Exact cases.  Activations and gradients in {-3..3} / 4, weights (256 a + b) / 1024 with a in {-3..3}, b in
  {-1, 0, 1} (10 significant bits: not representable in bf16, so an engine or pack that read the bf16_simt weights as
  bf16 fails), integer residuals and dW0.  Every product is a multiple of 2^-12 and every partial sum is below 2^24
  such units (K <= 4608 terms of at most 3 * 769), so every fp32 sum is exact in any order: fp32 outputs must equal the
  float64 reference exactly, bf16 outputs its round-to-nearest-even.  wgrad: products are multiples of 2^-4, at most
  9 such units, over at most 2^20 pixels.  This is what catches index, tap, parity and tail bugs: one dropped term of a
  K = 4608 sum is about the size of the worst-case bound below.

  Random cases.  Signed normal operands; bf16_simt rounds activations / gradients / residuals to bf16 (they are stored
  so) and keeps the weights in fp32 as given.  Reference on the decoded stored operands; S = the same ops on |a|, |b|.
    |got - ref| <= u_store |ref| + (1 + u_store) (gamma_n S + E_res)
  * fprop / dgrad: one fmaf chain per output over K = taps * channels terms in k order (zero-padded terms add exact
    zeros): each fmaf rounds once, so |acc - ref| <= gamma_K S with gamma_n = n u / (1 - n u), u = 2^-24.
  * dgrad residual: v = acc + res, one more rounding: E_res = u (S + |res|) bounds u |acc + res| to first order.
  * store: fp32 as computed (u_store = 0); bf16 round-to-nearest, u_store = 2^-8 relative to the stored value, hence
    relative to |ref| plus (1 + u_store) times the accumulation error.
  * wgrad: each split is a chain of at most kchunk fmaf; k_wgrad_reduce adds the splits in order (splits - 1 adds after
    the first) and then adds that sum into dW (one add; a single split adds its accumulator into dW directly), so
    |(out - dW0) - ref| <= gamma_(kchunk + splits + 1) (S + |dW0|), out - dW0 formed exactly in float64.
  A fprop / dgrad output is NaN before the launch (the in-place dgrad's holds its residual), so an element that is never
  written fails; the fp32 wgrad is run twice from the same dW0 and must agree bit for bit; `test_wgrad_split_order`
  pins k_wgrad_reduce's order with partials whose fp32 sum depends on it.

B. The im2col stem (mapnet_test_stem_im2col) in fp32, bf16_simt, bf16 and tc_split at posenet_bs64 (B = 64),
mapnet_n32t3 (96), 7Scenes (B = 4, 256x341: Wc = 171 is odd), a 97x65 frame (the zero halo reaches both edges) and
the widest frame launch_stem_im2col's 48 KB of shared memory allows (W = 570: 21 staged rows of W + 6 floats plus the
192-entry k -> offset table; 579, which a check that left the table out used to accept, failed at launch).
  * patch matrix, bit for bit against F.unfold of x reordered to k = (kh*7 + kw)*3 + c: fp32 exactly, bf16 its
    round-to-nearest-even, tc_split the fp16 hi / lo planes split_f16 makes (hi = fp16(x), lo = fp16(x - hi); also
    |hi + lo - x| <= max(2^-22 |x|, 2^-25)); columns 147..191 all-zero bit patterns.
  * fprop, per element, K = 192: the CUDA-core modes one fmaf chain (gamma_192); bf16 12 truncating wgmma instructions
    (2^-23 relative each); tc_split the plan's taps x split channels / 16 instructions plus 2 * 2^-22 + 2^-44 of the
    hi / lo split of both operands (x, w, dy drawn with magnitudes in [2^-3, 2^3]; zeros split exactly), fp32 store.
    The bf16 modes' weights are the pack's bf16 roundings (bf16_simt's pack rounds its fp32 row too).
  * BatchNorm statistics of the tensor-core epilogue, as tests/test_gpu_stem_head.py checks them.
  * wgrad in the [64,3,7,7] .grad layout (NaN before the call, so a padded column leaking through k_unpack_wgrads or a
    missed element fails): the CUDA-core chain as in A; the tensor cores 4 truncating instructions per 64-pixel tile,
    tiles_per_split tiles, and one fp32 add per split when there are several (strict: + the split and the 3 adds of
    the four hi / lo cells; dy arrives scaled by 2^8 and out_scale = 2^-8 is exact).
  * exact cases in all four modes: x, w, dy in {-3..3} / 4 are exact in bf16 and split exactly into hi + lo = x,
    lo = 0, so every mode's stem output and gradient is fully determined (at most 147 * 9 units of 2^-4 per output,
    2^20 * 9 per gradient element).
  * tensor-core plans asserted from mapnet_test_plan_describe(kind, B, Hc, Wc, 192, 64, 1, 1, flags).

C. The tensor-core training step on the im2col stem: a fixture replaces _lib.Trunk by a handle made with
mapnet_test_trunk_create(..., im2col_stem = 1) -- the stem Net falls back to when the driver rejects overlapped tensor
maps -- and the golden steps of tests/test_gpu_step.py run through tests/helpers.py at that file's tolerances.  A
profiler trace of one step shows that the patched handle runs k_stem_im2col and no k_stem_s2d (and the unpatched one
the opposite).

Every check prints max(err / bound), or that it is exact.
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

import test_gpu_conv_plans as CP
import test_gpu_step as STEP

NSM = 132
U_BF16 = 2.0 ** -8
U_FP32 = 2.0 ** -24
TRUNC = 2.0 ** -23          # one ulp per truncating wgmma accumulation
SPLIT = 2.0 ** -22          # hi/lo fp16 split of one operand
GSCALE = 8                  # strict-mode gradients arrive scaled by 2^GSCALE; the wgrad multiplies by 2^-GSCALE
SIMT_PREC = ["fp32", "bf16_simt"]
TRAIN_PREC = ["fp32", "bf16_simt", "bf16", "tc_split"]
KINDS = {"fprop": 0, "dgrad": 1, "wgrad": 2}
STEM_K = 192                # the patch-matrix row: 7 * 7 * 3 = 147 taps padded to 192


def _model_cases():
    """the CUDA-core cases of A: (id, (B, H, W, Ci, Co, k, stride))"""
    out, seen = [], set()
    for name, prec, geom, *_ in CP.CASES:
        if prec != "bf16" or name.endswith(".coherent") or geom in seen:
            continue
        if name.startswith(("posenet_bs64.", "7scenes_b4.")) or name == "mapnetpp_n16t10.layer1":
            out.append((name, geom))
            seen.add(geom)
    return out


CONV_CASES = _model_cases() + [
    ("posenet_bs64.stem_view", (64, 128, 128, STEM_K, 64, 1, 1)),
    ("7scenes_b4.stem_view", (4, 128, 171, STEM_K, 64, 1, 1)),
    ("tail.c4_c12", (3, 9, 11, 4, 12, 3, 1)),
    ("tail.c12_c20_s2", (2, 13, 7, 12, 20, 3, 2)),
    ("tail.c20_c4_1x1s2", (2, 10, 9, 20, 4, 1, 2)),
    ("tail.map2x7x5_s2", (2, 7, 5, 20, 12, 3, 2)),
]

# (id, (B, H, W), {precision: (fprop plan (BN, items, taps, Cs), wgrad plan (BN, pixel tiles, splits, tiles/split))})
# -- the tensor-core plans of the stem's GEMM view (Hc x Wc pixels, Ci = 192, 1x1)
STEM_CASES = [
    ("posenet_bs64", (64, 256, 256), {"bf16": ((64, 8192, 1, 192), (64, 16384, 132, 125)),
                                      "tc_split": ((64, 8192, 2, 384), (128, 16384, 88, 187))}),
    ("mapnet_n32t3", (96, 256, 256), {"bf16": ((64, 12288, 1, 192), (64, 24576, 132, 187)),
                                      "tc_split": ((64, 12288, 2, 384), (128, 24576, 88, 280))}),
    ("7scenes_b4", (4, 256, 341), {"bf16": ((64, 1024, 1, 192), (64, 1536, 128, 12)),
                                   "tc_split": ((64, 1024, 2, 384), (128, 1536, 86, 18))}),
    ("halo_97x65", (3, 97, 65), {"bf16": ((64, 75, 1, 192), (64, 147, 74, 2)),
                                 "tc_split": ((64, 75, 2, 384), (128, 147, 74, 2))}),
    ("widest_64x570", (2, 64, 570), {"bf16": ((64, 192, 1, 192), (64, 320, 107, 3)),
                                     "tc_split": ((64, 192, 2, 384), (128, 320, 80, 4))}),
]
MAX_IM2COL_W = 570          # 21 staged rows of W + 6 floats and the 192-entry table in 48 KB of shared memory


# ------------------------------------------------------------------------------------------------------------------
# host-side geometry and plans
# ------------------------------------------------------------------------------------------------------------------
def cdiv(a, b):
    return -(-a // b)


def out_hw(geom):
    B, H, W, Ci, Co, k, s = geom
    p = (k - 1) // 2
    return (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1


def simt_wgrad_plan(geom):
    """launch_conv_simt_wgrad's split-K plan: (splits, kchunk, pixels of the last split, kchunk clamped to 256)"""
    B, H, W, Ci, Co, k, s = geom
    Ho, Wo = out_hw(geom)
    gm, gn = cdiv(Co, 64), cdiv(k * k * Ci, 64)
    Kt = B * Ho * Wo
    splits = max(1, NSM * 4 // (gm * gn))
    kchunk = cdiv(cdiv(Kt, splits), 16) * 16
    clamped = kchunk < 256
    kchunk = max(kchunk, 256)
    splits = cdiv(Kt, kchunk)
    return splits, kchunk, Kt - (splits - 1) * kchunk, clamped


def stem_hw(H, W):
    return (H - 1) // 2 + 1, (W - 1) // 2 + 1


def stem_view_plan(kind, B, Hc, Wc, precision):
    buf = ctypes.create_string_buffer(1 << 17)
    flags = 2 if precision == "tc_split" else 0
    _lib.check(_lib.lib().mapnet_test_plan_describe(kind, B, Hc, Wc, STEM_K, 64, 1, 1, flags, buf, len(buf)),
               "mapnet_test_plan_describe")
    p = json.loads(buf.value.decode())
    if kind == 2:
        P = p["wgrad"]
        return (P["BN"], P["n_pix_tiles"], P["splits"], P["tiles_per_split"])
    assert len(p["launches"]) == 1
    L = p["launches"][0]
    return (p["BN"], L["n_tiles_m"] * L["n_tiles_n"], len(L["classes"][0]["taps"]), L["Cs"])


# ------------------------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------------------------
def check_elements(what, got, ref, bound):
    """every element within its bound (NaN fails); prints and returns max(err / bound)"""
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
    print("simt-stem %-64s max err/bound %.3g" % (what, ratio))
    return ratio


def check_exact(what, got, ref):
    """got == ref element for element (float64 values; NaN fails)"""
    same = got == ref
    if not bool(same.all()):
        bad = (~same).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError("%s: %d of %d elements differ from the exact result (%d NaN); first at index %s (shape %s): "
                             "got %r ref %r" % (what, bad.shape[0], got.numel(), int(torch.isnan(got).sum()), i,
                                                tuple(got.shape), float(got[i]), float(ref[i])))
    print("simt-stem %-64s exact (%d elements)" % (what, got.numel()))


def gamma(n):
    return n * U_FP32 / (1.0 - n * U_FP32)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ints(shape, g, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").double()


def _logu(shape, g):
    """fp32 values of magnitude in [2^-3, 2^3], random sign: inside fp16's window for the hi/lo split"""
    e = torch.rand(shape, generator=g, device="cuda") * 6.0 - 3.0
    s = torch.where(torch.rand(shape, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    return (s * torch.exp2(e)).float()


def _sum_bound(stored_abs_terms, tiles_per_cta):
    return (4 + 3 + tiles_per_cta + 3 + 1) * U_FP32 * stored_abs_terms + 1e-30


nhwc = lambda t: t.permute(0, 2, 3, 1)
nchw = lambda t: t.permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------------------------
# A. CUDA-core engines
# ------------------------------------------------------------------------------------------------------------------
def run_simt(prec, kind, geom, in0, in1, wmat, residual, out):
    B, H, W, Ci, Co, k, s = geom
    ptr = lambda t: None if t is None else t.data_ptr()
    _lib.check(_lib.lib().mapnet_test_conv_simt(_lib.PREC[prec], kind, B, H, W, Ci, Co, k, s, ptr(in0), ptr(in1),
                                                ptr(wmat), ptr(residual), ptr(out), _lib.stream_ptr()),
               "mapnet_test_conv_simt")


def conv_refs(geom, x, w, dy, absolute=False):
    """float64 fprop, dgrad and wgrad (.grad layout [Co][Ci][k][k]) of NCHW operands"""
    B, H, W, Ci, Co, k, s = geom
    p = (k - 1) // 2
    if absolute:
        x, w, dy = x.abs(), w.abs(), dy.abs()
    y = F.conv2d(x, w, None, s, p)
    dx = torch.nn.grad.conv2d_input(x.shape, w, dy, s, p)
    dw = torch.nn.grad.conv2d_weight(x, w.shape, dy, s, p)
    return y, dx, dw


def engine_outputs(prec, geom, x, w, dy, res, dw0, twice=False):
    """the engine's fprop, dgrad (separate residual), dgrad in place and wgrad of float64 NCHW operands already on the
    stored grid; returns float64 NCHW / [Co][Ci][k][k] tensors"""
    act = torch.float32 if prec == "fp32" else torch.bfloat16
    B, H, W, Ci, Co, k, s = geom
    Ho, Wo = out_hw(geom)
    xs = nhwc(x).contiguous().to(act)
    dys = nhwc(dy).contiguous().to(act)
    ress = nhwc(res).contiguous().to(act)
    w_krsc = w.permute(0, 2, 3, 1).contiguous().float()
    w_dg = w.permute(1, 2, 3, 0).contiguous().float()
    out = {}
    y = torch.full((B, Ho, Wo, Co), float("nan"), dtype=act, device="cuda")
    run_simt(prec, 0, geom, xs, None, w_krsc, None, y)
    out["fprop"] = nchw(y.double())
    dx = torch.full((B, H, W, Ci), float("nan"), dtype=act, device="cuda")
    run_simt(prec, 1, geom, dys, None, w_dg, ress, dx)
    out["dgrad"] = nchw(dx.double())
    dxi = ress.clone()
    run_simt(prec, 1, geom, dys, None, w_dg, dxi, dxi)
    out["dgrad_inplace"] = nchw(dxi.double())
    dw = dw0.permute(0, 2, 3, 1).contiguous().float()
    run_simt(prec, 2, geom, xs, dys, None, None, dw)
    out["wgrad"] = dw.permute(0, 3, 1, 2).double()
    if twice:
        dw2 = dw0.permute(0, 2, 3, 1).contiguous().float()
        run_simt(prec, 2, geom, xs, dys, None, None, dw2)
        assert torch.equal(dw.view(torch.int32), dw2.view(torch.int32)), "fp32 wgrad differs between two runs"
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SIMT_PREC)
@pytest.mark.parametrize("name,geom", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_cuda_core_engines(name, geom, prec):
    t0 = time.time()
    B, H, W, Ci, Co, k, s = geom
    Ho, Wo = out_hw(geom)
    splits, kchunk, last, clamped = simt_wgrad_plan(geom)
    what = "%s %s %s" % (prec, name, geom)
    g = _gen(5000 + CONV_CASES.index((name, geom)) * 2 + SIMT_PREC.index(prec))
    rnd = lambda t: t if prec == "fp32" else t.float().bfloat16().double()

    # ---- exact operands ----
    x = _ints((B, Ci, H, W), g, -3, 3) / 4
    w = (_ints((Co, Ci, k, k), g, -3, 3) * 256 + _ints((Co, Ci, k, k), g, -1, 1)) / 1024
    dy = _ints((B, Co, Ho, Wo), g, -3, 3) / 4
    res = _ints((B, Ci, H, W), g, -4, 4)
    dw0 = _ints((Co, Ci, k, k), g, -4, 4)
    got = engine_outputs(prec, geom, x, w, dy, res, dw0)
    y, dx, dw = conv_refs(geom, x, w, dy)
    store = (lambda t: t) if prec == "fp32" else (lambda t: t.float().bfloat16().double())
    check_exact(what + " exact fprop", got["fprop"], store(y))
    del y
    check_exact(what + " exact dgrad + residual", got["dgrad"], store(dx + res))
    check_exact(what + " exact dgrad in place", got["dgrad_inplace"], store(dx + res))
    del dx
    check_exact(what + " exact wgrad (%d splits of %d)" % (splits, kchunk), got["wgrad"], dw0 + dw)
    del got, dw

    # ---- random operands ----
    x = rnd(torch.randn((B, Ci, H, W), generator=g, device="cuda").double())
    w = (torch.randn((Co, Ci, k, k), generator=g, device="cuda") * (2.0 / (Ci * k * k)) ** 0.5).double()
    dy = rnd(torch.randn((B, Co, Ho, Wo), generator=g, device="cuda").double())
    res = rnd(torch.randn((B, Ci, H, W), generator=g, device="cuda").double())
    dw0 = torch.randn((Co, Ci, k, k), generator=g, device="cuda").double()
    got = engine_outputs(prec, geom, x, w, dy, res, dw0, twice=prec == "fp32")
    assert torch.equal(got["dgrad"], got["dgrad_inplace"]), what + ": dgrad in place differs from a separate residual"
    u = 0.0 if prec == "fp32" else U_BF16
    y, dx, dw = conv_refs(geom, x, w, dy)
    Sy, Sdx, Sdw = conv_refs(geom, x, w, dy, absolute=True)
    check_elements(what + " fprop", got["fprop"], y, u * y.abs() + (1 + u) * gamma(k * k * Ci) * Sy)
    del y, Sy
    ref = dx + res
    check_elements(what + " dgrad + residual", got["dgrad"], ref,
                   u * ref.abs() + (1 + u) * (gamma(k * k * Co) * Sdx + U_FP32 * (Sdx + res.abs())))
    del dx, Sdx, ref
    check_elements(what + " wgrad (%d splits of %d, last %d)" % (splits, kchunk, last), got["wgrad"] - dw0, dw,
                   gamma(kchunk + splits + 1) * (Sdw + dw0.abs()))
    print("simt-stem %-64s %.1f s" % (what, time.time() - t0))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", SIMT_PREC)
def test_wgrad_split_order(prec):
    """k_wgrad_reduce adds the splits of launch_conv_simt_wgrad in order 0, 1, ... and then adds that sum into dW.  With
    x = 1 and dy nonzero only at the first pixel of each split, split z's partial is exactly dy there: 2^24 for split 0
    and 1 for the others, so s = 2^24 in that order (each + 1 is a tie that rounds to even), while the reversed order
    sums the 175 ones first and gives 2^24 + 176.  With dW0 = 3 the in-order result is 2^24 + 4."""
    geom = (64, 128, 128, STEM_K, 64, 1, 1)           # the stem view: 176 splits
    B, H, W, Ci, Co, k, s = geom
    splits, kchunk, last, _ = simt_wgrad_plan(geom)
    assert splits > 100
    act = torch.float32 if prec == "fp32" else torch.bfloat16
    x = torch.ones((B, H, W, Ci), dtype=act, device="cuda")
    dy = torch.zeros((B * H * W, Co), dtype=act, device="cuda")
    dy[0] = 2.0 ** 24
    dy[kchunk * torch.arange(1, splits, device="cuda")] = 1.0
    dw0 = torch.full((Co, 1, 1, Ci), 3.0, dtype=torch.float32, device="cuda")
    dw = dw0.clone()
    run_simt(prec, 2, geom, x, dy.view(B, H, W, Co), None, None, dw)
    torch.cuda.synchronize()
    sacc = np.float32(0.0)
    for z in range(splits):
        sacc = np.float32(sacc + np.float32(2.0 ** 24 if z == 0 else 1.0))
    want = float(np.float32(np.float32(3.0) + sacc))
    assert want == 2.0 ** 24 + 4.0        # the in-order sum; the reversed order gives 2^24 + 180
    vals = torch.unique(dw)
    assert vals.numel() == 1 and float(vals[0]) == want, (prec, vals[:8].tolist(), want)
    print("simt-stem %-64s in order (%d splits of %d)" % ("%s wgrad split order" % prec, splits, kchunk))


# ------------------------------------------------------------------------------------------------------------------
# B. the im2col stem
# ------------------------------------------------------------------------------------------------------------------
def im2col_ref(x):
    """[B*Hc*Wc][147] patch matrix of NCHW x, k = (kh*7 + kw)*3 + c"""
    B = x.shape[0]
    u = F.unfold(x, 7, padding=3, stride=2)                # [B, 3*49, L], row c*49 + kh*7 + kw
    return u.view(B, 3, 49, -1).permute(0, 3, 2, 1).reshape(-1, 147)


def decode_split(a, M):
    """hsplit patch matrix -> (hi, lo) fp16 [M][192]: per 8 channels 8 hi then 8 lo"""
    p = a.view(torch.float16).view(M, STEM_K // 8, 2, 8)
    return p[:, :, 0, :].reshape(M, STEM_K), p[:, :, 1, :].reshape(M, STEM_K)


def check_patch_matrix(what, prec, A, x, M):
    ref = im2col_ref(x)
    if prec == "tc_split":
        hi, lo = decode_split(A, M)
        rh = ref.half()
        rl = (ref - rh.float()).half()
        for name, got, want in (("hi", hi[:, :147], rh), ("lo", lo[:, :147], rl)):
            same = got.view(torch.int16) == want.view(torch.int16)
            assert bool(same.all()), "%s: patch matrix %s plane differs in %d elements" % (what, name, int((~same).sum()))
        err = (hi[:, :147].double() + lo[:, :147].double() - ref.double()).abs()
        assert bool((err <= torch.clamp(ref.double().abs() * SPLIT, min=2.0 ** -25)).all()), what
        pad = torch.cat([hi[:, 147:], lo[:, 147:]], 1).view(torch.int16)
    else:
        want = ref if prec == "fp32" else ref.bfloat16()
        bits = torch.int32 if prec == "fp32" else torch.int16
        same = A[:, :147].view(bits) == want.view(bits)
        assert bool(same.all()), "%s: patch matrix differs in %d elements" % (what, int((~same).sum()))
        pad = A[:, 147:].view(bits)
    assert bool((pad == 0).all()), "%s: %d nonzero padding columns" % (what, int((pad != 0).sum()))
    print("simt-stem %-64s patch matrix bitwise (%d x 192)" % (what, M))


def run_stem(prec, B, H, W, x, w, dy_in, out_scale, sums, want_a):
    Hc, Wc = stem_hw(H, W)
    M = B * Hc * Wc
    yt = torch.float32 if prec in ("fp32", "tc_split") else torch.bfloat16
    at = {"fp32": torch.float32, "bf16_simt": torch.bfloat16, "bf16": torch.bfloat16, "tc_split": torch.int32}[prec]
    A = torch.empty((M, STEM_K), dtype=at, device="cuda") if want_a else None
    y = torch.full((B, Hc, Wc, 64), float("nan"), dtype=yt, device="cuda")
    dw = torch.full((64, 3, 7, 7), float("nan"), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().mapnet_test_stem_im2col(
        _lib.PREC[prec], B, H, W, x.data_ptr(), w.data_ptr(), None if A is None else A.data_ptr(), y.data_ptr(),
        dy_in.data_ptr(), dw.data_ptr(), float(out_scale),
        None if sums is None else sums.ctypes.data_as(ctypes.c_void_p), _lib.stream_ptr()), "mapnet_test_stem_im2col")
    torch.cuda.synchronize()
    return A, y, dw


def _stem_wgrad(x, dy):
    ww = torch.zeros((64, 3, 7, 7), dtype=torch.float64, device="cuda", requires_grad=True)
    return torch.autograd.grad(F.conv2d(x, ww, None, 2, 3), ww, dy)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", TRAIN_PREC)
@pytest.mark.parametrize("case", STEM_CASES, ids=[c[0] for c in STEM_CASES])
def test_im2col_stem(case, prec):
    name, (B, H, W), plans = case
    t0 = time.time()
    Hc, Wc = stem_hw(H, W)
    M = B * Hc * Wc
    tc = prec in ("bf16", "tc_split")
    strict = prec == "tc_split"
    if tc:
        fplan = stem_view_plan(0, B, Hc, Wc, prec)
        wplan = stem_view_plan(2, B, Hc, Wc, prec)
        assert (fplan, wplan) == plans[prec], (name, prec, fplan, wplan)
    what = "%s stem %s %s" % (prec, name, (B, H, W))
    g = _gen(7000 + STEM_CASES.index(case) * 4 + TRAIN_PREC.index(prec))
    yt = torch.float32 if prec in ("fp32", "tc_split") else torch.bfloat16
    dscale = 2.0 ** GSCALE if strict else 1.0
    out_scale = 2.0 ** -GSCALE if strict else 0.0
    to_dy = lambda dy: (nhwc(dy) * dscale).contiguous().to(yt)

    # ---- exact operands: every mode's output and gradient is fully determined ----
    x = (_ints((B, 3, H, W), g, -3, 3) / 4).float()
    w = (_ints((64, 3, 7, 7), g, -3, 3) / 4).float()
    dy = _ints((B, 64, Hc, Wc), g, -3, 3) / 4
    A, y, dw = run_stem(prec, B, H, W, x, w, to_dy(dy), out_scale, None, True)
    check_patch_matrix(what + " exact", prec, A, x, M)
    del A
    ref = nhwc(F.conv2d(x.double(), w.double(), None, 2, 3))
    check_exact(what + " exact fprop", y.double(), ref if yt == torch.float32 else ref.float().bfloat16().double())
    del ref, y
    check_exact(what + " exact wgrad", dw.double(), _stem_wgrad(x.double(), dy))
    del x, w, dy, dw

    # ---- random operands ----
    if strict:
        x, w, dy = _logu((B, 3, H, W), g), _logu((64, 3, 7, 7), g), _logu((B, 64, Hc, Wc), g).double()
    else:
        x = torch.randn((B, 3, H, W), generator=g, device="cuda")
        w = torch.randn((64, 3, 7, 7), generator=g, device="cuda") * (2.0 / 147) ** 0.5
        dy = torch.randn((B, 64, Hc, Wc), generator=g, device="cuda").double()
        if yt == torch.bfloat16:
            dy = dy.float().bfloat16().double()
    sums = np.full((2, 64), np.nan, dtype=np.float64) if tc else None
    A, y, dw = run_stem(prec, B, H, W, x, w, to_dy(dy), out_scale, sums, True)
    check_patch_matrix(what, prec, A, x, M)
    del A
    bf_ops = prec in ("bf16", "bf16_simt")
    xr = x.bfloat16().double() if bf_ops else x.double()
    wr = w.bfloat16().double() if bf_ops else w.double()
    del x, w
    ref = nhwc(F.conv2d(xr, wr, None, 2, 3))
    S = nhwc(F.conv2d(xr.abs(), wr.abs(), None, 2, 3))
    if prec == "bf16":
        gam = fplan[2] * fplan[3] // 16 * TRUNC
    elif strict:
        gam = fplan[2] * fplan[3] // 16 * TRUNC + 2 * SPLIT + SPLIT ** 2
    else:
        gam = gamma(STEM_K)
    u = U_BF16 if yt == torch.bfloat16 else 0.0
    got = y.double()
    del y
    check_elements(what + " fprop", got, ref, u * ref.abs() + (1 + u) * gam * S)
    del ref, S
    if tc:
        st = got.reshape(-1, 64)
        tpc = math.ceil(fplan[1] / NSM)
        sums = torch.from_numpy(sums).cuda()
        for j, (terms, n_extra) in enumerate(((st, 0), (st * st, 1))):
            bound = _sum_bound(terms.abs().sum(0), tpc + n_extra)
            check_elements(what + (" sum y" if j == 0 else " sum y^2"), sums[j], terms.sum(0), bound)
        del st
    del got
    ref = _stem_wgrad(xr, dy)
    S = _stem_wgrad(xr.abs(), dy.abs())
    if tc:
        gw = 4 * wplan[3] * TRUNC + (wplan[2] if wplan[2] > 1 else 0) * U_FP32
        if strict:
            gw += 2 * SPLIT + SPLIT ** 2 + 3 * U_FP32
        bound = (1 + U_FP32) * gw * S
        plan = "splits %d x %d tiles" % (wplan[2], wplan[3])
    else:
        splits, kchunk, _, _ = simt_wgrad_plan((B, Hc, Wc, STEM_K, 64, 1, 1))
        bound = gamma(kchunk + splits + 1) * S
        plan = "%d splits of %d" % (splits, kchunk)
    check_elements(what + " wgrad " + plan, dw.double(), ref, bound)
    print("simt-stem %-64s %.1f s" % (what, time.time() - t0))


# ------------------------------------------------------------------------------------------------------------------
# C. the tensor-core training step on the im2col stem
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def im2col_trunks(monkeypatch):
    """_lib.Trunk handles made with the im2col stem (mapnet_test_trunk_create(..., im2col_stem = 1))"""
    class Im2colTrunk(_lib.Trunk):
        def __init__(self, max_B, H, W, feat_dim, precision):
            self.h = ctypes.c_void_p()
            self.max_B, self.H, self.W, self.feat_dim, self.precision = max_B, H, W, feat_dim, precision
            self.trainable = None
            _lib.check(_lib.lib().mapnet_test_trunk_create(ctypes.byref(self.h), max_B, H, W, feat_dim,
                                                           _lib.PREC[precision], 1), "mapnet_test_trunk_create")
    monkeypatch.setattr(_lib, "Trunk", Im2colTrunk)
    return Im2colTrunk


def golden_step(name, precision, tol):
    from helpers import load_golden, make_product_model, make_product_criterion, product_step, compare_with_golden
    from oracle import weights
    g, cfg = load_golden(name)
    st = weights.make_state(int(g["seed"]))
    x, targ = weights.make_inputs(cfg, int(g["seed"]))
    kind = cfg["kind"]
    model, net = make_product_model(st, kind, precision, filter_nans=kind.startswith("online"))
    crit = make_product_criterion(kind)
    model.train()
    loss, pred, grads, sgrads = product_step(model, net, crit, x, targ, lr=cfg.get("lr", 1e-4), wd=cfg.get("wd", 5e-4),
                                             clip=cfg.get("clip", 0.0))
    torch.cuda.synchronize()
    errs = compare_with_golden(g, loss, pred, grads, sgrads, net, crit, tol)
    print("simt-stem %-64s loss %.2e pred %.2e grad %.2e grad_full %.2e" % (
        "%s im2col-stem step %s" % (precision, name), errs["loss"], errs["pred"], errs["grad_norm"], errs["grad_full"]))


STEP_CASES = [("tc_split", n) for n in STEP.TINY + ["posenet_b64_256"]] + \
             [("bf16", n) for n in ("posenet_b8_256", "posenet_b64_256")]


@pytest.mark.gpu
@pytest.mark.parametrize("prec,name", STEP_CASES, ids=["%s-%s" % c for c in STEP_CASES])
def test_training_step_on_the_im2col_stem(im2col_trunks, prec, name):
    golden_step(name, prec, STEP.TOL_TC_SPLIT if prec == "tc_split" else STEP.TOL_BF16)


def _stem_kernels(precision):
    """names of the stem kernels one training step of a fresh model launches"""
    from helpers import make_product_model, make_product_criterion
    from oracle import weights
    from torch.profiler import profile, ProfilerActivity
    cfg = dict(kind="posenet", N=4, H=64, W=64)
    x, targ = weights.make_inputs(cfg, 7)
    model, net = make_product_model(weights.make_state(7), "posenet", precision)
    crit = make_product_criterion("posenet")
    model.train()
    x, targ = x.cuda(), targ.cuda()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        crit(model(x), targ).backward()
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    return {k for k in ("k_stem_im2col", "k_stem_s2d") if any(k in n for n in names)}


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "tc_split"])
def test_patched_handle_runs_the_im2col_stem(im2col_trunks, prec, monkeypatch):
    assert _stem_kernels(prec) == {"k_stem_im2col"}
    monkeypatch.undo()
    assert _stem_kernels(prec) == {"k_stem_s2d"}
