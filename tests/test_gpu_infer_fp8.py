"""GPU tests of the fp8 inference engine (csrc/conv_tc.cu k_f8_conv, csrc/infer.cu, Predictor(precision='fp8')): one
e4m3 conv against fp64 on the dequantized operands, calibration (reproducible, powers of two, no saturation, the
emulation's scales), the whole network against the fp8-emulating oracle, and the Predictor's semantics."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fp8_emulation import fp8_engine_emulation, pow2_scale, quantize_e4m3
from test_gpu_infer import _device_flat, _oracle_eval, _rel, _state_with_batch_stats

pytestmark = pytest.mark.gpu


def _lib():
    from geomapnet_b200 import _lib
    return _lib


def _codes(v):
    """e4m3 values (already representable) -> their bytes"""
    return v.to(torch.float8_e4m3fn).view(torch.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# 1. one conv
# ---------------------------------------------------------------------------------------------------------------------
# (Ci, Co, k, stride, B, Hi, Wi, residual, relu, out_f8): Cin = 64 (64-byte k-blocks) at N tiles of 64 (Co 64) and 128
# (Co 128 over 128 M tiles), 3x3/s1 at 128 and 256 channels, 3x3/s2 on a ragged width (88 -> 44), the 1x1/s2 downsample
# with bf16 out (Cin 64 and 128), conv2 with e4m3 and bf16 residuals, 512 -> 512 (K = 4608, the longest accumulation)
CASES = [
    (64, 64, 3, 1, 3, 16, 16, "f8", True, True),
    (64, 128, 3, 1, 4, 64, 64, None, True, True),
    (64, 128, 3, 2, 3, 22, 88, None, True, True),
    (128, 128, 3, 1, 3, 12, 12, None, True, True),
    (256, 256, 3, 1, 3, 8, 8, "bf16", True, True),
    (128, 256, 3, 2, 2, 22, 88, None, True, True),
    (64, 128, 1, 2, 3, 16, 16, None, False, False),
    (256, 512, 1, 2, 3, 16, 16, None, False, False),
    (128, 128, 3, 1, 3, 12, 12, "f8", True, True),
    (512, 512, 3, 1, 4, 8, 8, "f8", True, True),
]

# The e4m3 products are exact, but the tensor cores' accumulation of them is not fp32-exact: measured on an H100 it adds
# up to tau = 6.3e-4 of max|ref| (512 -> 512, K = 4608; 6e-5 .. 3e-4 on the shorter convs) beyond the one e4m3 (or bf16)
# rounding of the output, about 2^-11 -- fewer bits than an fp32 accumulator keeps.  TAU is 2x the largest measurement.
# An accumulation error that crosses a rounding midpoint moves an output by one step: measured, 0.4 .. 1.3 % of e4m3
# outputs and 2.5 .. 6.2 % of bf16 outputs differ from the exactly rounded fp64 result; the bounds are 2x that.  A layout
# or scale error would move most outputs.
TAU = 1.3e-3
MISMATCH_FRAC = {True: 0.027, False: 0.125}     # by out_f8


@pytest.mark.parametrize("case", CASES, ids=lambda c: "ci%d_co%d_k%d_s%d_%dx%d%s%s" % (
    c[0], c[1], c[2], c[3], c[5], c[6], "_res" + c[7] if c[7] else "", "_f8out" if c[9] else "_bf16out"))
def test_fp8_conv_matches_fp64(case):
    Ci, Co, k, s, B, Hi, Wi, res, relu, out_f8 = case
    L = _lib()
    g = torch.Generator().manual_seed(Ci * 7 + Co + k + Wi)
    pad = (k - 1) // 2
    Ho, Wo = (Hi + 2 * pad - k) // s + 1, (Wi + 2 * pad - k) // s + 1
    # e4m3 operands (the engine's input is already quantized); weights scaled per output channel as the pack does
    x = quantize_e4m3(torch.randn(B, Hi, Wi, Ci, generator=g) * 2.0)
    w = quantize_e4m3(torch.randn(Co, k, k, Ci, generator=g) * 64.0)
    S = ((1.0 + 0.3 * torch.randn(Co, generator=g)) * (2.0 / (Ci * k * k)) ** 0.5 / 64.0).float()
    shift = (0.2 * torch.randn(Co, generator=g)).float()
    ref = F.conv2d(x.permute(0, 3, 1, 2).double().cuda(), w.permute(0, 3, 1, 2).double().cuda(), None, s, pad)
    ref = ref.permute(0, 2, 3, 1) * S.double().cuda() + shift.double().cuda()
    s_res = torch.tensor([0.25], device="cuda")
    rin = None
    if res == "f8":
        r8 = quantize_e4m3(torch.randn(B, Ho, Wo, Co, generator=g) * 8.0)
        ref = ref + r8.double().cuda() * 0.25
        rin = _codes(r8).cuda()
    elif res == "bf16":
        rb = torch.randn(B, Ho, Wo, Co, generator=g).to(torch.bfloat16)
        ref = ref + rb.double().cuda()
        rin = rb.cuda()
    if relu:
        ref = ref.clamp_min(0)
    flags = (1 if relu else 0) | (2 if res == "f8" else 0) | (4 if out_f8 else 0)
    s_out = pow2_scale(float(ref.abs().max()))
    out_inv = torch.tensor([1.0 / s_out], device="cuda")
    xb, wb, Sd, shd = _codes(x).cuda(), _codes(w).cuda(), S.cuda(), shift.cuda()
    args = lambda fl, out, amax: (B, Hi, Wi, Ci, Co, k, s, xb.data_ptr(), wb.data_ptr(), Sd.data_ptr(), shd.data_ptr(),
                                  rin.data_ptr() if rin is not None else None, s_res.data_ptr(), out_inv.data_ptr(), fl,
                                  out, amax, L.stream_ptr())
    out = torch.zeros(B, Ho, Wo, Co, dtype=torch.uint8 if out_f8 else torch.bfloat16, device="cuda")
    L.check(L.lib().mapnet_test_conv_fp8(*args(flags, out.data_ptr(), None)), "mapnet_test_conv_fp8")
    mx = float(ref.abs().max())
    if out_f8:
        got = out.view(torch.float8_e4m3fn).double() * s_out
        exact = quantize_e4m3((ref / s_out).float()).double() * s_out
        bound = ref.abs() * 2.0 ** -4 + 2.0 ** -10 * s_out + TAU * mx
        frac = float((got != exact).double().mean())
    else:
        got = out.double()
        exact = ref.float().to(torch.bfloat16).double()
        bound = ref.abs() * 2.0 ** -8 + TAU * mx
        frac = float((got != exact).double().mean())
    err = (got - ref).abs()
    # tau: what the fp32 accumulation adds beyond the output rounding, relative to max|ref|
    tau = float((err - (bound - TAU * mx)).clamp_min(0).max() / mx)
    print(case, "max err / bound %.3f, tau %.2e, outputs != exactly rounded %.4f" % (float((err / bound).max()), tau, frac))
    assert bool((err <= bound).all()), float((err / bound).max())
    assert frac <= MISMATCH_FRAC[out_f8], frac
    if out_f8:
        # the calibration pass of the same launch: max |f| of the output, nothing stored
        amax = torch.zeros(1, dtype=torch.int32, device="cuda")
        before = out.clone()
        L.check(L.lib().mapnet_test_conv_fp8(*args(flags | 8, out.data_ptr(), amax.data_ptr())), "mapnet_test_conv_fp8")
        a = float(amax.view(torch.float32))
        assert abs(a - mx) <= 2 * TAU * mx + 1e-6 * mx, (a, mx)
        assert torch.equal(out, before)


# ---------------------------------------------------------------------------------------------------------------------
# 2. calibration, 3. whole network
# ---------------------------------------------------------------------------------------------------------------------
def _frames(kind, n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*((n,) if kind == "posenet" else n), 3, H, W, generator=g)


def _check_scales_match_emulation(scales, emu_scales, emu_amax):
    """engine scales against the emulation's progressive rule.  The tensor cores' accumulation (test_fp8_conv_matches_fp64:
    up to 6.3e-4 of max|ref| per conv) flips an occasional e4m3 rounding by one step, and such flips compound through the
    blocks, so the deep tensors' amax drifts by a few percent and a scale may land one power of two away.  Measured on an
    H100 (B = 8, 256x256): 30 of 33 scales equal, three layer3 / layer4 tensors (19, 21, 28) a factor 2 apart.  Asserted:
    every scale within a factor 2, at most 6 of 33 different.  Returns the indices that agree."""
    assert len(scales) == len(emu_scales) == 33
    diff = [i for i, (a, b) in enumerate(zip(scales, emu_scales)) if a != b]
    print("scales different from the emulation's:", [(i, scales[i], emu_scales[i], emu_amax[i]) for i in diff])
    assert all(max(a, b) <= 2 * min(a, b) for a, b in zip(scales, emu_scales))
    assert len(diff) <= 6, diff
    return [i for i in range(33) if i not in diff]


def test_calibration_is_reproducible_powers_of_two_without_saturation():
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    st = weights.make_state(5)
    x = _frames("posenet", 8, 256, 256, 3)
    st_b = _state_with_batch_stats(st, x)
    model, net = make_product_model(st_b, "posenet", "bf16")
    pr = Predictor(model, max_batch=8, precision="fp8", calibration=x.cuda())
    s1, p1 = pr.act_scales, pr(x.cuda())
    pr2 = Predictor(model, max_batch=8, precision="fp8", calibration=x.cuda())
    s2, p2 = pr2.act_scales, pr2(x.cuda())
    assert s1 == s2 and torch.equal(p1, p2)                     # bitwise reproducible
    for s in s1:
        m, _ = np.frexp(s)
        assert m == 0.5, s                                      # powers of two
    with torch.no_grad():
        _, emu_scales, emu_amax = fp8_engine_emulation({k: v.cuda() for k, v in st_b.items()}, x.cuda())
    same = _check_scales_match_emulation(s1, emu_scales, emu_amax)
    # no calibrated tensor saturates on the calibration frames: amax / s <= 448, with the emulation's amax where it
    # follows the engine's values (the scales agree; elsewhere the two have drifted apart, see above)
    worst = max(emu_amax[i] / s1[i] for i in same)
    print("fp8 scales:", s1, "largest amax / scale on the calibration frames %.1f" % worst)
    assert worst <= 448.0 * (1 + 1e-3), worst
    pr.close(); pr2.close()


# Measured on an H100 (max |difference| / max |pose|): fp8 Predictor vs the fp8 emulation with the engine's scales 0.071
# (256x341) .. 0.311 (MapNet 128x128); vs the fp32 oracle 0.126 .. 0.391, vs the bf16 Predictor 0.133 .. 0.391.  With
# 3 mantissa bits one flipped rounding moves a value by 6 .. 12 %, and these random-weight networks amplify it over 33
# quantized tensors, so the emulation pins the rounding points (scales, operands, epilogue order) and the per-conv test
# pins the arithmetic; the bounds are 2x the measurements.
EMU_BOUND = 0.65
DRIFT_BOUND = 0.8


@pytest.mark.parametrize("shape", [("posenet", 8, 256, 256), ("posenet", 64, 256, 256), ("posenet", 2, 256, 341),
                                   ("mapnet", (3, 3), 128, 128)],
                         ids=lambda s: "%s_%s_%dx%d" % (s[0], s[1], s[2], s[3]))
def test_fp8_predictor_matches_fp8_emulation(shape):
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    kind, n, H, W = shape
    st = weights.make_state(11)
    x = _frames(kind, n, H, W, H * W + 1)
    frames = x.reshape(-1, 3, H, W)
    st_b = _state_with_batch_stats(st, frames[:16])
    model, net = make_product_model(st_b, kind, "bf16")
    mb = max(8, frames.shape[0])
    pr = Predictor(model, max_batch=mb, precision="fp8", calibration=x.cuda())
    got = pr(x.cuda()).reshape(-1, 6)
    scales = pr.act_scales
    prb = Predictor(model, max_batch=mb)
    bf = prb(x.cuda()).reshape(-1, 6)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            emu, emu_scales, emu_amax = fp8_engine_emulation({k: v.cuda() for k, v in st_b.items()}, frames.cuda(), scales)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    e_emu = _rel(got, emu)
    e_ref = _rel(got.cpu(), _oracle_eval(st_b, frames))
    e_bf = _rel(got, bf)
    print(shape, "fp8 vs fp8 emulation %.2e, vs fp32 oracle %.2e, vs bf16 Predictor %.2e" % (e_emu, e_ref, e_bf))
    # The emulation uses the engine's own scales and rounding points; what remains is the fp32 accumulation order,
    # which flips an occasional e4m3 rounding of one step and propagates.
    assert e_emu <= EMU_BOUND, e_emu
    # the drift fp8 adds to the pose is a property of e4m3 (3 mantissa bits), stated loosely
    assert e_ref <= DRIFT_BOUND and e_bf <= DRIFT_BOUND, (e_ref, e_bf)
    pr.close(); prb.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. semantics
# ---------------------------------------------------------------------------------------------------------------------
def test_fp8_graph_replay_chunking_refresh_and_launches():
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    from geomapnet_b200.common.optimizer import Optimizer
    L = _lib()
    lib = L.lib()
    st = weights.make_state(13)
    model, net = make_product_model(st, "posenet", "tc_split")
    mb, H, W = 8, 64, 96
    x = torch.randn(2 * mb + 3, 3, H, W, generator=torch.Generator().manual_seed(2)).cuda()
    pr = Predictor(model, max_batch=mb, precision="fp8", calibration=x[:mb])
    eng = pr._engine(H, W)
    for B in (1, 5, mb):
        graphed, graphed2 = pr(x[:B]), pr(x[:B])
        eager = torch.empty(B, 6, device="cuda")
        eng.forward(x[:B].contiguous(), eager, 0.0, 0)
        assert torch.equal(graphed, eager) and torch.equal(graphed2, eager), B
    chunked = pr(x)
    singles = torch.cat([pr(x[i:i + mb]) for i in range(0, x.shape[0], mb)])
    assert torch.equal(chunked, singles)
    # launches per call: the bf16 Predictor's (36 convs + stem operand + pool + head); the calibration adds none
    for B in (1, 4):
        c0 = lib.mapnet_launch_count()
        eng.forward(x[:B].contiguous(), torch.empty(B, 6, device="cuda"), 0.0, 0)
        assert lib.mapnet_launch_count() - c0 == 36 + 2 + 6, (B, lib.mapnet_launch_count() - c0)
    # refresh() after training steps equals a freshly built fp8 Predictor, bitwise (scales and poses)
    before = pr(x)
    opt = Optimizer(params=model.parameters(), method="adam", base_lr=1e-2, weight_decay=0.0)
    model.train()
    for _ in range(2):
        out = model(x[:4].clone().requires_grad_(True))
        opt.learner.zero_grad()
        out.square().sum().backward()
        opt.learner.step()
    with torch.no_grad():
        model(x[:4])
    assert torch.equal(pr(x), before)                  # frozen until refresh
    pr.refresh()
    fresh = Predictor(model, max_batch=mb, precision="fp8", calibration=x[:mb])
    after = pr(x)
    assert not torch.equal(after, before)
    assert pr.act_scales == fresh.act_scales and torch.equal(after, fresh(x))
    pr.close(); fresh.close()


def test_fp8_errors_before_any_launch():
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    L = _lib()
    lib = L.lib()
    st = weights.make_state(4)
    model, net = make_product_model(st, "posenet", "bf16")
    _device_flat(net)
    H, W = 64, 64
    x = torch.randn(4, 3, H, W, device="cuda")
    n0 = lib.mapnet_launch_count()
    with pytest.raises(ValueError, match="calibration"):
        Predictor(model, max_batch=4, precision="fp8")
    with pytest.raises(ValueError, match="max_batch"):
        Predictor(model, max_batch=4, precision="fp8", calibration=torch.randn(5, 3, H, W, device="cuda"))
    with pytest.raises(ValueError, match="max_batch"):
        Predictor(model, max_batch=4, precision="fp8", calibration=torch.randn(2, 3, 3, H, W, device="cuda"))
    assert lib.mapnet_launch_count() == n0
    pr = Predictor(model, max_batch=4, precision="fp8", calibration=x)
    n1 = lib.mapnet_launch_count()
    with pytest.raises(ValueError, match="calibrated at 64x64"):
        pr(torch.randn(2, 3, 64, 96, device="cuda"))
    assert lib.mapnet_launch_count() == n1
    pr.close()
    # the engine: a forward after a load but before a calibration, a calibration on a bf16 handle
    eng = L.Infer(4, H, W, net.feat_dim, "fp8")
    eng.load(net._flat, net._bufs)
    n2 = lib.mapnet_launch_count()
    with pytest.raises(RuntimeError, match="mapnet_infer_calibrate"):
        eng.forward(x, torch.empty(4, 6, device="cuda"), 0.0, 0)
    with pytest.raises(RuntimeError, match="outside"):
        eng.calibrate(torch.randn(5, 3, H, W, device="cuda"))
    assert lib.mapnet_launch_count() == n2
    bf = L.Infer(4, H, W, net.feat_dim, "bf16")
    bf.load(net._flat, net._bufs)
    n3 = lib.mapnet_launch_count()
    with pytest.raises(RuntimeError, match="only the fp8 engine"):
        bf.calibrate(x)
    assert lib.mapnet_launch_count() == n3
    torch.cuda.synchronize()
    eng.close(); bf.close()
