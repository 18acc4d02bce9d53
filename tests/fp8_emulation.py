"""CPU / torch emulation of the fp8 inference engine's arithmetic (csrc/infer.cu, conv_tc.cu k_f8_conv).

The engine's roundings are: the stem on the bf16 engine (bf16 operands, one bf16 rounding after its epilogue), then for
every other conv e4m3 operands, fp32 accumulation, the fp32 affine map f = acc * S + shift with S = bn_scale * s_in *
s_w (powers of two: exact), the residual (e4m3 r * s_res, exact, or the bf16 downsample output), the ReLU and one
e4m3 rounding of f / s_out (round to nearest even, saturating at +-448).  Every scale is the power of two
2^ceil(log2(amax / 448)) of its tensor (weights: of each output channel's row), so scaling is exact and the emulation
below reproduces the engine's rounding points; only the order of the fp32 accumulation differs."""
import numpy as np
import torch
import torch.nn.functional as F

E4M3_MAX = 448.0


def quantize_e4m3(t):
    """e4m3 round to nearest even with saturation, as cvt.rn.satfinite.e4m3x2.f32: torch's cast rounds to nearest even
    but does not saturate (500.0 -> NaN), so the values are clamped to +-448 first (NaN stays NaN)."""
    return t.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).to(t.dtype)


def e4m3_rne_satfinite_numpy(x):
    """from-scratch reference of the same rounding on float32 values: 3 mantissa bits, exponent bias 7, subnormal quantum
    2^-9, round half to even, |result| <= 448, NaN -> NaN"""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    a = np.abs(x)
    _, k = np.frexp(np.where(a > 0, a, 1.0))            # a = m * 2^k, m in [0.5, 1): binade exponent k - 1
    e = np.maximum(k - 1, -6)                           # below 2^-6 the quantum stays 2^-9 (subnormals)
    quantum = np.ldexp(1.0, e - 3)
    r = np.rint(a / quantum) * quantum                  # np.rint rounds half to even; a / quantum is exact
    r = np.minimum(r, E4M3_MAX)
    out = np.copysign(r, x)
    return np.where(np.isnan(x), np.nan, out).astype(np.float32)


def pow2_scale(amax):
    """the smallest power of two s with 448 * s >= amax (1 for amax 0), from the exponent as f8_pow2_scale does"""
    a = np.float32(amax)
    if not a > 0:
        return 1.0
    if not np.isfinite(a):
        return 2.0 ** 120
    m, k = np.frexp(a)
    e = k - 9 if m <= np.float32(0.875) else k - 8
    return float(2.0 ** max(int(e), -126))


def weight_scales(w):
    """per output channel power-of-two scales of a conv weight [Co, ...] and the e4m3 values w / s"""
    amax = w.abs().reshape(w.shape[0], -1).amax(1)
    s = torch.tensor([pow2_scale(float(v)) for v in amax], dtype=torch.float32, device=w.device)
    return s, quantize_e4m3(w / s.view(-1, *([1] * (w.dim() - 1))))


def _eval_affine(st, p):
    """the eval-mode BatchNorm scale / shift (k_bn_eval_scale's formula, fp32)"""
    inv = 1.0 / torch.sqrt(st[p + ".running_var"] + 1e-5)
    sc = st[p + ".weight"] * inv
    return sc, st[p + ".bias"] - st[p + ".running_mean"] * sc


def fp8_engine_emulation(st, x, act_scales=None):
    """pred [N,6] of the fp8 engine's arithmetic on frames x [N,3,H,W] (st: fp32 state dict, tensors on one device).
    act_scales None: take the 33 activation scales progressively from x (the engine's calibration rule); otherwise use
    the given ones.  Returns (pred, scales, amaxes)."""
    from oracle import mapnet_oracle as O
    rb = lambda t: t.to(torch.bfloat16).float()
    fe = "feature_extractor."
    calib = act_scales is None
    scales = [] if calib else [float(s) for s in act_scales]
    amaxes = []
    idx = [0]

    def take(f):
        amaxes.append(float(f.abs().max()))
        if calib:
            scales.append(pow2_scale(amaxes[-1]))
        s = scales[idx[0]]
        idx[0] += 1
        return s

    def conv8(z, zs, name, bn, stride, pad):
        """acc * S + shift of one e4m3 conv (acc in fp64 from exact products, rounded to fp32 as the accumulator holds it)"""
        sw, w8 = weight_scales(st[name])
        sc, sh = _eval_affine(st, bn)
        S = sc * np.float32(zs) * sw
        acc = F.conv2d(z.double(), w8.double(), None, stride, pad).float()
        return acc * S[None, :, None, None] + sh[None, :, None, None]

    sc, sh = _eval_affine(st, fe + "bn1")
    y0 = rb(F.relu(F.conv2d(rb(x), rb(st[fe + "conv1.weight"]), None, 2, 3) * sc[None, :, None, None] + sh[None, :, None, None]))
    zs = take(y0)
    z = quantize_e4m3(F.max_pool2d(y0, 3, 2, 1) / np.float32(zs))
    inpl = 64
    for li, (planes, nblk, stride) in enumerate(O.STAGES, start=1):
        for b in range(nblk):
            p = "%slayer%d.%d." % (fe, li, b)
            s = stride if b == 0 else 1
            f = F.relu(conv8(z, zs, p + "conv1.weight", p + "bn1", s, 1))
            hs = take(f)
            h = quantize_e4m3(f / np.float32(hs))
            if s != 1 or inpl != planes:
                idt = rb(conv8(z, zs, p + "downsample.0.weight", p + "downsample.1", s, 0))
            else:
                idt = z * np.float32(zs)
            f = F.relu(conv8(h, hs, p + "conv2.weight", p + "bn2", 1, 1) + idt)
            zs = take(f)
            z = quantize_e4m3(f / np.float32(zs))
            inpl = planes
    feat = z.mean(dim=(2, 3)) * np.float32(zs)
    f = F.relu(F.linear(feat, st[fe + "fc.weight"], st[fe + "fc.bias"]))
    pred = torch.cat((F.linear(f, st["fc_xyz.weight"], st["fc_xyz.bias"]), F.linear(f, st["fc_wpqr.weight"], st["fc_wpqr.bias"])), 1)
    return pred, scales, amaxes
