"""GPU tests of the eval-mode inference engine (csrc/infer.cu) and its Predictor (geomapnet_b200/inference.py): the
fused affine epilogue against torch, whole-network parity against the oracle's eval forward, agreement with the live
eval path, snapshot semantics, graph replay, dropout and launch counts."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

EPS = 1e-5


def _lib():
    from geomapnet_b200 import _lib
    return _lib


def _round_f16x2(t):
    c = t.clamp(-65504.0, 65504.0)
    hi = c.to(torch.float16).to(t.dtype)
    return hi + (c - hi).to(torch.float16).to(t.dtype)


def _planes_to_f32(raw, shape):
    """hi/lo plane storage (common.cuh: hsplit; per 8 channels 8 fp16 hi then 8 fp16 lo) -> fp32 [.., C]"""
    h = raw.view(torch.float16).reshape(*shape[:-1], shape[-1] // 8, 2, 8).float()
    return (h[..., 0, :] + h[..., 1, :]).reshape(shape)


# ---------------------------------------------------------------------------------------------------------------------
# 1. one conv with the inference epilogue against torch
# ---------------------------------------------------------------------------------------------------------------------
# (Ci, Co, k, stride, Hi, Wi, residual, relu): the stem, 3x3/s1 at both tile widths, 3x3/s2 on a ragged width
# (88 -> 44), the 1x1/s2 downsample (no ReLU), conv2 with a residual
CASES = [
    (3, 64, 7, 2, 40, 88, False, True),
    (64, 64, 3, 1, 16, 16, True, True),
    (128, 128, 3, 1, 12, 12, False, True),
    (256, 256, 3, 1, 8, 8, True, True),
    (64, 128, 3, 2, 22, 88, False, True),
    (64, 128, 1, 2, 16, 16, False, False),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "k%d_s%d_%dx%d_co%d%s%s" % (c[2], c[3], c[4], c[5], c[1],
                                                                                  "_res" if c[6] else "", "_relu" if c[7] else ""))
@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
def test_affine_epilogue_matches_torch(precision, case):
    Ci, Co, k, s, Hi, Wi, res, relu = case
    L = _lib().lib()
    g = torch.Generator().manual_seed(Ci * 7 + Co + k)
    B = 3
    pad = (k - 1) // 2
    Ho, Wo = (Hi + 2 * pad - k) // s + 1, (Wi + 2 * pad - k) // s + 1
    x = torch.randn(B, Ci, Hi, Wi, generator=g)
    w = torch.randn(Co, Ci, k, k, generator=g) * (2.0 / (Ci * k * k)) ** 0.5
    scale = (1.0 + 0.3 * torch.randn(Co, generator=g)).cuda()
    shift = (0.2 * torch.randn(Co, generator=g)).cuda()
    r = torch.randn(B, Ho, Wo, Co, generator=g) if res else None
    sp = precision == "tc_split"
    rnd = _round_f16x2 if sp else (lambda t: t.to(torch.bfloat16).float())
    # operands as the engine stores them; products exact, accumulation in fp64 here
    ref = F.conv2d(rnd(x).double().cuda(), rnd(w).double().cuda(), None, s, pad).permute(0, 2, 3, 1)
    ref = ref * scale.double() + shift.double()
    flags = 1 if relu else 0
    res_split = sp and res and Co == 64          # identity branch (block input planes); Co 256: a downsample output, fp32
    out_split = sp and k != 7 and relu           # conv1 / conv2 write the next conv's operand planes
    flags |= (2 if res_split else 0) | (4 if out_split else 0)
    if res:
        rr = rnd(r) if (res_split or not sp) else r
        ref = ref + rr.double().cuda()
    if relu:
        ref = ref.clamp_min(0)
    if k == 7:
        xin, win = x.cuda(), w.cuda()                                              # fp32 NCHW image, fp32 OIHW
    elif sp:
        xin, win = x.permute(0, 2, 3, 1).contiguous().cuda(), w.permute(0, 2, 3, 1).contiguous().cuda()
    else:
        xin = x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16).cuda()
        win = w.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16).cuda()
    rin = None
    if res:
        rin = r.cuda() if sp else r.to(torch.bfloat16).cuda()
    if sp:
        out = torch.zeros(B, Ho, Wo, Co, dtype=torch.float32, device="cuda")
    else:
        out = torch.zeros(B, Ho, Wo, Co, dtype=torch.bfloat16, device="cuda")
    _lib().check(L.mapnet_test_conv_affine(_lib().PREC[precision], B, Hi, Wi, Ci, Co, k, s, xin.data_ptr(), win.data_ptr(),
                                           scale.data_ptr(), shift.data_ptr(), rin.data_ptr() if rin is not None else None,
                                           flags, out.data_ptr(), _lib().stream_ptr()), "mapnet_test_conv_affine")
    got = _planes_to_f32(out, out.shape) if out_split else out.float()
    err = (got.double() - ref).abs()
    scale_ref = ref.abs().max()
    if sp:
        # strict mode: exact hi/lo products, the tensor cores' fp32 accumulation (it truncates, so the error grows with
        # K) and one 22-bit rounding when the output is stored as planes: the strict engine's per-conv bound of
        # test_gpu_kernels.test_conv_engines (1e-4 of the output's magnitude; measured up to 1.5e-5 here)
        e = float(err.max() / scale_ref)
        print(precision, case, "max err / max|ref| %.2e" % e)
        assert e <= 1e-4, e
    else:
        # one bf16 rounding of the fp32 result (2^-8 relative; fp32 accumulation adds ~1e-6 of the magnitude)
        bound = ref.abs() * 2.0 ** -8 + 1e-5 * scale_ref
        print(precision, case, "max err / bound %.3f" % float((err / bound).max()))
        assert bool((err <= bound).all()), float((err / bound).max())


# ---------------------------------------------------------------------------------------------------------------------
# helpers: models, realistic running statistics
# ---------------------------------------------------------------------------------------------------------------------
def _state_with_batch_stats(st, x):
    """running statistics = the batch statistics of a training-mode forward on x (what a trained net's are like: every
    BatchNorm normalises its input), recovered from one momentum update of the oracle's buffers"""
    from oracle import mapnet_oracle as O
    s0 = {k: v.clone() for k, v in st.items()}
    for k in s0:
        if k.endswith("running_mean"):
            s0[k].zero_()
        elif k.endswith("running_var"):
            s0[k].fill_(1.0)
    bufs = {}
    with torch.no_grad():
        O.trunk_forward({k: v.cuda() for k, v in s0.items()}, x.cuda(), training=True, bufs_out=bufs)
    out = dict(s0)
    for k, v in bufs.items():
        if k.endswith("running_mean"):
            out[k] = (v / O.BN_MOMENTUM).cpu()
        else:
            out[k] = ((v - (1 - O.BN_MOMENTUM)) / O.BN_MOMENTUM).cpu()
    return out


def _oracle_eval(st, x, kind="posenet"):
    """the oracle's eval forward in fp64 (on the GPU for speed: fp64 keeps cuDNN's algorithm choice out of the bound)"""
    from oracle import mapnet_oracle as O
    with torch.no_grad():
        stc = {k: (v.double() if v.is_floating_point() else v).cuda() for k, v in st.items()}
        f = O.posenet_forward if kind == "posenet" else O.mapnet_forward
        return f(stc, x.double().cuda(), training=False).cpu()


def _device_flat(net):
    """bind the model's parameters / buffers to its flat device buffers (what its first forward does)"""
    dev = torch.device("cuda", torch.cuda.current_device())
    if not net._is_flat(dev):
        net._reflatten(dev)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


# ---------------------------------------------------------------------------------------------------------------------
# 2. whole network, strict mode, against the oracle's eval forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [("posenet", 3, 64, 96), ("posenet", 2, 72, 88), ("posenet", 2, 256, 341),
                                   ("posenet", 64, 256, 256), ("mapnet", (3, 3), 64, 64)],
                         ids=lambda s: "%s_%s_%dx%d" % (s[0], s[1], s[2], s[3]))
def test_tc_split_predictor_matches_oracle_eval(shape):
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    kind, n, H, W = shape
    st = weights.make_state(11)
    g = torch.Generator().manual_seed(H * W)
    x = torch.randn(*((n,) if kind == "posenet" else n), 3, H, W, generator=g)
    frames = x.reshape(-1, 3, H, W)
    # realistic normalisation: the running statistics of a training-mode batch -> the 1e-4 bound
    st_b = _state_with_batch_stats(st, frames[:16])
    model, net = make_product_model(st_b, kind, "tc_split")
    pr = Predictor(model, max_batch=64)
    e = _rel(pr(x.cuda()).cpu(), _oracle_eval(st_b, x, kind))
    # untouched (0, 1) statistics: activations grow layer by layer -> the existing eval test's 3e-4
    st0 = {k: (torch.zeros_like(v) if k.endswith("running_mean") else torch.ones_like(v) if k.endswith("running_var")
               else v) for k, v in st.items()}
    model0, _ = make_product_model(st0, kind, "tc_split")
    pr0 = Predictor(model0, max_batch=64)
    e0 = _rel(pr0(x.cuda()).cpu(), _oracle_eval(st0, x, kind))
    print(shape, "batch-stat rel err %.2e, (0,1)-stat rel err %.2e" % (e, e0))
    pr.close(); pr0.close()
    # The engine is bitwise equal to the live eval path (test_predictor_matches_live_eval_path), so this is the strict
    # mode's eval-mode error.  With realistic statistics it exceeds the training step's 1e-4: the eval-mode BatchNorm
    # computes y*s + (beta - mean*s) in fp32 (k_bn_eval_scale, as mapnet_forward(training=0) does), which cancels where
    # |mean| >> std, and eval mode does not re-normalise the error away layer by layer.  Measured on an H100: 2.0e-4 ..
    # 5.1e-4 against the fp32 oracle; the bound is 2x that.
    assert e <= 1e-3, e
    assert e0 <= 3e-4, e0


# ---------------------------------------------------------------------------------------------------------------------
# 3. against the live eval path
# ---------------------------------------------------------------------------------------------------------------------
def _bf16_engine_emulation(st, x):
    """the bf16 engine's rounding points: conv operands bf16 (weights rounded, activations stored bf16), fp32
    accumulation, scale / shift as k_bn_eval_scale computes them, ONE rounding after affine (+ residual) (+ ReLU)"""
    from oracle import mapnet_oracle as O
    rb = lambda t: t.to(torch.bfloat16).float()
    fe = "feature_extractor."

    def aff(y, p):
        inv = 1.0 / torch.sqrt(st[p + ".running_var"] + 1e-5)
        sc = st[p + ".weight"] * inv
        sh = st[p + ".bias"] - st[p + ".running_mean"] * sc
        return y * sc[None, :, None, None] + sh[None, :, None, None]

    conv = lambda z, name, s, p: F.conv2d(z, rb(st[name]), None, s, p)
    z = rb(F.relu(aff(conv(rb(x), fe + "conv1.weight", 2, 3), fe + "bn1")))
    z = F.max_pool2d(z, 3, 2, 1)
    inpl = 64
    for li, (planes, nblk, stride) in enumerate(O.STAGES, start=1):
        for b in range(nblk):
            p = "%slayer%d.%d." % (fe, li, b)
            s = stride if b == 0 else 1
            h = rb(F.relu(aff(conv(z, p + "conv1.weight", s, 1), p + "bn1")))
            idt = z
            if s != 1 or inpl != planes:
                idt = rb(aff(conv(z, p + "downsample.0.weight", s, 0), p + "downsample.1"))
            z = rb(F.relu(aff(conv(h, p + "conv2.weight", 1, 1), p + "bn2") + idt))
            inpl = planes
    f = F.relu(F.linear(z.mean(dim=(2, 3)), st[fe + "fc.weight"], st[fe + "fc.bias"]))
    return torch.cat((F.linear(f, st["fc_xyz.weight"], st["fc_xyz.bias"]), F.linear(f, st["fc_wpqr.weight"], st["fc_wpqr.bias"])), 1)


def test_predictor_matches_live_eval_path():
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    st = weights.make_state(5)
    x = torch.randn(8, 3, 256, 256, generator=torch.Generator().manual_seed(3))
    st_b = _state_with_batch_stats(st, x)
    # tc_split: the scale and shift are the same k_bn_eval_scale results on both sides; only where the affine map is
    # applied moves (the conv epilogue on the fp32 accumulator vs k_bn_apply on the stored fp32 conv output), so the two
    # differ at most by FMA contraction of the fp32 arithmetic.  Both apply ONE fused multiply-add to the same fp32
    # accumulator value (the live path stores it exactly in fp32 first) and the fprop plans are the same, so measured:
    # 0 (bitwise equal); the bound leaves room for a contraction the compiler may choose differently.
    model, net = make_product_model(st_b, "posenet", "tc_split")
    model.eval()
    with torch.no_grad():
        live = model(x.cuda())
    pr = Predictor(model, max_batch=8)
    e = _rel(pr(x.cuda()), live)
    print("tc_split Predictor vs model.eval(): %.2e" % e)
    assert e <= 2e-5, e
    pr.close()
    # bf16: the engine rounds once per conv after the epilogue, the live path rounds the conv output before BatchNorm:
    # compared with an emulation of the engine's own rounding points, at the bf16 forward bound of
    # test_step_bf16_matches_bf16_emulating_oracle
    model, net = make_product_model(st_b, "posenet", "bf16")
    pr = Predictor(model, max_batch=8)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            emu = _bf16_engine_emulation({k: v.cuda() for k, v in st_b.items()}, x.cuda())
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    e_emu = _rel(pr(x.cuda()), emu)
    e_ref = _rel(pr(x.cuda()).cpu(), _oracle_eval(st_b, x))
    print("bf16 Predictor vs bf16 engine emulation: %.2e, vs fp32 oracle: %.2e" % (e_emu, e_ref))
    assert e_emu <= 7e-2, e_emu
    pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. snapshot semantics, 5. graph replay
# ---------------------------------------------------------------------------------------------------------------------
def test_snapshot_is_frozen_until_refresh():
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    from geomapnet_b200.common.optimizer import Optimizer
    st = weights.make_state(9)
    model, net = make_product_model(st, "posenet", "bf16")
    x = torch.randn(4, 3, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    pr = Predictor(model, max_batch=4)
    before = pr(x)
    opt = Optimizer(params=model.parameters(), method="adam", base_lr=1e-2, weight_decay=0.0)
    model.train()
    for _ in range(3):
        out = model(x.clone().requires_grad_(True))
        opt.learner.zero_grad()
        out.square().sum().backward()
        opt.learner.step()
    with torch.no_grad():
        model(x)                      # a training-mode forward moves the running statistics too
    assert torch.equal(pr(x), before)
    pr.refresh()
    fresh = Predictor(model, max_batch=4)
    after = pr(x)
    assert not torch.equal(after, before)
    assert torch.equal(after, fresh(x))
    pr.close(); fresh.close()


def test_graph_replay_equals_eager_and_chunking():
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    L = _lib()
    st = weights.make_state(13)
    model, net = make_product_model(st, "posenet", "tc_split")
    mb = 16
    pr = Predictor(model, max_batch=mb)
    x = torch.randn(2 * mb + 5, 3, 64, 96, generator=torch.Generator().manual_seed(2)).cuda()
    eng = pr._engine(64, 96)
    for B in (1, 5, mb):
        graphed = pr(x[:B])
        graphed2 = pr(x[:B])                            # replay of the captured graph
        eager = torch.empty(B, 6, device="cuda")
        eng.forward(x[:B].contiguous(), eager, 0.0, 0)
        assert torch.equal(graphed, eager) and torch.equal(graphed2, eager), B
    chunked = pr(x)                                     # 16 + 16 + 5 frames
    singles = torch.cat([pr(x[i:i + mb]) for i in range(0, x.shape[0], mb)])
    assert torch.equal(chunked, singles)
    # the tile plan changes with B, the arithmetic per frame may too: frame-by-frame within the live-path bound
    one_by_one = torch.cat([pr(x[i:i + 1]) for i in range(0, 8)])
    assert _rel(chunked[:8], one_by_one) <= 2e-5
    with pytest.raises(RuntimeError, match="no CPU path"):
        pr(x.cpu())
    with pytest.raises(ValueError, match="expected input"):
        pr(x[:, :2])
    pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. dropout, 7. launch counts and errors
# ---------------------------------------------------------------------------------------------------------------------
def test_dropout_mask_follows_the_live_forward():
    from oracle import weights
    from helpers import make_product_model
    L = _lib()
    lib = L.lib()
    st = weights.make_state(4)
    model, net = make_product_model(st, "posenet", "tc_split", droprate=0.5)
    _device_flat(net)
    B, H, W = 6, 64, 64
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(8)).cuda()
    trunk = L.Trunk(B, H, W, net.feat_dim, "tc_split")
    eng = L.Infer(B, H, W, net.feat_dim, "tc_split")
    eng.load(net._flat, net._bufs)
    seed, step = 1234, 17
    live = torch.empty(B, 6, device="cuda")
    L.check(lib.mapnet_forward(trunk.h, x.data_ptr(), net._flat.data_ptr(), net._bufs.data_ptr(), B, 0, 0.5, seed, step,
                               live.data_ptr(), L.stream_ptr()), "mapnet_forward")
    got = torch.empty(B, 6, device="cuda")
    eng.forward(x, got, 0.5, seed, step)
    e = _rel(got, live)
    print("droprate 0.5, same (seed, step): %.2e" % e)
    assert e <= 2e-5, e
    other = torch.empty(B, 6, device="cuda")
    eng.forward(x, other, 0.5, seed, step + 1)
    assert _rel(other, live) > 1e-3                   # a different step draws a different mask
    trunk.close(); eng.close()


def test_launch_count_and_errors_before_any_launch():
    from oracle import weights
    from helpers import make_product_model
    L = _lib()
    lib = L.lib()
    st = weights.make_state(4)
    model, net = make_product_model(st, "posenet", "bf16")
    _device_flat(net)
    H, W = 64, 64
    eng = L.Infer(4, H, W, net.feat_dim, "bf16")
    x = torch.randn(4, 3, H, W, device="cuda")
    pred = torch.empty(4, 6, device="cuda")
    # a forward before a load, a batch above max_B: refused without a launch
    n0 = lib.mapnet_launch_count()
    with pytest.raises(RuntimeError, match="no snapshot loaded"):
        eng.forward(x, pred, 0.0, 0)
    eng.load(net._flat, net._bufs)
    n1 = lib.mapnet_launch_count()
    assert n1 > n0                     # the load packs weights and computes the 36 scale / shift pairs
    big = torch.randn(5, 3, H, W, device="cuda")
    with pytest.raises(RuntimeError, match="outside"):
        eng.forward(big, torch.empty(5, 6, device="cuda"), 0.0, 0)
    assert lib.mapnet_launch_count() == n1
    h = ctypes.c_void_p()
    assert lib.mapnet_infer_create(ctypes.byref(h), 4, H, W, 2048, L.PREC["fp32"]) != 0
    assert lib.mapnet_launch_count() == n1
    # launches per forward: 36 convs + stem operand + pool + head (global average pool, fc with its split-K reduction
    # at small B, fc_xyz, fc_wpqr); no BatchNorm launch, no weight pack
    for B, head in ((1, 6), (4, 6)):
        c0 = lib.mapnet_launch_count()
        eng.forward(x[:B].contiguous(), pred[:B], 0.0, 0)
        assert lib.mapnet_launch_count() - c0 == 36 + 2 + head, (B, lib.mapnet_launch_count() - c0)
    torch.cuda.synchronize()
    eng.close()
