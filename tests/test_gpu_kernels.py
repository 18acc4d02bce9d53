"""Per-kernel GPU parity through the C ABI: conv engines vs torch conv2d (the
third-party arithmetic the reference calls), fused criterion vs the reference's
autograd goldens, fused Adam vs torch.optim.Adam (common/optimizer.py:21-23)."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from geomapnet_b200 import _lib


def _conv_case(precision, B, H, W, Ci, Co, k, stride, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, k, k, generator=g) * (2.0 / (Ci * k * k)) ** 0.5
    pad = (k - 1) // 2
    if precision not in ("fp32", "tc_split"):
        x = x.bfloat16().float(); w = w.bfloat16().float()
    xr = x.clone().requires_grad_(True); wr = w.clone().requires_grad_(True)
    y = F.conv2d(xr, wr, None, stride, pad)
    dy = torch.randn(y.shape, generator=g)
    if precision not in ("fp32", "tc_split"):
        dy = dy.bfloat16().float()
    y.backward(dy)
    return x, w, dy, y.detach(), xr.grad, wr.grad


def _run_conv(precision, kind, x_nhwc, other_nhwc, wmat, out, geom):
    B, H, W, Ci, Co, k, stride = geom
    L = _lib.lib()
    _lib.check(L.mapnet_test_conv(_lib.PREC[precision], kind, B, H, W, Ci, Co, k, stride, x_nhwc.data_ptr(),
                                  other_nhwc.data_ptr() if other_nhwc is not None else None,
                                  wmat.data_ptr() if wmat is not None else None, out.data_ptr(),
                                  _lib.stream_ptr()), "mapnet_test_conv")
    torch.cuda.synchronize()


CASES = [(2, 16, 16, 64, 64, 3, 1), (2, 16, 16, 64, 128, 3, 2), (2, 16, 16, 64, 128, 1, 2),
         (3, 9, 11, 128, 128, 3, 1), (2, 18, 22, 64, 128, 3, 2), (1, 8, 8, 256, 512, 3, 2),
         (2, 8, 8, 512, 512, 3, 1), (1, 32, 32, 192, 64, 1, 1), (4, 64, 64, 64, 64, 3, 1),
         (2, 16, 16, 128, 256, 1, 2), (3, 17, 13, 128, 256, 3, 2)]


@pytest.mark.parametrize("precision", ["fp32", "bf16_simt", "bf16", "tc_split"])
@pytest.mark.parametrize("geom", CASES)
def test_conv_engines(precision, geom):
    """tc_split (strict tensor-core mode): UNROUNDED fp32 operands in, fp32 out -- the entry point cuts them into
    fp16 hi/lo planes (22 significant bits) and the wgmma engines form all four hi/lo products; the bound is the
    fp32 CUDA-core engine's."""
    B, H, W, Ci, Co, k, stride = geom
    x, w, dy, y, dx, dw = _conv_case(precision, *geom)
    act = torch.float32 if precision in ("fp32", "tc_split") else torch.bfloat16
    wt = torch.bfloat16 if precision == "bf16" else torch.float32
    xn = x.permute(0, 2, 3, 1).contiguous().to(act).cuda()
    dyn = dy.permute(0, 2, 3, 1).contiguous().to(act).cuda()
    w_krsc = w.permute(0, 2, 3, 1).contiguous().to(wt).cuda()          # [Co][kh][kw][Ci]
    w_dg = w.permute(1, 2, 3, 0).contiguous().to(wt).cuda()            # [Ci][kh][kw][Co]
    # bf16: output rounding 2^-8 relative.  tc_split: fp32 outputs; what is left is the tensor core's fp32 accumulation
    # (the tensor cores' fp32 accumulation truncates instead of rounding, so the error grows with K)
    tol = {"fp32": 2e-5, "tc_split": 1e-4}.get(precision, 1.2e-2)
    errs = []
    # fprop
    out = torch.empty(y.permute(0, 2, 3, 1).shape, dtype=act, device="cuda")
    _run_conv(precision, 0, xn, None, w_krsc, out, geom)
    ref = y.permute(0, 2, 3, 1)
    errs.append(float((out.float().cpu() - ref).abs().max() / ref.abs().max()))
    # dgrad
    out = torch.empty(xn.shape, dtype=act, device="cuda")
    _run_conv(precision, 1, dyn, None, w_dg, out, geom)
    ref = dx.permute(0, 2, 3, 1)
    errs.append(float((out.float().cpu() - ref).abs().max() / ref.abs().max()))
    # wgrad (fp32 accumulators, accumulated into a zeroed buffer)
    out = torch.zeros(w_krsc.shape, dtype=torch.float32, device="cuda")
    _run_conv(precision, 2, xn, dyn, None, out, geom)
    ref = dw.permute(0, 2, 3, 1)
    errs.append(float((out.cpu() - ref).abs().max() / ref.abs().max()))
    print("conv-engine", precision, geom, "fprop %.2e dgrad %.2e wgrad %.2e" % tuple(errs))
    assert errs[0] < tol and errs[1] < tol and errs[2] < max(5e-5, tol if precision == "tc_split" else 0.0), errs


@pytest.mark.parametrize("shape", [(2, 64, 64), (3, 97, 65), (4, 256, 256)])
def test_tensor_core_stem_matches_conv2d(shape):
    """The bf16 stem (space-to-depth image + overlapped TMA view, layout.cu / conv_tc.cu) against torch's
    7x7/s2/p3 conv2d on the same bf16-rounded operands: output and weight gradient (the stem has no input
    gradient).  Odd sizes exercise the zero halo of the space-to-depth image."""
    B, H, W = shape
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 3, H, W, generator=g)
    w = torch.randn(64, 3, 7, 7, generator=g) * (2.0 / 147) ** 0.5
    xr = x.bfloat16().float(); wr = w.bfloat16().float().requires_grad_(True)
    y = F.conv2d(xr, wr, None, 2, 3)
    dy = torch.randn(y.shape, generator=g).bfloat16().float()
    y.backward(dy)
    Hc, Wc = y.shape[2], y.shape[3]
    xd = x.cuda().contiguous(); wd = w.cuda().contiguous()
    out = torch.empty(B, Hc, Wc, 64, dtype=torch.bfloat16, device="cuda")
    dyn = dy.permute(0, 2, 3, 1).contiguous().bfloat16().cuda()
    dw = torch.zeros(64, 3, 7, 7, dtype=torch.float32, device="cuda")
    L = _lib.lib()
    _lib.check(L.mapnet_test_stem(B, H, W, xd.data_ptr(), wd.data_ptr(), out.data_ptr(), dyn.data_ptr(), dw.data_ptr(),
                                  _lib.stream_ptr()), "mapnet_test_stem")
    torch.cuda.synchronize()
    ref = y.detach().permute(0, 2, 3, 1)
    assert float((out.float().cpu() - ref).abs().max() / ref.abs().max()) < 1.2e-2      # bf16 output rounding
    assert float((dw.cpu() - wr.grad).abs().max() / wr.grad.abs().max()) < 5e-5


# the three downsampling blocks of ResNet-34 at their real channel counts (small batch / maps), plus odd sizes
SHORTCUT_CASES = [(2, 64, 64, 64, 128), (2, 32, 32, 128, 256), (2, 16, 16, 256, 512), (3, 17, 13, 128, 256),
                  (2, 18, 22, 64, 128), (1, 9, 7, 256, 512), (9, 16, 16, 256, 512)]


@pytest.mark.parametrize("geom", SHORTCUT_CASES)
def test_merged_stride2_dgrad_with_folded_shortcut(geom):
    """d(block input) of a downsampling BasicBlock in ONE wgmma launch: the four parity classes of the 3x3/s2
    conv1 dgrad plus the 1x1/s2 downsample dgrad as an extra tap of class (0,0) (conv_tc.cu,
    tc_plan_add_shortcut), against torch autograd through both convs on the same bf16-rounded operands."""
    B, H, W, Ci, Co = geom
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, Ci, H, W, generator=g).bfloat16().float().requires_grad_(True)
    w1 = (torch.randn(Co, Ci, 3, 3, generator=g) * (2.0 / (Ci * 9)) ** 0.5).bfloat16().float()
    w2 = (torch.randn(Co, Ci, 1, 1, generator=g) * (2.0 / Ci) ** 0.5).bfloat16().float()
    y1 = F.conv2d(x, w1, None, 2, 1)
    y2 = F.conv2d(x, w2, None, 2, 0)
    assert y1.shape == y2.shape
    dy1 = torch.randn(y1.shape, generator=g).bfloat16().float()
    dy2 = torch.randn(y2.shape, generator=g).bfloat16().float()
    (y1 * dy1).sum().backward(retain_graph=True)
    dx1 = x.grad.clone()
    (y2 * dy2).sum().backward()
    dx = x.grad                                                   # dx1 + shortcut part
    d1 = dy1.permute(0, 2, 3, 1).contiguous().bfloat16().cuda()
    d2 = dy2.permute(0, 2, 3, 1).contiguous().bfloat16().cuda()
    w1_dg = w1.permute(1, 2, 3, 0).contiguous().bfloat16().cuda()           # [Ci][kh][kw][Co]
    w2_dg = w2.permute(1, 2, 3, 0).contiguous().bfloat16().cuda()           # [Ci][1][1][Co]
    out = torch.full((B, H, W, Ci), float("nan"), dtype=torch.bfloat16, device="cuda")
    L = _lib.lib()
    _lib.check(L.mapnet_test_dgrad_shortcut(B, H, W, Ci, Co, d1.data_ptr(), d2.data_ptr(), w1_dg.data_ptr(),
                                            w2_dg.data_ptr(), out.data_ptr(), _lib.stream_ptr()),
               "mapnet_test_dgrad_shortcut")
    torch.cuda.synchronize()
    ref = dx.permute(0, 2, 3, 1)
    got = out.float().cpu()
    assert bool(torch.isfinite(got).all()), "some output pixel class was not written"
    assert float((got - ref).abs().max() / ref.abs().max()) < 1.2e-2         # bf16 output rounding
    # the shortcut must really be in there: without it the error is O(1)
    assert float((got - dx1.permute(0, 2, 3, 1)).abs().max() / ref.abs().max()) > 0.1


CRIT_KEYS = ["posenet_n64t1", "posenet_n7t1", "mapnet_n32t3", "mapnet_n5t2", "online_n16t10",
             "online_n3t4", "online_gps_n16t10", "online_gps_n2t6"]


@pytest.mark.parametrize("key", CRIT_KEYS)
def test_fused_criterion_vs_reference_autograd(key, golden_dir):
    from helpers import make_product_criterion
    gold = np.load(os.path.join(golden_dir, "pose_math.npz"))
    kind = key.rsplit("_n", 1)[0]
    pred = torch.tensor(gold["crit_pred_" + key]).cuda().requires_grad_(True)
    targ = torch.tensor(gold["crit_targ_" + key]).cuda()
    crit = make_product_criterion(kind)
    loss = crit(pred, targ)
    assert tuple(loss.shape) == (1,)
    loss.backward()
    ref_loss = float(gold["crit_loss_" + key].reshape(-1)[0])
    assert abs(float(loss) - ref_loss) <= 2e-6 * abs(ref_loss) + 1e-6
    ref_d = gold["crit_dpred_" + key]
    assert np.abs(pred.grad.cpu().numpy() - ref_d).max() <= 1e-4 * np.abs(ref_d).max() + 1e-7
    ref_ds = gold["crit_ds_" + key]
    got = [float(p.grad) for _, p in crit.named_parameters()]
    for i in range(len(ref_ds)):
        if not np.isnan(ref_ds[i]):
            assert abs(got[i] - ref_ds[i]) <= 2e-6 * abs(ref_ds[i]) + 1e-6


def test_fused_adam_matches_torch_adam():
    from geomapnet_b200.common.optimizer import FusedAdam
    torch.manual_seed(0)
    flat = torch.randn(10240, device="cuda")
    shapes = [(100, 50), (4999,), (1,)]
    offs = [0, 5056, 10112]
    ps, qs = [], []
    for s, o in zip(shapes, offs):
        n = int(np.prod(s))
        ps.append(torch.nn.Parameter(flat[o:o + n].view(s)))
        qs.append(torch.nn.Parameter(flat[o:o + n].view(s).clone()))
    a = FusedAdam(ps, lr=1e-2, weight_decay=5e-4)
    b = torch.optim.Adam(qs, lr=1e-2, weight_decay=5e-4)
    gflat = torch.zeros_like(flat)
    for it in range(5):
        g = torch.randn_like(flat)
        gflat.copy_(g)
        for p, q, s, o in zip(ps, qs, shapes, offs):
            n = int(np.prod(s))
            p.grad = gflat[o:o + n].view(s)
            q.grad = g[o:o + n].view(s).clone()
        a.step(); b.step()
    for p, q in zip(ps, qs):
        assert torch.allclose(p, q, rtol=2e-5, atol=1e-6)
    sd = a.state_dict()
    assert set(sd["state"][0].keys()) >= {"step", "exp_avg", "exp_avg_sq"}


def test_fused_adam_clip_matches_clip_grad_norm():
    from geomapnet_b200.common.optimizer import FusedAdam
    torch.manual_seed(1)
    p = torch.nn.Parameter(torch.randn(4096, device="cuda")); q = torch.nn.Parameter(p.detach().clone())
    g = torch.randn(4096, device="cuda") * 3
    p.grad = g.clone(); q.grad = g.clone()
    a = FusedAdam([p], lr=1e-3); b = torch.optim.Adam([q], lr=1e-3)
    torch.nn.utils.clip_grad_norm_([q], 5.0)
    a.step(max_grad_norm=5.0); b.step()
    assert torch.allclose(p, q, rtol=1e-5, atol=1e-7)


# ---------------------------------------------------------------------------------------------------------------------
# the FUSED epilogues of the wgmma engines against torch (not product-vs-product): BatchNorm statistics in fprop,
# ReLU gate + BatchNorm-backward reductions (+ residual) in dgrad
# ---------------------------------------------------------------------------------------------------------------------
EPI_CASES = [(2, 16, 16, 64, 64, 3, 1), (3, 9, 11, 128, 128, 3, 1), (2, 18, 22, 64, 128, 3, 2), (1, 8, 8, 256, 512, 3, 2),
             (2, 8, 8, 512, 512, 3, 1), (4, 64, 64, 64, 64, 3, 1), (2, 16, 16, 128, 256, 1, 2)]


def _run_epilogue(kind, geom, in0, wmat, residual, y, zmask, yd, mscale, mshift, out, C):
    B, H, W, Ci, Co, k, stride = geom
    sums = np.zeros((3, C), dtype=np.float64)
    ptr = lambda t: t.data_ptr() if t is not None else None
    _lib.check(_lib.lib().mapnet_test_conv_epilogue(
        kind, B, H, W, Ci, Co, k, stride, ptr(in0), ptr(wmat), ptr(residual), ptr(y), ptr(zmask), ptr(yd), ptr(mscale),
        ptr(mshift), ptr(out), sums.ctypes.data_as(ctypes.c_void_p), _lib.stream_ptr()), "mapnet_test_conv_epilogue")
    torch.cuda.synchronize()
    return sums


@pytest.mark.parametrize("geom", EPI_CASES)
def test_fprop_fused_batchnorm_statistics_vs_torch(geom):
    """out = conv(x, w) stored as bf16; (sum, sum of squares) per channel of the STORED values, accumulated in the conv
    epilogue -- what BatchNorm's training-mode forward then normalises with."""
    B, H, W, Ci, Co, k, stride = geom
    x, w, dy, y, dx, dw = _conv_case("bf16", *geom)
    xn = x.permute(0, 2, 3, 1).contiguous().bfloat16().cuda()
    w_krsc = w.permute(0, 2, 3, 1).contiguous().bfloat16().cuda()
    out = torch.empty(y.permute(0, 2, 3, 1).shape, dtype=torch.bfloat16, device="cuda")
    sums = _run_epilogue(0, geom, xn, w_krsc, None, None, None, None, None, None, out, Co)
    ref = y.permute(0, 2, 3, 1)
    assert float((out.float().cpu() - ref).abs().max() / ref.abs().max()) < 1.2e-2
    stored = out.float().cpu().double().reshape(-1, Co)           # the statistics are those of the stored tensor
    s0, s1 = stored.sum(0).numpy(), (stored * stored).sum(0).numpy()
    assert np.abs(sums[0] - s0).max() <= 2e-5 * np.abs(stored).sum(0).max().item()
    assert np.abs(sums[1] - s1).max() <= 2e-5 * s1.max()


@pytest.mark.parametrize("variant", ["ymask", "zmask", "zmask_res", "zmask_res_yd"])
@pytest.mark.parametrize("geom", EPI_CASES)
def test_dgrad_fused_relu_gate_and_batchnorm_backward_sums_vs_torch(geom, variant):
    """g = [gate] * (conv_dgrad(dy, w) [+ residual]) stored as bf16 and (sum g, sum g*y [, sum g*yd]) of the stored
    values: the ReLU backward and the reduction half of BatchNorm's backward of the layer that CONSUMES this gradient,
    fused into the dgrad epilogue.  Gate: the post-ReLU tensor's sign (zmask) or the recomputed activation
    mscale * y + mshift > 0."""
    B, H, W, Ci, Co, k, stride = geom
    x, w, dy, yref, dx, dw = _conv_case("bf16", *geom)
    gen = torch.Generator().manual_seed(1)
    shape = (B, H, W, Ci)                                           # the dgrad output is shaped like the conv input
    dyn = dy.permute(0, 2, 3, 1).contiguous().bfloat16().cuda()
    w_dg = w.permute(1, 2, 3, 0).contiguous().bfloat16().cuda()
    ybn = torch.randn(shape, generator=gen).bfloat16()              # the consumer BatchNorm's input (a forward conv output)
    ydn = torch.randn(shape, generator=gen).bfloat16()
    res = torch.randn(shape, generator=gen).bfloat16()
    msc = (torch.rand(Ci, generator=gen) + 0.5)
    msh = torch.randn(Ci, generator=gen) * 0.3
    z = torch.relu(torch.randn(shape, generator=gen)).bfloat16()    # post-ReLU tensor: zeros where the gate is closed
    use_z = variant != "ymask"
    use_res = "res" in variant
    use_yd = variant.endswith("yd")
    out = torch.empty(shape, dtype=torch.bfloat16, device="cuda")
    sums = _run_epilogue(1, geom, dyn, w_dg, res.cuda() if use_res else None, ybn.cuda(), z.cuda() if use_z else None,
                         ydn.cuda() if use_yd else None, None if use_z else msc.cuda(), None if use_z else msh.cuda(), out, Ci)
    g = dx.permute(0, 2, 3, 1).float()
    if use_res:
        g = g + res.float()
    gate = (z.float() > 0) if use_z else ((ybn.float() * msc + msh) > 0)
    g = torch.where(gate, g, torch.zeros_like(g))
    got = out.float().cpu()
    assert float((got - g).abs().max() / g.abs().max()) < 1.2e-2
    assert torch.equal(got == 0, ~gate | (got == 0)) and bool((got[~gate] == 0).all())     # closed gates store exact zeros
    st = got.double().reshape(-1, Ci)
    yy, yd2 = ybn.double().reshape(-1, Ci), ydn.double().reshape(-1, Ci)
    scale = st.abs().sum(0).max().item()
    assert np.abs(sums[0] - st.sum(0).numpy()).max() <= 2e-5 * scale
    assert np.abs(sums[1] - (st * yy).sum(0).numpy()).max() <= 2e-5 * (st.abs() * yy.abs()).sum(0).max().item()
    if use_yd:
        assert np.abs(sums[2] - (st * yd2).sum(0).numpy()).max() <= 2e-5 * (st.abs() * yd2.abs()).sum(0).max().item()
