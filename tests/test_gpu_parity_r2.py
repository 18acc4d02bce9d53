"""GPU parity, second layer of evidence (through the reference-facing nn.Module surface and the C ABI):

 * the NaN filter of models/posenet.py:28-34 on the DEVICE -- degenerate rotations through the fused criterion
   (NaN positions of d pred) and through the whole step with filter_nans=True (hook semantics: whole fc_wpqr rows /
   whole samples drop out), against the oracle, which tests/test_oracle_pinning.py pins to the reference module's
   own hook;
 * the bf16 tensor-core product against the ORACLE RUN WITH THE SAME ROUNDING POINTS (oracle emulate="bf16",
   fixtures tests/golden/emu_bf16_*.npz).  Measured: only ~2x closer than to the fp32 reference -- two bf16
   implementations that round at the same points still differ at the percent level after 36 layers (summation order moves
   individual roundings and ReLU masks); the bounds document that noise floor, kernel correctness is carried by the
   per-conv and per-epilogue unit tests (tests/test_gpu_kernels.py) and by the strict mode;
 * the strict tensor-core product against the f16x2-emulating oracle;
 * multi-step trajectories with gradient clipping and learnable criterion scalars (clip_grad_norm_ covers
   model.parameters() only: common/train.py:357-358).
"""
import os

import numpy as np
import pytest
import torch

from helpers import (GOLDEN, SVALS, load_golden, make_product_model, make_product_criterion, product_step)

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------
# a5: NaN filter on the device
# ------------------------------------------------------------------------------------------------------------------
def test_criterion_nan_positions_match_reference_on_degenerate_rotations(golden_dir):
    """tests/golden/pose_math.npz:vos_degen_*: identical consecutive rotations -> the reference's calc_vos backward
    yields NaN in d pred (acos'(1) * 0).  The fused criterion must produce NaN in exactly the same entries (they are
    what filter_hook later removes) and the reference's values everywhere else."""
    from oracle import mapnet_oracle as O
    gold = np.load(os.path.join(golden_dir, "pose_math.npz"))
    poses = torch.tensor(gold["vos_degen_in"])                     # [2,3,6], all rotations equal
    N, T = poses.shape[0], poses.shape[1]
    g = torch.Generator().manual_seed(3)
    abs_part = torch.randn(N, T, 6, generator=g) * 0.3
    pred = torch.cat([abs_part, poses], 1)                          # [N, 2T, 6]: T absolute poses | T poses for the VOs
    targ = torch.randn(N, 2 * T - 1, 6, generator=g) * 0.3
    # oracle (CPU, the reference's arithmetic)
    pr = pred.clone().requires_grad_(True)
    S = {k: torch.tensor([v], requires_grad=True) for k, v in SVALS.items()}
    lo = O.criterion("online", pr, targ, S)
    lo.backward()
    ref_d = pr.grad.numpy()
    assert np.isnan(ref_d).any(), "the degenerate input was meant to produce NaN gradients"
    assert np.isnan(ref_d[:, :T]).sum() == 0 and np.isnan(ref_d[:, T:, :3]).sum() == 0
    # product
    crit = make_product_criterion("online")
    pd = pred.cuda().requires_grad_(True)
    loss = crit(pd, targ.cuda())
    loss.backward()
    got = pd.grad.cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(ref_d)), (np.isnan(got).sum(), np.isnan(ref_d).sum())
    fin = ~np.isnan(ref_d)
    assert np.abs(got[fin] - ref_d[fin]).max() <= 1e-4 * np.abs(ref_d[fin]).max() + 1e-7
    assert abs(float(loss) - float(lo)) <= 2e-6 * abs(float(lo)) + 1e-6


@pytest.mark.parametrize("precision", ["fp32", "tc_split", "bf16"])
def test_filter_nans_step_matches_reference_hook_semantics(precision):
    """fc_wpqr = 0 -> every predicted rotation is the identity -> NaN in d pred[..., 3:] for the VO half.  With
    filter_nans=True the reference zeroes the NaNs of fc_wpqr's bias / input / weight gradients; the step must come out
    finite and equal to the oracle's (pinned to the reference hook in tests/test_oracle_pinning.py)."""
    from oracle import weights, mapnet_oracle as O
    st = weights.make_state(3)
    st["fc_wpqr.weight"] = torch.zeros_like(st["fc_wpqr.weight"])
    st["fc_wpqr.bias"] = torch.zeros_like(st["fc_wpqr.bias"])
    cfg = dict(kind="online", N=2, T=4, H=64, W=64)
    x, targ = weights.make_inputs(cfg, 3)
    r = O.train_step("online", st, x, targ, SVALS, filter_nans=True, do_step=False)
    model, net = make_product_model(st, "online", precision, filter_nans=True)
    crit = make_product_criterion("online")
    model.train()
    loss, pred, grads, sgrads = product_step(model, net, crit, x, targ, do_step=False)
    for n, gt in grads.items():
        assert bool(torch.isfinite(gt).all()), n
    tight = precision != "bf16"
    assert abs(float(loss) - float(r["loss"])) <= (1e-4 if tight else 5e-2) * abs(float(r["loss"]))
    # the head sees the hook directly: rows of fc_wpqr wiped by a NaN stay wiped, the others carry the reference values
    for n in ("fc_wpqr.weight", "fc_wpqr.bias", "fc_xyz.weight", "fc_xyz.bias"):
        ref = r["grads"][n]
        got = grads[n].cpu()
        # which output rows are wiped entirely (element-wise zeros also come from dead ReLU features, which bf16 may flip)
        wiped_ref = [bool((ref[j] == 0).all()) for j in range(3)]
        wiped_got = [bool((got[j] == 0).all()) for j in range(3)]
        if n.endswith(".weight"):
            assert wiped_got == wiped_ref, (n, wiped_got, wiped_ref)
        else:
            # a bias gradient is a sum of +-c terms (L1 loss): it can be exactly 0 without any wipe when the signs balance
            # (seen in bf16, where one flipped sign balanced fc_xyz.bias[2]) -- only "wiped in the reference => wiped here"
            assert all(g or not w for g, w in zip(wiped_got, wiped_ref)), (n, wiped_got, wiped_ref)
        # bf16 on this 8-frame 64x64 config is at its noise floor (2x2 maps and 8-sample BatchNorm statistics at layer4:
        # measured 0.37 .. 0.67 on these tensors, moving with every change of a summation order): in that mode the test is
        # about the hook STRUCTURE asserted above; the value bound only says "error smaller than the signal"
        assert float((got - ref).norm()) <= (2e-3 if tight else 1.0) * float(ref.norm()) + 1e-12, n
    assert any(bool((r["grads"]["fc_wpqr.weight"][j] == 0).all()) for j in range(3)), "no fc_wpqr row was wiped"
    # and the trunk receives nothing from the samples whose rotation gradient was NaN
    ref = r["grads"]["feature_extractor.fc.weight"]
    e = float((grads["feature_extractor.fc.weight"].cpu() - ref).norm() / ref.norm())
    print("filter_nans", precision, "fc.weight rel err", e)
    assert e <= (5e-3 if tight else 1.0), e
    # without the filter the same step is NaN -- the test input really exercises the hook
    model2, net2 = make_product_model(st, "online", precision, filter_nans=False)
    model2.train()
    _, _, grads2, _ = product_step(model2, net2, make_product_criterion("online"), x, targ, do_step=False)
    assert bool(torch.isnan(grads2["fc_wpqr.weight"]).any())


# ------------------------------------------------------------------------------------------------------------------
# product vs the oracle run with the product's rounding points
# ------------------------------------------------------------------------------------------------------------------
def _emu(emulate, name):
    e = np.load(os.path.join(GOLDEN, "emu_%s_%s.npz" % (emulate, name)), allow_pickle=False)
    return e


def _vs_emulated(emulate, precision, name):
    from oracle import weights
    e = _emu(emulate, name)
    g, cfg = load_golden(name)
    st = weights.make_state(int(e["seed"]))
    x, targ = weights.make_inputs(cfg, int(e["seed"]))
    assert abs(float(x.double().sum()) - float(e["x_checksum"])) < 1e-6 * max(1.0, abs(float(e["x_checksum"])))
    kind = cfg["kind"]
    model, net = make_product_model(st, kind, precision, filter_nans=kind.startswith("online"))
    crit = make_product_criterion(kind)
    model.train()
    loss, pred, grads, _ = product_step(model, net, crit, x, targ, do_step=False)
    out = {"loss": abs(float(loss) - float(e["loss"])) / abs(float(e["loss"]))}
    p = pred.cpu().numpy().reshape(e["pred"].shape)
    out["pred"] = float(np.abs(p - e["pred"]).max() / np.abs(e["pred"]).max())
    # the same two numbers against the fp32 REFERENCE golden, for the side-by-side picture
    out["loss_vs_fp32_ref"] = abs(float(loss) - float(g["loss"])) / abs(float(g["loss"]))
    out["pred_vs_fp32_ref"] = float(np.abs(p - g["pred"].reshape(p.shape)).max() / np.abs(g["pred"]).max())
    gn = 0.0
    for i, n in enumerate(e["grad_names"]):
        t = float(grads[str(n)].double().norm())
        gn = max(gn, abs(t - float(e["grad_norm"][i])) / (float(e["grad_norm"][i]) + 1e-30))
    out["grad_norm"] = gn
    per = {}
    for i, n in enumerate(e["grad_full_names"]):
        ref = e["grad_full_%d" % i].astype(np.float64)
        t = grads[str(n)].double().cpu().flatten().numpy()
        t = t[::max(1, t.size // 40000)]
        per[str(n)] = float(np.linalg.norm(t - ref) / (np.linalg.norm(ref) + 1e-30))
    out["grad_full"] = per
    print("vs-emulated-oracle", emulate, precision, name, {k: (("%.3e" % v) if isinstance(v, float) else v) for k, v in out.items()})
    return out


@pytest.mark.parametrize("name", ["posenet_b8_256", "posenet_b64_256", "mapnet_n32t3_256", "online_n16t10_256"])
def test_step_bf16_matches_bf16_emulating_oracle(name):
    """Identical rounding points on both sides (bf16 operands, bf16-stored activations and gradients, fp32
    accumulation / BN / loss).  The product sits only ~2x closer to the emulating oracle than to the fp32 reference.
    Rounding at the same
    POINTS does not make two bf16 implementations agree: a different fp32 summation order moves individual bf16
    roundings / ReLU masks, and 36 conv+BN layers at random initialisation amplify that to the percent level.  The
    independent CUDA-core bf16 engine differs from the wgmma one by the same amount
    (test_tensor_core_path_matches_cuda_core_path_on_bf16: pose 2.9e-2).  So these bounds (~2x measured) document the
    bf16 noise floor; kernel CORRECTNESS is carried by the per-conv / per-epilogue unit tests (bit-level operands
    against torch) and by the strict tensor-core mode, which meets 1e-4.  The tail of the backward pass (head, last
    conv) is compared element-wise."""
    r = _vs_emulated("bf16", "bf16", name)
    assert r["loss"] <= 1.5e-2, r
    assert r["pred"] <= 7e-2, r
    assert r["pred"] <= r["pred_vs_fp32_ref"], r        # closer to the oracle that rounds like it than to fp32
    assert r["grad_full"]["fc_wpqr.weight"] <= 7e-2, r
    assert r["grad_full"]["feature_extractor.fc.weight"] <= 9e-2, r
    assert r["grad_full"]["feature_extractor.layer4.2.conv2.weight"] <= 7e-1, r


@pytest.mark.parametrize("name", ["posenet_b8_256", "posenet_b64_256"])
def test_step_tc_split_matches_f16x2_emulating_oracle(name):
    r = _vs_emulated("f16x2", "tc_split", name)
    assert r["loss"] <= 1e-4 and r["pred"] <= 1e-4, r
    # measured: head 1e-6 .. 3e-6, last conv 4e-3 .. 6e-3 (first ReLU-mask flips), early layers 1.3e-2
    assert r["grad_full"]["fc_wpqr.weight"] <= 1e-4 and r["grad_full"]["feature_extractor.fc.weight"] <= 1e-4, r
    assert r["grad_full"]["feature_extractor.layer4.2.conv2.weight"] <= 1.5e-2, r
    assert max(r["grad_full"].values()) <= 4e-2, r


# ------------------------------------------------------------------------------------------------------------------
# multi-step trajectory with clipping + learnable criterion scalars (ADVICE r1: the clip covers the model group only)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "tc_split"])
def test_multi_step_clip_with_learnable_scalars_matches_oracle_trainer(precision):
    """Six steps with max_grad_norm small enough to always clip and learnable sax/saq/srx/srq, against
    oracle.OracleTrainer, which clips list(P.values()) only and lets Adam see the criterion scalars' gradients unscaled
    (common/train.py:357-359, scripts/train.py:104-110).  One step cannot tell (Adam's first step is scale invariant);
    over several steps a per-step-varying clip coefficient applied to the scalars changes m / sqrt(v) and their
    trajectory.  The model group's learning rate is tiny so that both sides see (nearly) the same network each step --
    with a visible rate the 22 M sign-like Adam updates make the loss trajectory chaotic within three steps."""
    from oracle import weights, mapnet_oracle as O
    from geomapnet_b200.common.optimizer import Optimizer
    st = weights.make_state(5)
    cfg = dict(kind="mapnet", N=2, T=3, H=64, W=64)
    lr_model, lr_s, clip, steps = 1e-7, 1e-2, 0.05, 6
    xs = [weights.make_inputs(cfg, 20 + i) for i in range(steps)]
    tr = O.OracleTrainer("mapnet", st, SVALS, lr=lr_model, weight_decay=0.0, max_grad_norm=clip, droprate=0.0)
    tr.opt.param_groups[1]["lr"] = lr_s
    ref_losses = [tr.step(x, t) for x, t in xs]
    model, net = make_product_model(st, "mapnet", precision)
    crit = make_product_criterion("mapnet")
    model.train()
    opt = Optimizer(params=[{"params": model.parameters()}, {"params": list(crit.parameters())}], method="adam",
                    base_lr=lr_model, weight_decay=0.0)
    opt.learner.param_groups[1]["lr"] = lr_s
    losses = []
    for x, t in xs:
        loss = crit(model(x.cuda()), t.cuda())
        opt.learner.zero_grad()
        loss.backward()
        opt.learner.step(max_grad_norm=clip)
        losses.append(float(loss))
    print("multi-step", precision, losses, ref_losses)
    for a, b in zip(losses, ref_losses):
        assert abs(a - b) <= 2e-3 * abs(b), (losses, ref_losses)
    moved = 0.0
    for k in ("sax", "saq", "srx", "srq"):
        got, ref = float(getattr(crit, k)), float(tr.S[k])
        moved = max(moved, abs(ref - SVALS[k]))
        assert abs(got - ref) <= 0.05 * lr_s, (k, got, ref, SVALS[k])
    assert moved >= 3 * lr_s, "the scalars were meant to move by several steps"
