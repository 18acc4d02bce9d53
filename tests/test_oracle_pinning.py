"""The CPU oracle (oracle/mapnet_oracle.py) pinned against outputs of the REFERENCE: the committed goldens in
tests/golden/, made by oracle/make_goldens.py from the reference's own modules (live_reference.npz holds what the
reference modules computed on the configs below, gradients as fixed-stride samples plus full norms)."""
import ast
import os

import numpy as np
import pytest
import torch

from oracle import mapnet_oracle as O
from oracle import weights

SV = dict(sax=0.0, saq=-3.0, srx=0.0, srq=-3.0)


def _golden(golden_dir, name):
    g = np.load(os.path.join(golden_dir, "step_%s.npz" % name))
    return g, ast.literal_eval(str(g["cfg"]))


@pytest.mark.parametrize("name", ["posenet_tiny", "posenet_ragged", "mapnet_tiny", "online_tiny", "online_gps_tiny",
                                  "posenet_7scenes_b4"])
def test_oracle_step_matches_reference_golden(golden_dir, name):
    g, cfg = _golden(golden_dir, name)
    st = weights.make_state(int(g["seed"]))
    x, targ = weights.make_inputs(cfg, int(g["seed"]))
    if "x" in g.files:
        assert np.array_equal(x.numpy(), g["x"]), "input generator drifted"
    if "x_head" in g.files:
        assert np.array_equal(x.numpy().reshape(-1)[:g["x_head"].size], g["x_head"]), "input generator drifted"
    assert abs(float(x.double().sum()) - float(g["x_checksum"])) < 1e-6 * max(1.0, abs(float(g["x_checksum"])))
    assert np.array_equal(targ.numpy(), g["targ"])
    r = O.train_step(cfg["kind"], st, x, targ, SV, lr=cfg.get("lr", 1e-4), weight_decay=cfg.get("wd", 5e-4),
                     max_grad_norm=cfg.get("clip", 0.0), filter_nans=cfg["kind"].startswith("online"))
    # same torch build on both sides -> the restatement reproduces the reference bit for bit
    # (tolerances only guard against thread-count dependent reduction order)
    assert abs(float(r["loss"]) - float(g["loss"])) <= 1e-6 * abs(float(g["loss"]))
    np.testing.assert_allclose(r["pred"].numpy().reshape(g["pred"].shape), g["pred"], rtol=1e-5, atol=1e-6)
    for i, n in enumerate(g["grad_names"]):
        t = r["grads"][str(n)].double()
        assert abs(float(t.norm()) - g["grad_norm"][i]) <= 1e-4 * g["grad_norm"][i] + 1e-12, str(n)
    for i, n in enumerate(g["post_names"]):
        t = r["new_state"][str(n)].double()
        assert abs(float(t.norm()) - g["post_norm"][i]) <= 1e-5 * g["post_norm"][i] + 1e-12, str(n)
    for i, n in enumerate(g["sgrad_names"]):
        if not np.isnan(g["sgrads"][i]):
            assert abs(float(r["sgrads"][str(n)]) - g["sgrads"][i]) <= 1e-5 * abs(g["sgrads"][i]) + 1e-7


def test_oracle_pose_math_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "pose_math.npz"))
    v = torch.tensor(g["qexp_in"])
    np.testing.assert_allclose(O.qexp_t(v).numpy(), g["qexp_out"], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(O.qlog_t(torch.tensor(g["qexp_out"])).numpy(), g["qlog_out"], rtol=1e-6, atol=1e-7)
    for key in ("n5t3", "n16t5", "n3t2", "n4t7"):
        p = torch.tensor(g["vos_in_" + key]).requires_grad_(True)
        np.testing.assert_allclose(O.calc_vos_simple(p).detach().numpy(), g["vos_simple_" + key], rtol=0, atol=0)
        vv = O.calc_vos(p)
        np.testing.assert_allclose(vv.detach().numpy(), g["vos_" + key], rtol=1e-5, atol=1e-6)
        (vv * torch.tensor(g["vos_w_" + key])).sum().backward()
        np.testing.assert_allclose(p.grad.numpy(), g["vos_grad_" + key], rtol=1e-4, atol=1e-5)


def test_known_answer_properties():
    """SURVEY.md section 4 (iii),(iv),(vi): qlog(qexp(v)) == v for |v| < pi; |qexp(v)| = 1;
    calc_vos_simple is a plain difference."""
    g = torch.Generator().manual_seed(1)
    v = torch.randn(100, 3, generator=g)
    v = v / v.norm(dim=1, keepdim=True) * (torch.rand(100, 1, generator=g) * 3.0)
    q = O.qexp_t(v)
    assert float((q.norm(dim=1) - 1).abs().max()) < 1e-6
    assert float((O.qlog_t(q) - v).abs().max()) < 1e-5
    p = torch.randn(4, 5, 6, generator=g)
    assert torch.equal(O.calc_vos_simple(p), p[:, 1:] - p[:, :-1])


def test_flop_model():
    macs, conv1 = O.conv_macs_per_image(256, 256)
    assert macs == 4784652288                      # SURVEY.md section 8d, hook-measured on the live module
    assert abs(O.train_flops_per_image(256, 256) - 28.400e9) < 0.01e9


def _live(golden_dir):
    return np.load(os.path.join(golden_dir, "live_reference.npz"))


def _check_grad_samples(L, prefix, grads):
    """oracle gradients vs the reference's: full norms and the stored fixed-stride samples"""
    for i, k in enumerate(L[prefix + "grad_names"]):
        v = grads[str(k)].detach().double().flatten()
        ref_norm = float(L[prefix + "grad_norm"][i])
        assert abs(float(v.norm()) - ref_norm) <= 1e-5 * ref_norm + 1e-12, k
        sample = v[::int(L[prefix + "grad_stride"][i])].numpy()
        assert float(np.linalg.norm(sample - L[prefix + "grad_%d" % i])) <= 1e-5 * ref_norm + 1e-12, k


@pytest.mark.parametrize("kind,cfg", [("posenet", dict(kind="posenet", N=2, H=64, W=64)),
                                      ("online", dict(kind="online", N=2, T=4, H=64, W=64))])
def test_oracle_matches_live_reference(golden_dir, kind, cfg):
    L = _live(golden_dir)
    st = weights.make_state(3)
    x, targ = weights.make_inputs(cfg, 3)
    r = O.train_step(kind, st, x, targ, SV)
    loss = float(L["step_%s_loss" % kind])
    out = torch.from_numpy(L["step_%s_out" % kind])
    assert abs(float(r["loss"]) - loss) <= 1e-6 * abs(loss)
    assert float((out - r["pred"].view_as(out)).abs().max()) <= 1e-6
    _check_grad_samples(L, "step_%s_" % kind, r["grads"])


def test_oracle_nan_filter_matches_live_reference_hook(golden_dir):
    """models/posenet.py:28-34,50-51 with a NaN-producing gradient: degenerate state (fc_wpqr = 0 -> every predicted
    rotation is the identity -> qlog's backward gives NaN, the case the hook exists for) through the reference
    MapNet + MapNetOnlineCriterion with filter_nans=True, against the oracle.  The hook zeroes NaNs of the Linear's
    bias / input / weight gradients: whole weight rows and whole samples drop out, not single entries."""
    L = _live(golden_dir)
    st = weights.make_state(3)
    st["fc_wpqr.weight"] = torch.zeros_like(st["fc_wpqr.weight"])
    st["fc_wpqr.bias"] = torch.zeros_like(st["fc_wpqr.bias"])
    cfg = dict(kind="online", N=2, T=4, H=64, W=64)
    x, targ = weights.make_inputs(cfg, 3)
    r = O.train_step("online", st, x, targ, SV, filter_nans=True, do_step=False)
    # the unfiltered gradient really is NaN in the rotation half
    r_nofilter = O.train_step("online", st, x, targ, SV, filter_nans=False, do_step=False)
    assert bool(torch.isnan(r_nofilter["grads"]["fc_wpqr.weight"]).any())
    assert bool(L["nanfilter_all_finite"].all())
    for k in L["nanfilter_grad_names"]:
        assert bool(torch.isfinite(r["grads"][str(k)]).all()), k
    _check_grad_samples(L, "nanfilter_", r["grads"])
    ref_w = torch.from_numpy(L["nanfilter_fc_wpqr_weight"])
    assert float((ref_w - r["grads"]["fc_wpqr.weight"]).norm()) <= 1e-5 * float(ref_w.norm()) + 1e-12
    n_zero_rows = sum(int(bool((ref_w[j] == 0).all())) for j in range(3))
    assert n_zero_rows >= 1, "the degenerate input was meant to wipe at least one fc_wpqr row"


def test_baseline_config0_plumbing_single_frame(golden_dir):
    """BASELINE.json configs[0] / SURVEY.md section 8d "Config 1 (plumbing)": PoseNet ResNet-34 on ONE synthetic 256x256 frame,
    PoseNetCriterion(sax=0, saq=-3), seed 7, on the CPU: a [1,6] output and a finite loss -- through the oracle, and
    against what the reference modules computed (tests/golden/live_reference.npz)."""
    st = weights.make_state(7)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(1, 3, 256, 256, generator=g)
    targ = torch.randn(1, 6, generator=g)
    r = O.train_step("posenet", st, x, targ, SV, do_step=False)
    assert tuple(r["pred"].shape) == (1, 6) and bool(torch.isfinite(r["pred"]).all())
    assert np.isfinite(float(r["loss"]))
    # the criterion value follows from the prediction: exp(-sax) L1(t) + sax + exp(-saq) L1(q) + saq (criterion.py:42-52)
    want = float((r["pred"][:, :3] - targ[:, :3]).abs().mean() + 0.0
                 + np.exp(3.0) * (r["pred"][:, 3:] - targ[:, 3:]).abs().mean() - 3.0)
    assert abs(float(r["loss"]) - want) <= 1e-5 * abs(want)
    L = _live(golden_dir)
    loss, out = float(L["config0_loss"]), torch.from_numpy(L["config0_out"])
    assert tuple(out.shape) == (1, 6)
    assert abs(loss - float(r["loss"])) <= 1e-6 * abs(loss)
    assert float((out - r["pred"]).abs().max()) <= 1e-6
