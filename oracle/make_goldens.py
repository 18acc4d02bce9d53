"""Regenerate tests/golden/*.npz by RUNNING THE REFERENCE (build container only).

TEST INFRASTRUCTURE.  Usage:  python -m oracle.make_goldens [--full]

Every golden holds the outputs of the reference's own modules
(models/posenet.py, common/criterion.py, common/pose_utils.py, executed from
the reference tree through oracle.ref_loader) on seed-generated inputs and
seed-generated weights (oracle.weights).  Inputs/weights are NOT stored for the
large configs -- they are regenerated from the seed on the test side; a
checksum of each guards against generator drift.
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

from . import ref_loader, weights

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

SVALS = dict(sax=0.0, saq=-3.0, srx=0.0, srq=-3.0)   # scripts/train.py:59-66 + mapnet.ini beta/gamma

# name -> cfg.  T is the frame count the MODEL sees per tuple.
STEP_CONFIGS = {
    "posenet_tiny":     dict(kind="posenet", N=4, H=64, W=64),
    "posenet_ragged":   dict(kind="posenet", N=3, H=72, W=88),
    "mapnet_tiny":      dict(kind="mapnet", N=2, T=3, H=64, W=64),
    "online_tiny":      dict(kind="online", N=2, T=6, H=64, W=64, lr=1e-5, wd=0.0, clip=5.0),
    "online_gps_tiny":  dict(kind="online_gps", N=2, T=6, H=64, W=64, lr=1e-5, wd=0.0, clip=5.0),
    "posenet_b8_256":   dict(kind="posenet", N=8, H=256, W=256),
    # the shape real 7Scenes frames (640x480) reach the net with after Resize(256), no crop
    # (scripts/train.py:119-128; SURVEY.md section 8d): odd width, feature maps 128x171 ... 8x11
    "posenet_7scenes_b4": dict(kind="posenet", N=4, H=256, W=341),
}
FULL_CONFIGS = {
    "posenet_b64_256":  dict(kind="posenet", N=64, H=256, W=256),            # BASELINE configs[1]
    "mapnet_n32t3_256": dict(kind="mapnet", N=32, T=3, H=256, W=256),        # BASELINE configs[2]
    # BASELINE configs[4] per-GPU shape: MapNet++ steps=5 through MFOnline (2T = 10 frames), bs16 = 160 frames,
    # MapNetOnlineCriterion, lr 1e-5, wd 0, max_grad_norm 5, filter_nans (mapnet++_7Scenes.ini:15-20)
    "online_n16t10_256": dict(kind="online", N=16, T=10, H=256, W=256, lr=1e-5, wd=0.0, clip=5.0),
}


def _crit(ns, kind):
    if kind == "posenet":
        return ns.PoseNetCriterion(sax=SVALS["sax"], saq=SVALS["saq"], learn_beta=True)
    kw = dict(sax=SVALS["sax"], saq=SVALS["saq"], srx=SVALS["srx"], srq=SVALS["srq"],
              learn_beta=True, learn_gamma=True)
    if kind == "mapnet":
        return ns.MapNetCriterion(**kw)
    return ns.MapNetOnlineCriterion(gps_mode=(kind == "online_gps"), **kw)


# Gradient tensors kept ELEMENT-WISE (a per-tensor norm cannot see a gradient written in the wrong layout): one per
# stage of the backward pass -- the stem, the first block, a downsample conv, the last conv, the first fc.  Tensors
# larger than FULL_CAP elements are sampled with a fixed stride (deterministic; the rule is stored with the data).
FULL_GRAD_NAMES = ["feature_extractor.conv1.weight", "feature_extractor.layer1.0.conv1.weight",
                   "feature_extractor.layer2.0.downsample.0.weight", "feature_extractor.layer3.0.conv1.weight",
                   "feature_extractor.layer4.2.conv2.weight", "feature_extractor.fc.weight", "fc_wpqr.weight",
                   "feature_extractor.layer1.0.bn1.weight", "feature_extractor.layer4.2.bn2.bias"]
FULL_CAP = 40000


def sample_stride(numel):
    return max(1, numel // FULL_CAP)


def tensor_stats(t):
    t = t.detach().double().flatten()
    head = torch.zeros(8, dtype=torch.float64)
    n = min(8, t.numel())
    head[:n] = t[:n]
    return float(t.sum()), float(t.norm()), head.numpy()


def run_step_config(name, cfg, seed=7):
    ns = ref_loader.load()
    st = weights.make_state(seed)
    x, targ = weights.make_inputs(cfg, seed)
    kind = cfg["kind"]
    model = ref_loader.build_reference_model(st, "posenet" if kind == "posenet" else "mapnet",
                                             droprate=0.0, filter_nans=kind.startswith("online"))
    model.train()
    crit = _crit(ns, kind)
    t0 = time.time()
    loss, pred, grads, cgrads = ref_loader.reference_step(
        model, crit, x, targ, lr=cfg.get("lr", 1e-4), weight_decay=cfg.get("wd", 5e-4),
        max_grad_norm=cfg.get("clip", 0.0))
    dt = time.time() - t0
    names = [k.replace("mapnet.", "", 1) for k in grads.keys()]
    gsum, gnorm, ghead = [], [], []
    for k in grads:
        s, n, h = tensor_stats(grads[k])
        gsum.append(s), gnorm.append(n), ghead.append(h)
    post = model.state_dict()
    pnames, psum, pnorm, phead = [], [], [], []
    for k, v in post.items():
        if k.endswith("num_batches_tracked"):
            continue
        s, n, h = tensor_stats(v)
        pnames.append(k.replace("mapnet.", "", 1)), psum.append(s), pnorm.append(n), phead.append(h)
    out = dict(
        name=name, seed=seed, cfg=repr(cfg), ref_seconds=dt,
        x_checksum=float(x.double().sum()), targ=targ.numpy(),
        pred=pred.numpy(), loss=np.float64(loss),
        grad_names=np.array(names), grad_sum=np.array(gsum), grad_norm=np.array(gnorm),
        grad_head=np.stack(ghead),
        post_names=np.array(pnames), post_sum=np.array(psum), post_norm=np.array(pnorm),
        post_head=np.stack(phead),
        grad_full_names=np.array(FULL_GRAD_NAMES),
        sgrad_names=np.array(list(cgrads.keys())),
        sgrads=np.array([float(v) if v is not None else np.nan for v in cgrads.values()]),
        post_svals=np.array([float(p.detach()) for _, p in crit.named_parameters()]),
    )
    by_name = dict(zip(names, grads.values()))
    for i, n in enumerate(FULL_GRAD_NAMES):
        t = by_name[n].detach().flatten()
        out["grad_full_%d" % i] = t[::sample_stride(t.numel())].numpy().copy()
    if x.numel() <= 6 * 3 * 64 * 64:
        out["x"] = x.numpy()
    elif x.numel() <= 4 * 6 * 3 * 64 * 64:       # keeps the file under 1 MB; the tail is covered by x_checksum
        out["x_head"] = x.flatten()[:1 << 16].numpy().copy()
    np.savez_compressed(os.path.join(GOLD, "step_%s.npz" % name), **out)
    print("golden step_%s: loss=%.6f  ref time %.2fs" % (name, loss, dt), flush=True)


# (emulation mode, config): fixtures of the ORACLE (not of the reference) run with the product's rounding points,
# see mapnet_oracle.py `emulate`.  They separate "the narrow format is coarse" from "the kernel is wrong": the bf16
# product is ~4e-2 off the fp32 reference on the pose, but must sit much closer to the oracle that rounds where it does.
EMU_CONFIGS = [("bf16", "posenet_b8_256"), ("bf16", "posenet_b64_256"), ("bf16", "mapnet_n32t3_256"),
               ("bf16", "online_n16t10_256"), ("f16x2", "posenet_b8_256"), ("f16x2", "posenet_b64_256")]


def run_emulated(emulate, name, seed=7):
    from . import mapnet_oracle as O
    cfg = dict(STEP_CONFIGS, **FULL_CONFIGS)[name]
    st = weights.make_state(seed)
    x, targ = weights.make_inputs(cfg, seed)
    kind = cfg["kind"]
    t0 = time.time()
    r = O.train_step(kind, st, x, targ, SVALS, lr=cfg.get("lr", 1e-4), weight_decay=cfg.get("wd", 5e-4),
                     max_grad_norm=cfg.get("clip", 0.0), emulate=emulate, do_step=False,
                     filter_nans=kind.startswith("online"))
    names = list(r["grads"].keys())
    out = dict(name=name, emulate=emulate, seed=seed, cfg=repr(cfg), oracle_seconds=time.time() - t0,
               x_checksum=float(x.double().sum()), loss=np.float64(float(r["loss"])), pred=r["pred"].numpy(),
               grad_names=np.array(names), grad_norm=np.array([float(r["grads"][k].double().norm()) for k in names]),
               grad_full_names=np.array(FULL_GRAD_NAMES))
    for i, n in enumerate(FULL_GRAD_NAMES):
        t = r["grads"][n].detach().flatten()
        out["grad_full_%d" % i] = t[::sample_stride(t.numel())].numpy().copy()
    np.savez_compressed(os.path.join(GOLD, "emu_%s_%s.npz" % (emulate, name)), **out)
    print("oracle fixture emu_%s_%s: loss=%.6f  (%.1fs)" % (emulate, name, float(r["loss"]), out["oracle_seconds"]), flush=True)


def run_pose_math(seed=7):
    """Known-answer vectors for the torch pose math and criteria alone
    (common/pose_utils.py:21-260, common/criterion.py), incl. edge cases."""
    ns = ref_loader.load()
    pu = ns.pose_utils
    g = torch.Generator().manual_seed(seed)
    out = {}
    v = torch.randn(64, 3, generator=g)
    v[0] = 0.0                      # zero rotation: clamp(1e-8) path (pose_utils.py:80)
    v[1] = torch.tensor([1e-9, 0, 0])
    v[2] = torch.tensor([3.0, 0.5, -0.2])   # |v| > pi/2
    out["qexp_in"] = v.numpy()
    out["qexp_out"] = pu.qexp_t(v).numpy()
    q = pu.qexp_t(v)
    out["qlog_out"] = pu.qlog_t(q).numpy()
    for N, T in ((5, 3), (16, 5), (3, 2), (4, 7)):
        poses = torch.cat([torch.randn(N, T, 3, generator=g), 0.8 * torch.randn(N, T, 3, generator=g)], 2)
        poses.requires_grad_(True)
        vs = pu.calc_vos_simple(poses)
        vv = pu.calc_vos(poses)
        w = torch.randn(vv.shape, generator=g)
        (vv * w).sum().backward()
        key = "n%dt%d" % (N, T)
        out["vos_in_" + key] = poses.detach().numpy()
        out["vos_simple_" + key] = vs.detach().numpy()
        out["vos_" + key] = vv.detach().numpy()
        out["vos_w_" + key] = w.numpy()
        out["vos_grad_" + key] = poses.grad.numpy()
    # criteria with gradients
    for kind, N, T in (("posenet", 64, 1), ("posenet", 7, 1), ("mapnet", 32, 3), ("mapnet", 5, 2),
                       ("online", 16, 10), ("online", 3, 4), ("online_gps", 16, 10), ("online_gps", 2, 6)):
        cfg = dict(kind=kind, N=N, T=T, H=1, W=1)
        _, targ = weights.make_inputs(cfg, seed + N)
        if kind == "posenet":
            pred = targ.clone()
        else:   # the model predicts T absolute poses per tuple
            _, pred = weights.make_inputs(dict(kind="mapnet", N=N, T=T, H=1, W=1), seed + N)
        pred = pred + 0.3 * torch.randn(pred.shape, generator=g)
        pred.requires_grad_(True)
        crit = _crit(ns, kind)
        loss = crit(pred, targ)
        loss.backward()
        key = "%s_n%dt%d" % (kind, N, T)
        out["crit_pred_" + key] = pred.detach().numpy()
        out["crit_targ_" + key] = targ.numpy()
        out["crit_loss_" + key] = loss.detach().numpy()
        out["crit_dpred_" + key] = pred.grad.numpy()
        out["crit_ds_" + key] = np.array([float(p.grad) if p.grad is not None else np.nan
                                          for _, p in crit.named_parameters()])
    # degenerate: identical consecutive predicted rotations -> NaN gradient in the
    # reference (acos'(1) * 0), the case filter_hook exists for (posenet.py:28-34)
    poses = torch.zeros(2, 3, 6)
    poses[:, :, :3] = torch.randn(2, 3, 3, generator=g)
    poses[:, :, 3:] = torch.tensor([0.1, 0.2, -0.1])
    poses.requires_grad_(True)
    vv = pu.calc_vos(poses)
    vv.sum().backward()
    out["vos_degen_in"] = poses.detach().numpy()
    out["vos_degen_out"] = vv.detach().numpy()
    out["vos_degen_grad"] = poses.grad.numpy()
    np.savez_compressed(os.path.join(GOLD, "pose_math.npz"), **out)
    print("golden pose_math: %d arrays" % len(out), flush=True)


def run_pgo(seed=7):
    """Known-answer vectors of the reference's pose-graph optimisation (common/pose_utils.py:458-804), made by running
    its own PoseGraph / PoseGraphFC classes from source (oracle.pgo_oracle.load_reference): windows of predicted poses,
    VOs and covariances in -> optimised poses out.  Includes the covariances scripts/eval.py derives from a trained
    criterion (exp of the learned log-variances) and a degenerate window (all poses equal)."""
    from . import pgo_oracle as P
    ns = P.load_reference()
    rng = np.random.default_rng(seed)

    def rand_poses(n):
        t = rng.normal(size=(n, 3)).cumsum(0) * 0.3
        v = rng.normal(size=(n, 3)) * 0.4
        q = np.stack([np.concatenate(([np.cos(np.linalg.norm(a))], np.sinc(np.linalg.norm(a) / np.pi) * a)) for a in v])
        return np.hstack((t, q))

    out = {}
    cases = [(3, False, 8, (1.0, 1.0, 1.0, 1.0)), (5, False, 6, (1.0, 0.05, 1.0, 0.05)), (7, False, 5, (2.0, 0.5, 0.5, 0.2)),
             (4, True, 5, (1.0, 1.0, 1.0, 1.0)), (6, True, 4, (1.0, 0.05, 1.0, 0.05)), (16, False, 2, (1.0, 1.0, 1.0, 1.0))]
    for ci, (n, fc, w, sig) in enumerate(cases):
        P_in, V_in, ref = [], [], []
        for k in range(w):
            gt = rand_poses(n)
            if ci == 0 and k == 0:
                gt = np.tile(gt[:1], (n, 1))                    # degenerate: identical poses
            pred = gt + rng.normal(size=gt.shape) * 0.05
            E = P.edges(n, fc)
            vos = np.zeros((len(E), 7))
            for e, (i, j) in enumerate(E):
                vos[e, :3] = P.rotate_vector(gt[j, :3] - gt[i, :3], P.qinverse(gt[i, 3:]))
                vos[e, 3:] = P.qmult(P.qinverse(gt[i, 3:]), gt[j, 3:])
            vos += rng.normal(size=vos.shape) * 0.01
            r = ns["optimize_poses"](pred_poses=pred.copy(), vos=vos.copy(), fc_vos=fc, sax=sig[0], saq=sig[1], srx=sig[2], srq=sig[3])
            P_in.append(pred); V_in.append(vos); ref.append(r)
        out["case%d_cfg" % ci] = np.array([n, int(fc), w] + list(sig), dtype=np.float64)
        out["case%d_poses" % ci] = np.stack(P_in); out["case%d_vos" % ci] = np.stack(V_in); out["case%d_out" % ci] = np.stack(ref)
    # optimize_poses with target_poses instead of VOs (:793-799)
    gt = rand_poses(5); pred = gt + rng.normal(size=gt.shape) * 0.05
    out["targ_pred"] = pred; out["targ_gt"] = gt
    out["targ_out"] = ns["optimize_poses"](pred_poses=pred.copy(), target_poses=gt.copy(), sax=1.0, saq=1.0, srx=0.1, srq=0.1)
    # eval.py:163-167 qexp of predicted log-quaternions (numpy float32 arithmetic) and the angular error metric
    lq = (rng.normal(size=(64, 3)) * 0.8).astype(np.float32); lq[0] = 0
    out["qexp_in"] = lq
    out["qexp_out"] = np.asarray([ns["qexp"](p) for p in lq])
    qa, qb = rand_poses(32)[:, 3:], rand_poses(32)[:, 3:]
    out["qerr_a"] = qa; out["qerr_b"] = qb
    out["qerr_deg"] = np.asarray([ns["quaternion_angular_error"](a, b) for a, b in zip(qa, qb)])
    np.savez_compressed(os.path.join(GOLD, "pgo.npz"), **out)
    print("golden pgo: %d arrays" % len(out), flush=True)


def run_keys():
    """The reference module's state_dict / named_parameters key order (drop-in
    contract for common/train.py:22-53,198-204)."""
    import torchvision
    ns = ref_loader.load()
    net = ns.PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False)
    mp = ns.MapNet(mapnet=net)
    np.savez_compressed(
        os.path.join(GOLD, "keys.npz"),
        posenet_state_keys=np.array(list(net.state_dict().keys())),
        posenet_param_names=np.array([n for n, _ in net.named_parameters()]),
        posenet_param_shapes=np.array([repr(tuple(p.shape)) for _, p in net.named_parameters()]),
        mapnet_state_keys=np.array(list(mp.state_dict().keys())),
        n_params=np.int64(sum(p.numel() for p in net.parameters())))
    print("golden keys: %d state entries" % len(net.state_dict()), flush=True)


LIVE_SAMPLE = 256       # entries per gradient tensor kept by run_live (fixed stride)
INIT_SAMPLE = 64        # entries per initial state tensor kept by run_live (fixed stride)


def _grad_samples(prefix, grads, out):
    names = [k.replace("mapnet.", "", 1) for k in grads]
    out[prefix + "grad_names"] = np.array(names)
    out[prefix + "grad_norm"] = np.array([float(v.double().norm()) for v in grads.values()])
    out[prefix + "grad_stride"] = np.array([max(1, v.numel() // LIVE_SAMPLE) for v in grads.values()], dtype=np.int64)
    for i, v in enumerate(grads.values()):
        out[prefix + "grad_%d" % i] = v.detach().flatten()[::max(1, v.numel() // LIVE_SAMPLE)].numpy().copy()


def run_live():
    """tests/golden/live_reference.npz: what the tests that once executed the reference live compared against --
    training steps of the reference modules, its NaN-filter hook, the one-frame plumbing config, the PoseGraph
    classes and numpy helpers, MF.get_indices, the reference PoseNet's seeded initialisation, and the reference
    module's state_dict / criterion layout."""
    import torchvision
    from . import pgo_oracle as P
    ns = ref_loader.load()
    out = {}
    for kind, cfg in (("posenet", dict(kind="posenet", N=2, H=64, W=64)),
                      ("online", dict(kind="online", N=2, T=4, H=64, W=64))):
        st = weights.make_state(3)
        x, targ = weights.make_inputs(cfg, 3)
        model = ref_loader.build_reference_model(st, "posenet" if kind == "posenet" else "mapnet")
        model.train()
        if kind == "posenet":
            crit = ns.PoseNetCriterion(sax=0.0, saq=-3.0, learn_beta=True)
        else:
            crit = ns.MapNetOnlineCriterion(sax=0.0, saq=-3.0, srx=0.0, srq=-3.0, learn_beta=True, learn_gamma=True)
        loss, o, grads, _ = ref_loader.reference_step(model, crit, x, targ)
        out["step_%s_loss" % kind] = np.float64(loss)
        out["step_%s_out" % kind] = o.numpy()
        _grad_samples("step_%s_" % kind, grads, out)
    # NaN filter hook (degenerate fc_wpqr = 0)
    st = weights.make_state(3)
    st["fc_wpqr.weight"] = torch.zeros_like(st["fc_wpqr.weight"])
    st["fc_wpqr.bias"] = torch.zeros_like(st["fc_wpqr.bias"])
    cfg = dict(kind="online", N=2, T=4, H=64, W=64)
    x, targ = weights.make_inputs(cfg, 3)
    model = ref_loader.build_reference_model(st, "mapnet", filter_nans=True)
    model.train()
    crit = ns.MapNetOnlineCriterion(sax=0.0, saq=-3.0, srx=0.0, srq=-3.0, learn_beta=True, learn_gamma=True)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, _, grads, _ = ref_loader.reference_step(model, crit, x, targ, do_step=False)
    _grad_samples("nanfilter_", grads, out)
    out["nanfilter_all_finite"] = np.array([bool(torch.isfinite(v).all()) for v in grads.values()])
    out["nanfilter_fc_wpqr_weight"] = grads["mapnet.fc_wpqr.weight"].numpy()
    # BASELINE configs[0]: one 256x256 frame
    st = weights.make_state(7)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(1, 3, 256, 256, generator=g)
    targ = torch.randn(1, 6, generator=g)
    model = ref_loader.build_reference_model(st, "posenet")
    model.train()
    loss, o, _, _ = ref_loader.reference_step(model, ns.PoseNetCriterion(sax=0.0, saq=-3.0, learn_beta=True), x, targ,
                                              do_step=False)
    out["config0_loss"] = np.float64(loss)
    out["config0_out"] = o.numpy()
    # PoseGraph classes and numpy helpers (common/pose_utils.py:306-804)
    pns = P.load_reference()
    rng = np.random.default_rng(11)
    for ci, (N, fc) in enumerate([(3, False), (6, False), (5, True)]):
        t = rng.normal(size=(N, 3)).cumsum(0) * 0.3
        v = rng.normal(size=(N, 3)) * 0.4
        q = np.stack([np.concatenate(([np.cos(np.linalg.norm(a))], np.sinc(np.linalg.norm(a) / np.pi) * a)) for a in v])
        gt = np.hstack((t, q))
        pred = gt + rng.normal(size=gt.shape) * 0.05
        E = P.edges(N, fc)
        vos = np.stack([np.concatenate((P.rotate_vector(gt[j, :3] - gt[i, :3], P.qinverse(gt[i, 3:])),
                                        P.qmult(P.qinverse(gt[i, 3:]), gt[j, 3:]))) for i, j in E])
        out["pgo%d_pred" % ci], out["pgo%d_vos" % ci], out["pgo%d_fc" % ci] = pred, vos, np.bool_(fc)
        out["pgo%d_out" % ci] = pns["optimize_poses"](pred_poses=pred.copy(), vos=vos.copy(), fc_vos=fc, sax=1.5, saq=0.3,
                                                     srx=0.7, srq=0.1)
    for name in ("dpq_q", "dpsq_q", "dpsq_p", "dqstq_t", "m_rot"):
        xx = rng.normal(size=(4, 1))
        out["pgohelper_%s_in" % name], out["pgohelper_%s_out" % name] = xx, pns[name](xx)
    # MF.get_indices (dataset_loaders/composite.py:60-75) on the cases tests/test_preprocess_host.py walks
    get_indices = _reference_mf_get_indices()
    from types import SimpleNamespace
    rows = []
    for steps, skip, L in [(3, 10, 1000), (5, 10, 47), (2, 1, 5), (4, 3, 30), (3, 10, 12)]:
        for nodup in (False, True):
            me = SimpleNamespace(variable_skip=False, skip=skip, steps=steps, no_duplicates=nodup, dset=range(L))
            n = (L - (steps - 1) * skip) if nodup else L
            for index in list(range(0, min(n, 40))) + [max(n - 1, 0)]:
                rows.append([steps, skip, L, int(nodup), index] + list(get_indices(me, index)) + [-1] * (5 - steps))
    out["mf_cases"] = np.array(rows, dtype=np.int64)
    me = SimpleNamespace(variable_skip=True, skip=7, steps=5, no_duplicates=False, dset=range(500))
    np.random.seed(3)
    out["mf_variable_skip"] = np.asarray(get_indices(me, 250), dtype=np.int64)
    # initialisation: the reference PoseNet's state_dict right after torch.manual_seed(11), without and with pretrained
    # (models/posenet.py:50-66): per-tensor sums and a fixed-stride sample of the exact values
    for pretrained in (False, True):
        torch.manual_seed(11)
        r = ns.PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=pretrained)
        sd = r.state_dict()
        tag = "init_pre%d_" % int(pretrained)
        out[tag + "keys"] = np.array(list(sd.keys()))
        out[tag + "sum"] = np.array([float(v.double().sum()) for v in sd.values()])
        out[tag + "stride"] = np.array([max(1, v.numel() // INIT_SAMPLE) for v in sd.values()], dtype=np.int64)
        for i, v in enumerate(sd.values()):
            out[tag + "%d" % i] = v.flatten()[::max(1, v.numel() // INIT_SAMPLE)].numpy().copy()
    # state_dict layout of the reference MapNet and its criterion (strict load_state_dict checks names and shapes)
    net = ns.PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False)
    mp = ns.MapNet(mapnet=net)
    out["mapnet_state_keys"] = np.array(list(mp.state_dict().keys()))
    out["mapnet_state_shapes"] = np.array([repr(tuple(v.shape)) for v in mp.state_dict().values()])
    rc = ns.MapNetCriterion(sax=1.0, saq=1.0, srx=1.0, srq=1.0, learn_beta=True, learn_gamma=True)
    out["mapnet_criterion_state_keys"] = np.array(list(rc.state_dict().keys()))
    np.savez_compressed(os.path.join(GOLD, "live_reference.npz"), **out)
    print("golden live_reference: %d arrays" % len(out), flush=True)


def _reference_mf_get_indices():
    """MF.get_indices executed from the reference's own source text with the Python-2 integer divisions spelled `//`
    (the module itself imports py2-only dataset code)."""
    path = os.path.join(ref_loader.REF_ROOT, "dataset_loaders", "composite.py")
    src = open(path).read().split("\n")
    start = next(i for i, l in enumerate(src) if l.strip().startswith("def get_indices"))
    end = next(i for i in range(start + 1, len(src)) if src[i].strip().startswith("def "))
    body = "\n".join(l[2:] for l in src[start:end])
    body = body.replace("len(offsets) / 2", "len(offsets) // 2").replace("self.steps/2", "self.steps//2").replace("np.int)", "int)")
    ns = {"np": np}
    exec(body, ns)
    return ns["get_indices"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true", help="also the BASELINE full-size configs (minutes)")
    ap.add_argument("--only", default=None)
    ap.add_argument("--emulated", action="store_true", help="only the oracle-with-product-rounding fixtures (emu_*.npz)")
    a = ap.parse_args()
    if not ref_loader.available():
        sys.exit("reference tree not available; goldens can only be regenerated in the build container")
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    if a.emulated:
        for emulate, name in EMU_CONFIGS:
            run_emulated(emulate, name)
        return
    if a.only == "pgo":
        run_pgo()
        return
    if a.only == "live":
        run_live()
        return
    if a.only is None:
        run_keys()
        run_pose_math()
        run_pgo()
    cfgs = dict(STEP_CONFIGS)
    if a.full:
        cfgs.update(FULL_CONFIGS)
    for name, cfg in cfgs.items():
        if a.only and a.only != name:
            continue
        run_step_config(name, cfg)


if __name__ == "__main__":
    main()
