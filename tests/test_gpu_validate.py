"""GPU run of inference.validate (the trainer's validation pass over a DeviceLoader) and graph.train_val: batch losses
bit for bit those of calling the criterion batch by batch on the same DeviceLoader batches, each distinct frame through
the engine once when nothing is random, dropout and ColorJitter in the reference's per-batch order, live models,
a float64 restatement, and train_val's schedule, checkpoints and resume."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

L_SEQ, H_IN, W_IN, STEPS, SKIP, BS = 23, 120, 160, 3, 2, 4      # 6 batches: 4, 4, 4, 4, 4, 3
STATS = (np.array([0.45, 0.5, 0.55]), np.array([0.22, 0.25, 0.2]))


def _seq(L, seed):
    rng = np.random.default_rng(seed)
    fr = (rng.random((L, H_IN, W_IN, 3)) * 256).astype(np.uint8)
    t = rng.standard_normal((L, 3)).cumsum(0) * 0.2
    v = rng.standard_normal((L, 3))
    v = v / np.linalg.norm(v, axis=1, keepdims=True) * (rng.random((L, 1)) - 0.5) * math.pi
    return fr, np.concatenate([t, v], 1).astype(np.float32)


def _dataset(kind, cj=0.0, seed=1, L=L_SEQ):
    from geomapnet_b200.data import DeviceDataset
    fr, poses = _seq(L, seed)
    return DeviceDataset(fr, STATS[0], STATS[1], poses=poses, steps=None if kind == "posenet" else STEPS, skip=SKIP,
                         variable_skip=kind != "posenet", color_jitter=cj, size=96, max_batch=BS, chunk=16)


def _model(kind, precision, droprate=0.0):
    from oracle import weights
    from helpers import make_product_model
    st = weights.make_state(7)
    model, _ = make_product_model(st, kind, precision, droprate=droprate)
    return model, st


def _crit(kind):
    from helpers import make_product_criterion
    return make_product_criterion(kind, learn=False)


def _seed(s=5):
    torch.manual_seed(s)
    np.random.seed(s)


def _loop(fn, loader, crit):
    """the reference's val loop restated: one criterion call and one .item() per DeviceLoader batch"""
    with torch.no_grad():
        return [float(crit(fn(x), t)) for x, t in loader]


def _count_frames(ds):
    seen = []
    orig = ds.assemble_frames

    def counting(frames, x_out):
        seen.append(len(frames))
        return orig(frames, x_out)
    ds.assemble_frames = counting
    return seen


@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
@pytest.mark.parametrize("kind", ["posenet", "mapnet"])
def test_losses_equal_per_batch_criterion(kind, precision):
    """droprate 0, no ColorJitter: each distinct frame of the pass through the engine once.  The losses are bit for bit
    the criterion's on every batch gathered from those per-frame predictions, and the criterion's on the Predictor
    called batch by batch on the DeviceLoader's batches (the reference's loop); their mean is AverageMeter's."""
    from geomapnet_b200.data import DeviceLoader
    from geomapnet_b200.inference import Predictor, validate
    model, _ = _model(kind, precision)
    ds = _dataset(kind)
    crit = _crit(kind)
    loader = DeviceLoader(ds, BS, shuffle=True)
    pr = Predictor(model, max_batch=16)
    seen = _count_frames(ds)
    _seed()
    avg, losses = validate(pr, loader, crit)
    state = torch.get_rng_state(), np.random.get_state()[2]
    _seed()
    tab = ds.val_tables(BS, True, True)
    assert torch.equal(torch.get_rng_state(), state[0]) and np.random.get_state()[2] == state[1]
    frames = tab["frames"]
    assert sum(seen) == len(frames) <= L_SEQ               # each distinct frame of the pass through the engine once
    B = min(16, ds.max_batch * ds.frames_per_item)         # validate's chunks of distinct frames
    x = torch.empty(len(frames), 3, ds.Ho, ds.Wo, device="cuda")
    for lo in range(0, len(frames), B):
        ds.assemble_frames(frames[lo:lo + B], x[lo:lo + B])
    pred6 = torch.cat([pr(x[lo:lo + B]) for lo in range(0, len(frames), B)])
    items = tab["batch_items"]
    exp = []
    for b in range(len(items) - 1):
        rows = torch.as_tensor(tab["pred_rows"][items[b]:items[b + 1]], dtype=torch.long, device="cuda")
        t = ds.poses[torch.as_tensor(tab["targ_rows"][items[b]:items[b + 1]], dtype=torch.long, device="cuda")]
        p = pred6[rows]
        if kind == "posenet":
            p, t = p[:, 0], t[:, 0]
        exp.append(float(crit(p, t)))
    assert len(losses) == len(exp) == 6 and all(type(v) is float for v in losses)
    assert losses == exp, (losses, exp)
    s = 0.0
    for v in exp:                                  # AverageMeter: sum += val * 1; avg = sum / count
        s += v * 1
    assert avg == s / len(exp)
    _seed()
    ref = _loop(pr, loader, crit)
    assert losses == ref, (losses, ref)
    pr.close(); ds.close()


def test_dropout_and_jitter_follow_the_per_batch_loop():
    """droprate 0.5 and ColorJitter 0.7: every batch assembled with its jitter draws and run on its own; two passes
    equal two per-batch loops of a fresh Predictor with the same seed (the engine's dropout counter included)"""
    from geomapnet_b200.data import DeviceLoader
    from geomapnet_b200.inference import Predictor, validate
    model, _ = _model("mapnet", "tc_split", droprate=0.5)
    ds = _dataset("mapnet", cj=0.7)
    crit = _crit("mapnet")
    loader = DeviceLoader(ds, BS, shuffle=True)
    pr = Predictor(model)
    seen = _count_frames(ds)
    _seed(9)
    got = [validate(pr, loader, crit) for _ in range(2)]
    assert seen == []                              # no frame-list assembly: whole jittered batches
    fresh = Predictor(model)
    _seed(9)
    ref = [_loop(fresh, loader, crit) for _ in range(2)]
    assert [g[1] for g in got] == ref, (got, ref)
    assert got[0][1] != got[1][1]                  # the masks moved on
    pr.close(); fresh.close(); ds.close()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_live_model(precision):
    """a live bf16 model gives the Predictor's result; an fp32 one its own eval forward, batch by batch (bitwise with
    jitter, where each batch runs on its own; within 1e-5 relative when each distinct frame runs once)"""
    from geomapnet_b200.data import DeviceLoader
    from geomapnet_b200.inference import Predictor, validate
    crit = _crit("mapnet")
    for cj in (0.0, 0.7):
        model, _ = _model("mapnet", precision)
        ds = _dataset("mapnet", cj=cj)
        loader = DeviceLoader(ds, BS, shuffle=True)
        _seed(3)
        avg, got = validate(model, loader, crit)
        assert model.training                                  # the mode is restored
        _seed(3)
        if precision == "bf16":
            pr = Predictor(model)
            assert validate(pr, loader, crit) == (avg, got)
            pr.close()
        else:
            model.eval()
            ref = _loop(model, loader, crit)
            model.train()
            if cj:
                assert got == ref
            else:
                assert max(abs(a - b) / abs(b) for a, b in zip(got, ref)) <= 1e-5, (got, ref)
        ds.close()


def _f64_loss(p, t, s):
    """MapNetCriterion.forward (common/criterion.py:76-109) in float64: pred, targ [N,T,6]"""
    def l1(a, b):
        return (a - b).abs().mean()
    vp, vt = p[:, 1:] - p[:, :-1], t[:, 1:] - t[:, :-1]                 # calc_vos_simple
    return (math.exp(-s["sax"]) * l1(p[..., :3], t[..., :3]) + s["sax"] + math.exp(-s["saq"]) * l1(p[..., 3:], t[..., 3:])
            + s["saq"] + math.exp(-s["srx"]) * l1(vp[..., :3], vt[..., :3]) + s["srx"]
            + math.exp(-s["srq"]) * l1(vp[..., 3:], vt[..., 3:]) + s["srq"])


def test_tc_split_matches_float64_restatement():
    from oracle import mapnet_oracle as O
    from geomapnet_b200.common.criterion import MapNetCriterion
    from geomapnet_b200.data import DeviceLoader
    from geomapnet_b200.inference import Predictor, validate
    model, st = _model("mapnet", "tc_split")
    ds = _dataset("mapnet")
    crit = MapNetCriterion().cuda()                # scripts/train.py's val_criterion: all four sigma 0
    loader = DeviceLoader(ds, BS, shuffle=True)
    pr = Predictor(model, max_batch=16)
    _seed(4)
    avg, got = validate(pr, loader, crit)
    _seed(4)
    stc = {k: (v.double() if v.is_floating_point() else v).cuda() for k, v in st.items()}
    ref = []
    with torch.no_grad():
        for x, t in loader:
            ref.append(float(_f64_loss(O.mapnet_forward(stc, x.double(), training=False), t.double(),
                                       dict(sax=0.0, saq=0.0, srx=0.0, srq=0.0))))
    ratio = max(abs(a - b) / abs(b) for a, b in zip(got, ref))
    print("tc_split validate vs float64 oracle: max relative loss error %.2e" % ratio)
    assert ratio <= 2e-4          # measured 1.3e-4 on an H100: the engine's strict-mode forward, not the loss
    assert abs(avg - sum(ref) / len(ref)) <= 2e-4 * abs(sum(ref) / len(ref))
    pr.close(); ds.close()


def _train_setup(st):
    from helpers import make_product_model
    from geomapnet_b200.common.optimizer import Optimizer
    model, _ = make_product_model(st, "mapnet", "bf16")
    crit = _crit("mapnet")
    opt = Optimizer([{"params": model.parameters()}], "adam", 1e-4, 5e-4)
    return model, crit, opt


def test_train_val_schedule_checkpoints_and_resume(tmp_path):
    """3 epochs, val_freq 2, snapshot 2: validates at epochs 0 and 2, writes epoch_000, epoch_002 and epoch_003, equals
    validate / train_epoch called by hand from the same seeds, and a resume from epoch_002 reproduces epoch 2 on"""
    from oracle import weights
    from geomapnet_b200.common.checkpoint import checkpoint_filename, load_checkpoint
    from geomapnet_b200.common.criterion import MapNetCriterion
    from geomapnet_b200.data import DeviceLoader
    from geomapnet_b200.graph import train_epoch, train_val
    from geomapnet_b200.inference import Predictor, validate
    st = weights.make_state(7)
    tr_ds, va_ds = _dataset("mapnet", cj=0.7, seed=2, L=19), _dataset("mapnet", seed=3, L=13)
    tr, va = DeviceLoader(tr_ds, BS, shuffle=True), DeviceLoader(va_ds, BS, shuffle=True)
    run = str(tmp_path / "run")
    os.makedirs(run)
    model, crit, opt = _train_setup(st)
    _seed(11)
    out = train_val(model, tr, va, crit, MapNetCriterion(), opt, 3, 2, 2, run, max_grad_norm=5.0)
    assert sorted(out["val"]) == [0, 2] and sorted(out["train"]) == [0, 1, 2]
    assert sorted(os.listdir(run)) == ["epoch_000.pth.tar", "epoch_002.pth.tar", "epoch_003.pth.tar"]
    final = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    # by hand
    model2, crit2, opt2 = _train_setup(st)
    pr, steps, val, train = Predictor(model2), {}, {}, {}
    _seed(11)
    for epoch in range(3):
        if epoch == 2:
            rng2 = torch.get_rng_state(), np.random.get_state()
        if epoch % 2 == 0:
            pr.refresh()
            val[epoch] = validate(pr, va, MapNetCriterion())[0]
        opt2.adjust_lr(epoch)
        model2.train()
        train[epoch] = train_epoch(tr, model2, crit2, opt2, max_grad_norm=5.0, steps=steps)
    pr.close()
    assert out["val"] == val and out["train"] == train, (out, val, train)
    # resume from epoch_002 with the RNG streams of epoch 2
    model3, crit3, opt3 = _train_setup(st)
    start = load_checkpoint(checkpoint_filename(run, 2), model3, opt3, crit3, resume_optim=True)
    assert start == 2
    torch.set_rng_state(rng2[0])
    np.random.set_state(rng2[1])
    res = str(tmp_path / "resume")
    os.makedirs(res)
    again = train_val(model3, tr, va, crit3, MapNetCriterion(), opt3, 3, 2, 2, res, max_grad_norm=5.0, start_epoch=start)
    assert again["val"] == {2: out["val"][2]} and again["train"] == {2: out["train"][2]}
    assert sorted(os.listdir(res)) == ["epoch_002.pth.tar", "epoch_003.pth.tar"]
    for k, v in model3.state_dict().items():
        assert torch.equal(v.detach().cpu(), final[k]), k
    tr_ds.close(); va_ds.close()
