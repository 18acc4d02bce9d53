"""CPU restatement of the reference MapNet training hot path -- TEST INFRASTRUCTURE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference leg may import this (see oracle/__init__.py).  The product
(geomapnet_b200/) never does; it fails loudly when its CUDA library is missing.

Each function cites the reference file:line (relative to /root/reference) it
restates.  The third-party arithmetic the reference calls (torchvision
resnet34 graph, torch conv/BN/linear/Adam -- SURVEY.md section 8c) is expressed with
torch.nn.functional on plain tensors; there is no nn.Module, no torchvision
import and no dependence on /root/reference at run time, so it travels to the
GPU box.  Pinned against the reference itself by tests/test_oracle_pinning.py
(build container) and tests/golden/*.npz (everywhere).

Floating point: fp32 by default (what the reference computes in); pass float64
tensors for a higher-precision arbiter.  ``emulate="bf16"`` reproduces the
rounding points of the product's bf16 tensor-core path (operands of every conv
rounded to bf16, stored activations AND stored gradients rounded to bf16, fp32
accumulation/BN math); ``emulate="f16x2"`` those of the strict tensor-core mode
(conv operands = fp16 hi + lo planes, 22 significant bits; everything else fp32).
"""
import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

from .weights import STAGES

# --------------------------------------------------------------------------
# L1 pose math -- common/pose_utils.py:21-260 (torch section)
# --------------------------------------------------------------------------


def vdot(v1, v2):
    """common/pose_utils.py:21-30"""
    return (v1 * v2).sum(1)


def normalize(x, dim=1):
    """common/pose_utils.py:32-42 (p=2)"""
    return x / x.norm(p=2, dim=dim).unsqueeze(dim)


def qmult(q1, q2):
    """common/pose_utils.py:44-62 -- Hamilton product followed by normalize."""
    q1s, q1v = q1[:, :1], q1[:, 1:]
    q2s, q2v = q2[:, :1], q2[:, 1:]
    qs = q1s * q2s - vdot(q1v, q2v).unsqueeze(1)   # ref: [N,1]*[N,1] - [N] with N==1 per call
    qv = q1v * q2s + q2v * q1s + torch.cross(q1v, q2v, dim=1)
    return normalize(torch.cat((qs, qv), dim=1), dim=1)


def qinv(q):
    """common/pose_utils.py:64-71"""
    return torch.cat((q[:, :1], -q[:, 1:]), dim=1)


def qexp_t(q):
    """common/pose_utils.py:73-84"""
    n = torch.norm(q, p=2, dim=1, keepdim=True)
    n = torch.clamp(n, min=1e-8)
    q = q * torch.sin(n)
    q = q / n
    return torch.cat((torch.cos(n), q), dim=1)


def qlog_t(q):
    """common/pose_utils.py:86-96"""
    n = torch.norm(q[:, 1:], p=2, dim=1, keepdim=True)
    n = torch.clamp(n, min=1e-8)
    q = q[:, 1:] * torch.acos(torch.clamp(q[:, :1], min=-1.0, max=1.0))
    return q / n


def rotate_vec_by_q(t, q):
    """common/pose_utils.py:120-132: t + 2 qs (qv x t) + 2 qv x (qv x t)"""
    qs, qv = q[:, :1], q[:, 1:]
    b = torch.cross(qv, t, dim=1)
    c = 2 * torch.cross(qv, b, dim=1)
    b = 2 * b * qs
    return t + b + c


def compose_pose_quaternion(p1, p2):
    """common/pose_utils.py:134-146"""
    p1t, p1q = p1[:, :3], p1[:, 3:]
    p2t, p2q = p2[:, :3], p2[:, 3:]
    q = qmult(p1q, p2q)
    t = p1t + rotate_vec_by_q(p2t, p1q)
    return torch.cat((t, q), dim=1)


def invert_pose_quaternion(p):
    """common/pose_utils.py:148-157"""
    t, q = p[:, :3], p[:, 3:]
    q_inv = qinv(q)
    tinv = -rotate_vec_by_q(t, q_inv)
    return torch.cat((tinv, q_inv), dim=1)


def calc_vo(p0, p1):
    """common/pose_utils.py:159-165"""
    return compose_pose_quaternion(invert_pose_quaternion(p0), p1)


def calc_vo_logq(p0, p1):
    """common/pose_utils.py:167-179"""
    q0 = qexp_t(p0[:, 3:])
    q1 = qexp_t(p1[:, 3:])
    vos = calc_vo(torch.cat((p0[:, :3], q0), dim=1), torch.cat((p1[:, :3], q1), dim=1))
    vos_q = qlog_t(vos[:, 3:])
    return torch.cat((vos[:, :3], vos_q), dim=1)


def calc_vos_simple(poses):
    """common/pose_utils.py:234-246 -- plain subtraction of consecutive 6-vectors
    (the reference's Python double loop, vectorised; same arithmetic per element)."""
    return poses[:, 1:] - poses[:, :-1]


def calc_vos(poses):
    """common/pose_utils.py:248-260 -- calc_vo_logq on every consecutive pair
    (the reference loops over n and i; all pairs are independent, so they are
    batched here -- elementwise arithmetic per pair is unchanged)."""
    N, T = poses.shape[0], poses.shape[1]
    p0 = poses[:, :-1].reshape(-1, 6)
    p1 = poses[:, 1:].reshape(-1, 6)
    return calc_vo_logq(p0, p1).view(N, T - 1, 6)


# --------------------------------------------------------------------------
# L3 criteria -- common/criterion.py
# --------------------------------------------------------------------------


def _l1(a, b):
    """nn.L1Loss(): mean over all elements (criterion.py:34 default t/q_loss_fn)."""
    return (a - b).abs().mean()


def posenet_criterion(pred, targ, sax, saq):
    """common/criterion.py:42-52.  sax/saq: 1-element tensors."""
    return torch.exp(-sax) * _l1(pred[:, :3], targ[:, :3]) + sax + \
        torch.exp(-saq) * _l1(pred[:, 3:], targ[:, 3:]) + saq


def mapnet_criterion(pred, targ, sax, saq, srx, srq):
    """common/criterion.py:76-109"""
    p, t = pred.reshape(-1, 6), targ.reshape(-1, 6)
    abs_loss = torch.exp(-sax) * _l1(p[:, :3], t[:, :3]) + sax + \
        torch.exp(-saq) * _l1(p[:, 3:], t[:, 3:]) + saq
    pv = calc_vos_simple(pred).reshape(-1, 6)
    tv = calc_vos_simple(targ).reshape(-1, 6)
    vo_loss = torch.exp(-srx) * _l1(pv[:, :3], tv[:, :3]) + srx + \
        torch.exp(-srq) * _l1(pv[:, 3:], tv[:, 3:]) + srq
    return abs_loss + vo_loss


def mapnet_online_criterion(pred, targ, sax, saq, srx, srq, gps_mode=False):
    """common/criterion.py:137-184 (T = s[1] / 2 at :150 is py2 integer division)."""
    T = pred.shape[1] // 2
    pred_abs = pred[:, :T].reshape(-1, 6)
    pred_vos = pred[:, T:]
    targ_abs = targ[:, :T].reshape(-1, 6)
    targ_vos = targ[:, T:].reshape(-1, 6)
    abs_loss = torch.exp(-sax) * _l1(pred_abs[:, :3], targ_abs[:, :3]) + sax + \
        torch.exp(-saq) * _l1(pred_abs[:, 3:], targ_abs[:, 3:]) + saq
    if not gps_mode:
        pred_vos = calc_vos(pred_vos)                      # :166-167
    pred_vos = pred_vos.reshape(-1, 6)
    idx = 2 if gps_mode else 3                             # :173
    vo_loss = torch.exp(-srx) * _l1(pred_vos[:, :idx], targ_vos[:, :idx]) + srx
    if not gps_mode:
        vo_loss = vo_loss + torch.exp(-srq) * _l1(pred_vos[:, 3:], targ_vos[:, 3:]) + srq
    return abs_loss + vo_loss


def criterion(kind, pred, targ, s):
    """Dispatch.  s = dict(sax, saq[, srx, srq]) of 1-element tensors."""
    if kind == "posenet":
        return posenet_criterion(pred, targ, s["sax"], s["saq"])
    if kind == "mapnet":
        return mapnet_criterion(pred, targ, s["sax"], s["saq"], s["srx"], s["srq"])
    if kind in ("online", "online_gps"):
        return mapnet_online_criterion(pred, targ, s["sax"], s["saq"], s["srx"], s["srq"],
                                       gps_mode=(kind == "online_gps"))
    raise ValueError(kind)


# --------------------------------------------------------------------------
# L2/L0 model -- models/posenet.py:65-73, :93-97 around torchvision resnet34
# --------------------------------------------------------------------------

BN_EPS = 1e-5       # torch.nn.BatchNorm2d default, used by torchvision resnet
BN_MOMENTUM = 0.1


def _round_bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def _round_f16x2(t):
    """hi + lo with hi = fp16(t), lo = fp16(t - hi): the 22 significant bits the strict tensor-core mode's operand
    planes carry (geomapnet_b200/csrc/common.cuh: hsplit; saturating at the fp16 range)."""
    c = t.clamp(-65504.0, 65504.0)
    hi = c.to(torch.float16).to(t.dtype)
    return hi + (c - hi).to(torch.float16).to(t.dtype)


class _RoundBoth(torch.autograd.Function):
    """A tensor the product STORES in a narrow format: rounded on the way forward, and the gradient that flows back
    through this point (the product stores that one too) rounded the same way."""

    @staticmethod
    def forward(ctx, t, fn):
        ctx.fn = fn
        return fn(t)

    @staticmethod
    def backward(ctx, g):
        return ctx.fn(g), None


class _RoundFwd(torch.autograd.Function):
    """An operand copy (packed weights): rounded forward, gradient untouched (wgrad accumulates in fp32)."""

    @staticmethod
    def forward(ctx, t, fn):
        return fn(t)

    @staticmethod
    def backward(ctx, g):
        return g, None


def _rb(t, emulate):
    """storage rounding point of an activation / conv output (and of the gradient w.r.t. it)"""
    if emulate == "bf16":
        return _RoundBoth.apply(t, _round_bf16)
    return t


def _conv(x, w, stride, pad, emulate):
    if emulate == "f16x2":
        # strict tensor-core mode (precision tc_split): conv operands -- activations, weights and, in the backward
        # pass, the gradient w.r.t. the conv output -- carry 22 significant bits; all four hi/lo products are
        # formed and accumulated in fp32; conv outputs and everything element-wise stay fp32.
        y = F.conv2d(_RoundFwd.apply(x, _round_f16x2), _RoundFwd.apply(w, _round_f16x2), None, stride, pad)
        return _GradRound.apply(y)
    # operands rounded to bf16 (x already is when it is a stored activation);
    # products exact in fp32, fp32 accumulate -- what wgmma does.
    y = F.conv2d(_rb(x, emulate), _RoundFwd.apply(w, _round_bf16) if emulate == "bf16" else w, None, stride, pad)
    return _rb(y, emulate)      # conv output is stored (bf16) before BN reads it


class _GradRound(torch.autograd.Function):
    """identity forward; the gradient w.r.t. a conv output is a backward conv OPERAND in the strict mode"""

    @staticmethod
    def forward(ctx, t):
        return t.view_as(t)

    @staticmethod
    def backward(ctx, g):
        return _round_f16x2(g)


def _bn(y, st, prefix, training, bufs_out):
    w, b = st[prefix + ".weight"], st[prefix + ".bias"]
    rm, rv = st[prefix + ".running_mean"], st[prefix + ".running_var"]
    if training:
        rm2, rv2 = rm.clone(), rv.clone()
        out = F.batch_norm(y, rm2, rv2, w, b, True, BN_MOMENTUM, BN_EPS)
        if bufs_out is not None:
            bufs_out[prefix + ".running_mean"] = rm2.detach()
            bufs_out[prefix + ".running_var"] = rv2.detach()
        return out
    return F.batch_norm(y, rm, rv, w, b, False, BN_MOMENTUM, BN_EPS)


def trunk_forward(st, x, training=True, emulate=None, bufs_out=None, taps=None):
    """torchvision ResNet.forward with BasicBlock [3,4,6,3] (3rd party; run at
    models/posenet.py:66), avgpool=AdaptiveAvgPool2d(1) (posenet.py:44), up to
    and including fc 512->feat_dim (posenet.py:45-46).
    x: [B,3,H,W].  Returns [B, feat_dim]."""
    fe = "feature_extractor."
    y = _conv(x, st[fe + "conv1.weight"], 2, 3, emulate)
    z = F.relu(_bn(y, st, fe + "bn1", training, bufs_out))
    z = F.max_pool2d(z, 3, 2, 1)
    z = _rb(z, emulate)
    if taps is not None:
        taps["stem"] = z
    inpl = 64
    for li, (planes, nblk, stride) in enumerate(STAGES, start=1):
        for b in range(nblk):
            p = "%slayer%d.%d." % (fe, li, b)
            s = stride if b == 0 else 1
            idt = z
            y1 = _conv(z, st[p + "conv1.weight"], s, 1, emulate)
            h = _rb(F.relu(_bn(y1, st, p + "bn1", training, bufs_out)), emulate)
            y2 = _conv(h, st[p + "conv2.weight"], 1, 1, emulate)
            o = _bn(y2, st, p + "bn2", training, bufs_out)
            if s != 1 or inpl != planes:
                yd = _conv(z, st[p + "downsample.0.weight"], s, 0, emulate)
                idt = _bn(yd, st, p + "downsample.1", training, bufs_out)
            z = _rb(F.relu(o + idt), emulate)
            inpl = planes
            if taps is not None:
                taps["layer%d.%d" % (li, b)] = z
    feat = z.mean(dim=(2, 3))                       # AdaptiveAvgPool2d(1) + flatten
    if taps is not None:
        taps["gap"] = feat
    return F.linear(feat, st[fe + "fc.weight"], st[fe + "fc.bias"])


class _LinearNanFiltered(torch.autograd.Function):
    """fc_wpqr with the backward hook of models/posenet.py:28-34,50-51: `filter_hook` clones every entry of the
    Linear's grad_input -- the gradients w.r.t. bias, input and weight -- and sets their NaN entries to zero.
    (Pinned against the reference module itself by tests/test_oracle_pinning.py with a NaN-producing gradient.)"""

    @staticmethod
    def forward(ctx, f, w, b):
        ctx.save_for_backward(f, w)
        return F.linear(f, w, b)

    @staticmethod
    def backward(ctx, g):
        f, w = ctx.saved_tensors
        gf, gw, gb = g @ w, g.t() @ f, g.sum(0)
        return tuple(torch.where(torch.isnan(t), torch.zeros_like(t), t) for t in (gf, gw, gb))


def posenet_forward(st, x, training=True, drop_mask=None, emulate=None, bufs_out=None,
                    taps=None, filter_nans=False):
    """models/posenet.py:65-73.  drop_mask: None (droprate 0, the :68 guard) or a
    [B,feat_dim] tensor already scaled by 1/(1-p) (injected dropout mask)."""
    f = trunk_forward(st, x, training, emulate, bufs_out, taps)
    f = F.relu(f)
    if drop_mask is not None:
        f = f * drop_mask
    xyz = F.linear(f, st["fc_xyz.weight"], st["fc_xyz.bias"])
    if filter_nans:
        wpqr = _LinearNanFiltered.apply(f, st["fc_wpqr.weight"], st["fc_wpqr.bias"])
    else:
        wpqr = F.linear(f, st["fc_wpqr.weight"], st["fc_wpqr.bias"])
    return torch.cat((xyz, wpqr), 1)


def mapnet_forward(st, x, **kw):
    """models/posenet.py:93-97: fold T into the batch (BN statistics span N*T)."""
    s = x.shape
    poses = posenet_forward(st, x.reshape(-1, *s[2:]), **kw)
    return poses.view(s[0], s[1], -1)


def model_forward(kind, st, x, **kw):
    if kind == "posenet":
        return posenet_forward(st, x, **kw)
    return mapnet_forward(st, x, **kw)


# --------------------------------------------------------------------------
# L4 step -- common/train.py:339-361 + common/optimizer.py:21-23
# --------------------------------------------------------------------------

TRAINABLE_KINDS = ("conv", "bn_w", "bn_b", "fc_w", "fc_b")


def split_state(st):
    params = OrderedDict((k, v) for k, v in st.items()
                         if not (k.endswith("running_mean") or k.endswith("running_var")
                                 or k.endswith("num_batches_tracked")))
    bufs = OrderedDict((k, v) for k, v in st.items() if k not in params)
    return params, bufs


def train_step(kind, st, x, targ, svals, learn=(True, True), lr=1e-4, weight_decay=5e-4,
               max_grad_norm=0.0, emulate=None, drop_mask=None, adam_state=None,
               do_step=True, filter_nans=False):
    """One step_feedfwd (common/train.py:339-361) on plain tensors.

    kind   posenet | mapnet | online | online_gps
    st     state dict (oracle.weights.make_state layout); NOT modified
    svals  dict sax/saq[/srx/srq] -> python floats
    learn  (learn_beta, learn_gamma) -> which scalars are trainable (scripts/train.py:104-110)
    Returns dict(loss, pred, grads{name}, sgrads{name}, new_state, new_svals, adam_state).
    """
    dt, dev = x.dtype, x.device
    params, bufs = split_state(st)
    P = OrderedDict((k, v.detach().to(dev, dt).clone().requires_grad_(True)) for k, v in params.items())
    full = OrderedDict(P)
    for k, v in bufs.items():
        full[k] = v.detach().to(dev) if v.dtype == torch.int64 else v.detach().to(dev, dt)
    S = OrderedDict()
    for name in (("sax", "saq") if kind == "posenet" else ("sax", "saq", "srx", "srq")):
        trainable = learn[0] if name in ("sax", "saq") else learn[1]
        S[name] = torch.tensor([svals[name]], dtype=dt, device=dev, requires_grad=trainable)

    bufs_out = {}
    mkind = "posenet" if kind == "posenet" else "mapnet"
    pred = model_forward(mkind, full, x, training=True, drop_mask=drop_mask, emulate=emulate,
                         bufs_out=bufs_out, filter_nans=filter_nans)
    loss = criterion(kind, pred, targ, S)
    loss.backward()
    grads = OrderedDict((k, v.grad.detach().clone()) for k, v in P.items())
    sgrads = OrderedDict((k, (v.grad.detach().clone() if v.grad is not None else None))
                         for k, v in S.items())
    out = dict(loss=loss.detach().clone(), pred=pred.detach().clone(), grads=grads, sgrads=sgrads)

    if do_step:
        plist = list(P.values())
        groups = [{"params": plist}]
        sl = [v for v in S.values() if v.requires_grad]
        if sl:
            groups.append({"params": sl})
        opt = torch.optim.Adam(groups, lr=lr, weight_decay=weight_decay)   # optimizer.py:21-23
        if adam_state is not None:
            opt.load_state_dict(adam_state)
        if max_grad_norm > 0.0:                                            # train.py:357-358
            torch.nn.utils.clip_grad_norm_(plist, max_grad_norm)
        opt.step()
        new_state = OrderedDict()
        for k, v in st.items():
            if k in P:
                new_state[k] = P[k].detach().clone()
            elif k in bufs_out:
                new_state[k] = bufs_out[k].clone()
            elif k.endswith("num_batches_tracked"):
                new_state[k] = v + 1
            else:
                new_state[k] = v.clone()
        out["new_state"] = new_state
        out["new_svals"] = {k: float(v.detach()) for k, v in S.items()}
        out["adam_state"] = opt.state_dict()
    return out


class OracleTrainer(object):
    """Persistent-state version of train_step for TIMING the CPU path (bench.py's
    cpu_baseline / --impl reference): parameters, Adam state and criterion scalars live
    across steps exactly as in common/train.py (no per-step cloning), so a timed step is
    only forward + loss + zero_grad + backward + [clip] + Adam.step (train.py:339-361)."""

    def __init__(self, kind, st, svals, learn=(True, True), lr=1e-4, weight_decay=5e-4, max_grad_norm=0.0,
                 droprate=0.0):
        self.kind, self.max_grad_norm, self.droprate = kind, max_grad_norm, droprate
        params, bufs = split_state(st)
        self.P = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in params.items())
        self.full = OrderedDict(self.P)
        for k, v in bufs.items():
            self.full[k] = v.detach().clone()
        self.S = OrderedDict()
        for name in (("sax", "saq") if kind == "posenet" else ("sax", "saq", "srx", "srq")):
            trainable = learn[0] if name in ("sax", "saq") else learn[1]
            self.S[name] = torch.tensor([svals[name]], dtype=torch.float32, requires_grad=trainable)
        groups = [{"params": list(self.P.values())}]
        sl = [v for v in self.S.values() if v.requires_grad]
        if sl:
            groups.append({"params": sl})
        self.opt = torch.optim.Adam(groups, lr=lr, weight_decay=weight_decay)

    def step(self, x, targ):
        bufs_out = {}
        mask = None
        if self.droprate > 0:
            B = x.shape[0] if x.dim() == 4 else x.shape[0] * x.shape[1]
            keep = (torch.rand(B, self.full["feature_extractor.fc.bias"].numel()) >= self.droprate).float()
            mask = keep / (1.0 - self.droprate)
        x = x.clone().requires_grad_(True)                               # train.py:339
        pred = model_forward("posenet" if self.kind == "posenet" else "mapnet", self.full, x, training=True,
                             drop_mask=mask, bufs_out=bufs_out)
        loss = criterion(self.kind, pred, targ, self.S)
        self.opt.zero_grad()
        loss.backward()
        if self.max_grad_norm > 0.0:
            torch.nn.utils.clip_grad_norm_(list(self.P.values()), self.max_grad_norm)
        self.opt.step()
        for k, v in bufs_out.items():
            self.full[k] = v
        return float(loss.item())                                         # train.py:361


# --------------------------------------------------------------------------
# FLOP model used by bench.py's roofline (SURVEY.md section 8d)
# --------------------------------------------------------------------------


def conv_macs_per_image(H=256, W=256):
    """Forward conv MACs per image of the ResNet-34 trunk; 4 784 652 288 at 256x256."""
    def out(n, k, s, p):
        return (n + 2 * p - k) // s + 1
    h, w = out(H, 7, 2, 3), out(W, 7, 2, 3)
    macs = h * w * 64 * 3 * 49
    conv1 = macs
    h, w = out(h, 3, 2, 1), out(w, 3, 2, 1)
    inpl = 64
    for planes, nblk, stride in STAGES:
        for b in range(nblk):
            s = stride if b == 0 else 1
            h2, w2 = out(h, 3, s, 1), out(w, 3, s, 1)
            macs += h2 * w2 * planes * inpl * 9
            macs += h2 * w2 * planes * planes * 9
            if s != 1 or inpl != planes:
                macs += h2 * w2 * planes * inpl
            h, w, inpl = h2, w2, planes
    return macs, conv1


def train_flops_per_image(H=256, W=256):
    """3x fwd conv FLOPs minus conv1's dgrad (no parameter needs d loss/d input)."""
    macs, conv1 = conv_macs_per_image(H, W)
    return 2.0 * (3 * macs - conv1)
