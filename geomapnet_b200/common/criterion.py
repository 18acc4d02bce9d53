"""Fused GPU criteria behind the reference's nn.Module surface.

Host-side mirror of /root/reference/common/criterion.py: PoseNetCriterion
(:33-52), MapNetCriterion (:54-109), MapNetOnlineCriterion (:111-184) with the
same constructor keywords, the same four 1-element nn.Parameters
(sax, saq, srx, srq; requires_grad = learn_beta / learn_gamma) and the same
``forward(pred, targ) -> tensor of shape [1]``.  Forward AND backward are one
CUDA launch (csrc/loss.cu); calc_vos_simple / calc_vos
(/root/reference/common/pose_utils.py:234-260) are folded into it.
QuaternionLoss (:15-31) is unused by scripts/train.py and out of scope.
"""
import torch
from torch import nn

from .. import _lib

__all__ = ["PoseNetCriterion", "MapNetCriterion", "MapNetOnlineCriterion"]


class _LossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mode, pred, targ, sax, saq, srx, srq):
        if not pred.is_cuda:
            raise RuntimeError("geomapnet_b200 criteria have no CPU path: pred must be a CUDA tensor")
        dev = pred.device
        p = pred.detach().contiguous().float()
        t = targ.detach().to(dev).contiguous().float()
        if mode == "posenet":
            if p.dim() != 2 or p.shape[1] != 6 or t.shape != p.shape:
                raise ValueError("PoseNetCriterion wants pred, targ [N,6]; got %s, %s"
                                 % (tuple(p.shape), tuple(t.shape)))
            N, Tp, Tt = p.shape[0], 1, 1
        else:
            if p.dim() != 3 or p.shape[2] != 6 or t.dim() != 3 or t.shape[2] != 6 or t.shape[0] != p.shape[0]:
                raise ValueError("criterion wants pred [N,T,6], targ [N,T',6]; got %s, %s"
                                 % (tuple(p.shape), tuple(t.shape)))
            N, Tp, Tt = p.shape[0], p.shape[1], t.shape[1]
        if N == 0:
            raise ValueError("empty batch")
        zero = torch.zeros(1, dtype=torch.float32, device=dev)
        s4 = torch.cat([v.detach().float().to(dev).reshape(1) if v is not None else zero
                        for v in (sax, saq, srx, srq)])
        out = torch.empty(5, dtype=torch.float32, device=dev)      # loss, ds[4]
        dpred = torch.empty_like(p)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().mapnet_loss_fwd_bwd(
                _lib.LOSS_MODE[mode], p.data_ptr(), t.data_ptr(), N, Tp, Tt, s4.data_ptr(),
                out.data_ptr(), dpred.data_ptr(), out.data_ptr() + 4, _lib.stream_ptr()),
                "mapnet_loss_fwd_bwd")
        ctx.save_for_backward(dpred, out)
        ctx.pred_shape = pred.shape
        ctx.has = [v is not None for v in (sax, saq, srx, srq)]
        return out[:1].clone()

    @staticmethod
    def backward(ctx, g):
        dpred, out = ctx.saved_tensors
        g = g.reshape(())
        gp = (dpred * g).view(ctx.pred_shape) if ctx.needs_input_grad[1] else None
        gs = []
        for k in range(4):
            if ctx.has[k] and ctx.needs_input_grad[3 + k]:
                gs.append((out[1 + k] * g).reshape(1))
            else:
                gs.append(None)
        return (None, gp, None) + tuple(gs)


def _check_l1(fn, which):
    if not isinstance(fn, nn.L1Loss) or getattr(fn, "reduction", "mean") != "mean":
        raise NotImplementedError("geomapnet_b200 criteria fuse nn.L1Loss() (the reference default, "
                                  "common/criterion.py:34) -- %s=%r is not supported" % (which, fn))


class PoseNetCriterion(nn.Module):
    def __init__(self, t_loss_fn=nn.L1Loss(), q_loss_fn=nn.L1Loss(), sax=0.0, saq=0.0, learn_beta=False):
        super(PoseNetCriterion, self).__init__()
        _check_l1(t_loss_fn, "t_loss_fn")
        _check_l1(q_loss_fn, "q_loss_fn")
        self.t_loss_fn = t_loss_fn
        self.q_loss_fn = q_loss_fn
        self.sax = nn.Parameter(torch.Tensor([sax]), requires_grad=learn_beta)
        self.saq = nn.Parameter(torch.Tensor([saq]), requires_grad=learn_beta)

    def forward(self, pred, targ):
        """pred, targ: N x 6  ->  loss [1]   (common/criterion.py:42-52)"""
        return _LossFn.apply("posenet", pred, targ, self.sax, self.saq, None, None)


class MapNetCriterion(nn.Module):
    def __init__(self, t_loss_fn=nn.L1Loss(), q_loss_fn=nn.L1Loss(), sax=0.0, saq=0.0, srx=0, srq=0.0,
                 learn_beta=False, learn_gamma=False):
        super(MapNetCriterion, self).__init__()
        _check_l1(t_loss_fn, "t_loss_fn")
        _check_l1(q_loss_fn, "q_loss_fn")
        self.t_loss_fn = t_loss_fn
        self.q_loss_fn = q_loss_fn
        self.sax = nn.Parameter(torch.Tensor([sax]), requires_grad=learn_beta)
        self.saq = nn.Parameter(torch.Tensor([saq]), requires_grad=learn_beta)
        self.srx = nn.Parameter(torch.Tensor([srx]), requires_grad=learn_gamma)
        self.srq = nn.Parameter(torch.Tensor([srq]), requires_grad=learn_gamma)

    def forward(self, pred, targ):
        """pred, targ: N x T x 6  ->  loss [1]   (common/criterion.py:76-109)"""
        return _LossFn.apply("mapnet", pred, targ, self.sax, self.saq, self.srx, self.srq)


class MapNetOnlineCriterion(nn.Module):
    def __init__(self, t_loss_fn=nn.L1Loss(), q_loss_fn=nn.L1Loss(), sax=0.0, saq=0.0, srx=0, srq=0.0,
                 learn_beta=False, learn_gamma=False, gps_mode=False):
        super(MapNetOnlineCriterion, self).__init__()
        _check_l1(t_loss_fn, "t_loss_fn")
        _check_l1(q_loss_fn, "q_loss_fn")
        self.t_loss_fn = t_loss_fn
        self.q_loss_fn = q_loss_fn
        self.sax = nn.Parameter(torch.Tensor([sax]), requires_grad=learn_beta)
        self.saq = nn.Parameter(torch.Tensor([saq]), requires_grad=learn_beta)
        self.srx = nn.Parameter(torch.Tensor([srx]), requires_grad=learn_gamma)
        self.srq = nn.Parameter(torch.Tensor([srq]), requires_grad=learn_gamma)
        self.gps_mode = gps_mode

    def forward(self, pred, targ):
        """pred: N x 2T x 6, targ: N x (2T-1) x 6 (2T in gps_mode)  (common/criterion.py:137-184)"""
        return _LossFn.apply("online_gps" if self.gps_mode else "online", pred, targ,
                             self.sax, self.saq, self.srx, self.srq)
