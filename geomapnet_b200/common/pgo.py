"""Pose-graph optimisation of predicted pose windows on the GPU, batched.

Host-side mirror of /root/reference/common/pose_utils.py:775-804 ``optimize_poses(pred_poses, vos=None, fc_vos=False,
target_poses=None, sax=1, saq=1, srx=1, srq=1)`` (PoseGraph / PoseGraphFC.optimize, :458-773), which
scripts/eval.py:172-178 calls once per frame; ``optimize_pose_windows`` runs the same Gauss-Newton for W windows in ONE
launch (csrc/pgo.cu, one thread block per window, fp64).  No CPU path.

robust_c=c (both batched entry points) gives the absolute factors the Cauchy loss rho(s) = c^2 log(1 + s / c^2) of their
squared whitened residual s, solved by iteratively reweighted Gauss-Newton: each iteration weighs slot k's absolute
factor by w_k = 1 / (1 + s_k / c^2) at the iteration's starting state.  c is in multiples of sigma; a frame whose
prediction is far off stops pulling on its window instead of pulling in proportion to its error.
"""
import ctypes
import math

import numpy as np
import torch

from .. import _lib

__all__ = ["optimize_poses", "optimize_pose_windows", "optimize_pose_windows_cov", "vos_from_target_poses",
           "check_robust_c"]


def check_robust_c(robust_c):
    """robust_c as a float, or None (no robust loss) for None; ValueError for anything but a finite real number > 0"""
    if robust_c is None:
        return None
    if isinstance(robust_c, (bool, np.bool_)) or not isinstance(robust_c, (int, float, np.integer, np.floating)):
        raise ValueError("robust_c must be None or a finite number > 0 (the Cauchy scale in sigmas), got %r"
                         % (robust_c,))
    c = float(robust_c)
    if not (math.isfinite(c) and c > 0):
        raise ValueError("robust_c must be None or a finite number > 0 (the Cauchy scale in sigmas), got %r" % (c,))
    return c


def _qmult(a, b):
    w = a[..., 0] * b[..., 0] - a[..., 1] * b[..., 1] - a[..., 2] * b[..., 2] - a[..., 3] * b[..., 3]
    x = a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0] + a[..., 2] * b[..., 3] - a[..., 3] * b[..., 2]
    y = a[..., 0] * b[..., 2] - a[..., 1] * b[..., 3] + a[..., 2] * b[..., 0] + a[..., 3] * b[..., 1]
    z = a[..., 0] * b[..., 3] + a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1] + a[..., 3] * b[..., 0]
    return torch.stack((w, x, y, z), -1)


def vos_from_target_poses(target_poses):
    """pose_utils.py:793-799: VOs in the frame of the poses -- plain translation differences and q0^-1 * q1.
    target_poses: [..., N, 7] -> [..., N-1, 7]"""
    t = torch.as_tensor(target_poses, dtype=torch.float64)
    q0, q1 = t[..., :-1, 3:], t[..., 1:, 3:]
    qinv = torch.cat((q0[..., :1], -q0[..., 1:]), -1) / (q0 * q0).sum(-1, keepdim=True)
    return torch.cat((t[..., 1:, :3] - t[..., :-1, :3], _qmult(qinv, q1)), -1)


def optimize_pose_windows(pred_poses, vos, fc_vos=False, sax=1.0, saq=1.0, srx=1.0, srq=1.0, n_iters=10, device=None,
                          exact_solve=False, robust_c=None):
    """pred_poses [W,N,7] (translation + quaternion wxyz), vos [W,N-1,7] (or [W,N(N-1)/2,7] when fc_vos: every pair
    i<j in row-major order) -> optimised poses [W,N,7] float64 on the device.  Raises if a window's normal matrix
    is not positive definite (scipy's cholesky would raise LinAlgError in the reference).

    exact_solve=False reproduces the reference's linear solve literally: pose_utils.py:605-608 calls
    ``slin.solve_triangular(R.T, -b)`` with scipy's default ``lower=False``, which reads only the diagonal of the
    (lower-triangular) R', so its step is R^-1 diag(R)^-1 (-b) rather than H^-1 (-b).  That is what scripts/eval.py
    computes; exact_solve=True takes the Gauss-Newton step instead.

    robust_c=c: the absolute factors take the Cauchy loss of scale c (module docstring; residual (t - t0) / sqrt(sax),
    (q - q0) / sqrt(saq)), with the same step rule; returns (poses, w [W,N]), w each slot's weight at the returned
    state.  A bad robust_c raises ValueError before anything is launched."""
    c = check_robust_c(robust_c)
    if device is None:
        device = pred_poses.device if torch.is_tensor(pred_poses) and pred_poses.is_cuda else torch.device("cuda")
    p = torch.as_tensor(pred_poses, dtype=torch.float64).to(device).contiguous()
    v = torch.as_tensor(vos, dtype=torch.float64).to(device).contiguous()
    if p.dim() != 3 or p.shape[2] != 7:
        raise ValueError("pred_poses must be [W,N,7], got %s" % (tuple(p.shape),))
    W, N, _ = p.shape
    E = N * (N - 1) // 2 if fc_vos else N - 1
    if tuple(v.shape) != (W, E, 7):
        raise ValueError("vos must be [%d,%d,7], got %s" % (W, E, tuple(v.shape)))
    out = torch.empty_like(p)
    status = torch.zeros(1, dtype=torch.int32, device=device)
    with torch.cuda.device(device):
        if c is None:
            _lib.check(_lib.lib().mapnet_pgo_optimize(p.data_ptr(), v.data_ptr(), out.data_ptr(), W, N,
                                                      1 if fc_vos else 0, float(sax), float(saq), float(srx),
                                                      float(srq), int(n_iters), 1 if exact_solve else 0,
                                                      status.data_ptr(), _lib.stream_ptr()), "mapnet_pgo_optimize")
        else:
            w = torch.empty((W, N), dtype=torch.float64, device=device)
            _lib.check(_lib.lib().mapnet_pgo_optimize_robust(p.data_ptr(), v.data_ptr(), out.data_ptr(), W, N,
                                                             1 if fc_vos else 0, float(sax), float(saq), float(srx),
                                                             float(srq), int(n_iters), 1 if exact_solve else 0, c,
                                                             w.data_ptr(), status.data_ptr(), _lib.stream_ptr()),
                       "mapnet_pgo_optimize_robust")
    if int(status.item()) != 0:
        raise np.linalg.LinAlgError("pose graph: normal matrix of a window is not positive definite")
    return out if c is None else (out, w)


def optimize_pose_windows_cov(pred_poses, abs_cov7, vos, fc_vos=False, srx=1.0, srq=1.0, n_iters=10, robust_c=None):
    """Covariance-weighted pose graph (csrc/pgo.cu, k_pgo_cov): pred_poses [W,N,7] (translation + quaternion wxyz),
    abs_cov7 [W,N,7,7] the covariance S7 of each absolute pose, vos as for optimize_pose_windows.  Slot k's absolute
    factor has residual C^-1 (z_k - p_k) with S7 = C C' (lower Cholesky factor); the relative factors (srx, srq), state
    and manifold update are optimize_pose_windows'; every iteration takes the exact Gauss-Newton step.  Returns
    (poses [W,N,7], cov [W,N,6,6]) float64 on the device: cov is each slot's posterior covariance, the 6 x 6 diagonal
    block of the inverse normal matrix at the returned state, in (t, log q) coordinates.  Raises
    np.linalg.LinAlgError if a window's normal matrix (or one of its S7) is not positive definite.

    robust_c=c: the absolute factors take the Cauchy loss of scale c (module docstring; residual C^-1 (z_k - p_k)), and
    the posterior is the inverse normal matrix at the returned state with the weights at that state; returns (poses,
    cov, w [W,N]), w each slot's weight at the returned state.  A bad robust_c raises ValueError before any launch."""
    rc = check_robust_c(robust_c)
    device = pred_poses.device if torch.is_tensor(pred_poses) and pred_poses.is_cuda else torch.device("cuda")
    p = torch.as_tensor(pred_poses, dtype=torch.float64).to(device).contiguous()
    c = torch.as_tensor(abs_cov7, dtype=torch.float64).to(device).contiguous()
    v = torch.as_tensor(vos, dtype=torch.float64).to(device).contiguous()
    if p.dim() != 3 or p.shape[2] != 7:
        raise ValueError("pred_poses must be [W,N,7], got %s" % (tuple(p.shape),))
    W, N, _ = p.shape
    E = N * (N - 1) // 2 if fc_vos else N - 1
    if tuple(c.shape) != (W, N, 7, 7):
        raise ValueError("abs_cov7 must be [%d,%d,7,7], got %s" % (W, N, tuple(c.shape)))
    if tuple(v.shape) != (W, E, 7):
        raise ValueError("vos must be [%d,%d,7], got %s" % (W, E, tuple(v.shape)))
    out = torch.empty_like(p)
    cov = torch.empty((W, N, 6, 6), dtype=torch.float64, device=device)
    status = torch.zeros(1, dtype=torch.int32, device=device)
    with torch.cuda.device(device):
        if rc is None:
            _lib.check(_lib.lib().mapnet_pgo_optimize_cov(p.data_ptr(), c.data_ptr(), v.data_ptr(), out.data_ptr(),
                                                          cov.data_ptr(), W, N, 1 if fc_vos else 0, float(srx),
                                                          float(srq), int(n_iters), status.data_ptr(),
                                                          _lib.stream_ptr()), "mapnet_pgo_optimize_cov")
        else:
            w = torch.empty((W, N), dtype=torch.float64, device=device)
            _lib.check(_lib.lib().mapnet_pgo_optimize_cov_robust(p.data_ptr(), c.data_ptr(), v.data_ptr(),
                                                                 out.data_ptr(), cov.data_ptr(), W, N,
                                                                 1 if fc_vos else 0, float(srx), float(srq),
                                                                 int(n_iters), rc, w.data_ptr(), status.data_ptr(),
                                                                 _lib.stream_ptr()), "mapnet_pgo_optimize_cov_robust")
    if int(status.item()) != 0:
        raise np.linalg.LinAlgError("pose graph: normal matrix of a window is not positive definite")
    return (out, cov) if rc is None else (out, cov, w)


def optimize_poses(pred_poses, vos=None, fc_vos=False, target_poses=None, sax=1, saq=1, srx=1, srq=1):
    """The reference's signature and return value (one window, numpy [N,7]); see optimize_pose_windows for batches."""
    if vos is None:
        if target_poses is None:
            print('Specify either VO or target poses')
            return None
        if fc_vos:
            raise ValueError("fc_vos needs explicit VOs (the reference derives only consecutive VOs from target poses)")
        vos = vos_from_target_poses(np.asarray(target_poses, dtype=np.float64))
    p = torch.as_tensor(np.asarray(pred_poses, dtype=np.float64))[None]
    v = torch.as_tensor(np.asarray(vos, dtype=np.float64))[None]
    return optimize_pose_windows(p, v, fc_vos=fc_vos, sax=sax, saq=saq, srx=srx, srq=srq)[0].cpu().numpy()
