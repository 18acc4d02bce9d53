"""The CPU restatement of the reference's pose-graph optimisation (oracle/pgo_oracle.py) pinned against the committed
goldens tests/golden/pgo.npz and live_reference.npz, made by oracle/make_goldens.py from the reference's own
PoseGraph / PoseGraphFC classes and numpy helpers (common/pose_utils.py:306-804)."""
import os

import numpy as np

from oracle import pgo_oracle as P


def _cases(golden_dir):
    g = np.load(os.path.join(golden_dir, "pgo.npz"))
    i = 0
    while "case%d_cfg" % i in g.files:
        cfg = g["case%d_cfg" % i]
        yield i, int(cfg[0]), bool(cfg[1]), tuple(cfg[3:7]), g["case%d_poses" % i], g["case%d_vos" % i], g["case%d_out" % i]
        i += 1


def test_pgo_oracle_matches_reference_goldens(golden_dir):
    n = 0
    for ci, N, fc, sig, poses, vos, ref in _cases(golden_dir):
        for w in range(len(poses)):
            got = P.optimize_poses(poses[w], vos[w], fc, sax=sig[0], saq=sig[1], srx=sig[2], srq=sig[3])
            assert np.abs(got - ref[w]).max() <= 1e-11, (ci, w)
            n += 1
    assert n >= 30
    g = np.load(os.path.join(golden_dir, "pgo.npz"))
    got = P.optimize_poses(g["targ_pred"], target_poses=g["targ_gt"], sax=1.0, saq=1.0, srx=0.1, srq=0.1)
    assert np.abs(got - g["targ_out"]).max() <= 1e-11


def test_reference_step_is_not_the_gauss_newton_step(golden_dir):
    """pose_utils.py:605-608: solve_triangular(R.T, -b) with scipy's default lower=False reads only the diagonal of R'.
    The restatement must reproduce THAT (goldens above); the true Gauss-Newton step is a different iteration."""
    for ci, N, fc, sig, poses, vos, ref in _cases(golden_dir):
        if ci != 2:
            continue
        exact = P.optimize(poses[0], vos[0], *sig, fc=fc, exact_solve=True)
        lit = P.optimize(poses[0], vos[0], *sig, fc=fc, n_iters=1)
        ex1 = P.optimize(poses[0], vos[0], *sig, fc=fc, n_iters=1, exact_solve=True)
        assert np.abs(lit - ex1).max() > 1e-4            # the first steps differ ...
        assert np.abs(exact - ref[0]).max() < 5e-2       # ... although both iterations settle near the same poses


def test_pgo_oracle_matches_live_reference_classes(golden_dir):
    L = np.load(os.path.join(golden_dir, "live_reference.npz"))
    for ci in range(3):
        pred, vos, fc = L["pgo%d_pred" % ci], L["pgo%d_vos" % ci], bool(L["pgo%d_fc" % ci])
        got = P.optimize_poses(pred, vos, fc, sax=1.5, saq=0.3, srx=0.7, srq=0.1)
        assert np.abs(L["pgo%d_out" % ci] - got).max() <= 1e-12
    # the numpy helpers one by one
    for name in ("dpq_q", "dpsq_q", "dpsq_p", "dqstq_t", "m_rot"):
        x = L["pgohelper_%s_in" % name]
        assert np.abs(L["pgohelper_%s_out" % name] - getattr(P, name)(x)).max() <= 1e-15, name
