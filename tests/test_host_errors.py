"""Error behaviour and small host-side helpers of the product modules that need no device.

The reference's convention is plain Python exceptions before any work is done (`raise NotImplementedError`
scripts/train.py:84,101; `KeyError` common/train.py:42; `optimize_poses` prints and returns None without VOs,
common/pose_utils.py:789-792).  These checks run BEFORE any launch, so they are testable on the CPU."""
import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def built():
    from geomapnet_b200 import build
    build.build(verbose=False)


def test_unknown_precision_is_rejected(built):
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet
    with pytest.raises(ValueError, match="precision"):
        PoseNet(torchvision.models.resnet34(weights=None), pretrained=False, precision="fp8")
    for prec in ("bf16", "tc_split", "fp32", "bf16_simt"):       # the four engines share one parameter table
        m = PoseNet(torchvision.models.resnet34(weights=None), pretrained=False, precision=prec)
        assert len(m.state_dict()) == 222 and m.precision == prec


def test_fused_adam_rejects_invalid_hyper_parameters():
    from geomapnet_b200.common.optimizer import FusedAdam, Optimizer
    p = [torch.nn.Parameter(torch.zeros(4))]
    for kw in (dict(lr=-1e-3), dict(eps=-1e-8), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)), dict(weight_decay=-1.0)):
        with pytest.raises(ValueError):
            FusedAdam(p, **kw)
    with pytest.raises(Exception):
        Optimizer(params=p, method="adagrad", base_lr=1e-3, weight_decay=0.0)      # the reference knows sgd / adam / rmsprop


def test_tuple_sharding_never_splits_a_tuple_and_needs_equal_shards():
    from geomapnet_b200.ddp import shard_tuples
    x = torch.arange(8 * 3 * 2).view(8, 3, 2)                   # [N, T, ...]
    parts = [shard_tuples(x, r, 4) for r in range(4)]
    assert all(p.shape == (2, 3, 2) for p in parts) and torch.equal(torch.cat(parts, 0), x)
    with pytest.raises(ValueError, match="divisible"):
        shard_tuples(x, 0, 3)


def test_color_jitter_sampler_ranges_follow_torchvision_check_input():
    from geomapnet_b200.data import ColorJitterSampler
    s = ColorJitterSampler(0.7, 0.7, 0.7, 0.5)                  # scripts/train.py:123-124 with color_jitter = 0.7
    assert s.brightness == (pytest.approx(0.3), pytest.approx(1.7)) and s.hue == (-0.5, 0.5)
    assert ColorJitterSampler(1.5).brightness == (0.0, 2.5)     # lower end clipped at 0
    off = ColorJitterSampler()                                  # nothing enabled: neutral factors, still a valid record
    assert off.brightness is None and off.hue is None
    rec = off.sample(3)
    assert rec.dtype == torch.uint8 and tuple(rec.shape) == (3, 32)
    fac = rec.numpy().view(np.float32).reshape(3, 8)[:, 4:]
    assert np.array_equal(fac, np.tile(np.float32([1, 1, 1, 0]), (3, 1)))
    order = rec.numpy().view(np.int32).reshape(3, 8)[:, :4]
    assert all(sorted(o) == [0, 1, 2, 3] for o in order.tolist())
    with pytest.raises(ValueError):
        ColorJitterSampler(brightness=-0.1)
    with pytest.raises(ValueError):
        ColorJitterSampler(hue=0.6)


def test_image_pipeline_rejects_bad_statistics():
    from geomapnet_b200.data import ImagePipeline, resize_output_size
    with pytest.raises(ValueError, match="std"):
        ImagePipeline([0.5, 0.5, 0.5], [0.2, 0.0, 0.2])
    # torchvision.transforms.Resize(256) on 480x640 (7Scenes) and 960x1280 (RobotCar centre camera): shorter side -> 256
    assert resize_output_size(480, 640) == (256, 341) and resize_output_size(960, 1280) == (256, 341)
    assert resize_output_size(640, 480) == (341, 256) and resize_output_size(300, 300) == (256, 256)


def test_optimize_poses_without_vos_behaves_like_the_reference(capsys):
    """common/pose_utils.py:789-792: neither VOs nor target poses -> a printed message and None, no exception."""
    from geomapnet_b200.common import pgo
    assert pgo.optimize_poses(np.zeros((3, 7))) is None
    assert "Specify either VO or target poses" in capsys.readouterr().out
    with pytest.raises(ValueError, match="fc_vos"):
        pgo.optimize_poses(np.zeros((3, 7)), target_poses=np.zeros((3, 7)), fc_vos=True)


def test_vos_from_target_poses_is_the_reference_arithmetic(golden_dir):
    """common/pose_utils.py:793-799: VO translation = plain difference, rotation = q0^-1 * q1 -- against the oracle's
    numpy restatement (pinned to the reference in tests/test_pgo_oracle.py)."""
    from geomapnet_b200.common import pgo
    from oracle import pgo_oracle as P
    rng = np.random.default_rng(4)
    q = rng.normal(size=(2, 5, 4)); q /= np.linalg.norm(q, axis=-1, keepdims=True)
    poses = np.concatenate((rng.normal(size=(2, 5, 3)), q), -1)
    got = pgo.vos_from_target_poses(poses).numpy()
    assert got.shape == (2, 4, 7)
    for w in range(2):
        for i in range(4):
            ref = np.concatenate((poses[w, i + 1, :3] - poses[w, i, :3], P.qmult(P.qinverse(poses[w, i, 3:]), poses[w, i + 1, 3:])))
            assert np.abs(got[w, i] - ref).max() <= 1e-14


def test_mf_tuple_lengths_and_clipping():
    """dataset_loaders/composite.py:64-75,105-109: offsets centred on the middle frame, clipped at the sequence ends;
    no_duplicates shortens the dataset instead of repeating frames."""
    from geomapnet_b200.data import tuples as T
    assert T.mf_offsets(3, 10).tolist() == [-10, 0, 10]
    assert T.mf_indices(0, 100, 3, 10).tolist() == [0, 0, 10]              # clipped at the start: frame 0 repeats
    assert T.mf_indices(99, 100, 3, 10).tolist() == [89, 99, 99]
    assert T.mf_indices(0, 100, 3, 10, no_duplicates=True).tolist() == [0, 10, 20]
    assert T.mf_len(100, 3, 10) == 100 and T.mf_len(100, 3, 10, no_duplicates=True) == 80
    tr, va = T.mfonline_indices(85, 100, 100, 5, 2)
    assert tr.tolist() == [81, 83, 85, 87, 89] and va.tolist() == [(85 % 92) + k for k in (0, 2, 4, 6, 8)]
    idx = T.batch_frame_indices([0, 50], 100, 3, 10)
    assert idx.dtype == np.int32 and idx.tolist() == [0, 0, 10, 40, 50, 60]


def _rc_and_message(fn, *args):
    from geomapnet_b200 import _lib
    rc = fn(*args)
    msg = _lib.lib().mapnet_last_error()
    return rc, (msg.decode() if msg else "")


def test_element_wise_test_entry_points_fail_with_a_message(built):
    """mapnet_test_bn_forward / _bn_backward / _stem_pool / _gap check their arguments before they touch the device:
    on any host a bad call returns non-zero with a message (the pointers below are never dereferenced); on a host
    without a device so does a well-formed call."""
    from geomapnet_b200 import _lib
    L = _lib.lib()
    buf = np.zeros(64, dtype=np.float32)
    h = buf.ctypes.data
    fwd = lambda prec, res_mode, source, M, C, res, nrep=8: _rc_and_message(
        L.mapnet_test_bn_forward, prec, res_mode, 1, source, M, C, h, res, h, h, h, nrep, h, None)
    cases = [
        (fwd(1, 0, 1, 64, 96, None), "multiple of 64"),                  # the apply kernels take 64-channel slices
        (fwd(1, 2, 0, 64, 64, None), "res_mode 2 needs res"),           # the downsample branch is missing
        (fwd(4, 0, 0, 64, 64, None), "not a training precision"),       # fp8 has no training element-wise path
        (fwd(1, 3, 0, 64, 64, None), "res_mode 3"),
        (fwd(1, 0, 1, 64, 64, None, nrep=33), "nrep"),                   # more replicas than a slot has
        (_rc_and_message(L.mapnet_test_bn_backward, 1, 0, 1, 64, 64, h, None, h, None, h, None, None, h, None, 0, 0.0,
                         h, None), "zmask is given exactly when gate == 1"),
        (_rc_and_message(L.mapnet_test_bn_backward, 3, 2, 0, 64, 64, h, None, h, None, h, None, None, h, None, 0, 0.0,
                         h, None), "neither 0 (reduce) nor 1 (lazy)"),
        (_rc_and_message(L.mapnet_test_stem_pool, 1, 1, 1, 1, 7, 9, h, h, h, h, h, h, h, h, 8, h, None),
         "lazy backward needs even Hc, Wc"),
        (_rc_and_message(L.mapnet_test_stem_pool, 4, 0, 0, 1, 8, 8, h, h, h, None, None, None, h, None, 8, h, None),
         "fp8 is the inference pool"),
        (_rc_and_message(L.mapnet_test_gap, 7, 2, 4, 512, h, h, h, h, None), "not a training precision"),
        (_rc_and_message(L.mapnet_test_gap, 1, 2, 4, 12, h, h, h, h, None), "bad shape"),
    ]
    for (rc, msg), want in cases:
        assert rc != 0 and want in msg, (rc, msg, want)
    if torch.cuda.is_available():       # the well-formed calls below would run (the pointers are host memory)
        return
    # without a CUDA device, well-formed calls fail with a message instead of crashing
    buf = np.zeros(64 * 15 * 2, dtype=np.float32)
    h = buf.ctypes.data
    calls = [
        (L.mapnet_test_bn_forward, 1, 0, 1, 0, 64, 64, h, None, h, h, None, 0, h, None),
        (L.mapnet_test_bn_backward, 1, 0, 0, 64, 64, h, None, h, None, h, None, None, h, None, 0, 0.0, h, None),
        (L.mapnet_test_stem_pool, 1, 0, 0, 1, 8, 8, h, h, h, None, None, None, h, None, 0, h, None),
        (L.mapnet_test_gap, 1, 2, 4, 512, h, h, h, h, None),
    ]
    for fn, *args in calls:
        rc, msg = _rc_and_message(fn, *args)
        assert rc != 0 and "no CUDA device" in msg, (fn.__name__, rc, msg)


def test_conv_ex_test_entry_point_fails_with_a_message(built):
    """mapnet_test_conv_ex checks its arguments before it touches the device (the pointers below are never
    dereferenced); on a host without a device a well-formed call fails with a message too."""
    from geomapnet_b200 import _lib
    L = _lib.lib()
    buf = np.zeros(64, dtype=np.float32)
    h = buf.ctypes.data
    ex = lambda prec, kind, Ci, k, stride, in1, wmat, res, scale: _rc_and_message(
        L.mapnet_test_conv_ex, prec, kind, 2, 8, 8, Ci, 64, k, stride, h, in1, wmat, res, scale, h, None)
    cases = [
        (ex(0, 0, 64, 3, 1, None, h, None, 0.0), "not a tensor-core training precision"),   # fp32 is mapnet_test_conv's
        (ex(1, 3, 64, 3, 1, None, h, None, 0.0), "kind 3"),
        (ex(1, 0, 96, 3, 1, None, h, None, 0.0), "bad shape"),                               # 64-channel k-blocks
        (ex(1, 0, 64, 5, 1, None, h, None, 0.0), "bad shape"),
        (ex(1, 2, 64, 3, 1, None, None, None, 0.0), "null argument"),                        # wgrad needs dy
        (ex(1, 0, 64, 3, 1, None, None, None, 0.0), "null argument"),                        # fprop needs weights
        (ex(1, 0, 64, 3, 1, None, h, h, 0.0), "a residual is a dgrad feature"),
        (ex(1, 1, 64, 3, 1, None, h, None, 0.5), "out_scale"),                               # bf16 has no gradient scale
        (ex(3, 0, 64, 3, 1, None, h, None, 0.5), "out_scale"),                               # nor does strict fprop
        (ex(3, 1, 64, 3, 1, None, h, None, -0.5), "out_scale"),
        (ex(3, 2, 64, 3, 1, h, None, None, float("inf")), "out_scale"),
    ]
    for (rc, msg), want in cases:
        assert rc != 0 and want in msg, (rc, msg, want)
    if torch.cuda.is_available():
        return
    for prec, kind, in1, wmat, res, scale in ((1, 0, None, h, None, 0.0), (3, 1, None, h, h, 0.25), (3, 2, h, None, None, 0.25)):
        rc, msg = ex(prec, kind, 64, 3, 2, in1, wmat, res, scale)
        assert rc != 0 and "no CUDA device" in msg, (prec, kind, rc, msg)
