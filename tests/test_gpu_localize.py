"""GPU tests of localisation from camera frames: the fused vertical-resize + Normalize + space-to-depth kernel
(csrc/preprocess.cu, k_pre_resize_v_s2d) against k_stem_s2d over ImagePipeline's float32 output, bit for bit, and
inference.Localizer against the three-call chain post(Predictor(ImagePipeline(frames))) -- bitwise, in every engine
precision, with dropout, across snapshot refreshes, for every input form, and one library launch fewer per call."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# data/7Scenes/chess/stats.txt of the reference: row 0 the mean, row 1 the variance (Normalize takes its square root)
CHESS_MEAN = [5.009650708326967017e-01, 4.413125411911532625e-01, 4.458285283490354689e-01]
CHESS_STD = [float(np.sqrt(v)) for v in (4.329720281018845096e-02, 5.278270383679337097e-02, 4.760929057962018374e-02)]
POSE_M, POSE_S = [0.5, -1.25, 2.0], [1.5, 0.75, 2.5]
SIZES = [(480, 640), (960, 1280), (256, 256), (200, 300), (481, 643), (640, 480)]


def _lib():
    from geomapnet_b200 import _lib
    return _lib


def _frames(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, H, W, 3), dtype=torch.uint8, generator=g)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the stem operand, bitwise
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", SIZES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("precision", ["bf16", "tc_split"])
def test_fused_stem_operand_is_bitwise_k_stem_s2d_over_image_pipeline(precision, hw):
    from geomapnet_b200.data import ImagePipeline, resize_output_size
    L = _lib()
    lib = L.lib()
    H, W = hw
    Ho, Wo = resize_output_size(H, W, 256)
    hc, wc = (Ho - 1) // 2 + 1, (Wo - 1) // 2 + 1
    Hs, Wsp = hc + 3, (wc + 6) // 4 * 4
    elt = 4 if precision == "tc_split" else 2          # hi/lo fp16 planes: 4 bytes per element
    pipe = ImagePipeline(CHESS_MEAN, CHESS_STD, 256)
    fp = ctypes.POINTER(ctypes.c_float)
    for B in (1, 3, 64):
        frames = _frames(B, H, W, H * 7 + W + B).cuda()
        x = pipe(frames)
        pre = ctypes.c_void_p()
        L.check(lib.mapnet_preprocess_create(ctypes.byref(pre), H, W, 256, B), "mapnet_preprocess_create")
        try:
            # both buffers start from the same non-zero pattern: the zero halo and channels 12..15 must be written
            fused = torch.full((B * Hs * Wsp * 16 * elt,), 0xA5, dtype=torch.uint8, device="cuda")
            ref = fused.clone()
            L.check(lib.mapnet_test_stem_operand(L.PREC[precision], pre, frames.data_ptr(), None, B,
                                                 pipe.mean.ctypes.data_as(fp), pipe.std.ctypes.data_as(fp),
                                                 fused.data_ptr(), L.stream_ptr()), "mapnet_test_stem_operand(frames)")
            L.check(lib.mapnet_test_stem_operand(L.PREC[precision], pre, None, x.data_ptr(), B, None, None,
                                                 ref.data_ptr(), L.stream_ptr()), "mapnet_test_stem_operand(x)")
            torch.cuda.synchronize()
        finally:
            lib.mapnet_preprocess_destroy(pre)
        assert not bool((ref == 0xA5).all())
        diff = int((fused != ref).sum())
        assert diff == 0, (precision, hw, B, diff)
        # the padding channels and the halo are zero bytes
        blocks = ref.view(B, Hs, Wsp, 16 * elt)
        if precision == "bf16":
            assert int(blocks[..., 24:].count_nonzero()) == 0
        assert int(blocks[:, :2].count_nonzero()) == 0 and int(blocks[:, :, :2].count_nonzero()) == 0


# ---------------------------------------------------------------------------------------------------------------------
# helpers: predictors and the three-call chain
# ---------------------------------------------------------------------------------------------------------------------
def _predictor(kind, precision, seed=5, max_batch=4, droprate=0.0, calib_frames=None):
    from oracle import weights
    from helpers import make_product_model
    from geomapnet_b200.inference import Predictor
    from geomapnet_b200.data import ImagePipeline
    st = weights.make_state(seed)
    model, net = make_product_model(st, kind, "bf16" if precision == "fp8" else precision, droprate=droprate)
    if precision != "fp8":
        return Predictor(model, max_batch=max_batch), model, net
    calib = ImagePipeline(CHESS_MEAN, CHESS_STD)(calib_frames.cuda())
    return Predictor(model, max_batch=max_batch, precision="fp8", calibration=calib), model, net


def _chain(pr, frames, pose_m=None, pose_s=None):
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.inference import post
    return post(pr(ImagePipeline(CHESS_MEAN, CHESS_STD, 256)(frames.cuda())), pose_m, pose_s)


# ---------------------------------------------------------------------------------------------------------------------
# 2. poses, bitwise
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["posenet", "mapnet"])
@pytest.mark.parametrize("precision", ["bf16", "tc_split", "fp8"])
def test_localizer_is_bitwise_the_three_call_chain(precision, kind):
    from geomapnet_b200.inference import Localizer
    mb = 4
    frames = _frames(2 * mb + 1, 480, 640, 11)
    pr, _, _ = _predictor(kind, precision, max_batch=mb, calib_frames=frames[:mb])
    plain = Localizer(pr, CHESS_MEAN, CHESS_STD)
    metric = Localizer(pr, CHESS_MEAN, CHESS_STD, pose_m=POSE_M, pose_s=POSE_S)
    for n in (1, 3, mb, 2 * mb + 1):                    # B = 1, odd, max_batch, and chunks of max_batch
        f = frames[:n].cuda()
        got, want = plain(f), _chain(pr, f)
        assert got.dtype == torch.float64 and tuple(got.shape) == (n, 7)
        assert torch.equal(got, want), (precision, kind, n, float((got - want).abs().max()))
        got, want = metric(f), _chain(pr, f, POSE_M, POSE_S)
        assert torch.equal(got, want), (precision, kind, n, "pose_m/pose_s")
        assert torch.equal(metric(f), got)              # graph replay
    assert not torch.equal(plain(frames[:3].cuda()), metric(frames[:3].cuda()))
    plain.close(); metric.close(); pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. dropout, 4. snapshots
# ---------------------------------------------------------------------------------------------------------------------
def test_dropout_masks_follow_the_predictors_sequence_of_calls():
    from geomapnet_b200.inference import Localizer
    pa, _, _ = _predictor("posenet", "bf16", seed=3, droprate=0.5)
    pb, _, _ = _predictor("posenet", "bf16", seed=3, droprate=0.5)
    pb.seed = pa.seed
    loc = Localizer(pa, CHESS_MEAN, CHESS_STD)
    f640 = _frames(4, 480, 640, 1)
    f643 = _frames(4, 481, 643, 2)            # resizes to 256x342: a second engine
    f641 = _frames(4, 480, 641, 3)            # resizes to 256x341 as 480x640 does: a new graph, no new engine shape
    calls = [f640[:2], f640[:2], f640[:3], f643[:2], f640[:2], f641[:2], f641[:3], f643[:2], f640[:1], f640[:2]]
    prev = None
    for k, f in enumerate(calls):
        got, want = loc(f.cuda()), _chain(pb, f)
        assert torch.equal(got, want), (k, tuple(f.shape))
        if k == 1:
            assert not torch.equal(got, prev)         # the same frames again: a new mask
        prev = got
    loc.close(); pa.close(); pb.close()


@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_refresh_changes_the_localizer_output_to_the_new_snapshot(precision):
    from geomapnet_b200.inference import Localizer
    from geomapnet_b200.common.optimizer import Optimizer
    frames = _frames(3, 480, 640, 21)
    pr, model, _ = _predictor("posenet", precision, seed=9, calib_frames=frames)
    loc = Localizer(pr, CHESS_MEAN, CHESS_STD, pose_m=POSE_M, pose_s=POSE_S)
    f = frames.cuda()
    before = loc(f)
    opt = Optimizer(params=model.parameters(), method="adam", base_lr=1e-2, weight_decay=0.0)
    model.train()
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    out = model(x.requires_grad_(True))
    opt.learner.zero_grad()
    out.square().sum().backward()
    opt.learner.step()
    assert torch.equal(loc(f), before)                  # frozen until refresh
    pr.refresh()
    after = loc(f)
    assert not torch.equal(after, before)
    assert torch.equal(after, _chain(pr, f, POSE_M, POSE_S))
    loc.close(); pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. input forms, 6. launches
# ---------------------------------------------------------------------------------------------------------------------
def test_host_tensors_arrays_and_cuda_frames_agree():
    from geomapnet_b200.inference import Localizer
    pr, _, _ = _predictor("posenet", "bf16", seed=2)
    loc = Localizer(pr, CHESS_MEAN, CHESS_STD)
    frames = _frames(3, 480, 640, 5)
    ref = loc(frames.cuda())
    assert ref.is_cuda
    for form in (frames, frames.numpy(), frames.pin_memory()):
        assert torch.equal(loc(form), ref)
    one = loc(frames[1].numpy())
    assert tuple(one.shape) == (7,) and one.is_cuda
    assert torch.equal(one, loc(frames[1:2].cuda())[0])
    assert torch.equal(loc(frames[1].cuda()), one)
    loc.close(); pr.close()


def test_one_library_launch_fewer_than_the_chain():
    """2 preprocess launches + 43 engine launches + mapnet_pose_post against the chain's 2 + 44 + 1: counted on the eager
    run before the capture (the capture calls the library once more; a replay makes no library call)"""
    from geomapnet_b200.data import ImagePipeline
    from geomapnet_b200.inference import Localizer, post
    lib = _lib().lib()
    pr, _, _ = _predictor("posenet", "bf16", seed=4)
    loc = Localizer(pr, CHESS_MEAN, CHESS_STD, pose_m=POSE_M, pose_s=POSE_S)
    pipe = ImagePipeline(CHESS_MEAN, CHESS_STD)
    pr._engine(256, 341)                                # the engine's creation and snapshot load are not counted
    for B in (1, 4):
        f = _frames(B, 480, 640, B).cuda()
        c0 = lib.mapnet_launch_count()
        loc(f)
        c1 = lib.mapnet_launch_count()
        assert c1 - c0 == 2 * (2 + 43 + 1), (B, c1 - c0)
        loc(f)
        assert lib.mapnet_launch_count() == c1          # replay
        x = pipe(f)
        c2 = lib.mapnet_launch_count()
        assert c2 - c1 == 2
        pred = torch.empty(B, 6, device="cuda")
        pr._engine(256, 341).forward(x, pred, 0.0, 0)
        c3 = lib.mapnet_launch_count()
        assert c3 - c2 == 44
        post(pred, POSE_M, POSE_S)
        assert lib.mapnet_launch_count() - c3 == 1
    torch.cuda.synchronize()
    loc.close(); pr.close()
