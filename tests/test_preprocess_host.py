"""Image pre-processing arithmetic (SURVEY.md section 8 row f2) on the CPU: geomapnet_b200/csrc/preprocess_core.h --
the functions the CUDA kernels call -- compiled for the host (tests/_hostpre.cpp) and compared BIT FOR BIT with the
third-party code the reference's transform stack runs (scripts/train.py:119-128): Pillow's 8-bit bilinear resize and
torchvision's ToTensor / Normalize."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PIL = pytest.importorskip("PIL.Image")
T = pytest.importorskip("torchvision.transforms")


@pytest.fixture(scope="module")
def hp():
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libhostpre.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "_hostpre.cpp")])
    return ctypes.CDLL(so)


def run_host(hp, img, size, mean32, std32):
    H, W, _ = img.shape
    Ho, Wo = ctypes.c_int(), ctypes.c_int()
    hp.hp_output_size(H, W, size, ctypes.byref(Ho), ctypes.byref(Wo))
    Ho, Wo = Ho.value, Wo.value
    u8 = np.zeros((Ho, Wo, 3), np.uint8)
    f = np.zeros((3, Ho, Wo), np.float32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    hp.hp_preprocess(p(img), H, W, Ho, Wo, p(mean32), p(std32), p(u8), p(f))
    return u8, f


# (H, W): 7Scenes 480x640, RobotCar-like 960x1280, portrait, square, tiny (upscaling), odd sizes
SIZES = [(480, 640), (960, 1280), (640, 480), (256, 256), (100, 100), (97, 65), (600, 401), (31, 500), (257, 255)]


@pytest.mark.parametrize("hw", SIZES)
def test_resize_totensor_normalize_bit_exact(hp, hw):
    H, W = hw
    rng = np.random.default_rng(H * 1000 + W)
    img = (rng.random((H, W, 3)) * 256).astype(np.uint8)
    img[: H // 4, : W // 4] = 255; img[-(H // 5):, -(W // 5):] = 0        # saturated regions: the clip8 edges
    stats_mean = rng.random(3) * 0.5 + 0.25                               # float64, as np.loadtxt(stats.txt) gives them
    stats_var = rng.random(3) * 0.08 + 0.01
    tf = T.Compose([T.Resize(256), T.ToTensor(), T.Normalize(mean=stats_mean, std=np.sqrt(stats_var))])
    pil = PIL.fromarray(img)
    ref = tf(pil).numpy()
    u8, f = run_host(hp, img, 256, stats_mean.astype(np.float32), np.sqrt(stats_var).astype(np.float32))
    assert f.shape == ref.shape
    ref_u8 = np.asarray(pil.resize((ref.shape[2], ref.shape[1]), PIL.BILINEAR))
    assert np.array_equal(u8, ref_u8), "resized uint8 image differs from Pillow in %d samples" % int((u8 != ref_u8).sum())
    assert np.array_equal(f.view(np.uint32), ref.view(np.uint32)), "float32 output differs, max abs %g" % float(np.abs(f - ref).max())


def test_other_target_sizes_and_python_size_helper(hp):
    from geomapnet_b200.data.preprocess import resize_output_size
    rng = np.random.default_rng(5)
    for (H, W, size) in [(480, 640, 128), (480, 640, 224), (120, 90, 300), (64, 64, 64)]:
        img = (rng.random((H, W, 3)) * 256).astype(np.uint8)
        mean = np.float32([0.5, 0.5, 0.5]); std = np.float32([0.25, 0.25, 0.25])
        ref = T.Compose([T.Resize(size), T.ToTensor(), T.Normalize(mean=mean.tolist(), std=std.tolist())])(PIL.fromarray(img)).numpy()
        u8, f = run_host(hp, img, size, mean, std)
        assert (f.shape[1], f.shape[2]) == resize_output_size(H, W, size) == (ref.shape[1], ref.shape[2])
        assert np.array_equal(f.view(np.uint32), ref.view(np.uint32))


def test_pipeline_rejects_cpu_tensors_and_bad_input():
    from geomapnet_b200.data import ImagePipeline
    pipe = ImagePipeline([0.5, 0.5, 0.5], [0.2, 0.2, 0.2])
    with pytest.raises(RuntimeError, match="no CPU path"):
        pipe(torch.zeros(2, 48, 64, 3, dtype=torch.uint8))
    with pytest.raises(ValueError):
        ImagePipeline([0.5, 0.5, 0.5], [0.2, 0.0, 0.2])
    # mean / std are rounded to float32 the way torchvision's Normalize does
    p2 = ImagePipeline(np.array([0.1, 0.2, 0.3]), np.sqrt(np.array([0.01, 0.02, 0.03])))
    assert p2.mean.dtype == np.float32 and p2.std[1] == np.float32(np.sqrt(0.02))


# ---------------------------------------------------------------------------------------------------------------
# ColorJitter (scripts/train.py:121-126): arithmetic, random draws; MF / MFOnline index arithmetic
# ---------------------------------------------------------------------------------------------------------------
def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def test_hsv_conversions_bit_exact_over_all_colours(hp):
    """every 8-bit RGB triple through Pillow's RGB->HSV and every HSV triple through HSV->RGB"""
    g = np.arange(256, dtype=np.uint8)
    cube = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(4096, 4096, 3).copy()
    out = np.zeros_like(cube)
    hp.hj_rgb2hsv(_p(cube), _p(out), ctypes.c_longlong(4096 * 4096))
    assert np.array_equal(out, np.asarray(PIL.fromarray(cube).convert("HSV")))
    hp.hj_hsv2rgb(_p(cube), _p(out), ctypes.c_longlong(4096 * 4096))
    assert np.array_equal(out, np.asarray(PIL.fromarray(cube, "HSV").convert("RGB")))


@pytest.mark.parametrize("op", [0, 1, 2, 3])
def test_jitter_adjustments_bit_exact(hp, op):
    import torchvision.transforms.functional as F
    rng = np.random.default_rng(op)
    img = (rng.random((97, 131, 3)) * 256).astype(np.uint8)
    img[:20, :20] = 255; img[-10:] = 0
    pil = PIL.fromarray(img)
    fn = [F.adjust_brightness, F.adjust_contrast, F.adjust_saturation, F.adjust_hue][op]
    factors = [0.0, 0.3, 0.7, 1.0, 1.35, 2.0] if op < 3 else [-0.5, -0.31, -0.001, 0.0, 0.12, 0.5]
    factors += [float(np.float32(rng.uniform(0.3, 1.7) if op < 3 else rng.uniform(-0.5, 0.5))) for _ in range(6)]
    for f in factors:
        f32 = float(np.float32(f))
        a = img.copy()
        hp.hj_apply(_p(a), ctypes.c_longlong(97 * 131), op, ctypes.c_float(f32))
        assert np.array_equal(a, np.asarray(fn(pil, f32))), (op, f)


def test_color_jitter_sampler_draws_what_torchvision_draws(hp):
    """same torch seed -> the same order and factors as ColorJitter.get_params, and the composed result on an image is
    what the reference's transform (scripts/train.py:123-124: brightness = contrast = saturation = cj, hue = 0.5) gives"""
    from geomapnet_b200.data import ColorJitterSampler
    cj = 0.7
    tv = T.ColorJitter(brightness=cj, contrast=cj, saturation=cj, hue=0.5)
    rng = np.random.default_rng(3)
    imgs = (rng.random((5, 64, 48, 3)) * 256).astype(np.uint8)
    torch.manual_seed(11)
    ref = [np.asarray(tv(PIL.fromarray(im))) for im in imgs]
    torch.manual_seed(11)
    rec = ColorJitterSampler(cj, cj, cj, 0.5).sample(5).numpy()
    order = rec.view(np.int32).reshape(5, 8)[:, :4]
    factor = rec.view(np.float32).reshape(5, 8)[:, 4:]
    torch.manual_seed(11)
    for i in range(5):
        fn_idx, b, c, s, h = T.ColorJitter.get_params(tv.brightness, tv.contrast, tv.saturation, tv.hue)
        assert list(order[i]) == fn_idx.tolist()
        assert np.array_equal(factor[i], np.float32([b, c, s, h]))
        a = imgs[i].copy()
        for op in order[i]:
            hp.hj_apply(_p(a), ctypes.c_longlong(64 * 48), int(op), ctypes.c_float(float(factor[i][op])))
        assert np.array_equal(a, ref[i]), i
    # disabled adjustments consume no random numbers and stay neutral
    torch.manual_seed(5)
    r0 = ColorJitterSampler(0.0, 0.2, 0.0, 0.0).sample(1).numpy().view(np.float32).reshape(8)[4:]
    assert r0[0] == 1.0 and r0[2] == 1.0 and r0[3] == 0.0 and 0.8 <= r0[1] <= 1.2


def test_tuple_indices_match_reference_mf(golden_dir):
    """tuples.mf_indices against MF.get_indices / __len__ of the reference (dataset_loaders/composite.py:60-75,
    105-109), as stored in tests/golden/live_reference.npz by oracle/make_goldens.py."""
    from geomapnet_b200.data import tuples
    L = np.load(os.path.join(golden_dir, "live_reference.npz"))
    cases = L["mf_cases"]
    seen = set()
    for row in cases:
        steps, skip, length, nodup, index = (int(v) for v in row[:5])
        n = tuples.mf_len(length, steps, skip, bool(nodup))
        assert n == (length - (steps - 1) * skip if nodup else length)
        got = tuples.mf_indices(index, length, steps, skip, bool(nodup))
        assert np.array_equal(row[5:5 + steps], got), (steps, skip, length, nodup, index)
        seen.add((steps, skip, length, nodup))
    assert len(seen) == 10
    # variable_skip consumes np.random exactly as the reference does
    np.random.seed(3); got = tuples.mf_indices(250, 500, 5, 7, variable_skip=True)
    assert np.array_equal(L["mf_variable_skip"], got)
    # MFOnline: train tuple | validation tuple (no_duplicates), both modulo their dataset length
    tr, va = tuples.mfonline_indices(123, 100, 60, 5, 10)
    assert np.array_equal(tr, tuples.mf_indices(123 % 100, 100, 5, 10)) and \
        np.array_equal(va, tuples.mf_indices(123 % (60 - 40), 60, 5, 10, no_duplicates=True))
    flat = tuples.batch_frame_indices([0, 7, 999], 1000, 3, 10)
    assert flat.dtype == np.int32 and flat.tolist() == [0, 0, 10, 0, 7, 17, 989, 999, 999]
