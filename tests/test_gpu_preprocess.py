"""GPU run of the input-pipeline kernels (geomapnet_b200/csrc/preprocess.cu, SURVEY.md section 8 row f2) against Pillow /
torchvision, bit for bit: Resize(256) -> [ColorJitter] -> ToTensor -> Normalize (scripts/train.py:119-128) and the
MF tuple gather (dataset_loaders/composite.py:60-97)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("hw,n", [((480, 640), 8), ((97, 65), 3), ((600, 401), 2), ((100, 100), 5)])
def test_gpu_pipeline_matches_pillow_and_torchvision(hw, n):
    from PIL import Image
    import torchvision.transforms as T
    from geomapnet_b200.data import ImagePipeline
    H, W = hw
    rng = np.random.default_rng(H + W + n)
    frames = (rng.random((n, H, W, 3)) * 256).astype(np.uint8)
    stats_mean = rng.random(3) * 0.5 + 0.25
    stats_var = rng.random(3) * 0.08 + 0.01
    tf = T.Compose([T.Resize(256), T.ToTensor(), T.Normalize(mean=stats_mean, std=np.sqrt(stats_var))])
    ref = torch.stack([tf(Image.fromarray(f)) for f in frames]).numpy()
    pipe = ImagePipeline(stats_mean, np.sqrt(stats_var))
    out, u8 = pipe(torch.from_numpy(frames).cuda(), return_u8=True)
    torch.cuda.synchronize()
    ref_u8 = np.stack([np.asarray(Image.fromarray(f).resize((ref.shape[3], ref.shape[2]), Image.BILINEAR)) for f in frames])
    assert np.array_equal(u8.cpu().numpy(), ref_u8)
    got = out.cpu().numpy()
    assert got.shape == ref.shape and np.array_equal(got.view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("hw", [(480, 640), (120, 90)])
def test_gpu_tuple_gather_and_color_jitter_match_the_reference_transform(hw):
    """A [N,T] minibatch of MF tuples cut from a device-resident sequence with ColorJitter on: the same frames through
    the reference's transform stack (scripts/train.py:119-128 with color_jitter = 0.7) image by image, same torch seed.
    Bit-identical uint8 image after the jitter and bit-identical float32 tensor."""
    from PIL import Image
    import torchvision.transforms as T
    from geomapnet_b200.data import ImagePipeline, ColorJitterSampler, tuples
    H, W = hw
    rng = np.random.default_rng(H)
    L, steps, skip, cj = 40, 3, 10, 0.7
    seq = (rng.random((L, H, W, 3)) * 256).astype(np.uint8)
    seq[3, : H // 3] = 255; seq[17, :, : W // 4] = 0
    stats_mean, stats_var = rng.random(3) * 0.5 + 0.25, rng.random(3) * 0.08 + 0.01
    idx = tuples.batch_frame_indices([0, 5, 19, 39], L, steps, skip)          # [N*T] frame numbers, clipped at the ends
    assert idx.tolist()[:3] == [0, 0, 10] and idx.tolist()[-3:] == [29, 39, 39]
    tf = T.Compose([T.Resize(256), T.ColorJitter(brightness=cj, contrast=cj, saturation=cj, hue=0.5)])
    tail = T.Compose([T.ToTensor(), T.Normalize(mean=stats_mean, std=np.sqrt(stats_var))])
    torch.manual_seed(21)
    ref_u8 = [tf(Image.fromarray(seq[i])) for i in idx]
    ref = torch.stack([tail(im) for im in ref_u8]).numpy()
    torch.manual_seed(21)
    jit = ColorJitterSampler(cj, cj, cj, 0.5).sample(len(idx))
    pipe = ImagePipeline(stats_mean, np.sqrt(stats_var))
    out, u8 = pipe(torch.from_numpy(seq).cuda(), index=idx, jitter=jit, return_u8=True)
    torch.cuda.synchronize()
    assert np.array_equal(u8.cpu().numpy(), np.stack([np.asarray(im) for im in ref_u8]))
    got = out.cpu().numpy()
    assert got.shape == ref.shape and np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    # the gather alone (no jitter) equals pre-processing the gathered frames
    a = pipe(torch.from_numpy(seq).cuda(), index=idx)
    b = pipe(torch.from_numpy(seq[idx]).cuda())
    assert torch.equal(a, b)
    # MapNet's input layout: [N, T, 3, H', W'] is a view of the result
    x = out.view(4, steps, 3, out.shape[2], out.shape[3])
    assert x.is_contiguous()


def test_gpu_pipeline_throughput_is_reported():
    """HBM-bound byte work: algorithmic bytes = uint8 frame in + fp32 tensor out.  Not a pass/fail bar -- prints the GB/s
    tools/bench_preprocess.py records under profiles/ and checks the launch count."""
    from geomapnet_b200 import _lib
    from geomapnet_b200.data import ImagePipeline
    frames = torch.randint(0, 256, (64, 480, 640, 3), dtype=torch.uint8, device="cuda")
    pipe = ImagePipeline([0.5, 0.5, 0.5], [0.25, 0.25, 0.25])
    pipe(frames)
    torch.cuda.synchronize()
    lc = _lib.lib().mapnet_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        out = pipe(frames)
    e1.record()
    torch.cuda.synchronize()
    assert (_lib.lib().mapnet_launch_count() - lc) == 20          # two kernels per call
    ms = e0.elapsed_time(e1) / 10
    gb = (frames.numel() + out.numel() * 4) / 1e9
    print("input-pipeline 64 x 480x640 -> 256x341: %.3f ms, %.0f img/s, %.1f GB/s algorithmic" % (ms, 64 / ms * 1e3, gb / ms * 1e3))
