"""Throughput of the GPU input pipeline (SURVEY.md 8f, row f2) on one GPU: Resize(256) -> [ColorJitter] -> ToTensor ->
Normalize over 64 frames of 480x640 (the 7-Scenes frame size), with and without the tuple gather and the jitter.
HBM-bound byte work: algorithmic bytes = uint8 frames in + fp32 tensor out.  usage: python tools/bench_preprocess.py [out.json]"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from geomapnet_b200.data import ImagePipeline, ColorJitterSampler

def main():
    torch.manual_seed(0)
    L, n = 256, 64
    seq = torch.randint(0, 256, (L, 480, 640, 3), dtype=torch.uint8, device="cuda")
    pipe = ImagePipeline([0.5, 0.5, 0.5], [0.25, 0.25, 0.25])
    idx = torch.randint(0, L, (n,), dtype=torch.int32)
    jit = ColorJitterSampler(0.7, 0.7, 0.7, 0.5).sample(n)
    peaks = None
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peaks = json.load(open(p))
    res = {}
    for name, kw in (("resize+normalize", dict(index=None, jitter=None)), ("gather", dict(index=idx, jitter=None)),
                     ("gather+jitter", dict(index=idx, jitter=jit))):
        frames = seq[:n] if kw["index"] is None else seq
        for _ in range(3):
            out = pipe(frames, **kw)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            out = pipe(frames, **kw)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 20
        gb = (n * 480 * 640 * 3 + out.numel() * 4) / 1e9
        res[name] = {"ms": ms, "img_per_s": n / ms * 1e3, "algorithmic_GBps": gb / ms * 1e3}
        print("%-18s %.3f ms  %.0f img/s  %.0f GB/s algorithmic" % (name, ms, n / ms * 1e3, gb / ms * 1e3), flush=True)
    res["note"] = ("64 frames 480x640x3 u8 -> 64x3x256x341 fp32; host index/jitter record upload (a few hundred bytes) is inside the "
                   "timed region; the 64-frame working set (59 MB in, 67 MB out) is about the size of L2, so this is an upper "
                   "bound of what a cold pipeline sees")
    if peaks:
        res["measured_peaks"] = peaks
    if len(sys.argv) > 1:
        json.dump(res, open(sys.argv[1], "w"), indent=1)

if __name__ == "__main__":
    main()
