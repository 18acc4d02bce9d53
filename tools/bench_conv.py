"""Micro-benchmark of the wgmma conv engines per ResNet-34 layer shape (GPU box).
usage: python tools/bench_conv.py [B]   (env MAPNET_TC_BN=64|128 forces the N tile, MAPNET_TC_DEBUG skips parts of the work)"""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from geomapnet_b200 import _lib
B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
L = _lib.lib()
shapes = [("layer1 3x3 64->64", 64, 64, 64, 64, 3, 1), ("layer2 3x3 128->128", 32, 32, 128, 128, 3, 1),
          ("layer3 3x3 256->256", 16, 16, 256, 256, 3, 1), ("layer4 3x3 512->512", 8, 8, 512, 512, 3, 1),
          ("layer2.0 3x3s2 64->128", 64, 64, 64, 128, 3, 2), ("stem gemm 192->64", 128, 128, 192, 64, 1, 1)]
for name, H, W, Ci, Co, k, s in shapes:
    Ho = (H + 2 * ((k - 1) // 2) - k) // s + 1
    x = torch.randn(B, H, W, Ci, device="cuda").bfloat16()
    dy = torch.randn(B, Ho, Ho, Co, device="cuda").bfloat16()
    w = (torch.randn(Co, k, k, Ci, device="cuda") * 0.05).bfloat16()
    wd = (torch.randn(Ci, k, k, Co, device="cuda") * 0.05).bfloat16()
    flops = 2.0 * B * Ho * Ho * Co * k * k * Ci
    res = []
    for kind, a, b_, wm, out in ((0, x, None, w, torch.empty_like(dy)), (1, dy, None, wd, torch.empty_like(x)),
                                (2, x, dy, None, torch.zeros(Co, k, k, Ci, device="cuda"))):
        if kind == 1 and name.startswith("stem"):
            res.append("   -   "); continue
        ms = ctypes.c_float()
        rc = L.mapnet_bench_conv(kind, B, H, W, Ci, Co, k, s, a.data_ptr(), b_.data_ptr() if b_ is not None else None,
                                 wm.data_ptr() if wm is not None else None, out.data_ptr(), 20, ctypes.byref(ms))
        if rc != 0:
            res.append("ERR %s" % L.mapnet_last_error().decode()[:60]); continue
        res.append("%6.1fus %5.0fTF" % (ms.value * 1000, flops / (ms.value * 1e-3) / 1e12))
    print("%-26s fprop %s | dgrad %s | wgrad %s" % (name, res[0], res[1], res[2]), flush=True)
