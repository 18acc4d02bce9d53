"""Micro-benchmark of the wgmma conv engines per ResNet-34 layer shape (GPU box).
usage: python tools/bench_conv.py [B]   (env MAPNET_TC_BN=64|128 forces the N tile, MAPNET_TC_DEBUG skips parts of the work)
Then the stride-1 3x3 wgrads on every wgrad engine (taps/BN: 0 = per-tap k_tc_wgrad, 3 or 9 = k_halo_wgrad)."""
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

# wgrad of the stride-1 3x3 convs on each engine with the same K partition: the per-tap engine (taps 0) and the halo
# engines (3 or 9 filter taps per CTA), timed in turn for 3 rounds; the median per engine, * marks the planner's choice
import json
print("wgrad engines, B = %d: median of 3 alternating rounds of 20 launches (* = planned)" % B, flush=True)
for name, H, W, Ci, Co, k, s in shapes:
    if k != 3 or s != 1:
        continue
    buf = ctypes.create_string_buffer(1 << 17)
    assert L.mapnet_test_plan_describe(2, B, H, W, Ci, Co, k, s, 0, buf, len(buf)) == 0
    P = json.loads(buf.value.decode())["wgrad"]
    eng = P["engine"]
    x = torch.randn(B, H, W, Ci, device="cuda").bfloat16()
    dy = torch.randn(B, H, W, Co, device="cuda").bfloat16()
    dw = torch.zeros(Co, 9, Ci, device="cuda")
    flops = 2.0 * B * H * W * Co * 9 * Ci
    engines = [(0, 0)] + [(t, bn) for t, bn in ((3, 64), (3, 128), (9, 64)) if Co % bn == 0]
    times = {e: [] for e in engines}
    for _ in range(3):
        for t, bn in engines:
            ms = ctypes.c_float()
            rc = L.mapnet_test_wgrad(t, bn, B, H, W, Ci, Co, k, s, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), 20,
                                     ctypes.byref(ms))
            assert rc == 0, L.mapnet_last_error().decode()
            times[(t, bn)].append(ms.value)
    cells = []
    for t, bn in engines:
        m = sorted(times[(t, bn)])[1]
        bn = bn if t else P["BN"]
        mark = "*" if (t, bn) == (eng["taps"], eng["BN"]) else " "
        cells.append("%s%d/%-3d %6.1fus %4.0fTF" % (mark, t, bn, m * 1000, flops / (m * 1e-3) / 1e12))
    print("%-26s %s" % (name, " | ".join(cells)), flush=True)
