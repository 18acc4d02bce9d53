"""Host-side checks of the fp8 inference engine (no GPU needed): the emulation's e4m3 quantizer against a from-scratch
reference, the power-of-two scale rule, the fp8 arena, argument errors before any device work, the exported symbols,
and the build: the e4m3 wgmma kernels compile without spills into QGMMA / TMA / mbarrier code while the six bf16 conv
engines keep their names and register counts."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from fp8_emulation import e4m3_rne_satfinite_numpy, pow2_scale, quantize_e4m3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "geomapnet_b200", "csrc", "_obj", "conv_tc.o.log")


@pytest.fixture(scope="module")
def L():
    from geomapnet_b200 import build, _lib
    build.build(verbose=False)
    return _lib.lib()


# ---------------------------------------------------------------------------------------------------------------------
# quantizer and scale rule
# ---------------------------------------------------------------------------------------------------------------------
def test_quantizer_matches_a_from_scratch_e4m3_rne_satfinite():
    # a dense sweep of fp32 bit patterns over every binade e4m3 reaches and beyond (2^-12 .. 2^10), both signs: every
    # 2^12-th pattern plus the neighbours of every e4m3 value and of every midpoint between two (ties and their
    # neighbours), the subnormals, +-448 and the overflow region
    sweep = np.arange(0x39800000, 0x44800000, 1 << 12, dtype=np.uint32).view(np.float32)
    grid = np.array(sorted(set(float(v) for v in torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).float()
                               .numpy() if np.isfinite(v) and v >= 0)), dtype=np.float32)
    mids = ((grid[1:].astype(np.float64) + grid[:-1]) / 2).astype(np.float32)
    pts = np.concatenate([grid, mids, [448.0, 464.0, 479.0, 480.0, 500.0, 1e6, 3e38, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -11]])
    near = np.concatenate([np.nextafter(pts.astype(np.float32), np.float32(np.inf)),
                           np.nextafter(pts.astype(np.float32), np.float32(0)), pts.astype(np.float32)])
    x = np.concatenate([sweep, near, [0.0]]).astype(np.float32)
    x = np.concatenate([x, -x])
    ref = e4m3_rne_satfinite_numpy(x)
    got = quantize_e4m3(torch.from_numpy(x)).numpy()
    assert np.array_equal(ref, got, equal_nan=True), x[np.flatnonzero(ref != got)[:8]]
    # the properties the comparison rests on: ties to even, saturation instead of NaN, subnormals
    q = lambda v: float(quantize_e4m3(torch.tensor([v], dtype=torch.float32))[0])
    assert q(500.0) == 448.0 and q(-1e30) == -448.0 and q(464.0) == 448.0
    assert q(17.0) == 16.0 and q(19.0) == 20.0               # midpoints: 16 = 1.000b * 2^4 (even), 20 = 1.010b * 2^4
    assert q(2.0 ** -9) == 2.0 ** -9 and q(2.0 ** -10) == 0.0 and q(3 * 2.0 ** -10) == 2.0 ** -8
    assert np.isnan(q(float("nan")))
    # torch's own cast does not saturate: the reason the quantizer clamps first
    assert torch.isnan(torch.tensor([500.0]).to(torch.float8_e4m3fn).float()).all()


def test_scale_rule_is_a_power_of_two_that_fits_amax():
    assert pow2_scale(0.0) == 1.0
    rng = np.random.default_rng(0)
    vals = np.concatenate([rng.lognormal(0, 6, 2000).astype(np.float32), [448.0, 448.0 * 2 ** -3, 449.0, 1e-30, 3e38]])
    for a in vals:
        s = pow2_scale(a)
        m, _ = np.frexp(s)
        assert m == 0.5, (a, s)                              # a power of two
        assert 448.0 * s >= a and 448.0 * s / 2 < a, (a, s)  # the smallest one with amax / s <= 448
    assert pow2_scale(448.0) == 1.0 and pow2_scale(449.0) == 2.0 and pow2_scale(224.0) == 0.5


# ---------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------
def _arena_from_shapes(B, H, W, feat_dim=2048):
    """bf16 stem image and stem output, three rotating e4m3 block tensors, the bf16 downsample output, the head, and the
    scale slots (33 amax, 33 scales, 33 inverses, the pool's 128-entry map)"""
    conv = lambda n, k, s, p: (n + 2 * p - k) // s + 1
    hc, wc = conv(H, 7, 2, 3), conv(W, 7, 2, 3)
    hp, wp = conv(hc, 3, 2, 1), conv(wc, 3, 2, 1)
    wsp = (wc + 6) // 4 * 4
    a0 = (hc + 3) * wsp * 16 * 2
    y0 = hc * wc * 64 * 2
    act = hp * wp * 64
    h2, w2 = conv(hp, 3, 2, 1), conv(wp, 3, 2, 1)
    ds = h2 * w2 * 128 * 2
    head = (512 + 3 * feat_dim) * 4
    return B * (a0 + y0 + 3 * act + ds + head) + 4 * (3 * 33 + 128)


def test_fp8_arena_matches_the_shapes_and_is_below_bf16(L):
    from geomapnet_b200._lib import PREC, INFER_PREC
    for B, H, W in ((1, 256, 256), (64, 256, 256), (8, 256, 341)):
        got = L.mapnet_infer_arena_bytes(B, H, W, INFER_PREC["fp8"])
        assert got == _arena_from_shapes(B, H, W), (B, H, W, got)
        assert got < L.mapnet_infer_arena_bytes(B, H, W, PREC["bf16"])
    print("fp8 inference arena at 256x256: %.2f MB per image" % (L.mapnet_infer_arena_bytes(64, 256, 256, 4) / 64e6))


def test_fp8_argument_errors_before_any_device_work(L):
    from geomapnet_b200._lib import PREC, INFER_PREC
    assert INFER_PREC["fp8"] == 4 and "fp8" not in PREC       # training precisions are unchanged
    h = ctypes.c_void_p()
    assert L.mapnet_trunk_create(ctypes.byref(h), 0, 256, 256, 2048, 4) != 0      # inference only
    assert not h.value and b"precision" in L.mapnet_last_error()
    assert L.mapnet_infer_calibrate(None, None, 1, None) != 0
    assert L.mapnet_infer_act_scales(None, None, 0) != 0
    # k = 5 and a calibration pass without an amax slot are refused before a device is looked for
    assert L.mapnet_test_conv_fp8(1, 8, 8, 64, 64, 5, 1, 1, 1, 1, 1, None, None, None, 0, 1, None, None) != 0
    assert L.mapnet_test_conv_fp8(1, 8, 8, 64, 64, 3, 1, 1, 1, 1, 1, None, None, None, 8, None, None, None) != 0


def test_fp8_symbols_are_exported(L):
    from geomapnet_b200 import _lib
    for name in ("mapnet_infer_calibrate", "mapnet_infer_act_scales", "mapnet_test_conv_fp8"):
        assert name in _lib.EXPORTED and hasattr(L, name)
    hdr = open(os.path.join(ROOT, "include", "mapnet_b200.h")).read()
    assert re.search(r"#define MAPNET_PREC_FP8 4\b", hdr)


# ---------------------------------------------------------------------------------------------------------------------
# build evidence
# ---------------------------------------------------------------------------------------------------------------------
def _ptxas_entries(text):
    """{mangled kernel name: (registers, spill store bytes, spill load bytes)} from the ptxas -v log"""
    out = {}
    for m in re.finditer(r"Compiling entry function '(\w+)'[^\n]*\n(?:[^\n]*Function properties[^\n]*\n)?\s*(\d+) bytes stack "
                         r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) registers", text):
        out[m.group(1)] = (int(m.group(5)), int(m.group(3)), int(m.group(4)))
    return out


def test_fp8_kernels_compile_without_spills_and_bf16_engines_are_unchanged(L):
    ent = _ptxas_entries(open(LOG).read())
    f8 = {n: v for n, v in ent.items() if "k_f8_conv" in n}
    # k_f8_conv<BN, KB>: N tiles of 64 and 128, 128- and 64-byte k-blocks
    assert {re.search(r"k_f8_convILi\d+ELi\d+E", n).group(0) for n in f8} == \
        {"k_f8_convILi%dELi%dE" % (bn, kb) for bn in (64, 128) for kb in (64, 128)}, sorted(f8)
    for n, (regs, st, ld) in f8.items():
        print(n[:40], regs, "registers")
        assert st == 0 and ld == 0, (n, st, ld)
    # the six bf16 engines: same names, same register counts as before the fp8 engine was added
    regs = {re.search(r"k_tc_(conv|wgrad)ILi\d+E(Lb[01]E)?", n).group(0): v[0] for n, v in ent.items()
            if "k_tc_conv" in n or "k_tc_wgrad" in n}
    assert regs == {"k_tc_convILi64ELb0E": 148, "k_tc_convILi128ELb0E": 166, "k_tc_convILi64ELb1E": 144,
                    "k_tc_convILi128ELb1E": 163, "k_tc_wgradILi64E": 74, "k_tc_wgradILi128E": 95}, regs


def test_fp8_sass_uses_e4m3_wgmma_tma_and_mbarriers(L):
    from geomapnet_b200 import build
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    r = subprocess.run([exe, "-sass", build.OUT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-1000:]
    bodies, name = {}, None
    for line in r.stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            bodies[name] = []
        elif name:
            bodies[name].append(line)
    f8 = {n: "\n".join(b) for n, b in bodies.items() if "k_f8_conv" in n}
    assert len(f8) == 4, sorted(f8)
    for n, b in f8.items():
        bn = re.search(r"k_f8_convILi(\d+)E", n).group(1)
        # FP8 wgmma is QGMMA in SASS (bf16 / fp16 wgmma is HGMMA)
        assert ("QGMMA.64x%sx32.F32.E4M3.E4M3" % bn) in b, n
        assert "HGMMA" not in b and not re.search(r"\bHMMA\.", b), n
        assert "UTMALDG.4D" in b and "UTMALDG.2D" in b, n
        assert "SYNCS.ARRIVE.TRANS64" in b and "WARPGROUP.DEPBAR" in b, n
