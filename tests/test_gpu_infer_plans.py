"""The inference conv engines (csrc/conv_tc.cu) one launch at a time, at the tile plans the inference benchmarks run,
checked element by element against float64: k_f8_conv (fp8, with every epilogue variant infer.cu uses and its EPI_AMAX
calibration pass) and k_tc_conv's eval-mode affine epilogue (EPI_AFFINE) in bf16 and strict (tc_split) mode.

Cases are the distinct ResNet-34 conv geometries behind a 256x256 frame at B = 1, 8 and 64 (bench_infer*) and a 256x341
frame (Resize(256) of 480x640: ragged widths 171, 86, 43, 22 and 11) at B = 1 and 64 (bench_localize, bench_sample),
plus fp8 layer1 at B = 256 (2 048 M tiles x 4: about 62 work items per persistent CTA).  Each conv runs with the
epilogue the schedule gives it: fp8 conv1 ReLU + e4m3 out; conv2 e4m3 residual x s_res (identity blocks) or bf16
residual (downsampling blocks), ReLU, e4m3 out; the 1x1/s2 downsample bf16 out without ReLU.  Affine: the 7x7 stem
(space-to-depth 4x1 conv, ReLU), conv1 (ReLU), the downsample (no ReLU), conv2 (residual, ReLU); strict mode stores
conv1 / conv2 outputs as fp16 hi/lo planes (the next conv's operand), reads an identity residual as planes and a
downsample's as fp32, and stores the stem and the downsample in fp32.  A case states the plan it expects (N tile BN,
work items against the 132 persistent CTAs, fp8 k-block bytes) and asserts it from mapnet_test_plan_describe before
launching; `test_case_list_covers_the_inference_plans` (host only) checks that the list still reaches the plans that
matter.

Reference.  float64 on the GPU: F.conv2d on the decoded stored operands (e4m3 and bf16 decode exactly; strict mode
takes the fp32 inputs), then the epilogue.  S = sum |a*b| per element from the same conv on |a| and |b|, times |scale|.

Per-element bound.  |got - ref| <= eps_store(|ref|) + (1 + u_store) * E, E = |scale| * gamma * S + E_epi (+ E_res):
  * gamma, bf16 / tc_split: a wgmma instruction adds 16 exact products and the fp32 accumulation truncates, one ulp
    (TRUNC = 2^-23) relative to the running sum, which is at most S; K / 16 instructions, K = taps * channels (strict:
    four times longer, the hi/lo products).  Strict mode cuts each operand into fp16 hi + lo planes,
    x = (hi + lo)(1 + d), |d| <= SPLIT = 2^-22 for |x| in [2^-3, 2^3] (where the operands are drawn), so a product
    carries 2 SPLIT + SPLIT^2.
  * gamma, fp8: e4m3 products are exact, but how Hopper's e4m3 wgmma accumulates is not documented, so the per-
    instruction error is measured: gamma = (K / 32 instructions) * U_F8ACC.  `test_fp8_accumulation_per_instruction`
    runs a coherent case (non-negative operands, so every running sum grows monotonically and the errors add up) and
    reads the accumulator back exactly: one pixel value per output channel is cancelled by the epilogue's shift, so the
    bf16 output holds the accumulation error itself.  Measured on an H100 80GB HBM3 (700 W power limit): max |acc - T|
    / ((K/32) S) = 5.9e-4 (Ci 512, K = 4608) and 4.9e-4 (Ci 64, K = 576), no error positive (acc <= T), to a
    resolution of 2.4e-6.  That is about 2^-11 of S per instruction, 4 000 times fp32's truncation (TRUNC = 2^-23).
    U_F8ACC is 2x the largest measurement: the coherent running sums grow from 0 to S, and the bound charges every
    instruction against S.
  * E_epi: the epilogue's fp32 arithmetic acc * scale + shift (+ residual), at most four roundings (the product, the
    shift, the residual's hi + lo, its add) of U_FP32 = 2^-24 of |scale| S + |shift| + |residual|.  The residual's own
    split (strict identity residuals, cut into planes from fp32): E_res = SPLIT |r| + 2^-25.  ReLU is 1-Lipschitz.
  * eps_store: bf16 rounds to 8 significant bits, u_store = 2^-8 |ref|; e4m3 to 4, 2^-4 |ref|, plus half its subnormal
    quantum 2^-10 s_out (the output scale s_out is a power of two, f / s_out is exact); fp32 outputs are stored as
    computed; hi/lo planes keep 22 bits, SPLIT |ref| + 2^-25 (half lo's subnormal quantum).
Every case prints max(err / bound).  The fp8 bound is wide where gamma * S dominates (layer4: K = 4608), so each fp8
case also keeps test_gpu_infer_fp8's check that few outputs differ from the exactly rounded float64 result: an
accumulation error moves an output only when it crosses a rounding midpoint, a layout or tile error moves most.

Every element is written exactly once: outputs are NaN before the launch (bf16 NaN, e4m3fn code 0x7F, fp32 NaN, fp16
NaN planes) and a NaN left behind fails the check.  The EPI_AMAX pass leaves the output bytes untouched, and its amax
equals max |f| of the float64 reference within the largest bound without the store term.  A failure names the first
wrong element, its work item, CTA and which of that CTA's tiles it is, and how many wrong tiles are a CTA's first.
"""
import ctypes
import json
import time
import zlib

import pytest
import torch
import torch.nn.functional as F

from fp8_emulation import pow2_scale, quantize_e4m3
from geomapnet_b200 import _lib
from test_gpu_infer_fp8 import MISMATCH_FRAC

NSM = 132
U_BF16 = 2.0 ** -8
U_FP32 = 2.0 ** -24
U_E4M3 = 2.0 ** -4
E4M3_HALF_SUB = 2.0 ** -10     # half of e4m3's subnormal quantum 2^-9
PLANE_HALF_SUB = 2.0 ** -25    # half of fp16's subnormal quantum 2^-24
TRUNC = 2.0 ** -23             # one ulp per truncating bf16 / fp16 wgmma accumulation
SPLIT = 2.0 ** -22             # hi/lo fp16 split of one value
U_F8ACC = 1.2e-3               # e4m3 wgmma accumulation, per instruction, relative to S (2x the H100 measurement)
N_EPI = 4                      # fp32 roundings of the affine epilogue
S_RES = 0.25                   # power-of-two scale of an e4m3 residual

# (name, batch, frame H, frame W) of the inference benchmarks
CONFIGS = [("256x256.b1", 1, 256, 256), ("256x256.b8", 8, 256, 256), ("256x256.b64", 64, 256, 256),
           ("256x341.b1", 1, 256, 341), ("256x341.b64", 64, 256, 341)]


def resnet34_convs(H, W):
    """(role, (Hi, Wi, Ci, Co, k, stride)) of the distinct conv launches of ResNet-34 on an H x W frame; the stem's Hi x
    Wi is the frame.  layerN.1.conv2 stands for every identity block's conv2 (and, in shape, its conv1)."""
    h, w = (H - 1) // 2 + 1, (W - 1) // 2 + 1          # stem 7x7/s2
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1          # max pool 3x3/s2
    out = [("stem", (H, W, 3, 64, 7, 2)), ("layer1.0.conv1", (h, w, 64, 64, 3, 1)),
           ("layer1.0.conv2", (h, w, 64, 64, 3, 1))]
    c = 64
    for n, co in ((2, 128), (3, 256), (4, 512)):
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        out += [("layer%d.0.conv1" % n, (h, w, c, co, 3, 2)), ("layer%d.0.downsample" % n, (h, w, c, co, 1, 2)),
                ("layer%d.0.conv2" % n, (ho, wo, co, co, 3, 1)), ("layer%d.1.conv2" % n, (ho, wo, co, co, 3, 1))]
        h, w, c = ho, wo, co
    return out


def epilogue(engine, role):
    """the epilogue variant infer.cu runs this conv with (None: not run on this engine, or the same launch as another
    case)"""
    identity = role.startswith("layer1.") or ".1." in role      # conv2 whose residual is the block input
    if engine == "fp8":                                         # the stem stays on the bf16 engine
        return None if role == "stem" else "relu_f8out" if role.endswith("conv1") else "bf16out" \
            if role.endswith("downsample") else "f8res" if identity else "bf16res"
    if engine == "bf16":
        if ".1." in role:
            return None
        return "plain" if role.endswith("downsample") else "res_relu" if role.endswith("conv2") else "relu"
    return "relu_f32out" if role == "stem" else "relu_hout" if role.endswith("conv1") else "f32out" \
        if role.endswith("downsample") else "hres_hout" if identity else "f32res_hout"


# (mapnet_test_conv_fp8 / mapnet_test_conv_affine flags, residual kind, output kind)
F8_EPI = {"relu_f8out": (1 | 4, None, "e4m3"), "f8res": (1 | 2 | 4, "e4m3", "e4m3"), "bf16res": (1 | 4, "bf16", "e4m3"),
          "bf16out": (0, None, "bf16")}
AFF_EPI = {"relu": (1, None, "bf16"), "plain": (0, None, "bf16"), "res_relu": (1, "bf16", "bf16"),
           "relu_f32out": (1, None, "fp32"), "relu_hout": (1 | 4, None, "planes"), "f32out": (0, None, "fp32"),
           "f32res_hout": (1 | 4, "fp32", "planes"), "hres_hout": (1 | 2 | 4, "planes", "planes")}

# strict mode: every role at 256x256 B = 64, a subset elsewhere
STRICT = {"256x256.b64": None,
          "256x341.b64": {"stem", "layer1.0.conv2", "layer3.0.conv1", "layer3.0.downsample", "layer3.0.conv2",
                          "layer4.1.conv2"},
          "256x341.b1": {"layer2.1.conv2", "layer4.0.conv1"}}


def _cases():
    f8, aff = [], []
    for cfg, B, H, W in CONFIGS:
        for role, (hi, wi, ci, co, k, s) in resnet34_convs(H, W):
            geom = (B, hi, wi, ci, co, k, s)
            if epilogue("fp8", role):
                f8.append(("fp8", cfg, role, geom, epilogue("fp8", role)))
            if epilogue("bf16", role):
                aff.append(("bf16", cfg, role, geom, epilogue("bf16", role)))
            if cfg in STRICT and (STRICT[cfg] is None or role in STRICT[cfg]):
                aff.append(("tc_split", cfg, role, geom, epilogue("tc_split", role)))
    f8.append(("fp8", "256x256.b256", "layer1.0.conv2", (256, 64, 64, 64, 64, 3, 1), "f8res"))
    return f8, aff


F8_CASES, AFF_CASES = _cases()


def case_id(c):
    return "%s-%s.%s" % (c[0], c[1], c[2])


# the plan each case expects: (BN, work items) and, fp8, the k-block bytes
PLANS = {"fp8-256x256.b1.layer1.0.conv1": (64, 32, 64), "fp8-256x256.b1.layer1.0.conv2": (64, 32, 64),
         "fp8-256x256.b1.layer2.0.conv1": (64, 16, 64), "fp8-256x256.b1.layer2.0.downsample": (64, 16, 64),
         "fp8-256x256.b1.layer2.0.conv2": (64, 16, 128), "fp8-256x256.b1.layer2.1.conv2": (64, 16, 128),
         "fp8-256x256.b1.layer3.0.conv1": (64, 8, 128), "fp8-256x256.b1.layer3.0.downsample": (64, 8, 128),
         "fp8-256x256.b1.layer3.0.conv2": (64, 8, 128), "fp8-256x256.b1.layer3.1.conv2": (64, 8, 128),
         "fp8-256x256.b1.layer4.0.conv1": (64, 8, 128), "fp8-256x256.b1.layer4.0.downsample": (64, 8, 128),
         "fp8-256x256.b1.layer4.0.conv2": (64, 8, 128), "fp8-256x256.b1.layer4.1.conv2": (64, 8, 128),
         "fp8-256x256.b8.layer1.0.conv1": (64, 256, 64), "fp8-256x256.b8.layer1.0.conv2": (64, 256, 64),
         "fp8-256x256.b8.layer2.0.conv1": (64, 128, 64), "fp8-256x256.b8.layer2.0.downsample": (64, 128, 64),
         "fp8-256x256.b8.layer2.0.conv2": (64, 128, 128), "fp8-256x256.b8.layer2.1.conv2": (64, 128, 128),
         "fp8-256x256.b8.layer3.0.conv1": (64, 64, 128), "fp8-256x256.b8.layer3.0.downsample": (64, 64, 128),
         "fp8-256x256.b8.layer3.0.conv2": (64, 64, 128), "fp8-256x256.b8.layer3.1.conv2": (64, 64, 128),
         "fp8-256x256.b8.layer4.0.conv1": (64, 32, 128), "fp8-256x256.b8.layer4.0.downsample": (64, 32, 128),
         "fp8-256x256.b8.layer4.0.conv2": (64, 32, 128), "fp8-256x256.b8.layer4.1.conv2": (64, 32, 128),
         "fp8-256x256.b64.layer1.0.conv1": (64, 2048, 64), "fp8-256x256.b64.layer1.0.conv2": (64, 2048, 64),
         "fp8-256x256.b64.layer2.0.conv1": (128, 512, 64), "fp8-256x256.b64.layer2.0.downsample": (128, 512, 64),
         "fp8-256x256.b64.layer2.0.conv2": (128, 512, 128), "fp8-256x256.b64.layer2.1.conv2": (128, 512, 128),
         "fp8-256x256.b64.layer3.0.conv1": (128, 256, 128), "fp8-256x256.b64.layer3.0.downsample": (128, 256, 128),
         "fp8-256x256.b64.layer3.0.conv2": (128, 256, 128), "fp8-256x256.b64.layer3.1.conv2": (128, 256, 128),
         "fp8-256x256.b64.layer4.0.conv1": (128, 128, 128), "fp8-256x256.b64.layer4.0.downsample": (128, 128, 128),
         "fp8-256x256.b64.layer4.0.conv2": (128, 128, 128), "fp8-256x256.b64.layer4.1.conv2": (128, 128, 128),
         "fp8-256x341.b1.layer1.0.conv1": (64, 64, 64), "fp8-256x341.b1.layer1.0.conv2": (64, 64, 64),
         "fp8-256x341.b1.layer2.0.conv1": (64, 32, 64), "fp8-256x341.b1.layer2.0.downsample": (64, 32, 64),
         "fp8-256x341.b1.layer2.0.conv2": (64, 32, 128), "fp8-256x341.b1.layer2.1.conv2": (64, 32, 128),
         "fp8-256x341.b1.layer3.0.conv1": (64, 16, 128), "fp8-256x341.b1.layer3.0.downsample": (64, 16, 128),
         "fp8-256x341.b1.layer3.0.conv2": (64, 16, 128), "fp8-256x341.b1.layer3.1.conv2": (64, 16, 128),
         "fp8-256x341.b1.layer4.0.conv1": (64, 8, 128), "fp8-256x341.b1.layer4.0.downsample": (64, 8, 128),
         "fp8-256x341.b1.layer4.0.conv2": (64, 8, 128), "fp8-256x341.b1.layer4.1.conv2": (64, 8, 128),
         "fp8-256x341.b64.layer1.0.conv1": (64, 4096, 64), "fp8-256x341.b64.layer1.0.conv2": (64, 4096, 64),
         "fp8-256x341.b64.layer2.0.conv1": (128, 1024, 64), "fp8-256x341.b64.layer2.0.downsample": (128, 1024, 64),
         "fp8-256x341.b64.layer2.0.conv2": (128, 1024, 128), "fp8-256x341.b64.layer2.1.conv2": (128, 1024, 128),
         "fp8-256x341.b64.layer3.0.conv1": (128, 512, 128), "fp8-256x341.b64.layer3.0.downsample": (128, 512, 128),
         "fp8-256x341.b64.layer3.0.conv2": (128, 512, 128), "fp8-256x341.b64.layer3.1.conv2": (128, 512, 128),
         "fp8-256x341.b64.layer4.0.conv1": (128, 256, 128), "fp8-256x341.b64.layer4.0.downsample": (128, 256, 128),
         "fp8-256x341.b64.layer4.0.conv2": (128, 256, 128), "fp8-256x341.b64.layer4.1.conv2": (128, 256, 128),
         "fp8-256x256.b256.layer1.0.conv2": (64, 8192, 64), "bf16-256x256.b1.stem": (64, 128),
         "bf16-256x256.b1.layer1.0.conv1": (64, 32), "bf16-256x256.b1.layer1.0.conv2": (64, 32),
         "bf16-256x256.b1.layer2.0.conv1": (64, 16), "bf16-256x256.b1.layer2.0.downsample": (64, 16),
         "bf16-256x256.b1.layer2.0.conv2": (64, 16), "bf16-256x256.b1.layer3.0.conv1": (64, 8),
         "bf16-256x256.b1.layer3.0.downsample": (64, 8), "bf16-256x256.b1.layer3.0.conv2": (64, 8),
         "bf16-256x256.b1.layer4.0.conv1": (64, 8), "bf16-256x256.b1.layer4.0.downsample": (64, 8),
         "bf16-256x256.b1.layer4.0.conv2": (64, 8), "bf16-256x256.b8.stem": (64, 1024),
         "bf16-256x256.b8.layer1.0.conv1": (64, 256), "bf16-256x256.b8.layer1.0.conv2": (64, 256),
         "bf16-256x256.b8.layer2.0.conv1": (64, 128), "bf16-256x256.b8.layer2.0.downsample": (64, 128),
         "bf16-256x256.b8.layer2.0.conv2": (64, 128), "bf16-256x256.b8.layer3.0.conv1": (64, 64),
         "bf16-256x256.b8.layer3.0.downsample": (64, 64), "bf16-256x256.b8.layer3.0.conv2": (64, 64),
         "bf16-256x256.b8.layer4.0.conv1": (64, 32), "bf16-256x256.b8.layer4.0.downsample": (64, 32),
         "bf16-256x256.b8.layer4.0.conv2": (64, 32), "bf16-256x256.b64.stem": (64, 8192),
         "tc_split-256x256.b64.stem": (64, 8192), "bf16-256x256.b64.layer1.0.conv1": (64, 2048),
         "tc_split-256x256.b64.layer1.0.conv1": (64, 2048), "bf16-256x256.b64.layer1.0.conv2": (64, 2048),
         "tc_split-256x256.b64.layer1.0.conv2": (64, 2048), "bf16-256x256.b64.layer2.0.conv1": (128, 512),
         "tc_split-256x256.b64.layer2.0.conv1": (128, 512), "bf16-256x256.b64.layer2.0.downsample": (128, 512),
         "tc_split-256x256.b64.layer2.0.downsample": (128, 512), "bf16-256x256.b64.layer2.0.conv2": (128, 512),
         "tc_split-256x256.b64.layer2.0.conv2": (128, 512), "tc_split-256x256.b64.layer2.1.conv2": (128, 512),
         "bf16-256x256.b64.layer3.0.conv1": (128, 256), "tc_split-256x256.b64.layer3.0.conv1": (128, 256),
         "bf16-256x256.b64.layer3.0.downsample": (128, 256), "tc_split-256x256.b64.layer3.0.downsample": (128, 256),
         "bf16-256x256.b64.layer3.0.conv2": (128, 256), "tc_split-256x256.b64.layer3.0.conv2": (128, 256),
         "tc_split-256x256.b64.layer3.1.conv2": (128, 256), "bf16-256x256.b64.layer4.0.conv1": (128, 128),
         "tc_split-256x256.b64.layer4.0.conv1": (128, 128), "bf16-256x256.b64.layer4.0.downsample": (128, 128),
         "tc_split-256x256.b64.layer4.0.downsample": (128, 128), "bf16-256x256.b64.layer4.0.conv2": (128, 128),
         "tc_split-256x256.b64.layer4.0.conv2": (128, 128), "tc_split-256x256.b64.layer4.1.conv2": (128, 128),
         "bf16-256x341.b1.stem": (64, 256), "bf16-256x341.b1.layer1.0.conv1": (64, 64),
         "bf16-256x341.b1.layer1.0.conv2": (64, 64), "bf16-256x341.b1.layer2.0.conv1": (64, 32),
         "bf16-256x341.b1.layer2.0.downsample": (64, 32), "bf16-256x341.b1.layer2.0.conv2": (64, 32),
         "tc_split-256x341.b1.layer2.1.conv2": (64, 32), "bf16-256x341.b1.layer3.0.conv1": (64, 16),
         "bf16-256x341.b1.layer3.0.downsample": (64, 16), "bf16-256x341.b1.layer3.0.conv2": (64, 16),
         "bf16-256x341.b1.layer4.0.conv1": (64, 8), "tc_split-256x341.b1.layer4.0.conv1": (64, 8),
         "bf16-256x341.b1.layer4.0.downsample": (64, 8), "bf16-256x341.b1.layer4.0.conv2": (64, 8),
         "bf16-256x341.b64.stem": (64, 16384), "tc_split-256x341.b64.stem": (64, 16384),
         "bf16-256x341.b64.layer1.0.conv1": (64, 4096), "bf16-256x341.b64.layer1.0.conv2": (64, 4096),
         "tc_split-256x341.b64.layer1.0.conv2": (64, 4096), "bf16-256x341.b64.layer2.0.conv1": (128, 1024),
         "bf16-256x341.b64.layer2.0.downsample": (128, 1024), "bf16-256x341.b64.layer2.0.conv2": (128, 1024),
         "bf16-256x341.b64.layer3.0.conv1": (128, 512), "tc_split-256x341.b64.layer3.0.conv1": (128, 512),
         "bf16-256x341.b64.layer3.0.downsample": (128, 512), "tc_split-256x341.b64.layer3.0.downsample": (128, 512),
         "bf16-256x341.b64.layer3.0.conv2": (128, 512), "tc_split-256x341.b64.layer3.0.conv2": (128, 512),
         "bf16-256x341.b64.layer4.0.conv1": (128, 256), "bf16-256x341.b64.layer4.0.downsample": (128, 256),
         "bf16-256x341.b64.layer4.0.conv2": (128, 256), "tc_split-256x341.b64.layer4.1.conv2": (128, 256)}


def describe(engine, geom):
    """the engine's plan of one fprop (host only)"""
    B, H, W, Ci, Co, k, s = geom
    buf = ctypes.create_string_buffer(1 << 16)
    flags = {"bf16": 0, "tc_split": 2, "fp8": 4}[engine]
    _lib.check(_lib.lib().mapnet_test_plan_describe(0, B, H, W, Ci, Co, k, s, flags, buf, len(buf)),
               "mapnet_test_plan_describe")
    return json.loads(buf.value.decode())


def plan_summary(case):
    p = describe(case[0], case[3])
    assert len(p["launches"]) == 1
    L = p["launches"][0]
    assert len(L["classes"]) == 1
    return dict(BN=p["BN"], kb=p["f8_kb"], items=L["n_tiles_m"] * L["n_tiles_n"], box=(L["TW"], L["TH"], L["TN"]),
                taps=len(L["classes"][0]["taps"]), Cs=L["Cs"], L=L)


def expected_plan(case):
    s = plan_summary(case)
    want = PLANS[case_id(case)]
    got = (s["BN"], s["items"], s["kb"]) if case[0] == "fp8" else (s["BN"], s["items"])
    assert got == want, (case_id(case), got, want)
    return s


def test_case_list_covers_the_inference_plans():
    """Host only: every case's plan is the one it states, and the list still reaches the inference plans that matter."""
    from geomapnet_b200 import build
    build.build(verbose=False)
    assert len(PLANS) == len(F8_CASES) + len(AFF_CASES)
    f8 = [(c, expected_plan(c)) for c in F8_CASES]
    aff = [(c, expected_plan(c)) for c in AFF_CASES]
    assert any(s["items"] >= 16 * NSM for _, s in f8), "no fp8 launch with >= 16 work items per CTA"
    assert any(s["items"] > NSM and s["items"] % NSM for _, s in f8), "no fp8 launch with a ragged last wave"
    assert {s["kb"] for _, s in f8} == {64, 128}, "fp8 k-blocks: need 64 and 128 bytes"
    assert {s["BN"] for _, s in f8} == {64, 128}, "fp8: need BN 64 and 128"
    for eng in ("bf16", "tc_split"):
        assert {s["BN"] for c, s in aff if c[0] == eng} == {64, 128}, "%s affine: need BN 64 and 128" % eng
    assert any(c[3][6] == 2 and c[3][5] == 3 and c[3][2] % 2 for c, _ in f8), \
        "no stride-2 fp8 conv on an odd (ragged) width: its parity views differ in width"
    assert any(c[3][0] == 1 and s["items"] < NSM for c, s in f8 + aff), "no B = 1 launch with fewer items than CTAs"
    for eng in ("bf16", "tc_split"):
        assert any(c[2] == "stem" and c[0] == eng and s["items"] >= 16 * NSM for c, s in aff), \
            "no %s stem with >= 16 work items per CTA" % eng
    assert any(s["box"] == (128, 1, 1) for _, s in f8) and any(s["box"] == (128, 1, 1) for _, s in aff), \
        "no 128x1 pixel box"
    # every epilogue variant the schedule uses is run
    assert {c[4] for c in F8_CASES} == set(F8_EPI) and {c[4] for c in AFF_CASES} == set(AFF_EPI)


# ------------------------------------------------------------------------------------------------------------------
# operands, references, the per-element check
# ------------------------------------------------------------------------------------------------------------------
def _gen(name):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(name.encode()))


def _bf16(shape, g, scale=1.0, positive=False):
    t = torch.randn(shape, generator=g, device="cuda")
    return ((t.abs() if positive else t) * scale).bfloat16().double()


def _logu(shape, g):
    """fp32 values of magnitude in [2^-3, 2^3], random sign: inside fp16's window for the hi/lo split"""
    e = torch.rand(shape, generator=g, device="cuda") * 6.0 - 3.0
    s = torch.where(torch.rand(shape, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    return (s * torch.exp2(e)).float().double()


nhwc = lambda t: t.permute(0, 2, 3, 1)


def _codes(v):
    """e4m3 values (already representable) -> their bytes"""
    return v.float().to(torch.float8_e4m3fn).view(torch.uint8)


def _conv_ref(x, w, s, pad):
    """NHWC float64 (value, sum |a*b|) of an NCHW conv"""
    return nhwc(F.conv2d(x, w, None, s, pad)), nhwc(F.conv2d(x.abs(), w.abs(), None, s, pad))


def _where(idx, plan):
    """work item, CTA and the CTA's tile number of output elements idx [n, 4] (NHWC)"""
    L = plan["L"]
    n, h, w, c = idx.unbind(1)
    tm = w // L["TW"] + L["tiles_w"] * (h // L["TH"] + L["tiles_h"] * (n // L["TN"]))
    item = tm * L["n_tiles_n"] + c // plan["BN"]
    grid = min(plan["items"], NSM)
    return item, item % grid, item // grid


def check_elements(what, got, ref, bound, plan):
    """every element within its bound (NaN fails); prints and returns max(err / bound)"""
    err = (got - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        item, cta, j = _where(bad, plan)
        i = tuple(bad[0].tolist())
        raise AssertionError(
            "%s: %d of %d elements outside the bound (%d NaN) in %d of %d work items (%d of them a CTA's first tile, "
            "the earliest a CTA's tile #%d); first at NHWC %s: item %d, CTA %d, its tile #%d: got %r ref %r "
            "bound %r" % (
                what, bad.shape[0], got.numel(), int(torch.isnan(got).sum()), int(item.unique().numel()), plan["items"],
                int(item[j == 0].unique().numel()), int(j.min()), i, int(item[0]), int(cta[0]), int(j[0]),
                float(got[i]), float(ref[i]), float(bound[i])))
    ratio = float((err / bound).max())
    print("infer-plans %-58s max err/bound %.3g" % (what, ratio))
    return ratio


def _epi_error(sc, gamma, S, sh, r_abs):
    """E: the accumulation error through |scale| plus the epilogue's fp32 roundings"""
    a = sc.abs() * S
    return a * gamma + N_EPI * U_FP32 * (1 + gamma) * (a + sh.abs() + r_abs)


# ------------------------------------------------------------------------------------------------------------------
# fp8: k_f8_conv
# ------------------------------------------------------------------------------------------------------------------
def _run_f8(geom, x8, w8, sc, sh, rin, flags, out, amax=None):
    B, H, W, Ci, Co, k, s = geom
    s_res = torch.tensor([S_RES], device="cuda")
    ptr = lambda t: t.data_ptr() if t is not None else None
    _lib.check(_lib.lib().mapnet_test_conv_fp8(B, H, W, Ci, Co, k, s, x8.data_ptr(), w8.data_ptr(), sc.data_ptr(),
                                               sh.data_ptr(), ptr(rin), s_res.data_ptr(), ptr(out[1]), flags,
                                               ptr(out[0]), ptr(amax), _lib.stream_ptr()), "mapnet_test_conv_fp8")
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("case", F8_CASES, ids=case_id)
def test_fp8_conv_at_inference_plan(case):
    eng, cfg, role, geom, epi = case
    plan = expected_plan(case)
    t0 = time.time()
    B, H, W, Ci, Co, k, s = geom
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    flags, res, outk = F8_EPI[epi]
    g = _gen(case_id(case))
    # the distributions of test_gpu_infer_fp8 (its mismatch fractions were measured on them): e4m3 operands, weights
    # scaled per output channel as the pack does
    x = quantize_e4m3(torch.randn((B, H, W, Ci), generator=g, device="cuda") * 2.0)
    w = quantize_e4m3(torch.randn((Co, k, k, Ci), generator=g, device="cuda") * 64.0)
    sc = ((1.0 + 0.3 * torch.randn(Co, generator=g, device="cuda")) * (2.0 / (Ci * k * k)) ** 0.5 / 64.0).float()
    sh = (0.2 * torch.randn(Co, generator=g, device="cuda")).float()
    acc, S = _conv_ref(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), s, pad)
    x8, w8 = _codes(x), _codes(w)
    del x, w
    ref = acc * sc.double() + sh.double()
    del acc
    rin, r_abs = None, 0.0
    if res == "e4m3":
        r8 = quantize_e4m3(torch.randn((B, Ho, Wo, Co), generator=g, device="cuda") * 8.0)
        ref += r8.double() * S_RES
        r_abs = r8.double().abs() * S_RES
        rin = _codes(r8)
    elif res == "bf16":
        rin = torch.randn((B, Ho, Wo, Co), generator=g, device="cuda").bfloat16()
        ref += rin.double()
        r_abs = rin.double().abs()
    if flags & 1:
        ref.clamp_(min=0)
    gamma = plan["taps"] * plan["Cs"] // 32 * U_F8ACC
    E = _epi_error(sc.double(), gamma, S, sh.double(), r_abs)
    del S, r_abs
    if outk == "e4m3":
        s_out = pow2_scale(float(ref.abs().max()))
        out_inv = torch.tensor([1.0 / s_out], device="cuda")
        out = torch.full((B, Ho, Wo, Co), 0x7F, dtype=torch.uint8, device="cuda")        # e4m3fn NaN
        _run_f8(geom, x8, w8, sc, sh, rin, flags, (out, out_inv))
        got = out.view(torch.float8_e4m3fn).double() * s_out
        exact = quantize_e4m3((ref / s_out).float()).double() * s_out
        bound = U_E4M3 * ref.abs() + E4M3_HALF_SUB * s_out + (1 + U_E4M3) * E
    else:
        out = torch.full((B, Ho, Wo, Co), float("nan"), dtype=torch.bfloat16, device="cuda")
        _run_f8(geom, x8, w8, sc, sh, rin, flags, (out, None))
        got = out.double()
        exact = ref.float().bfloat16().double()
        bound = U_BF16 * ref.abs() + (1 + U_BF16) * E
    what = "fp8 %s.%s %s BN%d kb%d %d items" % (cfg, role, epi, plan["BN"], plan["kb"], plan["items"])
    check_elements(what, got, ref, bound, plan)
    frac = float((got != exact).double().mean())
    print("infer-plans %-58s outputs != exactly rounded %.4f" % (what, frac))
    assert frac <= MISMATCH_FRAC[outk == "e4m3"], (what, frac)
    if outk == "e4m3":
        # the calibration pass of the same launch: max |f| into amax, the output bytes untouched
        before = out.clone()
        amax = torch.zeros(1, dtype=torch.int32, device="cuda")
        _run_f8(geom, x8, w8, sc, sh, rin, flags | 8, (out, out_inv), amax)
        a, m, e = float(amax.view(torch.float32)), float(ref.abs().max()), float(E.max())
        assert torch.equal(out, before), "%s: the EPI_AMAX pass wrote the output" % what
        assert abs(a - m) <= e, (what, a, m, e)
        print("infer-plans %-58s amax %.6g ref %.6g err/bound %.3g" % (what, a, m, abs(a - m) / e))
    print("infer-plans %-58s %.1f s" % (what, time.time() - t0))


# ((B, H, W, Ci, Co, k, s), draws): one 3x3 conv per k-block width, the longest accumulation (K = 4608) and layer1's
MEASURE = [((1, 8, 8, 512, 512, 3, 1), 4), ((1, 16, 16, 64, 64, 3, 1), 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("geom,draws", MEASURE, ids=["ci512", "ci64"])
def test_fp8_accumulation_per_instruction(geom, draws):
    """U_F8ACC from a coherent case: non-negative e4m3 operands, constant over the pixels of the one image, so every
    interior output of channel c is the same exact sum T[c] (no ReLU: its values are non-negative anyway).  The epilogue
    runs with scale 2^-16 (exact) and shift = -fp32(2^-16 T[c]): f = 2^-16 acc - fl(2^-16 T) is exact in fp32 (the two
    are within a factor two), so the bf16 output holds 2^-16 (acc - T) up to 2^-8 of itself and 2^-24 T."""
    B, H, W, Ci, Co, k, s = geom
    plan = plan_summary(("fp8", "", "", geom, ""))
    n_instr = plan["taps"] * plan["Cs"] // 32
    worst, res, lo, hi = 0.0, 0.0, 0.0, 0.0
    for d in range(draws):
        g = _gen("measure-%d-%d" % (Ci, d))
        xv = quantize_e4m3(torch.randn(Ci, generator=g, device="cuda").abs() * 2.0)
        w = quantize_e4m3(torch.randn((Co, k, k, Ci), generator=g, device="cuda").abs() * 64.0)
        T = (w.double().sum((1, 2)) * xv.double()).sum(1)                    # exact: multiples of 2^-18 below 2^30
        sc = torch.full((Co,), 2.0 ** -16, device="cuda")
        sh = (-(T * 2.0 ** -16)).float()
        x = xv.expand(B, H, W, Ci).contiguous()
        out = torch.full((B, H, W, Co), float("nan"), dtype=torch.bfloat16, device="cuda")
        _run_f8(geom, _codes(x), _codes(w), sc, sh, None, 0, (out, None))
        f = out[:, 1:-1, 1:-1, :].double()                                   # interior pixels: all nine taps
        err = (f - sh.double()) / 2.0 ** -16 - T                              # acc - T
        resolution = (U_BF16 * f.abs() / 2.0 ** -16 + 2 * U_FP32 * T).max()
        rel = err / (n_instr * T)
        worst, lo, hi = max(worst, float(rel.abs().max())), min(lo, float(rel.min())), max(hi, float(rel.max()))
        res = max(res, float(resolution / T.min() / n_instr))
        assert not bool(torch.isnan(f).any())
    print("infer-plans fp8 accumulation, Ci %d, K %d (%d instructions): max |acc - T| / (K/32 * T) = %.3g, signed "
          "%.3g .. %.3g (resolution %.2g), U_F8ACC %.3g" % (Ci, plan["taps"] * Ci, n_instr, worst, lo, hi, res,
                                                             U_F8ACC))
    assert worst <= U_F8ACC, (worst, U_F8ACC)


# ------------------------------------------------------------------------------------------------------------------
# affine: k_tc_conv with EPI_AFFINE, bf16 and strict mode
# ------------------------------------------------------------------------------------------------------------------
def _planes(t):
    """hi/lo plane storage (common.cuh: hsplit; per 8 channels 8 fp16 hi then 8 fp16 lo) -> float64 [.., C]"""
    h = t.reshape(*t.shape[:-1], t.shape[-1] // 16, 2, 8).double()
    return (h[..., 0, :] + h[..., 1, :]).reshape(*t.shape[:-1], t.shape[-1] // 2)


@pytest.mark.gpu
@pytest.mark.parametrize("case", AFF_CASES, ids=case_id)
def test_affine_conv_at_inference_plan(case):
    eng, cfg, role, geom, epi = case
    plan = expected_plan(case)
    t0 = time.time()
    B, H, W, Ci, Co, k, s = geom
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    flags, res, outk = AFF_EPI[epi]
    strict = eng == "tc_split"
    g = _gen(case_id(case))
    if strict:
        x, w = _logu((B, Ci, H, W), g), _logu((Co, Ci, k, k), g)
    else:       # post-ReLU activations; the stem's normalized image is signed
        x = _bf16((B, Ci, H, W), g, positive=k != 7)
        w = _bf16((Co, Ci, k, k), g, (2.0 / (Ci * k * k)) ** 0.5)
    sc = (torch.rand(Co, generator=g, device="cuda") + 0.5).float()
    sh = (0.2 * torch.randn(Co, generator=g, device="cuda")).float()
    acc, S = _conv_ref(x, w, s, pad)
    op = torch.float32 if strict else torch.bfloat16
    if k == 7:      # the stem: fp32 NCHW image and OIHW weights, cut into the engine's operand form inside
        xin, win = x.float(), w.float()
    else:
        xin, win = nhwc(x).contiguous().to(op), w.permute(0, 2, 3, 1).contiguous().to(op)
    del x, w
    ref = acc * sc.double() + sh.double()
    del acc
    rin, r_abs, e_res = None, 0.0, 0.0
    if res is not None:
        r = _logu((B, Ho, Wo, Co), g) if strict else _bf16((B, Ho, Wo, Co), g)
        rin = r.to(op)
        ref += r
        r_abs = r.abs()
        if res == "planes":
            e_res = SPLIT * r_abs + PLANE_HALF_SUB
        del r
    if flags & 1:
        ref.clamp_(min=0)
    gamma = plan["taps"] * plan["Cs"] // 16 * TRUNC + (2 * SPLIT + SPLIT ** 2 if strict else 0.0)
    E = _epi_error(sc.double(), gamma, S, sh.double(), r_abs) + e_res
    del S, r_abs, e_res
    if outk == "planes":
        out = torch.full((B, Ho, Wo, 2 * Co), float("nan"), dtype=torch.float16, device="cuda")
        u, a = SPLIT, PLANE_HALF_SUB
    else:
        out = torch.full((B, Ho, Wo, Co), float("nan"), dtype=op, device="cuda")
        u, a = (0.0, 0.0) if outk == "fp32" else (U_BF16, 0.0)
    ptr = lambda t: t.data_ptr() if t is not None else None
    _lib.check(_lib.lib().mapnet_test_conv_affine(_lib.PREC[eng], B, H, W, Ci, Co, k, s, xin.data_ptr(), win.data_ptr(),
                                                  sc.data_ptr(), sh.data_ptr(), ptr(rin), flags, out.data_ptr(),
                                                  _lib.stream_ptr()), "mapnet_test_conv_affine")
    torch.cuda.synchronize()
    got = _planes(out) if outk == "planes" else out.double()
    bound = u * ref.abs() + a + (1 + u) * E
    what = "%s %s.%s %s BN%d %d items" % (eng, cfg, role, epi, plan["BN"], plan["items"])
    check_elements(what, got, ref, bound, plan)
    print("infer-plans %-58s %.1f s" % (what, time.time() - t0))
