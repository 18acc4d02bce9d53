"""Static evidence that the built library's hot path is the Hopper one (no GPU needed): cuobjdump -sass of
libmapnet_b200.so must contain the wgmma / TMA / mbarrier instructions the conv engines are written around, for
sm_90a, and none of the Ampere-style warp-level tensor-core instructions a compatibility path would leave behind."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sass():
    from geomapnet_b200 import build
    so = build.build(verbose=False)
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    r = subprocess.run([exe, "-sass", so], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-1000:]
    return r.stdout


def _kernel_bodies(sass):
    """{demangled-ish function name: SASS text}"""
    out, name, buf = {}, None, []
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                out[name] = "\n".join(buf)
            name, buf = m.group(1), []
        elif name:
            buf.append(line)
    if name:
        out[name] = "\n".join(buf)
    return out


def test_library_targets_sm_90a_only(sass):
    # every device function in the fat binary is sm_90a code (the CUDA runtime's own empty stub image is ignored)
    arch, per_arch = None, {}
    for line in sass.splitlines():
        m = re.match(r"arch = (sm_\w+)", line)
        if m:
            arch = m.group(1)
        elif re.match(r"\s*Function : ", line):
            per_arch[arch] = per_arch.get(arch, 0) + 1
    assert set(per_arch) == {"sm_90a"} and per_arch["sm_90a"] > 50, per_arch


def test_six_conv_engines_use_wgmma_tma_and_mbarriers(sass):
    k = _kernel_bodies(sass)
    conv = {n: b for n, b in k.items() if "k_tc_conv" in n or "k_tc_wgrad" in n}
    # training fprop / dgrad, inference fprop (eval-mode epilogues) and wgrad, each with N tiles of 64 and 128
    # (mangled: k_tc_conv<BN, AFF> = k_tc_convILi<BN>ELb<AFF>E..., k_tc_wgrad<BN> = k_tc_wgradILi<BN>EE...)
    names = {re.search(r"k_tc_(conv|wgrad)ILi\d+E(Lb[01]E)?", n).group(0) for n in conv}
    expected = {"k_tc_convILi%dELb%dE" % (bn, aff) for bn in (64, 128) for aff in (0, 1)} | \
               {"k_tc_wgradILi%dE" % bn for bn in (64, 128)}
    assert len(conv) == 6 and names == expected, sorted(conv)
    for n, b in conv.items():
        assert "HGMMA" in b, "no wgmma in %s" % n                        # warpgroup MMA, accumulator in registers
        assert "UTMALDG" in b, "no TMA tensor load in %s" % n          # cp.async.bulk.tensor
        assert "SYNCS.ARRIVE.TRANS64" in b, "no mbarrier transaction arrive in %s" % n
        assert "WARPGROUP.DEPBAR" in b, "no wgmma.wait_group in %s" % n
        assert not re.search(r"\bHMMA\.", b), "legacy tensor-core instruction in %s" % n
    # im2col happens in the load: the fprop / dgrad / wgrad engines read activations through 4-D tensor maps
    assert all("UTMALDG.4D" in b for n, b in conv.items())
    # wgrad writes every dW element with plain stores (one writer per element; split-K partials are added up in a fixed
    # order by k_wgrad_reduce): no float atomics, so the gradient is the same from run to run
    wgrad = [b for n, b in conv.items() if "k_tc_wgrad" in n]
    assert wgrad and all("STG.E" in b and not re.search(r"\b(RED|REDG|ATOMG)\.E\.ADD\.F32", b) for b in wgrad)


def test_bandwidth_kernels_are_vectorised(sass):
    k = _kernel_bodies(sass)
    for key in ("k_bn_apply", "k_bn_bwd_apply", "k_adam"):
        bodies = [b for n, b in k.items() if key in n]
        assert bodies, key
        for b in bodies:
            assert re.search(r"LDG\.E\.(128|64)|LDG\.E\.\w*\.?128", b), "%s has no 128-bit global loads" % key
            assert re.search(r"STG\.E\.(128|64)", b), "%s has no wide global stores" % key
