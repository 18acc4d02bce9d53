"""Frozen parameters, host side (no GPU): the mapnet_trunk_set_trainable entry point, its argument checks on a spec-only
handle, and the mask PoseNet derives from requires_grad."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from geomapnet_b200 import build
    return build.build(verbose=False)


def _spec():
    from geomapnet_b200 import _lib
    return _lib.Trunk(0, 256, 256, 2048, "bf16")


def test_set_trainable_declared_and_exported(built):
    from geomapnet_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mapnet_b200.h")).read(), flags=re.S)
    assert re.search(r"int\s+mapnet_trunk_set_trainable\s*\(\s*mapnet_trunk_t\s*\*\s*h\s*,\s*const\s+uint8_t\s*\*\s*"
                     r"host_mask\s*,\s*int\s+n\s*\)\s*;", hdr)
    assert "mapnet_trunk_set_trainable" in _lib.EXPORTED
    assert hasattr(ctypes.CDLL(built), "mapnet_trunk_set_trainable")
    assert _lib.lib().mapnet_abi_version() == 2


def test_set_trainable_rejects_bad_arguments_on_spec_handle(built):
    from geomapnet_b200 import _lib
    L = _lib.lib()
    t = _spec()
    try:
        n = sum(1 for e in t.table()[0] if e[1] == 0)
        assert n == 114       # 36 conv weights, 36 BatchNorm (gamma, beta), 3 Linear (weight, bias)
        for bad in (n - 1, n + 1, 0, -1):
            buf = (ctypes.c_uint8 * max(bad, 1))(*([1] * max(bad, 1)))
            assert L.mapnet_trunk_set_trainable(t.h, buf, bad) != 0
            msg = L.mapnet_last_error().decode()
            assert "set_trainable" in msg and str(n) in msg, msg
        assert L.mapnet_trunk_set_trainable(t.h, None, n) != 0
        assert "null mask" in L.mapnet_last_error().decode()
        assert L.mapnet_trunk_set_trainable(None, (ctypes.c_uint8 * n)(), n) != 0
        assert "null handle" in L.mapnet_last_error().decode()
        # a valid mask is host-only: accepted without a device
        assert L.mapnet_trunk_set_trainable(t.h, (ctypes.c_uint8 * n)(*([0, 1] * (n // 2))), n) == 0
        with pytest.raises(_lib.MapNetLibError, match="set_trainable"):
            t.set_trainable([True] * (n - 1))
    finally:
        t.close()


def test_trunk_passes_mask_only_when_it_changes(built, monkeypatch):
    from geomapnet_b200 import _lib
    t = _spec()
    try:
        n = sum(1 for e in t.table()[0] if e[1] == 0)
        calls = []
        real = _lib.lib().mapnet_trunk_set_trainable

        class Wrap(object):
            def __getattr__(self, name):
                return getattr(real_lib, name)

            def mapnet_trunk_set_trainable(self, h, buf, k):
                calls.append(list(buf)[:k])
                return real(h, buf, k)
        real_lib = _lib.lib()
        monkeypatch.setattr(_lib, "lib", lambda: Wrap())
        t.set_trainable([True] * n)
        t.set_trainable([True] * n)
        assert calls == [[1] * n]
        mask = [i % 3 == 0 for i in range(n)]
        t.set_trainable(mask)
        t.set_trainable(tuple(mask))
        assert calls[1:] == [[int(m) for m in mask]]
        t.set_trainable([True] * n)             # back to all: passed, since the handle holds another mask
        assert len(calls) == 3 and calls[2] == [1] * n
    finally:
        monkeypatch.undo()
        t.close()


def test_mask_follows_table_order(built):
    import torchvision
    from geomapnet_b200.models.posenet import PoseNet
    torch.manual_seed(0)
    m = PoseNet(torchvision.models.resnet34(weights=None), droprate=0.0, pretrained=False)
    t = _spec()
    try:
        names = [e[0] for e in t.table()[0] if e[1] == 0]
    finally:
        t.close()
    assert [nm for nm, _ in m.named_parameters()] == names
    assert m.trainable_mask() == (True,) * len(names)
    for p in m.feature_extractor.parameters():
        p.requires_grad_(False)
    m.feature_extractor.layer4.requires_grad_(True)
    m.feature_extractor.bn1.bias.requires_grad_(True)
    want = tuple(nm.startswith("feature_extractor.layer4.") or nm == "feature_extractor.bn1.bias"
                 or not nm.startswith("feature_extractor.") for nm in names)
    assert m.trainable_mask() == tuple(dict(m.named_parameters())[nm].requires_grad for nm in names) == want
    assert want[names.index("feature_extractor.bn1.bias")] and not want[names.index("feature_extractor.bn1.weight")]
    assert not want[names.index("feature_extractor.fc.weight")] and want[names.index("fc_xyz.weight")]
