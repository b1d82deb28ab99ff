"""CPU: the UNet's handle lifecycle around a parameter re-commit (no GPU), against a fake library that records its calls.  The library
re-applies the geometry on commit, so a re-commit issues no dawn_unet_set_geometry; it changes graph_generation(), and a
frame-sharded UNet raises on its next use (init_shard must run again on every rank)."""
import contextlib
import unittest.mock as um

import pytest
import torch

from tests import gpu_common as G

DEV, GEOM = torch.device("cuda", 0), (4, 8, 8)


class _FakeLib:
    def __init__(self, calls):
        self.calls = calls

    def __getattr__(self, name):
        def f(*a):
            self.calls.append((name, a[1].decode()) if name == "dawn_unet_set_param" else name)
            return 0
        return f


@pytest.fixture
def calls():
    from dawn_pytorch_b200 import _lib, unet
    calls = []
    fake = _FakeLib(calls)
    with um.patch.object(_lib, "lib", fake), um.patch.object(unet, "lib", fake), \
            um.patch("torch.cuda.device", lambda idx: contextlib.nullcontext()):
        yield calls


def _ready_net(calls):
    """a UNet whose handle was created, committed and given GEOM"""
    from dawn_pytorch_b200 import DynamicNfUnet3D
    net = DynamicNfUnet3D(**G.CTOR).eval()
    net._ensure(DEV, *GEOM)
    params = {c[1] for c in calls if isinstance(c, tuple)}
    assert params == set(net.state_dict()) | {"aux.time_freqs", "aux.rel_bias"}
    assert [c for c in calls if not isinstance(c, tuple)] == ["dawn_unet_create", "dawn_unet_commit_params", "dawn_unet_set_geometry"]
    calls.clear()
    return net


def test_recommit_keeps_the_geometry_and_changes_the_graph_generation(calls):
    net = _ready_net(calls)
    gen = net.graph_generation()
    net._ensure(DEV, *GEOM)
    assert calls == [] and net.graph_generation() == gen
    net.load_state_dict(net.state_dict())
    net._ensure(DEV, *GEOM)
    assert [c for c in calls if not isinstance(c, tuple)] == ["dawn_unet_commit_params"]
    assert net.graph_generation() != gen
    gen = net.graph_generation()
    calls.clear()
    net.float()                                                   # .to() / .float() / .cuda() also re-commit
    net._ensure(DEV, *GEOM)
    assert [c for c in calls if not isinstance(c, tuple)] == ["dawn_unet_commit_params"]
    assert net.graph_generation() != gen


def test_a_sharded_unet_raises_after_a_recommit(calls):
    from dawn_pytorch_b200._lib import DawnError
    net = _ready_net(calls)
    net._shard = (0, 2, GEOM)                                     # what init_shard leaves on rank 0 of 2
    assert net.shard_info() == (0, 2)
    net.load_state_dict(net.state_dict())
    for _ in range(2):                                            # every use until init_shard runs again
        with pytest.raises(DawnError, match="call init_shard again"):
            net._ensure(DEV, *GEOM)
    assert net.shard_info() == (0, 1)
    assert [c for c in calls if not isinstance(c, tuple)] == ["dawn_unet_commit_params"]
