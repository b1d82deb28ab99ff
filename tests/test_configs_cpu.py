"""CPU: at every configuration of tests/config_cases.py the module's state_dict schema is the reference's and the UNet library
accepts it; configurations it does not implement are refused with a message (dawn_unet_create needs no GPU)."""
import ctypes

import pytest

from tests import config_cases as CC


def create(cfg):
    from dawn_pytorch_b200 import _lib
    h = ctypes.c_void_p()
    rc = _lib.lib.dawn_unet_create(ctypes.byref(cfg), ctypes.byref(h))
    if rc == 0:
        _lib.lib.dawn_unet_destroy(h)
    return rc, _lib.lib.dawn_last_error().decode()


def cfg_of(**kw):
    """the library configuration of dim128 with fields replaced (dim_mults sets n_levels too)"""
    from dawn_pytorch_b200 import DynamicNfUnet3D
    cfg = DynamicNfUnet3D(**CC.ctor("dim128"))._cfg
    for k, v in kw.items():
        if k == "dim_mults":
            cfg.n_levels = len(v)
            for i, m in enumerate(v):
                cfg.dim_mults[i] = m
        else:
            setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("tag", CC.TAGS)
def test_state_dict_schema_equals_reference(tag):
    """the module's state_dict names and shapes, in order, are the reference's at the same configuration"""
    sch, rep = CC.schema(tag), CC.report(tag)
    assert (len(sch), CC.schema_digest(sch)) == (rep["schema_entries"], rep["schema_digest"])


@pytest.mark.parametrize("tag", CC.TAGS)
def test_create_accepts_config(tag):
    from dawn_pytorch_b200 import DynamicNfUnet3D
    rc, err = create(DynamicNfUnet3D(**CC.ctor(tag))._cfg)
    assert rc == 0, err


@pytest.mark.parametrize("kw,msg", [
    (dict(dim=0), "dim must be 64 or 128"),
    (dict(dim=96), "dim must be 64 or 128"),
    (dict(dim=192), "dim must be 64 or 128"),
    (dict(dim_mults=(1, 2, 4, 16)), "[1, 1024]"),                   # 128 x 16 = 2048 channels
    (dict(dim_mults=(1, 0, 2)), "[1, 1024]"),
    (dict(dim_mults=(1,)), "n_levels"),
    (dict(dim_mults=(1, 1, 1, 1, 1, 1, 1)), "n_levels"),
    (dict(init_kernel_size=9), "init kernel"),
    (dict(win_width=121), "win_width"),
    (dict(win_width=0), "win_width"),
])
def test_create_refuses_unsupported(kw, msg):
    rc, err = create(cfg_of(**kw))
    assert rc == -1 and msg in err, err
