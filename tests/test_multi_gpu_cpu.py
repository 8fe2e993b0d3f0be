"""garage_bm_create_on_devices without a GPU: the device lists it refuses before any CUDA context exists, and the
device metrics call's argument checks (DESIGN.md section 5.13)."""
import ctypes as C
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import garage_b200 as G  # noqa: E402
from garage_b200 import block_manager as BM  # noqa: E402

E_INVALID, E_NODEVICE = -1, -5


def _no_cuda():
    import torch

    return not torch.cuda.is_available()


def _create(tmp_path, devices, n=None, null_list=False):
    """garage_bm_create_on_devices of a file-store default config -> rc (a created manager is destroyed)"""
    L = BM.load_library()
    cfg = BM.Config()
    L.garage_bm_default_config(C.byref(cfg))
    keep = str(tmp_path / "store").encode()
    cfg.data_dir = keep
    arr = (C.c_int * max(1, len(devices)))(*devices)
    h = C.c_void_p()
    rc = L.garage_bm_create_on_devices(C.byref(h), C.byref(cfg), None, 0, None if null_list else arr,
                                       len(devices) if n is None else n)
    if rc == 0:
        L.garage_bm_destroy(h)
    assert rc == 0 or not h.value
    return rc


@pytest.mark.parametrize("case", ["null_list", "zero", "negative_count", "seventeen", "negative_device",
                                  "negative_device_later"])
def test_bad_device_lists_are_refused_before_any_context(tmp_path, case):
    devices, kw = {
        "null_list": ([0], {"null_list": True}), "zero": ([0], {"n": 0}), "negative_count": ([0], {"n": -1}),
        "seventeen": ([0] * 17, {}), "negative_device": ([-1], {}), "negative_device_later": ([0, 0, -2], {}),
    }[case]
    assert _create(tmp_path, devices, **kw) == E_INVALID
    assert not (tmp_path / "store").exists(), "nothing may be created before the check"


@pytest.mark.skipif(not _no_cuda(), reason="checks the no-GPU behaviour")
def test_no_device_is_nodevice_as_for_garage_bm_create(tmp_path):
    assert G.load_library().garage_ec_device_count() == 0
    assert _create(tmp_path, [0]) == E_NODEVICE
    assert _create(tmp_path, [0, 1]) == E_NODEVICE
    with pytest.raises(BM.BlockManagerError) as e:
        BM.BlockManager(4, 2, cuda_devices=[0, 0])
    assert e.value.code == E_NODEVICE


def test_config_refusals_still_come_first(tmp_path):
    """a list that is fine does not hide a configuration garage_bm_create refuses"""
    L = BM.load_library()
    cfg = BM.Config()
    L.garage_bm_default_config(C.byref(cfg))
    cfg.parity_shards = 0
    arr = (C.c_int * 2)(0, 0)
    h = C.c_void_p()
    assert L.garage_bm_create_on_devices(C.byref(h), C.byref(cfg), None, 0, arr, 2) == E_INVALID and not h.value


def test_device_metrics_argument_checks():
    L = BM.load_library()
    n = C.c_int(0)
    out = (BM.DeviceMetrics * 1)()
    assert L.garage_bm_get_device_metrics(None, out, 1, C.byref(n)) == E_INVALID
