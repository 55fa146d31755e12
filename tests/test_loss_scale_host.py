"""CPU: argument checks of the dynamic loss scale (monoflex_b200/loss_scale.py) and of its C entry points
(mf_unscale_accumulate, mf_loss_scale_update), which fail before anything reaches a device; its checkpoint layout is
torch.amp.GradScaler's."""
import ctypes
import os

import pytest
import torch

from conftest import ROOT


@pytest.fixture(scope="module")
def lib():
    path = os.path.join(ROOT, "monoflex_b200", "libmonoflex_b200.so")
    if not os.path.exists(path):
        import __graft_entry__
        __graft_entry__.build()
    from monoflex_b200 import _lib
    return _lib.load()


DUMMY = 16                                                             # never dereferenced: the call fails first


@pytest.mark.parametrize("kw", [dict(init_scale=0.0), dict(init_scale=-1.0), dict(init_scale=float("inf")),
                                dict(init_scale=float("nan")), dict(init_scale=1e39), dict(init_scale="65536"),
                                dict(growth_factor=1.0), dict(growth_factor=0.5), dict(growth_factor=float("inf")),
                                dict(backoff_factor=0.0), dict(backoff_factor=1.0), dict(backoff_factor=1.5),
                                dict(growth_interval=0), dict(growth_interval=2.0), dict(growth_interval=True),
                                dict(growth_interval=2 ** 31)])
def test_dynamic_loss_scale_rejects_bad_arguments(kw):
    from monoflex_b200.loss_scale import DynamicLossScale
    with pytest.raises(ValueError):
        DynamicLossScale(**kw)


def _cpu_scaler(scale, tracker):
    """a DynamicLossScale whose state sits in host tensors: only its checkpoint methods are used"""
    from monoflex_b200.loss_scale import DynamicLossScale
    s = DynamicLossScale.__new__(DynamicLossScale)
    s.growth_factor, s.backoff_factor, s.growth_interval = 2.0, 0.5, 2000
    s.scale = torch.full((), scale, dtype=torch.float32)
    s.growth_tracker = torch.full((), tracker, dtype=torch.int32)
    s.optimizer = None
    return s


def test_state_dict_has_grad_scalers_keys_and_types():
    want = torch.amp.GradScaler("cpu").state_dict()
    got = _cpu_scaler(2.0 ** 16, 0).state_dict()
    assert set(got) == set(want)
    assert {k: type(v) for k, v in got.items()} == {k: type(v) for k, v in want.items()}
    assert got == want


def test_state_dict_loads_from_and_into_grad_scaler():
    ref = torch.amp.GradScaler("cpu", init_scale=1024.0, growth_factor=4.0, backoff_factor=0.25, growth_interval=7)
    sd = ref.state_dict()
    sd["_growth_tracker"] = 3
    s = _cpu_scaler(1.0, 0)
    s.load_state_dict(sd)
    assert (s.get_scale(), s.growth_factor, s.backoff_factor, s.growth_interval) == (1024.0, 4.0, 0.25, 7)
    assert int(s.growth_tracker) == 3
    back = torch.amp.GradScaler("cpu")
    back.load_state_dict(s.state_dict())
    assert back.state_dict() == sd
    with pytest.raises(RuntimeError, match="missing keys"):
        s.load_state_dict({"scale": 1.0})
    with pytest.raises(ValueError):
        s.load_state_dict(dict(sd, backoff_factor=2.0))


def test_trainer_argument_resolution(monkeypatch):
    from monoflex_b200 import loss_scale
    monkeypatch.delenv("MF_LOSS_SCALE", raising=False)
    assert loss_scale.resolve(None) == (None, None)
    assert loss_scale.resolve(256) == (256.0, None)
    s = _cpu_scaler(8.0, 0)
    assert loss_scale.resolve(s) == (None, s)


def _unscale(lib, dst=None, src=None, numels=None, count=1, scale=DUMMY):
    arr = (ctypes.c_ulonglong * 1)(DUMMY)
    n = (ctypes.c_longlong * 1)(4 if numels is None else numels)
    dst = ctypes.addressof(arr) if dst is None else dst
    src = ctypes.addressof(arr) if src is None else src
    return lib.mf_unscale_accumulate(dst, src, ctypes.addressof(n), None, count, scale, None)


def test_unscale_accumulate_argument_checks(lib):
    cap = lib.mf_unscale_max_tensors()
    assert cap >= 300                                                  # the detector's ~280 gradients in one launch
    assert _unscale(lib, count=cap + 1) != 0 and b"in one launch" in lib.mf_last_error()
    assert _unscale(lib, count=-1) != 0 and b"in one launch" in lib.mf_last_error()
    assert _unscale(lib, scale=None) != 0 and b"scale (device float) is NULL" in lib.mf_last_error()
    for kw in (dict(dst=0), dict(src=0)):
        assert _unscale(lib, **kw) != 0 and b"not NULL" in lib.mf_last_error()
    assert _unscale(lib, numels=-1) != 0 and b"elements" in lib.mf_last_error()
    assert _unscale(lib, numels=2 ** 31) != 0 and b"elements" in lib.mf_last_error()
    null = (ctypes.c_ulonglong * 1)(0)
    assert _unscale(lib, dst=ctypes.addressof(null)) != 0 and b"NULL dst or src" in lib.mf_last_error()
    assert _unscale(lib, count=0) == 0                                 # nothing to do: no launch
    assert _unscale(lib, numels=0) == 0                                # empty tensors are skipped: no launch


@pytest.mark.parametrize("args", [(2.0, 0.5, 0), (1.0, 0.5, 10), (2.0, 1.0, 10), (2.0, 0.0, 10), (float("nan"), 0.5, 10)])
def test_loss_scale_update_argument_checks(lib, args):
    assert lib.mf_loss_scale_update(DUMMY, DUMMY, DUMMY, args[0], args[1], args[2], None) != 0
    assert b"growth_factor > 1" in lib.mf_last_error()


def test_loss_scale_update_needs_device_pointers(lib):
    for ptrs in ((None, DUMMY, DUMMY), (DUMMY, None, DUMMY), (DUMMY, DUMMY, None)):
        assert lib.mf_loss_scale_update(*ptrs, 2.0, 0.5, 10, None) != 0
        assert b"not NULL" in lib.mf_last_error()
