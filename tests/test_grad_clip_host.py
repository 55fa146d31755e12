"""CPU: argument checks of the clipping AdamW entry point (mf_adamw_step_dyn_clip), which fail before any launch."""
import ctypes
import os

import pytest

from conftest import ROOT


@pytest.fixture(scope="module")
def lib():
    path = os.path.join(ROOT, "monoflex_b200", "libmonoflex_b200.so")
    if not os.path.exists(path):
        import __graft_entry__
        __graft_entry__.build()
    from monoflex_b200 import _lib
    return _lib.load()


def test_clip_needs_partials_and_norm_output(lib):
    dummy = 16                                                         # never dereferenced: the call fails first
    for partials, norm_out in ((None, dummy), (dummy, None)):
        rc = lib.mf_adamw_step_dyn_clip(dummy, dummy, dummy, dummy, dummy, 4, 0.9, 0.99, 1e-8, 1e-5, 1.0, 1.0, dummy, dummy, 1,
                                        1.0, partials, norm_out, None)
        assert rc != 0
        assert b"partials buffer and total_norm_out" in lib.mf_last_error()
