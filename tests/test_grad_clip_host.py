"""CPU: argument checks of the optimiser step (mf_optim_step_dyn), which fail before any launch."""
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


DUMMY = 16                                                             # never dereferenced: the call fails first


def _step(lib, rule=0, hyper=DUMMY, max_norm=0.0, partials=DUMMY, norm_out=DUMMY):
    return lib.mf_optim_step_dyn(rule, DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, 4, hyper, 0.99, 1e-8, 1.0, DUMMY, DUMMY, max_norm,
                                 partials, norm_out, None)


def test_optim_step_clip_needs_partials_and_norm_output(lib):
    for partials, norm_out in ((None, DUMMY), (DUMMY, None)):
        assert _step(lib, max_norm=1.0, partials=partials, norm_out=norm_out) != 0
        assert b"partials buffer and total_norm_out" in lib.mf_last_error()


def test_step_needs_hyper_block(lib):
    assert _step(lib, hyper=None) != 0
    assert b"hyper (device double[4]) is NULL" in lib.mf_last_error()


@pytest.mark.parametrize("rule", [-1, 2])
def test_step_refuses_unknown_rule(lib, rule):
    assert _step(lib, rule=rule) != 0
    assert ("rule %d" % rule).encode() in lib.mf_last_error()
