"""CPU: the C-ABI library loads without a GPU driver and exports every symbol include/monoflex_b200.h declares; the
ctypes table monoflex_b200/_lib.py derives from the header covers the same set with the right types; csrc/ defines each
entry point exactly once; product modules keep the reference's state_dict keys."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT


def header_symbols():
    src = open(os.path.join(ROOT, "include", "monoflex_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mf_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    path = os.path.join(ROOT, "monoflex_b200", "libmonoflex_b200.so")
    if not os.path.exists(path):
        import __graft_entry__
        __graft_entry__.build()
    return ctypes.CDLL(path)


def test_library_exports_every_declared_symbol(lib):
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), "missing export %s" % s


def test_ctypes_table_matches_header():
    from monoflex_b200 import _lib
    assert sorted(list(_lib.SIGNATURES) + ["mf_last_error"]) == header_symbols()


def test_derived_bindings_cover_header():
    """The prototypes parsed from the header include every symbol this independent name scan finds."""
    from monoflex_b200 import _lib
    assert sorted(_lib._PROTOTYPES) == header_symbols()


def test_derived_ctypes_types():
    from monoflex_b200 import _lib
    sig, proto = _lib.SIGNATURES, _lib._PROTOTYPES
    assert sig["mf_bn_sync_forward_apply"][5] is ctypes.c_double
    assert sig["mf_loss_scale_update"][3:5] == [ctypes.c_double, ctypes.c_double]
    assert sig["mf_adamw_step_p2p"][4:6] == [ctypes.c_ulonglong, ctypes.c_ulonglong]
    assert sig["mf_kitti_eval_statistics"][14] is ctypes.c_size_t
    assert sig["mf_sigmoid_clamp"] == [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    assert sig["mf_version"] == [] and proto["mf_last_error"][1] == []
    workspace = [name for name in sig if name.endswith("_workspace")]
    assert len(workspace) == 5
    assert {proto[name][0] for name in workspace} == {ctypes.c_size_t}
    assert proto["mf_last_error"][0] is ctypes.c_char_p
    assert {proto[name][0] for name in sig if name not in workspace} == {ctypes.c_int}


def test_unknown_parameter_type_is_refused():
    from monoflex_b200 import _lib
    assert _lib.parse_header("int mf_ok(const void* x, unsigned long long n, void* stream);")["mf_ok"][1] == \
        [ctypes.c_void_p, ctypes.c_ulonglong, ctypes.c_void_p]
    with pytest.raises(RuntimeError, match="mf_bad"):
        _lib.parse_header("int mf_bad(const float* x, short n, void* stream);")
    with pytest.raises(RuntimeError, match="mf_bad_ret"):
        _lib.parse_header("float mf_bad_ret(void);")


def test_each_entry_point_defined_once_beside_its_kernels():
    """Every header symbol has exactly one definition under csrc/, and csrc/ defines no mf_* function the header lacks."""
    csrc = os.path.join(ROOT, "monoflex_b200", "csrc")
    defined = []
    for name in sorted(os.listdir(csrc)):
        if name.endswith(".cu"):
            src = re.sub(r"/\*.*?\*/|//[^\n]*", "", open(os.path.join(csrc, name)).read(), flags=re.S)
            defined += re.findall(r"\b(?:int|size_t|char\s*\*)\s*\b(mf_[a-z0-9_]+)\s*\([^;{}]*\)\s*\{", src)
    assert sorted(defined) == header_symbols()


def test_version_and_error_string(lib):
    lib.mf_last_error.restype = ctypes.c_char_p
    assert lib.mf_version() == 100
    assert lib.mf_set_conv_impl(7) != 0
    assert b"impl must be 0 or 1" in lib.mf_last_error()
    assert lib.mf_dcn_v2_psroi_pooling_forward() == -2
    assert b"not built" in lib.mf_last_error()


# the layout entry points that take pair rows or fp16 rows by their lo offsets, called with offsets they must refuse before
# any CUDA call (no device needed): (name, args without the stream)
P = 16                  # a non-null pointer that is never dereferenced
BAD_LO = [
    ("mf_maxpool2_nhwc_f16", (P, 64, 0, P, 64, 32, 2, 4, 4, 32)),                       # fp16 x, pair y
    ("mf_maxpool2_nhwc_f16", (P, 64, 32, P, 64, 0, 2, 4, 4, 32)),                       # pair x, fp16 y
    ("mf_maxpool2_nhwc_f16", (P, 64, 36, P, 64, 32, 2, 4, 4, 32)),                      # x_lo not a multiple of 8
    ("mf_upsample_add_nhwc_f16", (P, 64, 32, P, P, 64, 0, P, 64, 32, 2, 4, 4, 32, 2)),  # fp16 skip, pair x and y
    ("mf_upsample_add_nhwc_f16", (P, 64, 0, P, None, 0, 0, P, 64, 32, 2, 4, 4, 32, 4)),  # fp16 x, pair y, no skip
    ("mf_upsample_add_nhwc_f16", (P, 64, 32, P, P, 64, 36, P, 64, 32, 2, 4, 4, 32, 2)),  # skip_lo not a multiple of 8
    ("mf_edge_gather", (P, 1024, 516, 0, 256, P, P, P, 2, 4, 4, 8, 16, 16)),             # feat_lo not a multiple of 8
    ("mf_edge_head_add", (P, 512, 260, P, P, 2, P, P, P, 3, 0, 2, 8, 4, 4)),             # t_lo not a multiple of 8
]


@pytest.mark.parametrize("name,args", BAD_LO, ids=["%s-%d" % (n, i) for i, (n, _) in enumerate(BAD_LO)])
def test_row_format_errors(name, args):
    """mixed row formats and lo offsets off the 16-byte grid are refused with a message, before any CUDA call"""
    from monoflex_b200 import _lib
    lib = _lib.load()
    assert getattr(lib, name)(*args, None) == -1
    assert b"lo offsets must all be 0" in lib.mf_last_error()


def test_conv_block_n(lib):
    assert [lib.mf_conv_block_n(c) for c in (3, 16, 27, 32, 64, 128, 256, 2304)] == [16, 16, 32, 32, 64, 128, 128, 128]


def test_state_dict_keys_match_reference_layout():
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.config import default_cfg
    from monoflex_b200.model.detector import KeypointDetector
    m = KeypointDetector(default_cfg())
    sd = syn.make_state_dict(0)
    assert set(m.state_dict()) == set(sd)
    for k, v in m.state_dict().items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
    assert sum(p.numel() for p in m.parameters()) == 20952538      # SURVEY §8 [probe]
    m.load_state_dict(sd)
    for key in ("backbone.base.level3.tree1.tree2.conv1.weight", "backbone.dla_up.ida_1.proj_2.conv.conv_offset_mask.bias",
                "backbone.ida_up.up_2.weight", "heads.predictor.reg_features.5.0.weight",
                "heads.predictor.reg_heads.5.1.bias", "heads.predictor.trunc_offset_conv.0.weight"):
        assert key in sd


def test_no_cpu_fallback():
    """The product path refuses CPU tensors / training mode instead of silently falling back."""
    from monoflex_b200.config import default_cfg
    from monoflex_b200.model.detector import KeypointDetector
    m = KeypointDetector(default_cfg(width=64, height=64)).eval()
    with pytest.raises(RuntimeError):
        m.backbone(torch.zeros(1, 3, 64, 64))
    m.train()
    with pytest.raises(ValueError):
        m(torch.zeros(1, 3, 64, 64))
