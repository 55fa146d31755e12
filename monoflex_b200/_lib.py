"""ctypes binding of libmonoflex_b200.so (include/monoflex_b200.h). There is NO fallback: if the shared library is
missing or a call fails, a RuntimeError is raised (the reference's AT_ASSERTM/AT_ERROR also surface as RuntimeError,
/root/reference/model/backbone/DCNv2/src/dcn_v2.h:25-45)."""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmonoflex_b200.so")
_lib = None

HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "monoflex_b200.h")

_ARG_TYPES = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "unsigned long long": ctypes.c_ulonglong,
              "float": ctypes.c_float, "double": ctypes.c_double, "size_t": ctypes.c_size_t}
_RET_TYPES = {"int": ctypes.c_int, "size_t": ctypes.c_size_t, "const char*": ctypes.c_char_p}


def parse_header(text):
    """{name: (restype, argtypes)} of every mf_* prototype in the C header `text`: any pointer is c_void_p, the scalar
    types map as in _ARG_TYPES. A type without a ctypes mapping raises RuntimeError naming the symbol."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", " ", text, flags=re.M)
    table = {}
    for ret, name, params in re.findall(r"([A-Za-z_][\w\s]*\**)\s*\b(mf_\w+)\s*\(([^)]*)\)\s*;", text):
        ret = re.sub(r"\s+", " ", ret).replace(" *", "*").strip()
        if ret not in _RET_TYPES:
            raise RuntimeError("monoflex_b200.h: %s returns %r, which has no ctypes mapping here" % (name, ret))
        args = []
        for param in params.split(","):
            words = [w for w in re.findall(r"\w+", param) if w != "const"]
            if "*" in param:
                args.append(ctypes.c_void_p)
            elif words != ["void"]:
                ctype = " ".join(words[:-1])                      # the last word is the parameter's name
                if ctype not in _ARG_TYPES:
                    raise RuntimeError("monoflex_b200.h: %s takes %r, which has no ctypes mapping here" % (name, param.strip()))
                args.append(_ARG_TYPES[ctype])
        table[name] = (_RET_TYPES[ret], args)
    return table


with open(HEADER_PATH) as _f:
    _PROTOTYPES = parse_header(_f.read())
# name -> argtypes of the entry points that return a status or a size (all but mf_last_error, which returns the message),
# derived from include/monoflex_b200.h
SIGNATURES = {name: args for name, (restype, args) in _PROTOTYPES.items() if restype is not ctypes.c_char_p}


def load():
    """dlopen the in-tree library (built by __graft_entry__.build()); raises if absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("monoflex_b200: %s not built - run `python __graft_entry__.py` (nvcc, sm_90a). "
                               "There is no CPU or PyTorch fallback." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in _PROTOTYPES.items():
            fn = getattr(lib, name)
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
        if os.environ.get("MF_CONV_IMPL"):            # diagnostics only: 1 = CUDA-core cross-check kernels
            lib.mf_set_conv_impl(int(os.environ["MF_CONV_IMPL"]))
    return _lib


def call(name, *args):
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (name, rc, lib.mf_last_error().decode()))
    return rc


def ptr(t):
    """device pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream
