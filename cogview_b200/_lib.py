"""ctypes binding of libcogview_b200.so (the C ABI declared in include/cogview_b200.h).

The argument and result types of every cv_* function are parsed from that header, so the header is the only place a
signature is written down; a type the parser does not know fails when the library is loaded, not inside a kernel.
There is no CPU or PyTorch fallback: if the library is missing or a call fails, this raises.
"""
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libcogview_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "cogview_b200.h")

_lib = None

_SCALARS = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "long long": ctypes.c_longlong, "float": ctypes.c_float,
            "uint64_t": ctypes.c_uint64, "uint32_t": ctypes.c_uint32}
_PROTOTYPE = re.compile(r"^\s*([A-Za-z_][\w ]*?\**)\s*\b(cv_\w+)\s*\(([^)]*)\)\s*;", re.M)


class CogViewB200Error(RuntimeError):
    pass


def _ctype(name, decl, is_return=False):
    if "*" in decl:
        return ctypes.c_char_p if is_return and decl.replace(" ", "") == "constchar*" else ctypes.c_void_p
    t = " ".join(w for w in decl.split() if w != "const")
    if t not in _SCALARS:
        raise CogViewB200Error("%s: C type %r has no ctypes mapping" % (name, decl))
    return _SCALARS[t]


def signatures(text):
    """{name: (restype, argtypes)} for every cv_* prototype of the header text `text`."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    sigs = {}
    for ret, name, params in _PROTOTYPE.findall(text):
        params = params.strip()
        argtypes = []
        if params != "void":
            for p in params.split(","):
                decl = re.sub(r"\w+$", "", p.strip())          # drop the parameter name
                argtypes.append(_ctype(name, decl.strip()))
        sigs[name] = (_ctype(name, ret.strip(), is_return=True), argtypes)
    return sigs


def lib():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CogViewB200Error(
                "libcogview_b200.so not found at %s — build it with `python -m cogview_b200.csrc.build` "
                "(there is no fallback path)" % LIB_PATH)
        handle = ctypes.CDLL(LIB_PATH)
        with open(HEADER_PATH) as f:
            for name, (restype, argtypes) in signatures(f.read()).items():
                fn = getattr(handle, name)
                fn.restype, fn.argtypes = restype, argtypes
        _lib = handle
    return _lib


def check(rc, name="call"):
    if rc != 0:
        msg = lib().cv_last_error()
        raise CogViewB200Error("%s failed (rc=%d): %s" % (name, rc, msg.decode() if msg else "?"))


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return 0 if t is None else t.data_ptr()


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise CogViewB200Error("cogview_b200 kernels need CUDA tensors; got a %s tensor (no CPU fallback)"
                                   % t.device)
