"""ctypes binding of libgoliath_b200.so — the thin C-ABI extension (include/goliath_b200.h).

The product path has NO CPU fallback: if the CUDA library is missing, or a tensor is not on a CUDA
device, every op raises.  Build with `python -m goliath_b200.build` (nvcc, sm_90a).
"""
import ctypes
import os
import re
import types

import torch  # noqa: F401  (loads libcudart.so.12 first so the C library binds to the same runtime)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgoliath_b200.so")
_lib = None
_kernels = None

HEADER = os.path.join(_HERE, os.pardir, "include", "goliath_b200.h")

# C parameter / return type -> ctypes type; every pointer binds as c_void_p
_CTYPES = {"int": ctypes.c_int, "float": ctypes.c_float, "int64_t": ctypes.c_int64, "long long": ctypes.c_int64,
           "size_t": ctypes.c_size_t, "unsigned long long": ctypes.c_ulonglong, "void": None}


class GoliathB200Error(RuntimeError):
    pass


def _ctype(t, proto, named=True):
    """ctypes type of the C type `t` (a parameter with its name when `named`, else a return type) of `proto`."""
    if "*" in t:
        return ctypes.c_void_p
    key = " ".join(re.sub(r"\bconst\b", " ", t).split()[:-1 if named else None])
    if key not in _CTYPES or (named and key == "void"):
        raise GoliathB200Error("unsupported C type %r in prototype %s" % (t, proto))
    return _CTYPES[key]


def parse_header(text):
    """name -> (restype, argtypes) for every `ret gb_name(params);` prototype in `text`, and the set of launchers:
    the entry points whose last parameter is `void* stream`.  A type outside _CTYPES raises, naming the prototype."""
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    sigs, launchers = {}, set()
    for ret, name, params in re.findall(r"^\s*([A-Za-z_][\w ]*?\**)\s*\b(gb_\w+)\s*\(([^)]*)\)\s*;", text,
                                        flags=re.M):
        params = [" ".join(p.split()) for p in params.split(",")]
        if params == ["void"]:
            params = []
        proto = "%s(%s)" % (name, ", ".join(params))
        sigs[name] = (_ctype(ret, proto, named=False), [_ctype(p, proto) for p in params])
        if params and re.fullmatch(r"void ?\* ?stream", params[-1]):
            launchers.add(name)
    return sigs, frozenset(launchers)


with open(HEADER) as _f:
    # name -> (restype, argtypes) of every symbol include/goliath_b200.h declares
    SIGNATURES, LAUNCHERS = parse_header(_f.read())


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GoliathB200Error(
                "libgoliath_b200.so is not built (%s). Run `python -m goliath_b200.build`; there is no CPU "
                "fallback." % LIB_PATH
            )
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def _launcher(fn, name):
    """`fn` called as the header declares it without the trailing stream: a tensor passes as its data_ptr(), None as
    NULL, anything else unchanged.  It launches on the current stream of the first CUDA tensor's device (else of the
    current device) and raises GoliathB200Error on a nonzero return.  No synchronisation, no allocation: safe inside
    CUDA graph capture."""
    Tensor, current_device, current_stream = torch.Tensor, torch.cuda.current_device, torch.cuda.current_stream

    def launch(*args):
        dev = None
        for a in args:
            if isinstance(a, Tensor) and a.is_cuda:
                dev = a.get_device()
                break
        ptrs = [a.data_ptr() if isinstance(a, Tensor) else a for a in args]
        if dev is None or dev == current_device():
            err = fn(*ptrs, current_stream(dev).cuda_stream)
        else:
            with torch.cuda.device(dev):
                err = fn(*ptrs, current_stream(dev).cuda_stream)
        if err != 0:
            raise GoliathB200Error("%s failed: CUDA error %d" % (name, err))
        return 0

    launch.__name__ = name
    return launch


def kernels():
    """Every entry point of the header as an attribute of one namespace: the launchers (LAUNCHERS) wrapped by
    _launcher, the queries, setters and sizers as the plain ctypes functions."""
    global _kernels
    if _kernels is None:
        L = lib()
        _kernels = types.SimpleNamespace(**{n: _launcher(getattr(L, n), n) if n in LAUNCHERS else getattr(L, n)
                                            for n in SIGNATURES})
    return _kernels


def check(err, what):
    if err != 0:
        raise GoliathB200Error("%s failed: CUDA error %d" % (what, err))


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_ptr(device=None):
    return torch.cuda.current_stream(device).cuda_stream


def check_input(t, name, dtype=torch.float32):
    """Same contract as the reference's CHECK_INPUT (extensions/sgutils/utils.h): CUDA + contiguous."""
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor" % name)
    if not t.is_contiguous():
        raise RuntimeError("%s must be contiguous" % name)
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError("%s must have dtype %s (got %s)" % (name, dtype, t.dtype))
