"""ctypes binding of the C-ABI library (include/unispeech_b200.h).

The product path has no CPU / PyTorch fallback: if the shared library is missing, or the device is not
sm_90, calls raise.  Functions take torch CUDA tensors and pass raw device pointers + the current stream.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import Optional

import torch

_LIB_PATH = Path(__file__).resolve().parent / "lib" / "libunispeech_b200.so"
_lib = None


class Epilogue(C.Structure):
    _fields_ = [
        ("bias", C.c_void_p),
        ("res1", C.c_void_p), ("res1_bs", C.c_longlong), ("res1_ld", C.c_longlong),
        ("res2", C.c_void_p), ("res2_bs", C.c_longlong), ("res2_ld", C.c_longlong),
        ("gelu_aux", C.c_void_p), ("aux_bs", C.c_longlong), ("aux_ld", C.c_longlong),
        ("out_pre", C.c_void_p), ("pre_bs", C.c_longlong), ("pre_ld", C.c_longlong),
        ("colsum", C.c_void_p),
        ("gelu", C.c_int),
        ("dgelu", C.c_int),
    ]


def lib_path() -> Path:
    return _LIB_PATH


def load():
    """Load the shared library (once). Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise RuntimeError(
            f"{_LIB_PATH} is missing: build it with `python -m unispeech_b200.build` "
            "(there is no CPU or PyTorch fallback for the hot path)"
        )
    lib = C.CDLL(str(_LIB_PATH))
    _bind_prototypes(lib)
    _lib = lib
    return lib


_CTYPES = {"int": C.c_int, "long long": C.c_longlong, "unsigned long long": C.c_ulonglong, "size_t": C.c_size_t,
           "uint32_t": C.c_uint32, "float": C.c_float, "double": C.c_double, "b200s_stream": C.c_void_p, "unsigned": C.c_uint,
           "unsigned int": C.c_uint, "uint8_t": C.c_uint8, "int64_t": C.c_int64}
_RESTYPES = {"int": C.c_int, "long long": C.c_longlong, "uint32_t": C.c_uint32, "const char*": C.c_char_p, "void": None,
             "double": C.c_double, "float": C.c_float}


def _bind_prototypes(lib):
    """Declare `argtypes` / `restype` of every entry point ONCE, from the prototypes of include/unispeech_b200.h.  The wrappers
    then pass plain Python ints / floats (raw device pointers, strides, sizes) instead of one ctypes object per argument
    (15-20 arguments per call, ~6400 calls per WavLM-Large step)."""
    import re
    hdr = Path(__file__).resolve().parent.parent / "include" / "unispeech_b200.h"
    src = hdr.read_text()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    protos = re.findall(r"\b(int|long long|uint32_t|const char\s*\*|void|double|float)\s+(b200s_\w+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S)
    if len(protos) < 40:
        raise RuntimeError(f"could not read the C prototypes from {hdr}")
    for ret, name, params in protos:
        args = []
        if params.strip() not in ("", "void"):
            for prm in params.split(","):
                prm = " ".join(prm.split())
                if "*" in prm:
                    args.append(C.c_void_p)
                    continue
                t = re.sub(r"\b\w+$", "", prm).strip() if re.search(r"\s\w+$", prm) else prm
                t = t.replace("const ", "").strip()
                if t not in _CTYPES:
                    raise RuntimeError(f"{hdr}: unknown parameter type {prm!r} in {name}")
                args.append(_CTYPES[t])
        fn = getattr(lib, name, None)
        if fn is None:
            raise RuntimeError(f"{_LIB_PATH} does not export {name} (stale build? run `python -m unispeech_b200.build`)")
        fn.argtypes = args
        fn.restype = _RESTYPES[" ".join(ret.split()).replace(" *", "*")]


def _check(rc: int):
    if rc != 0:
        msg = load().b200s_last_error()
        raise RuntimeError(f"unispeech_b200 C-ABI call failed ({rc}): {msg.decode() if msg else '?'}")


def check_device():
    _check(load().b200s_check_device())


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def stream_ptr() -> int:
    """Raw cudaStream_t of torch's current stream (an int: every entry point has its argtypes declared).
    `torch.cuda.current_stream()` costs ~13 us per call (device-index and availability checks) and is needed once per kernel
    launch, so the raw C accessor is used when present."""
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


def ptr(t: Optional[torch.Tensor]) -> int:
    """Raw device (or host) address of a tensor's first element, 0 for None."""
    return 0 if t is None else t.data_ptr()


def ll(v) -> int:
    return int(v)


_fn_cache = {}


def _resolve(name: str):
    fn = getattr(load(), name)
    if fn.argtypes is None:   # a symbol without a prototype in the header would get 32-bit ints for its pointers
        raise RuntimeError(f"{name} has no prototype in include/unispeech_b200.h")
    _fn_cache[name] = fn
    return fn


def call(name: str, *args):
    fn = _fn_cache.get(name)
    if fn is None:
        fn = _resolve(name)
    rc = fn(*args)
    if rc:
        _check(rc)


def make_epilogue(bias=None, res1=None, res1_bs=0, res1_ld=0, res2=None, res2_bs=0, res2_ld=0,
                  gelu_aux=None, aux_bs=0, aux_ld=0, out_pre=None, pre_bs=0, pre_ld=0, colsum=None,
                  gelu=False, dgelu=False) -> Epilogue:
    e = Epilogue()
    e.bias = bias.data_ptr() if bias is not None else None
    e.res1 = res1.data_ptr() if res1 is not None else None
    e.res1_bs, e.res1_ld = int(res1_bs), int(res1_ld)
    e.res2 = res2.data_ptr() if res2 is not None else None
    e.res2_bs, e.res2_ld = int(res2_bs), int(res2_ld)
    e.gelu_aux = gelu_aux.data_ptr() if gelu_aux is not None else None
    e.aux_bs, e.aux_ld = int(aux_bs), int(aux_ld)
    e.out_pre = out_pre.data_ptr() if out_pre is not None else None
    e.pre_bs, e.pre_ld = int(pre_bs), int(pre_ld)
    e.colsum = colsum.data_ptr() if colsum is not None else None
    e.gelu = int(gelu)    # 1: out_pre <- pre-activation, 2: out_pre <- gelu'(pre-activation)
    e.dgelu = int(dgelu)  # 1: aux is the pre-activation, 2: aux already is gelu'(.)
    return e
