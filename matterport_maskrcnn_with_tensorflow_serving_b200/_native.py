"""ctypes binding of lib/libmrx.so (C ABI: include/mrx.h).

The header is the only declaration of the ABI: every `#define MRX_<NAME> <integer>` is a module
attribute here, and every `mrx_*` prototype gives the restype and argtypes of its function.  A
pointer parameter takes a torch tensor whose dtype holds the C element type (see `Pointer`).

There is no CPU fallback: if the library is missing or a call fails, this raises.
PyTorch is imported first so that libmrx.so resolves libcudart.so.12 to the CUDA
runtime instance torch already loaded (shared device / stream state).
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
import re

import torch

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
# MRX_LIB=<file name under lib/> selects another build of the library (development only:
# e.g. libmrx_dev.so built with MRX_NVCC_FLAGS=-DMRX_DEV); the default is the shipped one
LIB_PATH = os.path.join(_PKG_DIR, "lib", os.environ.get("MRX_LIB", "libmrx.so"))
HEADER_PATH = os.path.join(os.path.dirname(_PKG_DIR), "include", "mrx.h")


class MrxError(RuntimeError):
    """A libmrx call returned a negative status."""


class Pointer(C.c_void_p):
    """A pointer parameter of the header, one subclass per C element type (`element`).  A torch
    tensor (device, pinned or CPU memory) passes its data_ptr() when it is contiguous and its
    dtype holds the element type; anything else goes through as c_void_p takes it (None, an
    integer address, c_void_p, byref(...), bytes), a ctypes array only when its elements have the
    element's size.  Wrong arguments raise TypeError, which ctypes reports as
    ctypes.ArgumentError."""
    element = "void"


# C element type of a pointer parameter -> (bytes, tensor dtypes that hold it; None: any).
# unsigned int data lives in int32 tensors (torch has few uint32 kernels); void * is the element
# of a void ** out-parameter, given as byref(c_void_p()).
_ELEMENTS = {
    "void": (None, None),
    "unsigned char": (1, (torch.uint8,)),
    "short": (2, (torch.int16,)),
    "int": (4, (torch.int32,)),
    "unsigned int": (4, (torch.int32, torch.uint32)),
    "float": (4, (torch.float32,)),
    "long long": (8, (torch.int64,)),
    "double": (8, (torch.float64,)),
    "void *": (8, ()),
}


def _pointer_type(element, size, dtypes):
    """The `Pointer` subclass of one element type."""
    dtypes = None if dtypes is None else frozenset(dtypes)

    # runs for every pointer of every launch: its names are locals
    def from_param(obj, _tensor=torch.Tensor, _void_p=C.c_void_p):
        if isinstance(obj, _tensor):
            if (dtypes is None or obj.dtype in dtypes) and obj.is_contiguous():
                return _void_p(obj.data_ptr())
            got = str(obj.dtype) if obj.is_contiguous() else "non-contiguous"
            raise TypeError(f"{element} * parameter: got a {got} tensor")
        if isinstance(obj, C.Array) and size is not None and C.sizeof(obj._type_) != size:
            raise TypeError(f"{element} * parameter: got an array of {obj._type_.__name__}")
        return _void_p.from_param(obj)

    return type(f"Pointer[{element}]", (Pointer,),
                {"element": element, "from_param": staticmethod(from_param)})


_POINTERS = {e: _pointer_type(e, size, dtypes) for e, (size, dtypes) in _ELEMENTS.items()}
_SCALARS = {"int": C.c_int, "unsigned int": C.c_uint, "long long": C.c_longlong,
            "unsigned long long": C.c_ulonglong, "double": C.c_double}
_RESTYPES = {"int": C.c_int, "const char *": C.c_char_p}


def _words(decl):
    """A C declaration with one space between its words and around each '*'."""
    return " ".join(decl.replace("*", " * ").split())


def _parameter(fn, param):
    """The ctypes argtype of one parameter declaration (in `_words` form) of function `fn`."""
    m = re.fullmatch(r"(?:const )?([a-z]+(?: [a-z]+)*)((?: \*)*) \w+", param)
    if m is None:
        kind = None
    elif not m.group(2):
        kind = _SCALARS.get(m.group(1))
    else:   # the element type: one '*' fewer
        kind = _POINTERS.get(m.group(1) + " *" * (m.group(2).count("*") - 1))
    if kind is None:
        raise ValueError(f"mrx.h: {fn}: no binding for the parameter {param!r}")
    return kind


def parse_header(text):
    """(constants, signatures) of a header's text: constants {MRX_NAME: int} of every object-like
    `#define MRX_*` (a decimal integer, possibly negative, or `(a << b)`), signatures
    {mrx_name: (restype, argtypes)} of every `mrx_*` prototype.  A define or prototype it cannot
    read, or a type outside its tables, raises ValueError naming it."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    constants = {}
    for name, value in re.findall(r"^[ \t]*#[ \t]*define[ \t]+(MRX_\w+)[ \t]+(\S.*?)[ \t]*$",
                                  text, flags=re.M):
        m = re.fullmatch(r"(-?\d+)|\( *(\d+) *<< *(\d+) *\)", value)
        if m is None:
            raise ValueError(f"mrx.h: {name}: {value!r} is not an integer constant")
        constants[name] = int(m.group(1)) if m.group(1) else int(m.group(2)) << int(m.group(3))
    body = re.sub(r"^[ \t]*#.*$", "", text, flags=re.M)
    signatures = {}
    for ret, fn, params in re.findall(r"([^;{}]*?)\b(mrx_\w+)\s*\(([^;{}]*)\)\s*;", body):
        restype = _RESTYPES.get(_words(ret))
        if restype is None:
            raise ValueError(f"mrx.h: {fn}: no binding for the return type {_words(ret)!r}")
        params = [_words(p) for p in params.split(",")]
        signatures[fn] = (restype, [] if params == ["void"] else
                          [_parameter(fn, p) for p in params])
    unread = sorted(set(re.findall(r"\b(mrx_\w+)\s*\(", body)) - set(signatures))
    if unread:
        raise ValueError(f"mrx.h: cannot read the declaration of {', '.join(unread)}")
    return constants, signatures


def _read_header(header_path=HEADER_PATH):
    with open(header_path) as f:
        return parse_header(f.read())


_CONSTANTS, SIGNATURES = _read_header()   # SIGNATURES: name -> (restype, argtypes)
globals().update(_CONSTANTS)
ABI_VERSION = _CONSTANTS["MRX_ABI_VERSION"]


def contour_scratch_bytes(total_segments):
    """MRX_CONTOUR_SCRATCH_BYTES(S): device scratch of mrx_contours_write for S segments."""
    return 48 * int(total_segments) + 256


def rle_string_bound(total_changes, n_instances):
    """MRX_RLE_STRING_BOUND(T, n): bytes of mrx_rle_strings' output for T value changes (runs
    T + n) over n instances; every count takes at most 7 characters."""
    return 7 * (int(total_changes) + int(n_instances))


_lib = None


def declared_symbols(header_path=HEADER_PATH):
    """Function names declared in include/mrx.h (used by the symbol-export test)."""
    return sorted(_read_header(header_path)[1])


def load(build_if_missing=True):
    """Load libmrx.so (building it in-tree first if it is absent). Raises on failure."""
    global _lib
    if _lib is not None:
        return _lib

    default_lib = os.path.basename(LIB_PATH) == "libmrx.so"
    if build_if_missing and default_lib:
        # cheap when nothing changed (a digest of the sources against lib/libmrx.stamp); a stale
        # library whose ABI number happens to match is rebuilt instead of silently used.  Without
        # nvcc (a deployment box) the prebuilt library is used as it is.
        from . import build as _build
        try:
            _build.build()
        except RuntimeError:
            if not os.path.exists(LIB_PATH):
                raise
    if not os.path.exists(LIB_PATH):
        raise MrxError(f"{LIB_PATH} is missing; run __graft_entry__.build()")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    got = lib.mrx_abi_version()
    if got != ABI_VERSION:
        raise MrxError(f"libmrx ABI {got} != expected {ABI_VERSION}; rebuild the library")
    _lib = lib
    return lib


def check(rc, what):
    if rc != _CONSTANTS["MRX_OK"]:
        msg = load().mrx_last_error()
        raise MrxError(f"{what} failed (status {rc}): {msg.decode() if msg else ''}")


def int_array(values):
    arr = (C.c_int * len(values))(*[int(v) for v in values])
    return arr


def double_array(values):
    arr = (C.c_double * len(values))(*[float(v) for v in values])
    return arr


# The current stream's raw handle.  Every launch asks for it, and the pipeline launches ask
# whether a stream is current on every step: torch.cuda.current_stream() builds a Stream object
# each time (7 us of host time on an H100 host, measured) where this read takes 0.5 us.  These are
# the calls torch's own kernel launchers make; tests/test_gpu_streams.py checks them against
# torch.cuda.current_stream().
def _current_handle(device_index):
    return torch._C._cuda_getCurrentRawStream(device_index)


def stream_ptr(stream=None):
    """cudaStream_t of a torch.cuda.Stream (or the current stream) as an integer."""
    if stream is None:
        return C.c_void_p(_current_handle(torch._C._cuda_getDevice()))
    return C.c_void_p(stream.cuda_stream)


def on_stream(stream):
    """The context of the pipeline launches' `stream` argument: `torch.cuda.stream(stream)`, or
    none when `stream` is None or already current on the current device.  Callers hand these
    launches the current stream on every step, and entering torch's context costs 19 us of host
    time on an H100 host (measured), which the device waits for ahead of a 0.44 ms packed expand
    step."""
    if stream is None or (stream.device_index == torch._C._cuda_getDevice() and
                          stream.cuda_stream == _current_handle(stream.device_index)):
        return contextlib.nullcontext()
    return torch.cuda.stream(stream)


class DeviceBytes:
    """`__cuda_array_interface__` view of raw device memory, so that torch can wrap memory it did
    not allocate (peer memory, the canvas of mrx_device_alloc); torch keeps the object alive for
    as long as the tensor's storage lives."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1",
                                         "data": (int(ptr), False), "version": 2}


def require_cuda():
    if not torch.cuda.is_available():
        raise MrxError("no CUDA device: this package has no CPU fallback "
                       "(the CPU restatement under oracle/ is test infrastructure only)")
