"""CPU tests of the ctypes binding derived from include/mrx.h: the header parser, the constants
it gives, and the pointer parameter type on real calls that return before touching CUDA."""
import ctypes as C

import numpy as np
import pytest
import torch

from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N

SYNTHETIC = """
/* a comment with mrx_not_a_function(int x) in it */
#define MRX_ANSWER   42   /* trailing comment */
#define MRX_NEGATIVE -3
#define MRX_BIG (1 << 30)
#define MRX_LIKE_A_FUNCTION(n) (2 * (n))
int mrx_good(const float *d_in, unsigned int *d_out, void **d_ptr, long long n,
             unsigned long long bytes, double alpha, void *stream);
const char *mrx_text(void);
"""


def test_parser_reads_a_synthetic_header():
    constants, signatures = N.parse_header(SYNTHETIC)
    assert constants == {"MRX_ANSWER": 42, "MRX_NEGATIVE": -3, "MRX_BIG": 1 << 30}
    assert sorted(signatures) == ["mrx_good", "mrx_text"]
    res, args = signatures["mrx_good"]
    assert res is C.c_int
    assert [a.element for a in args[:3]] == ["float", "unsigned int", "void *"]
    assert args[3:6] == [C.c_longlong, C.c_ulonglong, C.c_double]
    assert args[6].element == "void" and all(issubclass(a, N.Pointer) for a in args[:3])
    assert signatures["mrx_text"] == (C.c_char_p, [])


@pytest.mark.parametrize("decl, name", [
    ("int mrx_bad(float x);", "mrx_bad"),                         # scalar outside the table
    ("int mrx_bad(const long *d_x);", "mrx_bad"),                 # element outside the table
    ("float mrx_bad(int x);", "mrx_bad"),                         # return type
    ("int mrx_bad(int (*cb)(int));", "mrx_bad"),                  # a declaration it cannot read
    ("#define MRX_ODD 0x10", "MRX_ODD"),                          # not a decimal constant
])
def test_parser_refuses_what_it_has_no_binding_for(decl, name):
    with pytest.raises(ValueError, match=name):
        N.parse_header(SYNTHETIC + decl + "\n")


def test_constants_of_the_real_header():
    assert N.MRX_MAX_BATCH == 4096
    assert N.MRX_GEOM_INTS == 8
    assert N.MRX_MAX_IOU_THRESHOLDS == 64
    assert N.MRX_MAX_CONTOUR_SEGMENTS == 1 << 30
    assert (N.MRX_OK, N.MRX_E_INVALID, N.MRX_E_UNSUPPORTED) == (0, -1, -2)
    assert N.ABI_VERSION == N.MRX_ABI_VERSION == 17
    assert N.declared_symbols() == sorted(N.SIGNATURES)


def _ranks_args():
    """mrx_coco_ranks over B = 0 images of R = 4 rows: checked, then nothing launched."""
    i32 = lambda *shape: torch.zeros(shape, dtype=torch.int32)   # noqa: E731
    return [i32(1, 4), torch.zeros(1, 4, dtype=torch.float64), N.MRX_F64, i32(1), i32(3), 3, 10,
            i32(1, 4), i32(1, 4), torch.zeros(1, 4, dtype=torch.uint8), i32(1, 4), 0, 4, None]


def _ranks(**replace):
    args = _ranks_args()
    for k, v in replace.items():
        args[int(k[1:])] = v
    return N.load().mrx_coco_ranks(*args)


def test_tensors_of_the_declared_element_types_reach_the_library():
    assert _ranks() == N.MRX_OK
    assert _ranks(a1=torch.zeros(1, 4, dtype=torch.float32), a2=N.MRX_F32) == N.MRX_OK  # void *


@pytest.mark.parametrize("what, k, bad", [
    ("int64 tensor for const int *", 0, torch.zeros(1, 4, dtype=torch.int64)),
    ("bool tensor for unsigned char *", 9, torch.zeros(1, 4, dtype=torch.bool)),
    ("non-contiguous view", 0, torch.zeros(4, 2, dtype=torch.int32).t()),
    ("NumPy array", 0, np.zeros((1, 4), np.int32)),
    ("array of double for const int *", 4, N.double_array([0, 1, 2])),
])
def test_wrong_pointer_arguments_raise(what, k, bad):
    with pytest.raises(C.ArgumentError):
        _ranks(**{f"a{k}": bad})


def test_raw_pointers_reach_the_library():
    assert _ranks(a0=None) == N.MRX_E_INVALID             # NULL: the library's own check
    assert N.load().mrx_last_error().decode().startswith("mrx_coco_ranks:")
    x = C.c_int(0)
    for raw in (16, C.c_void_p(16), C.byref(x), N.int_array([0, 0, 0])):
        assert _ranks(a0=raw) == N.MRX_OK


def test_unsigned_int_takes_int32_and_uint32_bits():
    lib = N.load()
    for dt in (torch.int32, torch.uint32):
        runs = torch.zeros(4, dtype=dt)
        assert lib.mrx_rle_strings(runs, 16, 16, 0, 4, 16, 16, None) == N.MRX_OK
    with pytest.raises(C.ArgumentError):
        lib.mrx_rle_strings(torch.zeros(4, dtype=torch.int64), 16, 16, 0, 4, 16, 16, None)
