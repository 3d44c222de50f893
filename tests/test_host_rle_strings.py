"""CPU tests of mrx_rle_strings' argument checks (no device needed: every refused call returns
before anything reaches the GPU)."""
import ctypes as C

import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N


@pytest.mark.parametrize("what,null,B,R", [
    ("null run lengths", 0, 1, 100),
    ("null instance offsets", 1, 1, 100),
    ("null counts", 2, 1, 100),
    ("null string offsets", 3, 1, 100),
    ("null strings", 4, 1, 100),
    ("null pointer with B = 0", 4, 0, 100),
    ("B > MRX_MAX_BATCH", None, N.MRX_MAX_BATCH + 1, 100),
    ("B < 0", None, -1, 100),
    ("R = 0", None, 1, 0),
    ("R = 65535", None, 1, 65535),
])
def test_rle_strings_refuses_bad_arguments(what, null, B, R):
    lib = N.load()
    p = [C.c_void_p(16)] * 5
    if null is not None:
        p[null] = None
    assert lib.mrx_rle_strings(p[0], p[1], p[2], B, R, p[3], p[4], None) == -1, what
    assert lib.mrx_last_error().decode().startswith("mrx_rle_strings:"), what


def test_rle_strings_empty_batch_launches_nothing():
    lib = N.load()
    p = C.c_void_p(16)
    assert lib.mrx_rle_strings(p, p, p, 0, 100, p, p, None) == 0


def test_string_bound():
    assert N.rle_string_bound(0, 1) == 7
    assert N.rle_string_bound(10, 3) == 91
