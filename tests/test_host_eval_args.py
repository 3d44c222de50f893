"""CPU tests of the argument checks of mrx_mask_extents, mrx_mask_overlaps and mrx_mask_matches (no
device needed: every refused call returns before anything reaches the GPU)."""
import ctypes as C

import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N

P = C.c_void_p(16)


def _refused(rc, fn, what):
    assert rc == -1, what
    assert N.load().mrx_last_error().decode().startswith(fn + ":"), what


@pytest.mark.parametrize("what,null,B,R", [
    *[(f"null pointer {i}", i, 1, 100) for i in range(7)],
    ("null pointer with B = 0", 6, 0, 100),
    ("B > MRX_MAX_BATCH", None, N.MRX_MAX_BATCH + 1, 100),
    ("B < 0", None, -1, 100),
    ("R = 0", None, 1, 0),
    ("R = 65535", None, 1, 65535),
])
def test_extents_refuses_bad_arguments(what, null, B, R):
    p = [P] * 7
    if null is not None:
        p[null] = None
    _refused(N.load().mrx_mask_extents(*p, B, R, None), "mrx_mask_extents", what)


def _overlaps_args(null=None, B=1, R1=100, R2=100, base=P):
    p = [base, P, P, P, P, base, P, P, P, P, P, P]
    if null is not None:
        p[null] = None
    return (*p[:5], R1, *p[5:10], R2, p[10], p[11], B, None)


@pytest.mark.parametrize("what,kw", [
    *[(f"null pointer {i}", dict(null=i)) for i in range(12)],
    ("null pointer with B = 0", dict(null=11, B=0)),
    ("B > MRX_MAX_BATCH", dict(B=N.MRX_MAX_BATCH + 1)),
    ("B < 0", dict(B=-1)),
    ("R1 = 0", dict(R1=0)),
    ("R2 = 0", dict(R2=0)),
    ("R2 = 65535", dict(R2=65535)),
    ("misaligned planes", dict(base=C.c_void_p(18))),
])
def test_overlaps_refuses_bad_arguments(what, kw):
    _refused(N.load().mrx_mask_overlaps(*_overlaps_args(**kw)), "mrx_mask_overlaps", what)


def _matches_args(null=None, B=1, R1=100, R2=100, T=1, dtype=N.MRX_F32):
    p = [P] * 10
    thr = N.double_array([0.5] * max(T, 1))
    args = [p[0], p[1], p[2], p[3], dtype, p[4], p[5], thr, T, 0.0, p[6], p[7], p[8], B, R1, R2, None]
    if null is not None:
        args[[0, 1, 2, 3, 5, 6, 7, 10, 11, 12][null]] = None
    return args


@pytest.mark.parametrize("what,kw", [
    *[(f"null pointer {i}", dict(null=i)) for i in range(10)],
    ("null thresholds with B = 0", dict(null=6, B=0)),
    ("B > MRX_MAX_BATCH", dict(B=N.MRX_MAX_BATCH + 1)),
    ("B < 0", dict(B=-1)),
    ("R1 = 0", dict(R1=0)),
    ("R1 = 65535", dict(R1=65535)),
    ("R2 = 0", dict(R2=0)),
    ("T = 0", dict(T=0)),
    ("T above MRX_MAX_IOU_THRESHOLDS", dict(T=N.MRX_MAX_IOU_THRESHOLDS + 1)),
    ("bad score dtype", dict(dtype=2)),
])
def test_matches_refuses_bad_arguments(what, kw):
    _refused(N.load().mrx_mask_matches(*_matches_args(**kw)), "mrx_mask_matches", what)


def test_empty_batches_launch_nothing():
    lib = N.load()
    assert lib.mrx_mask_extents(*[P] * 7, 0, 100, None) == 0
    assert lib.mrx_mask_overlaps(*_overlaps_args(B=0)) == 0
    assert lib.mrx_mask_matches(*_matches_args(B=0, T=N.MRX_MAX_IOU_THRESHOLDS)) == 0
