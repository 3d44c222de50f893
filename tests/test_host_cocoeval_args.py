"""CPU tests of the argument checks of mrx_coco_ranks, mrx_coco_ious and mrx_coco_match (no device
needed: every refused call returns before anything reaches the GPU)."""
import ctypes as C

import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N

P = C.c_void_p(16)


def _refused(rc, fn, what):
    assert rc == -1, what
    assert N.load().mrx_last_error().decode().startswith(fn + ":"), what


def _ranks_args(null=None, B=1, R=100, C_=81, max_det=100, dtype=N.MRX_F32):
    p = [P] * 8
    if null is not None:
        p[null] = None
    return (p[0], p[1], dtype, p[2], p[3], C_, max_det, p[4], p[5], p[6], p[7], B, R, None)


@pytest.mark.parametrize("what,kw", [
    *[(f"null pointer {i}", dict(null=i)) for i in range(8)],
    ("null pointer with B = 0", dict(null=7, B=0)),
    ("B > MRX_MAX_BATCH", dict(B=N.MRX_MAX_BATCH + 1)),
    ("B < 0", dict(B=-1)),
    ("R = 0", dict(R=0)),
    ("R = 65535", dict(R=65535)),
    ("C = 0", dict(C_=0)),
    ("max_det = 0", dict(max_det=0)),
    ("bad score dtype", dict(dtype=2)),
])
def test_ranks_refuses_bad_arguments(what, kw):
    _refused(N.load().mrx_coco_ranks(*_ranks_args(**kw)), "mrx_coco_ranks", what)


def _ious_args(null=None, B=1, R1=100, R2=100, base=P):
    p = [base, P, P, P, P, P, P, base, P, P, P, P, P, P, P, P]
    if null is not None:
        p[null] = None
    return (*p[:7], R1, *p[7:14], R2, p[14], p[15], B, None)


@pytest.mark.parametrize("what,kw", [
    *[(f"null pointer {i}", dict(null=i)) for i in range(16)],
    ("null pointer with B = 0", dict(null=15, B=0)),
    ("B > MRX_MAX_BATCH", dict(B=N.MRX_MAX_BATCH + 1)),
    ("B < 0", dict(B=-1)),
    ("R1 = 0", dict(R1=0)),
    ("R1 = 65535", dict(R1=65535)),
    ("R2 = 0", dict(R2=0)),
    ("R2 = 65535", dict(R2=65535)),
    ("misaligned planes", dict(base=C.c_void_p(18))),
])
def test_ious_refuses_bad_arguments(what, kw):
    _refused(N.load().mrx_coco_ious(*_ious_args(**kw)), "mrx_coco_ious", what)


def _match_args(null=None, B=1, R1=100, R2=100, T=10, A=4):
    p = [P] * 12
    thr = N.double_array([0.5] * max(T, 1))
    rng = N.double_array([0.0, 1e10] * max(A, 1))
    args = [*p[:10], thr, T, rng, A, p[10], p[11], B, R1, R2, None]
    if null is not None:
        args[[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 15][null]] = None
    return args


@pytest.mark.parametrize("what,kw", [
    *[(f"null pointer {i}", dict(null=i)) for i in range(14)],
    ("null thresholds with B = 0", dict(null=10, B=0)),
    ("B > MRX_MAX_BATCH", dict(B=N.MRX_MAX_BATCH + 1)),
    ("B < 0", dict(B=-1)),
    ("R1 = 0", dict(R1=0)),
    ("R1 = 65535", dict(R1=65535)),
    ("R2 = 0", dict(R2=0)),
    ("R2 = 65535", dict(R2=65535)),
    ("T = 0", dict(T=0)),
    ("T above MRX_MAX_IOU_THRESHOLDS", dict(T=N.MRX_MAX_IOU_THRESHOLDS + 1)),
    ("A = 0", dict(A=0)),
    ("A above MRX_MAX_AREA_RANGES", dict(A=N.MRX_MAX_AREA_RANGES + 1)),
])
def test_match_refuses_bad_arguments(what, kw):
    _refused(N.load().mrx_coco_match(*_match_args(**kw)), "mrx_coco_match", what)


def test_empty_batches_launch_nothing():
    lib = N.load()
    assert lib.mrx_coco_ranks(*_ranks_args(B=0)) == 0
    assert lib.mrx_coco_ious(*_ious_args(B=0)) == 0
    assert lib.mrx_coco_match(*_match_args(B=0, T=N.MRX_MAX_IOU_THRESHOLDS,
                                           A=N.MRX_MAX_AREA_RANGES)) == 0
