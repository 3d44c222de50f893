"""The output slots of a planned batch (mrx.h, "Output slots"): every entry point that writes or
reads the canvas or the packed planes checks them the same way, and mrx_pack_masks refuses a
batch before it writes anything."""
import ctypes as C

import numpy as np
import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import BatchLayout


# The entry points that write or read the slots, as (base, off, counts, geom, B, R) -> status;
# every other argument is a non-null placeholder and every extent is valid.
def _slot_entry_points(lib):
    p = C.c_void_p(16)
    ll = C.c_longlong
    return {
        "mrx_mask_expand": lambda base, off, cnt, geom, B, R: lib.mrx_mask_expand(
            p, p, p, cnt, geom, off, base, B, R, 28, 28, 0, 0, p, None),
        "mrx_mask_expand_values": lambda base, off, cnt, geom, B, R: lib.mrx_mask_expand_values(
            p, p, p, cnt, geom, off, base, p, B, R, 28, 28, p, None),
        "mrx_mask_expand_packed": lambda base, off, cnt, geom, B, R: lib.mrx_mask_expand_packed(
            p, p, p, cnt, geom, off, base, B, R, 28, 28, 16, p, None),
        "mrx_pack_masks": lambda base, off, cnt, geom, B, R: lib.mrx_pack_masks(
            base, off, cnt, geom, p, p, B, R, 16, 16, None),
        "mrx_composite_masks": lambda base, off, cnt, geom, B, R: lib.mrx_composite_masks(
            base, off, cnt, geom, p, p, p, p, C.c_double(0.5), p, B, R, ll(256), None),
        "mrx_contours_count": lambda base, off, cnt, geom, B, R: lib.mrx_contours_count(
            base, off, cnt, geom, p, p, p, B, R, 16, None),
        "mrx_contours_write": lambda base, off, cnt, geom, B, R: lib.mrx_contours_write(
            base, off, cnt, geom, p, p, p, ll(10), ll(4), p, p, p, p, B, R, 16, None),
    }


# (what is wrong, null argument, B, R); every row is MRX_E_INVALID.  The R rows take B = 0, so
# that a build without the R bound returns at B = 0 instead of launching on placeholders.
BAD_SLOTS = [
    ("null slot base", "base", 1, 100),
    ("null offsets", "off", 1, 100),
    ("null counts", "counts", 1, 100),
    ("null geom", "geom", 1, 100),
    ("B > MRX_MAX_BATCH", None, N.MRX_MAX_BATCH + 1, 100),
    ("R = 0", None, 0, 0),
    ("R = 65535", None, 0, 65535),
]


@pytest.mark.parametrize("fn", ["mrx_mask_expand", "mrx_mask_expand_values",
                                "mrx_mask_expand_packed", "mrx_pack_masks", "mrx_composite_masks",
                                "mrx_contours_count", "mrx_contours_write"])
def test_slot_checks_agree(fn):
    """Every entry point that writes or reads the output slots refuses the same bad slots with the
    same status and names itself in the message."""
    lib = N.load()
    call = _slot_entry_points(lib)[fn]
    for what, null, B, R in BAD_SLOTS:
        args = {k: (None if k == null else C.c_void_p(16)) for k in ("base", "off", "counts", "geom")}
        assert call(args["base"], args["off"], args["counts"], args["geom"], B, R) == -1, what
        msg = lib.mrx_last_error().decode()
        assert msg.startswith(fn + ":"), (what, msg)


@pytest.mark.gpu
def test_pack_masks_refuses_before_writing(cuda_device):
    """Past the largest R whose pack_bytes_kernel fits in shared memory, mrx_pack_masks returns
    MRX_E_UNSUPPORTED with the packed buffer untouched, although the direct form of
    pack_quads_kernel could take the image with N % 4 == 0.  At the largest R that fits, both
    forms write np.packbits of the canvas."""
    import torch

    lib = N.load()
    sms, major, minor, optin = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    N.check(lib.mrx_device_props(torch.cuda.current_device(), C.byref(sms), C.byref(major),
                                 C.byref(minor), C.byref(optin)), "mrx_device_props")
    r_fit = (optin.value - 32) // 256      # pack_bytes_kernel: 256 * R + 32 bytes
    # eight runs of at least 32 * R + 16 bytes: too many for the staged form, so it is the direct
    # form of pack_quads_kernel (N % 4 == 0) and pack_bytes_kernel (the other image)
    assert 8 * (32 * r_fit + 16) + 1024 > optin.value // 4
    counts = [40, 37]
    rng = np.random.default_rng(5)
    masks = [rng.random((16, 16, n)) < 0.4 for n in counts]
    for R, status in [(r_fit + 1, -2), (r_fit, 0)]:
        layout = BatchLayout([[16, 16, 16, 16, 0, 0, 16, 16]] * 2, R)
        canvas = np.zeros(int(layout.canvas_off[-1]), np.uint8)
        for b, m in enumerate(masks):
            lo, hi = layout.canvas_span(b, counts[b])
            canvas[lo:hi] = m.reshape(-1)
        dev = torch.device("cuda", torch.cuda.current_device())
        d_canvas = torch.from_numpy(canvas).to(dev)
        d_canvas_off = torch.from_numpy(layout.canvas_off[:-1].copy()).to(dev)
        d_packed_off = torch.from_numpy(layout.packed_off[:-1].copy()).to(dev)
        d_counts = torch.tensor(counts, dtype=torch.int32, device=dev)
        d_geom = torch.from_numpy(layout.geom).to(dev)
        d_packed = torch.full((int(layout.packed_off[-1]),), 0xAA, dtype=torch.uint8, device=dev)
        rc = lib.mrx_pack_masks(d_canvas, d_canvas_off, d_counts, d_geom, d_packed, d_packed_off,
                                2, R, 16, 16, N.stream_ptr(None))
        assert rc == status, (R, lib.mrx_last_error())
        packed = d_packed.cpu().numpy()
        if status:
            assert lib.mrx_last_error().decode().startswith("mrx_pack_masks:")
            assert (packed == 0xAA).all(), f"R={R}: refused, but the packed buffer was written"
            continue
        for b, m in enumerate(masks):
            lo, hi = layout.packed_span(b, counts[b])
            want = np.packbits(m.transpose(2, 0, 1), axis=-1)
            assert np.array_equal(packed[lo:hi].reshape(layout.packed_shape(b, counts[b])), want), b
