"""Response decode / request encode of the TF-Serving call without the Python list detour
(SURVEY.md 8f rank 1; reference: serve.py:49-76 and :131-136).

The reference turns `result.outputs[name].float_val` -- a protobuf repeated field -- into an
ndarray with `np.array(...)`: every float becomes a Python object first.  For the mask tensor
(100 x 28 x 28 x 81 = 6.35 M floats) that costs ~0.9 s per image on this host, ~400x the
whole device-side unmold.  On the wire a packed repeated float field IS a little-endian
float32 array, so the values can be taken straight from the serialized message:

    tensor_proto_to_ndarray(outputs[name])      # ~0.02 s: serialize once (C++), slice, frombuffer

This module parses just enough of the protobuf wire format of `tensorflow.TensorProto`
(public schema: dtype = 1, tensor_shape = 2, tensor_content = 4, float_val = 5,
double_val = 6; TensorShapeProto.dim = 2, Dim.size = 1) to do that, and builds the request
tensors the way `tf.make_tensor_proto(ndarray)` does (values in `tensor_content`).  It has no
TensorFlow dependency; anything with `SerializeToString()` or raw bytes is accepted.
"""
from __future__ import annotations

import numpy as np

DT_FLOAT = 1
DT_DOUBLE = 2
_NP_OF_DT = {DT_FLOAT: np.dtype("<f4"), DT_DOUBLE: np.dtype("<f8")}
_DT_OF_NP = {np.dtype("float32"): DT_FLOAT, np.dtype("float64"): DT_DOUBLE}


def _varint(buf, pos):
    """Decode one base-128 varint at `pos`; returns (value, next_pos)."""
    result = 0
    shift = 0
    while True:
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7
        if shift > 63:
            raise ValueError("malformed varint")


def _fields(buf, start=0, end=None):
    """Yield (field_number, wire_type, value_or_slice_bounds) over one message's bytes.
    Length-delimited values are yielded as (lo, hi) bounds into `buf` (no copy)."""
    pos = start
    end = len(buf) if end is None else end
    while pos < end:
        key, pos = _varint(buf, pos)
        num, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
            yield num, wt, v
        elif wt == 1:
            yield num, wt, (pos, pos + 8)
            pos += 8
        elif wt == 2:
            n, pos = _varint(buf, pos)
            yield num, wt, (pos, pos + n)
            pos += n
        elif wt == 5:
            yield num, wt, (pos, pos + 4)
            pos += 4
        else:
            raise ValueError(f"unsupported wire type {wt}")
    if pos != end:
        raise ValueError("truncated message")


def _shape_of(buf, lo, hi):
    dims = []
    for num, wt, v in _fields(buf, lo, hi):
        if num == 2 and wt == 2:                    # TensorShapeProto.dim
            size = 0
            for n2, w2, v2 in _fields(buf, v[0], v[1]):
                if n2 == 1 and w2 == 0:             # Dim.size (int64 varint)
                    size = v2 - (1 << 64) if v2 >= (1 << 63) else v2
            dims.append(size)
    return dims


def tensor_proto_to_ndarray(tensor, dtype=None):
    """ndarray of a TensorProto given as a message (anything with SerializeToString) or as
    serialized bytes.  Values come from `tensor_content` if present, else from the packed (or
    unpacked) `float_val` / `double_val`; the result is shaped by `tensor_shape` when that is
    present and consistent, else 1-D.  No per-element Python objects are created.
    `dtype`: optional final dtype (e.g. np.float64 to match `np.array(float_val)`)."""
    buf = tensor if isinstance(tensor, (bytes, bytearray, memoryview)) else tensor.SerializeToString()
    buf = bytes(buf) if not isinstance(buf, bytes) else buf
    dt = None
    shape = None
    content = None
    packed = []          # (field dtype, lo, hi) runs of packed values
    singles = []         # (field dtype, lo, hi) unpacked elements
    for num, wt, v in _fields(buf):
        if num == 1 and wt == 0:
            dt = v
        elif num == 2 and wt == 2:
            shape = _shape_of(buf, v[0], v[1])
        elif num == 4 and wt == 2:
            content = v
        elif num == 5 and wt == 2:
            packed.append((np.dtype("<f4"), v[0], v[1]))
        elif num == 5 and wt == 5:
            singles.append((np.dtype("<f4"), v[0], v[1]))
        elif num == 6 and wt == 2:
            packed.append((np.dtype("<f8"), v[0], v[1]))
        elif num == 6 and wt == 1:
            singles.append((np.dtype("<f8"), v[0], v[1]))
    for d, lo, hi in packed + singles:
        if (hi - lo) % d.itemsize:
            raise ValueError(f"TensorProto value field of {hi - lo} bytes is not a whole number "
                             f"of {d.itemsize}-byte elements")
    if content is not None and content[1] > content[0]:
        if dt not in _NP_OF_DT:
            raise ValueError(f"tensor_content with unsupported dtype enum {dt}")
        if (content[1] - content[0]) % _NP_OF_DT[dt].itemsize:
            raise ValueError(f"tensor_content of {content[1] - content[0]} bytes is not a whole "
                             f"number of {_NP_OF_DT[dt].itemsize}-byte elements")
        arr = np.frombuffer(buf, dtype=_NP_OF_DT[dt], count=(content[1] - content[0]) // _NP_OF_DT[dt].itemsize,
                            offset=content[0])
    elif len(packed) == 1 and not singles:
        d, lo, hi = packed[0]
        arr = np.frombuffer(buf, dtype=d, count=(hi - lo) // d.itemsize, offset=lo)
    elif packed or singles:
        runs = sorted(packed + singles, key=lambda r: r[1])     # wire order = element order
        d = runs[0][0]
        arr = np.concatenate([np.frombuffer(buf, dtype=d, count=(hi - lo) // d.itemsize, offset=lo)
                              for _, lo, hi in runs])
    else:
        arr = np.empty((0,), dtype=_NP_OF_DT.get(dt, np.dtype("<f4")))
    if shape and all(s >= 0 for s in shape):
        if int(np.prod(shape)) != arr.size:
            # TensorFlow allows a single repeated value to stand for a whole tensor; anything
            # else is a malformed message
            if arr.size == 1:
                arr = np.full(shape, arr.reshape(-1)[0], dtype=arr.dtype)
            else:
                raise ValueError(f"tensor_shape {list(shape)} does not match the {arr.size} "
                                 "values of the message")
        else:
            arr = arr.reshape(shape)
    if dtype is not None and arr.dtype != np.dtype(dtype):
        arr = arr.astype(dtype)
    return arr


def decode_predict_outputs(detection_tensor, mask_tensor, det_shape, mask_shape,
                           mask_dtype=np.float32):
    """What serve.py:131-136 computes from `result.outputs[...]`:
        detections = np.array(float_val).reshape((-1, *OUT_DETECTION_SHAPE))   (float64)
        masks      = np.array(float_val).reshape((-1, *OUT_MASK_SHAPE))
    Detections are returned as float64 exactly like the reference (600 values; the box
    arithmetic downstream depends on that dtype).  Masks stay float32 by default: the values
    are the same numbers (float64(float32) is exact), and `unmold_detections` accepts both."""
    det = tensor_proto_to_ndarray(detection_tensor).reshape(-1).astype(np.float64)
    msk = tensor_proto_to_ndarray(mask_tensor).reshape(-1)
    if msk.dtype != np.dtype(mask_dtype):
        msk = msk.astype(mask_dtype)
    return det.reshape((-1, *det_shape)), msk.reshape((-1, *mask_shape))


def _put_varint(out, v):
    v = int(v)
    if v < 0:
        # protobuf encodes negative int64 as the 10-byte two's complement varint
        v &= (1 << 64) - 1
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return


def ndarray_to_tensor_proto_bytes(arr, shape=None):
    """Serialized `TensorProto` for a float32 / float64 ndarray: dtype, tensor_shape and the
    raw values in `tensor_content` -- what `tf.make_tensor_proto(arr, shape=...)` produces for
    an ndarray (serve.py:49-76).  Parse with `TensorProto.FromString` on the TF side, or send
    as-is inside a hand-built PredictRequest."""
    arr = np.ascontiguousarray(arr)
    if arr.dtype not in _DT_OF_NP:
        raise ValueError(f"unsupported dtype {arr.dtype}")
    dims = list(arr.shape if shape is None else shape)
    if any(int(d) < 0 for d in dims):
        raise ValueError(f"negative dimension in shape {dims} (a request tensor is fully shaped)")
    if int(np.prod(dims)) != arr.size:
        raise ValueError("shape does not match the number of elements")
    shape_msg = bytearray()
    for s in dims:
        dim = bytearray()
        dim.append((1 << 3) | 0)                 # Dim.size
        _put_varint(dim, int(s))
        shape_msg.append((2 << 3) | 2)           # TensorShapeProto.dim
        _put_varint(shape_msg, len(dim))
        shape_msg += dim
    out = bytearray()
    out.append((1 << 3) | 0)                     # dtype
    _put_varint(out, _DT_OF_NP[arr.dtype])
    out.append((2 << 3) | 2)                     # tensor_shape
    _put_varint(out, len(shape_msg))
    out += shape_msg
    payload = arr.astype(arr.dtype.newbyteorder("<"), copy=False).tobytes()
    out.append((4 << 3) | 2)                     # tensor_content
    _put_varint(out, len(payload))
    return bytes(out) + payload
