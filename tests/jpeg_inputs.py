"""JPEG test inputs: files made with cv2.imencode at test time, and hand-spliced variants."""
from __future__ import annotations

import struct

import numpy as np

from matterport_maskrcnn_with_tensorflow_serving_b200 import synth

SAMPLINGS = {"444": 0x111111, "422": 0x211111, "420": 0x221111, "440": 0x121111, "411": 0x411111}


def image(rng, h, w, kind="smooth", gray=False):
    """synth_rgb_image (smooth gradients) or uniform noise, RGB (or one channel)."""
    if kind == "noise":
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    else:
        img = synth.synth_rgb_image(rng, h, w)
    return np.ascontiguousarray(img[:, :, 0]) if gray else img


def encode(img, quality=90, sampling="420", rst=0, optimize=False, progressive=False):
    """cv2.imencode of an RGB (or 2-D grayscale) image; returns the file's bytes."""
    import cv2

    src = img if img.ndim == 2 else img[:, :, ::-1]
    params = [cv2.IMWRITE_JPEG_QUALITY, int(quality),
              cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLINGS[sampling],
              cv2.IMWRITE_JPEG_RST_INTERVAL, int(rst),
              cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize),
              cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)]
    ok, buf = cv2.imencode(".jpg", src, params)
    assert ok
    return buf.tobytes()


def cv2_decode(blob):
    """What load_img returns for the file: cv2.imdecode(IMREAD_COLOR) then BGR -> RGB."""
    import cv2

    bgr = cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)
    return None if bgr is None else cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)


def segments(blob):
    """(marker, start, end) of each header segment up to and including SOS."""
    out, pos = [], 2
    while True:
        code = blob[pos + 1]
        length = struct.unpack(">H", blob[pos + 2:pos + 4])[0]
        out.append((code, pos, pos + 2 + length))
        pos += 2 + length
        if code == 0xDA:
            return out


def scan_start(blob):
    return segments(blob)[-1][2]


def with_exif(blob, orientation, big_endian=False):
    """An APP1 Exif segment whose IFD0 holds only the orientation tag, after SOI."""
    e = ">" if big_endian else "<"
    tiff = (b"MM" if big_endian else b"II") + struct.pack(e + "HI", 42, 8)
    tiff += struct.pack(e + "H", 1) + struct.pack(e + "HHIHH", 0x0112, 3, 1, orientation, 0)
    tiff += struct.pack(e + "I", 0)
    payload = b"Exif\x00\x00" + tiff
    return blob[:2] + b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload + blob[2:]


def with_dqt16(blob):
    """Every DQT table rewritten with 16-bit entries (same values)."""
    out, last = bytearray(), 0
    for code, s, e in segments(blob):
        if code != 0xDB:
            continue
        seg = blob[s + 4:e]
        new, q = bytearray(), 0
        while q < len(seg):
            tq = seg[q] & 15
            vals = np.frombuffer(seg[q + 1:q + 65], np.uint8).astype(">u2")
            new += bytes([0x10 | tq]) + vals.tobytes()
            q += 65
        out += blob[last:s] + b"\xff\xdb" + struct.pack(">H", len(new) + 2) + new
        last = e
    return bytes(out + blob[last:])


def without_jfif_with_adobe(blob, transform=0):
    """The JFIF APP0 dropped and an Adobe APP14 segment with `transform` added."""
    out, last = bytearray(blob[:2]), 2
    for code, s, e in segments(blob):
        if code == 0xE0:
            out += blob[last:s]
            last = e
    adobe = b"Adobe" + struct.pack(">HHHB", 100, 0, 0, transform)
    out = out[:2] + b"\xff\xee" + struct.pack(">H", len(adobe) + 2) + adobe + out[2:]
    return bytes(out + blob[last:])


def with_wrong_rst(blob):
    """The first RST0 of the scan renumbered RST1."""
    s = scan_start(blob)
    i = blob.index(b"\xff\xd0", s)
    return blob[:i] + b"\xff\xd1" + blob[i + 2:]


def truncated(blob, frac=0.5):
    """The scan cut at `frac` of its length, then EOI."""
    s = scan_start(blob)
    cut = s + int((len(blob) - 2 - s) * frac)
    if blob[cut - 1] == 0xFF:
        cut -= 1
    return blob[:cut] + b"\xff\xd9"


def with_bad_code(blob, frac=0.5):
    """32 one bits (stuffed 0xFF bytes) in the middle of the scan: no baseline table assigns an
    all-ones code, so the decoder meets an invalid code there."""
    s = scan_start(blob)
    i = s + int((len(blob) - 2 - s) * frac)
    while blob[i - 1] == 0xFF or blob[i] == 0xFF:
        i += 1
    return blob[:i] + b"\xff\x00" * 4 + blob[i + 4:]


def with_second_scan(blob):
    """The SOS segment and scan repeated before EOI."""
    sos = segments(blob)[-1][1]
    return blob[:-2] + blob[sos:-2] + b"\xff\xd9"
