"""The EXIF orientation both device decoders apply (a JPEG APP1 segment, a PNG eXIf chunk)."""
from __future__ import annotations

import struct


def orientation(tiff):
    """IFD0 tag 0x0112 of EXIF data in TIFF layout ("II" or "MM" byte order first), or 1 when the
    tag is missing, out of range or the data is malformed."""
    t = bytes(tiff)
    if t[:2] == b"II":
        e = "<"
    elif t[:2] == b"MM":
        e = ">"
    else:
        return 1
    try:
        if struct.unpack(e + "H", t[2:4])[0] != 42:
            return 1
        ifd = struct.unpack(e + "I", t[4:8])[0]
        n = struct.unpack(e + "H", t[ifd:ifd + 2])[0]
        for i in range(n):
            p = ifd + 2 + 12 * i
            tag, typ, cnt = struct.unpack(e + "HHI", t[p:p + 8])
            if tag == 0x0112 and typ == 3:
                v = struct.unpack(e + "H", t[p + 8:p + 10])[0]
                return v if 1 <= v <= 8 else 1
    except struct.error:
        return 1
    return 1
