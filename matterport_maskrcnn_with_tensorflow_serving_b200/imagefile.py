"""Image files by their signature: the one place that tells a JPEG file (FF D8) from a PNG file
(89 50 4E 47 0D 0A 1A 0A) and hands each to its decoder's plan.  Anything else raises
ValueError naming the image's index."""
from __future__ import annotations

from . import jpeg, png
from .jpeg import _as_bytes

JPEG, PNG = "jpeg", "png"


def kind(blob, index=0):
    """JPEG or PNG for a file's bytes."""
    data = _as_bytes(blob, index)
    if data[:2] == b"\xff\xd8":
        return JPEG
    if data[:8] == png.SIGNATURE:
        return PNG
    raise ValueError(f"image {index}: neither a JPEG nor a PNG file")


def shape(blob, index=0):
    """(H, W, 3) of the decoded, oriented image, from the headers alone."""
    if kind(blob, index) == PNG:
        return png.parse(blob, index).shape
    return jpeg.parse(blob, index).shape


def plan_batch(blobs, index=None):
    """A batch of files split by format: ([(plan, positions in blobs)], the decoded shape of every
    file, the format of every file).  JPEG files go to `jpeg.plan_batch`, PNG files to one
    `png.DecodePlan`; each keeps the caller's index for its refusals."""
    index = list(range(len(blobs))) if index is None else list(index)
    kinds = [kind(b, i) for b, i in zip(blobs, index)]
    plans, shapes = [], [None] * len(blobs)
    jpos = [k for k, f in enumerate(kinds) if f == JPEG]
    if jpos:
        jplans, jshapes = jpeg.plan_batch([blobs[k] for k in jpos], index=[index[k] for k in jpos])
        plans += [(plan, [jpos[k] for k in pos]) for plan, pos in jplans]
        for k, sh in zip(jpos, jshapes):
            shapes[k] = sh
    ppos = [k for k, f in enumerate(kinds) if f == PNG]
    if ppos:
        plan = png.DecodePlan([blobs[k] for k in ppos], index=[index[k] for k in ppos])
        plans.append((plan, ppos))
        for k, sh in zip(ppos, plan.shapes):
            shapes[k] = sh
    return plans, shapes, kinds
