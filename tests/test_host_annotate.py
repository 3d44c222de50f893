"""The host halves of the annotated overlay (DESIGN.md section 3.25), checked against cv2 on the CPU:
the contour segment rule mrx_annotate_draw rasterises, the caption stencils, the colour table,
the argument checks of both entry points, and the mutant table of tools/mutate_annotate.py."""
import os
import sys

import cv2
import numpy as np
import pytest
import torch

import annotate_oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import visualize

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

# every step between edge midpoints a contour makes, in half pixels
STEPS = [(1, 1), (1, -1), (-1, 1), (-1, -1), (2, 0), (-2, 0), (0, 2), (0, -2)]


@pytest.mark.parametrize("H,W", [(1, 1), (5, 6), (2, 9), (7, 3)])
def test_segment_rule_equals_polylines_shift1(H, W):
    """Every step from every start point with coordinates in [-1/2, W - 1/2] x [-1/2, H - 1/2]
    (both parities, every border position, steps that leave the image) sets the pixels cv2 sets."""
    cases = 0
    for dx, dy in STEPS:
        for ax in range(-1, 2 * W):
            for ay in range(-1, 2 * H):
                bx, by = ax + dx, ay + dy
                if not (-1 <= bx <= 2 * W - 1 and -1 <= by <= 2 * H - 1):
                    continue
                img = np.zeros((H, W), np.uint8)
                cv2.polylines(img, [np.array([[ax, ay], [bx, by]], np.int32)], False, 255, 1,
                              cv2.LINE_8, shift=1)
                want = {(int(x), int(y)) for y, x in zip(*np.nonzero(img))}
                got = visualize.segment_pixels((ax / 2, ay / 2), (bx / 2, by / 2), H, W)
                assert got == want, ((ax, ay), (bx, by))
                cases += 1
    assert cases > 8 * H * W


def test_outline_is_its_rounded_vertices():
    """A polyline of such steps is the union of its segments: the rule needs no segment order."""
    rng = np.random.default_rng(3)
    H, W = 9, 11
    for _ in range(300):
        pts = [(int(rng.integers(-1, 2 * W)), int(rng.integers(-1, 2 * H)))]
        while len(pts) < 12:
            dx, dy = STEPS[int(rng.integers(8))]
            q = (pts[-1][0] + dx, pts[-1][1] + dy)
            if -1 <= q[0] <= 2 * W - 1 and -1 <= q[1] <= 2 * H - 1:
                pts.append(q)
        img = np.zeros((H, W), np.uint8)
        cv2.polylines(img, [np.array(pts, np.int32)], False, 255, 1, cv2.LINE_8, shift=1)
        got = set()
        for p, q in zip(pts[:-1], pts[1:]):
            got |= visualize.segment_pixels((p[0] / 2, p[1] / 2), (q[0] / 2, q[1] / 2), H, W)
        assert got == {(int(x), int(y)) for y, x in zip(*np.nonzero(img))}


def _stencil_image(texts, boxes, hw):
    out = np.zeros(hw, np.uint8)
    for y0, x0, st in visualize.caption_patches(texts, boxes, hw):
        out[y0:y0 + st.shape[0], x0:x0 + st.shape[1]] |= st.astype(np.uint8) * 255
    return out


def _put_text(texts, boxes, hw):
    img = np.zeros(hw, np.uint8)
    for text, box in zip(texts, boxes):
        if np.any(box):
            cv2.putText(img, text, (int(box[1]), int(box[0]) + 8), cv2.FONT_HERSHEY_SIMPLEX, 0.5,
                        255, 1, cv2.LINE_8)
    return img


@pytest.mark.parametrize("hw", [(40, 60), (13, 200), (100, 17), (1, 1), (9, 9)])
def test_caption_patches_equal_put_text(hw):
    """Captions off every edge, at the corners and past the bottom (y1 + 8 >= H)."""
    H, W = hw
    rng = np.random.default_rng(H * 1000 + W)
    texts = ["class_1 0.987", "BG", "Wyg|_@ 0.001", "x", "class_80 1.000", "a long caption text"]
    for trial in range(300):
        y1 = int(rng.integers(-20, H + 20))
        x1 = int(rng.integers(-120, W + 5))
        text = texts[trial % len(texts)]
        boxes = np.array([[y1, x1, y1 + 5, x1 + 5]])
        if not boxes.any():
            continue
        assert np.array_equal(_stencil_image([text], boxes, hw), _put_text([text], boxes, hw)), \
            (hw, y1, x1, text)
    for y1, x1 in [(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (H, 1), (H + 7, 2),
                   (H - 8, W - 3), (-8, -3)]:
        boxes = np.array([[y1, x1, H, W]])
        assert np.array_equal(_stencil_image(["class_9 0.5"], boxes, hw),
                              _put_text(["class_9 0.5"], boxes, hw)), (y1, x1)


def test_caption_strings_follow_upstream():
    names = ["BG", "dent", "scratch"]
    assert visualize.caption_strings(3, [1, 2, 1], names, np.float32([0.98765, 0.0, 1.0])) == \
        ["dent 0.988", "scratch", "dent 1.000"]
    assert visualize.caption_strings(2, [1, 2], names, None) == ["dent", "scratch"]
    assert visualize.caption_strings(2, None, None, None, ["mine", ""]) == ["mine", ""]
    # an empty caption list means "none given", as upstream's `if not captions`
    assert visualize.caption_strings(1, [2], names, [0.5], []) == ["scratch 0.500"]
    with pytest.raises(ValueError):
        visualize.caption_strings(1, [1], None, [0.5])


def test_empty_and_custom_captions_and_score_zero():
    hw = (48, 64)
    boxes = np.array([[10, 5, 30, 40], [0, 0, 0, 0], [40, 50, 48, 64], [20, 30, 40, 60]])
    texts = visualize.caption_strings(4, [1, 2, 1, 2], ["BG", "a", "b"], [0.0, 0.9, 0.25, 0.5],
                                      ["", "skipped", "custom", "x y"])
    assert texts == ["", "skipped", "custom", "x y"]
    want = _put_text(texts, boxes, hw)
    assert np.array_equal(_stencil_image(texts, boxes, hw), want)
    # score 0: the label alone
    texts = visualize.caption_strings(1, [1], ["BG", "a"], [0.0])
    assert texts == ["a"]


def test_caption_stencils_pack_bits():
    boxes = [np.array([[10, 5, 30, 40], [30, 50, 40, 60]]), np.zeros((0, 4)),
             np.array([[0, 0, 0, 0], [3, 2, 9, 9]])]
    hws = [(40, 60), (8, 8), (12, 30)]
    recs, bits = visualize.caption_stencils(boxes, hws, captions=[["ab", "cd"], [], ["x", "yz"]])
    assert recs.dtype == np.int64 and recs.shape[1] == 6
    canvases = [np.zeros(hw, np.uint8) for hw in hws]
    for b, y0, x0, h, w, off in recs:
        st = np.unpackbits(bits[off:off + (h * w + 7) // 8])[:h * w].reshape(h, w)
        assert 0 <= y0 and y0 + h <= hws[b][0] and 0 <= x0 and x0 + w <= hws[b][1]
        canvases[b][y0:y0 + h, x0:x0 + w] |= st * 255
    assert np.array_equal(canvases[0], _put_text(["ab", "cd"], boxes[0], hws[0]))
    assert not canvases[1].any()
    assert np.array_equal(canvases[2], _put_text(["yz"], boxes[2][1:], hws[2]))


def test_color_table_equals_what_cv2_draws():
    halves = [(k + 0.5) / 255.0 for k in (0, 1, 126, 127, 253, 254)]
    colors = [tuple(halves[i:i + 3]) for i in range(0, 6, 3)]
    # 255 * c exactly k + 1/2 (cvRound rounds half to even), negative, above 1, out of int32 range
    colors += [(-0.001, -1.0, -0.5 / 255), (1.0, 1.5, 300.0), (1e8, 1e10, -1e10),
               (float("inf"), float("nan"), 0.5), (0.2, 0.4, 0.6)]
    for c in colors[:2]:
        assert all(float(255.0 * v) % 1 == 0.5 for v in c)
    tab = visualize.color_table(colors, len(colors) + 2)
    assert tab.dtype == np.uint8 and not tab[len(colors):].any()
    for k, col in enumerate(colors):
        img = np.zeros((2, 2, 3), np.uint8)
        cv2.rectangle(img, (0, 0), (1, 1), tuple(255.0 * float(v) for v in col), 1, cv2.LINE_8)
        assert np.array_equal(tab[k], img[0, 0]), (col, tab[k], img[0, 0])


def test_oracle_program_runs_on_the_cpu():
    """The test oracle's call sequence: captions over boxes over outlines, later over earlier."""
    img = np.zeros((30, 40, 3), np.uint8)
    boxes = np.array([[2, 3, 20, 30], [5, 5, 25, 35]])
    contours = [[np.array([[4.5, 4.0], [5.0, 4.5], [4.5, 5.0], [4.0, 4.5], [4.5, 4.0]])], []]
    out = annotate_oracle.annotate(img, boxes, [(1, 0, 0), (0, 0, 1)], contours,
                                   captions=["", ""])
    assert tuple(out[5, 10]) == (0, 0, 255) and tuple(out[2, 10]) == (255, 0, 0)
    assert tuple(out[4, 5]) == (255, 0, 0)


# ------------------------------------------------------------------ argument checks (no device work)
def _i32(*shape):
    return torch.zeros(shape, dtype=torch.int32)


def _i64(*shape):
    return torch.zeros(shape, dtype=torch.int64)


def _draw(**replace):
    args = [_i32(1), _i32(1, 8), _i32(1, 2, 4), torch.zeros(4, 2, dtype=torch.float64), _i64(2),
            _i64(3), 4, 1, _i32(16), _i64(1), 0, 2, 16, None]
    for k, v in replace.items():
        args[int(k[1:])] = v
    return N.load().mrx_annotate_draw(*args)


def _resolve(**replace):
    args = [_i32(1, 8), _i32(16), _i64(1), torch.zeros(1, 2, 3, dtype=torch.uint8),
            torch.zeros(48, dtype=torch.uint8), _i64(1), torch.zeros(4, dtype=torch.uint8),
            _i64(1, 6), 1, 0, 2, 16, None]
    for k, v in replace.items():
        args[int(k[1:])] = v
    return N.load().mrx_annotate_resolve(*args)


@pytest.mark.parametrize("replace, status", [
    ({}, "MRX_OK"),
    ({"a3": None, "a4": None, "a5": None, "a6": 0}, "MRX_OK"),   # no outline
    ({"a0": None}, "MRX_E_INVALID"), ({"a1": None}, "MRX_E_INVALID"),
    ({"a2": None}, "MRX_E_INVALID"), ({"a8": None}, "MRX_E_INVALID"),
    ({"a9": None}, "MRX_E_INVALID"), ({"a3": None}, "MRX_E_INVALID"),
    ({"a5": None}, "MRX_E_INVALID"), ({"a6": -1}, "MRX_E_INVALID"),
    ({"a10": -1}, "MRX_E_INVALID"), ({"a10": N.MRX_MAX_BATCH + 1}, "MRX_E_INVALID"),
    ({"a11": 0}, "MRX_E_INVALID"), ({"a11": 65535}, "MRX_E_INVALID"),
    ({"a12": -1}, "MRX_E_INVALID"), ({"a12": (1 << 31) - 1}, "MRX_E_INVALID"),
])
def test_draw_refusals_with_float64_vertices(replace, status):
    assert _draw(**replace) == getattr(N, status)
    if status != "MRX_OK":
        assert N.load().mrx_last_error().decode().startswith("mrx_annotate_draw")


def test_draw_binding_refuses_float32_vertices():
    """The vertices are float64 (mrx.h, mrx_contours_write): float32 rounds halves past 2^23, and
    a float32 buffer read as float64 would draw garbage, so the binding refuses it."""
    with pytest.raises(Exception, match=r"double \* parameter: got a torch.float32 tensor"):
        _draw(a3=torch.zeros(4, 2))


@pytest.mark.parametrize("replace, status", [
    ({}, "MRX_OK"),
    ({"a6": None, "a7": None, "a8": 0}, "MRX_OK"),                # no caption
    ({"a0": None}, "MRX_E_INVALID"), ({"a1": None}, "MRX_E_INVALID"),
    ({"a2": None}, "MRX_E_INVALID"), ({"a3": None}, "MRX_E_INVALID"),
    ({"a4": None}, "MRX_E_INVALID"), ({"a5": None}, "MRX_E_INVALID"),
    ({"a6": None}, "MRX_E_INVALID"), ({"a7": None}, "MRX_E_INVALID"),
    ({"a8": -1}, "MRX_E_INVALID"), ({"a9": -1}, "MRX_E_INVALID"),
    ({"a9": N.MRX_MAX_BATCH + 1}, "MRX_E_INVALID"), ({"a10": 0}, "MRX_E_INVALID"),
    ({"a11": -1}, "MRX_E_INVALID"),
])
def test_resolve_refusals(replace, status):
    assert _resolve(**replace) == getattr(N, status)
    if status != "MRX_OK":
        assert N.load().mrx_last_error().decode().startswith("mrx_annotate_resolve")


def test_mutant_table_matches_the_sources():
    import mutate_annotate
    from test_host_mutants import check_table

    check_table(mutate_annotate, ROOT)
