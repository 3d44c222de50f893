"""The picture `display_instances(..., annotate=True)` promises (DESIGN.md section 3.25): the OpenCV
calls below on the overlay, in RGB order, at the image's own resolution.  cv2 is the
specification; this module only states the call sequence."""
import cv2
import numpy as np


def annotate(overlay, boxes, colors, contours, class_ids=None, class_names=None, scores=None,
             captions=None, show_bbox=True):
    """overlay uint8 [H, W, 3]; boxes [N, 4] (y1, x1, y2, x2); colors N RGB triples; contours[k]:
    the (x, y) float polygons of instance k (`contour_oracle.mask_polygons`)."""
    img = np.ascontiguousarray(overlay).copy()
    boxes = np.asarray(boxes).reshape(-1, 4)
    kept = [k for k in range(boxes.shape[0]) if np.any(boxes[k])]
    for k in kept:
        y1, x1, y2, x2 = (int(v) for v in boxes[k])
        col = tuple(255.0 * float(c) for c in colors[k])
        if show_bbox:
            cv2.rectangle(img, (x1, y1), (x2, y2), col, 1, cv2.LINE_8)
        for v in contours[k]:
            cv2.polylines(img, [np.int32(2 * np.asarray(v))], False, col, 1, cv2.LINE_8, shift=1)
    for k in kept:
        y1, x1 = int(boxes[k][0]), int(boxes[k][1])
        if captions:
            cap = captions[k]
        else:
            score = scores[k] if scores is not None else None
            label = class_names[int(class_ids[k])]
            cap = "{} {:.3f}".format(label, score) if score else label
        cv2.putText(img, cap, (x1, y1 + 8), cv2.FONT_HERSHEY_SIMPLEX, 0.5, (255, 255, 255), 1,
                    cv2.LINE_8)
    return img
