"""CPU restatement of upstream Matterport `mrcnn.utils.extract_bboxes`, the ground-truth boxes
`load_image_gt` computes from the masks.  TEST INFRASTRUCTURE ONLY."""
import numpy as np


def extract_bboxes(mask):
    """[UPSTREAM mrcnn.utils.extract_bboxes] boxes [N, (y1, x1, y2, x2)] int32 of masks [H, W, N]:
    the tight box with exclusive ends, all zeros for an empty mask."""
    boxes = np.zeros([mask.shape[-1], 4], dtype=np.int32)
    for i in range(mask.shape[-1]):
        m = mask[:, :, i]
        horizontal_indicies = np.where(np.any(m, axis=0))[0]
        vertical_indicies = np.where(np.any(m, axis=1))[0]
        if horizontal_indicies.shape[0]:
            x1, x2 = horizontal_indicies[[0, -1]]
            y1, y2 = vertical_indicies[[0, -1]]
            x2 += 1
            y2 += 1
        else:
            x1, x2, y1, y2 = 0, 0, 0, 0
        boxes[i] = np.array([y1, x1, y2, x2])
    return boxes.astype(np.int32)
