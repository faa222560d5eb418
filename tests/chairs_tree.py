"""Tiny Flying Chairs trees for the reader and pretraining tests: cv2-written .ppm frames and Middlebury .flo files in the release layout
(<root>/data/NNNNN_img1.ppm, NNNNN_img2.ppm, NNNNN_flow.flo, optional <root>/FlyingChairs_train_val.txt)."""
import os

import cv2
import numpy as np

CH, CW = 384, 512


def write_flo(path, uv, tag=202021.25):
    """float32 [H,W,2] (u, v) -> Middlebury .flo."""
    h, w = uv.shape[:2]
    with open(path, 'wb') as f:
        f.write(np.array([tag], '<f4').tobytes() + np.array([w, h], '<i4').tobytes() + np.ascontiguousarray(uv, '<f4').tobytes())


def pattern(seed, h=CH, w=CW):
    """A smooth uint8 BGR frame (low-frequency sinusoids), so that resized and warped copies stay well conditioned."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = np.zeros((h, w, 3))
    for c in range(3):
        for _ in range(3):
            fy, fx, ph = rng.uniform(0.005, 0.03), rng.uniform(0.005, 0.03), rng.uniform(0, 6.3)
            out[..., c] += np.sin(fy * y * 6.28 + fx * x * 6.28 + ph)
    return np.clip(127.5 + 40.0 * out, 0, 255).astype(np.uint8)


def shifted(frame, dx, dy):
    """frame2(x, y) = frame1(x - dx, y - dy): the content moves by (dx, dy) pixels (Middlebury u = dx, v = dy); edges repeat."""
    h, w = frame.shape[:2]
    yi = np.clip(np.arange(h) - dy, 0, h - 1)
    xi = np.clip(np.arange(w) - dx, 0, w - 1)
    return np.ascontiguousarray(frame[yi][:, xi])


def make_chairs_tree(root, n=6, labels=None, shift=(4, 2), flows=None):
    """n translated pairs (frame 2 = frame 1 moved by `shift` = (dx, dy), flow (dx, dy) everywhere unless flows[i] is given); labels =
    the split file's labels (None: no split file) -> root."""
    data = os.path.join(str(root), 'data')
    os.makedirs(data, exist_ok=True)
    for i in range(n):
        stem = os.path.join(data, '%05d' % (i + 1))
        a = pattern(i)
        cv2.imwrite(stem + '_img1.ppm', a)
        cv2.imwrite(stem + '_img2.ppm', shifted(a, *shift))
        uv = flows[i] if flows is not None else np.broadcast_to(np.array(shift, np.float32), (CH, CW, 2))
        write_flo(stem + '_flow.flo', uv)
    if labels is not None:
        with open(os.path.join(str(root), 'FlyingChairs_train_val.txt'), 'w') as f:
            f.write('\n'.join(str(v) for v in labels) + '\n')
    return str(root)
