"""Host-side Flying Chairs reader for the recover-net pretraining (the dataset the reference's README names for it): frame pairs with
their ground-truth optical flow, fed as pinned torch tensors like the other readers' batches.

Release layout: <root>/data/NNNNN_img1.ppm, NNNNN_img2.ppm, NNNNN_flow.flo (384x512), and optionally <root>/FlyingChairs_train_val.txt
with one label per pair in file-name order (1 = train, 2 = val; 22,232 / 640 pairs in the release).  Without that file every pair is a
training pair.  Frames go through the same host routine as the other readers (RGB in [-0.5, 0.5], legacy bilinear to 384x640); the flow
is resampled to that grid with its vectors rescaled to 384x640 pixel units, and handed over in the channel order and sign of PWC-Net's
output (pwc_flow_from_uv).  Training pairs get the DAVIS reader's augmentation (same draws, same order), applied to the flow field and
to its vectors; validation pairs are ordered and not augmented.
"""
import os
import random

import numpy as np

from .davis2016_data_utils import ORIG_H, ORIG_W, Davis2016Reader, _Iter, crop_resized, flip, legacy_resize, train_augmentation

FLO_TAG = 202021.25
SPLIT_FILE = 'FlyingChairs_train_val.txt'
TRAIN, VAL = 1, 2


def read_flo(path):
    """Middlebury .flo -> float32 [H,W,2] (u, v): float32 tag 202021.25, int32 width, int32 height, then H*W*2 little-endian float32.
    IOError naming the file on a wrong tag, a size that does not match the header, or non-finite values."""
    with open(path, 'rb') as f:
        data = f.read()
    if len(data) < 12 or np.frombuffer(data, '<f4', 1, 0)[0] != np.float32(FLO_TAG):
        raise IOError('%s: not a Middlebury .flo file (wrong tag)' % path)
    w, h = (int(v) for v in np.frombuffer(data, '<i4', 2, 4))
    if w < 1 or h < 1 or len(data) != 12 + 8 * h * w:
        raise IOError('%s: %d bytes do not hold the %dx%d flow field of its header (truncated?)' % (path, len(data), w, h))
    flow = np.frombuffer(data, '<f4', 2 * h * w, 12).reshape(h, w, 2).astype(np.float32)
    if not np.isfinite(flow).all():
        raise IOError('%s: non-finite flow values' % path)
    return flow


def pwc_flow_from_uv(uv):
    """Middlebury flow (u, v) [...,2] -> the flow PWC-Net hands to the recover net: channel 0 = -v, channel 1 = -u.

    Derivation.  PWC-Net aligns frame 2 with frame 1 by warping frame 2's features with its flow estimate (model_pwcnet.py, warp:
    dense_image_warp(c2, flow)), and dense_image_warp (core_warp.py:153-202, oracle.pwcnet.dense_image_warp) reads
        out[j, i] = c2[j - flow[j, i, 0], i - flow[j, i, 1]]        (j = row, i = column).
    A warp that reproduces frame 1 must read frame 2 where pixel (i, j) of frame 1 has moved to.  Middlebury's (u, v) is that motion:
    frame1(i, j) = frame2(i + u, j + v).  Equating the sampling positions, j - flow0 = j + v and i - flow1 = i + u, so flow0 = -v and
    flow1 = -u: the field that makes the network's own warp consistent is (row, column) ordered and points from frame 2 back to frame 1.
    This follows from the warp alone; it has not been compared with the output of a trained PWC-Net checkpoint."""
    return np.stack([-uv[..., 1], -uv[..., 0]], axis=-1)


def flow_to_grid(uv):
    """(u, v) flow at any size -> legacy bilinear resize to 384x640 with the vectors rescaled to that grid's pixels (x by 640/W, y by
    384/H)."""
    h, w = uv.shape[:2]
    out = legacy_resize(np.ascontiguousarray(uv, dtype=np.float32), ORIG_H, ORIG_W)
    return out * np.array([ORIG_W / w, ORIG_H / h], np.float32)


def augment_flow(uv, case, y0, x0, ch, cw):
    """train_augmentation's flip and crop applied to a (u, v) field on the 384x640 grid: the field is flipped and cropped like the frames,
    and its vectors follow -- a left-right flip negates u, a top-down flip negates v, the 180-degree rotation both, and resizing the
    ch x cw crop back to the full grid scales u by W/cw and v by H/ch."""
    h, w = uv.shape[:2]
    sign = np.array([(1, 1), (-1, -1), (-1, 1), (1, -1)][case], np.float32)
    out = crop_resized(flip(uv, case), y0, x0, ch, cw)
    return out * (sign * np.array([w / cw, h / ch], np.float32))


class FlyingChairsReader(object):
    """Pairs of <root>/data with their train / val split; image_inputs() and test_inputs() return the other readers' batch iterators
    (thread pool, CIS_READER_PREFETCH, shard) whose batches are (img1 [B,384,640,3], img2 [B,384,640,3], flow [B,384,640,2], names)."""

    def __init__(self, root_dir, num_threads=6, seed=8964):
        self.root_dir, self.num_threads = root_dir, num_threads
        self.rng = random.Random(seed)
        self.prefetch = int(os.environ.get('CIS_READER_PREFETCH', '3'))     # training batches decoded ahead (0 = synchronous)
        self.train_crop = 1.0
        data = os.path.join(root_dir, 'data')
        stems = sorted(f[:-len('_img1.ppm')] for f in os.listdir(data) if f.endswith('_img1.ppm')) if os.path.isdir(data) else []
        if not stems:
            raise IOError('Did not find any Flying Chairs pair (data/NNNNN_img1.ppm) under %s' % root_dir)
        pairs = [tuple(os.path.join(data, s + suf) for suf in ('_img1.ppm', '_img2.ppm', '_flow.flo')) for s in stems]
        split = os.path.join(root_dir, SPLIT_FILE)
        self.has_split = os.path.isfile(split)
        labels = np.loadtxt(split, dtype=np.int64, ndmin=1) if self.has_split else np.full(len(pairs), TRAIN)
        if len(labels) != len(pairs) or not np.isin(labels, (TRAIN, VAL)).all():
            raise IOError('%s: needs one label 1 (train) or 2 (val) per pair, %d pairs found' % (split, len(pairs)))
        self.train_pairs = [p for p, lb in zip(pairs, labels) if lb == TRAIN]
        self.val_pairs = [p for p, lb in zip(pairs, labels) if lb == VAL]
        self.train_samples, self.val_samples = len(self.train_pairs), len(self.val_pairs)
        print('Found {} Flying Chairs pairs: {} train, {} val.'.format(len(pairs), self.train_samples, self.val_samples))

    @staticmethod
    def _read(pair):
        """-> frame 1, frame 2 (384x640 RGB in [-0.5, 0.5]) and the (u, v) flow on that grid."""
        a, b = Davis2016Reader.preprocess_image(pair[0]), Davis2016Reader.preprocess_image(pair[1])
        return a, b, flow_to_grid(read_flo(pair[2]))

    def _train_sample(self, pair, seed):
        a, b, uv = self._read(pair)
        h, w = a.shape[:2]
        aug = train_augmentation(random.Random(seed), self.train_crop, h, w)
        a, b = crop_resized(flip(a, aug[0]), *aug[1:]), crop_resized(flip(b, aug[0]), *aug[1:])
        return a.astype(np.float32), b.astype(np.float32), pwc_flow_from_uv(augment_flow(uv, *aug)), pair[0]

    def _test_sample(self, pair, seed):
        a, b, uv = self._read(pair)
        return a, b, pwc_flow_from_uv(uv), pair[0]

    def image_inputs(self, batch_size=32, train_crop=1.0):
        """Endless shuffled iterator of augmented training pairs (label 1)."""
        self.train_crop = train_crop
        return _Iter(self, self.train_pairs, train=True, shuffle=True, num_threads=self.num_threads, prefetch=self.prefetch)

    def test_inputs(self, batch_size=32):
        """Ordered iterator of the validation pairs (label 2), not augmented.  IOError without a split file."""
        if not self.val_pairs:
            raise IOError('No Flying Chairs validation pairs: %s is missing or labels none' % os.path.join(self.root_dir, SPLIT_FILE))
        return _Iter(self, self.val_pairs, train=False, shuffle=False, num_threads=self.num_threads, prefetch=self.prefetch)
