"""Tiny DAVIS2016 / FBMS / SegTrackV2 trees and supplied-flow trees for the --flow_dir tests."""
import os

import cv2
import numpy as np


def _frame(rng, i, h, w):
    img = (rng.rand(h, w, 3) * 255).astype(np.uint8)
    img[:, :, 0] = i * 20                                   # blue (BGR) encodes the frame index
    return img


def _mask(i, h, w):
    m = np.zeros((h, w), np.uint8)
    m[h // 5:h // 2 + 2, w // 4 + i:w // 2 + i] = 255
    return m


def make_davis_tree(root, seqs=(('train', ('bear', 'bus')), ('val', ('cows',))), n=6, h=48, w=80):
    root = str(root)
    rng = np.random.RandomState(0)
    lines = {}
    for part, names in seqs:
        for s in names:
            os.makedirs(os.path.join(root, 'JPEGImages/480p', s))
            os.makedirs(os.path.join(root, 'Annotations/480p', s))
            for i in range(n):
                cv2.imwrite(os.path.join(root, 'JPEGImages/480p', s, '%05d.jpg' % i), _frame(rng, i, h, w), [cv2.IMWRITE_JPEG_QUALITY, 100])
                cv2.imwrite(os.path.join(root, 'Annotations/480p', s, '%05d.png' % i), _mask(i, h, w))
                lines.setdefault(part, []).append('/JPEGImages/480p/%s/%05d.jpg /Annotations/480p/%s/%05d.png' % (s, i, s, i))
    os.makedirs(os.path.join(root, 'ImageSets/480p'))
    for part in ('train', 'val'):
        open(os.path.join(root, 'ImageSets/480p', part + '.txt'), 'w').write('\n'.join(lines.get(part, [])) + '\n')
    open(os.path.join(root, 'ImageSets/480p', 'trainval.txt'), 'w').write('\n'.join(lines.get('train', []) + lines.get('val', [])) + '\n')
    return root


def make_fbms_tree(root, n=8, h=40, w=64):
    root = str(root)
    rng = np.random.RandomState(1)
    for part, cats in (('Trainingset', ['cars1']), ('Testset', ['cats01', 'marple7'])):
        for c in cats:
            d = os.path.join(root, part, c)
            os.makedirs(os.path.join(d, 'GroundTruth'))
            with open(os.path.join(d, c + '.bmf'), 'w') as f:
                f.write('%d 1\n' % n + ''.join('%s_%02d.ppm\n' % (c, i + 1) for i in range(n)))
            for i in range(n):
                cv2.imwrite(os.path.join(d, '%s_%02d.jpg' % (c, i + 1)), _frame(rng, i, h, w), [cv2.IMWRITE_JPEG_QUALITY, 100])
            for k in (1, 4, 8):
                cv2.imwrite(os.path.join(d, 'GroundTruth', '%s_%03d.pgm' % (c, k)), _mask(k, h, w))
    return root


def make_segtrack_tree(root, seqs=('birdfall', 'frog'), n=6, h=40, w=64):
    root = str(root)
    rng = np.random.RandomState(2)
    os.makedirs(os.path.join(root, 'ImageSets'))
    open(os.path.join(root, 'ImageSets/all.txt'), 'w').write(''.join('*%s\n' % s for s in seqs))
    for s in seqs:
        os.makedirs(os.path.join(root, 'JPEGImages', s))
        os.makedirs(os.path.join(root, 'GroundTruth', s))
        names = ['%s_%05d' % (s, i) for i in range(n)]
        open(os.path.join(root, 'ImageSets', s + '.txt'), 'w').write('header\n' + ''.join(nm + '\n' for nm in names))
        for i, nm in enumerate(names):
            cv2.imwrite(os.path.join(root, 'JPEGImages', s, nm + '.png'), _frame(rng, i, h, w))
            cv2.imwrite(os.path.join(root, 'GroundTruth', s, nm + '.png'), _mask(i, h, w))
    return root


def make_tree(dataset, root):
    return {'DAVIS2016': make_davis_tree, 'FBMS': make_fbms_tree, 'SEGTRACK': make_segtrack_tree}[dataset](root)


def reader(dataset, root, flow_dir='', seed=3, **kw):
    from unsupervised_detection_b200.data.davis2016_data_utils import Davis2016Reader
    from unsupervised_detection_b200.data.fbms_data_utils import FBMS59Reader
    from unsupervised_detection_b200.data.segtrackv2_data_utils import SegTrackV2Reader
    cls = {'DAVIS2016': Davis2016Reader, 'FBMS': FBMS59Reader, 'SEGTRACK': SegTrackV2Reader}[dataset]
    kw.setdefault('max_temporal_len', 3)
    kw.setdefault('min_temporal_len', 1)
    return cls(root, num_threads=2, seed=seed, flow_dir=flow_dir, **kw)


def random_uv(seed, h, w):
    """A smooth-ish seeded (u, v) field in pixels of an h x w grid."""
    rng = np.random.RandomState(seed)
    lo = rng.randn(3, 4, 2).astype(np.float32) * 4
    return cv2.resize(lo, (w, h), interpolation=cv2.INTER_CUBIC).astype(np.float32) + rng.randn(h, w, 2).astype(np.float32) * 0.1


def write_flows(rd, flow_dir, pairs, size=(30, 52)):
    """One random .flo of resolution `size` per (f1, f2) in `pairs` under flow_dir -> {pair: uv}."""
    from unsupervised_detection_b200.data.davis2016_data_utils import flow_file
    from unsupervised_detection_b200.data.flyingchairs_data_utils import write_flo
    out = {}
    for k, (f1, f2) in enumerate(pairs):
        uv = random_uv(k, *size)
        write_flo(flow_file(str(flow_dir), rd.root_dir, f1, f2), uv)
        out[(f1, f2)] = uv
    return out
