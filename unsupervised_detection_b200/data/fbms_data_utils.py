"""Host-side FBMS59 reader (SURVEY 8f-2): the reference's data/fbms_data_utils.py:20-389 restated on top of the DAVIS2016
reader's numpy/OpenCV pipeline (same preprocessing, sampling and augmentation; see davis2016_data_utils.py).

Folder contract: `<root>/{Trainingset,Testset}/<category>/<category>.bmf` (first line = header, then one frame file name per
line; `.ppm`/`.pgm` names are mapped to `.jpg`, :73-76) and `<category>/GroundTruth/*.pgm | *_gt.ppm` for evaluation.

Differences from the reference, on purpose:
  * ground-truth masks are binarised IN MEMORY with the reference's thresholds (:107-121: 0.1, marple2 0.4, marple7 0.05,
    >0.99 -> 0 for the .ppm flavour).  The reference writes them back into the dataset folder as `.jpg` and re-reads those;
    this reader never writes into the dataset, so its masks lack only the JPEG compression noise of that round trip.
  * test batches are (img_1, img_2, seg_1, fnames) like the other readers; the per-category sample counts the reference appends
    to every sample (:148, used to weight categories) are kept in `samples_per_cat` / `batch_samples_per_cat()`.
"""
import os
import re

import cv2
import numpy as np

from .davis2016_data_utils import Davis2016Reader, _Iter, central_crop_box, nn_resize, ORIG_H, ORIG_W


def _read_bmf(path):
    """File names listed in a .bmf (np.loadtxt(..., skiprows=1) of the reference, first column)."""
    if not os.path.isfile(path):
        raise IOError("Not found file {}".format(path))
    with open(path) as f:
        lines = [l.split() for l in f.read().splitlines()[1:]]
    return [l[0].split('.')[0] + '.jpg' for l in lines if l]


def find_gt(directory):
    """fbms_data_utils.py:156-177 -> (sorted annotation file names, their frame numbers, type_weird)."""
    all_files = os.listdir(directory)
    type_weird = any(f.endswith('ppm') for f in all_files)
    if not type_weird:
        files = [f for f in all_files if f.endswith('pgm')]
        try:
            key = lambda x: int(x.split('.')[0].split('_')[-1])
            files = sorted(files, key=key)
        except ValueError:
            key = lambda x: int(re.search(r'\d+', x).group())
            files = sorted(files, key=key)
        return files, [key(f) for f in files], type_weird
    files = [f for f in all_files if f.endswith('ppm') and 'PROB' not in f]
    key = lambda x: int(x.split('_')[1])
    files = sorted(files, key=key)
    return files, [key(f) for f in files], type_weird


def binarise_gt(path, category, type_weird):
    """The one-off GT preprocessing of :107-121 -> uint8 {0,255} [H,W]."""
    m = cv2.imread(path)
    if m is None:
        raise IOError("Could not read annotation %s" % path)
    m = cv2.cvtColor(m, cv2.COLOR_BGR2GRAY) / 255.0
    if type_weird:
        m[m > 0.99] = 0.0
    thr = 0.05 if category == 'marple7' else (0.4 if category == 'marple2' else 0.1)
    return np.asarray((m > thr) * 255, dtype=np.uint8)


def test_offsets(numbers, t):
    """:124-137: index of the second frame for every annotated frame (frame numbers rebased to 0, shift t, mirrored at the two
    ends of the annotated range, clamped to the sequence)."""
    numbers = np.array(numbers) - np.min(numbers)
    seq_len = np.max(numbers)
    offsets = numbers + t
    if offsets[0] < numbers[0]:
        offsets[0] += 2 * abs(t)
    if offsets[-1] > numbers[-1]:
        offsets[-1] -= 2 * abs(t)
    return numbers, np.clip(offsets, 0, seq_len)


class DirectoryIterator(object):
    """fbms_data_utils.py:20-154."""
    PARTS = {'train': ['Trainingset'], 'val': ['Testset'], 'trainval': ['Trainingset', 'Testset']}

    def __init__(self, directory, part='train', for_testing=False, test_temporal_t=1):
        self.directory = directory
        self.num_experiments = 0
        self.samples = 0
        self.samples_per_cat = {}
        self.image_filenames, self.annotation_filenames, self.test_tuples = [], [], []
        dirs = [os.path.join(directory, d) for d in self.PARTS[part]]
        for d in dirs:
            if not os.path.isdir(d):
                raise IOError("Directory {} file not found".format(d))
        for d in dirs:
            for cat in sorted(os.listdir(d)):
                names = [os.path.join(d, cat, f) for f in _read_bmf(os.path.join(d, cat, cat + ".bmf"))]
                if not for_testing:
                    self.samples += len(names)
                    self.image_filenames.append(names)
                    continue
                gt_dir = os.path.join(d, cat, 'GroundTruth')
                ann, numbers, weird = find_gt(gt_dir)
                numbers, offsets = test_offsets(numbers, test_temporal_t)
                for i, k in enumerate(numbers):
                    self.test_tuples.append((names[k], names[offsets[i]], os.path.join(gt_dir, ann[i]), cat, weird, len(ann)))
                self.samples += len(ann)
                self.samples_per_cat[cat] = len(ann)
                self.num_experiments += 1
        if self.samples == 0:
            raise IOError("Did not find any file in the dataset folder")
        if not for_testing:
            self.num_experiments = len(self.image_filenames)
        print('Found {} images belonging to {} experiments.'.format(self.samples, self.num_experiments))


class FBMS59Reader(Davis2016Reader):
    """fbms_data_utils.py:179-389.  image_inputs / augmentation / central cropping are inherited (identical code in the
    reference); only the directory layout and the test tuples differ."""

    def __init__(self, root_dir, max_temporal_len=3, min_temporal_len=2, num_threads=6, seed=8964, flow_dir=''):
        Davis2016Reader.__init__(self, root_dir, max_temporal_len, min_temporal_len, num_threads, seed, flow_dir)

    def get_filenames_list(self, partition):
        it = DirectoryIterator(self.root_dir, partition)
        self.val_samples = it.samples
        return it.image_filenames, it.annotation_filenames

    def get_test_tuples(self, partition, test_temporal_t=1):
        it = DirectoryIterator(self.root_dir, partition, for_testing=True, test_temporal_t=test_temporal_t)
        self.val_samples = it.samples
        self.samples_per_cat = it.samples_per_cat
        self.num_categories = len(it.samples_per_cat)
        return it.test_tuples

    def _test_frames(self, tup):
        return tup[0], tup[1]

    def _test_sample(self, tup, seed):
        """test_dataset_map :337-359."""
        f1, f2, ann, cat, weird, _ = tup
        a, b = self.preprocess_image(f1), self.preprocess_image(f2)
        s = nn_resize(binarise_gt(ann, cat, weird).astype(np.float32)[..., None] / np.float32(255.0), ORIG_H, ORIG_W)
        c = self.test_crop
        sample = (self.central_cropping(a, c).astype(np.float32), self.central_cropping(b, c).astype(np.float32),
                  self.central_cropping(s, c).astype(np.float32), f1)
        return self._with_flow(sample, f1, f2, 0, central_crop_box(ORIG_H, ORIG_W, c))

    def test_inputs(self, batch_size=32, partition='val', t_len=2, with_fname=False, test_crop=1.0):
        """:311-335 -> ordered iterator over the annotated frames of every category."""
        tuples = self.get_test_tuples(partition, t_len)
        self.test_crop = test_crop
        return _Iter(self, tuples, train=False, shuffle=False, num_threads=self.num_threads, prefetch=self.prefetch)

    def batch_samples_per_cat(self, fnames):
        """The 5th element of the reference's test batch: number of annotated frames of each sample's category."""
        return np.array([self.samples_per_cat[os.path.basename(os.path.dirname(f))] for f in fnames], np.float32)
