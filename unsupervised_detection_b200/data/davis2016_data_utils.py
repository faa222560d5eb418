"""Host-side DAVIS2016 reader (SURVEY.md section 8f-2): the reference's tf.data pipeline (data/davis2016_data_utils.py:6-354,
data/aug_flips.py:35-45) restated with numpy + OpenCV + a thread pool, feeding pinned torch tensors to AdversarialLearner.

Same folder contract (`ImageSets/480p/{train,val,trainval}.txt` listing `/JPEGImages/480p/<seq>/<frame>.jpg
/Annotations/480p/<seq>/<frame>.png`), same sampling (frame pairs with a temporal shift in [min,max]_temporal_len forward from
the head of a sequence / backward from its tail), same preprocessing (x/255-0.5, legacy-bilinear resize to 384x640, random
flips applied to both frames, random / central crop resized back).  JPEG decoding and augmentation stay on the CPU.

Supplied flow (flow_dir, not in the reference): the flow of a frame pair is one Middlebury .flo file under flow_dir (flow_file gives its
name), read next to the frames and added to every batch as a fifth element, (img1, img2, seg1, fnames, flow [B,384,640,2]) in PWC-Net's
channel order and sign.  It goes through the Flying Chairs conversion: resampled to 384x640 with its vectors rescaled
(flow_to_grid), then flipped and cropped with the frames' own draws (augment_flow) for a training pair, or cut to the same central
test_crop box for a test pair, and finally pwc_flow_from_uv.  This is a geometric transform of the field: PWC-Net run on the augmented
frames gives the same flow only for no flip and a crop of 1.0.  Without flow_dir every batch is what it was.
"""
import collections
import copy
import os
import queue
import random
import threading
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import torch

from .. import _lib

ORIG_H, ORIG_W = 384, 640   # preprocess_image :87-90


def flow_file(flow_dir, root_dir, f1, f2):
    """The .flo file of the frame pair (f1, f2), frame paths under root_dir: <flow_dir>/<directory of f1 relative to root_dir>/<file
    name of f1 without extension>__<file name of f2 without extension>.flo, e.g. JPEGImages/480p/bear/00003__00001.flo for frame 3 to
    frame 1.  One file per ordered pair, so every temporal shift and direction has its own.  The two frames must share a directory
    (the readers never pair frames of two sequences); ValueError otherwise, and for a frame outside root_dir."""
    d1, d2 = (os.path.dirname(os.path.relpath(f, root_dir)) for f in (f1, f2))
    if d1 != d2 or d1 == os.pardir or d1.startswith(os.pardir + os.sep):
        raise ValueError('frame pair %s, %s: both frames must lie in one directory under %s' % (f1, f2, root_dir))
    stem = lambda f: os.path.splitext(os.path.basename(f))[0]
    return os.path.join(flow_dir, d1, '%s__%s.flo' % (stem(f1), stem(f2)))


class DirectoryIterator(object):
    """davis2016_data_utils.py:6-65."""

    def __init__(self, directory, part='train'):
        self.directory = directory
        name_division = {'train': 'ImageSets/480p/train.txt', 'val': 'ImageSets/480p/val.txt', 'trainval': 'ImageSets/480p/trainval.txt'}
        if part not in name_division:
            raise IOError("Partition file not found")
        part_file = os.path.join(directory, name_division[part])
        if not os.path.isfile(part_file):
            raise IOError("Partition file not found")
        self.components = np.loadtxt(part_file, dtype=str, ndmin=2)
        self.samples = 0
        self.image_filenames = []
        self.annotation_filenames = []
        self._parse_components(self.components)
        if self.samples == 0:
            raise IOError("Did not find any file in the dataset folder")
        self.num_experiments = len(self.image_filenames)
        print('Found {} images belonging to {} experiments.'.format(self.samples, self.num_experiments))

    def _parse_components(self, components):
        current_experiment, cur_f, cur_a = '', None, None
        for string in components:
            folder_name = string[0].split('/')[3]
            if folder_name != current_experiment:
                current_experiment = folder_name
                if cur_f is not None:
                    self.image_filenames.append(cur_f)
                    self.annotation_filenames.append(cur_a)
                cur_f, cur_a = [], []
            cur_f.append(os.path.join(self.directory, string[0][1:]))
            cur_a.append(os.path.join(self.directory, string[1][1:]))
            self.samples += 1
        if cur_f is not None:
            self.image_filenames.append(cur_f)
            self.annotation_filenames.append(cur_a)


def legacy_resize(x, oh, ow):
    """tf.image.resize_images (legacy bilinear, App. A.6) on an HWC float32 array -- libcis_b200's host routine
    (cis_host_resize_bilinear_legacy, ~2 ms per 384x640x3 frame, GIL released); bit-identical to `legacy_resize_numpy`."""
    h, w = x.shape[:2]
    if (h, w) == (oh, ow):
        return x
    x = np.ascontiguousarray(x, dtype=np.float32)
    if x.ndim == 2:
        x = x[..., None]
    out = np.empty((oh, ow, x.shape[2]), np.float32)
    _lib.check(_lib.load().cis_host_resize_bilinear_legacy(x.ctypes.data, h, w, x.shape[2], out.ctypes.data, oh, ow), 'host resize')
    return out


def legacy_resize_numpy(x, oh, ow):
    """The same resize written with numpy gathers (about 15x slower): the restatement the C routine is tested against."""
    h, w = x.shape[:2]
    if (h, w) == (oh, ow):
        return x

    def ax(n_in, n_out):
        s = np.arange(n_out, dtype=np.float32) * np.float32(n_in / n_out)
        lo = np.floor(s).astype(np.int64)
        return lo, np.minimum(lo + 1, n_in - 1), (s - lo).astype(np.float32)
    hl, hh, hf = ax(h, oh)
    wl, wh, wf = ax(w, ow)
    top, bot = x[hl], x[hh]
    wf = wf[None, :, None]
    t = top[:, wl] + (top[:, wh] - top[:, wl]) * wf
    b = bot[:, wl] + (bot[:, wh] - bot[:, wl]) * wf
    return t + (b - t) * hf[:, None, None]


def nn_resize(x, oh, ow):
    """tf.image.resize_images(method=NEAREST_NEIGHBOR), align_corners=False."""
    h, w = x.shape[:2]
    yi = np.minimum(np.floor(np.arange(oh, dtype=np.float32) * np.float32(h / oh)).astype(np.int64), h - 1)
    xi = np.minimum(np.floor(np.arange(ow, dtype=np.float32) * np.float32(w / ow)).astype(np.int64), w - 1)
    return x[yi][:, xi]


def train_augmentation(r, train_crop, h, w):
    """The random draws of one training sample's augmentation (augment_pair :136-148 + aug_flips.random_flip_images), in the reference's
    order, from the random.Random r: the flip case (0 keep | 1 rotate 180 | 2 left-right | 3 top-down, 25 % each), then the crop
    fraction pct in [train_crop, 1) and the crop's corner (random_crop_image_pair :101-128) -> (case, y0, x0, ch, cw)."""
    case = r.randrange(4)
    pct = train_crop + r.random() * (1 - train_crop)
    ch, cw = int(h * pct), int(w * pct)
    y0, x0 = r.randint(0, h - ch), r.randint(0, w - cw)
    return case, y0, x0, ch, cw


def flip(x, case):
    """The flip of train_augmentation's case on an HWC array (a view)."""
    return (x, x[::-1, ::-1], x[:, ::-1], x[::-1])[case]


def crop_resized(x, y0, x0, ch, cw):
    """The crop [y0:y0+ch, x0:x0+cw] of an HWC array, legacy-bilinear resized back to the array's size."""
    h, w = x.shape[:2]
    return legacy_resize(np.ascontiguousarray(x[y0:y0 + ch, x0:x0 + cw]), h, w)


def central_crop_box(h, w, frac):
    """tf.image.central_crop geometry: offset = int((dim - dim*frac)/2), size = dim - 2*offset."""
    y0 = int((h - h * frac) / 2)
    x0 = int((w - w * frac) / 2)
    return y0, x0, h - 2 * y0, w - 2 * x0


class _Iter(object):
    """Endless batch iterator with the interface AdversarialLearner uses: .batch(n) -> (img1, img2, seg1, fnames).

    `prefetch` > 0 keeps that many batches decoded ahead of the consumer in a background thread (the reference's
    `dataset.prefetch(3 * batch_size)`, davis2016_data_utils.py:226): host decoding / augmentation of the next batches overlaps the
    GPU step that consumes the current one.  For a constant batch size, order and content are the same with or without prefetching
    (one producer, FIFO queue, iterator-private random stream); changing the batch size restarts the producer and drops what it had
    decoded ahead.  state() / restore() save and resume the stream at the consumer's position, which resumable training stores."""

    def __init__(self, reader, pairs, train, shuffle, num_threads, prefetch=0):
        # Snapshot of the reader as it is NOW (file lists, temporal shift, crops): a later image_inputs()/test_inputs() call on the
        # same reader rebinds those attributes for ITS iterator and must not change what this one decodes -- the reference gets the
        # same isolation from tf.gather(self.filenames) being captured as a graph constant when each dataset map is traced.
        self.reader, self.view = reader, copy.copy(reader)
        self.pairs, self.train, self.shuffle = list(pairs), train, shuffle
        self.pool = ThreadPoolExecutor(max_workers=max(1, num_threads))
        self.rng = random.Random(reader.rng.getrandbits(64))     # private stream: iterators of one reader do not interleave draws
        self.pos = 0
        self.order = list(range(len(self.pairs)))
        if shuffle:
            self.rng.shuffle(self.order)
        self.prefetch = prefetch
        self._q = self._thread = self._qn = None
        self._stop = threading.Event()
        self._at = self._position()                 # state(): the stream position of the next batch batch() returns

    def _position(self):
        return {'rng': self.rng.getstate(), 'pos': self.pos, 'order': list(self.order)}

    def state(self):
        """The stream position of the next batch batch() returns (not of what the background producer has drawn ahead): random state,
        list position and order.  restore(state()) on an iterator over the same pairs makes it return the same batches from there."""
        return self._at

    def restore(self, state):
        """Continue from a position state() returned; batches decoded ahead are dropped."""
        self.close()
        self.rng.setstate(state['rng'])
        self.pos, self.order = state['pos'], list(state['order'])
        self._at = self._position()

    def shard(self, rank, world, global_batch):
        """Data-parallel evaluation: global batch k is samples [k*B, (k+1)*B) of the ordered list (wrapping at the end, like
        dataset.repeat); rank r reads its contiguous slice of every global batch, so the ranks together see each global batch exactly
        once.  Ordered iterators only (training iterators are shuffled per rank instead)."""
        self.global_names = [self._name_of(pr) for pr in self.pairs]      # first-frame file name of every list position
        if world <= 1:
            return self
        assert not self.shuffle and global_batch % world == 0
        lb, n = global_batch // world, len(self.pairs)
        steps = -(-n // global_batch)
        self.close()
        self.order = [(k * global_batch + rank * lb + j) % n for k in range(steps) for j in range(lb)]
        self.pos = 0
        self._at = self._position()
        return self

    def _name_of(self, pair):
        return pair[0] if isinstance(pair[0], str) else self.view.filenames[int(pair[0])]

    def _next_index(self):
        if self.pos >= len(self.order):          # dataset.repeat(None) (+ reshuffle_each_iteration)
            self.pos = 0
            if self.shuffle:
                self.rng.shuffle(self.order)
        i = self.order[self.pos]
        self.pos += 1
        return i

    def _submit(self, n):
        """Draw the next n samples (indices + augmentation seeds, in stream order) and hand them to the thread pool -> (their futures, the
        stream position after the draws)."""
        idx = [self._next_index() for _ in range(n)]
        fn = self.view._train_sample if self.train else self.view._test_sample
        seeds = [self.rng.getrandbits(32) for _ in idx]
        return [self.pool.submit(fn, self.pairs[i], sd) for i, sd in zip(idx, seeds)], self._position()

    @staticmethod
    def _collect(drawn):
        """_submit's (futures, position) -> ([img1, img2, seg1, fnames] (+ [flow] when the samples carry a supplied flow field as a fifth
        element), position)."""
        futs, at = drawn
        res = [f.result() for f in futs]
        out = [torch.from_numpy(np.stack([r[k] for r in res])) for k in range(3)] + [[r[3] for r in res]]
        return (out + [torch.from_numpy(np.stack([r[4] for r in res]))] if len(res[0]) > 4 else out), at

    def _make(self, n):
        return self._collect(self._submit(n))

    def _producer(self, n, q, stop):
        inflight = collections.deque()           # several batches are decoded concurrently so all pool threads stay busy
        while not stop.is_set():
            while len(inflight) < max(1, self.prefetch):
                inflight.append(self._submit(n))
            try:
                item = self._collect(inflight.popleft())
            except Exception as e:               # surfaces in the consumer's batch() call
                item = e
            while not stop.is_set():
                try:
                    q.put(item, timeout=0.1)
                    break
                except queue.Full:
                    continue
            if isinstance(item, Exception):
                break
        for futs, _ in inflight:
            for f in futs:
                f.cancel()

    def close(self):
        """Stop the background producer (batches already decoded ahead are dropped)."""
        if self._thread is not None:
            self._stop.set()
            self._thread.join(timeout=5)
            self._q = self._thread = self._qn = None
            self._stop = threading.Event()

    def __del__(self):
        try:
            self._stop.set()
        except Exception:
            pass

    def batch(self, n, pinned=True):
        if self.prefetch > 0:
            if self._qn != n:                    # (re)start the producer for this batch size
                self.close()
                self._q, self._qn = queue.Queue(maxsize=self.prefetch), n
                self._thread = threading.Thread(target=self._producer, args=(n, self._q, self._stop), daemon=True)
                self._thread.start()
            item = self._q.get()
            if isinstance(item, Exception):
                self.close()
                raise item
            out, self._at = item
        else:
            out, self._at = self._make(n)
        ts = out[:3] + out[4:]
        if pinned and torch.cuda.is_available():
            ts = [t.pin_memory() for t in ts]
        return (ts[0], ts[1], ts[2], out[3]) + tuple(ts[3:])


class Davis2016Reader(object):
    """davis2016_data_utils.py:68-354."""

    def __init__(self, root_dir, max_temporal_len=3, min_temporal_len=1, num_threads=6, seed=8964, flow_dir=''):
        """flow_dir: root of the supplied .flo files (flow_file); '' = frames only."""
        self.root_dir, self.flow_dir = root_dir, flow_dir
        self.max_temporal_len, self.min_temporal_len = max_temporal_len, min_temporal_len
        assert min_temporal_len < max_temporal_len, "Temporal lenghts are not consistenst"
        assert min_temporal_len > 0, "Min temporal len should be positive"
        self.num_threads = num_threads
        self.rng = random.Random(seed)
        self.prefetch = int(os.environ.get('CIS_READER_PREFETCH', '3'))     # training batches decoded ahead (0 = synchronous)

    def get_filenames_list(self, partition):
        it = DirectoryIterator(self.root_dir, partition)
        self.val_samples = it.samples
        return it.image_filenames, it.annotation_filenames

    # ---- preprocessing (:84-99)
    @staticmethod
    def preprocess_image(path):
        bgr = cv2.imread(path, cv2.IMREAD_COLOR)
        if bgr is None:
            raise IOError("Could not read image %s" % path)
        # BGR uint8 -> RGB float (v/255 - 0.5) -> legacy bilinear 384x640 in one pass of libcis_b200's host routine
        bgr = np.ascontiguousarray(bgr)
        out = np.empty((ORIG_H, ORIG_W, 3), np.float32)
        _lib.check(_lib.load().cis_host_bgr8_to_rgb_resized(bgr.ctypes.data, bgr.shape[0], bgr.shape[1], out.ctypes.data, ORIG_H, ORIG_W),
                   'host preprocess')
        return out

    @staticmethod
    def preprocess_mask(path):
        m = cv2.imread(path, cv2.IMREAD_GRAYSCALE)
        if m is None:
            raise IOError("Could not read annotation %s" % path)
        return nn_resize(m.astype(np.float32)[..., None] / np.float32(255.0), ORIG_H, ORIG_W)

    @staticmethod
    def central_cropping(img, frac, nearest=False):
        h, w = img.shape[:2]
        y0, x0, ch, cw = central_crop_box(h, w, frac)
        c = img[y0:y0 + ch, x0:x0 + cw]
        return nn_resize(c, h, w) if nearest else legacy_resize(c, h, w)   # the reference resizes masks bilinearly here too (:133)

    # ---- supplied flow
    def flow_path(self, f1, f2):
        """The .flo file of the frame pair (f1, f2) under self.flow_dir (flow_file)."""
        return flow_file(self.flow_dir, self.root_dir, f1, f2)

    def _with_flow(self, sample, f1, f2, case, box):
        """sample + (the supplied flow of (f1, f2) after flip `case` and crop `box` = (y0, x0, ch, cw) of the 384x640 grid,) when a
        flow_dir is set.  IOError naming the file when it is missing or unreadable."""
        if not self.flow_dir:
            return sample
        from .flyingchairs_data_utils import augment_flow, flow_to_grid, pwc_flow_from_uv, read_flo
        path = self.flow_path(f1, f2)
        if not os.path.isfile(path):
            raise IOError('missing flow file %s (frame pair %s -> %s)' % (path, f1, f2))
        return sample + (pwc_flow_from_uv(augment_flow(flow_to_grid(read_flo(path)), case, *box)).astype(np.float32),)

    # ---- samples
    def _train_frames(self, pair, t_shift):
        """(frame 1, frame 2) file names of training pair `pair` = (index of frame 1, direction) at temporal shift t_shift."""
        i1, direction = pair
        return self.filenames[i1], self.filenames[int(t_shift * direction + i1)]

    def _test_frames(self, pair):
        """(frame 1, frame 2) file names of test pair `pair`."""
        i1, direction = pair
        return self.filenames[i1], self.filenames[int(self.test_t_len * direction + i1)]

    def _train_sample(self, pair, seed):
        """dataset_map :150-178 + augment_pair :136-148 + aug_flips.random_flip_images."""
        r = random.Random(seed)
        f1, f2 = self._train_frames(pair, r.randint(self.min_temporal_len, self.max_temporal_len))
        a, b = self.preprocess_image(f1), self.preprocess_image(f2)
        h, w = a.shape[:2]
        case, y0, x0, ch, cw = train_augmentation(r, self.train_crop, h, w)
        a = crop_resized(flip(a, case), y0, x0, ch, cw)
        b = crop_resized(flip(b, case), y0, x0, ch, cw)
        sample = a.astype(np.float32), b.astype(np.float32), np.ones((h, w, 1), np.float32), f1
        return self._with_flow(sample, f1, f2, case, (y0, x0, ch, cw))

    def _test_sample(self, pair, seed):
        """test_dataset_map :293-326."""
        f1, f2 = self._test_frames(pair)
        a, b = self.preprocess_image(f1), self.preprocess_image(f2)
        s = self.preprocess_mask(self.annotation_filenames[pair[0]])
        c = self.test_crop
        sample = (self.central_cropping(a, c).astype(np.float32), self.central_cropping(b, c).astype(np.float32),
                  self.central_cropping(s, c).astype(np.float32), f1)
        return self._with_flow(sample, f1, f2, 0, central_crop_box(ORIG_H, ORIG_W, c))

    # ---- the frame pairs a partition can draw (the files export_flow.py writes and a flow_dir must hold).  They are read off the
    # iterators themselves, built on a copy of the reader so that neither its state nor its random stream moves.
    def _probe(self):
        rd = copy.copy(self)
        rd.rng, rd.prefetch = random.Random(0), 0
        return rd

    def train_frame_pairs(self, partition='train'):
        """Every (frame 1, frame 2) file pair image_inputs(partition=partition) can draw: each forward / backward pair at each shift in
        [min_temporal_len, max_temporal_len]."""
        it = self._probe().image_inputs(partition=partition)
        shifts = range(self.min_temporal_len, self.max_temporal_len + 1)
        return [it.view._train_frames(pr, s) for pr in it.pairs for s in shifts]

    def test_frame_pairs(self, partition='val', t_len=2):
        """The (frame 1, frame 2) file pairs of test_inputs(partition=partition, t_len=t_len), in its order."""
        it = self._probe().test_inputs(partition=partition, t_len=t_len)
        return [it.view._test_frames(pr) for pr in it.pairs]

    def frame_pairs(self, partition, t_len):
        """Sorted, without repeats: every pair a training iterator and a test iterator at temporal shift t_len of `partition` read."""
        return sorted(set(self.train_frame_pairs(partition)) | set(self.test_frame_pairs(partition, t_len)))

    # ---- iterators
    def image_inputs(self, batch_size=32, partition='train', train_crop=1.0, num_threads=6):
        """:180-230 -> endless shuffled iterator of augmented training pairs."""
        t_len = self.max_temporal_len
        file_list, _ = self.get_filenames_list(partition)
        self.train_crop = train_crop
        pairs, N = [], 0
        for fnames in file_list:
            pairs += [(i, 1.0) for i in range(N, N + len(fnames) - t_len)]       # forward from the head
            N += len(fnames)
        N = 0
        for fnames in file_list:
            pairs += [(i, -1.0) for i in range(N + t_len, N + len(fnames))]      # backward from the tail
            N += len(fnames)
        self.filenames = [f for fl in file_list for f in fl]
        return _Iter(self, pairs, train=True, shuffle=True, num_threads=self.num_threads, prefetch=self.prefetch)

    def test_inputs(self, batch_size=32, partition='val', t_len=2, with_fname=False, test_crop=1.0):
        """:233-290 -> ordered iterator (img_1, img_2, seg_1, fname); time(img2)-time(img1) = t_len except at sequence ends."""
        file_list, ann_list = self.get_filenames_list(partition)
        self.test_crop = test_crop
        first, last, N = [], [], 0
        for fnames in file_list:
            if t_len < 0:
                last += list(range(N + abs(t_len), N + len(fnames)))
                first += list(range(N, N + abs(t_len)))
            elif t_len > 0:
                first += list(range(N, N + len(fnames) - t_len))
                last += list(range(N + len(fnames) - t_len, N + len(fnames)))
            N += len(fnames)
        self.test_t_len = abs(t_len)
        self.filenames = [f for fl in file_list for f in fl]
        self.annotation_filenames = [f for fl in ann_list for f in fl]
        pairs = [(i, 1.0) for i in first] + [(i, -1.0) for i in last]
        # ordered: the FIFO prefetch queue keeps the list order even with several decoding threads (the reference pins num_threads=1 for that)
        return _Iter(self, pairs, train=False, shuffle=False, num_threads=self.num_threads, prefetch=self.prefetch)
