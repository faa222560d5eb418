"""Flying Chairs reader (data/flyingchairs_data_utils.py) on a tiny cv2-written tree: .flo parsing and its errors, the train / val split,
the flow's resampling, augmentation and vector transform against closed forms, and the channel convention pinned by the warp."""
import os
import random

import numpy as np
import pytest
import torch

from chairs_tree import CH, CW, make_chairs_tree, pattern, shifted, write_flo
from unsupervised_detection_b200.data import flyingchairs_data_utils as FC
from unsupervised_detection_b200.data.davis2016_data_utils import train_augmentation


def test_flo_round_trip(tmp_path):
    uv = np.random.default_rng(0).normal(size=(7, 11, 2)).astype(np.float32)
    p = str(tmp_path / 'a.flo')
    write_flo(p, uv)
    got = FC.read_flo(p)
    assert got.dtype == np.float32 and got.shape == (7, 11, 2) and np.array_equal(got, uv)


def test_flo_errors_name_the_file(tmp_path):
    uv = np.zeros((4, 5, 2), np.float32)
    bad_tag, trunc, nan = (str(tmp_path / n) for n in ('tag.flo', 'trunc.flo', 'nan.flo'))
    write_flo(bad_tag, uv, tag=1.0)
    write_flo(trunc, uv)
    with open(trunc, 'r+b') as f:
        f.truncate(12 + 8 * 20 - 4)
    uv_nan = uv.copy()
    uv_nan[2, 3, 1] = np.nan
    write_flo(nan, uv_nan)
    for path, what in ((bad_tag, 'tag'), (trunc, 'truncated'), (nan, 'non-finite')):
        with pytest.raises(IOError) as e:
            FC.read_flo(path)
        assert path in str(e.value) and what in str(e.value)
    with open(trunc, 'wb') as f:
        f.write(b'\x00' * 5)
    with pytest.raises(IOError):
        FC.read_flo(trunc)


def test_split_counts_with_and_without_the_split_file(tmp_path):
    root = make_chairs_tree(tmp_path / 'split', n=5, labels=[1, 2, 1, 1, 2])
    rd = FC.FlyingChairsReader(root, num_threads=1)
    assert (rd.train_samples, rd.val_samples, rd.has_split) == (3, 2, True)
    assert [os.path.basename(p[0]) for p in rd.val_pairs] == ['00002_img1.ppm', '00005_img1.ppm']
    root = make_chairs_tree(tmp_path / 'nosplit', n=4)
    rd = FC.FlyingChairsReader(root, num_threads=1)
    assert (rd.train_samples, rd.val_samples, rd.has_split) == (4, 0, False)
    with pytest.raises(IOError):
        rd.test_inputs()
    bad = make_chairs_tree(tmp_path / 'bad', n=3, labels=[1, 2])
    with pytest.raises(IOError):
        FC.FlyingChairsReader(bad)
    with pytest.raises(IOError):
        FC.FlyingChairsReader(str(tmp_path / 'empty'))


def _linear(a, b, c, d, e, f):
    y, x = np.mgrid[0:CH, 0:CW].astype(np.float32)
    return np.stack([a + b * x + c * y, d + e * x + f * y], -1).astype(np.float32)


def _closed_form(coef, case, y0, x0, ch, cw):
    """The converted flow at every 384x640 pixel for the linear source field `coef`: crop-resize -> flip -> grid -> source."""
    a, b, c, d, e, f = coef
    yy, xx = np.mgrid[0:384, 0:640].astype(np.float64)
    xf, yf = x0 + xx * (cw / 640.0), y0 + yy * (ch / 384.0)                # position in the flipped 384x640 grid
    xg = 639.0 - xf if case in (1, 2) else xf
    yg = 383.0 - yf if case in (1, 3) else yf
    xs, ys = xg * (CW / 640.0), yg                                         # position in the 384x512 source
    su = -1.0 if case in (1, 2) else 1.0
    sv = -1.0 if case in (1, 3) else 1.0
    u = (a + b * xs + c * ys) * (640.0 / CW) * su * (640.0 / cw)
    v = (d + e * xs + f * ys) * sv * (384.0 / ch)
    return np.stack([-v, -u], -1)


def _seeds_for_every_case(train_crop):
    seen = {}
    for sd in range(200):
        case = train_augmentation(random.Random(sd), train_crop, 384, 640)[0]
        seen.setdefault(case, sd)
        if len(seen) == 4:
            return [seen[k] for k in range(4)]
    raise AssertionError('no seed for every flip case')


@pytest.mark.parametrize('field', ['constant', 'linear'])
@pytest.mark.parametrize('train_crop', [1.0, 0.9])
def test_training_flow_matches_the_closed_form(tmp_path, field, train_crop):
    coef = (1.5, 0.0, 0.0, -2.25, 0.0, 0.0) if field == 'constant' else (0.7, 0.011, -0.006, -1.2, 0.004, 0.013)
    root = make_chairs_tree(tmp_path, n=1, flows=[_linear(*coef)])
    rd = FC.FlyingChairsReader(root, num_threads=1)
    rd.train_crop = train_crop
    for sd in _seeds_for_every_case(train_crop):
        case, y0, x0, ch, cw = train_augmentation(random.Random(sd), train_crop, 384, 640)
        a, b, flow, name = rd._train_sample(rd.train_pairs[0], sd)
        assert flow.shape == (384, 640, 2) and flow.dtype == np.float32 and a.shape == (384, 640, 3) and name == rd.train_pairs[0][0]
        ref = _closed_form(coef, case, y0, x0, ch, cw)
        if train_crop == 1.0:
            assert (ch, cw) == (384, 640)
        inner = (slice(None), slice(None)) if field == 'constant' else (slice(4, -4), slice(4, -4))
        err = np.abs(flow[inner] - ref[inner]).max()
        assert err <= 2e-4 * max(1.0, np.abs(ref).max()), (case, y0, x0, ch, cw, err)
    # validation pairs: the same conversion without augmentation
    _, _, flow, _ = rd._test_sample(rd.train_pairs[0], 0)
    ref = _closed_form(coef, 0, 0, 0, 384, 640)
    assert np.abs(flow[4:-4, 4:-4] - ref[4:-4, 4:-4]).max() <= 2e-4 * max(1.0, np.abs(ref).max())


def test_frames_get_the_same_augmentation_as_the_davis_reader(tmp_path):
    from unsupervised_detection_b200.data.davis2016_data_utils import Davis2016Reader, crop_resized, flip
    root = make_chairs_tree(tmp_path, n=1)
    rd = FC.FlyingChairsReader(root, num_threads=1)
    rd.train_crop = 0.8
    pair = rd.train_pairs[0]
    for sd in _seeds_for_every_case(0.8):
        case, y0, x0, ch, cw = train_augmentation(random.Random(sd), 0.8, 384, 640)
        a, b, _, _ = rd._train_sample(pair, sd)
        for got, path in ((a, pair[0]), (b, pair[1])):
            assert np.array_equal(got, crop_resized(flip(Davis2016Reader.preprocess_image(path), case), y0, x0, ch, cw))


def test_warping_frame_2_with_the_converted_flow_reproduces_frame_1(tmp_path):
    """Pins pwc_flow_from_uv: with the flow as the reader hands it over, PWC-Net's own warp (oracle dense_image_warp) maps frame 2
    onto frame 1.  The unconverted (u, v) field does not."""
    from oracle.pwcnet import dense_image_warp
    root = make_chairs_tree(tmp_path, n=1, shift=(4, 2))               # 4 px at 512 wide = 5 px at 640 wide; 2 px vertically
    rd = FC.FlyingChairsReader(root, num_threads=1)
    a, b, flow, _ = rd._test_sample(rd.train_pairs[0], 0)
    assert np.allclose(flow[..., 0], -2.0) and np.allclose(flow[..., 1], -5.0)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x))[None].double()
    warped = dense_image_warp(t(b), t(flow))[0].numpy()
    inner = (slice(4, -8), slice(4, -8))
    assert np.abs(warped[inner] - a[inner]).max() < 1e-3
    uv = np.stack([-flow[..., 1], -flow[..., 0]], -1)                   # back to Middlebury (u, v)
    assert np.abs(dense_image_warp(t(b), t(uv))[0].numpy()[inner] - a[inner]).max() > 0.05


def test_batches_are_pinned_shaped_and_sharded(tmp_path, monkeypatch):
    monkeypatch.setenv('CIS_READER_PREFETCH', '2')
    root = make_chairs_tree(tmp_path, n=6, labels=[1, 1, 1, 2, 2, 2])
    rd = FC.FlyingChairsReader(root, num_threads=2)
    it = rd.image_inputs(batch_size=2, train_crop=0.9)
    img1, img2, flow, names = it.batch(2)
    assert img1.shape == (2, 384, 640, 3) and img2.shape == (2, 384, 640, 3) and flow.shape == (2, 384, 640, 2) and len(names) == 2
    assert all(n in [p[0] for p in rd.train_pairs] for n in names)
    it.close()
    # the val iterator is ordered and unaugmented; shard gives rank r its slice of every global batch
    full = rd.test_inputs().shard(0, 1, 2)
    seq = [full.batch(1)[3][0] for _ in range(3)]
    full.close()
    assert seq == [p[0] for p in rd.val_pairs]
    r1 = rd.test_inputs().shard(1, 2, 2)
    got = [r1.batch(1)[3][0] for _ in range(2)]
    r1.close()
    assert got == [rd.val_pairs[1][0], rd.val_pairs[0][0]]              # global batches [0,1], [2,0(wrap)]: rank 1 reads 1, then 0
