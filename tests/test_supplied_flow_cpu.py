"""Supplied optical flow (--flow_dir), host side: the .flo naming rule, the readers' flow batches against the Flying Chairs conversion on
tiny DAVIS / FBMS / SegTrack trees, the export format round trip, the launch plans of the input-flow generator graph, and the flag and
usage errors."""
import os
import random

import numpy as np
import pytest
import torch

from flow_trees import make_tree, reader, write_flows
from unsupervised_detection_b200.data.davis2016_data_utils import ORIG_H, ORIG_W, central_crop_box, flow_file, train_augmentation
from unsupervised_detection_b200.data.flyingchairs_data_utils import (augment_flow, flow_to_grid, pwc_flow_from_uv, read_flo,
                                                                      uv_from_pwc_flow, write_flo)

DATASETS = ['DAVIS2016', 'FBMS', 'SEGTRACK']
# (training partition, test partition) of each tree
PARTS = {'DAVIS2016': ('train', 'val'), 'FBMS': ('train', 'val'), 'SEGTRACK': (None, None)}


@pytest.fixture(scope='module', params=DATASETS)
def tree(request, tmp_path_factory):
    ds = request.param
    root = make_tree(ds, tmp_path_factory.mktemp(ds.lower()))
    flow_dir = str(tmp_path_factory.mktemp(ds.lower() + '_flow'))
    rd = reader(ds, root)
    tp, vp = PARTS[ds]
    pairs = sorted(set(rd.frame_pairs(tp, 1)) | set(rd.frame_pairs(vp, 1)) | set(rd.frame_pairs(vp, -2)))
    uv = write_flows(rd, flow_dir, pairs)
    return ds, root, flow_dir, uv


def _flow_of(uv, case, box):
    return pwc_flow_from_uv(augment_flow(flow_to_grid(uv), case, *box))


# ------------------------------------------------------------------------------------------------ naming and format
def test_flow_file_names_one_file_per_ordered_pair(tmp_path):
    r = str(tmp_path / 'ds')
    f = lambda n: os.path.join(r, 'JPEGImages/480p/bear', n)
    assert flow_file('/fl', r, f('00003.jpg'), f('00001.jpg')) == '/fl/JPEGImages/480p/bear/00003__00001.flo'
    assert flow_file('/fl', r, f('00001.jpg'), f('00003.jpg')) != flow_file('/fl', r, f('00003.jpg'), f('00001.jpg'))
    with pytest.raises(ValueError):
        flow_file('/fl', r, f('00001.jpg'), os.path.join(r, 'JPEGImages/480p/bus/00002.jpg'))
    with pytest.raises(ValueError):
        flow_file('/fl', r, '/elsewhere/a.jpg', '/elsewhere/b.jpg')


def test_write_flo_round_trips_and_inverts_pwc_flow(tmp_path):
    f = np.random.RandomState(4).randn(ORIG_H, ORIG_W, 2).astype(np.float32) * 7
    p = str(tmp_path / 'a' / 'b.flo')
    write_flo(p, uv_from_pwc_flow(f))
    assert os.listdir(str(tmp_path / 'a')) == ['b.flo']                    # no temporary left behind
    back = read_flo(p)
    assert np.array_equal(pwc_flow_from_uv(back), f)
    # a 384x640 field passes the readers' conversion unchanged (no flip, crop 1.0): export then read is bit for bit
    assert np.array_equal(_flow_of(back, 0, central_crop_box(ORIG_H, ORIG_W, 1.0)), f)
    assert np.array_equal(_flow_of(back, 0, (0, 0, ORIG_H, ORIG_W)), f)


# ------------------------------------------------------------------------------------------------ readers
def test_every_listed_pair_resolves(tree):
    """Training iterators draw random shifts and directions, test iterators their fixed shift: every file they open is one the pair
    lists name (the lists are all the flow tree holds)."""
    ds, root, flow_dir, uv = tree
    tp, vp = PARTS[ds]
    rd = reader(ds, root, flow_dir=flow_dir)
    it = rd.image_inputs(batch_size=4, partition=tp, train_crop=0.8)
    n = 0
    for _ in range(12):
        b = it.batch(4, pinned=False)
        assert len(b) == 5 and b[4].shape == (4, ORIG_H, ORIG_W, 2) and b[4].dtype == torch.float32
        n += 4
    it.close()
    for t_len in (1, -2):
        it = rd.test_inputs(batch_size=2, partition=vp, t_len=t_len, test_crop=0.9)
        for _ in range(-(-len(it.pairs) // 2)):
            assert it.batch(2, pinned=False)[4].shape == (2, ORIG_H, ORIG_W, 2)
        it.close()
    # every shift in [min, max] in both directions is listed
    pairs = rd.train_frame_pairs(tp)
    assert len(pairs) == len(set(pairs)) == 3 * len(rd._probe().image_inputs(partition=tp).pairs)


def test_a_missing_flow_file_raises_ioerror_with_its_path(tree, tmp_path):
    ds, root, flow_dir, uv = tree
    tp, vp = PARTS[ds]
    rd = reader(ds, root, flow_dir=str(tmp_path))                         # an empty flow tree
    it = rd.test_inputs(batch_size=1, partition=vp, t_len=1)
    f1, f2 = rd.test_frame_pairs(vp, 1)[0]
    with pytest.raises(IOError) as e:
        it.batch(1, pinned=False)
    assert flow_file(str(tmp_path), root, f1, f2) in str(e.value)
    it.close()


def test_training_flow_follows_the_frames_draws(tree):
    ds, root, flow_dir, uv = tree
    tp, _ = PARTS[ds]
    plain, rd = reader(ds, root), reader(ds, root, flow_dir=flow_dir)
    it_p, it_f = plain.image_inputs(partition=tp, train_crop=0.7), rd.image_inputs(partition=tp, train_crop=0.7)
    cases = set()
    for k, pair in enumerate(it_f.pairs[:16]):
        seed = 1000 + k
        r = random.Random(seed)
        f1, f2 = it_f.view._train_frames(pair, r.randint(rd.min_temporal_len, rd.max_temporal_len))
        draws = train_augmentation(r, 0.7, ORIG_H, ORIG_W)
        cases.add(draws[0])
        got = it_f.view._train_sample(pair, seed)
        ref = it_p.view._train_sample(pair, seed)
        assert len(ref) == 4 and len(got) == 5
        for a, b in zip(got[:3], ref[:3]):
            assert np.array_equal(a, b)                                    # the frames do not change with a flow_dir
        assert got[3] == ref[3] == f1
        assert np.array_equal(got[4], _flow_of(uv[(f1, f2)], draws[0], draws[1:]))
    assert len(cases) >= 3
    it_p.close()
    it_f.close()


@pytest.mark.parametrize('crop', [0.9, 1.0])
def test_test_flow_follows_the_test_crop_box(tree, crop):
    ds, root, flow_dir, uv = tree
    _, vp = PARTS[ds]
    rd = reader(ds, root, flow_dir=flow_dir)
    it = rd.test_inputs(batch_size=3, partition=vp, t_len=-2, test_crop=crop)
    pairs = rd.test_frame_pairs(vp, -2)
    b = it.batch(3, pinned=False)
    it.close()
    for j in range(3):
        ref = _flow_of(uv[pairs[j]], 0, central_crop_box(ORIG_H, ORIG_W, crop))
        assert b[3][j] == pairs[j][0] and np.array_equal(b[4][j].numpy(), ref)


def test_batches_without_flow_dir_are_unchanged(tree):
    """Same seed with and without flow_dir: the same frames, masks and names, in the same order; no fifth element without it."""
    ds, root, flow_dir, uv = tree
    tp, vp = PARTS[ds]
    a, b = reader(ds, root, seed=11), reader(ds, root, seed=11, flow_dir=flow_dir)
    for mk in (lambda r: r.image_inputs(partition=tp, train_crop=0.8), lambda r: r.test_inputs(partition=vp, t_len=1, test_crop=0.9)):
        ia, ib = mk(a), mk(b)
        for _ in range(3):
            x, y = ia.batch(2, pinned=False), ib.batch(2, pinned=False)
            assert len(x) == 4 and len(y) == 5
            assert all(torch.equal(p, q) for p, q in zip(x[:3], y[:3])) and x[3] == y[3]
        ia.close()
        ib.close()


def test_listing_moves_no_reader_state(tmp_path):
    root = make_tree('DAVIS2016', tmp_path / 'd')
    a, b = reader('DAVIS2016', root, seed=5), reader('DAVIS2016', root, seed=5)
    a.frame_pairs('train', 2)
    x, y = a.image_inputs(partition='train').batch(2, pinned=False), b.image_inputs(partition='train').batch(2, pinned=False)
    assert all(torch.equal(p, q) for p, q in zip(x[:3], y[:3]))


# ------------------------------------------------------------------------------------------------ graph plans
SMALL = dict(pwc_hw=(128, 192))


@pytest.mark.parametrize('train', [True, False])
def test_input_flow_generator_graph_is_the_default_graph_minus_pwcnet(train):
    from plan_digest import digest, filled_uninitialized
    from unsupervised_detection_b200.step_graph import CISGraph

    def plans(g, prefix):
        out = [('prefix', prefix), ('rest', g._pipe_rest), ('masks_tail', g._sub_plan('m', g._mask_plan.ops[g._pwc_ops:])),
               ('pack_gen', g.pack_gen), ('pack_rec', g.pack_rec)]
        for m in sorted(g.bwd):
            out += [('bwd' + m, g.bwd[m]), ('adam' + m, g.adam[m])]
        return out
    with filled_uninitialized():
        d = CISGraph(64, 96, 2, device='cpu', train=train, **SMALL)
        i = CISGraph(64, 96, 2, device='cpu', train=train, masks='generator', flow_source='input', **SMALL)
    assert not i.with_pwc and i.staged and i.img2 is None and i.inputs == (i.img1, i.flow_full) and not i.pack_pwc.ops
    assert sorted(i.bwd) == sorted(d.bwd) == (['G', 'R'] if train else [])
    # the input graph's prefix is the default graph's two resizes after PWC-Net; everything after take_stage is op for op the same
    assert [op[2] for op in i.fwd.ops[:i._pwc_ops]] == ['cis_resize_bilinear_f32'] * 2
    assert i.fwd.ops[i._pwc_ops][2] == d.fwd.ops[d._pwc_ops][2] == 'take_stage'
    assert len(i.fwd.ops) == len(d.fwd.ops) - d._pwc_ops + i._pwc_ops
    dd = digest(plans(d, d._sub_plan('p', d.fwd.ops[d._pwc_ops - 2:d._pwc_ops])))
    di = digest(plans(i, i._sub_plan('p', i.fwd.ops[:i._pwc_ops])))
    strip = lambda lines: [ln for ln in lines if not ln.startswith('storage ')]
    assert strip(di) == strip(dd)
    assert [ln.split()[2] for ln in di if ln.startswith('storage ')] == [ln.split()[2] for ln in dd if ln.startswith('storage ')]


def test_input_flow_needs_a_named_mask_source_and_the_staged_inputs():
    from unsupervised_detection_b200.step_graph import CISGraph
    with pytest.raises(ValueError):
        CISGraph(32, 48, 1, device='cpu', flow_source='input', pwc_hw=(64, 96))                  # masks not named
    assert CISGraph(32, 48, 1, device='cpu', with_pwc=False).masks == 'generator'               # without supplied flow: the default
    for masks in ('generator', 'boxes'):
        with pytest.raises(ValueError):
            CISGraph(32, 48, 1, device='cpu', masks=masks, flow_source='input', with_pwc=False)
    with pytest.raises(ValueError):
        CISGraph(32, 48, 1, device='cpu', flow_source='gt', pwc_hw=(64, 96))
    g = CISGraph(32, 48, 1, device='cpu', masks='generator', flow_source='input', pwc_hw=(64, 96))
    assert g.masks == 'generator' and sorted(g.bwd) == ['G', 'R'] and not g.with_pwc
    with pytest.raises(ValueError):
        g.forward_flow()                                                   # no PWC-Net to run


# ------------------------------------------------------------------------------------------------ learner, flags, usage errors
def test_learner_uploads_the_supplied_flow():
    from types import SimpleNamespace as NS
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    L = AdversarialLearner()
    img1, img2, seg, flow = (torch.zeros(1) for _ in range(4))
    L.config, L.graph = NS(dataset='DAVIS2016', flow_dir='/f'), NS(flow_source='input')
    up = L._uploads((img1, img2, seg, ['n'], flow))
    assert up[0] is img1 and up[1] is flow
    up = L._uploads((img1, img2, flow, ['n']))                            # a Flying Chairs batch
    assert up[0] is img1 and up[1] is flow
    L.graph = NS(flow_source='pwc')
    up = L._uploads((img1, img2, seg, ['n']))
    assert up[0] is img1 and up[1] is img2
    assert L._flow_source() == 'input'
    L.config = NS(dataset='DAVIS2016')
    assert L._flow_source() == 'pwc' and L.flow_dir() == ''


def _exits(main, argv):
    with pytest.raises(SystemExit) as e:
        main(argv)
    return e.value.code


def test_flow_dir_flag_and_usage_errors(monkeypatch, tmp_path):
    import export_flow as EF
    import pretrain_recover as PR
    import test_generator as TG
    import test_generator_ensemble as TGE
    import train as TR
    from unsupervised_detection_b200.common_flags import FLAG_NAMES, FLAGS
    assert len(FLAG_NAMES) == 31 and 'flow_dir' not in FLAG_NAMES and FLAGS['flow_dir'].default == ''
    fd = str(tmp_path)
    seen = []
    monkeypatch.setattr(TR, 'run', lambda cfg: seen.append(('train', cfg.flow_dir)))
    monkeypatch.setattr(PR, 'run', lambda cfg: seen.append(('pretrain', cfg.flow_dir)))
    monkeypatch.setattr(TG, '_test_masks', lambda: seen.append(('test', FLAGS.flow_dir)))
    monkeypatch.setattr(TGE, '_test_masks', lambda: seen.append(('ensemble', FLAGS.flow_dir)))
    monkeypatch.setattr(EF, 'export', lambda cfg: seen.append(('export', cfg.flow_dir)))
    ck = '--checkpoint_dir=%s' % (tmp_path / 'ck')
    try:
        TR.main(['train.py'])
        TR.main(['train.py', '--flow_dir=' + fd])
        TG.main(['test_generator.py', '--dataset=FBMS', '--flow_dir=' + fd])
        TGE.main(['test_generator_ensemble.py', '--dataset=SEGTRACK', '--flow_dir=' + fd])
        PR.main(['pretrain_recover.py', ck, '--pretrain_flow=gt', '--flow_dir=' + fd])
        EF.main(['export_flow.py', '--flow_dir=' + str(tmp_path / 'new'), '--flow_ckpt=synthetic'])
        assert seen == [('train', ''), ('train', fd), ('test', fd), ('ensemble', fd), ('pretrain', fd), ('export', str(tmp_path / 'new'))]
        for bad in (['--dataset=SYNTHETIC', '--flow_dir=' + fd], ['--flow_dir=' + str(tmp_path / 'absent')]):
            assert _exits(TR.main, ['train.py'] + bad)
        for bad in (['--flow_dir=' + fd], ['--dataset=FLYINGCHAIRS', '--pretrain_flow=gt', '--flow_dir=' + fd],
                    ['--pretrain_flow=gt', '--flow_dir=' + fd, '--validate']):
            assert _exits(PR.main, ['pretrain_recover.py', ck] + bad)
        for bad in (['--flow_ckpt=synthetic'], ['--flow_dir=' + fd], ['--dataset=SYNTHETIC', '--flow_ckpt=synthetic', '--flow_dir=' + fd]):
            assert _exits(EF.main, ['export_flow.py'] + bad)
    finally:
        FLAGS.unparse_flags()


def test_pretraining_on_a_mask_dataset_needs_gt_with_a_flow_dir():
    from unsupervised_detection_b200.common_flags import Config
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner, has_flow
    assert has_flow('DAVIS2016', '/f') and not has_flow('DAVIS2016', '') and has_flow('FLYINGCHAIRS', '') and not has_flow('SYNTHETIC', '/f')
    for pf, fd in (('gt', ''), ('pwc', '/f')):
        L = AdversarialLearner()
        L.config = Config(dataset='DAVIS2016')
        L.config.pretrain_flow, L.config.flow_dir = pf, fd
        L._init_dist = lambda: None
        with pytest.raises(ValueError):
            L.build_pretrain_graph()


def test_export_pairs_are_the_readers_lists(tmp_path):
    import export_flow as EF
    from unsupervised_detection_b200.common_flags import Config
    root = make_tree('DAVIS2016', tmp_path / 'd')
    cfg = Config(dataset='DAVIS2016', root_dir=root, train_partition='train', test_partition='val', test_temporal_shift=-1)
    rd = EF.make_reader(cfg)
    got = EF.export_pairs(cfg, rd)
    want = set(pr for p in ('train', 'val') for pr in rd.train_frame_pairs(p) + rd.test_frame_pairs(p, -1))
    assert got == sorted(want) and len(got) == len(set(got))
    assert all(os.path.dirname(a) == os.path.dirname(b) and a != b for a, b in got)


def test_the_learner_refuses_a_flow_dir_it_cannot_read(tmp_path):
    """test_generator*.py parse --flow_dir through the learner's import and meet these errors when the learner opens the dataset."""
    from unsupervised_detection_b200.common_flags import Config
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    root = make_tree('DAVIS2016', tmp_path / 'd')
    for ds, fd, err in (('SYNTHETIC', str(tmp_path), ValueError), ('DAVIS2016', str(tmp_path / 'absent'), IOError)):
        L = AdversarialLearner()
        L.config = Config(dataset=ds, root_dir=root, num_threads=1)
        L.config.flow_dir = fd
        with pytest.raises(err):
            L.load_training_data()
    L = AdversarialLearner()
    L.config = Config(dataset='DAVIS2016', root_dir=root, num_threads=1, train_partition='train')
    L.config.flow_dir = str(tmp_path)
    L.load_training_data()
    assert L.dataset_reader.flow_dir == str(tmp_path)
    L.reader.close()
    L.val_reader.close()
