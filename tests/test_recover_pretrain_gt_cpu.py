"""Recover-net pretraining on ground-truth flow, host side: the launch plans of CISGraph(flow_source='input'), the validation box offsets,
the FLYINGCHAIRS dataset gate, the --pretrain_flow / --validate flags and the epoch-end validation of the pretraining loop (GPU parts
stubbed)."""
import pytest

from chairs_tree import make_chairs_tree
from unsupervised_detection_b200.common_flags import FLAG_NAMES, Config
from unsupervised_detection_b200.step_graph import CISGraph

SMALL = dict(pwc_hw=(128, 192), box=(6, 32, 9, 48))


@pytest.fixture(scope='module')
def graphs():
    return (CISGraph(64, 96, 2, device='cpu', masks='boxes', flow_source='input', sample_offset=4, **SMALL),
            CISGraph(64, 96, 2, device='cpu', masks='boxes', sample_offset=4, **SMALL))


def test_input_flow_graph_builds_no_pwcnet(graphs):
    g, _ = graphs
    names = [op[2] for op in g.fwd.ops]
    assert 'cis_warp_costvol' not in names and g.pack_pwc.ops == [] and g.pwc_store.entries == []
    assert not g.with_pwc and g.img2 is None and g.flow_source == 'input'
    assert g.inputs == (g.img1, g.flow_full) and tuple(g.flow_full.shape) == (2, 128, 192, 2)
    assert 'pwcnet/' not in ''.join(g.export_params())


def test_input_flow_prefix_is_exactly_the_two_resizes(graphs):
    g, pwc = graphs
    pre = g.fwd.ops[:g._pwc_ops]
    assert [op[2] for op in pre] == ['cis_resize_bilinear_f32'] * 2 and g.fwd.ops[g._pwc_ops][2] == 'take_stage'
    assert pre[0][1] == (g.img1.data_ptr(), 2, 128, 192, 3, g.image_st.data_ptr(), 64, 96, 1.0)
    assert pre[1][1] == (g.flow_full.data_ptr(), 2, 128, 192, 2, g.flow_st.data_ptr(), 64, 96, 1.0 / 80.0)
    # the same two launches end PWC-Net's prefix; everything after the hand-over is the PWC-fed boxes graph, op for op
    assert [op[2] for op in pwc.fwd.ops[pwc._pwc_ops - 2:pwc._pwc_ops]] == ['cis_resize_bilinear_f32'] * 2
    assert pwc.fwd.ops[pwc._pwc_ops - 1][1][1:5] == pre[1][1][1:5] and pwc.fwd.ops[pwc._pwc_ops - 1][1][6:] == pre[1][1][6:]
    rest = lambda gr: [(op[2], op[4]) for op in gr.fwd.ops[gr._pwc_ops:]]
    assert rest(g) == rest(pwc)
    assert [op[2] for op in g.bwd['R'].ops] == [op[2] for op in pwc.bwd['R'].ops] and sorted(g.bwd) == ['R']
    assert g._pipe_pwc.ops == pre


def test_input_flow_needs_boxes_and_the_staged_inputs():
    with pytest.raises(ValueError):
        CISGraph(32, 48, 1, device='cpu', flow_source='input', pwc_hw=(64, 96))                  # masks='generator'
    with pytest.raises(ValueError):
        CISGraph(32, 48, 1, device='cpu', masks='boxes', flow_source='input', with_pwc=False)
    with pytest.raises(ValueError):
        CISGraph(32, 48, 1, device='cpu', masks='boxes', flow_source='gt', pwc_hw=(64, 96))


def test_set_sample_offset_rewrites_every_box_launch():
    g = CISGraph(32, 48, 2, device='cpu', masks='boxes', flow_source='input', pwc_hw=(64, 96), train=False)
    assert g.epe_sums.shape == (2, 4) and g._epe_scratch.numel() == 2 * 256
    g.set_sample_offset(17)
    for plan in (g.fwd, g._mask_plan, g._pipe_rest):
        box = [op for op in plan.ops if op[2] == 'cis_box_masks']
        assert len(box) == 1 and box[0][1][1:8] == (2, 32, 48) + g.box
        assert box[0][1][8] == 17 and box[0][1][9] == g.step_state.data_ptr() and box[0][1][10] == g.seed
    assert g.sample_offset == 17
    with pytest.raises(ValueError):
        g.set_sample_offset(-1)
    g.graphs['x'] = object()
    with pytest.raises(ValueError):
        g.set_sample_offset(3)
    with pytest.raises(ValueError):
        CISGraph(32, 48, 1, device='cpu', with_pwc=False).set_sample_offset(0)


def test_flyingchairs_is_a_pretraining_dataset_only(tmp_path):
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    root = make_chairs_tree(tmp_path, n=3, labels=[1, 1, 2])
    L = AdversarialLearner()
    L.config = Config(dataset='FLYINGCHAIRS', root_dir=root, num_threads=1)
    with pytest.raises(IOError):
        L.load_training_data()                             # train.py: no masks to validate IoU on
    L._pretrain = True
    L.load_training_data()
    assert L.num_samples_val == 1 and L.dataset_reader.train_samples == 2
    L.reader.close()


def test_pretrain_flags(monkeypatch, tmp_path):
    import pretrain_recover as PR
    from unsupervised_detection_b200.common_flags import FLAGS
    assert len(FLAG_NAMES) == 31 and 'pretrain_flow' not in FLAG_NAMES and 'validate' not in FLAG_NAMES
    assert FLAGS['pretrain_flow'].default == 'pwc' and FLAGS['validate'].default is False
    split = make_chairs_tree(tmp_path / 'split', n=2, labels=[1, 2])
    nosplit = make_chairs_tree(tmp_path / 'nosplit', n=2)
    seen = []
    monkeypatch.setattr(PR, 'run', lambda cfg: seen.append((cfg.dataset, cfg.pretrain_flow, cfg.validate, cfg.flow_ckpt)))
    ck = '--checkpoint_dir=%s' % (tmp_path / 'ck')

    def main(*args):
        FLAGS.unparse_flags()
        PR.main(['pretrain_recover.py'] + list(args))
    try:
        main(ck)
        main(ck, '--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit, '--pretrain_flow=gt')           # no --flow_ckpt needed
        main(ck, '--dataset=FLYINGCHAIRS', '--root_dir=' + split, '--pretrain_flow=gt', '--validate')
        main(ck, '--dataset=FLYINGCHAIRS', '--root_dir=' + split, '--validate')                        # PWC-Net flow, validated
        assert seen == [('DAVIS2016', 'pwc', False, ''), ('FLYINGCHAIRS', 'gt', False, ''), ('FLYINGCHAIRS', 'gt', True, ''),
                        ('FLYINGCHAIRS', 'pwc', True, '')]
        for bad in (['--pretrain_flow=gt'], ['--dataset=SYNTHETIC', '--pretrain_flow=gt'], ['--pretrain_flow=flo'],
                    ['--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit, '--pretrain_flow=gt', '--validate'],
                    ['--validate'], ['--dataset=SYNTHETIC', '--validate']):
            with pytest.raises(SystemExit):
                main(ck, *bad)
    finally:
        FLAGS.unparse_flags()
    assert len(seen) == 4


def test_gt_flow_on_a_dataset_without_flow_is_refused():
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    L = AdversarialLearner()
    L.config = Config(dataset='DAVIS2016')
    L.config.pretrain_flow = 'gt'
    L._init_dist = lambda: None
    with pytest.raises(ValueError):
        L.build_pretrain_graph()


def test_pretrain_loop_validates_every_epoch_and_keeps_the_best(capsys, tmp_path):
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    from unsupervised_detection_b200.summary import read_events

    class Reader(object):
        def batch(self, b):
            return ('i', 'j', 'f', [])

    class Graph(object):
        box = (1, 2, 3, 4)

        class rec_store(object):
            @staticmethod
            def real_count():
                return 5

    class Stub(AdversarialLearner):
        def build_pretrain_graph(self):
            self.rank, self.world, self.local_batch = 0, 1, 2
            self.reader, self.graph = Reader(), Graph()
            self.train_steps_per_epoch = 2
            self.saved, self.epes = [], iter([(3.0, 1.0), (2.0, 1.5), (2.5, 0.5), (1.0, 0.25)])

        def pretrain_step(self, batch, next_batch=None, fetch_losses=False, use_graph=True):
            self.global_step += 1
            return {'global_step': self.global_step}

        def validate_recover(self):
            return next(self.epes)

        def save_recover(self, checkpoint_dir, epoch):
            self.saved.append(epoch)

    L = Stub()
    cfg = Config(max_epochs=4, save_freq=2, summary_freq=100, checkpoint_dir=str(tmp_path))
    cfg.validate = True
    L.pretrain_recover(cfg)
    assert L.saved == ['best', 2, 'best', 4, 'best']                   # recover-<epoch> first, then the epoch's validation
    out = capsys.readouterr().out
    assert out.count('Validation EPE (boxes)') == 4 and 'Epoch [3] Validation EPE (boxes): 2.5000' in out
    L.summary_writer.close()
    ev = [e for e in read_events(L.summary_writer.path)[1:] if e['values']]
    assert [(e['step'], e['values'][0]['tag'], e['values'][0]['simple_value']) for e in ev] == [
        (1, 'Validation EPE', 3.0), (2, 'Validation EPE', 2.0), (3, 'Validation EPE', 2.5), (4, 'Validation EPE', 1.0)]


@pytest.mark.parametrize('flow_source', ['pwc', 'input'])
def test_validation_feeds_the_right_pair_and_sums_only_real_val_pairs(flow_source):
    """validate_recover with the graphs stubbed (CISGraph.feed's signature kept): each Chairs batch (img1, img2, flow, names) is fed as
    (img1, img2) on PWC-Net's flow and (img1, flow) on ground-truth flow, every batch gets its global val index as the box offset, and
    the pairs that only pad the last global batch add nothing."""
    import torch
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner

    n, lb = 5, 2
    batches = [tuple(torch.full((lb, 1), float(10 * k + j)) for j in range(3)) + (['n%d' % k] * lb,) for k in range(3)]

    class It(object):
        def __init__(self):
            self.k, self.closed = 0, False

        def shard(self, rank, world, gb):
            assert (rank, world, gb) == (0, 1, lb)
            return self

        def batch(self, b):
            assert b == lb
            self.k += 1
            return batches[self.k - 1]

        def close(self):
            self.closed = True

    class Reader(object):
        def test_inputs(self, batch_size):
            self.it = It()
            return self.it

    class ValGraph(object):
        def __init__(self):
            self.fed, self.offsets = [], []

        def load_params(self, p):
            self.params = p

        def set_sample_offset(self, off):
            self.offsets.append(off)

        def feed(self, img1, img2):                        # CISGraph.feed(img1, img2)
            self.fed.append((float(img1[0, 0]), float(img2[0, 0])))

        def forward(self):
            pass

        def masked_epe(self):                              # per sample {m*e, (1-m)*e, m, 1-m}
            return torch.tensor([[1.0, 2.0, 4.0, 8.0]] * lb, dtype=torch.float64)

    class Graph(object):
        box = (1, 2, 3, 4)

        def export_params(self):
            return {'w': 1}

    L = AdversarialLearner()
    L.config = Config(batch_size=lb, flow_normalizer=80.0)
    L.local_batch, L.num_samples_val, L.dataset_reader = lb, n, Reader()
    L.graph, L.val_graph = Graph(), ValGraph()
    L.graph.flow_source = flow_source
    epe = L.validate_recover()
    second = 2 if flow_source == 'input' else 1
    assert L.val_graph.fed == [(10.0 * k, 10.0 * k + second) for k in range(3)]
    assert L.val_graph.offsets == [0, 2, 4] and L.dataset_reader.it.closed
    assert epe == (1.0 / 4.0 * 80.0, 2.0 / 8.0 * 80.0)            # 5 real pairs: the sums' ratios, the padding pair left out
    assert L._uploads(batches[0]) == (batches[0][0], batches[0][second]) and L._uploads(None) is None
