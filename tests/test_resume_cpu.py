"""--resumable, host side: the flag and its usage errors, the launch plans of the learners' graphs (unchanged by the flag), the readers'
state() / restore() round trips at the consumer's position, the state file (atomic write, the newest two kept, a stale .tmp ignored), its
mismatch checks, and the epoch loop continued from a state file with the GPU parts stubbed."""
import os
import sys

import pytest
import torch

import plan_digest
from chairs_tree import make_chairs_tree
from flow_trees import make_tree, reader as tree_reader, write_flows
from unsupervised_detection_b200 import resume_flags, train_state
from unsupervised_detection_b200.common_flags import FLAG_NAMES, FLAGS, Config
from unsupervised_detection_b200.data.synthetic import SyntheticReader
from unsupervised_detection_b200.engine import ParamStore
from unsupervised_detection_b200.models import adversarial_learner as AL, flow_learner as FL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _cfg(**kw):
    c = Config()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


# ------------------------------------------------------------------------------------------------ the flag
def test_flag_is_defined_once_outside_the_reference_surface_and_dumped(monkeypatch, tmp_path, capsys):
    import pretrain_recover
    import train
    import train_flow
    assert len(FLAG_NAMES) == 31 and 'resumable' not in FLAG_NAMES and FLAGS['resumable'].default is False
    monkeypatch.setattr(AL.AdversarialLearner, 'train', lambda self, config: None)
    monkeypatch.setattr(AL.AdversarialLearner, 'pretrain_recover', lambda self, config: None)
    monkeypatch.setattr(FL.FlowLearner, 'train_flow', lambda self, config: None)
    for mod in (train, pretrain_recover, train_flow):
        cfg = _cfg(checkpoint_dir=str(tmp_path), resumable=True, flow_dir='', ema_decay=0.0, box_min=0.1, box_max=0.5, pretrain_flow='pwc',
                   validate=False, flow_loss='multiscale', smooth_weight=3.0, learning_rate=1e-4, lr_boundaries=[], weight_decay=4e-4,
                   flow_aug=False)
        mod.run(cfg)
        assert "'resumable': True" in capsys.readouterr().out, mod.__name__


def test_usage_errors(monkeypatch, tmp_path):
    import pretrain_recover
    import train
    import train_flow
    args = ['--dataset=FLYINGCHAIRS', '--root_dir=%s' % tmp_path, '--resumable']
    seen = []
    try:
        for mod in (train, pretrain_recover, train_flow):
            monkeypatch.setattr(mod, 'run', lambda config: seen.append(config.resumable))
            FLAGS.unparse_flags()
            mod.main(['x', '--checkpoint_dir=%s' % tmp_path] + args)
            FLAGS.unparse_flags()
            with pytest.raises(SystemExit, match='checkpoint_dir'):
                mod.main(['x'] + args)
            FLAGS.unparse_flags()
            with pytest.raises(SystemExit, match='resume_train'):
                mod.main(['x', '--checkpoint_dir=%s' % tmp_path, '--resume_train'] + args)

            def mismatch(config):
                raise resume_flags.StateMismatch('--resumable: f was written with --batch_size=4, this run has --batch_size=8')
            monkeypatch.setattr(mod, 'run', mismatch)
            FLAGS.unparse_flags()
            with pytest.raises(SystemExit, match='--batch_size=4, this run has --batch_size=8'):
                mod.main(['x', '--checkpoint_dir=%s' % tmp_path] + args)
    finally:
        FLAGS.unparse_flags()
    assert seen == [True] * 3
    resume_flags.check(_cfg())                           # off: nothing to check


def _state(**kw):
    st = dict(format=train_state.FORMAT, kind='flow', epoch=1, world=1, flags=train_state.trajectory(_cfg()), frozen_crc=None)
    st.update(kw)
    return st


def test_mismatch_checks_name_the_flag_and_both_values():
    flags = train_state.trajectory(_cfg())
    train_state.check(_state(), 'f', 'flow', 1, flags, None)
    with pytest.raises(resume_flags.StateMismatch, match='written by train_flow.py, not train.py'):
        train_state.check(_state(), 'f', 'adversarial', 1, flags, None)
    with pytest.raises(resume_flags.StateMismatch, match='written by 1 ranks, this run has 2'):
        train_state.check(_state(), 'f', 'flow', 2, flags, None)
    for name, v in (('batch_size', 8), ('img_width', 512), ('beta1', 0.5), ('dataset', 'FBMS'), ('train_crop', 1.0)):
        other = train_state.trajectory(_cfg(**{name: v}))
        with pytest.raises(resume_flags.StateMismatch, match='--%s=%r, this run has --%s=%r' % (name, FLAGS[name].default, name, v)):
            train_state.check(_state(), 'f', 'flow', 1, other, None)
    other = train_state.trajectory(_cfg(lr_boundaries=['10']))
    with pytest.raises(resume_flags.StateMismatch, match='lr_boundaries'):
        train_state.check(_state(flags=train_state.trajectory(_cfg(lr_boundaries=[]))), 'f', 'flow', 1, other, None)
    other = train_state.trajectory(_cfg(flow_dir='/some/dir'))
    assert other['flow_dir'] is True
    with pytest.raises(resume_flags.StateMismatch, match='flow_dir'):
        train_state.check(_state(), 'f', 'flow', 1, other, None)
    with pytest.raises(resume_flags.StateMismatch, match='other PWC-Net parameters'):
        train_state.check(_state(kind='adversarial', frozen_crc=1234), 'f', 'adversarial', 1, flags, 5678)
    # flags that may change when a run is continued
    same = train_state.trajectory(_cfg(max_epochs=99, root_dir='/x', num_threads=1, summary_freq=7, save_freq=3))
    assert same == flags


# ------------------------------------------------------------------------------------------------ the state file
def test_state_file_is_written_atomically_and_the_newest_two_are_kept(tmp_path):
    d = str(tmp_path)
    assert train_state.newest(d) is None and train_state.newest(str(tmp_path / 'missing')) is None
    open(os.path.join(d, 'train_state-7.pt.tmp'), 'wb').write(b'an interrupted write')
    assert train_state.newest(d) is None                # a stale .tmp is not a state
    for e in (1, 2, 3):
        p = train_state.write(d, _state(epoch=e, t=torch.arange(e)))
        assert p == os.path.join(d, 'train_state-%d.pt' % e)
    assert sorted(os.listdir(d)) == ['train_state-2.pt', 'train_state-3.pt']     # the .tmp is removed, the newest two stay
    st = train_state.load(train_state.newest(d))
    assert st['epoch'] == 3 and torch.equal(st['t'], torch.arange(3))
    train_state.write(d, _state(epoch=10))              # numeric, not lexical, order
    assert train_state.epochs(d) == [3, 10]
    torch.save(_state(format=99), os.path.join(d, 'train_state-11.pt'))
    with pytest.raises(resume_flags.StateMismatch, match='format 99'):
        train_state.load(train_state.newest(d))


# ------------------------------------------------------------------------------------------------ readers
def _same_batches(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert len(x) == len(y)
        for u, v in zip(x, y):
            assert (torch.equal(u, v) if torch.is_tensor(u) else u == v)


def _round_trip(make, B, skip, n):
    """Stream A: `skip` batches, state(), then n batches.  Stream B: a fresh iterator restored to that state, n batches.  Equal."""
    a = make()
    for _ in range(skip):
        a.batch(B, pinned=False)
    st = a.state()
    want = [a.batch(B, pinned=False) for _ in range(n)]
    b = make()
    b.batch(B, pinned=False)                            # an iterator that has moved on (and started its producer) restores too
    b.restore(st)
    got = [b.batch(B, pinned=False) for _ in range(n)]
    for it in (a, b):
        getattr(it, 'close', lambda: None)()
    _same_batches(want, got)
    return want


@pytest.mark.parametrize('prefetch', [0, 3])
@pytest.mark.parametrize('dataset', ['DAVIS2016', 'FBMS', 'SEGTRACK'])
def test_mask_reader_round_trip(tmp_path, dataset, prefetch):
    root = make_tree(dataset, str(tmp_path / 'tree'))

    def train_it():
        rd = tree_reader(dataset, root)
        rd.prefetch = prefetch
        return rd.image_inputs(partition='train', train_crop=0.8)
    n = len(train_it().pairs)
    got = _round_trip(train_it, 5, 1, -(-2 * n // 5) + 1)        # two passes and more: the reshuffles at the end of the pair list
    assert len({nm for b in got for nm in b[3]}) > 1

    def val_it():
        rd = tree_reader(dataset, root)
        rd.prefetch = prefetch
        return rd.test_inputs(batch_size=2, partition='val').shard(0, 1, 2)
    _round_trip(val_it, 2, 1, len(val_it().pairs) + 1)           # the ordered validation reader wraps at the end of its list


@pytest.mark.parametrize('prefetch', [0, 2])
def test_reader_round_trip_with_supplied_flow(tmp_path, prefetch):
    root = make_tree('DAVIS2016', str(tmp_path / 'tree'))
    fdir = tmp_path / 'flo'
    write_flows(tree_reader('DAVIS2016', root), fdir, tree_reader('DAVIS2016', root).train_frame_pairs('train'))

    def train_it():
        rd = tree_reader('DAVIS2016', root, flow_dir=str(fdir))
        rd.prefetch = prefetch
        return rd.image_inputs(partition='train', train_crop=0.8)
    got = _round_trip(train_it, 4, 2, 8)
    assert len(got[0]) == 5 and got[0][4].shape == (4, 384, 640, 2)


@pytest.mark.parametrize('prefetch', [0, 2])
def test_flying_chairs_round_trip(tmp_path, prefetch):
    from unsupervised_detection_b200.data.flyingchairs_data_utils import FlyingChairsReader
    root = make_chairs_tree(str(tmp_path / 'chairs'), n=5)

    def train_it():
        rd = FlyingChairsReader(root, num_threads=2, seed=5)
        rd.prefetch = prefetch
        return rd.image_inputs(batch_size=2, train_crop=0.8)
    _round_trip(train_it, 2, 1, 6)                      # 5 pairs: 12 samples from position 2 cross two reshuffles


def test_state_is_the_consumers_position_with_prefetch(tmp_path):
    root = make_tree('DAVIS2016', str(tmp_path / 'tree'))
    its = []
    for p in (0, 3):
        rd = tree_reader('DAVIS2016', root)
        rd.prefetch, rd.num_threads = p, 3
        its.append(rd.image_inputs(partition='train'))
    for k in range(6):
        assert its[0].state() == its[1].state(), k     # the producer of the second one has drawn up to 3 batches further
        _same_batches([its[0].batch(3, pinned=False)], [its[1].batch(3, pinned=False)])
    its[1].close()


def test_synthetic_reader_round_trip():
    _round_trip(lambda: SyntheticReader(32, 48, seed=11), 2, 2, 3)


# ------------------------------------------------------------------------------------------------ launch plans with the flag off
def _cpu_graphs(monkeypatch):
    """The learners build their graphs on the CPU, PWC-Net at a small size, so that plan_digest can read them."""
    def init_dist(self):
        self.world, self.rank, self.local_rank, self.device = 1, 0, 0, 'cpu'
    monkeypatch.setattr(AL.AdversarialLearner, '_init_dist', init_dist)
    cis = AL.CISGraph
    monkeypatch.setattr(AL, 'CISGraph', lambda *a, **kw: cis(*a, pwc_hw=(128, 192), **kw))


def _plans(g):
    return dict(plan_digest.graph_plans(g)) if hasattr(g, 'gen_store') else {p: getattr(g, p) for p in ('aug', 'fwd', 'bwd', 'adam', 'pack')}


@pytest.mark.parametrize('kind', ['adversarial', 'pretrain_recover', 'flow'])
def test_learner_plans_are_unchanged_and_nothing_is_read_without_a_state(monkeypatch, tmp_path, kind):
    _cpu_graphs(monkeypatch)
    kw = dict(img_height=64, img_width=96, batch_size=1, dataset='SYNTHETIC', flow_ckpt='synthetic', ema_decay=0.0, flow_dir='')
    if kind == 'flow':
        kw.update(img_height=128, img_width=128, dataset='FLYINGCHAIRS', root_dir=make_chairs_tree(str(tmp_path / 'chairs'), n=2),
                  flow_ckpt='', flow_aug=True)
    digests = []
    with plan_digest.filled_uninitialized():
        for resumable in (False, True):
            L = (FL.FlowLearner if kind == 'flow' else AL.AdversarialLearner)()
            L.config, L._kind = _cfg(resumable=resumable, checkpoint_dir=str(tmp_path / 'ck'), **kw), kind
            getattr(L, {'adversarial': 'build_train_graph', 'pretrain_recover': 'build_pretrain_graph', 'flow': 'build_flow_graph'}[kind])()
            if resumable:
                assert L._resume() == (0, None)         # no state file: a fresh start, nothing loaded
            digests.append(plan_digest.digest(list(_plans(L.graph).items())))
    assert digests[0] == digests[1]
    assert not os.path.exists(str(tmp_path / 'ck'))


# ------------------------------------------------------------------------------------------------ the epoch loop, GPU parts stubbed
class _Reader(object):
    def __init__(self):
        self.n = 0

    def batch(self, b):
        self.n += 1
        return ('img1_%d' % self.n, 'img2_%d' % self.n, 'flow_%d' % self.n, [])

    def state(self):
        return self.n

    def restore(self, n):
        self.n = n


class _Graph(object):
    H, W, loss = 64, 128, 'multiscale'

    def __init__(self):
        from collections import namedtuple
        self.options = namedtuple('Options', 'search_range')(4)
        self.store = ParamStore('cpu')
        self.store.declare('pwcnet/w', (3,))
        self.store.finalize(True)
        self.step_state = torch.zeros(1, dtype=torch.int64)
        self.lr = []

    def set_lr(self, lr):
        self.lr.append(lr)


VALS = {3: 3.0, 6: 2.0, 9: 2.5, 12: 1.0, 15: 1.5}                # validation value after global step k: epoch 3 is worse than epoch 2


class _Stub(FL.FlowLearner):
    def build_flow_graph(self):
        self.rank, self.world, self.local_batch = 0, 1, 2
        self.reader, self.graph = _Reader(), _Graph()
        self.train_steps_per_epoch = 3
        self.calls, self.saved = [], []

    def flow_step(self, batch, next_batch=None, fetch_losses=False, use_graph=True):
        self.global_step += 1
        self.graph.store.flat += self.global_step       # stands in for an optimiser step
        self.graph.store.m += 1
        self.graph.step_state += 1
        self.calls.append((batch[0], next_batch[0], fetch_losses))
        r = {'global_step': self.global_step}
        if fetch_losses:
            r.update((k, float(self.global_step)) for k in FL.SUMMARY_KEYS['multiscale'])
        return r

    def save_flow(self, checkpoint_dir, epoch):
        self.saved.append(epoch)

    def validate_flow(self):
        return VALS[self.global_step]


def _loop(ck, max_epochs, resumable=True):
    L = _Stub()
    cfg = _cfg(dataset='FLYINGCHAIRS', max_epochs=max_epochs, save_freq=10, summary_freq=2, checkpoint_dir=str(ck), resumable=resumable,
               lr_boundaries=['5'])
    cfg.validate = True
    L.train_flow(cfg)
    return L


def test_resumed_loop_continues_after_the_saved_epoch(tmp_path, capsys):
    full = _loop(tmp_path / 'full', 4)
    assert train_state.epochs(str(tmp_path / 'full')) == [3, 4]
    capsys.readouterr()
    first = _loop(tmp_path / 'ck', 2)
    assert 'No training state in' in capsys.readouterr().out
    rest = _loop(tmp_path / 'ck', 4)
    out = capsys.readouterr().out
    assert 'Resumed training state from %s (epoch 2)' % train_state.path(str(tmp_path / 'ck'), 2) in out
    assert 'Epoch: [ 3] [    2/    3]' in out          # the step count carries on, and with it the summary steps
    assert first.calls + rest.calls == full.calls
    assert rest.calls[0][0] == 'img1_7'                 # the batch drawn before the epoch ended is trained on again
    assert full.saved == ['best', 'best', 4, 'best'] and first.saved == ['best', 2, 'best']     # the last epoch is always saved
    assert rest.saved == [4, 'best']                    # epoch 3 (2.5) is worse than epoch 2 (2.0): no best checkpoint
    assert rest.min_val_epe == full.min_val_epe == 1.0
    assert rest.global_step == 12 and rest.graph.lr == [1e-4 / 2]        # past --lr_boundaries=5 on resuming
    for a, b in ((full, rest),):
        assert torch.equal(a.graph.store.flat, b.graph.store.flat) and torch.equal(a.graph.store.m, b.graph.store.m)
        assert torch.equal(a.graph.step_state, b.graph.step_state)
    # a finished run returns without a step; a larger max_epochs extends it
    done = _loop(tmp_path / 'ck', 4)
    assert done.calls == [] and 'training is complete' in capsys.readouterr().out
    more = _loop(tmp_path / 'ck', 5)
    assert more.calls[0][0] == 'img1_13' and len(more.calls) == 3


def test_no_state_file_without_the_flag(tmp_path):
    L = _loop(tmp_path, 2, resumable=False)
    assert len(L.calls) == 6 and train_state.epochs(str(tmp_path)) == []
