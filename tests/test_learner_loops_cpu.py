"""The learners' host-side loops with the GPU parts stubbed: train_flow's epoch loop (batch hand-over, summaries, progress lines,
checkpoints and the keep-the-best validation), the sharded validation passes of validate_flow / validate_unsup / validate_recover
(padding pairs left out, the iterator closed, the feed arguments) and their one all-reduce per pass on two ranks."""
import re

import pytest
import torch
from collections import namedtuple

from unsupervised_detection_b200.common_flags import Config
from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
from unsupervised_detection_b200.models.flow_learner import SUMMARY_KEYS, FlowLearner
from unsupervised_detection_b200.summary import read_events

N, LB = 5, 2                                            # a 5-pair val split read at local batch 2: the last pair of batch 3 only pads


# ------------------------------------------------------------------------------------------------ train_flow's loop
class _Reader(object):
    def __init__(self):
        self.n = 0

    def batch(self, b):
        self.n += 1
        return ('img1_%d' % self.n, 'img2_%d' % self.n, 'flow_%d' % self.n, [])


class _Store(object):
    def real_count(self):
        return 99


class _FlowGraph(object):
    store, H, W = _Store(), 64, 128
    options = namedtuple('Options', 'search_range')(4)

    def __init__(self, loss):
        self.loss = loss


@pytest.mark.parametrize('dataset,loss,tag', [('FLYINGCHAIRS', 'multiscale', 'Validation EPE (flow)'),
                                              ('DAVIS2016', 'unsupervised', 'Validation unsupervised flow loss')])
def test_train_flow_loop(capsys, tmp_path, dataset, loss, tag):
    """Each batch is stepped once and in order with the next one handed over; the losses are fetched, printed and written every
    summary_freq steps; pwcnet-<epoch> is saved every save_freq epochs and after the last one, before that epoch's validation, and
    pwcnet-best whenever the validation value drops."""
    keys = SUMMARY_KEYS[loss]

    class Stub(FlowLearner):
        def build_flow_graph(self):
            self.rank, self.world, self.local_batch = 0, 1, 2
            self.reader, self.graph = _Reader(), _FlowGraph(loss)
            self.train_steps_per_epoch = 3
            self.calls, self.saved, self.vals = [], [], iter([3.0, 2.0, 2.5, 1.0])

        def flow_step(self, batch, next_batch=None, fetch_losses=False, use_graph=True):
            self.global_step += 1
            self.calls.append((batch[0], next_batch[0], fetch_losses))
            r = {'global_step': self.global_step}
            if fetch_losses:
                r.update((k, self.global_step + i * 0.125) for i, k in enumerate(keys))
            return r

        def save_flow(self, checkpoint_dir, epoch):
            self.saved.append((checkpoint_dir, epoch, len(self.calls)))

        def validate_flow(self):
            assert dataset == 'FLYINGCHAIRS'
            return next(self.vals)

        def validate_unsup(self):
            assert dataset == 'DAVIS2016'
            return next(self.vals)

    L = Stub()
    cfg = Config(dataset=dataset, max_epochs=4, save_freq=3, summary_freq=2, checkpoint_dir=str(tmp_path))
    cfg.validate = True
    L.train_flow(cfg)
    assert [c[0] for c in L.calls] == ['img1_%d' % i for i in range(1, 13)]          # 4 epochs x 3 steps, each batch once, in order
    assert [c[1] for c in L.calls] == ['img1_%d' % i for i in range(2, 14)]          # step k is given batch k+1 to prefetch
    assert [i + 1 for i, c in enumerate(L.calls) if c[2]] == [2, 4, 6, 8, 10, 12]
    ck = str(tmp_path)
    assert L.saved == [(ck, 'best', 3), (ck, 'best', 6), (ck, 3, 9), (ck, 4, 12), (ck, 'best', 12)]
    assert L.min_val_epe == 1.0
    out = re.sub(r'time: \S+/it', 'time: T/it', capsys.readouterr().out)
    assert out.splitlines() == [
        'Number of PWC-Net params: 99',
        '-------------------------------------',
        "Training PWC-Net (%s loss) on 64x128, options {'search_range': 4}" % loss,
        '-------------------------------------',
        'Epoch: [ 1] [    2/    3] time: T/it flow_loss 2.0000',
        'Epoch [1] %s: 3.0000' % tag,
        'Epoch: [ 2] [    1/    3] time: T/it flow_loss 4.0000',
        'Epoch: [ 2] [    3/    3] time: T/it flow_loss 6.0000',
        'Epoch [2] %s: 2.0000' % tag,
        'Epoch: [ 3] [    2/    3] time: T/it flow_loss 8.0000',
        'Epoch [3] %s: 2.5000' % tag,
        'Epoch: [ 4] [    1/    3] time: T/it flow_loss 10.0000',
        'Epoch: [ 4] [    3/    3] time: T/it flow_loss 12.0000',
        'Epoch [4] %s: 1.0000' % tag,
        '-------------------------------',
        'Training completed successfully',
        '-------------------------------']
    L.summary_writer.close()
    ev = [(e['step'], [(v['tag'], v['simple_value']) for v in e['values']]) for e in read_events(L.summary_writer.path)[1:]]
    losses = lambda s: (s, [(k, s + i * 0.125) for i, k in enumerate(keys)])
    val = lambda epoch, v: (epoch, [(tag, v)])
    assert ev == [losses(2), val(1, 3.0), losses(4), losses(6), val(2, 2.0), losses(8), val(3, 2.5), losses(10), losses(12), val(4, 1.0)]


# ------------------------------------------------------------------------------------------------ the sharded validation passes
def _batch(k):
    """Val batch k of the local batch: (img1, img2, flow) hold 10k + j at sample j, 10k + j + 0.25 and 10k + j + 0.5."""
    return tuple(torch.arange(LB, dtype=torch.float32).view(LB, 1) + 10 * k + d for d in (0.0, 0.25, 0.5)) + (['n%d' % k] * LB,)


class _It(object):
    """test_inputs of the val split, sharded: rank r's batch k is its slice of global batch k."""

    def __init__(self, kw):
        self.kw, self.k, self.closed, self.sharded = kw, 0, False, None

    def shard(self, rank, world, gb):
        self.sharded = (rank, world, gb)
        return self

    def batch(self, b):
        assert b == LB
        rank, world, gb = self.sharded
        self.k += 1
        return _batch((self.k - 1) * world + rank)

    def close(self):
        self.closed = True


class _ValReader(object):
    def test_inputs(self, **kw):
        self.it = _It(kw)
        return self.it


def _pair(x):
    """Global val index of the sample that carries x (_batch: 10k + j at sample j of local batch k)."""
    return int(x) // 10 * LB + int(x) % 10


class _ValGraph(object):
    """FlowTrainGraph / CISGraph's validation surface: per-sample sums that name the pair they come from."""
    box, flow_source = (1, 2, 3, 4), 'pwc'

    def __init__(self):
        self.fed, self.offsets, self.summed = [], [], 0

    def feed(self, *args):
        self.fed.append(tuple(float(a[0, 0]) for a in args))
        self.rows = [float(v) for v in args[0][:, 0]]

    def forward(self):
        pass

    def epe(self):                                      # per sample {sum e, 0, pixels, 0}
        self.summed += 1
        return torch.tensor([[_pair(v) + 1.0, 0.0, 2.0, 0.0] for v in self.rows], dtype=torch.float64)

    def masked_epe(self):                               # per sample {m*e, (1-m)*e, m, 1-m}
        self.summed += 1
        return torch.tensor([[_pair(v) + 1.0, 1.0, 2.0, 4.0] for v in self.rows], dtype=torch.float64)

    def direction_objective(self):                      # 2B directions: pair n forward, then pair n backward
        self.summed += 1
        return torch.tensor([_pair(v) + 1.0 for v in self.rows] + [100.0 * (_pair(v) + 1.0) for v in self.rows], dtype=torch.float64)

    def set_sample_offset(self, off):
        self.offsets.append(off)

    def load_params(self, p):
        pass

    def export_params(self):
        return {}


def _learner(rank=0, world=1, cls=FlowLearner):
    L = cls()
    L.config = Config(dataset='FLYINGCHAIRS', batch_size=LB * world, test_temporal_shift=-2, test_crop=0.9, flow_normalizer=80.0)
    L.rank, L.world, L.local_batch, L.num_samples_val = rank, world, LB, N
    L.dataset_reader, L.graph, L.val_graph = _ValReader(), _ValGraph(), _ValGraph()
    return L


def test_validate_flow_leaves_out_the_padding_pair():
    L = _learner()
    epe = L.validate_flow()
    it, g = L.dataset_reader.it, L.graph
    assert it.kw == {'batch_size': LB} and it.sharded == (0, 1, LB) and it.closed
    assert g.fed == [(10.0 * k, 10.0 * k + 0.25, 10.0 * k + 0.5) for k in range(3)]      # (img1, img2, ground-truth flow)
    assert epe == (1 + 2 + 3 + 4 + 5) / 10.0                                             # pair 6 of batch 3 only pads


def test_validate_unsup_counts_both_directions_of_the_real_pairs():
    L = _learner()
    L.config.dataset = 'DAVIS2016'
    obj = L.validate_unsup()
    it, g = L.dataset_reader.it, L.graph
    assert it.kw == {'batch_size': LB, 't_len': -2, 'test_crop': 0.9, 'partition': 'val'} and it.sharded == (0, 1, LB) and it.closed
    assert g.fed == [(10.0 * k, 10.0 * k + 0.25) for k in range(3)]                      # the frames only
    assert obj == 101.0 * (1 + 2 + 3 + 4 + 5) / N                                         # forward + backward half, per real pair


def _all_reduces(monkeypatch):
    """Makes the learner see an initialised process group whose all-reduce records a copy of each tensor and leaves it as it is."""
    import torch.distributed as dist
    seen = []
    monkeypatch.setattr(dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(dist, 'all_reduce', lambda t: seen.append(t.clone()))
    return seen


@pytest.mark.parametrize('which', ['validate_flow', 'validate_unsup', 'validate_recover'])
def test_each_validation_pass_makes_one_all_reduce_on_two_ranks(monkeypatch, which):
    """Two ranks x local batch 2 over the 5 pairs: rank 0 reads pairs 1-2 and 5 (+ a padding pair), rank 1 pairs 3-4 and then only
    padding, which it runs but does not score.  Each rank all-reduces once; the two ranks' first sums add up to the whole split's."""
    seen = _all_reduces(monkeypatch)
    firsts = []
    for rank in (0, 1):
        L = _learner(rank, world=2, cls=AdversarialLearner if which == 'validate_recover' else FlowLearner)
        L.config.dataset = 'DAVIS2016' if which == 'validate_unsup' else 'FLYINGCHAIRS'
        getattr(L, which)()
        g = L.val_graph if which == 'validate_recover' else L.graph
        assert L.dataset_reader.it.sharded == (rank, 2, 2 * LB) and L.dataset_reader.it.closed
        assert len(g.fed) == 2 and g.summed == 2 - rank
        if which == 'validate_recover':
            assert g.offsets == [rank * LB, 2 * LB + rank * LB]
        assert len(seen) == rank + 1
        firsts.append(float(seen[-1][0]))
    assert sum(firsts) == (101.0 if which == 'validate_unsup' else 1.0) * (1 + 2 + 3 + 4 + 5)


def test_validation_iou_makes_one_all_reduce_on_two_ranks(monkeypatch):
    seen = _all_reduces(monkeypatch)
    gt = torch.zeros(LB, 16, 24, 1)
    gt[:, 4:12, 6:18] = 1.0

    class Graph(object):
        def forward(self):
            self.mask = torch.zeros(LB, 8, 12, 1)
            self.mask[:, 2:6, 3:9] = 0.9

    class Reader(object):
        def batch(self, b):
            return torch.zeros(b, 4, 4, 3), torch.zeros(b, 4, 4, 3), gt, ['a'] * b

    class Stub(AdversarialLearner):
        def feed(self, img1, img2):
            pass

        def save(self, sess, checkpoint_dir, step):
            self.saved.append(step)

    L = Stub()
    L.rank, L.world, L.local_batch, L.saved = 0, 2, LB, []
    L.config = Config(batch_size=2 * LB, save_freq=1)
    L.graph, L.val_reader, L.val_steps_per_epoch, L.min_val_iou = Graph(), Reader(), 3, -1.0e12
    L.epoch_end_callback(None, None, 1)
    assert len(seen) == 1 and abs(float(seen[0][0]) - 3 * LB) < 1e-5
    assert L.saved == ['best', 1] and abs(L.min_val_iou - 0.5) < 1e-6        # this rank's IoU sum over the global batch count
