"""--resumable end to end: each training script runs 2 epochs in one go, and again as 1 epoch that a new process continues to 2.  The two
runs end bit-identical: the final weights, Adam moments, moving averages and step counter (their state files), every printed loss and
validation line, and the best checkpoints.  A continuation that reads other PWC-Net parameters is a usage error.

The runs go through tests/probes/resume_worker.py in two processes: the first makes every uninterrupted run and every 1-epoch run, the
second every continuation, so each continuation starts from nothing but its files and the batch pays the start-up cost twice."""
import json
import os
import re
import socket
import subprocess
import sys

import pytest
import torch

from chairs_tree import make_chairs_tree
from flow_trees import make_davis_tree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


def _cases(chairs, davis):
    """{name: (script, args, best checkpoint or None)}"""
    small = ['--img_height=64', '--img_width=96', '--batch_size=2', '--save_freq=1', '--num_threads=2', '--resumable']
    flow = ['--img_height=128', '--img_width=128', '--batch_size=2', '--num_samples_train=4', '--summary_freq=1', '--save_freq=1',
            '--num_threads=2', '--validate', '--resumable']
    return {
        # 4 steps per epoch and a cycle of 1 recover + 2 generator steps: the epoch ends inside a cycle; summary steps every 2, the others
        # pipelined
        'cis': ('train.py', ['--dataset=SYNTHETIC', '--flow_ckpt=synthetic', '--num_samples_train=8', '--iters_rec=1', '--iters_gen=2',
                             '--ema_decay=0.999', '--summary_freq=2'] + small, 'model.best'),
        'boxes': ('pretrain_recover.py', ['--dataset=SYNTHETIC', '--flow_ckpt=synthetic', '--num_samples_train=6', '--summary_freq=1'] + small,
                  None),
        'chairs_gt': ('pretrain_recover.py', ['--dataset=FLYINGCHAIRS', '--root_dir=%s' % chairs, '--pretrain_flow=gt', '--validate',
                                              '--num_samples_train=4', '--summary_freq=1'] + small, 'recover-best'),
        # the rate halves after step 2, the last step of epoch 1: the continuation must set it
        'flow': ('train_flow.py', ['--dataset=FLYINGCHAIRS', '--root_dir=%s' % chairs, '--flow_aug', '--ema_decay=0.999',
                                   '--lr_boundaries=2'] + flow, 'pwcnet-best'),
        'unsup': ('train_flow.py', ['--dataset=DAVIS2016', '--root_dir=%s' % davis, '--flow_loss=unsupervised'] + flow, 'pwcnet-best'),
    }


def _worker(base, name, jobs):
    spec = base / (name + '.json')
    spec.write_text(json.dumps([[s, a, str(o)] for s, a, o in jobs]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'probes', 'resume_worker.py'), str(spec)],
                       env=dict(os.environ, PYTHONPATH=ROOT), cwd=str(base), capture_output=True, text=True, timeout=580)
    assert r.returncode == 0, r.stderr[-3000:]


@pytest.fixture(scope='module')
def runs(tmp_path_factory):
    base = tmp_path_factory.mktemp('resume')
    cases = _cases(make_chairs_tree(base / 'chairs', n=6, labels=[1, 1, 1, 1, 2, 2]), make_davis_tree(base / 'davis'))
    first, second = [], []
    for name, (script, args, _) in cases.items():
        d = base / name
        first += [(script, args + ['--max_epochs=2', '--checkpoint_dir=%s' % (d / 'full')], d.with_suffix('.full')),
                  (script, args + ['--max_epochs=1', '--checkpoint_dir=%s' % (d / 'ck')], d.with_suffix('.first'))]
        second.append((script, args + ['--max_epochs=2', '--checkpoint_dir=%s' % (d / 'ck')], d.with_suffix('.second')))
    _worker(base, 'first', first)
    # train.py continued with PWC-Net parameters that differ in one tensor from the ones it started with
    p = torch.load(str(base / 'cis' / 'full' / 'model-2.pt'))['params']
    pwc = {k: v for k, v in p.items() if k.startswith('pwcnet/')}
    k0 = sorted(pwc)[0]
    pwc[k0] = pwc[k0] + 1e-3
    torch.save({'params': pwc}, str(base / 'other_pwc.pt'))
    script, args, _ = cases['cis']
    args = ['--flow_ckpt=%s' % (base / 'other_pwc.pt') if a.startswith('--flow_ckpt') else a for a in args]
    second.append((script, args + ['--max_epochs=3', '--checkpoint_dir=%s' % (base / 'cis' / 'ck')], base / 'mismatch.out'))
    _worker(base, 'second', second)
    return base, {name: best for name, (_, _, best) in cases.items()}


def _lines(out):
    """The loss and validation lines, without their timing."""
    return [re.sub(r'time: \S+/it', '', ln) for ln in out.splitlines() if ln.startswith('Epoch')]


def _equal(a, b, where=''):
    if torch.is_tensor(a):
        assert torch.is_tensor(b) and a.dtype == b.dtype and torch.equal(a, b), where
    elif isinstance(a, dict):
        assert sorted(a) == sorted(b), where
        for k in a:
            _equal(a[k], b[k], '%s/%s' % (where, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, '%s[%d]' % (where, i))
    else:
        assert a == b, (where, a, b)


def _check(d, best):
    """The uninterrupted run in d/full and the interrupted one in d/ck ended alike -> the final state."""
    one, first, second = (d.with_suffix(s).read_text() for s in ('.full', '.first', '.second'))
    for out in (one, first, second):
        assert 'EXIT' not in out and 'completed successfully' in out, out[-2000:]
    assert 'No training state in' in first and 'Resumed training state from %s (epoch 1)' % (d / 'ck' / 'train_state-1.pt') in second
    assert _lines(one) and _lines(one) == _lines(first) + _lines(second)
    a, b = (torch.load(str(d / sub / 'train_state-2.pt'), weights_only=True) for sub in ('full', 'ck'))
    assert a['stores'] and int(a['step_state']) > 0
    _equal(a, b)
    if best:
        _equal(torch.load(str(d / 'full' / (best + '.pt')))['params'], torch.load(str(d / 'ck' / (best + '.pt')))['params'], best)
    return b


def test_train_py_pipelined_with_averages_and_a_mid_cycle_epoch_end(runs):
    base, best = runs
    st = _check(base / 'cis', best['cis'])
    assert st['step'] == 8 and st['global_step'] == 2 and st['frozen_crc'] is not None
    assert sorted(st['stores']) == ['FlownetS', 'MaskNet'] and 'shadow' in st['stores']['MaskNet']


def test_continuing_from_other_pwcnet_parameters_is_a_usage_error(runs):
    base, _ = runs
    out = (base / 'mismatch.out').read_text()
    assert 'EXIT --resumable:' in out and 'other PWC-Net parameters' in out, out[-2000:]
    assert not (base / 'cis' / 'ck' / 'train_state-3.pt').exists()


def test_pretrain_recover_on_boxes(runs):
    base, best = runs
    assert sorted(_check(base / 'boxes', best['boxes'])['stores']) == ['FlownetS']


def test_pretrain_recover_on_flying_chairs_ground_truth_with_validation(runs):
    base, best = runs
    _check(base / 'chairs_gt', best['chairs_gt'])


def test_train_flow_supervised_augmented_with_a_rate_boundary_at_the_epoch_end(runs):
    base, best = runs
    st = _check(base / 'flow', best['flow'])
    assert st['global_step'] == 4 and 'shadow' in st['stores']['pwcnet'] and st['frozen_crc'] is None


def test_train_flow_unsupervised_on_davis(runs):
    base, best = runs
    _check(base / 'unsup', best['unsup'])


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_train_flow_on_two_ranks(tmp_path):
    root = make_chairs_tree(tmp_path / 'chairs', n=10, labels=[1] * 8 + [2, 2])
    args = ['--dataset=FLYINGCHAIRS', '--root_dir=%s' % root, '--batch_size=4', '--num_samples_train=8', '--flow_aug', '--ema_decay=0.999',
            '--lr_boundaries=2', '--validate', '--img_height=128', '--img_width=128', '--summary_freq=1', '--save_freq=1', '--num_threads=2',
            '--resumable']
    outs = {}
    for name, epochs, sub in (('full', 2, 'full'), ('first', 1, 'ck'), ('second', 2, 'ck')):
        cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
               '--master-port', str(_free_port()), os.path.join(ROOT, 'train_flow.py')] + args + \
            ['--max_epochs=%d' % epochs, '--checkpoint_dir=%s' % (tmp_path / sub)]
        r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), cwd=str(tmp_path), capture_output=True, text=True, timeout=500)
        assert r.returncode == 0, r.stderr[-3000:]
        outs[name] = r.stdout
    assert 'Resumed training state from' in outs['second']
    assert _lines(outs['full']) and _lines(outs['full']) == _lines(outs['first']) + _lines(outs['second'])
    a, b = (torch.load(str(tmp_path / sub / 'train_state-2.pt'), weights_only=True) for sub in ('full', 'ck'))
    _equal(a, b)
    assert a['world'] == 2 and len(a['readers']) == 2 and a['readers'][0]['train'] != a['readers'][1]['train']
    _equal(torch.load(str(tmp_path / 'full' / 'pwcnet-best.pt'))['params'], torch.load(str(tmp_path / 'ck' / 'pwcnet-best.pt'))['params'])
