"""Moving average of the weights on the GPU: cis_ema_update bit for bit against its numpy fp32 restatement, its launches in the per-launch
harness, CIS training, recover pretraining and PWC-Net training with averaging on (live weights and losses unchanged, shadows equal to a
host recomputation, a validation pass on the shadows leaving training as it was), the three training scripts end to end, and two ranks."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import conv_launch_ref as R
import glue_launch_ref as G
import launch_suites as LS
import pwc_options_ref as REF
from oracle import params as OP
from unsupervised_detection_b200 import _lib
from unsupervised_detection_b200.flow_train_graph import FlowTrainGraph
from unsupervised_detection_b200.step_graph import CISGraph

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DECAY = 0.999


def ema_ref(shadow, param, decay, t):
    """cis_ema_update restated in numpy fp32 (numpy arrays in, the new shadow out): d = fp32(min(fp32 decay, (1 + t) / (10 + t)) in
    fp64), then shadow - (shadow - param) * (1 - d), each operation rounded to fp32."""
    d = np.float32(min(float(np.float32(decay)), (1.0 + t) / (10.0 + t)))
    k = np.float32(1.0) - d
    s = np.asarray(shadow, dtype=np.float32)
    return s - (s - np.asarray(param, dtype=np.float32)) * k


class EmaGlue(G.Glue):
    """glue_launch_ref's per-launch checker plus cis_ema_update: ema_ref from snapshots of shadow, param and the step read before the
    launch, bit-identical over [0, n); param and step_state unchanged; nothing outside the shadow written (the checker's stray-write
    test).  Negative control ema.t_off_by_one: the decay of step t + 1, made while it differs from step t's."""
    ARGS = 'shadow param n decay step_state'

    def _pre_ema_update(self, a):
        n = a['n']
        shadow, param = (self.mem.view(a[k], torch.float32, (n,)).clone() for k in ('shadow', 'param'))
        t = int(self.mem.view(a['step_state'], torch.int64, (1,)))
        s, p = shadow.cpu().numpy(), param.cpu().numpy()
        ctx = dict(ref=torch.from_numpy(ema_ref(s, p, a['decay'], t)), param=param, step=t, reads=[shadow, param],
                   dests=[(a['shadow'], torch.float32, 1, n, 0, n)])
        if self.controls is not None and ema_ref([1.0], [0.0], a['decay'], t)[0] != ema_ref([1.0], [0.0], a['decay'], t + 1)[0]:
            ctx['bad_t'] = torch.from_numpy(ema_ref(s, p, a['decay'], t + 1))
        return ctx

    def _post_ema_update(self, a, ctx):
        n = a['n']
        got = self.mem.view(a['shadow'], torch.float32, (n,)).cpu()
        self._rec('cis_ema_update', 'shadow', G.exact(got, ctx['ref']))
        self._rec('cis_ema_update', 'param unchanged', G.exact(self.mem.view(a['param'], torch.float32, (n,)), ctx['param']))
        step = int(self.mem.view(a['step_state'], torch.int64, (1,)))
        self._rec('cis_ema_update', 'step unchanged', 0.0 if step == ctx['step'] else float('inf'))
        if 'bad_t' in ctx:
            self._control('ema.t_off_by_one', G.exact(got, ctx['bad_t']))


def _st():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.detach().cpu().view(torch.int32)


# ------------------------------------------------------------------------------------------------ 1. the kernel
@pytest.mark.parametrize('n,t0,offset,decay', [(4096, 0, 0, DECAY),       # the num_updates warm-up: d = (1 + t) / (10 + t) < decay
                                               (1001, 0, 0, 0.9),         # odd n: a scalar tail after the float4 body
                                               (4103, 990, 0, DECAY),     # counter above 0: d reaches decay
                                               (999, 5, 1, 0.5)])         # 4-byte aligned only: the scalar path throughout
def test_ema_update_is_bit_identical_to_numpy(n, t0, offset, decay):
    gen = torch.Generator().manual_seed(n)
    base = torch.zeros(n + offset + 8, device='cuda')
    pbase = torch.zeros(n + offset + 8, device='cuda')
    shadow, param = base[offset:offset + n], pbase[offset:offset + n]
    s0 = torch.randn(n, generator=gen)
    s0[-3:] = 0.0                                                           # padding: zeros in both stay zero
    shadow.copy_(s0)
    step = torch.tensor([t0], dtype=torch.int64, device='cuda')
    ref = s0.numpy().copy()
    for k in range(20):
        p = torch.randn(n, generator=gen)
        p[-3:] = 0.0
        param.copy_(p)
        step += 1                                                           # what the optimiser launch does before the update
        _lib.call('cis_ema_update', shadow.data_ptr(), param.data_ptr(), n, decay, step.data_ptr(), _st())
        ref = ema_ref(ref, p.numpy(), decay, t0 + k + 1)
        assert torch.equal(_bits(shadow), torch.from_numpy(ref).view(torch.int32)), k
    assert not shadow[-3:].any() and not base[:offset].any() and not base[offset + n:].any()
    assert int(step) == t0 + 20


def test_ema_update_rejects_bad_arguments():
    s, p = torch.zeros(8, device='cuda'), torch.zeros(8, device='cuda')
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    good = [s.data_ptr(), p.data_ptr(), 8, 0.5, step.data_ptr()]
    for i, bad in ((0, None), (1, None), (4, None), (2, 0), (2, -1), (3, 0.0), (3, 1.0), (3, -0.5), (3, float('nan'))):
        args = list(good)
        args[i] = bad
        with pytest.raises(RuntimeError, match='cis_ema_update'):
            _lib.call('cis_ema_update', *args, _st())
    _lib.call('cis_ema_update', *good, _st())


# ------------------------------------------------------------------------------------------------ 2. the per-launch harness
def _walk_adam(monkeypatch, make, plans, prepare):
    """launch_suites.walk_plans over `plans` with EmaGlue as the glue checker (registered for this walk only)."""
    monkeypatch.setitem(G.ARGS, 'cis_ema_update', EmaGlue.ARGS)
    monkeypatch.setattr(G, 'Glue', EmaGlue)
    with R.recorded(pytest.MonkeyPatch()) as rec:
        g = make()
    prepare(g)
    return LS.walk_plans(rec, plans(g), controls=True, glue_controls=True)


def _noisy(stores, step_state, t):
    gen = torch.Generator().manual_seed(5)
    for st in stores:
        for _, _, n, off, _ in st.entries:
            st.grad[off:off + n] = 0.01 * torch.randn(n, generator=gen)
            st.shadow[off:off + n] += 0.01 * torch.randn(n, generator=gen).to(st.shadow.device)
    step_state.fill_(t)


@pytest.mark.parametrize('t', [0, 20000])
def test_every_ema_launch_of_the_optimiser_plans_is_checked(monkeypatch, t):
    def cis_prepare(g):
        g.load_params(OP.make_params(seed=4, jitter=0.1, nets=('MaskNet', 'FlownetS')))
        _noisy([g.gen_store, g.rec_store], g.step_state, t)
        g.avg_abs.fill_(1.0)
    r = _walk_adam(monkeypatch, lambda: CISGraph(64, 96, 1, with_pwc=False, ema_decay=DECAY),
                   lambda g: [('adam_G', g.adam['G']), ('adam_R', g.adam['R'])], cis_prepare)
    LS.assert_within_bounds(r)
    assert r['counts']['adam_G']['cis_ema_update'] == 1 and r['counts']['adam_R']['cis_ema_update'] == 1

    def flow_prepare(g):
        g.load_params(REF.make_params(3, jitter=0.1))
        _noisy([g.store], g.step_state, t)
    r2 = _walk_adam(monkeypatch, lambda: FlowTrainGraph(128, 192, 2, ema_decay=DECAY), lambda g: [('adam', g.adam)], flow_prepare)
    LS.assert_within_bounds(r2)
    assert r2['counts']['adam'] == {'cis_ema_update': 1, 'cis_adam_l2': 1}
    LS.report('ema t=%d' % t, r2['summary'], r2['controls'])
    if t == 0:          # the warm-up decay moves with t; at t = 20000 d = decay on both sides and the control is not made
        assert r['controls']['ema.t_off_by_one'] > 1 and r2['controls']['ema.t_off_by_one'] > 1


# ------------------------------------------------------------------------------------------------ 3. training with averaging on
class Shadows(object):
    """The host recomputation: every trained store's shadow from the live weights read after each step."""

    def __init__(self, stores):
        self.ref = {id(s): s.flat.cpu().numpy().copy() for s in stores}

    def step(self, store, t):
        self.ref[id(store)] = ema_ref(self.ref[id(store)], store.flat.cpu().numpy(), DECAY, t)
        assert torch.equal(_bits(store.shadow), torch.from_numpy(self.ref[id(store)]).view(torch.int32))


def _cis_batches(n, B, ph, pw):
    out = []
    for k in range(n):
        img1, img2, _ = LS.frames(B, ph, pw, 20 + k)
        out.append((img1.pin_memory(), img2.pin_memory()))
    return out


def _cis_run(masks, decay, validate_after=None):
    """Eight pipelined CUDA-graph steps, 1 recover : 3 generator (recover only for masks='boxes'), the learner's hand-over of each batch.
    -> (live params, losses per step, the graph).  validate_after=k: after step k a validation forward on the shadows of another batch."""
    B, H, W, ph, pw = 2, 64, 96, 128, 192
    g = CISGraph(H, W, B, with_pwc=True, pwc_hw=(ph, pw), masks=masks, ema_decay=decay)
    g.load_params(OP.make_params(seed=12, jitter=0.1))
    batches = _cis_batches(9, B, ph, pw)
    val = _cis_batches(1, B, ph, pw)[0]
    stores = [g.rec_store] + ([g.gen_store] if masks == 'generator' else [])
    host = Shadows(stores) if decay else None
    losses = []
    for k in range(8):
        mode = 'R' if masks == 'boxes' or k % 4 == 0 else 'G'
        if g.stage_for is not batches[k][0]:
            g.feed(*batches[k])
            g.prime_pipeline()
        ready = g.feed_next(*batches[k + 1])
        g.train_step(mode, use_graph=True, pipeline=True, inputs_ready=ready)
        g.pipeline_drain()
        losses.append(g.scalars[:4].tolist())
        if host is not None:
            host.step(g.store(mode), int(g.step_state))
        if validate_after == k:
            with g.averaged():
                g.feed(*val)
                g.forward()
                torch.cuda.synchronize()
                assert all(torch.equal(s.flat, s.shadow) for s in stores)
    torch.cuda.synchronize()
    live = {k: v.cpu() for k, v in g.export_params().items() if not k.endswith('/ExponentialMovingAverage')}
    return live, losses, g


def _same(a, b):
    assert a[1] == b[1]
    diff = [k for k in a[0] if not torch.equal(a[0][k], b[0][k])]
    assert not diff, diff[:5]


@pytest.mark.parametrize('masks', ['generator', 'boxes'])
def test_cis_training_is_unchanged_by_averaging_and_its_validation(masks):
    off = _cis_run(masks, 0.0)
    on = _cis_run(masks, DECAY)
    _same(off, on)
    assert any(not torch.equal(s.shadow, s.flat) for s in (on[2].rec_store,))
    _same(off, _cis_run(masks, DECAY, validate_after=4))
    if masks == 'boxes':
        assert on[2].gen_store.shadow is None


def _flow_run(loss, decay, validate_after=None):
    g = FlowTrainGraph(128, 128, 2, loss=loss, ema_decay=decay)
    g.load_params(REF.make_params(3, jitter=0.1))
    gen = torch.Generator().manual_seed(9)
    host = Shadows([g.store]) if decay else None
    losses = []
    for k in range(6):
        img1, img2, _ = LS.frames(2, 128, 128, 60 + k)
        g.feed(img1.cuda(), img2.cuda(), R.smooth(2, 128, 128, 2, 4.0, gen, div=24).cuda())
        g.train_step(use_graph=True)
        losses.append(g.losses())
        if host is not None:
            host.step(g.store, int(g.step_state))
        if validate_after == k:
            with g.averaged():
                g.forward()
                assert torch.equal(g.store.flat, g.store.shadow)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in g.store.export().items()}, losses, g


@pytest.mark.parametrize('loss', ['multiscale', 'unsupervised'])
def test_flow_training_is_unchanged_by_averaging_and_its_validation(loss):
    off = _flow_run(loss, 0.0)
    on = _flow_run(loss, DECAY)
    _same(off, on)
    assert not torch.equal(on[2].store.shadow, on[2].store.flat)
    _same(off, _flow_run(loss, DECAY, validate_after=2))


# ------------------------------------------------------------------------------------------------ 4. the scripts end to end
def _script(args, tmp_path):
    r = subprocess.run([sys.executable] + args, env=dict(os.environ, PYTHONPATH=ROOT), cwd=str(tmp_path), capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout


def _check_best(ck, epoch_base, best_base):
    """The epoch checkpoint holds every trained variable and its average (the two differ); the best one holds that epoch's averages under
    the plain names, in the .pt and in the bundle."""
    from unsupervised_detection_b200 import checkpoint as ckpt_io
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    ep = torch.load(str(ck / (epoch_base + '.pt')))['params']
    best = torch.load(str(ck / (best_base + '.pt')))['params']
    avg = sorted(k for k in ep if k.endswith('/ExponentialMovingAverage'))
    plain = [k[:-len('/ExponentialMovingAverage')] for k in avg]
    assert avg and all(p in ep for p in plain)
    assert any(not torch.equal(ep[p], ep[a]) for p, a in zip(plain, avg))
    got = AdversarialLearner._read_ckpt(str(ck / best_base), plain + avg)[0]
    for p, a in zip(plain, avg):
        assert torch.equal(best[p], ep[a]) and torch.equal(got[p].float(), ep[a]), p
    names = [v[0] for v in ckpt_io.list_variables(str(ck / epoch_base))]
    assert ckpt_io.to_tf_name(avg[0]) in names
    return plain


def test_scripts_write_averages_and_a_best_checkpoint_of_them(tmp_path):
    from chairs_tree import make_chairs_tree
    ema = '--ema_decay=%r' % DECAY
    # train.py: the validation IoU runs every epoch; model.best after the first one
    ck = tmp_path / 'cis'
    out = _script([os.path.join(ROOT, 'train.py'), '--dataset=SYNTHETIC', '--flow_ckpt=synthetic', '--img_height=64', '--img_width=96',
                   '--batch_size=2', '--num_samples_train=8', '--max_epochs=1', '--save_freq=1', '--summary_freq=100',
                   '--checkpoint_dir=%s' % ck, ema], tmp_path)
    assert 'Training completed successfully' in out and "'ema_decay': 0.999" in out
    plain = _check_best(ck, 'model-1', 'model.best')
    assert any(p.startswith('MaskNet/') for p in plain) and any(p.startswith('FlownetS/') for p in plain)
    assert not any(p.startswith('pwcnet/') for p in plain)
    out = _script([os.path.join(ROOT, 'test_generator.py'), '--dataset=SYNTHETIC', '--ckpt_file=%s' % (ck / 'model-1'), '--use_ema',
                   '--img_height=64', '--img_width=96', '--batch_size=2'], tmp_path)
    assert 'Success: Processed' in out
    # pretrain_recover.py and train_flow.py --validate on Flying Chairs with its split
    root = make_chairs_tree(tmp_path / 'chairs', n=4, labels=[1, 1, 2, 2])
    ck = tmp_path / 'rec'
    _script([os.path.join(ROOT, 'pretrain_recover.py'), '--dataset=FLYINGCHAIRS', '--root_dir=%s' % root, '--pretrain_flow=gt', '--validate',
             '--img_height=64', '--img_width=96', '--batch_size=2', '--num_samples_train=4', '--max_epochs=1', '--save_freq=1',
             '--num_threads=2', '--checkpoint_dir=%s' % ck, ema], tmp_path)
    assert all(p.startswith('FlownetS/') for p in _check_best(ck, 'recover-1', 'recover-best'))
    ck = tmp_path / 'flow'
    _script([os.path.join(ROOT, 'train_flow.py'), '--dataset=FLYINGCHAIRS', '--root_dir=%s' % root, '--validate', '--img_height=128',
             '--img_width=128', '--batch_size=2', '--num_samples_train=4', '--max_epochs=1', '--save_freq=1', '--num_threads=2',
             '--checkpoint_dir=%s' % ck, ema], tmp_path)
    assert all(p.startswith('pwcnet/') for p in _check_best(ck, 'pwcnet-1', 'pwcnet-best'))


# ------------------------------------------------------------------------------------------------ 5. two ranks
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_rank_nccl_training_keeps_identical_averages(tmp_path):
    GB, H, W, ph, pw = 4, 64, 96, 128, 192
    img1, img2, _ = LS.frames(GB, ph, pw, 31)
    torch.save(dict(GB=GB, H=H, W=W, ph=ph, pw=pw, img1=img1, img2=img2, params=OP.make_params(seed=12, jitter=0.1), modes='GGRG',
                    decay=DECAY), str(tmp_path / 'inputs.pt'))
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', str(_free_port()), os.path.join(ROOT, 'tests', 'probes', 'ema_dp_worker.py'), str(tmp_path)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=500)
    assert r.returncode == 0, r.stderr[-2000:]
    ranks = [torch.load(str(tmp_path / ('rank%d.pt' % i))) for i in range(2)]
    avg = [k for k in ranks[0] if k.endswith('/ExponentialMovingAverage')]
    assert avg and sorted(ranks[0]) == sorted(ranks[1])
    diff = [k for k in ranks[0] if not torch.equal(ranks[0][k], ranks[1][k])]
    assert not diff, diff[:5]
    assert np.mean([not torch.equal(ranks[0][k], ranks[0][k[:-len('/ExponentialMovingAverage')]]) for k in avg]) > 0.5
