"""Recover-net pretraining on ground-truth flow, on the GPU: cis_masked_epe against fp64 numpy, the flow_source='input' step against the
fp32 oracle, determinism and the pipelined schedule, the fixed validation pass, pretrain_recover.py on a tiny Flying Chairs tree end to
end, and 2 ranks against one GPU.

Run as a script (`torch.distributed.run ... tests/test_recover_pretrain_gt_gpu.py <dir> <chairs root>`) this file is the worker of the
2-rank test."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import losses as OL, params as OP  # noqa: E402
from unsupervised_detection_b200 import _lib  # noqa: E402
from unsupervised_detection_b200.step_graph import CISGraph, box_sides  # noqa: E402
from chairs_tree import make_chairs_tree  # noqa: E402
from test_parity_bench_sizes_gpu import smooth  # noqa: E402
from test_recover_pretrain_cpu import box_masks  # noqa: E402
from test_recover_pretrain_gpu import _free_port, _grad_check, _oracle_recover  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _st():
    return torch.cuda.current_stream().cuda_stream


def _epe_ref(pred, gt, m):
    e = np.sqrt(((pred.astype(np.float64) - gt.astype(np.float64)) ** 2).sum(-1))
    m = m.astype(np.float64)[..., 0]
    return np.stack([(m * e).sum((1, 2)), ((1 - m) * e).sum((1, 2)), m.sum((1, 2)), (1 - m).sum((1, 2))], 1)


@pytest.mark.parametrize('H,W', [(37, 53), (256, 448)])
@pytest.mark.parametrize('B', [1, 4, 7])
def test_masked_epe_matches_fp64_numpy_and_repeats_bit_for_bit(B, H, W):
    gen = torch.Generator().manual_seed(B * 1000 + H)
    pred, gt = torch.randn(B, H, W, 2, generator=gen).cuda(), torch.randn(B, H, W, 2, generator=gen).cuda()
    mask = torch.empty(B, H, W, 1, device='cuda')
    step = torch.full((1,), 3, dtype=torch.int64, device='cuda')
    _lib.call('cis_box_masks', mask.data_ptr(), B, H, W, *box_sides(0.1, 0.5, H, W), 5, step.data_ptr(), 8964, _st())
    scratch = torch.full((B * 256,), float('nan'), dtype=torch.float64, device='cuda')
    outs = []
    for _ in range(2):
        out = torch.full((B, 4), float('nan'), dtype=torch.float64, device='cuda')
        _lib.call('cis_masked_epe', pred.data_ptr(), gt.data_ptr(), mask.data_ptr(), B, H * W, scratch.data_ptr(), out.data_ptr(), _st())
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])
    ref = _epe_ref(pred.cpu().numpy(), gt.cpu().numpy(), mask.cpu().numpy())
    got = outs[0].numpy()
    assert np.all(np.abs(got - ref) <= 1e-12 * np.abs(ref)), np.abs(got - ref).max()
    assert np.array_equal(got[:, 2] + got[:, 3], np.full(B, float(H * W)))
    with pytest.raises(RuntimeError):
        _lib.call('cis_masked_epe', pred.data_ptr(), gt.data_ptr(), mask.data_ptr(), 0, H * W, scratch.data_ptr(), out.data_ptr(), _st())


# ------------------------------------------------------------------------------------------------ the step against the oracle
def test_gt_flow_pretrain_step_matches_the_oracle_64x96():
    # the inputs of test_recover_pretrain_gpu's oracle step, uploaded at twice the size: the legacy x2 downsample samples even pixels
    # exactly, so the staged path (resize, 1/flow_normalizer, hand-over) must give back that test's image and flow
    gen = torch.Generator().manual_seed(41)
    B, H, W, ph, pw = 2, 64, 96, 128, 192
    p = OP.make_params(seed=5, jitter=0.1, nets=('MaskNet', 'FlownetS'))
    up = lambda x: x.repeat_interleave(2, 1).repeat_interleave(2, 2).contiguous()
    img1 = up(torch.rand(B, H, W, 3, generator=gen) - 0.5)
    flow_full = up(smooth(B, H, W, 2, 0.3, gen) * 80.0)
    g = CISGraph(H, W, B, masks='boxes', flow_source='input', pwc_hw=(ph, pw))
    g.load_params(p)
    g.feed(img1, flow_full)
    pt = {k: v.clone() for k, v in p.items()}
    opt = OL.TFAdam()
    for t in range(3):
        g.forward()
        torch.cuda.synchronize()
        image, flow, m = g.image.cpu(), g.flow.cpu(), g.mask.cpu()
        if t == 0:
            # the same resize and normalisation as PWC-Net's output: legacy bilinear to HxW, / flow_normalizer
            from unsupervised_detection_b200.data.davis2016_data_utils import legacy_resize_numpy
            leg = np.stack([legacy_resize_numpy(flow_full[b].numpy(), H, W) for b in range(B)]) / np.float32(80.0)
            assert np.abs(flow.numpy() - leg).max() <= 1e-5 * np.abs(leg).max()
            assert np.abs(image.numpy() - np.stack([legacy_resize_numpy(img1[b].numpy(), H, W) for b in range(B)])).max() <= 1e-6
        assert torch.equal(m, box_masks(g.seed, t, 0, B, g.box, H, W))
        pr = {k: v.clone().requires_grad_(k.startswith('FlownetS/')) for k, v in pt.items()}
        L = _oracle_recover(image, flow, m, pr)
        ls = g.losses(full=True)
        assert abs(ls['recover'] - float(L['recover'])) <= 2e-3 * abs(float(L['recover'])), (ls['recover'], float(L['recover']))
        g.bwd['R'].run()
        torch.cuda.synchronize()
        names, grads = _grad_check(g, pr, L)
        clipped, _ = OL.clip_or_noise(list(grads), 0.2, can_change=False)
        opt.apply(pt, names, clipped)
        g.adam['R'].run()
        g.pack_rec.run()
        torch.cuda.synchronize()
        ex = g.export_params()
        worst = max(float((ex[n].cpu() - pt[n]).abs().max()) for n in names)
        mean = float(torch.cat([(ex[n].cpu() - pt[n]).abs().reshape(-1) for n in names]).mean())
        assert worst <= 2.5e-4 * (t + 1) and mean <= 1e-5 * (t + 2), (t, worst, mean)
    assert int(g.step_state.item()) == 3


def _batches(n, B, ph, pw, seed):
    gen = torch.Generator().manual_seed(seed)
    return [(smooth(B, ph, pw, 3, 0.25, gen).clamp(-0.5, 0.5).cuda(), smooth(B, ph, pw, 2, 20.0, gen).cuda()) for _ in range(n)]


def test_gt_flow_pretraining_is_deterministic_and_the_pipelined_schedule_bit_identical():
    B, H, W, ph, pw = 2, 64, 96, 128, 192
    p = OP.make_params(seed=9, jitter=0.1, nets=('MaskNet', 'FlownetS'))
    batches = _batches(9, B, ph, pw, 29)
    runs = []
    for pipelined in (False, False, True):
        g = CISGraph(H, W, B, pwc_hw=(ph, pw), masks='boxes', flow_source='input')
        g.load_params(p)
        losses = []
        if pipelined:
            g.img1.copy_(batches[0][0])
            g.flow_full.copy_(batches[0][1])
            g.prime_pipeline()
        for t in range(8):
            nxt = batches[t + 1] if pipelined else batches[t]
            if pipelined:
                torch.cuda.current_stream().wait_event(g.pipeline_inputs_free())
            g.img1.copy_(nxt[0])
            g.flow_full.copy_(nxt[1])
            ready = torch.cuda.Event()
            ready.record()
            g.train_step('R', use_graph=True, pipeline=pipelined, inputs_ready=ready)
            torch.cuda.synchronize()
            losses.append(g.losses())
            assert torch.equal(g.mask.cpu(), box_masks(g.seed, t, 0, B, g.box, H, W)), (pipelined, t)
        g.pipeline_drain()
        runs.append(({k: v.cpu() for k, v in g.export_params().items()}, losses))
    for other in runs[1:]:
        assert other[1] == runs[0][1]
        diff = [k for k in runs[0][0] if not torch.equal(runs[0][0][k], other[0][k])]
        assert not diff, diff[:5]
    assert any(not torch.equal(runs[0][0][k], p[k]) for k in p if k.startswith('FlownetS/'))


# ------------------------------------------------------------------------------------------------ validation and the CLI
def _chairs_learner(root, batch_size=2, pretrain_flow='gt'):
    from unsupervised_detection_b200.common_flags import Config
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    L = AdversarialLearner()
    L.config = Config(dataset='FLYINGCHAIRS', root_dir=root, img_height=64, img_width=96, batch_size=batch_size, num_threads=2,
                      flow_ckpt='synthetic')
    L.config.pretrain_flow = pretrain_flow
    L.build_pretrain_graph()
    return L


def test_validation_on_pwcnet_flow(tmp_path):
    """--validate with the default --pretrain_flow=pwc: the val graph runs PWC-Net on the val frame pairs (img1, img2) and scores the
    same boxes on every call; a training step on a Chairs batch moves the score."""
    root = make_chairs_tree(tmp_path, n=6, labels=[1, 1, 2, 2, 1, 2])
    L = _chairs_learner(root, pretrain_flow='pwc')
    assert L.graph.flow_source == 'pwc' and L.graph.with_pwc
    a = L.validate_recover()
    assert a == L.validate_recover() and all(math.isfinite(v) and v > 0 for v in a), a
    vg = L.val_graph
    assert vg.flow_source == 'pwc' and vg.sample_offset == 2
    it = L.dataset_reader.test_inputs()
    last = [it.batch(2) for _ in range(2)][-1]
    it.close()
    assert torch.equal(vg.img2.cpu(), last[1])                 # the second upload is frame 2, not the flow
    L.pretrain_step(L.reader.batch(2))
    torch.cuda.synchronize()
    assert L.validate_recover() != a


def test_validation_scores_fixed_boxes(tmp_path):
    root = make_chairs_tree(tmp_path, n=8, labels=[1, 1, 1, 2, 2, 2, 1, 2])
    L = _chairs_learner(root)
    a = L.validate_recover()
    b = L.validate_recover()
    assert a == b and all(math.isfinite(v) and v > 0 for v in a), (a, b)
    assert L.val_graph.sample_offset == 2 and int(L.val_graph.step_state.item()) == 0
    # the EPE restated on the host from the validation graph's own outputs, batch by batch
    vg, tot = L.val_graph, np.zeros(4)
    it = L.dataset_reader.test_inputs()
    for k in range(2):
        img1, _, flow, _ = it.batch(2)
        vg.set_sample_offset(2 * k)
        vg.feed(img1, flow)
        vg.forward()
        torch.cuda.synchronize()
        assert torch.equal(vg.mask.cpu(), box_masks(vg.seed, 0, 2 * k, 2, vg.box, 64, 96))
        tot += _epe_ref(vg.pred[:2].cpu().numpy(), vg.flow.cpu().numpy(), vg.mask.cpu().numpy()).sum(0)
    it.close()
    assert abs(tot[0] / tot[2] * 80.0 - a[0]) <= 1e-9 * a[0] and abs(tot[1] / tot[3] * 80.0 - a[1]) <= 1e-9 * a[1]
    L.pretrain_step(L.reader.batch(2))                 # new weights, new score
    torch.cuda.synchronize()
    assert L.validate_recover() != a


@pytest.mark.parametrize('flow', ['--pretrain_flow=gt', '--flow_ckpt=synthetic'])
def test_pretrain_recover_chairs_script_writes_best_and_train_loads_it(tmp_path, capsys, flow):
    root = make_chairs_tree(tmp_path / 'chairs', n=6, labels=[1, 1, 1, 1, 2, 2])
    ck = tmp_path / 'ck'
    cmd = [sys.executable, os.path.join(ROOT, 'pretrain_recover.py'), '--dataset=FLYINGCHAIRS', '--root_dir=%s' % root, flow,
           '--validate', '--img_height=64', '--img_width=96', '--batch_size=2', '--num_samples_train=4', '--max_epochs=2', '--save_freq=1',
           '--summary_freq=1', '--num_threads=2', '--checkpoint_dir=%s' % ck]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert 'Pretraining completed successfully' in r.stdout and r.stdout.count('Validation EPE (boxes)') == 2, r.stdout[-2000:]
    for base in ('recover-1', 'recover-2', 'recover-best'):
        for suf in ('.index', '.data-00000-of-00001', '.pt'):
            assert (ck / (base + suf)).is_file(), (base, suf)
    from unsupervised_detection_b200.common_flags import Config
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    from unsupervised_detection_b200.summary import read_events
    ev = [v for f in os.listdir(str(ck)) if f.startswith('events') for e in read_events(str(ck / f)) for v in e.get('values', [])]
    assert sum(v['tag'] == 'Validation EPE' for v in ev) == 2
    saved = torch.load(str(ck / 'recover-best.pt'))['params']
    for path in (str(ck / 'recover-best'), str(ck / 'recover-best.pt')):
        L = AdversarialLearner()
        L.config = Config(dataset='SYNTHETIC', flow_ckpt='synthetic', recover_ckpt=path, img_height=64, img_width=96, batch_size=2)
        L.build_train_graph()
        assert 'Recover net loaded from previous ckpt' in capsys.readouterr().out
        got = L.graph.rec_store.export()
        assert sorted(got) == sorted(saved) and all(torch.equal(got[k].cpu(), saved[k]) for k in saved)


# ------------------------------------------------------------------------------------------------ data parallelism
DP = dict(GB=4, steps=3)


def _run_dp(out, root):
    """3 steps on fixed global batches (each rank its slice), then validate_recover -> {params, epe} saved by rank 0 under `out`."""
    L = _chairs_learner(root, batch_size=DP['GB'])
    blob = torch.load(os.path.join(out, 'inputs.pt'))
    lb = L.local_batch
    sl = slice(L.rank * lb, (L.rank + 1) * lb)
    for img1, flow in blob['batches']:
        L.pretrain_step((img1[sl], None, flow[sl]), use_graph=True)
    epe = L.validate_recover()
    torch.cuda.synchronize()
    res = dict(params={k: v.cpu() for k, v in L.graph.rec_store.export().items()}, epe=epe)
    torch.save(res, os.path.join(out, 'world%d_rank%d.pt' % (L.world, L.rank)))
    return res


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_rank_gt_pretraining_and_validation_equal_one_gpu(tmp_path):
    root = make_chairs_tree(tmp_path / 'chairs', n=9, labels=[1, 1, 1, 1, 2, 2, 2, 2, 2])
    gen = torch.Generator().manual_seed(61)
    batches = [(smooth(DP['GB'], 384, 640, 3, 0.25, gen).clamp(-0.5, 0.5), smooth(DP['GB'], 384, 640, 2, 20.0, gen)) for _ in range(DP['steps'])]
    torch.save(dict(batches=batches), str(tmp_path / 'inputs.pt'))
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', str(_free_port()), os.path.abspath(__file__), str(tmp_path), root]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=500)
    assert r.returncode == 0, r.stderr[-2000:]
    ranks = [torch.load(str(tmp_path / ('world2_rank%d.pt' % i))) for i in range(2)]
    one = _run_dp(str(tmp_path), root)
    assert ranks[0]['epe'] == ranks[1]['epe']
    assert all(torch.equal(ranks[0]['params'][k], ranks[1]['params'][k]) for k in one['params'])
    for a, b in zip(one['epe'], ranks[0]['epe']):
        assert abs(a - b) <= 1e-4 * abs(a), (one['epe'], ranks[0]['epe'])
    worst = max(float((one['params'][k] - ranks[0]['params'][k]).abs().max()) for k in one['params'])
    assert worst <= 2.5e-4 * DP['steps'], worst


if __name__ == '__main__':
    _run_dp(sys.argv[1], sys.argv[2])
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()
