"""Recover-net pretraining on box-shaped occlusions, on the GPU: cis_box_masks against its Python restatement, the pretraining step against
the fp32 oracle (oracle.losses.loss_head + the oracle recover net, fed the kernel's masks), determinism and the pipelined schedule,
pretrain_recover.py end to end with its checkpoint read back by train.py's --recover_ckpt path, and 2-rank NCCL against one GPU.

Run as a script (`torch.distributed.run ... tests/test_recover_pretrain_gpu.py <dir>`) this file is the worker of the 2-rank test."""
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import losses as OL, nets as ON, params as OP  # noqa: E402
from unsupervised_detection_b200 import _lib  # noqa: E402
from unsupervised_detection_b200.step_graph import CISGraph, box_sides  # noqa: E402
from test_parity_bench_sizes_gpu import GRAD_TOL, VAR_TOL, smooth  # noqa: E402
from test_recover_pretrain_cpu import box_masks  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _st():
    return torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize('H,W', [(37, 53), (256, 448)])
@pytest.mark.parametrize('B', [1, 4, 7])
def test_box_kernel_matches_the_restatement_bit_for_bit(B, H, W):
    box = box_sides(0.1, 0.5, H, W)
    mask = torch.full((B, H, W, 1), -1.0, device='cuda')
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    prev = None
    for t in (0, 1, 2, 977, 2 ** 23 + 11):
        for off in (0, 3, 1000):
            step.fill_(t)
            _lib.call('cis_box_masks', mask.data_ptr(), B, H, W, *box, off, step.data_ptr(), 8964, _st())
            got = mask.cpu()
            ref = box_masks(8964, t, off, B, box, H, W)
            assert torch.equal(got, ref), (t, off, int((got != ref).sum()))
        if prev is not None:
            assert not torch.equal(got, prev)          # successive steps draw new boxes
        prev = got


def test_box_kernel_rejects_bad_sides():
    mask = torch.zeros(1, 8, 8, 1, device='cuda')
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    for box in ((0, 4, 1, 4), (3, 2, 1, 4), (1, 9, 1, 4), (1, 4, 1, 9)):
        with pytest.raises(RuntimeError):
            _lib.call('cis_box_masks', mask.data_ptr(), 1, 8, 8, *box, 0, step.data_ptr(), 1, _st())


# ------------------------------------------------------------------------------------------------ the step against the oracle
def _oracle_recover(image, flow, m, p):
    """adversarial_learner.py:107-172 with the mask m given: flow (x) (1-m), flow (x) m, the image-only prior -> loss_head dict."""
    pred = ON.recover_net(image, flow * (1.0 - m), m, p)
    pred_c = ON.recover_net(image, flow * m, 1.0 - m, p)
    pred_i = ON.recover_net(image, torch.zeros_like(flow), torch.ones_like(m), p)
    return OL.loss_head(flow, m, pred, pred_c, pred_i)


def _grad_check(g, pr, L):
    names = [n for n in pr if n.startswith('FlownetS/')]
    grads = torch.autograd.grad(L['recover'], [pr[n] for n in names])
    tot_ref = tot_err = bad_w = 0.0
    per = {}
    for n, gr in zip(names, grads):
        a, b = g.rec_store.view(n, 'grad').cpu().reshape(-1), gr.reshape(-1)
        e, r = float((a - b).norm()), float(b.norm())
        per[n] = (e / max(r, 1e-30), r)
        tot_ref += r * r
        tot_err += e * e
    for n, (rel, r) in per.items():
        if rel > VAR_TOL['R']:
            bad_w += r * r / tot_ref
    whole = (tot_err / tot_ref) ** 0.5
    assert whole <= GRAD_TOL['R'], whole
    assert bad_w <= 0.02, bad_w
    return names, grads


def test_pretrain_step_matches_the_oracle_64x96():
    gen = torch.Generator().manual_seed(41)
    B, H, W = 2, 64, 96
    p = OP.make_params(seed=5, jitter=0.1, nets=('MaskNet', 'FlownetS'))
    image = torch.rand(B, H, W, 3, generator=gen) - 0.5
    flow = smooth(B, H, W, 2, 0.3, gen)
    g = CISGraph(H, W, B, with_pwc=False, masks='boxes')
    g.load_params(p)
    g.image.copy_(image)
    g.flow.copy_(flow)
    pt = {k: v.clone() for k, v in p.items()}
    opt = OL.TFAdam()
    for t in range(3):
        g.forward()
        torch.cuda.synchronize()
        m = g.mask.cpu()
        assert torch.equal(m, box_masks(g.seed, t, 0, B, g.box, H, W))
        pr = {k: v.clone().requires_grad_(k.startswith('FlownetS/')) for k, v in pt.items()}
        L = _oracle_recover(image, flow, m, pr)
        ls = g.losses(full=True)
        assert abs(ls['recover'] - float(L['recover'])) <= 2e-3 * abs(float(L['recover'])), (ls['recover'], float(L['recover']))
        assert abs(ls['reconstruction_loss'] - float(L['rec'][0])) <= 2e-3 * max(1.0, float(L['rec'][0]))
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
        assert all(torch.equal(ex[n].cpu(), p[n]) for n in p if n.startswith('MaskNet/'))      # the generator is not trained
    assert int(g.step_state.item()) == 3


def test_pretrain_gradients_256x448_b4_with_pwcnet():
    gen = torch.Generator().manual_seed(43)
    B, H, W, ph, pw = 4, 256, 448, 384, 640
    p = OP.make_params(seed=6, jitter=0.1)
    g = CISGraph(H, W, B, with_pwc=True, masks='boxes')
    g.load_params(p)
    img1 = smooth(B, ph, pw, 3, 0.25, gen).clamp(-0.5, 0.5)
    g.img1.copy_(img1)
    g.img2.copy_(torch.roll(img1, shifts=(2, 3), dims=(1, 2)) + 0.01 * torch.randn(B, ph, pw, 3, generator=gen))
    g.step_state.fill_(5)
    g.forward()
    torch.cuda.synchronize()
    image, flow, m = g.image.cpu().clone(), g.flow.cpu().clone(), g.mask.cpu().clone()
    assert torch.equal(m, box_masks(g.seed, 5, 0, B, g.box, H, W))
    pr = {k: v.clone().requires_grad_(k.startswith('FlownetS/')) for k, v in p.items() if not k.startswith('pwcnet/')}
    L = _oracle_recover(image, flow, m, pr)
    assert abs(g.losses()['recover'] - float(L['recover'])) <= 2e-3 * abs(float(L['recover']))
    g.bwd['R'].run()
    torch.cuda.synchronize()
    _grad_check(g, pr, L)


def _batches(n, B, ph, pw, seed):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        a = smooth(B, ph, pw, 3, 0.25, gen).clamp(-0.5, 0.5)
        out.append((a.cuda(), (torch.roll(a, shifts=(1, 2), dims=(1, 2)) + 0.01 * torch.randn(B, ph, pw, 3, generator=gen)).cuda()))
    return out


def test_pretraining_is_deterministic_and_the_pipelined_schedule_bit_identical():
    """Two sequential 8-step runs end with bit-identical parameters; the pipelined schedule (PWC-Net of the next batch on a second stream,
    concurrent with this step's Adam update) gives the same parameters, losses and boxes -- the box kernel reads the Adam step counter
    after that update."""
    B, H, W, ph, pw = 2, 64, 96, 128, 192
    p = OP.make_params(seed=9, jitter=0.1)
    batches = _batches(9, B, ph, pw, 23)
    runs = []
    for pipelined in (False, False, True):
        g = CISGraph(H, W, B, with_pwc=True, pwc_hw=(ph, pw), masks='boxes')
        g.load_params(p)
        losses, masks = [], []
        if pipelined:
            g.img1.copy_(batches[0][0])
            g.img2.copy_(batches[0][1])
            g.prime_pipeline()
        for t in range(8):
            nxt = batches[t + 1] if pipelined else batches[t]
            if pipelined:
                torch.cuda.current_stream().wait_event(g.pipeline_inputs_free())
            g.img1.copy_(nxt[0])
            g.img2.copy_(nxt[1])
            ready = torch.cuda.Event()
            ready.record()
            g.train_step('R', use_graph=True, pipeline=pipelined, inputs_ready=ready)
            torch.cuda.synchronize()
            losses.append(g.losses())
            masks.append(g.mask.cpu())
            assert torch.equal(masks[-1], box_masks(g.seed, t, 0, B, g.box, H, W)), (pipelined, t)
        g.pipeline_drain()
        runs.append(({k: v.cpu() for k, v in g.export_params().items()}, losses))
    for other in runs[1:]:
        assert other[1] == runs[0][1]
        diff = [k for k in runs[0][0] if not torch.equal(runs[0][0][k], other[0][k])]
        assert not diff, diff[:5]
    assert any(not torch.equal(runs[0][0][k], p[k]) for k in p if k.startswith('FlownetS/'))


# ------------------------------------------------------------------------------------------------ CLI end to end
def test_pretrain_recover_script_writes_checkpoints_that_train_loads(tmp_path, capsys):
    ck = tmp_path / 'ck'
    env = dict(os.environ, PYTHONPATH=ROOT)
    cmd = [sys.executable, os.path.join(ROOT, 'pretrain_recover.py'), '--dataset=SYNTHETIC', '--flow_ckpt=synthetic', '--img_height=64',
           '--img_width=96', '--batch_size=2', '--num_samples_train=6', '--max_epochs=2', '--save_freq=1', '--summary_freq=2',
           '--checkpoint_dir=%s' % ck]
    r = subprocess.run(cmd, env=env, cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert 'Pretraining completed successfully' in r.stdout and r.stdout.count('loss_recover') == 3, r.stdout[-2000:]
    for n in (1, 2):
        for suf in ('.index', '.data-00000-of-00001', '.pt'):
            assert (ck / ('recover-%d%s' % (n, suf))).is_file(), (n, suf)
    from unsupervised_detection_b200.common_flags import Config
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    saved = torch.load(str(ck / 'recover-2.pt'))['params']
    for path in (str(ck / 'recover-2'), str(ck / 'recover-2.pt')):
        L = AdversarialLearner()
        L.config = Config(dataset='SYNTHETIC', flow_ckpt='synthetic', recover_ckpt=path, img_height=64, img_width=96, batch_size=2)
        L.build_train_graph()
        assert 'Recover net loaded from previous ckpt' in capsys.readouterr().out
        got = L.graph.rec_store.export()
        assert sorted(got) == sorted(saved)
        assert all(torch.equal(got[k].cpu(), saved[k]) for k in saved)
    first = torch.load(str(ck / 'recover-1.pt'))['params']
    assert any(not torch.equal(first[k], saved[k]) for k in saved)          # the second epoch moved the weights


# ------------------------------------------------------------------------------------------------ data parallelism
DP = dict(GB=4, H=64, W=96, ph=128, pw=192, steps=3)


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dp_worker(out):
    import torch.distributed as dist
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    blob = torch.load(os.path.join(out, 'inputs.pt'))
    b = DP['GB'] // world
    g = CISGraph(DP['H'], DP['W'], b, device='cuda:%d' % local, global_batch=DP['GB'], with_pwc=True, pwc_hw=(DP['ph'], DP['pw']),
                 masks='boxes', sample_offset=rank * b)
    g.load_params(blob['params'])
    sl = slice(rank * b, (rank + 1) * b)
    g.img1.copy_(blob['img1'][sl])
    g.img2.copy_(blob['img2'][sl])
    for _ in range(DP['steps']):
        g.train_step('R', allreduce=lambda t: dist.all_reduce(t), use_graph=True)
    torch.cuda.synchronize()
    res = {k: v.cpu() for k, v in g.rec_store.export().items()}
    res['__mask'] = g.mask.cpu()
    torch.save(res, os.path.join(out, 'rank%d.pt' % rank))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_rank_pretraining_equals_one_gpu_global_batch(tmp_path):
    gen = torch.Generator().manual_seed(47)
    GB, H, W, ph, pw = DP['GB'], DP['H'], DP['W'], DP['ph'], DP['pw']
    img1 = smooth(GB, ph, pw, 3, 0.25, gen).clamp(-0.5, 0.5)
    img2 = torch.roll(img1, shifts=(1, 2), dims=(1, 2)) + 0.01 * torch.randn(GB, ph, pw, 3, generator=gen)
    p = OP.make_params(seed=13, jitter=0.1)
    torch.save(dict(img1=img1, img2=img2, params=p), str(tmp_path / 'inputs.pt'))
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', str(_free_port()), os.path.abspath(__file__), str(tmp_path)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=500)
    assert r.returncode == 0, r.stderr[-2000:]
    ranks = [torch.load(str(tmp_path / ('rank%d.pt' % i))) for i in range(2)]
    g = CISGraph(H, W, GB, with_pwc=True, pwc_hw=(ph, pw), masks='boxes')
    g.load_params(p)
    g.img1.copy_(img1)
    g.img2.copy_(img2)
    for _ in range(DP['steps']):
        g.train_step('R', use_graph=True)
    torch.cuda.synchronize()
    assert torch.equal(torch.cat([ranks[0]['__mask'], ranks[1]['__mask']]), g.mask.cpu())   # the boxes of the global batch
    one = {k: v.cpu() for k, v in g.rec_store.export().items()}
    assert all(torch.equal(ranks[0][k], ranks[1][k]) for k in one)
    worst = max(float((one[k] - ranks[0][k]).abs().max()) for k in one)
    mean = float(torch.cat([(one[k] - ranks[0][k]).abs().reshape(-1) for k in one]).mean())
    moved = float(torch.cat([(one[k] - p[k]).abs().reshape(-1) for k in one]).mean())
    assert worst <= 2.5e-4 * DP['steps'] and mean <= 0.02 * moved, (worst, mean, moved)


if __name__ == '__main__':
    _dp_worker(sys.argv[1])
