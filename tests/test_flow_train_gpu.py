"""PWC-Net training on the GPU: the multi-scale loss kernels against the fp64 restatement (tests/flow_loss_ref.py), the gradient of a
whole step against fp64 autograd through the oracle, one cis_adam_l2 update, determinism and CUDA-graph replay, learning on a fixed
batch, train_flow.py end to end, and 2 ranks against one GPU.

Run as a script (`torch.distributed.run ... tests/test_flow_train_gpu.py <dir>`) this file is the worker of the 2-rank test."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import flow_loss_ref as FR  # noqa: E402
import pwc_options_ref as PO  # noqa: E402
from chairs_tree import make_chairs_tree, pattern, shifted  # noqa: E402
from unsupervised_detection_b200 import _lib  # noqa: E402
from unsupervised_detection_b200.flow_train_graph import ALPHAS, LEVELS, FlowTrainGraph  # noqa: E402
from unsupervised_detection_b200.params_init import init_pwcnet  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
NONDENSE = {'use_dense_cx': False, 'use_res_cx': False, 'search_range': 2}


def _st():
    return torch.cuda.current_stream().cuda_stream


def _smooth(B, H, W, C, amp, gen):
    lo = torch.randn(B, C, max(2, H // 16), max(2, W // 16), generator=gen)
    return (torch.nn.functional.interpolate(lo, size=(H, W), mode='bicubic', align_corners=False) * amp).permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------ 1. the loss kernels
@pytest.mark.parametrize('robust', [False, True])
# 64x128: level 6 is 1x2 and its target the legacy resize of 64 rows to 1 (the kernels take it; the graph needs 128, for the warp)
@pytest.mark.parametrize('H,W,gh,gw', [(384, 640, 384, 640), (64, 128, 64, 128), (128, 192, 128, 192), (128, 128, 384, 640)])
def test_loss_forward_and_backward_match_fp64(robust, H, W, gh, gw):
    B = 3
    gen = torch.Generator().manual_seed(H + W + robust)
    gt = _smooth(B, gh, gw, 2, 8.0, gen)
    gt[2] = 0.0                                                  # sample 2: ground truth 0 ...
    s0, s1 = H / gh, W / gw
    flows = []
    for l in LEVELS:
        g = FR.level_target(gt.double(), H >> l, W >> l, l, s0, s1).float()
        f = g + torch.randn(g.shape, generator=gen) * 0.5
        f[2] = 0.0                                               # ... and its flows 0: every difference is exactly 0
        flows.append(f.cuda().contiguous())
    pyr = _lib.CisFlowPyr()
    grads = []
    for i, l in enumerate(LEVELS):
        pitch, coff = (16, 2) if i == 1 else (8, 0)             # one level in a wider buffer at an offset
        gb = torch.zeros(B, H >> l, W >> l, pitch, dtype=torch.bfloat16, device='cuda')
        grads.append((gb, coff))
        pyr.flow[i], pyr.grad[i], pyr.pitch[i], pyr.c_off[i], pyr.accumulate[i] = flows[i].data_ptr(), gb.data_ptr(), pitch, coff, 0
        pyr.weight[i] = ALPHAS[i] / 4
    gtc = gt.cuda()
    args = (gtc.data_ptr(), B, H, W, gh, gw, s0, s1, int(robust), 0.01, 0.4)
    scratch = torch.full((5 * B * 64,), float('nan'), dtype=torch.float64, device='cuda')
    outs = []
    for _ in range(2):
        out = torch.full((B, 5), float('nan'), dtype=torch.float64, device='cuda')
        _lib.call('cis_flow_multiscale_loss', pyr, *args, scratch.data_ptr(), out.data_ptr(), _st())
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])
    with pytest.raises(RuntimeError, match='alignment'):          # gt is read as float pairs: 8-byte alignment is checked
        _lib.call('cis_flow_multiscale_loss', pyr, gtc.data_ptr() + 4, *args[1:], scratch.data_ptr(), out.data_ptr(), _st())
    fd = [f.cpu().double().requires_grad_(True) for f in flows]
    ref = FR.level_sums(fd, gt.double(), robust=robust, s0=s0, s1=s1)
    rel = ((outs[0] - ref.detach()).abs() / ref.detach().abs().clamp_min(1e-300))
    if not robust:
        assert torch.equal(outs[0][2], torch.zeros(5, dtype=torch.float64))
        rel[2] = 0
    print('MEASURED flow loss fwd %dx%d robust=%d worst rel %.2e' % (H, W, robust, float(rel.max())))
    assert float(rel.max()) <= 1e-6
    total = sum(ref[:, i].sum() * ALPHAS[i] / 4 for i in range(5))
    rg = torch.autograd.grad(total, fd)
    _lib.call('cis_flow_multiscale_loss_bwd', pyr, *args, _st())
    torch.cuda.synchronize()
    worst = 0.0
    for i, ((gb, coff), r) in enumerate(zip(grads, rg)):
        got = gb[..., coff:coff + 2].float().cpu().double()
        assert torch.isfinite(got).all()
        err = (got - r).abs() - 2 ** -8 * r.abs()              # bf16 rounding of a value computed in fp32
        worst = max(worst, float(((got - r).abs() / r.abs().clamp_min(1e-30)).max()))
        assert float(err.max()) <= 1e-5 * float(r.abs().max()), (i, float(err.max()))
        if not robust:
            assert float(got[2].abs().max()) == 0.0             # d = 0: gradient 0, not NaN
        pad = gb.float().cpu()
        pad[..., coff:coff + 2] = 0
        assert float(pad.abs().max()) == 0.0                    # nothing outside the level's two channels
    print('MEASURED flow loss bwd %dx%d robust=%d worst rel %.2e (bf16)' % (H, W, robust, worst))
    first = [gb.clone() for gb, _ in grads]
    for i in range(5):
        pyr.accumulate[i] = 1
    _lib.call('cis_flow_multiscale_loss_bwd', pyr, *args, _st())
    torch.cuda.synchronize()
    for (gb, coff), f0 in zip(grads, first):
        a, b = gb[..., coff:coff + 2].float(), f0[..., coff:coff + 2].float()
        assert float((a - 2 * b).abs().max()) <= 2 ** -7 * float(b.abs().max()) + 1e-30


# ------------------------------------------------------------------------------------------------ 2. the gradient of one whole step
def _golden():
    """The parameters (seed, jitter) and frames of the 64x64 PWC-Net fixture, the frames repeated to 128x128: the warp + cost volume
    needs level 6 to be at least 2x2."""
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'pwc_64x64.npz'))
    up = lambda a: torch.from_numpy(np.asarray(a)).float().repeat_interleave(2, 1).repeat_interleave(2, 2).contiguous()
    return z, up(z['img1']), up(z['img2'])


@pytest.mark.parametrize('options', [None, NONDENSE])
def test_step_gradient_matches_fp64_autograd(options):
    from test_pwc_grad_gpu import COS_MIN, GRAD_TOL, SCOPE_TOL, _cos, _rel_l2
    z, img1, img2 = _golden()
    B, H, W = img1.shape[0], img1.shape[1], img1.shape[2]
    p = PO.make_params(seed=int(z['seed']), jitter=float(z['jitter']), options=options)
    gt = _smooth(B, H, W, 2, 3.0, torch.Generator().manual_seed(7))
    g = FlowTrainGraph(H, W, B, options=options)
    g.load_params(p)
    g.feed(img1.cuda(), img2.cuda(), gt.cuda())
    g.forward()
    g.bwd.run()
    torch.cuda.synchronize()
    names = [e[0] for e in g.store.entries]
    got = {n: g.store.view(n, 'grad').cpu().double() + (4e-4 * p[n].double() if n.endswith('/kernel') else 0.0) for n in names}
    pd = {n: p[n].double().requires_grad_(True) for n in names}
    _, pyr, _, _ = PO.predict_from_img_pairs(img1.double(), img2.double(), pd, return_pyr=True, options=options)
    total, terms = FR.flow_loss(pyr, gt.double())
    ref = dict(zip(names, torch.autograd.grad(total + FR.l2_term(pd), [pd[n] for n in names])))
    L = g.losses()
    for l, t in zip(LEVELS, terms):
        assert abs(L['flow_loss_l%d' % l] - float(t)) <= 2e-2 * abs(float(t)), (l, L, float(t))
    rel = _rel_l2([got[n] for n in names], [ref[n] for n in names])
    scopes = {}
    for n in names:
        scopes.setdefault(n.split('/')[1], []).append(n)
    for sc, ns in sorted(scopes.items()):
        r = _rel_l2([got[n] for n in ns], [ref[n] for n in ns])
        print('MEASURED flow step %s scope %s rel L2 %.4f' % (options, sc, r))
        assert r <= SCOPE_TOL, sc
    cos = {n: _cos(got[n], ref[n]) for n in names if n.endswith('/kernel')}
    worst = min(cos, key=cos.get)
    print('MEASURED flow step %s params rel L2 %.4f, lowest kernel cosine %.4f (%s)' % (options, rel, cos[worst], worst))
    assert rel <= GRAD_TOL and cos[worst] >= COS_MIN


# ------------------------------------------------------------------------------------------------ 3. the optimiser
def test_adam_l2_update_matches_fp64():
    gen = torch.Generator().manual_seed(3)
    n = 5000
    seg = [(0, 1200), (1300, 1301), (2000, 4999)]
    w, gr = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 1e-3
    m, v = torch.randn(n, generator=gen) * 1e-3, torch.rand(n, generator=gen) * 1e-6
    dev = [t.clone().cuda() for t in (w, m, v, gr)]
    segd = torch.tensor([x for s in seg for x in s], dtype=torch.int64, device='cuda')
    step = torch.full((1,), 4, dtype=torch.int64, device='cuda')
    lr = torch.full((1,), 3e-4, device='cuda')
    wd, md, vd = w.double(), m.double(), v.double()
    for t, rate in ((5, 3e-4), (6, 1.5e-4)):
        lr.fill_(rate)
        _lib.call('cis_adam_l2', dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), dev[3].data_ptr(), n, segd.data_ptr(), len(seg), 4e-4,
                  lr.data_ptr(), 0.9, 0.999, 1e-8, step.data_ptr(), _st())
        mask = torch.zeros(n, dtype=torch.float64)
        for a, b in seg:
            mask[a:b] = 1
        g = gr.double() + 4e-4 * wd * mask
        md = 0.9 * md + 0.1 * g
        vd = 0.999 * vd + 0.001 * g * g
        wd = wd - rate * (1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t) * md / (vd.sqrt() + 1e-8)
    torch.cuda.synchronize()
    assert int(step.item()) == 6
    for got, want in ((dev[0], wd), (dev[1], md), (dev[2], vd)):
        err = (got.cpu().double() - want).abs().max()
        assert float(err) <= 2e-6 * float(want.abs().max()), float(err)
    # outside the segments (biases) the decay does not act: a zero gradient leaves those parameters exactly where they are
    z = [torch.zeros(n, device='cuda') for _ in range(3)]
    w0 = w.clone().cuda()
    _lib.call('cis_adam_l2', w0.data_ptr(), z[0].data_ptr(), z[1].data_ptr(), z[2].data_ptr(), n, segd.data_ptr(), len(seg), 4e-4,
              lr.data_ptr(), 0.9, 0.999, 1e-8, step.data_ptr(), _st())
    torch.cuda.synchronize()
    out = w0.cpu()
    assert torch.equal(out[1200:1300], w[1200:1300]) and torch.equal(out[4999:], w[4999:])
    assert not torch.equal(out[:1200], w[:1200])


# ------------------------------------------------------------------------------------------------ 4. determinism and CUDA graphs
def _batches(n, B, H, W, seed):
    gen = torch.Generator().manual_seed(seed)
    return [(_smooth(B, H, W, 3, 0.25, gen).clamp(-0.5, 0.5), _smooth(B, H, W, 3, 0.25, gen).clamp(-0.5, 0.5), _smooth(B, H, W, 2, 3.0, gen))
            for _ in range(n)]


def test_training_is_deterministic_and_graph_replay_bit_identical():
    B, H, W = 2, 128, 128
    batches = _batches(5, B, H, W, 11)
    runs = []
    for use_graph in (False, False, True):
        g = FlowTrainGraph(H, W, B)
        g.load_params(init_pwcnet(g.store.entries))
        losses = []
        for k, b in enumerate(batches):
            if use_graph and k + 1 < len(batches):
                g.prefetch(*(t.pin_memory() for t in batches[k + 1]))
            g.feed(*b)
            g.train_step(use_graph=use_graph)
            losses.append(g.losses())
        torch.cuda.synchronize()
        runs.append(({k: v.cpu() for k, v in g.export_params().items()}, losses))
    for other in runs[1:]:
        assert other[1] == runs[0][1]
        diff = [k for k in runs[0][0] if not torch.equal(runs[0][0][k], other[0][k])]
        assert not diff, diff[:5]


# ------------------------------------------------------------------------------------------------ 5. learning
def _translated_batch(B, H, W):
    img1, img2, flow = [], [], []
    for b in range(B):
        a = pattern(b, H, W)
        dx, dy = (4, 2) if b % 2 == 0 else (-3, 5)
        for dst, im in ((img1, a), (img2, shifted(a, dx, dy))):
            dst.append(torch.from_numpy(im[..., ::-1].astype(np.float32) / 255.0 - 0.5))
        flow.append(torch.tensor([-float(dy), -float(dx)]).expand(H, W, 2))       # PWC-Net's order and sign: (-v, -u)
    return torch.stack(img1), torch.stack(img2), torch.stack(flow).contiguous()


def test_training_cuts_the_epe_on_a_fixed_batch():
    B, H, W = 4, 128, 192
    img1, img2, flow = (t.cuda() for t in _translated_batch(B, H, W))
    g = FlowTrainGraph(H, W, B, lr=5e-4)
    g.load_params(init_pwcnet(g.store.entries))

    def epe():
        s = g.epe().cpu()
        return float(s[:, 0].sum() / s[:, 2].sum())
    g.feed(img1, img2, flow)
    g.forward()
    curve = [epe()]
    for k in range(150):
        g.train_step(use_graph=True)
        if (k + 1) % 25 == 0:
            g.forward()
            curve.append(epe())
    print('MEASURED flow training EPE every 25 steps: %s' % ', '.join('%.3f' % e for e in curve))
    # measured on an H100 80GB HBM3 (700 W): 4.303, 3.350, 1.645, 0.524, 0.446, 0.213, 0.176 -- the bound keeps a 5x margin
    assert all(np.isfinite(curve)) and curve[-1] < 0.2 * curve[0], curve


# ------------------------------------------------------------------------------------------------ 6. the script end to end
def test_train_flow_script_writes_checkpoints_that_flow_ckpt_loads(tmp_path, capsys):
    root = make_chairs_tree(tmp_path / 'chairs', n=4, labels=[1, 1, 2, 2])
    ck = tmp_path / 'ck'
    cmd = [sys.executable, os.path.join(ROOT, 'train_flow.py'), '--dataset=FLYINGCHAIRS', '--root_dir=%s' % root, '--validate',
           '--img_height=128', '--img_width=128', '--batch_size=2', '--num_samples_train=2', '--max_epochs=1', '--save_freq=1',
           '--summary_freq=1', '--num_threads=2', '--checkpoint_dir=%s' % ck]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert 'Training completed successfully' in r.stdout and r.stdout.count('Validation EPE (flow)') == 1, r.stdout[-2000:]
    for base in ('pwcnet-1', 'pwcnet-best'):
        for suf in ('.index', '.data-00000-of-00001', '.pt'):
            assert (ck / (base + suf)).is_file(), (base, suf)
    from unsupervised_detection_b200.common_flags import Config
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    from unsupervised_detection_b200.models.PWCNet.model_pwcnet import ModelPWCNet
    from unsupervised_detection_b200.summary import read_events
    ev = [v['tag'] for f in os.listdir(str(ck)) if f.startswith('events') for e in read_events(str(ck / f)) for v in e.get('values', [])]
    assert ev.count('Validation EPE (flow)') == 1 and ev.count('flow_loss_l2') == 1
    # --flow_ckpt of train.py reads it
    L = AdversarialLearner()
    L.config = Config(dataset='SYNTHETIC', flow_ckpt=str(ck / 'pwcnet-1'), img_height=64, img_width=96, batch_size=2)
    L.build_train_graph()
    assert 'Flow net loaded from' in capsys.readouterr().out
    p = {k: v.cpu() for k, v in L.graph.pwc_store.export().items()}
    # the functional predict_from_img_pairs with those weights against the training graph's forward on the same frames
    from unsupervised_detection_b200.data.flyingchairs_data_utils import FlyingChairsReader
    rd = FlyingChairsReader(root, num_threads=1)
    it = rd.test_inputs()
    img1, img2, flow, _ = it.batch(2)
    it.close()
    small = [torch.nn.functional.interpolate(t.permute(0, 3, 1, 2), size=(128, 128), mode='bilinear').permute(0, 2, 3, 1).contiguous()
             for t in (img1, img2)]
    g = FlowTrainGraph(128, 128, 2)
    g.load_params(p)
    g.feed(small[0].cuda(), small[1].cuda(), torch.zeros(2, 128, 128, 2, device='cuda'))
    g.forward()
    fn = ModelPWCNet.predict_from_img_pairs(small[0].cuda(), small[1].cuda(), params={k: v.cuda() for k, v in p.items()})
    torch.cuda.synchronize()
    d = float((fn - g.flow).abs().max())
    print('MEASURED functional vs training-graph flow max |diff| %.3e (max |flow| %.3e)' % (d, float(g.flow.abs().max())))
    assert d <= 1e-5 * max(1.0, float(g.flow.abs().max()))


# ------------------------------------------------------------------------------------------------ 7. data parallelism
# Why 2 ranks x batch 2 cannot equal 1 GPU x batch 4 bit for bit: every weight gradient is a sum over the batch's pixels, and the engine
# splits that sum into split-K slices sized from the local batch (engine.wgrad_splits), adds each rank's slices in a fixed order, and
# the all-reduce then adds the two ranks' fp32 sums.  The full batch adds the same terms in another grouping, so the gradients agree
# only to fp32 rounding, and Adam's m / sqrt(v) carries that into the parameters.  What must hold exactly is that the ranks agree with
# each other; against one GPU the checks are relative: the step-1 gradient to a small fraction of its norm, and the parameters after
# the steps to a small fraction of how far they moved from their start.  A wrong slice, a wrong 1 / global batch or a missing
# all-reduce changes the gradient by O(1) of its norm (the negative control below shows the margin).
DP = dict(GB=4, steps=3, H=128, W=128)
# Measured on an H100 80GB HBM3 (700 W) by test_sharded_batch_matches_the_full_batch: gradient rel L2 3.5e-4 (one half batch alone:
# 0.20), parameters 9.9e-3 of their movement.  Adam is nearly scale-invariant, so the parameter check alone would miss a wrong
# 1 / global batch; the gradient check catches it.
DP_GRAD_TOL, DP_PARAM_TOL = 5e-3, 3e-2


def _dp_metrics(full, part, init):
    """full / part = (step-1 flat gradient, final flat parameters) of the 1-GPU run and of one rank; init = the flat parameters at the
    start -> (gradient rel L2, mean |parameter difference| / mean |movement of the 1-GPU run|)."""
    grad = float((part[0] - full[0]).norm() / full[0].norm())
    moved = float((full[1] - init).abs().mean())
    return grad, float((part[1] - full[1]).abs().mean()) / moved


def _dp_step(g, batch, allreduce):
    """One eager step of `g` on `batch` (this rank's slice) -> the flat gradient after the all-reduce (a copy)."""
    g.feed(*batch)
    g.forward()
    g.bwd.run()
    if allreduce is not None:
        allreduce(g.store.grad)
    grad = g.store.grad.clone()
    g.adam.run()
    g.pack.run()
    return grad


def test_sharded_batch_matches_the_full_batch():
    """The arithmetic of a 2-rank job on one GPU: two graphs on the halves of each global batch (global_batch = 4), their gradients
    summed as the all-reduce does, against one graph on the whole batch."""
    H, W, GB = DP['H'], DP['W'], DP['GB']
    batches = [tuple(t.cuda() for t in b) for b in _batches(DP['steps'], GB, H, W, 5)]
    full = FlowTrainGraph(H, W, GB)
    halves = [FlowTrainGraph(H, W, GB // 2, global_batch=GB) for _ in range(2)]
    p = init_pwcnet(full.store.entries)
    for g in [full] + halves:
        g.load_params(p)
    init = full.store.flat.clone()
    for k, b in enumerate(batches):
        gf = _dp_step(full, b, None)
        parts = []
        for r, g in enumerate(halves):
            g.feed(*(t[r * 2:(r + 1) * 2] for t in b))
            g.forward()
            g.bwd.run()
            parts.append(g.store.grad.clone())
        summed = parts[0] + parts[1]
        for g in halves:
            g.store.grad.copy_(summed)
            g.adam.run()
            g.pack.run()
        if k == 0:
            first = (gf, summed, parts[0])
    torch.cuda.synchronize()
    assert torch.equal(halves[0].store.flat, halves[1].store.flat)
    grad, param = _dp_metrics((first[0], full.store.flat), (first[1], halves[0].store.flat), init)
    wrong = float((2 * first[2] - first[0]).norm() / first[0].norm())      # one half batch standing in for the whole
    print('MEASURED sharded vs full batch: step-1 gradient rel L2 %.3e (one half alone: %.3e), parameters mean |diff| / mean |moved| %.3e'
          % (grad, wrong, param))
    assert grad <= DP_GRAD_TOL and param <= DP_PARAM_TOL
    assert wrong >= 10 * DP_GRAD_TOL


def _run_dp(out):
    """DP['steps'] eager steps on fixed global batches (each rank its slice, one all-reduce per step) -> {step-1 gradient, final flat
    parameters, initial flat parameters} saved under `out`."""
    world = 1
    if int(os.environ.get('WORLD_SIZE', '1')) > 1:
        import torch.distributed as dist
        rank = int(os.environ['RANK'])
        torch.cuda.set_device(rank)
        dist.init_process_group('nccl', device_id=torch.device('cuda', rank))
        world = dist.get_world_size()
        allreduce = lambda t: dist.all_reduce(t)
    else:
        rank, allreduce = 0, None
    lb = DP['GB'] // world
    g = FlowTrainGraph(DP['H'], DP['W'], lb, global_batch=DP['GB'], device='cuda:%d' % rank)
    g.load_params(init_pwcnet(g.store.entries))
    init = g.store.flat.clone()
    blob = torch.load(os.path.join(out, 'inputs.pt'))
    sl = slice(rank * lb, (rank + 1) * lb)
    grads = [_dp_step(g, tuple(t[sl].cuda() for t in b), allreduce) for b in blob['batches']]
    torch.cuda.synchronize()
    res = dict(grad=grads[0].cpu(), flat=g.store.flat.cpu(), init=init.cpu())
    torch.save(res, os.path.join(out, 'world%d_rank%d.pt' % (world, rank)))
    return res


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_ranks_equal_one_gpu(tmp_path):
    from test_recover_pretrain_gpu import _free_port
    torch.save(dict(batches=_batches(DP['steps'], DP['GB'], DP['H'], DP['W'], 5)), str(tmp_path / 'inputs.pt'))
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', str(_free_port()), os.path.abspath(__file__), str(tmp_path)]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=500)
    assert r.returncode == 0, r.stderr[-2000:]
    ranks = [torch.load(str(tmp_path / ('world2_rank%d.pt' % i))) for i in range(2)]
    one = _run_dp(str(tmp_path))
    assert torch.equal(ranks[0]['grad'], ranks[1]['grad']) and torch.equal(ranks[0]['flat'], ranks[1]['flat'])
    assert torch.equal(ranks[0]['init'], one['init'])
    grad, param = _dp_metrics((one['grad'], one['flat']), (ranks[0]['grad'], ranks[0]['flat']), one['init'])
    print('MEASURED 2 ranks x batch 2 vs 1 GPU x batch 4: step-1 gradient rel L2 %.3e, parameters mean |diff| / mean |moved| %.3e'
          % (grad, param))
    assert grad <= DP_GRAD_TOL and param <= DP_PARAM_TOL


if __name__ == '__main__':
    _run_dp(sys.argv[1])
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()
