"""Unsupervised PWC-Net fine-tuning on the GPU: the census + smoothness loss kernels against the fp64 restatement
(tests/unsup_flow_loss_ref.py), the gradient of a whole step against fp64 autograd through the oracle PWC-Net, determinism and CUDA-graph
replay, learning a known translation without its flow, train_flow.py --flow_loss=unsupervised end to end, and a sharded batch against
the full one."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import flow_loss_ref as FR  # noqa: E402
import pwc_options_ref as PO  # noqa: E402
import unsup_flow_loss_ref as UR  # noqa: E402
from chairs_tree import make_chairs_tree  # noqa: E402
from flow_trees import make_davis_tree  # noqa: E402
from test_flow_train_gpu import (DP, DP_PARAM_TOL, _batches, _dp_metrics, _dp_step, _golden, _smooth,  # noqa: E402
                                 _translated_batch)
from unsupervised_detection_b200 import _lib  # noqa: E402
from unsupervised_detection_b200.flow_train_graph import FlowTrainGraph  # noqa: E402
from unsupervised_detection_b200.params_init import init_pwcnet  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
NONDENSE = {'use_dense_cx': False, 'use_res_cx': False, 'search_range': 2}
NEAR = 1e-4          # mask decisions and bilinear kinks closer than this to their threshold are not compared


def _st():
    return torch.cuda.current_stream().cuda_stream


def _inputs(B, H, W, seed):
    """Textured frames in [-0.5, 0.5] and smooth flows up to about 8 px; the backward flow is minus the forward one plus a smooth
    field, so that some pixels pass the consistency check and some fail it."""
    gen = torch.Generator().manual_seed(seed)
    frames = [(_smooth(B, H, W, 3, 0.3, gen) + 0.2 * (torch.rand(B, H, W, 3, generator=gen) - 0.5)).clamp(-0.5, 0.5) for _ in range(2)]
    ff = _smooth(B, H, W, 2, 3.0, gen)
    fb = -ff + _smooth(B, H, W, 2, 1.0, gen)
    return frames[0].contiguous(), frames[1].contiguous(), torch.cat([ff, fb]).contiguous()


def _near_mask_threshold(flow):
    """fp64 mask of flow, and where a decision is within NEAR of its threshold (occlusion test or the frame border)."""
    H, W = flow.shape[1], flow.shape[2]
    M, V, lhs, rhs = UR.mask(flow)
    qy, qx = UR.sample_points(flow)
    edge = torch.stack([qy.abs(), (qy - (H - 1)).abs(), qx.abs(), (qx - (W - 1)).abs()]).min(0)[0]
    return M, V, lhs, rhs, ((lhs - rhs).abs() < NEAR) | (edge < NEAR)


# ------------------------------------------------------------------------------------------------ 1. the loss kernels
@pytest.mark.parametrize('B,H,W', [(2, 384, 640), (2, 128, 192), (3, 70, 98)])
def test_loss_kernels_match_fp64(B, H, W):
    img1, img2, flow = _inputs(B, H, W, H + W)
    GB, lam = B + 1, 3.0
    N = 2 * B
    d = [t.cuda() for t in (img1, img2, flow)]
    warped, mask, coef = (torch.full((N, H, W), float('nan'), device='cuda') for _ in range(3))
    scratch = torch.full((2 * N * 64,), float('nan'), dtype=torch.float64, device='cuda')
    fwd = lambda out, fl=d[2].data_ptr(): _lib.call('cis_unsup_flow_loss', fl, d[0].data_ptr(), d[1].data_ptr(), B, H, W,
                                                      warped.data_ptr(), mask.data_ptr(), coef.data_ptr(), scratch.data_ptr(),
                                                      out.data_ptr(), _st())
    outs = []
    for _ in range(2):
        out = torch.full((N, 2), float('nan'), dtype=torch.float64, device='cuda')
        fwd(out)
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])
    with pytest.raises(RuntimeError, match='alignment'):          # the flow is read as float pairs: 8-byte alignment is checked
        fwd(out, d[2].data_ptr() + 4)
    with pytest.raises(RuntimeError, match='size'):
        _lib.call('cis_unsup_flow_loss', d[2].data_ptr(), d[0].data_ptr(), d[1].data_ptr(), B, 2, W, warped.data_ptr(), mask.data_ptr(),
                  coef.data_ptr(), scratch.data_ptr(), out.data_ptr(), _st())
    # the mask: equal to fp64 but for decisions within NEAR of their threshold; the inputs hold out-of-frame and occluded pixels.  The
    # fp64 reference runs on the device.
    fd = d[2].double()
    M, V, lhs, rhs, near = _near_mask_threshold(fd)
    gm = mask.double()
    assert bool((V == 0).any()) and bool(((V == 1) & (lhs > rhs)).any()) and bool((M == 1).any())
    assert int(((gm != M) & ~near).sum()) == 0
    print('MEASURED unsup mask %dx%d B=%d: %d of %d pixels differ from fp64, all within %g of the threshold (%d near it); out of frame '
          '%d, occluded %d' % (H, W, B, int((gm != M).sum()), M.numel(), NEAR, int(near.sum()), int((V == 0).sum()),
                               int(((V == 1) & (lhs > rhs)).sum())))
    m_used = torch.where(near, gm, M)
    fr = fd.clone().requires_grad_(True)
    ref, terms = UR.direction_sums(fr, d[0].double(), d[1].double(), m=m_used)
    rel = (outs[0] - ref.detach().cpu()).abs() / ref.detach().cpu().abs()
    print('MEASURED unsup loss fwd %dx%d B=%d worst rel %.2e' % (H, W, B, float(rel.max())))
    assert float(rel.max()) <= 1e-5
    assert float((warped.double() - terms['warped'].detach()).abs().max()) <= 1e-4      # T~ in [0, 255]
    kref = (m_used * 0.4 * (terms['c'].detach() + 0.01) ** -0.6)
    assert float((coef.double() - kref).abs().max()) <= 1e-4 * float(kref.abs().max())
    # the backward against autograd, away from the bilinear kinks and clamp edges of the pixel's own sample point
    loss = (ref[:, 0].sum() + lam * ref[:, 1].sum()) / (GB * H * W)
    (gref,) = torch.autograd.grad(loss, fr)
    dflow = torch.full((N, H, W, 2), float('nan'), device='cuda')
    _lib.call('cis_unsup_flow_loss_bwd', d[2].data_ptr(), d[0].data_ptr(), d[1].data_ptr(), B, H, W, warped.data_ptr(), coef.data_ptr(),
              1.0 / (GB * H * W), lam / (GB * H * W), dflow.data_ptr(), _st())
    torch.cuda.synchronize()
    got = dflow.double()
    assert torch.isfinite(got).all()
    qy, qx = UR.sample_points(fd)
    kink = ((qy - qy.round()).abs() < NEAR) | ((qx - qx.round()).abs() < NEAR)
    err = (got - gref).abs().amax(-1)[~kink]
    scale = float(gref.abs().max())
    print('MEASURED unsup loss bwd %dx%d B=%d max |err| / max |ref| %.2e (%d pixels at kinks left out)'
          % (H, W, B, float(err.max()) / scale, int(kink.sum())))
    assert float(err.max()) <= 1e-4 * scale


# ------------------------------------------------------------------------------------------------ 2. the gradient of one whole step
@pytest.mark.parametrize('options', [None, NONDENSE])
def test_step_gradient_matches_fp64_autograd(options):
    from test_pwc_grad_gpu import COS_MIN, GRAD_TOL, SCOPE_TOL, _cos, _rel_l2
    z, img1, img2 = _golden()
    B, H, W = img1.shape[0], img1.shape[1], img1.shape[2]
    p = PO.make_params(seed=int(z['seed']), jitter=float(z['jitter']), options=options)
    g = FlowTrainGraph(H, W, B, options=options, loss='unsupervised')
    g.load_params(p)
    g.feed(img1.cuda(), img2.cuda())
    g.forward()
    g.bwd.run()
    torch.cuda.synchronize()
    # the graph's mask against one recomputed in fp64 from the graph's own flows
    gm = g.mask.cpu().double()
    M, _, _, _, near = _near_mask_threshold(g.flow.cpu().double())
    assert int(((gm != M) & ~near).sum()) == 0
    names = [e[0] for e in g.store.entries]
    got = {n: g.store.view(n, 'grad').cpu().double() + (4e-4 * p[n].double() if n.endswith('/kernel') else 0.0) for n in names}
    pd = {n: p[n].double().requires_grad_(True) for n in names}
    S, T = UR.directions(img1.double(), img2.double())
    flow = PO.predict_from_img_pairs(S, T, pd, options=options)
    total = UR.loss(flow, img1.double(), img2.double(), m=gm)          # M carries no gradient: the graph's mask
    ref = dict(zip(names, torch.autograd.grad(total + FR.l2_term(pd), [pd[n] for n in names])))
    L = g.losses()
    assert abs(L['flow_loss'] - float(total)) <= 2e-2 * abs(float(total)), (L, float(total))
    assert L['flow_loss'] == pytest.approx(L['flow_loss_photo'] + L['flow_loss_smooth'], rel=1e-12)
    rel = _rel_l2([got[n] for n in names], [ref[n] for n in names])
    scopes = {}
    for n in names:
        scopes.setdefault(n.split('/')[1], []).append(n)
    for sc, ns in sorted(scopes.items()):
        r = _rel_l2([got[n] for n in ns], [ref[n] for n in ns])
        print('MEASURED unsup step %s scope %s rel L2 %.4f' % (options, sc, r))
        assert r <= SCOPE_TOL, sc
    cos = {n: _cos(got[n], ref[n]) for n in names if n.endswith('/kernel')}
    worst = min(cos, key=cos.get)
    print('MEASURED unsup step %s params rel L2 %.4f, lowest kernel cosine %.4f (%s)' % (options, rel, cos[worst], worst))
    assert rel <= GRAD_TOL and cos[worst] >= COS_MIN


# ------------------------------------------------------------------------------------------------ 3. determinism and CUDA graphs
def test_training_is_deterministic_and_graph_replay_bit_identical():
    B, H, W = 2, 128, 128
    batches = [b[:2] for b in _batches(5, B, H, W, 13)]
    runs = []
    for use_graph in (False, False, True):
        g = FlowTrainGraph(H, W, B, loss='unsupervised')
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


# ------------------------------------------------------------------------------------------------ 4. learning without ground truth
# The occlusion mask carries no gradient, and a pixel it masks costs nothing: the objective only teaches where the two directions' flows
# already agree.  From params_init.init_pwcnet they do not (the untrained network predicts nearly the same flow for a pair and its swap,
# so M covers 0-3 % of the pixels), and neither do they after supervised steps on the forward pairs alone, which on this two-translation
# batch teach a flow that ignores the order of the frames (M = 0).  Measured on an H100 80GB HBM3 (700 W): from either start 300
# unsupervised steps raised both the objective and the EPE.  So the run starts where fine-tuning starts in practice, from a network that
# computes flow: SUP_STEPS supervised steps on the pairs and their swaps (M covers ~70 % of the pixels), then UNSUP_STEPS unsupervised
# steps at rate 3e-5 (at 1e-4 the mask and the EPE oscillated).
SUP_STEPS, UNSUP_STEPS = 150, 200


def test_unsupervised_fine_tuning_cuts_the_objective_and_the_epe():
    B, H, W = 4, 128, 192
    img1, img2, flow = (t.cuda() for t in _translated_batch(B, H, W))
    sup = FlowTrainGraph(H, W, 2 * B, lr=5e-4)
    sup.load_params(init_pwcnet(sup.store.entries))
    sup.feed(torch.cat([img1, img2]), torch.cat([img2, img1]), torch.cat([flow, -flow]))
    for _ in range(SUP_STEPS):
        sup.train_step(use_graph=True)
    g = FlowTrainGraph(H, W, B, lr=3e-5, loss='unsupervised')
    g.load_params(sup.export_params())
    g.feed(img1, img2, flow)                   # the ground truth is uploaded for epe() only

    def point():
        g.forward()
        s = g.epe().cpu()
        return g.losses()['flow_loss'], float(s[:, 0].sum() / s[:, 2].sum()), float(g.mask.mean())
    curve = [point()]
    for k in range(UNSUP_STEPS):
        g.train_step(use_graph=True)
        if (k + 1) % 25 == 0:
            curve.append(point())
    obj, epe, m = ([c[i] for c in curve] for i in range(3))
    print('MEASURED unsupervised objective every 25 steps: %s' % ', '.join('%.4f' % v for v in obj))
    print('MEASURED unsupervised EPE every 25 steps: %s' % ', '.join('%.3f' % v for v in epe))
    print('MEASURED unsupervised visible fraction every 25 steps: %s' % ', '.join('%.2f' % v for v in m))
    # measured on an H100 80GB HBM3 (700 W): objective 1.968 -> 1.208, EPE 0.548 -> 0.343, M 0.70 -> 0.88, both falling at every
    # point; the bounds keep about half of each fall as margin
    assert m[0] >= 0.5
    assert all(torch.isfinite(torch.tensor(obj + epe)))
    assert obj[-1] < 0.8 * obj[0] and epe[-1] < 0.8 * epe[0], (obj, epe)


# ------------------------------------------------------------------------------------------------ 5. the script end to end
def _run(args, tmp_path):
    cmd = [sys.executable] + args
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout


def test_train_flow_unsupervised_on_davis_writes_checkpoints_that_flow_ckpt_loads(tmp_path):
    root = make_davis_tree(tmp_path / 'davis')
    ck = tmp_path / 'ck'
    common = ['--img_height=128', '--img_width=128', '--batch_size=2', '--num_samples_train=2', '--max_epochs=1', '--save_freq=1',
              '--summary_freq=1', '--num_threads=2']
    out = _run([os.path.join(ROOT, 'train_flow.py'), '--dataset=DAVIS2016', '--root_dir=%s' % root, '--flow_loss=unsupervised',
                '--validate', '--checkpoint_dir=%s' % ck] + common, tmp_path)
    assert 'Training completed successfully' in out and out.count('Validation unsupervised flow loss') == 1, out[-2000:]
    for base in ('pwcnet-1', 'pwcnet-best'):
        for suf in ('.index', '.data-00000-of-00001', '.pt'):
            assert (ck / (base + suf)).is_file(), (base, suf)
    from unsupervised_detection_b200.summary import read_events
    ev = [v['tag'] for f in os.listdir(str(ck)) if f.startswith('events') for e in read_events(str(ck / f)) for v in e.get('values', [])]
    assert ev.count('Validation unsupervised flow loss') == 1 and ev.count('flow_loss_smooth') == 1
    # --flow_ckpt of export_flow.py reads it
    fdir = tmp_path / 'flo'
    out = _run([os.path.join(ROOT, 'export_flow.py'), '--dataset=DAVIS2016', '--root_dir=%s' % root, '--flow_dir=%s' % fdir,
                '--flow_ckpt=%s' % (ck / 'pwcnet-1'), '--batch_size=2', '--num_threads=2'], tmp_path)
    assert any(f.endswith('.flo') for _, _, fs in os.walk(str(fdir)) for f in fs), out[-2000:]
    # on Flying Chairs the unsupervised loss validates with the end-point error
    chairs = make_chairs_tree(tmp_path / 'chairs', n=4, labels=[1, 1, 2, 2])
    out = _run([os.path.join(ROOT, 'train_flow.py'), '--dataset=FLYINGCHAIRS', '--root_dir=%s' % chairs, '--flow_loss=unsupervised',
                '--validate', '--checkpoint_dir=%s' % (tmp_path / 'ck2')] + common, tmp_path)
    assert 'Training completed successfully' in out and out.count('Validation EPE (flow)') == 1, out[-2000:]


# ------------------------------------------------------------------------------------------------ 6. data parallelism
# The network's forward is not bit-identical between batch 4 and batch 2 (final flows differ by up to 6e-3 px), and this objective is
# not smooth in the flow: sign(second difference) and the occlusion mask switch where the supervised loss bends smoothly.  So the
# step-1 gradient agrees less closely than the multi-scale loss's 5e-3.  Measured on an H100 80GB HBM3 (700 W): 8.8e-3 (one half batch
# alone: 0.14), parameters 9.8e-3 of their movement.
UNSUP_DP_GRAD_TOL = 2e-2
def test_sharded_batch_matches_the_full_batch():
    """Two graphs on the halves of each global batch (global_batch = 4), their gradients summed as the all-reduce does, against one
    graph on the whole batch (why they cannot agree bit for bit: tests/test_flow_train_gpu.py)."""
    H, W, GB = DP['H'], DP['W'], DP['GB']
    batches = [tuple(t.cuda() for t in b[:2]) for b in _batches(DP['steps'], GB, H, W, 5)]
    full = FlowTrainGraph(H, W, GB, loss='unsupervised')
    halves = [FlowTrainGraph(H, W, GB // 2, global_batch=GB, loss='unsupervised') for _ in range(2)]
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
    wrong = float((2 * first[2] - first[0]).norm() / first[0].norm())
    print('MEASURED unsup sharded vs full batch: step-1 gradient rel L2 %.3e (one half alone: %.3e), parameters mean |diff| / mean '
          '|moved| %.3e' % (grad, wrong, param))
    assert grad <= UNSUP_DP_GRAD_TOL and param <= DP_PARAM_TOL
    assert wrong >= 5 * UNSUP_DP_GRAD_TOL
