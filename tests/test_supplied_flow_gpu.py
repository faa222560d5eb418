"""Supplied optical flow (--flow_dir) on the GPU: the input-flow generator graph fed PWC-Net's own flow is bit-identical to the default
graph (train and test graphs, sequential and pipelined schedules), cis_crop_resize_flow_f32 against its host restatement, and the scripts
end to end on a tiny DAVIS tree with the synthetic PWC-Net."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from flow_trees import make_davis_tree  # noqa: E402
from oracle import params as OP  # noqa: E402
from test_parity_bench_sizes_gpu import smooth  # noqa: E402
from unsupervised_detection_b200 import _lib, params_init  # noqa: E402
from unsupervised_detection_b200.step_graph import CISGraph  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

B, H, W = 4, 256, 448
STEPS = 8


def _st():
    return torch.cuda.current_stream().cuda_stream


def _graphs(train=True):
    """The default graph and an input-flow graph with the same parameters."""
    d = CISGraph(H, W, B, train=train)
    i = CISGraph(H, W, B, train=train, masks='generator', flow_source='input')
    p = OP.make_params(seed=13, jitter=0.05, nets=('MaskNet', 'FlownetS'))
    p.update(params_init.init_pwcnet(d.pwc_store.entries))
    d.load_params(p)
    i.load_params(p)
    return d, i


def _frames(n, seed):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        a = smooth(B, 384, 640, 3, 0.25, gen).clamp(-0.5, 0.5)
        out.append((a.cuda(), torch.roll(a, shifts=(3, -5), dims=(1, 2)).cuda()))
    return out


def _pwc_flows(d, frames):
    """PWC-Net's flow_full of every frame pair, from the default graph itself."""
    out = []
    for a, b in frames:
        d.img1.copy_(a)
        d.img2.copy_(b)
        d.forward_flow()
        out.append(d.flow_full.clone())
    torch.cuda.synchronize()
    return out


def _run(g, uploads, pipelined):
    """STEPS alternating steps (1R:3G) on the uploads (what g.inputs takes per batch) -> per-step outputs and the final parameters."""
    rec = []
    if pipelined:
        for dst, src in zip(g.inputs, uploads[0]):
            dst.copy_(src)
        g.prime_pipeline()
    for t in range(STEPS):
        mode = 'R' if t % 4 == 0 else 'G'
        nxt = uploads[t + 1] if pipelined else uploads[t]
        if pipelined:
            torch.cuda.current_stream().wait_event(g.pipeline_inputs_free())
        for dst, src in zip(g.inputs, nxt):
            dst.copy_(src)
        ready = torch.cuda.Event()
        ready.record()
        g.train_step(mode, use_graph=True, pipeline=pipelined, inputs_ready=ready)
        torch.cuda.synchronize()
        rec.append(dict(image=g.image.cpu(), flow=g.flow.cpu(), mask=g.mask.cpu(), sums=g.sums.cpu(), grad=g.store(mode).grad.cpu()))
    g.pipeline_drain()
    torch.cuda.synchronize()
    return rec, {k: v.cpu() for k, v in g.export_params().items() if not k.startswith('pwcnet/')}


def _same(a, b, what):
    ra, pa = a
    rb, pb = b
    for t, (x, y) in enumerate(zip(ra, rb)):
        bad = [k for k in x if not torch.equal(x[k], y[k])]
        assert not bad, (what, t, bad)
    assert sorted(pa) == sorted(pb)
    bad = [k for k in pa if not torch.equal(pa[k], pb[k])]
    assert not bad, (what, bad[:5])


def test_input_flow_train_graph_is_bit_identical_to_the_default_graph():
    """The central check: the default graph on seeded frame pairs, and an input-flow graph with the same parameters fed the default
    graph's own flow_full, give the same image, flow, mask, five loss sums, both nets' gradients and, after 8 alternating steps, the
    same parameters -- in the sequential and in the pipelined schedule."""
    d, i = _graphs()
    frames = _frames(STEPS + 1, 5)
    flows = _pwc_flows(d, frames)
    # both nets' gradients on the first batch, before any update
    for g, up in ((d, frames[0]), (i, (frames[0][0], flows[0]))):
        for dst, src in zip(g.inputs, up):
            dst.copy_(src)
        g.forward()
        g.bwd['R'].run()
        g.bwd['G'].run()
    torch.cuda.synchronize()
    for name in ('image', 'flow', 'mask', 'sums', 'pred', 'scalars'):
        assert torch.equal(getattr(d, name).cpu(), getattr(i, name).cpu()), name
    for m in ('R', 'G'):
        assert torch.equal(d.store(m).grad.cpu(), i.store(m).grad.cpu()), m
    inputs = [(a, f) for (a, _), f in zip(frames, flows)]
    state = {k: v.clone() for k, v in d.export_params().items()}
    seq_d, seq_i = _run(d, frames, False), _run(i, inputs, False)
    _same(seq_d, seq_i, 'sequential')
    assert any(not torch.equal(seq_i[1][k], state[k].cpu()) for k in seq_i[1] if k.startswith('MaskNet/'))
    assert any(not torch.equal(seq_i[1][k], state[k].cpu()) for k in seq_i[1] if k.startswith('FlownetS/'))
    del d, i
    d, i = (CISGraph(H, W, B, masks='generator', flow_source=s) for s in ('pwc', 'input'))  # fresh Adam state and parameters for the pipelined schedule
    for g in (d, i):
        g.load_params(state)
    pipe_d, pipe_i = _run(d, frames, True), _run(i, inputs, True)
    _same(pipe_d, pipe_i, 'pipelined')
    _same(seq_i, pipe_i, 'input flow: sequential vs pipelined')


def test_input_flow_test_graph_gives_the_same_masks_and_pred():
    d, i = _graphs(train=False)
    frames = _frames(1, 9)
    (flow,) = _pwc_flows(d, frames)
    d.feed(*frames[0])
    i.feed(frames[0][0], flow)
    d.forward()
    i.forward()
    torch.cuda.synchronize()
    assert torch.equal(d.mask.cpu(), i.mask.cpu()) and torch.equal(d.pred.cpu(), i.pred.cpu())
    d.forward_masks(use_graph=True)
    i.forward_masks(use_graph=True)
    torch.cuda.synchronize()
    assert torch.equal(d.mask.cpu(), i.mask.cpu())


# ------------------------------------------------------------------------------------------------ the crop kernel
CROPS = [0.85, 0.9, 0.95, 1.0]


def test_flow_crop_kernel_matches_the_host_restatement():
    """cis_crop_resize_flow_f32 against crop_resized + the vector scale (rows by Hs/ch, columns by Ws/cw), within the bound the image
    crop kernel is held to (tests/test_kernels_gpu.py), relative to the field's magnitude."""
    from unsupervised_detection_b200.data.davis2016_data_utils import central_crop_box, crop_resized
    gen = torch.Generator().manual_seed(31)
    for hs, ws in ((96, 160), (384, 640)):
        fl = smooth(1, hs, ws, 2, 3.0, gen)
        src = fl.cuda()
        out = torch.empty(len(CROPS), hs, ws, 2, device='cuda')
        for k, c in enumerate(CROPS):
            y0, x0, ch, cw = central_crop_box(hs, ws, c)
            _lib.call('cis_crop_resize_flow_f32', src.data_ptr(), hs, ws, y0, x0, ch, cw, out[k].data_ptr(), hs, ws, hs / ch, ws / cw, _st())
        torch.cuda.synchronize()
        for k, c in enumerate(CROPS):
            y0, x0, ch, cw = central_crop_box(hs, ws, c)
            ref = crop_resized(fl[0].numpy(), y0, x0, ch, cw) * np.array([hs / ch, ws / cw], np.float32)
            got = out[k].cpu().numpy()
            assert np.abs(got - ref).max() <= 2e-6 * max(1.0, float(np.abs(ref).max())), (hs, c, np.abs(got - ref).max())
        assert torch.equal(out[3].cpu(), fl[0])                                  # crop 1.0 is the identity
    with pytest.raises(RuntimeError):
        _lib.call('cis_crop_resize_flow_f32', src.data_ptr(), hs, ws, 10, 0, hs, ws, out[0].data_ptr(), hs, ws, 1.0, 1.0, _st())


def _ensemble_learner(flow_source):
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    L = AdversarialLearner()
    L.test_crops = CROPS
    L.graph = CISGraph(64, 96, len(CROPS), train=False, masks='generator', flow_source=flow_source)
    return L


def test_device_crops_on_both_flow_sources():
    """_device_crops on the default path still cuts the frame pair with the image kernel (the same values as direct calls), and on an
    input-flow graph cuts frame 1 the same way and the flow with the new kernel."""
    from unsupervised_detection_b200.data.davis2016_data_utils import central_crop_box
    gen = torch.Generator().manual_seed(37)
    img1, img2 = torch.rand(1, 384, 640, 3, generator=gen) - 0.5, torch.rand(1, 384, 640, 3, generator=gen) - 0.5
    flow, gt = smooth(1, 384, 640, 2, 4.0, gen), (torch.rand(1, 384, 640, 1, generator=gen) > 0.5).float()
    Ld, Li = _ensemble_learner('pwc'), _ensemble_learner('input')
    gd, gi = Ld._device_crops(img1, img2, gt), Li._device_crops(img1, flow, gt)
    torch.cuda.synchronize()
    assert np.array_equal(gd, gi)
    d1, d2, df = img1.cuda(), img2.cuda(), flow.cuda()
    for k, c in enumerate(CROPS):
        y0, x0, ch, cw = central_crop_box(384, 640, c)
        ref = torch.empty(3, 384, 640, 3, device='cuda')
        rf = torch.empty(384, 640, 2, device='cuda')
        for src, dst in ((d1, ref[0]), (d2, ref[1])):
            _lib.call('cis_crop_resize_bilinear_f32', src.data_ptr(), 384, 640, 3, y0, x0, ch, cw, dst.data_ptr(), 384, 640, _st())
        _lib.call('cis_crop_resize_flow_f32', df.data_ptr(), 384, 640, y0, x0, ch, cw, rf.data_ptr(), 384, 640, 384 / ch, 640 / cw, _st())
        torch.cuda.synchronize()
        assert torch.equal(Ld.graph.img1[k], ref[0]) and torch.equal(Ld.graph.img2[k], ref[1]) and torch.equal(Li.graph.img1[k], ref[0])
        assert torch.equal(Li.graph.flow_full[k], rf)


# ------------------------------------------------------------------------------------------------ the scripts end to end
def _script(name, *args, cwd):
    cmd = [sys.executable, os.path.join(ROOT, name)] + list(args)
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT, CIS_READER_PREFETCH='0'), cwd=str(cwd), capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, (name, r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


def _report(out):
    return [ln for ln in out.splitlines() if re.match(r'(Category |The Average|Success)', ln)]


@pytest.fixture(scope='module')
def davis(tmp_path_factory):
    base = tmp_path_factory.mktemp('e2e')
    root = make_davis_tree(base / 'davis')
    flow_dir = str(base / 'flow')
    common = ['--dataset=DAVIS2016', '--root_dir=%s' % root, '--img_height=64', '--img_width=96', '--batch_size=2', '--num_threads=2',
              '--train_partition=train', '--test_partition=val', '--test_temporal_shift=1']
    out = _script('export_flow.py', *common, '--flow_dir=%s' % flow_dir, '--flow_ckpt=synthetic', cwd=base)
    assert 'Success: wrote the flow of' in out, out[-2000:]
    return base, root, flow_dir, common


def test_export_then_test_generator_equals_pwcnet_in_the_loop(davis):
    base, root, flow_dir, common = davis
    from export_flow import export_pairs, make_reader
    from unsupervised_detection_b200.common_flags import Config
    from unsupervised_detection_b200.data.davis2016_data_utils import flow_file
    cfg = Config(dataset='DAVIS2016', root_dir=root, train_partition='train', test_partition='val', test_temporal_shift=1)
    pairs = export_pairs(cfg, make_reader(cfg))
    assert pairs and all(os.path.isfile(flow_file(flow_dir, root, a, b)) for a, b in pairs)
    reps, mats = [], []
    for k, extra in enumerate(([], ['--flow_dir=%s' % flow_dir])):
        save = base / ('vis%d' % k)
        out = _script('test_generator.py', *common, '--test_crop=1.0', '--ckpt_file=synthetic', '--generate_visualization',
                      '--test_save_dir=%s' % save, *extra, cwd=base)
        reps.append(_report(out))
        import scipy.io as sio
        mats.append({f: sio.loadmat(str(save / 'cows' / f)) for f in sorted(os.listdir(str(save / 'cows'))) if f.endswith('.mat')})
    assert reps[0] == reps[1] and any(ln.startswith('Category cows') for ln in reps[0]), reps
    assert sorted(mats[0]) == sorted(mats[1]) and len(mats[0]) == 6
    for f in mats[0]:
        for key in ('pred_mask', 'flow', 'img1', 'gt_mask'):
            assert np.array_equal(mats[0][f][key], mats[1][f][key]), (f, key)


def test_train_on_supplied_flow_then_evaluate(davis):
    base, root, flow_dir, common = davis
    ck = base / 'ck'
    out = _script('train.py', *common, '--flow_dir=%s' % flow_dir, '--num_samples_train=4', '--max_epochs=1', '--save_freq=1',
                  '--summary_freq=1', '--checkpoint_dir=%s' % ck, cwd=base)
    assert 'Training completed successfully' in out and 'Validation IoU' in out, out[-2000:]
    saved = torch.load(str(ck / 'model.best.pt'))['params']
    assert not any(k.startswith('pwcnet/') for k in saved) and any(k.startswith('MaskNet/') for k in saved)
    out = _script('test_generator.py', *common, '--flow_dir=%s' % flow_dir, '--ckpt_file=%s' % (ck / 'model.best.pt'), cwd=base)
    assert 'Success: Processed' in out, out[-2000:]


def test_ensemble_on_supplied_flow_writes_its_buffers(davis):
    base, root, flow_dir, common = davis
    save = base / 'ens'
    out = _script('test_generator_ensemble.py', *common, '--flow_dir=%s' % flow_dir, '--ckpt_file=synthetic', '--generate_visualization',
                  '--test_save_dir=%s' % save, cwd=base)
    assert 'Success: Processed 6 frames' in out, out[-2000:]
    import scipy.io as sio
    m = sio.loadmat(str(save / 'cows' / 'result_1.mat'))
    assert all('%s_%03d' % (k, int(c * 100)) in m for k in ('img_1', 'pred_mask', 'gt_mask') for c in CROPS)
